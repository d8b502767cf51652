// itrquant_kernels.cuh -- inverse path of the TU loop and the fused TU round trip (SURVEY 8f rank 1).
//
//   inv_trquant_kernel   : TrQuant::invTransformNxN (CommonLib/TrQuant.cpp:318-348) = Quant::dequant (CommonLib/Quant.cpp:520-609,
//                          DeQuantCore :232-262) + TrQuant::xIT (:567-660; _fastInverseMM CommonLib/TrQuant_EMT.cpp:64-194, the B2..B8
//                          butterflies :231-636 equal the matrix product; AVX2 fastInvCore/roundClip CommonLib/x86/TrafoX86.h).
//                          Its RT instantiation ends the round trip with the slice's quantiser (vvb_tu_roundtrip_rdo*): the inverse of the
//                          quantiser's levels, then the same reconstruction and distortions as tu_roundtrip_kernel (rt_account, rt_zero_residual, rt_reduce).
//   tu_roundtrip_kernel  : the luma TU candidate body of IntraSearch::xIntraCodingTUBlock (EncoderLib/IntraSearch.cpp:1328-1429) and of
//                          InterSearch::xEstimateInterResidualQT (EncoderLib/InterSearch.cpp:3659-3714): residual = org - pred,
//                          transformNxN, (absSum > 0 ? invTransformNxN : zero residual), PelBuf::reconstruct (CommonLib/Buffer.cpp:719),
//                          SSE(org, reco) / SSE(orgResi, recResi) / SSE(0, orgResi) -- one kernel, the levels never leave shared memory.
//
// Exactness: dequantised coefficients and first-pass outputs are clipped to 16 bit by the reference itself (transformMinimum/Maximum,
// clipMinimum/Maximum = -2^15 .. 2^15-1), so both inverse passes run on IDP.2A (two int16 x int8 MACs) with int32 sums exactly as the
// scalar code; sums cannot overflow (64 * 32768 * 90 < 2^31).
#pragma once
#include "trquant_kernels.cuh"

namespace vvb {

// Inverse matrices: dst[q*N + j] (word) = bytes T[4q][j], T[4q+1][j], T[4q+2][j], T[4q+3][j]   for q < Q  (k runs over coefficients; rows >= keep are 0)
__device__ __forceinline__ void stage_matrix_inv( uint32_t* dst, const int8_t* __restrict__ table, int off, int N, int keep, int Q, int tid, int nthr )
{
  for( int i = tid; i < Q * N; i += nthr )
  {
    const int q = i / N, j = i - q * N;
    uint32_t v = 0;
    if( 4 * q < keep )
    {
      const int8_t* t = table + off + ( 4 * q ) * N + j;
      v = (uint32_t)(uint8_t) t[0] | ( (uint32_t)(uint8_t) t[N] << 8 ) | ( (uint32_t)(uint8_t) t[2 * N] << 16 ) | ( (uint32_t)(uint8_t) t[3 * N] << 24 );
    }
    dst[i] = v;
  }
}

__device__ __forceinline__ int clip16( int v ) { return max( -32768, min( 32767, v ) ); }

// Compile-time layout of the inverse scratch of one shape: cT [RW][RH/2 + 2] words (dequantised coefficients, transposed, k-pairs packed) and
// tT [H][RW/2] words (first-pass output, transposed, column pairs packed); MvI [RH/4][H], MhI [RW/4][W] inverse matrices.
template<int LW, int LH> struct InvShape
{
  using S = TuShape<LW, LH>;
  static constexpr int PITCH_C = S::RH / 2 + 2, PITCH_T = S::RW / 2;
  static constexpr int CT_WORDS = S::RW * PITCH_C, TT_WORDS = S::H * PITCH_T, WORDS = CT_WORDS + TT_WORDS;
  static constexpr int MAT_WORDS = ( S::RH / 4 ) * S::H + ( S::RW / 4 ) * S::W;
};

// Dequantise + inverse-transform one TU by one team.  qS: int16 levels [H][W] in shared memory; cT / tT: scratch (InvShape).
// out( y, x0, r0, r1, r2, r3 ) receives the residual of row y, columns x0..x0+3.  Contains __syncthreads(): all threads of the CTA call it;
// `active` masks the work (a team whose TU quantised to zero, or a tail team, only walks the barriers).
// LFN: the instantiation that carries the inverse LFNST (TrQuant::xInvLfnst); scanTab is only read there
template<int LW, int LH, bool LFN = false, class OUT>
__device__ __forceinline__ void team_inverse( const TuPar& par, const uint32_t* MvI, const uint32_t* MhI, const int16_t* qS, uint32_t* cT, uint32_t* tT,
                                              int tt, bool active, OUT out, const int32_t* __restrict__ scanTab )
{
  using S = TuShape<LW, LH>; using I = InvShape<LW, LH>;
  constexpr int W = S::W, H = S::H, T = S::T, RW = S::RW, RH = S::RH;
  const int lKW = LW == 5 ? par.lKeepW : S::LRW, lKH = LH == 5 ? par.lKeepH : S::LRH;
  const int keepW = 1 << lKW, keepH = 1 << lKH;
  if( par.ts )                                              // uniform over the launch: Quant::dequant without the transform shift + TrQuant::xITransformSkip (TrQuant.cpp:659-675)
  {
    const int sc = par.dqScale, sh = par.dqShift, inMax = par.dqInMax, inMin = -inMax - 1;
    const int add = sh > 0 ? 1 << ( sh - 1 ) : 0;
    for( int it = tt; active && it < H * W / 4; it += T )
    {
      const int y = it >> ( LW - 2 ), x0 = ( it & ( W / 4 - 1 ) ) << 2;
      int r[4];
#pragma unroll
      for( int k = 0; k < 4; k++ )
      {
        int c = max( inMin, min( inMax, (int) qS[y * W + x0 + k] ) );
        c = sh > 0 ? ( c * sc + add ) >> sh : (int)( (unsigned)( c * sc ) << ( -sh ) );
        r[k] = clip16( c );
      }
      out( y, x0, r[0], r[1], r[2], r[3] );
    }
    return;
  }
  // ---- dequant (DeQuantCore, Quant.cpp:232-262) + transpose: cT[i][k/2] = ( coef[k][i], coef[k+1][i] )
  {
    const int pairs = keepW << ( lKH - 1 );
    const int sc = par.dqScale, sh = par.dqShift, inMax = par.dqInMax, inMin = -inMax - 1;
    const int add = sh > 0 ? 1 << ( sh - 1 ) : 0;
#pragma unroll
    for( int k = 0; k < S::cdiv( RW * RH / 2, T ); k++ )
    {
      const int it = tt + k * T;
      if( active && it < pairs )
      {
        const int kp = it >> lKW, i = it & ( keepW - 1 );
        int c0 = max( inMin, min( inMax, (int) qS[( 2 * kp ) * W + i] ) );
        int c1 = max( inMin, min( inMax, (int) qS[( 2 * kp + 1 ) * W + i] ) );
        if( sh > 0 ) { c0 = ( c0 * sc + add ) >> sh; c1 = ( c1 * sc + add ) >> sh; }
        else         { c0 = (int)( (unsigned)( c0 * sc ) << ( -sh ) ); c1 = (int)( (unsigned)( c1 * sc ) << ( -sh ) ); }
        c0 = clip16( c0 ); c1 = clip16( c1 );
        if( LFN && par.lfnstIdx )
        {
          constexpr int K = ( LW >= 3 && LH >= 3 ) ? 8 : 4;      // xIT only reads the top-left K x K coefficients of an LFNST TU (TrQuant.cpp:590-602)
          if( i >= K || 2 * kp >= K ) { c0 = 0; c1 = 0; }
        }
        cT[i * I::PITCH_C + kp] = ( (uint32_t) c0 & 0xffffu ) | ( (uint32_t) c1 << 16 );
      }
    }
  }
  __syncthreads();
  if( LFN && par.lfnstIdx )                                   // uniform over the launch: TrQuant::xInvLfnst (TrQuant.cpp:838-940), xInvLfnstNxNCore (:190-213)
  {
    constexpr int K = ( LW >= 3 && LH >= 3 ) ? 8 : 4, NOUT = K == 8 ? 48 : 16;
    constexpr int ZIN = ( ( W == 4 && H == 4 ) || ( W == 8 && H == 8 ) ) ? 8 : 16;
    int16_t* c16 = reinterpret_cast<int16_t*>( cT );
    // the secondary coefficients: the first 16 scan positions = the top-left 4x4 group in diagonal order (table of the 8x8 region: same first group)
    const int32_t* fwd8 = scanTab + VVB_SCAN_TABLE_ENTRIES + 6 * 1024;
    constexpr int PER = S::cdiv( NOUT, T );
    int outv[PER];
    if( active )
    {
      int src[ZIN];
#pragma unroll
      for( int i = 0; i < ZIN; i++ )
      {
        const int p = __ldg( fwd8 + i ), x = p & 7, y = p >> 3;
        src[i] = c16[( x * I::PITCH_C + ( y >> 1 ) ) * 2 + ( y & 1 )];
      }
#pragma unroll
      for( int k = 0; k < PER; k++ )
      {
        const int j = min( tt + k * T, NOUT - 1 );
        int sum = 0;
#pragma unroll
        for( int i = 0; i < ZIN; i++ ) sum += src[i] * (int) __ldg( par.lfnstMat + i * NOUT + j );     // the inverse kernel is the transpose of the forward one
        outv[k] = clip16( ( sum + 64 ) >> 7 );
      }
    }
    __syncthreads();
    if( active )
#pragma unroll
      for( int k = 0; k < PER; k++ )
      {
        const int j = tt + k * T;
        if( j >= NOUT ) break;
        int a, b;                                              // the walk of :893-936: rows of 8 then rows of 4 (sub-block 8), rows of 4 (sub-block 4); transposed: columns
        if( K == 4 ) { b = j >> 2; a = j & 3; }
        else if( j < 32 ) { b = j >> 3; a = j & 7; }
        else { b = 4 + ( ( j - 32 ) >> 2 ); a = ( j - 32 ) & 3; }
        const int x = par.lfnstTranspose ? b : a, y = par.lfnstTranspose ? a : b;
        c16[( x * I::PITCH_C + ( y >> 1 ) ) * 2 + ( y & 1 )] = (int16_t) outv[k];
      }
    __syncthreads();
  }
  // ---- pass 1 (vertical, shift 7): tmp[i][j] = clip16( ( sum_{k<keepH} coef[k][i] * Tv[k][j] + 64 ) >> 7 ), two columns i per item;
  //      stored transposed and packed: tT[j][i/2] = ( tmp[i][j], tmp[i+1][j] ).  Kept rows k >= keepH of MvI are zero and cT beyond keepH is
  //      never read past Q, so the loop runs over the kept coefficients only.
  {
    const int items = ( keepW >> 1 ) << ( LH - 2 ), Q = keepH >> 2;
#pragma unroll
    for( int k = 0; k < S::cdiv( ( RW / 2 ) * ( H / 4 ), T ); k++ )
    {
      const int it = tt + k * T;
      if( active && it < items )
      {
        const int ip = it >> ( LH - 2 ), j0 = ( it & ( H / 4 - 1 ) ) << 2;
        int a0 = 0, a1 = 0, a2 = 0, a3 = 0, b0 = 0, b1 = 0, b2 = 0, b3 = 0;
        const uint2* ca = reinterpret_cast<const uint2*>( cT + ( 2 * ip ) * I::PITCH_C );
        const uint2* cb = reinterpret_cast<const uint2*>( cT + ( 2 * ip + 1 ) * I::PITCH_C );
        const uint32_t* mcol = MvI + j0;
#pragma unroll
        for( int q = 0; q < RH / 4; q++ )
        {
          if( LH != 5 || q < Q )
          {
            const uint2 va = ca[q], vb = cb[q];
            const uint4 m = *reinterpret_cast<const uint4*>( mcol + q * H );
            a0 = __dp2a_lo( (int) va.x, (int) m.x, a0 ); a0 = __dp2a_hi( (int) va.y, (int) m.x, a0 );
            a1 = __dp2a_lo( (int) va.x, (int) m.y, a1 ); a1 = __dp2a_hi( (int) va.y, (int) m.y, a1 );
            a2 = __dp2a_lo( (int) va.x, (int) m.z, a2 ); a2 = __dp2a_hi( (int) va.y, (int) m.z, a2 );
            a3 = __dp2a_lo( (int) va.x, (int) m.w, a3 ); a3 = __dp2a_hi( (int) va.y, (int) m.w, a3 );
            b0 = __dp2a_lo( (int) vb.x, (int) m.x, b0 ); b0 = __dp2a_hi( (int) vb.y, (int) m.x, b0 );
            b1 = __dp2a_lo( (int) vb.x, (int) m.y, b1 ); b1 = __dp2a_hi( (int) vb.y, (int) m.y, b1 );
            b2 = __dp2a_lo( (int) vb.x, (int) m.z, b2 ); b2 = __dp2a_hi( (int) vb.y, (int) m.z, b2 );
            b3 = __dp2a_lo( (int) vb.x, (int) m.w, b3 ); b3 = __dp2a_hi( (int) vb.y, (int) m.w, b3 );
          }
        }
#define VVB_P1( a, b ) ( ( (uint32_t) clip16( ( (a) + 64 ) >> 7 ) & 0xffffu ) | ( (uint32_t) clip16( ( (b) + 64 ) >> 7 ) << 16 ) )
        uint32_t* td = tT + j0 * I::PITCH_T + ip;
        td[0] = VVB_P1( a0, b0 ); td[I::PITCH_T] = VVB_P1( a1, b1 ); td[2 * I::PITCH_T] = VVB_P1( a2, b2 ); td[3 * I::PITCH_T] = VVB_P1( a3, b3 );
#undef VVB_P1
      }
    }
  }
  __syncthreads();
  // ---- pass 2 (horizontal, shift 20 - bitDepth): resi[y][x] = clip16( ( sum_{k<keepW} tmp[k][y] * Th[k][x] + rnd ) >> s2 )
  {
    const int s2 = par.s2Inv, r2 = 1 << ( s2 - 1 ), Q = keepW >> 2;
#pragma unroll
    for( int k = 0; k < S::cdiv( H * W / 4, T ); k++ )
    {
      const int it = tt + k * T;
      if( active )
      {
        const int y = it >> ( LW - 2 ), x0 = ( it & ( W / 4 - 1 ) ) << 2;
        int a0 = 0, a1 = 0, a2 = 0, a3 = 0;
        const uint2* tr = reinterpret_cast<const uint2*>( tT + y * I::PITCH_T );
        const uint32_t* mcol = MhI + x0;
#pragma unroll
        for( int q = 0; q < RW / 4; q++ )
        {
          if( LW != 5 || q < Q )
          {
            const uint2 tv = tr[q];
            const uint4 m = *reinterpret_cast<const uint4*>( mcol + q * W );
            a0 = __dp2a_lo( (int) tv.x, (int) m.x, a0 ); a0 = __dp2a_hi( (int) tv.y, (int) m.x, a0 );
            a1 = __dp2a_lo( (int) tv.x, (int) m.y, a1 ); a1 = __dp2a_hi( (int) tv.y, (int) m.y, a1 );
            a2 = __dp2a_lo( (int) tv.x, (int) m.z, a2 ); a2 = __dp2a_hi( (int) tv.y, (int) m.z, a2 );
            a3 = __dp2a_lo( (int) tv.x, (int) m.w, a3 ); a3 = __dp2a_hi( (int) tv.y, (int) m.w, a3 );
          }
        }
        out( y, x0, clip16( ( a0 + r2 ) >> s2 ), clip16( ( a1 + r2 ) >> s2 ), clip16( ( a2 + r2 ) >> s2 ), clip16( ( a3 + r2 ) >> s2 ) );
      }
    }
  }
}

// Dequantiser of dependent quantisation (DQIntern::Quantizer::dequantBlock, DepQuant.cpp:574-629): levels -> qIdx = 2 * level -+ (state >> 1), where `state` is the
// 4-state machine driven by the parities of the levels further up the scan, then ( qIdx * scale + add ) >> shift (or qIdx * ( scale << -shift )) in 64 bits, clipped
// to the 16-bit coefficient range.  One warp per TU: a lane folds the parities of its run of scan positions into a state -> state map (2 bits per state), the maps
// are combined across the warp in scan order (from the end of the scan down) with a shuffle scan, and each lane then walks its run with the state it starts from.
// qIdx reaches +-65535 for levels at the int16 extremes, so the block handed to the inverse kernel holds the clipped coefficients, which it reads with an identity
// dequantiser (scale 1, shift 0).
__device__ __forceinline__ unsigned dqd_compose( unsigned a, unsigned b )      // first a, then b
{
  unsigned r = 0;
#pragma unroll
  for( int s = 0; s < 4; s++ ) r |= ( ( b >> ( 2 * ( ( a >> ( 2 * s ) ) & 3u ) ) ) & 3u ) << ( 2 * s );
  return r;
}
__global__ void __launch_bounds__( 128 ) dq_dequant_levels_kernel( const int16_t* __restrict__ q, const int32_t* __restrict__ fwd, int w, int h, int lrw, int nScan, int n,
                                                                   int scale, int shift, int16_t* __restrict__ out )
{
  const int tu = blockIdx.x * 4 + ( threadIdx.x >> 5 ), lane = threadIdx.x & 31;
  if( tu >= n ) return;
  const int area = w * h, rw = 1 << lrw, rh = nScan >> lrw;
  const int16_t* qt = q + (size_t) tu * area;
  int16_t* ot = out + (size_t) tu * area;
  if( rw < w || rh < h )                                       // 64-sized TUs: nothing outside the scanned 32 x 32 region carries a level
    for( int i = lane; i < area; i += 32 ) { const int y = i / w, x = i - y * w; if( x >= rw || y >= rh ) ot[i] = 0; }
  const int run = nScan >= 32 ? nScan >> 5 : 1;                // scan positions per lane; lane 0 holds the END of the scan
  const int hi = nScan - 1 - lane * run;                       // first (highest) position of the lane's run
  const bool act = hi >= 0;
  unsigned m = 0xE4u;                                          // identity map
  for( int k = 0; act && k < run; k++ )
  {
    const int p = __ldg( fwd + hi - k );
    const int level = qt[( p >> lrw ) * w + ( p & ( rw - 1 ) )];
    m = dqd_compose( m, ( level & 1 ) ? 0x72u : 0xD8u );       // parity 1: 0->2 1->0 2->3 3->1 ; parity 0: 0->0 1->2 2->1 3->3  (the table 32040)
  }
  // exclusive scan of the maps over the lanes (lane 0 first)
  unsigned inc = m;
#pragma unroll
  for( int d = 1; d < 32; d <<= 1 )
  {
    const unsigned prev = __shfl_up_sync( 0xffffffffu, inc, d );
    if( lane >= d ) inc = dqd_compose( prev, inc );
  }
  unsigned exc = __shfl_up_sync( 0xffffffffu, inc, 1 );
  if( lane == 0 ) exc = 0xE4u;
  int state = (int)( exc & 3u );                               // the walk starts in state 0 at the end of the scan
  for( int k = 0; act && k < run; k++ )
  {
    const int p = __ldg( fwd + hi - k );
    const int idx = ( p >> lrw ) * w + ( p & ( rw - 1 ) );
    const int level = qt[idx];
    const long long qIdx = level ? 2 * level + ( level > 0 ? -( state >> 1 ) : ( state >> 1 ) ) : 0;
    const long long c = shift > 0 ? ( qIdx * scale + ( 1ll << ( shift - 1 ) ) ) >> shift : qIdx * ( (long long) scale << -shift );
    ot[idx] = (int16_t) max( -32768ll, min( 32767ll, c ) );
    state = ( 32040 >> ( ( state << 2 ) + ( ( level & 1 ) << 1 ) ) ) & 3;
  }
}

// ---------------------------------------------------------------------------------------------------------------------------------
// Epilogue of a TU round trip, shared by tu_roundtrip_kernel and the RT instantiation of inv_trquant_kernel.  The pieces work on the calling kernel's own
// locals (bases, strides, accumulators) and each kernel forms the bases itself, as the forward kernels do: gathering that state in a structure, or forming the
// bases in a helper that returns them through references, makes ptxas allocate tu_roundtrip_kernel differently, with spills in some instantiations.
// org / pred are either compact candidate pools [n][H][W] (planes == 0) or positions inside resident planes (vvb_block: x, y, start_x/start_y = displacement
// of the prediction).
struct TuResult { unsigned long long distReco, distResi, distZero; int absSum, lastPos; };     // == vvb_tu_result (32 bytes)

// residual r0..r3 of row y, columns x0..x0+3: PelBuf::reconstruct (clip to [0, pelMax]) into rBase (nullable) and the three SSEs of vvb_tu_result in 64 bits
template<int W>
__device__ __forceinline__ void rt_account( const int16_t* oBase, int so, const int16_t* pBase, int sp, bool al8, int pelMax, int16_t* rBase,
                                            unsigned long long& dReco, unsigned long long& dResi, unsigned long long& dZero, int y, int x0, int r0, int r1, int r2, int r3 )
{
  const int16_t* o = oBase + (ptrdiff_t) y * so + x0; const int16_t* p = pBase + (ptrdiff_t) y * sp + x0;
  const int r[4] = { r0, r1, r2, r3 };
  int rc[4], ovs[4], pvs[4];
  if( al8 )
  {
    const uint2 ow = __ldg( reinterpret_cast<const uint2*>( o ) ), pw = __ldg( reinterpret_cast<const uint2*>( p ) );
    ovs[0] = lo16( ow.x ); ovs[1] = hi16( ow.x ); ovs[2] = lo16( ow.y ); ovs[3] = hi16( ow.y );
    pvs[0] = lo16( pw.x ); pvs[1] = hi16( pw.x ); pvs[2] = lo16( pw.y ); pvs[3] = hi16( pw.y );
  }
  else
  {
#pragma unroll
    for( int c = 0; c < 4; c++ ) { ovs[c] = __ldg( o + c ); pvs[c] = __ldg( p + c ); }
  }
  unsigned sz = 0, sc = 0;
#pragma unroll
  for( int c = 0; c < 4; c++ )
  {
    const int ov = ovs[c], pv = pvs[c];
    rc[c] = max( 0, min( pelMax, pv + r[c] ) );
    const int dz = ov - pv;                 // original residual
    const long long dr = (long long) dz - r[c];
    const int dc = ov - rc[c];
    sz += (unsigned)( dz * dz ); sc += (unsigned)( dc * dc );          // 4 * (2^12)^2 < 2^32
    dResi += (unsigned long long)( dr * dr );
  }
  dZero += sz; dReco += sc;
  if( rBase )
  {
    uint2 ov2;
    ov2.x = ( (uint32_t) rc[0] & 0xffffu ) | ( (uint32_t) rc[1] << 16 );
    ov2.y = ( (uint32_t) rc[2] & 0xffffu ) | ( (uint32_t) rc[3] << 16 );
    *reinterpret_cast<uint2*>( rBase + y * W + x0 ) = ov2;
  }
}

// the residual of a live TU that quantised to zero (IntraSearch.cpp:1366-1369 piResi.fill(0)) through account( y, x0, 0, 0, 0, 0 )
template<int LW, int LH, class ACCOUNT>
__device__ __forceinline__ void rt_zero_residual( ACCOUNT account, int tt )
{
  using S = TuShape<LW, LH>;
#pragma unroll
  for( int k = 0; k < S::cdiv( S::H * S::W / 4, S::T ); k++ ) { const int it = tt + k * S::T; account( it >> ( LW - 2 ), ( it & ( S::W / 4 - 1 ) ) << 2, 0, 0, 0, 0 ); }
}

// team reduction of the three sums: shuffles inside the warp (teams of 4..16 lanes are aligned lane groups), then one shared atomic per warp and value into
// acc[0..2] for teams wider than a warp.  Contains __syncthreads() for teams wider than a warp: all threads of the CTA call it
template<int T>
__device__ __forceinline__ void rt_reduce( unsigned long long& dReco, unsigned long long& dResi, unsigned long long& dZero, unsigned long long* acc, int tt, bool live )
{
  constexpr int span = T < 32 ? T : 32;
#pragma unroll
  for( int off = span >> 1; off > 0; off >>= 1 )
  {
    dReco += __shfl_xor_sync( 0xffffffffu, dReco, off );
    dResi += __shfl_xor_sync( 0xffffffffu, dResi, off );
    dZero += __shfl_xor_sync( 0xffffffffu, dZero, off );
  }
  if( T > 32 )
  {
    if( tt == 0 ) { acc[0] = 0; acc[1] = 0; acc[2] = 0; }
    __syncthreads();
    if( live && ( tt & 31 ) == 0 ) { atomicAdd( &acc[0], dReco ); atomicAdd( &acc[1], dResi ); atomicAdd( &acc[2], dZero ); }
    __syncthreads();
    dReco = acc[0]; dResi = acc[1]; dZero = acc[2];
  }
}

// the inputs and outputs of the RT instantiation of inv_trquant_kernel: org / pred as for tu_roundtrip_kernel, the quantiser's abs_sum and last_pos per TU
struct RtIo
{
  int planes; Plane orgPlane, predPlane; const vvb_block* blocks; const int16_t* orgPool; const int16_t* predPool;
  int16_t* reco; TuResult* res; const int32_t* absSum; const int32_t* lastPos;
};

// RT adds four 64-bit accumulators per team (rt_reduce)
template<int LW, int LH, bool RT = false> static inline size_t inv_trquant_smem()
{
  using S = TuShape<LW, LH>; using I = InvShape<LW, LH>;
  return (size_t)( I::MAT_WORDS + S::NTEAMS * ( S::RESI_WORDS + I::WORDS ) + ( RT ? S::NTEAMS * 8 : 0 ) ) * 4;
}

// RT = false: levels -> residual (resiOut).  RT = true: the second half of a TU round trip whose levels (or, for dependent quantisation, dequantised
// coefficients read with an identity dequantiser) another kernel produced: TUs with io.absSum > 0 are inverted, the others get the zero residual, then
// the reconstruction and the distortions (rt_account, rt_zero_residual, rt_reduce) with the quantiser's abs_sum / last_pos (resiOut unused).  The RT instantiations ask for four resident
// CTAs per SM: left to its own register target, ptxas spilled a value in some of them
template<int LW, int LH, bool LFN, bool RT>
__global__ void __launch_bounds__( 128, RT ? 4 : 0 ) inv_trquant_kernel( const __grid_constant__ TuPar par, const int8_t* __restrict__ trTable, const int32_t* __restrict__ scanTab,
                                                             const int16_t* __restrict__ q, int n, int16_t* __restrict__ resiOut, const __grid_constant__ RtIo io )
{
  using S = TuShape<LW, LH>; using I = InvShape<LW, LH>;
  extern __shared__ __align__( 16 ) uint32_t smem[];
  constexpr int T = S::T, NTEAMS = S::NTEAMS, W = S::W, H = S::H;
  const int team = threadIdx.x / T, tt = threadIdx.x % T;
  uint32_t* MvI = smem;
  uint32_t* MhI = MvI + ( S::RH / 4 ) * H;
  uint32_t* teamBase = smem + I::MAT_WORDS;
  stage_matrix_inv( MvI, trTable, par.offV, H, par.keepH, S::RH / 4, threadIdx.x, blockDim.x );
  stage_matrix_inv( MhI, trTable, par.offH, W, par.keepW, S::RW / 4, threadIdx.x, blockDim.x );
  uint32_t* myQ = teamBase + team * ( S::RESI_WORDS + I::WORDS );
  uint32_t* cT  = myQ + S::RESI_WORDS;
  uint32_t* tT  = cT + I::CT_WORDS;
  unsigned long long* acc = reinterpret_cast<unsigned long long*>( teamBase + NTEAMS * ( S::RESI_WORDS + I::WORDS ) ) + team * 4;     // RT: [0] reco, [1] resi, [2] zero

  for( int base = blockIdx.x * NTEAMS; base < n; base += gridDim.x * NTEAMS )
  {
    const int tu = base + team;
    const bool live = tu < n;
    const int absSum = RT && live ? io.absSum[tu] : 0;
    const bool active = RT ? live && absSum > 0 : live;
    __syncthreads();
    {
      const uint32_t* src = reinterpret_cast<const uint32_t*>( q + (size_t)( live ? tu : 0 ) * W * H );
#pragma unroll
      for( int k = 0; k < S::RESI_WORDS / T; k++ ) if( active ) myQ[tt + k * T] = __ldg( src + tt + k * T );
    }
    __syncthreads();
    if constexpr( RT )
    {
      const int16_t* oBase; const int16_t* pBase; int so, sp;
      if( io.planes )
      {
        const vvb_block blk = io.blocks[live ? tu : 0];
        oBase = io.orgPlane.origin + (ptrdiff_t) blk.y * io.orgPlane.stride + blk.x;                 so = io.orgPlane.stride;
        pBase = io.predPlane.origin + (ptrdiff_t)( blk.y + blk.start_y ) * io.predPlane.stride + blk.x + blk.start_x;  sp = io.predPlane.stride;
      }
      else
      {
        oBase = io.orgPool + (size_t)( live ? tu : 0 ) * W * H;   so = W;
        pBase = io.predPool + (size_t)( live ? tu : 0 ) * W * H;  sp = W;
      }
      const bool al8 = ( ( ( reinterpret_cast<uintptr_t>( oBase ) | reinterpret_cast<uintptr_t>( pBase ) ) & 7 ) | ( ( so | sp ) & 3 ) ) == 0;   // 4-pel loads allowed
      unsigned long long dReco = 0, dResi = 0, dZero = 0;
      const int pelMax = par.pelMax;
      int16_t* rBase = io.reco ? io.reco + (size_t)( live ? tu : 0 ) * W * H : nullptr;
      auto account = [&]( int y, int x0, int r0, int r1, int r2, int r3 )
      {
        rt_account<W>( oBase, so, pBase, sp, al8, pelMax, rBase, dReco, dResi, dZero, y, x0, r0, r1, r2, r3 );
      };
      team_inverse<LW, LH, LFN>( par, MvI, MhI, reinterpret_cast<const int16_t*>( myQ ), cT, tT, tt, active, account, scanTab );
      if( live && !active ) rt_zero_residual<LW, LH>( account, tt );
      rt_reduce<T>( dReco, dResi, dZero, acc, tt, live );
      if( live && tt == 0 )
      {
        TuResult r;
        r.distReco = dReco; r.distResi = dResi; r.distZero = dZero;
        r.absSum = absSum; r.lastPos = io.lastPos[tu];
        io.res[tu] = r;
      }
    }
    else
    {
      int16_t* dst = resiOut + (size_t)( live ? tu : 0 ) * W * H;
      team_inverse<LW, LH, LFN>( par, MvI, MhI, reinterpret_cast<const int16_t*>( myQ ), cT, tT, tt, live,
                            [&]( int y, int x0, int r0, int r1, int r2, int r3 )
                            {
                              uint2 o;
                              o.x = ( (uint32_t) r0 & 0xffffu ) | ( (uint32_t) r1 << 16 );
                              o.y = ( (uint32_t) r2 & 0xffffu ) | ( (uint32_t) r3 << 16 );
                              *reinterpret_cast<uint2*>( dst + y * W + x0 ) = o;
                            }, scanTab );
    }
  }
}

// ---------------------------------------------------------------------------------------------------------------------------------
// Fused TU round trip with the plain quantiser: forward, quantiser, inverse and the epilogue (rt_account, rt_zero_residual, rt_reduce) in one kernel.

// smem: forward matrices + inverse matrices + per team ( forward view ; the inverse scratch aliases v.tmp / v.coef ) + 4 accumulators per team
template<int LW, int LH> static inline size_t tu_roundtrip_smem()
{
  using S = TuShape<LW, LH>; using I = InvShape<LW, LH>;
  static_assert( I::WORDS <= S::TMP_WORDS + S::COEF_WORDS, "inverse scratch must fit the forward tmp + coef areas" );
  return (size_t)( S::MAT_WORDS + I::MAT_WORDS + S::NTEAMS * ( S::TEAM_WORDS + 8 ) ) * 4;
}

template<int LW, int LH, bool EXT>
__global__ void __launch_bounds__( 128 ) tu_roundtrip_kernel( const __grid_constant__ TuPar par, const int8_t* __restrict__ trTable, const int32_t* __restrict__ scanTab,
                                                              const int planes, const __grid_constant__ Plane orgPlane, const __grid_constant__ Plane predPlane,
                                                              const vvb_block* __restrict__ blocks, const int16_t* __restrict__ orgPool, const int16_t* __restrict__ predPool, int n,
                                                              int16_t* __restrict__ qOut, int16_t* __restrict__ recoOut, TuResult* __restrict__ resOut, uint8_t* __restrict__ needRdoqOut )
{
  using S = TuShape<LW, LH>; using I = InvShape<LW, LH>;
  extern __shared__ __align__( 16 ) uint32_t smem[];
  constexpr int T = S::T, NTEAMS = S::NTEAMS, W = S::W, H = S::H;
  const int team = threadIdx.x / T, tt = threadIdx.x % T;
  uint32_t* MtH = smem;
  uint32_t* MtV = MtH + ( W / 4 ) * S::RW;
  uint32_t* MvI = smem + S::MAT_WORDS;
  uint32_t* MhI = MvI + ( S::RH / 4 ) * H;
  uint32_t* teamBase = MvI + I::MAT_WORDS;
  stage_matrix( MtH, trTable, par.offH, W, par.keepW, S::RW, threadIdx.x, blockDim.x );
  stage_matrix( MtV, trTable, par.offV, H, par.keepH, S::RH, threadIdx.x, blockDim.x );
  stage_matrix_inv( MvI, trTable, par.offV, H, par.keepH, S::RH / 4, threadIdx.x, blockDim.x );
  stage_matrix_inv( MhI, trTable, par.offH, W, par.keepW, S::RW / 4, threadIdx.x, blockDim.x );
  const TeamView v = team_view<S>( teamBase, team );
  unsigned long long* acc = reinterpret_cast<unsigned long long*>( teamBase + NTEAMS * S::TEAM_WORDS ) + team * 4;     // [0] reco, [1] resi, [2] zero

  for( int base = blockIdx.x * NTEAMS; base < n; base += gridDim.x * NTEAMS )
  {
    const int tu = base + team;
    const bool live = tu < n;
    const int16_t* oBase; const int16_t* pBase; int so, sp;
    if( planes )
    {
      const vvb_block blk = blocks[live ? tu : 0];
      oBase = orgPlane.origin + (ptrdiff_t) blk.y * orgPlane.stride + blk.x;                 so = orgPlane.stride;
      pBase = predPlane.origin + (ptrdiff_t)( blk.y + blk.start_y ) * predPlane.stride + blk.x + blk.start_x;  sp = predPlane.stride;
    }
    else
    {
      oBase = orgPool + (size_t)( live ? tu : 0 ) * W * H;   so = W;
      pBase = predPool + (size_t)( live ? tu : 0 ) * W * H;  sp = W;
    }
    const bool al8 = ( ( ( reinterpret_cast<uintptr_t>( oBase ) | reinterpret_cast<uintptr_t>( pBase ) ) & 7 ) | ( ( so | sp ) & 3 ) ) == 0;   // 4-pel loads allowed
    const int pos = team_forward<LW, LH, EXT>( par, MtH, MtV, v, scanTab, tt, live, org_pred_words<LW>( oBase, so, pBase, sp ) );
    const int absSum = v.red[4], lastQ1 = v.red[5];
    if( live )
    {
      uint32_t* dst = reinterpret_cast<uint32_t*>( qOut + (size_t) tu * W * H );
#pragma unroll
      for( int k = 0; k < S::RESI_WORDS / T; k++ ) dst[tt + k * T] = v.resi[tt + k * T];
    }
    // every thread has read absSum before any thread can pass the first barrier of team_inverse; red[] is only reset in the next team_forward
    const bool active = live && absSum > 0;
    unsigned long long dReco = 0, dResi = 0, dZero = 0;
    const int pelMax = par.pelMax;
    int16_t* rBase = recoOut ? recoOut + (size_t)( live ? tu : 0 ) * W * H : nullptr;
    auto account = [&]( int y, int x0, int r0, int r1, int r2, int r3 )
    {
      rt_account<W>( oBase, so, pBase, sp, al8, pelMax, rBase, dReco, dResi, dZero, y, x0, r0, r1, r2, r3 );
    };
    // inverse scratch aliases the forward tmp / coef areas (both dead once the levels are in v.resi)
    team_inverse<LW, LH, EXT>( par, MvI, MhI, reinterpret_cast<const int16_t*>( v.resi ), v.tmp, v.tmp + I::CT_WORDS, tt, active, account, scanTab );
    if( live && !active ) rt_zero_residual<LW, LH>( account, tt );
    rt_reduce<T>( dReco, dResi, dZero, acc, tt, live );
    if( live && tt == 0 )
    {
      TuResult r;
      r.distReco = dReco; r.distResi = dResi; r.distZero = dZero;
      r.absSum = absSum; r.lastPos = absSum ? lastQ1 - 1 : pos;
      resOut[tu] = r;
      if( needRdoqOut ) needRdoqOut[tu] = (uint8_t) v.red[6];
    }
  }
}

} // namespace vvb
