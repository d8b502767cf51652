// trquant_kernels.cuh -- forward 2-D integer transform (DCT-II / DST-VII / DCT-VIII) + plain quantiser, fused.
//
// Replaces TrQuant::xT (CommonLib/TrQuant.cpp:481-564; 1-D cores CommonLib/TrQuant_EMT.cpp:366-421,1973-2000,
// AVX2 CommonLib/x86/TrafoX86.h:310-640) followed by Quant::quant -> QuantCore (CommonLib/Quant.cpp:735-833,132-230)
// and Quant::xNeedRDOQ -> needRdoqCore (:835-891,264-278) for luma TUs without LFNST / transform skip / scaling lists.
//
// Exactness: all sums are int32 exactly as the scalar reference.  Products run on IDP.2A (two int16 x int8 MACs per
// instruction): stage 1 always (residuals are int16), stage 2 when every stage-1 output fits int16 (always true for
// real video -- it is also the domain in which the AVX2 path, which saturates at TrafoX86.h:364, equals the scalar one);
// otherwise stage 2 falls back to plain 32-bit IMAD so that the result still equals the scalar reference.
//
// One *team* of T threads (4..128) owns one TU; a 128-thread CTA runs 128/T teams in lock step.
#pragma once
#include "common.cuh"

namespace vvb {

struct TuPar
{
  int w, h, lw, lh;
  int trHor, trVer;
  int keepW, keepH;          // non-zeroed-out outputs (TrQuant.cpp:496-497)
  int s1, s2;                // shifts (TrQuant.cpp:544-545)
  int offH, offV;            // offsets of the two matrices inside the int8 table (row j, column k)
  int scale, qbits;          // g_quantScales entry, iQBits (Quant.cpp:767-769)
  long long add, addRdoq;    // (171|85) << (qbits-9) ; 171 << (qbitsRdoq-9)
  int scaleRdoq, qbitsRdoq;
  int useThres;              // thres / (scale << 2)   (Quant.cpp:173-180, thrVal = 8)
  int scanOff;               // offset (entries) of this shape's raster->scanpos table
  int dqScale, dqShift;      // g_invQuantScales entry, rightShift of Quant::dequant (may be <= 0)   (Quant.cpp:554-561,601)
  int dqDepScale, dqDepShift;   // the same for DepQuant::dequant, which runs at QP + 1 (DepQuant.cpp:1492-1514, dequantBlock :574-629); host side only
  int dqInMax;               // input clipping bound (Quant.cpp:606-607)
  int s2Inv;                 // second inverse shift 20 - bitDepth (TrQuant.cpp:609); the first is 7
  int pelMax;                // (1 << bitDepth) - 1, reconstruction clipping (Buffer.cpp:719)
  int lKeepW, lKeepH;        // log2 of keepW, keepH (powers of two: every index split is a shift)
  int q32;                   // qbits <= 30: (|c| * scale + add) fits 32 bit for |c| < 2^16 (always true for residuals inside the bit depth)
  unsigned add32;            // low 32 bits of add (valid when q32)
  int lfnstIdx, lfnstTranspose;   // cu.lfnstIdx (0 = off) and xGetTransposeFlag of the intra mode; the kernel matrix [outputs][inputs] (int8) of (set, index):
  const int8_t* lfnstMat;
  int lfnstMaxScan;          // last scan position the quantiser may look at: 7 (4x4 / 8x8 TUs) or 15 with LFNST (Quant.cpp:151-158), INT_MAX without
  int signHiding;            // slice->signDataHidingEnabled: Quant::quant runs xSignBitHidingHDQ after QuantCore (Quant.cpp:817-826)
  int ts;                    // transform skip: coefficients = residual (xTransformSkip), residual = dequantised coefficient (xITransformSkip)
  unsigned rdoqThr;          // smallest |c| with ((|c| * scaleRdoq + addRdoq) >> qbitsRdoq) != 0  (needRdoqCore as one compare)
};

// Compile-time geometry of one TU shape (W = 2^LW, H = 2^LH).  The kernels are instantiated per shape so that every loop has a constant trip
// count and every index split is a shift; only the number of kept outputs of a 32-wide / 32-high MTS dimension (16 instead of 32) stays a run-time value.
template<int LW, int LH> struct TuShape
{
  static constexpr int W = 1 << LW, H = 1 << LH;
  static constexpr int T  = ( W * H / 4 > 128 ) ? 128 : ( W * H / 4 < 4 ? 4 : W * H / 4 );   // threads per TU
  static constexpr int RW = W > 32 ? 32 : W, RH = H > 32 ? 32 : H;                            // scanned region = upper bound of the kept outputs
  static constexpr int LRW = LW > 5 ? 5 : LW, LRH = LH > 5 ? 5 : LH;
  static constexpr int RESI_WORDS = W * H / 2;         // int16 residual, later the int16 levels
  static constexpr int TMP_WORDS  = RW * H;            // int32 stage-1 output [keepW][H]
  static constexpr int COEF_WORDS = RW * RH;           // int32 coefficients of the scanned region
  static constexpr int TEAM_WORDS = RESI_WORDS + TMP_WORDS + COEF_WORDS + 8;
  static constexpr int MAT_WORDS  = ( W / 4 ) * RW + ( H / 4 ) * RH;                          // forward matrices MtH [W/4][RW], MtV [H/4][RH]
  static constexpr int NTEAMS = 128 / T;
  __host__ __device__ static constexpr int cdiv( int a, int b ) { return ( a + b - 1 ) / b; }
};

// Matrix staging: Mt[q][j] (32-bit word) = bytes T[j][4q..4q+3], row pitch `pitch` words; j fastest so that a thread's 4 consecutive j are one LDS.128
__device__ __forceinline__ void stage_matrix( uint32_t* dst, const int8_t* __restrict__ table, int off, int N, int keep, int pitch, int tid, int nthr )
{
  const int Q = N >> 2;
  for( int i = tid; i < Q * pitch; i += nthr )
  {
    const int q = i / pitch, j = i - q * pitch;
    dst[i] = j < keep ? *reinterpret_cast<const uint32_t*>( table + off + j * N + 4 * q ) : 0u;
  }
}

// Views into one team's shared memory.
struct TeamView
{
  uint32_t* resi;     // int16 residual [H][W] as words; holds the int16 levels after team_forward
  uint32_t* tmp;      // stage-1 output [keepW][H] (int32)
  int32_t*  coef;     // int32 coefficients of the scanned region [RH][RW]
  int*      red;      // [0] ovf, [1] lastNZ, [2] cgLo, [3] cgHi, [4] absSum, [5] lastQ+1, [6] rdoq
};

template<class S> __device__ __forceinline__ TeamView team_view( uint32_t* teamBase, int team )
{
  TeamView v;
  v.resi = teamBase + team * S::TEAM_WORDS;
  v.tmp  = v.resi + S::RESI_WORDS;
  v.coef = reinterpret_cast<int32_t*>( v.tmp + S::TMP_WORDS );
  v.red  = reinterpret_cast<int*>( v.coef + S::COEF_WORDS );
  return v;
}

// lanes of the calling thread's team inside its warp (teams of 4..16 threads are aligned lane groups; larger teams span whole warps)
template<int T> __device__ __forceinline__ unsigned team_lane_mask()
{
  if( T >= 32 ) return 0xffffffffu;
  const unsigned lane = threadIdx.x & 31u;
  return ( ( 1u << ( T & 31 ) ) - 1u ) << ( lane & ~(unsigned)( T - 1 ) );
}

#define VVB_SCAN_TABLE_ENTRIES ( 25 * 1024 )     // raster -> scan position tables of the 25 shapes; the scan position -> raster tables follow them

// Sign-bit hiding of one coefficient group by one thread: Quant::xSignBitHidingHDQ (CommonLib/Quant.cpp:377-518) for the group `cg` of a TU whose levels
// QuantCore has just produced.  Groups are independent of each other: the only state the reference carries from group to group is `lastCG` (1 exactly for
// the group that holds the last level) and lastScanPos, which can only move inside that group (a group is only touched when its first and last level are
// at least SBH_THRESHOLD = 4 apart, so one of them survives).  deltaU (Quant.cpp:221) is recomputed from the coefficient.  Returns the new last scan
// position + 1 when this is the top group and its last level was zeroed, 0 otherwise.
template<int LW, int LRW>
__device__ __noinline__ int sbh_group( const TuPar& par, const int32_t* coef, int16_t* q16, const int32_t* __restrict__ fwd, int cg, int lastScanPos )
{
  constexpr int RWM = ( 1 << LRW ) - 1;
  const int subPos = cg << 4;
  const bool top = cg == ( lastScanPos >> 4 );
  int pos[16]; int lev[16];
#pragma unroll
  for( int n = 0; n < 16; n++ ) { const int p = __ldg( fwd + subPos + n ); pos[n] = p; lev[n] = q16[( ( p >> LRW ) << LW ) + ( p & RWM )]; }
  int firstNZ = 16, lastNZ = -1, absSum = 0;
#pragma unroll
  for( int n = 15; n >= 0; n-- ) if( lev[n] && lastNZ < 0 ) lastNZ = n;
#pragma unroll
  for( int n = 0; n < 16; n++ ) if( lev[n] && firstNZ == 16 ) firstNZ = n;
#pragma unroll
  for( int n = 0; n < 16; n++ ) if( n >= firstNZ && n <= lastNZ ) absSum += lev[n];
  if( lastNZ - firstNZ < 4 ) return 0;                                        // SBH_THRESHOLD, CommonDef.h:272
  int firstLev = 0;
#pragma unroll
  for( int n = 0; n < 16; n++ ) if( n == firstNZ ) firstLev = lev[n];
  const unsigned signbit = firstLev > 0 ? 0u : 1u;
  if( signbit == ( (unsigned) absSum & 1u ) ) return 0;
  int curCost = 0x7fffffff, minCostInc = 0x7fffffff, minN = -1, finalChange = 0, curChange = 0;
  const int nStart = top ? lastNZ : 15;
#pragma unroll
  for( int n = 15; n >= 0; n-- )
  {
    if( n > nStart ) continue;
    const int c = coef[pos[n]];
    const long long t = (long long) abs( c ) * par.scale;
    const int mag = (int)( ( t + par.add ) >> par.qbits );
    const int dU = (int)( ( t - ( (long long) mag << par.qbits ) ) >> ( par.qbits - 8 ) );
    if( lev[n] != 0 )
    {
      if( dU > 0 ) { curCost = -dU; curChange = 1; }
      else if( n == firstNZ && abs( lev[n] ) == 1 ) curCost = 0x7fffffff;
      else { curCost = dU; curChange = -1; }
    }
    else if( n < firstNZ )
    {
      const unsigned thisSign = c >= 0 ? 0u : 1u;
      if( thisSign != signbit ) curCost = 0x7fffffff;
      else { curCost = -dU; curChange = 1; }
    }
    else { curCost = -dU; curChange = 1; }
    if( curCost < minCostInc ) { minCostInc = curCost; finalChange = curChange; minN = n; }
  }
  int minLev = 0, minPos = 0;
#pragma unroll
  for( int n = 0; n < 16; n++ ) if( n == minN ) { minLev = lev[n]; minPos = pos[n]; }
  if( minLev == 32767 || minLev == -32768 ) finalChange = -1;
  minLev = coef[minPos] >= 0 ? minLev + finalChange : minLev - finalChange;
  q16[( ( minPos >> LRW ) << LW ) + ( minPos & RWM )] = (int16_t) minLev;
  if( top && subPos + minN == lastScanPos && minLev == 0 )
  {
    int nl = -1;
#pragma unroll
    for( int n = 0; n < 16; n++ ) if( n < minN && lev[n] ) nl = n;           // the next level below inside the group (one exists: the first level survives)
    return subPos + nl + 1;
  }
  return 0;
}

// Plain quantiser of one TU by its team of T threads (Quant.cpp:132-230 QuantCore, :735-833 wrapper; needRdoqCore :264-278).
// coef: int32 [RH][RW] in shared memory; qWords: the level block int16 [H][W] (as words) in shared memory; inv: raster -> scan position.
// Every thread works on quads of 4 raster-consecutive coefficients (LDS.128 + one LDG.128 of scan positions); reductions are redux.sync inside
// the warp plus one shared atomic per warp for multi-warp teams.  Contains __syncthreads(); ends synchronised with red[4] = absSum,
// red[5] = last non-zero level's scan position + 1, red[6] = RDOQ flag; returns the final scan position (Quant.cpp:182-208).
// EXT: the instantiation that carries the LFNST position limit and the sign-bit hiding pass; the plain one (EXT = false) is the round-1 code path untouched
template<int LW, int LH, int T, bool EXT = true>
__device__ __forceinline__ int team_quantise( const TuPar& par, const int32_t* coef, uint32_t* qWords, int* red, const int32_t* __restrict__ inv, int tt, bool live )
{
  using S = TuShape<LW, LH>;
  constexpr int NQUADS = S::RW * S::RH / 4, ITERS = S::cdiv( NQUADS, T );
  constexpr bool CACHE = ITERS <= 4;                        // keep the quads and their scan positions in registers between the two passes
  const unsigned tmask = team_lane_mask<T>();
  constexpr bool multi = T > 32;
  const int4* c4 = reinterpret_cast<const int4*>( coef );
  const int4* s4 = reinterpret_cast<const int4*>( inv );
  const int useThres = par.useThres, maxScan = EXT ? par.lfnstMaxScan : 0x7fffffff; const unsigned rdoqThr = par.rdoqThr;
  // ---- pass 1: last non-zero scan position, coefficient groups holding a value above the threshold, RDOQ pre-check
  int lastNZ = 0; unsigned cgLo = 0, cgHi = 0, rd = 0;
  int4 cq[CACHE ? ITERS : 1], sq[CACHE ? ITERS : 1];
#pragma unroll
  for( int kk = 0; kk < ITERS; kk++ )
  {
    const int qi = tt + kk * T, k = CACHE ? kk : 0;
    cq[k] = make_int4( 0, 0, 0, 0 ); sq[k] = make_int4( 0, 0, 0, 0 );
    if( live && ( NQUADS % T == 0 || qi < NQUADS ) )
    {
      cq[k] = c4[qi];
      if( cq[k].x | cq[k].y | cq[k].z | cq[k].w )
      {
        sq[k] = __ldg( s4 + qi );
#define VVB_Q1( cv, sv ) if( cv ) { const int ac = abs( cv ); rd |= (unsigned) ac >= rdoqThr; if( !EXT || ( sv ) <= maxScan ) { lastNZ = max( lastNZ, sv ); \
          if( ac > useThres ) { const int cg = ( sv ) >> 4; if( NQUADS <= 128 || cg < 32 ) cgLo |= 1u << ( cg & 31 ); else cgHi |= 1u << ( cg - 32 ); } } }
        VVB_Q1( cq[k].x, sq[k].x ) VVB_Q1( cq[k].y, sq[k].y ) VVB_Q1( cq[k].z, sq[k].z ) VVB_Q1( cq[k].w, sq[k].w )
#undef VVB_Q1
      }
    }
  }
  lastNZ = __reduce_max_sync( tmask, lastNZ );
  cgLo   = __reduce_or_sync( tmask, cgLo );
  if( NQUADS > 128 ) cgHi = __reduce_or_sync( tmask, cgHi );
  rd     = __reduce_or_sync( tmask, rd );
  if( multi )
  {
    if( ( threadIdx.x & 31 ) == 0 )
    {
      if( lastNZ ) atomicMax( &red[1], lastNZ );
      if( cgLo ) atomicOr( reinterpret_cast<unsigned*>( &red[2] ), cgLo );
      if( cgHi ) atomicOr( reinterpret_cast<unsigned*>( &red[3] ), cgHi );
      if( rd ) atomicOr( &red[6], 1 );
    }
    __syncthreads();
    lastNZ = red[1]; cgLo = (unsigned) red[2]; cgHi = (unsigned) red[3];
  }
  else if( tt == 0 ) red[6] = (int) rd;
  // ---- final scan position after trailing-CG trimming (Quant.cpp:182-208)
  int pos = lastNZ;
  {
    const int initCg = pos >> 4;
    if( initCg >= 1 )
    {
      const unsigned long long mask = ( (unsigned long long) cgHi << 32 ) | cgLo;
      const unsigned long long m = mask & ( initCg >= 63 ? ~0ull : ( ( 1ull << ( initCg + 1 ) ) - 1ull ) ) & ~1ull;   // CGs 1..initCg
      if( m == 0 ) pos = 15;
      else { const int g = 63 - __clzll( (long long) m ); if( g != initCg ) pos = g * 16 + 15; }
    }
  }
  // ---- quantise (Quant.cpp:211-227): levels of the scanned region, zeros elsewhere
  if( S::W > S::RW || S::H > S::RH )
  {
#pragma unroll
    for( int k = 0; k < S::cdiv( S::RESI_WORDS, T ); k++ )
    {
      const int i = tt + k * T;
      const int y = i >> ( LW - 1 ), x = ( i & ( S::W / 2 - 1 ) ) << 1;
      if( live && i < S::RESI_WORDS && ( x >= S::RW || y >= S::RH ) ) qWords[i] = 0u;
    }
  }
  int sum = 0, lastQ = 0;                                   // lastQ holds scan position + 1
  const int qbits = par.qbits; const unsigned scale = (unsigned) par.scale, add32 = par.add32; const bool q32 = par.q32 != 0;
#pragma unroll
  for( int kk = 0; kk < ITERS; kk++ )
  {
    const int qi = tt + kk * T, k = CACHE ? kk : 0;
    if( live && ( NQUADS % T == 0 || qi < NQUADS ) )
    {
      if( !CACHE ) { cq[0] = c4[qi]; sq[0] = ( cq[0].x | cq[0].y | cq[0].z | cq[0].w ) ? __ldg( s4 + qi ) : make_int4( 0, 0, 0, 0 ); }
      int v0 = 0, v1 = 0, v2 = 0, v3 = 0;
#define VVB_Q2( cv, sv, vv ) if( ( cv ) && ( sv ) <= pos ) { \
        const unsigned ac = (unsigned) abs( cv ); \
        const int mag = ( q32 && ac < 65536u ) ? (int)( ( ac * scale + add32 ) >> qbits ) : (int)( ( (long long) ac * par.scale + par.add ) >> qbits ); \
        sum += mag; vv = min( 32767, mag ); if( ( cv ) < 0 ) vv = max( -32768, -mag ); if( vv ) lastQ = max( lastQ, ( sv ) + 1 ); }
      VVB_Q2( cq[k].x, sq[k].x, v0 ) VVB_Q2( cq[k].y, sq[k].y, v1 ) VVB_Q2( cq[k].z, sq[k].z, v2 ) VVB_Q2( cq[k].w, sq[k].w, v3 )
#undef VVB_Q2
      const int idx = qi << 2, y = idx >> S::LRW, x = idx & ( S::RW - 1 );
      uint2 o;
      o.x = ( (uint32_t) v0 & 0xffffu ) | ( (uint32_t) v1 << 16 );
      o.y = ( (uint32_t) v2 & 0xffffu ) | ( (uint32_t) v3 << 16 );
      *reinterpret_cast<uint2*>( qWords + ( ( ( y << LW ) + x ) >> 1 ) ) = o;
    }
  }
  sum   = __reduce_add_sync( tmask, sum );
  lastQ = __reduce_max_sync( tmask, lastQ );
  if( multi )
  {
    if( ( threadIdx.x & 31 ) == 0 ) { if( sum ) atomicAdd( &red[4], sum ); if( lastQ ) atomicMax( &red[5], lastQ ); }
  }
  else if( tt == 0 ) { red[4] = sum; red[5] = lastQ; }
  __syncthreads();
  if( EXT && par.signHiding )                                // uniform over the CTA
  {
    const int absSum = red[4], lastScanPos = red[5] - 1;     // scan position of the last level (Quant.cpp:806-816)
    __syncthreads();                                         // everybody has read red[5] before the top group's thread may rewrite it
    if( live && absSum >= 2 && lastScanPos >= 0 )
    {
      int16_t* q16 = reinterpret_cast<int16_t*>( qWords );
      for( int cg = tt; cg <= ( lastScanPos >> 4 ); cg += T )
      {
        const int nl = sbh_group<LW, S::LRW>( par, coef, q16, inv + VVB_SCAN_TABLE_ENTRIES, cg, lastScanPos );
        if( nl ) red[5] = nl;
      }
    }
    __syncthreads();
  }
  return pos;
}

// Forward transform + quantiser of one TU by one team.  `load( i )` returns residual word i (two int16, row-major compact).
// Contains __syncthreads(): every thread of the CTA must call it, `live` masks the work.  On return (all threads synchronised)
// v.resi holds the levels, v.coef the coefficients, v.red[4] absSum, v.red[5] lastQ+1, v.red[6] the RDOQ flag; returns the final scan pos.
template<int LW, int LH, bool EXT, class LOAD>
__device__ __forceinline__ int team_forward( const TuPar& par, const uint32_t* MtH, const uint32_t* MtV, const TeamView& v, const int32_t* __restrict__ scanTab,
                                             int tt, bool live, LOAD load )
{
  using S = TuShape<LW, LH>;
  constexpr int W = S::W, H = S::H, T = S::T, RW = S::RW, RH = S::RH;
  const int keepW = LW == 5 ? par.keepW : RW, keepH = LH == 5 ? par.keepH : RH;     // 16 for an MTS dimension of 32 (TrQuant.cpp:496-497)
  uint32_t* myResi = v.resi; int32_t* myTmp = reinterpret_cast<int32_t*>( v.tmp ); int32_t* myCoef = v.coef; int* myRed = v.red;
  __syncthreads();                                           // previous iteration's smem fully consumed; matrices visible
  if( tt < 8 ) myRed[tt] = 0;
  if( T < 8 && tt < 4 ) myRed[tt + 4] = 0;
#pragma unroll
  for( int k = 0; k < S::RESI_WORDS / T; k++ ) { const int i = tt + k * T; if( live ) myResi[i] = load( i ); }
  __syncthreads();
  const bool ts = EXT && par.ts != 0;                         // uniform over the launch
  if( ts )
  {
    // TrQuant::xTransformSkip (TrQuant.cpp:1050-1064): the residual is the coefficient block (sides <= 32: the scanned region is the whole TU)
    if( live )
      for( int i = tt; i < S::COEF_WORDS; i += T )
      {
        const uint32_t wv = myResi[i >> 1];
        myCoef[i] = ( i & 1 ) ? hi16( wv ) : lo16( wv );
      }
  }
  // ---- stage 1: tmp[j][i] = ( sum_k resi[i][k] * Th[j][k] + r1 ) >> s1   for i < H, j < keepW ; item = (row i, 4 outputs j0..j0+3)
  if( !ts )
  {
    const int s1 = par.s1, r1 = s1 > 0 ? 1 << ( s1 - 1 ) : 0;
    const int lJG = ( LW == 5 ? par.lKeepW : S::LRW ) - 2, items = H << lJG;
    int ovf = 0;
#pragma unroll
    for( int k = 0; k < S::cdiv( H * RW / 4, T ); k++ )
    {
      const int it = tt + k * T;
      if( live && it < items )
      {
        const int i = it >> lJG, j0 = ( it & ( ( 1 << lJG ) - 1 ) ) << 2;
        int a0 = 0, a1 = 0, a2 = 0, a3 = 0;
        const uint2* rrow = reinterpret_cast<const uint2*>( myResi + i * ( W / 2 ) );
        const uint32_t* mcol = MtH + j0;
#pragma unroll
        for( int q = 0; q < W / 4; q++ )
        {
          const uint2 rv = rrow[q];
          const uint4 m = *reinterpret_cast<const uint4*>( mcol + q * RW );
          a0 = __dp2a_lo( (int) rv.x, (int) m.x, a0 ); a0 = __dp2a_hi( (int) rv.y, (int) m.x, a0 );
          a1 = __dp2a_lo( (int) rv.x, (int) m.y, a1 ); a1 = __dp2a_hi( (int) rv.y, (int) m.y, a1 );
          a2 = __dp2a_lo( (int) rv.x, (int) m.z, a2 ); a2 = __dp2a_hi( (int) rv.y, (int) m.z, a2 );
          a3 = __dp2a_lo( (int) rv.x, (int) m.w, a3 ); a3 = __dp2a_hi( (int) rv.y, (int) m.w, a3 );
        }
        a0 = ( a0 + r1 ) >> s1; a1 = ( a1 + r1 ) >> s1; a2 = ( a2 + r1 ) >> s1; a3 = ( a3 + r1 ) >> s1;
        ovf |= ( a0 != (short) a0 ) | ( a1 != (short) a1 ) | ( a2 != (short) a2 ) | ( a3 != (short) a3 );
        int32_t* td = myTmp + j0 * H + i;
        td[0] = a0; td[H] = a1; td[2 * H] = a2; td[3 * H] = a3;
      }
    }
    if( ovf ) atomicOr( &myRed[0], 1 );
  }
  __syncthreads();
  // ---- stage 2: coef[j][i] = ( sum_k tmp[i][k] * Tv[j][k] + r2 ) >> s2   for i < keepW, j < keepH
  if( !ts )
  {
    const int s2 = par.s2, r2 = 1 << ( s2 - 1 );
    const int lJG = ( LH == 5 ? par.lKeepH : S::LRH ) - 2, items = keepW << lJG;
    const bool wide = myRed[0] != 0;
#pragma unroll
    for( int k = 0; k < S::cdiv( RW * RH / 4, T ); k++ )
    {
      const int it = tt + k * T;
      if( live && it < items )
      {
        const int i = it >> lJG, j0 = ( it & ( ( 1 << lJG ) - 1 ) ) << 2;
        int a0 = 0, a1 = 0, a2 = 0, a3 = 0;
        const int4* trow = reinterpret_cast<const int4*>( myTmp + i * H );
        const uint32_t* mcol = MtV + j0;
        if( !wide )
        {
#pragma unroll
          for( int q = 0; q < H / 4; q++ )
          {
            const int4 tv = trow[q];
            const uint32_t p0 = __byte_perm( (uint32_t) tv.x, (uint32_t) tv.y, 0x5410 );
            const uint32_t p1 = __byte_perm( (uint32_t) tv.z, (uint32_t) tv.w, 0x5410 );
            const uint4 m = *reinterpret_cast<const uint4*>( mcol + q * RH );
            a0 = __dp2a_lo( (int) p0, (int) m.x, a0 ); a0 = __dp2a_hi( (int) p1, (int) m.x, a0 );
            a1 = __dp2a_lo( (int) p0, (int) m.y, a1 ); a1 = __dp2a_hi( (int) p1, (int) m.y, a1 );
            a2 = __dp2a_lo( (int) p0, (int) m.z, a2 ); a2 = __dp2a_hi( (int) p1, (int) m.z, a2 );
            a3 = __dp2a_lo( (int) p0, (int) m.w, a3 ); a3 = __dp2a_hi( (int) p1, (int) m.w, a3 );
          }
        }
        else
        {
          for( int q = 0; q < H / 4; q++ )
          {
            const int4 tv = trow[q];
            const uint4 m = *reinterpret_cast<const uint4*>( mcol + q * RH );
#define VVB_MAC4( acc, mw ) acc += tv.x * (int)(signed char)( (mw) & 0xff ) + tv.y * (int)(signed char)( ( (mw) >> 8 ) & 0xff ) + tv.z * (int)(signed char)( ( (mw) >> 16 ) & 0xff ) + tv.w * (int)(signed char)( (mw) >> 24 )
            VVB_MAC4( a0, m.x ); VVB_MAC4( a1, m.y ); VVB_MAC4( a2, m.z ); VVB_MAC4( a3, m.w );
#undef VVB_MAC4
          }
        }
        a0 = ( a0 + r2 ) >> s2; a1 = ( a1 + r2 ) >> s2; a2 = ( a2 + r2 ) >> s2; a3 = ( a3 + r2 ) >> s2;
        int32_t* cd = myCoef + j0 * RW + i;
        cd[0] = a0; cd[RW] = a1; cd[2 * RW] = a2; cd[3 * RW] = a3;
      }
    }
    // rows/columns of the scanned region that were zeroed out (MTS 32 -> 16)
    if( ( LW == 5 || LH == 5 ) && live && ( keepW < RW || keepH < RH ) )
      for( int i = tt; i < S::COEF_WORDS; i += T )
      {
        const int y = i >> S::LRW, x = i & ( RW - 1 );
        if( x >= keepW || y >= keepH ) myCoef[i] = 0;
      }
  }
  __syncthreads();
  if( EXT && par.lfnstIdx )                                  // uniform over the CTA: TrQuant::xFwdLfnst (TrQuant.cpp:942-1048) between xT and the quantiser
  {
    constexpr int KEEP = ( LW >= 3 && LH >= 3 ) ? 8 : 4, NIN = KEEP == 8 ? 48 : 16;
    constexpr int ZOUT = ( ( W == 4 && H == 4 ) || ( W == 8 && H == 8 ) ) ? 8 : 16;
    // the primary transform keeps the top-left KEEP x KEEP outputs only (TrQuant.cpp:499-511)
    if( live )
      for( int i = tt; i < S::COEF_WORDS; i += T )
      {
        const int y = i >> S::LRW, x = i & ( RW - 1 );
        if( x >= KEEP || y >= KEEP ) myCoef[i] = 0;
      }
    __syncthreads();
    int32_t* lfOut = myTmp;                                  // the stage-1 buffer is free now
    if( live )
      for( int j = tt; j < ZOUT; j += T )
      {
        const int8_t* m = par.lfnstMat + j * NIN;
        int sum = 0;
#pragma unroll 4
        for( int i = 0; i < NIN; i++ )
        {
          int a, b;                                          // walk of :973-1019: rows of 8 then rows of 4 (sub-block 8), rows of 4 (sub-block 4); transposed: columns
          if( KEEP == 4 ) { b = i >> 2; a = i & 3; }
          else if( i < 32 ) { b = i >> 3; a = i & 7; }
          else { b = 4 + ( ( i - 32 ) >> 2 ); a = ( i - 32 ) & 3; }
          const int x = par.lfnstTranspose ? b : a, y = par.lfnstTranspose ? a : b;
          sum += myCoef[( y << S::LRW ) + x] * (int) __ldg( m + i );
        }
        lfOut[j] = ( sum + 64 ) >> 7;                        // xFwdLfnstNxNCore, :166-187
      }
    __syncthreads();
    if( live )
    {
      const int32_t* fwd8 = scanTab + VVB_SCAN_TABLE_ENTRIES + 6 * 1024;     // grouped 4x4 diagonal scan of an 8x8 region (= g_coefTopLeftDiagScan8x8 without the TU pitch)
      for( int j = tt; j < NIN; j += T )
      {
        const int p = __ldg( fwd8 + j );
        myCoef[( ( p >> 3 ) << S::LRW ) + ( p & 7 )] = j < ZOUT ? lfOut[j] : 0;
      }
    }
    __syncthreads();
  }
  return team_quantise<LW, LH, T, EXT>( par, myCoef, myResi, myRed, scanTab + par.scanOff, tt, live );
}

// results of team_forward -> global memory (q compact [H][W]; optional coefficients and per-TU scalars)
template<int LW, int LH>
__device__ __forceinline__ void team_forward_store( const TeamView& v, int pos, int tu, int tt, bool live,
                                                    int32_t* __restrict__ coefOut, int16_t* __restrict__ qOut, int32_t* __restrict__ absSumOut,
                                                    int32_t* __restrict__ lastPosOut, uint8_t* __restrict__ needRdoqOut )
{
  using S = TuShape<LW, LH>;
  constexpr int W = S::W, H = S::H, T = S::T;
  if( live )
  {
    uint32_t* dst = reinterpret_cast<uint32_t*>( qOut + (size_t) tu * W * H );
#pragma unroll
    for( int k = 0; k < S::RESI_WORDS / T; k++ ) dst[tt + k * T] = v.resi[tt + k * T];
    if( coefOut )
    {
      int32_t* cd = coefOut + (size_t) tu * W * H;
      for( int i = tt; i < W * H; i += T )
      {
        const int y = i >> LW, x = i & ( W - 1 );
        cd[i] = ( x < S::RW && y < S::RH ) ? v.coef[( y << S::LRW ) + x] : 0;
      }
    }
    if( tt == 0 )
    {
      const int sum = v.red[4];
      if( absSumOut )   absSumOut[tu]   = sum;
      if( lastPosOut )  lastPosOut[tu]  = sum ? v.red[5] - 1 : pos;      // Quant.cpp:806-816, :830
      if( needRdoqOut ) needRdoqOut[tu] = (uint8_t) v.red[6];
    }
  }
}

// Residual word i (two int16, row-major compact [H][W]) of a TU whose original starts at o (row pitch so pels) and whose prediction starts at p (pitch sp):
// org - pred (PelBuf::subtract, IntraSearch.cpp:1328), one word load from each where both rows allow it, single pels otherwise
template<int LW> __device__ __forceinline__ auto org_pred_words( const int16_t* o, int so, const int16_t* p, int sp )
{
  const bool al4 = ( ( ( reinterpret_cast<uintptr_t>( o ) | reinterpret_cast<uintptr_t>( p ) ) & 3 ) | ( ( so | sp ) & 1 ) ) == 0;   // word loads allowed
  return [=]( int i ) -> uint32_t
  {
    const int y = i >> ( LW - 1 ), x = ( i & ( ( 1 << ( LW - 1 ) ) - 1 ) ) << 1;
    const int16_t* oy = o + (ptrdiff_t) y * so + x; const int16_t* py = p + (ptrdiff_t) y * sp + x;
    if( al4 ) return __vsub2( __ldg( reinterpret_cast<const uint32_t*>( oy ) ), __ldg( reinterpret_cast<const uint32_t*>( py ) ) );
    const int d0 = (int) __ldg( oy ) - (int) __ldg( py ), d1 = (int) __ldg( oy + 1 ) - (int) __ldg( py + 1 );
    return ( (uint32_t) d0 & 0xffffu ) | ( (uint32_t) d1 << 16 );
  };
}

// where the forward kernels read the residual: the MODE of fwd_trquant_tc2_kernel (trquant_tc2_kernels.cuh) that fwd_trquant_kernel's SRC takes too
enum ResiMode { RESI_POOL = 0, RESI_PLANES = 1, RESI_TWO_POOLS = 2 };

// SRC = RESI_POOL: the residual of TU i is resi[i] of a compact pool [n][H][W].  SRC = RESI_PLANES: it is formed at load time, TU i sits at (blocks[i].x,
// blocks[i].y) of orgPlane, its prediction at (+start_x, +start_y) of predPlane -- no compact residual buffer, no extra launch.  SRC = RESI_TWO_POOLS: it is
// formed at load time from the original pool resi[i] and the prediction pool pred[i]
template<int LW, int LH, bool EXT, int SRC>
__global__ void __launch_bounds__( 128 ) fwd_trquant_kernel( const __grid_constant__ TuPar par, const int8_t* __restrict__ trTable, const int32_t* __restrict__ scanTab,
                                                             const int16_t* __restrict__ resi, const int16_t* __restrict__ pred,
                                                             const __grid_constant__ Plane orgPlane, const __grid_constant__ Plane predPlane,
                                                             const vvb_block* __restrict__ blocks, int n,
                                                             int32_t* __restrict__ coefOut, int16_t* __restrict__ qOut, int32_t* __restrict__ absSumOut,
                                                             int32_t* __restrict__ lastPosOut, uint8_t* __restrict__ needRdoqOut )
{
  using S = TuShape<LW, LH>;
  extern __shared__ __align__( 16 ) uint32_t smem[];
  constexpr int T = S::T, NTEAMS = S::NTEAMS;
  const int team = threadIdx.x / T, tt = threadIdx.x % T;
  // ---- matrices, shared by all teams of the CTA
  uint32_t* MtH = smem;                                        // [W/4][RW]
  uint32_t* MtV = MtH + ( S::W / 4 ) * S::RW;                  // [H/4][RH]
  uint32_t* teamBase = smem + S::MAT_WORDS;
  stage_matrix( MtH, trTable, par.offH, S::W, par.keepW, S::RW, threadIdx.x, blockDim.x );
  stage_matrix( MtV, trTable, par.offV, S::H, par.keepH, S::RH, threadIdx.x, blockDim.x );
  const TeamView v = team_view<S>( teamBase, team );

  for( int base = blockIdx.x * NTEAMS; base < n; base += gridDim.x * NTEAMS )
  {
    const int tu = base + team;
    const bool live = tu < n;
    int pos;
    if constexpr( SRC == RESI_PLANES )
    {
      const vvb_block blk = blocks[live ? tu : 0];
      const int so = orgPlane.stride, sp = predPlane.stride;
      pos = team_forward<LW, LH, EXT>( par, MtH, MtV, v, scanTab, tt, live,
                                       org_pred_words<LW>( orgPlane.origin + (ptrdiff_t) blk.y * so + blk.x, so,
                                                           predPlane.origin + (ptrdiff_t)( blk.y + blk.start_y ) * sp + blk.x + blk.start_x, sp ) );
    }
    else if constexpr( SRC == RESI_TWO_POOLS )
    {
      const size_t off = (size_t)( live ? tu : 0 ) * S::W * S::H;
      pos = team_forward<LW, LH, EXT>( par, MtH, MtV, v, scanTab, tt, live, org_pred_words<LW>( resi + off, S::W, pred + off, S::W ) );
    }
    else
    {
      const uint32_t* src = reinterpret_cast<const uint32_t*>( resi + (size_t)( live ? tu : 0 ) * S::W * S::H );
      pos = team_forward<LW, LH, EXT>( par, MtH, MtV, v, scanTab, tt, live, [&]( int i ) { return __ldg( src + i ); } );
    }
    team_forward_store<LW, LH>( v, pos, tu, tt, live, coefOut, qOut, absSumOut, lastPosOut, needRdoqOut );
  }
}

} // namespace vvb
