// itrquant_tc_kernels.cuh -- dequantiser + inverse 2-D transform of square TUs 8x8 .. 64x64 on the wgmma tensor cores, raw-byte operands as in
// trquant_tc2_kernels.cuh.  Simpler than the forward direction: the reference clips the dequantised coefficients and the first-pass outputs to 16 bit
// (Quant.cpp:232-262, TrQuant_EMT.cpp fastInverse: clipMinimum / clipMaximum), so both stages read int16 values = two byte planes (low u8, high s8):
//   stage 1 (vertical, shift 7):   A3[row (tu, column j)][2k + b] = byte b of the dequantised coefficient c[k][j]     (transposed 16-bit stores)
//                                  B3lo[y][2k] = Tv[k][y] , B3hi[y][2k+1] = Tv[k][y]      tmp[j][y] = clip16( ( Dlo + 256 * Dhi + 64 ) >> 7 )
//   stage 2 (horizontal, 20 - bd): A4[row (tu, y)][2j + b] = byte b of tmp[j][y]                                       (transposed 16-bit stores)
//                                  B4lo[x][2j] = Th[j][x] , B4hi[x][2j+1] = Th[j][x]      resi[y][x] = clip16( ( Dlo + 256 * Dhi + rnd ) >> s2 )
// Tile = 128 stage-2 rows = 128 / N TUs (at 64x64 the 64 stage-1 rows fill one m64 half; the threads of the other half load a copy that no MMA reads),
// one CTA of 128 threads = one warpgroup:
//   load + dequantise row k of the levels -> A3 ; MMA ; clip the accumulator registers -> A4 ; MMA ; clip -> staging rows ; thread = residual row (tu, y),
//   which goes out with 16-byte stores,
// or, for the fused TU round trip (RT), straight into reconstruction and the three distortions of tu_roundtrip_kernel (itrquant_kernels.cuh).
// Rows / columns beyond the kept coefficients (MTS at 32 keeps 16) have zero rows in the B operands, like the loops of team_inverse that never read them.
#pragma once
#include "trquant_tc2_kernels.cuh"
#include "itrquant_kernels.cuh"

namespace vvb {

template<int N> struct ItcShape
{
  static constexpr int KEEP = N > 32 ? 32 : N;             // coefficient rows / columns that can be non-zero (DCT-II zero-out at 64)
  static constexpr int TPT  = 128 / N;                     // TUs per tile: the stage-2 rows (tu, y) fill the 128 lanes
  static constexpr int DUP  = N / KEEP;                    // 64x64: the 64 stage-1 rows (tu, j) are written twice, so that all four warps read first-pass outputs (32 y each)
  static constexpr int NMMA = N < 16 ? 16 : N;             // outputs per MMA (y in stage 1, x in stage 2)
  static constexpr int K = 2 * KEEP < 32 ? 32 : 2 * KEEP, NCH = K / 16;
  static constexpr int SBO = 160, LBO = 16 * SBO + 16;     // as A2 of the forward engine: the transposed stores of a warp spread over the banks
  static constexpr int A_BYTES = NCH * LBO;                // A3 and A4 have the same geometry
  static constexpr int BCH = NMMA * 16, B_BYTES = NCH * BCH;
  static constexpr int LDR = N + 8;                        // int16 staging rows of the residual (16-byte aligned)
  static constexpr int SMEM = 2 * A_BYTES + 4 * B_BYTES + 128 * LDR * 2;   // A3 | A4 | B3lo | B3hi | B4lo | B4hi | staging
  static constexpr int CH = N < 16 ? 8 : 16;
};

// Host side: B3lo | B3hi | B4lo | B4hi in the canonical K-major layout [16-byte K chunk][row][16 B]
template<int N> static void itc_build_b_image( const int8_t* tab, int offH, int offV, int keepW, int keepH, unsigned char* out )
{
  using S = ItcShape<N>;
  for( int i = 0; i < S::B_BYTES; i++ )
  {
    const int c = i / S::BCH, r = ( i / 16 ) % S::NMMA, kb = c * 16 + ( i & 15 ), k = kb >> 1;
    const unsigned char v3 = ( r < N && k < keepH && k < S::KEEP ) ? (unsigned char) tab[offV + k * N + r] : 0;     // Tv[k][y = r]
    const unsigned char v4 = ( r < N && k < keepW && k < S::KEEP ) ? (unsigned char) tab[offH + k * N + r] : 0;     // Th[k][x = r]
    out[i] = ( kb & 1 ) ? 0 : v3;                 out[S::B_BYTES + i] = ( kb & 1 ) ? v3 : 0;
    out[2 * S::B_BYTES + i] = ( kb & 1 ) ? 0 : v4; out[3 * S::B_BYTES + i] = ( kb & 1 ) ? v4 : 0;
  }
}

// RT = false: levels -> residual.  RT = true: the second half of the fused TU round trip (levels, absSum, lastPos from the forward engine).
template<int N, bool RT>
__global__ void __launch_bounds__( 128, 4 ) inv_trquant_tc_kernel( const __grid_constant__ TuPar par, const uint4* __restrict__ bImage, const int16_t* __restrict__ q, int n,
                                                                   int16_t* __restrict__ resiOut,
                                                                   const int planes, const __grid_constant__ Plane orgPlane, const __grid_constant__ Plane predPlane,
                                                                   const vvb_block* __restrict__ blocks, const int16_t* __restrict__ orgPool, const int16_t* __restrict__ predPool,
                                                                   int16_t* __restrict__ recoOut, TuResult* __restrict__ resOut,
                                                                   const int32_t* __restrict__ absSumIn, const int32_t* __restrict__ lastPosIn )
{
  using S = ItcShape<N>;
  constexpr int TPT = S::TPT, NMMA = S::NMMA, CH = S::CH, KEEP = S::KEEP, DUP = S::DUP;
  extern __shared__ __align__( 128 ) unsigned char smemItc[];
  unsigned char* sA3 = smemItc;
  unsigned char* sA4 = smemItc + S::A_BYTES;
  unsigned char* sB  = smemItc + 2 * S::A_BYTES;
  int16_t* sR = reinterpret_cast<int16_t*>( sB + 4 * S::B_BYTES );

  const int tid = threadIdx.x, warp = tid >> 5;
  for( int i = tid; i < 4 * S::B_BYTES / 16; i += 128 ) reinterpret_cast<uint4*>( sB )[i] = __ldg( bImage + i );
  for( int i = tid; i < 2 * S::A_BYTES / 16; i += 128 ) reinterpret_cast<uint4*>( sA3 )[i] = make_uint4( 0, 0, 0, 0 );     // K padding (8x8) stays zero
  __syncthreads();
  const uint64_t dA3 = gmma_desc_kmajor( smem_u32( sA3 ), S::LBO, S::SBO ), dA4 = gmma_desc_kmajor( smem_u32( sA4 ), S::LBO, S::SBO );
  const uint64_t dB = gmma_desc_kmajor( smem_u32( sB ), S::BCH, 128 );
  const int numTiles = ( n + TPT - 1 ) / TPT;
  const int tl = tid / N, rr = tid % N;                       // stage 2: TU of the tile and row y of this thread
  const int r1 = tid % KEEP, t1 = ( tid / KEEP ) % TPT, cp = tid / ( KEEP * TPT );   // levels / stage 1: row k resp. column j, TU, copy (64x64 only)
  const int sc = par.dqScale, sh = par.dqShift, inMax = par.dqInMax, inMin = -inMax - 1;
  const int addQ = sh > 0 ? 1 << ( sh - 1 ) : 0;
  const int s2 = par.s2Inv, r2 = 1 << ( s2 - 1 );
  // transposed 16-bit store of element e (0..N-1) of this thread's row into row (tl, e) of an A operand, K position rr
  unsigned char* const stBase3 = sA3 + ( r1 >> 3 ) * S::LBO + ( ( cp * TPT + t1 ) * KEEP / 8 ) * S::SBO + ( r1 & 7 ) * 2;

  for( int tile = blockIdx.x; tile < numTiles; tile += gridDim.x )
  {
    const int tu = tile * TPT + tl;
    const bool live = tu < n;
    const bool active = live && ( !RT || absSumIn[tu] > 0 );   // a TU quantised to zero has residual 0 (IntraSearch.cpp:1366-1369)
    // ---- levels row k = r1 of TU t1 (the kept KEEP x KEEP corner) -> dequantise (DeQuantCore, Quant.cpp:232-262) -> A3 rows (copy, t1, j), K position k
    {
      const int tu1 = tile * TPT + t1;
      const bool act1 = tu1 < n && ( !RT || absSumIn[tu1] > 0 );
      const uint4* src = reinterpret_cast<const uint4*>( q + ( (size_t)( tu1 < n ? tu1 : 0 ) * N + r1 ) * N );
#pragma unroll
      for( int c = 0; c < KEEP / 8; c++ )
      {
        uint4 v = make_uint4( 0, 0, 0, 0 );
        if( act1 ) v = RT ? src[c] : __ldg( src + c );
        const uint32_t w[4] = { v.x, v.y, v.z, v.w };
#pragma unroll
        for( int e = 0; e < 8; e++ )
        {
          int cv = e & 1 ? hi16( w[e >> 1] ) : lo16( w[e >> 1] );
          cv = max( inMin, min( inMax, cv ) );
          cv = sh > 0 ? ( cv * sc + addQ ) >> sh : (int)( (unsigned)( cv * sc ) << ( -sh ) );
          cv = clip16( cv );
          const int j = 8 * c + e;
          *reinterpret_cast<int16_t*>( stBase3 + ( j >> 3 ) * S::SBO + ( j & 7 ) * 16 ) = (int16_t) cv;
        }
      }
    }
    fence_async_smem();
    __syncthreads();
    // ---- stage 1: Dlo / Dhi [rows (t1, column j) x y] (A3 read as u8 / s8); tmp[j][y] = clip16( ( Dlo + 256 * Dhi + 64 ) >> 7 ) -> A4 row (t1, y), K position j
    {
      constexpr int MH = DUP == 2 ? 1 : 2;                     // 64x64: the copy in rows 64..127 is not multiplied
      int lo[MH][NMMA / 2], hi[MH][NMMA / 2];
#pragma unroll
      for( int h = 0; h < MH; h++ ) { wg_hold( lo[h] ); wg_hold( hi[h] ); }
      wg_fence();
#pragma unroll
      for( int h = 0; h < MH; h++ )
#pragma unroll
        for( int ks = 0; ks < S::K / 32; ks++ )
        {
          const uint64_t da = dA3 + (uint64_t)( ( h * 8 * S::SBO + ks * 2 * S::LBO ) >> 4 );
          wgmma_i8<NMMA, false>( lo[h], da, dB + (uint64_t)( ( ks * 2 * S::BCH ) >> 4 ), ks > 0 );
          wgmma_i8<NMMA, true>( hi[h], da, dB + (uint64_t)( ( S::B_BYTES + ks * 2 * S::BCH ) >> 4 ), ks > 0 );
        }
      wg_commit();
      wg_wait0();
#pragma unroll
      for( int h = 0; h < MH; h++ ) { wg_hold( lo[h] ); wg_hold( hi[h] ); }
#pragma unroll
      for( int h = 0; h < MH; h++ )
#pragma unroll
        for( int i = 0; i < NMMA / 2; i++ )
        {
          const int r = h * 64 + wg_row( i ), y = wg_col( i ), j = r % KEEP, t = ( r / KEEP ) % TPT;
          if( y < N )
            *reinterpret_cast<int16_t*>( sA4 + ( j >> 3 ) * S::LBO + ( t * N / 8 + ( y >> 3 ) ) * S::SBO + ( j & 7 ) * 2 + ( y & 7 ) * 16 ) =
              (int16_t) clip16( ( ( hi[h][i] << 8 ) + lo[h][i] + 64 ) >> 7 );
        }
    }
    fence_async_smem();
    __syncthreads();
    // ---- stage 2: rows (tu, y) x columns x (A4 read as u8 / s8), one 64-row half at a time, each with accumulators of its own;
    //      resi = clip16( ( Dlo + 256 * Dhi + rnd ) >> s2 ) -> staging
    {
      int lo[2][NMMA / 2], hi[2][NMMA / 2];
#pragma unroll
      for( int h = 0; h < 2; h++ )
      {
        wg_fence();
#pragma unroll
        for( int ks = 0; ks < S::K / 32; ks++ )
        {
          const uint64_t da = dA4 + (uint64_t)( ( h * 8 * S::SBO + ks * 2 * S::LBO ) >> 4 );
          wgmma_i8<NMMA, false>( lo[h], da, dB + (uint64_t)( ( 2 * S::B_BYTES + ks * 2 * S::BCH ) >> 4 ), ks > 0 );
          wgmma_i8<NMMA, true>( hi[h], da, dB + (uint64_t)( ( 3 * S::B_BYTES + ks * 2 * S::BCH ) >> 4 ), ks > 0 );
        }
        wg_commit();
        wg_wait0();
        wg_hold( lo[h] ); wg_hold( hi[h] );
#pragma unroll
        for( int i = 0; i < NMMA / 2; i++ )
        {
          const int r = h * 64 + wg_row( i ), x = wg_col( i );
          if( x < N ) sR[r * S::LDR + x] = (int16_t) clip16( ( ( hi[h][i] << 8 ) + lo[h][i] + r2 ) >> s2 );
        }
      }
    }
    __syncthreads();
    // ---- residual row y = rr
    {
      int16_t* dst = RT ? nullptr : resiOut + ( (size_t)( live ? tu : 0 ) * N + rr ) * N;
      const int16_t* oRow = nullptr; const int16_t* pRow = nullptr; int16_t* rRow = nullptr;
      unsigned long long dReco = 0, dResi = 0, dZero = 0;
      if( RT )
      {
        if( planes )
        {
          const vvb_block blk = blocks[live ? tu : 0];
          oRow = orgPlane.origin + (ptrdiff_t)( blk.y + rr ) * orgPlane.stride + blk.x;
          pRow = predPlane.origin + (ptrdiff_t)( blk.y + blk.start_y + rr ) * predPlane.stride + blk.x + blk.start_x;
        }
        else
        {
          oRow = orgPool + ( (size_t)( live ? tu : 0 ) * N + rr ) * N;
          pRow = predPool + ( (size_t)( live ? tu : 0 ) * N + rr ) * N;
        }
        rRow = recoOut ? recoOut + ( (size_t)( live ? tu : 0 ) * N + rr ) * N : nullptr;
      }
      const int pelMax = par.pelMax;
#pragma unroll
      for( int c0 = 0; c0 < N; c0 += CH )
      {
        int r[CH];
#pragma unroll
        for( int k = 0; k < CH; k += 8 )
        {
          const uint4 v = *reinterpret_cast<const uint4*>( sR + tid * S::LDR + c0 + k );
          const uint32_t w[4] = { v.x, v.y, v.z, v.w };
#pragma unroll
          for( int e = 0; e < 8; e++ ) r[k + e] = active ? ( e & 1 ? hi16( w[e >> 1] ) : lo16( w[e >> 1] ) ) : 0;
        }
        if( !RT )
        {
          if( live )
#pragma unroll
            for( int k = 0; k < CH; k += 8 )
              *reinterpret_cast<uint4*>( dst + c0 + k ) = make_uint4( ( (uint32_t) r[k] & 0xffffu ) | ( (uint32_t) r[k + 1] << 16 ), ( (uint32_t) r[k + 2] & 0xffffu ) | ( (uint32_t) r[k + 3] << 16 ),
                                                                      ( (uint32_t) r[k + 4] & 0xffffu ) | ( (uint32_t) r[k + 5] << 16 ), ( (uint32_t) r[k + 6] & 0xffffu ) | ( (uint32_t) r[k + 7] << 16 ) );
        }
        else if( live )
        {
#pragma unroll
          for( int k = 0; k < CH; k += 8 )
          {
            int rc[8];
            unsigned sz = 0, scc = 0;
            uint32_t ow[4], pw[4];
            tc2_load8( oRow + c0 + k, ow ); tc2_load8( pRow + c0 + k, pw );
#pragma unroll
            for( int e = 0; e < 8; e++ )
            {
              const int ov = e & 1 ? hi16( ow[e >> 1] ) : lo16( ow[e >> 1] ), pv = e & 1 ? hi16( pw[e >> 1] ) : lo16( pw[e >> 1] );
              rc[e] = max( 0, min( pelMax, pv + r[k + e] ) );
              const int dz = ov - pv;
              const long long dr = (long long) dz - r[k + e];
              const int dc = ov - rc[e];
              sz += (unsigned)( dz * dz ); scc += (unsigned)( dc * dc );
              dResi += (unsigned long long)( dr * dr );
            }
            dZero += sz; dReco += scc;
            if( rRow )
              *reinterpret_cast<uint4*>( rRow + c0 + k ) = make_uint4( ( (uint32_t) rc[0] & 0xffffu ) | ( (uint32_t) rc[1] << 16 ), ( (uint32_t) rc[2] & 0xffffu ) | ( (uint32_t) rc[3] << 16 ),
                                                                       ( (uint32_t) rc[4] & 0xffffu ) | ( (uint32_t) rc[5] << 16 ), ( (uint32_t) rc[6] & 0xffffu ) | ( (uint32_t) rc[7] << 16 ) );
          }
        }
      }
      if( RT )
      {
        // the N lanes (tl, y) of a TU: aligned lane groups of 8 / 16 lanes, a whole warp, or two warps (64x64)
#pragma unroll
        for( int off = ( N > 32 ? 32 : N ) / 2; off > 0; off >>= 1 )
        {
          dReco += __shfl_xor_sync( 0xffffffffu, dReco, off );
          dResi += __shfl_xor_sync( 0xffffffffu, dResi, off );
          dZero += __shfl_xor_sync( 0xffffffffu, dZero, off );
        }
        if( N > 32 )
        {
          __shared__ unsigned long long sAcc[4][3];
          if( ( tid & 31 ) == 0 ) { sAcc[warp][0] = dReco; sAcc[warp][1] = dResi; sAcc[warp][2] = dZero; }
          __syncthreads();
          dReco = sAcc[2 * tl][0] + sAcc[2 * tl + 1][0]; dResi = sAcc[2 * tl][1] + sAcc[2 * tl + 1][1]; dZero = sAcc[2 * tl][2] + sAcc[2 * tl + 1][2];
        }
        if( live && rr == 0 )
        {
          TuResult t;
          t.distReco = dReco; t.distResi = dResi; t.distZero = dZero; t.absSum = absSumIn[tu]; t.lastPos = lastPosIn[tu];
          resOut[tu] = t;
        }
      }
    }
    __syncthreads();
  }
}

} // namespace vvb
