// trquant_tc_kernels.cuh -- forward 2-D integer transform on the Hopper tensor cores (wgmma, s8 x s8 -> s32, register
// accumulators) + the same fused quantiser as trquant_kernels.cuh.  Square TUs 16x16, 32x32, 64x64.
//
// Exact-integer strategy (SURVEY.md 7-3): the transform is pure int32 (TrQuant_EMT.cpp:1973-2000), the matrices fit s8
// (|T| <= 91), so both stages run as s8 x s8 -> s32 MMAs on byte planes of the left operand:
//   stage 1:  r   = r1*2^7  + r0               (r0 in [0,127], r1 = r >> 7, |r| < 2^14)        -> 2 MMAs per K step
//   stage 2:  tmp = t2*2^14 + t1*2^7 + t0      (t0,t1 in [0,127], t2 = tmp >> 14, |tmp| < 2^21) -> 3 MMAs per K step
// and the epilogue recombines  sum = (d2 << 14) + (d1 << 7) + d0  in int32 before the rounding shift.  No value is ever
// rounded, so the coefficients equal the scalar reference bit for bit (also where the AVX2 path would saturate).
//
// Tile = 128 stacked rows = 128/N TUs.  A operands are written to shared memory by the threads themselves in the canonical
// K-major no-swizzle layout ([16-byte K chunk][row][16 B]: SBO = 128 B, LBO = rows*16 B), B = the transform matrix rows in
// the same layout, D lives in the registers of the warpgroup (two m64 halves of the 128 rows).  Stage-1 results are scattered
// transposed (bytes) into the stage-2 A operand, so the second transform is again "rows x matrix".
#pragma once
#include "common.cuh"
#include "trquant_kernels.cuh"

namespace vvb {

__device__ __forceinline__ uint32_t smem_u32( const void* p ) { return (uint32_t) __cvta_generic_to_shared( p ); }

// wgmma shared-memory descriptor, K-major, no swizzle (PTX ISA, "Matrix Descriptor Format"): start address, leading byte offset = stride between the
// 16-byte K chunks of a k32 step, stride byte offset = stride between 8-row groups; base offset 0, layout type 0
__device__ __forceinline__ uint64_t gmma_desc_kmajor( uint32_t smemAddr, uint32_t lboBytes, uint32_t sboBytes )
{
  uint64_t d = 0;
  d |= (uint64_t)( ( smemAddr >> 4 ) & 0x3fffu );           // start address, bits [0,14)
  d |= (uint64_t)( ( lboBytes >> 4 ) & 0x3fffu ) << 16;     // leading byte offset, bits [16,30)
  d |= (uint64_t)( ( sboBytes >> 4 ) & 0x3fffu ) << 32;     // stride byte offset, bits [32,46)
  return d;
}

// D[64 x NN] (+)= A[64 x 32 B] * B[NN x 32 B]^T, A read as u8 (AS = false) or s8 (AS = true), B as s8, s32 accumulators; issued by the whole warpgroup
// (the 128 threads of the CTA).  accumulate = 0 starts the chain.  Register i of a thread holds row wg_row( i ), column wg_col( i ) of D.
template<int NN, bool AS> __device__ __forceinline__ void wgmma_i8( int (&d)[NN / 2], uint64_t descA, uint64_t descB, int accumulate );
template<> __device__ __forceinline__ void wgmma_i8<16, false>( int (&d)[8], uint64_t descA, uint64_t descB, int accumulate )
{
  asm volatile( "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %10, 0;\n\t"
                "wgmma.mma_async.sync.aligned.m64n16k32.s32.u8.s8 {%0,%1,%2,%3,%4,%5,%6,%7}, %8, %9, p;\n\t}\n"
                : "+r"( d[0] ), "+r"( d[1] ), "+r"( d[2] ), "+r"( d[3] ), "+r"( d[4] ), "+r"( d[5] ), "+r"( d[6] ), "+r"( d[7] )
                : "l"( descA ), "l"( descB ), "r"( accumulate ) : "memory" );
}
template<> __device__ __forceinline__ void wgmma_i8<16, true>( int (&d)[8], uint64_t descA, uint64_t descB, int accumulate )
{
  asm volatile( "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %10, 0;\n\t"
                "wgmma.mma_async.sync.aligned.m64n16k32.s32.s8.s8 {%0,%1,%2,%3,%4,%5,%6,%7}, %8, %9, p;\n\t}\n"
                : "+r"( d[0] ), "+r"( d[1] ), "+r"( d[2] ), "+r"( d[3] ), "+r"( d[4] ), "+r"( d[5] ), "+r"( d[6] ), "+r"( d[7] )
                : "l"( descA ), "l"( descB ), "r"( accumulate ) : "memory" );
}
template<> __device__ __forceinline__ void wgmma_i8<32, false>( int (&d)[16], uint64_t descA, uint64_t descB, int accumulate )
{
  asm volatile( "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %18, 0;\n\t"
                "wgmma.mma_async.sync.aligned.m64n32k32.s32.u8.s8 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15}, %16, %17, p;\n\t}\n"
                : "+r"( d[0] ), "+r"( d[1] ), "+r"( d[2] ), "+r"( d[3] ), "+r"( d[4] ), "+r"( d[5] ), "+r"( d[6] ), "+r"( d[7] ), "+r"( d[8] ), "+r"( d[9] ), "+r"( d[10] ), "+r"( d[11] ), "+r"( d[12] ), "+r"( d[13] ), "+r"( d[14] ), "+r"( d[15] )
                : "l"( descA ), "l"( descB ), "r"( accumulate ) : "memory" );
}
template<> __device__ __forceinline__ void wgmma_i8<32, true>( int (&d)[16], uint64_t descA, uint64_t descB, int accumulate )
{
  asm volatile( "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %18, 0;\n\t"
                "wgmma.mma_async.sync.aligned.m64n32k32.s32.s8.s8 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15}, %16, %17, p;\n\t}\n"
                : "+r"( d[0] ), "+r"( d[1] ), "+r"( d[2] ), "+r"( d[3] ), "+r"( d[4] ), "+r"( d[5] ), "+r"( d[6] ), "+r"( d[7] ), "+r"( d[8] ), "+r"( d[9] ), "+r"( d[10] ), "+r"( d[11] ), "+r"( d[12] ), "+r"( d[13] ), "+r"( d[14] ), "+r"( d[15] )
                : "l"( descA ), "l"( descB ), "r"( accumulate ) : "memory" );
}
template<> __device__ __forceinline__ void wgmma_i8<64, false>( int (&d)[32], uint64_t descA, uint64_t descB, int accumulate )
{
  asm volatile( "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
                "wgmma.mma_async.sync.aligned.m64n64k32.s32.u8.s8 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31}, %32, %33, p;\n\t}\n"
                : "+r"( d[0] ), "+r"( d[1] ), "+r"( d[2] ), "+r"( d[3] ), "+r"( d[4] ), "+r"( d[5] ), "+r"( d[6] ), "+r"( d[7] ), "+r"( d[8] ), "+r"( d[9] ), "+r"( d[10] ), "+r"( d[11] ), "+r"( d[12] ), "+r"( d[13] ), "+r"( d[14] ), "+r"( d[15] ), "+r"( d[16] ), "+r"( d[17] ), "+r"( d[18] ), "+r"( d[19] ), "+r"( d[20] ), "+r"( d[21] ), "+r"( d[22] ), "+r"( d[23] ), "+r"( d[24] ), "+r"( d[25] ), "+r"( d[26] ), "+r"( d[27] ), "+r"( d[28] ), "+r"( d[29] ), "+r"( d[30] ), "+r"( d[31] )
                : "l"( descA ), "l"( descB ), "r"( accumulate ) : "memory" );
}
template<> __device__ __forceinline__ void wgmma_i8<64, true>( int (&d)[32], uint64_t descA, uint64_t descB, int accumulate )
{
  asm volatile( "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
                "wgmma.mma_async.sync.aligned.m64n64k32.s32.s8.s8 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31}, %32, %33, p;\n\t}\n"
                : "+r"( d[0] ), "+r"( d[1] ), "+r"( d[2] ), "+r"( d[3] ), "+r"( d[4] ), "+r"( d[5] ), "+r"( d[6] ), "+r"( d[7] ), "+r"( d[8] ), "+r"( d[9] ), "+r"( d[10] ), "+r"( d[11] ), "+r"( d[12] ), "+r"( d[13] ), "+r"( d[14] ), "+r"( d[15] ), "+r"( d[16] ), "+r"( d[17] ), "+r"( d[18] ), "+r"( d[19] ), "+r"( d[20] ), "+r"( d[21] ), "+r"( d[22] ), "+r"( d[23] ), "+r"( d[24] ), "+r"( d[25] ), "+r"( d[26] ), "+r"( d[27] ), "+r"( d[28] ), "+r"( d[29] ), "+r"( d[30] ), "+r"( d[31] )
                : "l"( descA ), "l"( descB ), "r"( accumulate ) : "memory" );
}


__device__ __forceinline__ int wg_row( int i ) { return ( ( threadIdx.x >> 5 ) << 4 ) + ( ( threadIdx.x & 31 ) >> 2 ) + ( i & 2 ) * 4; }
__device__ __forceinline__ int wg_col( int i ) { return ( i >> 2 ) * 8 + ( threadIdx.x & 3 ) * 2 + ( i & 1 ); }
__device__ __forceinline__ void wg_fence()  { asm volatile( "wgmma.fence.sync.aligned;" ::: "memory" ); }
__device__ __forceinline__ void wg_commit() { asm volatile( "wgmma.commit_group.sync.aligned;" ::: "memory" ); }
__device__ __forceinline__ void wg_wait0()  { asm volatile( "wgmma.wait_group.sync.aligned 0;" ::: "memory" ); }
// the compiler does not know that wgmma writes its accumulator registers asynchronously: pinning every register here (before the first MMA of a group
// and after wgmma.wait_group) keeps it from reading, moving or reusing them while MMAs are in flight
template<int R> __device__ __forceinline__ void wg_hold( int (&d)[R] )
{
#pragma unroll
  for( int i = 0; i < R; i++ ) asm volatile( "" : "+r"( d[i] ) :: "memory" );
}
__device__ __forceinline__ void fence_async_smem() { asm volatile( "fence.proxy.async.shared::cta;" ::: "memory" ); }

// N = TU size (16, 32, 64).  KB = bytes of K per operand row = max(32, N); KEEP = N > 32 ? 32 : N (zero-out, DCT-II only at 64).
template<int N>
__global__ void __launch_bounds__( 128 ) fwd_trquant_tc_kernel( const __grid_constant__ TuPar par, const int8_t* __restrict__ trTable, const int32_t* __restrict__ scanTab,
                                                                const int16_t* __restrict__ resi, int n,
                                                                int32_t* __restrict__ coefOut, int16_t* __restrict__ qOut, int32_t* __restrict__ absSumOut,
                                                                int32_t* __restrict__ lastPosOut, uint8_t* __restrict__ needRdoqOut )
{
  constexpr int KB   = N < 32 ? 32 : N;          // operand row length in bytes (K elements, zero padded to a multiple of 32)
  constexpr int NCH  = KB / 16;                  // 16-byte K chunks
  constexpr int TPT  = 128 / N;                  // TUs per 128-row tile
  constexpr int KEEP = N > 32 ? 32 : N;          // kept outputs per dimension for DCT-II
  constexpr int A_BYTES = NCH * 128 * 16;        // one byte-plane operand of 128 rows
  constexpr int B_BYTES = NCH * 32 * 16 * ( KEEP > 32 ? 2 : 1 );   // matrix rows (<= 32 kept rows, padded to 32)
  constexpr int REGION = KEEP * KEEP;            // scanned coefficients per TU

  extern __shared__ __align__( 128 ) unsigned char smemTc[];
  unsigned char* sA   = smemTc;                              // 3 byte planes (stage 1 uses 2)
  unsigned char* sBh  = sA + 3 * A_BYTES;                    // horizontal matrix, rows j < keepW
  unsigned char* sBv  = sBh + B_BYTES;                       // vertical matrix, rows j < keepH
  int32_t*       sCoef = reinterpret_cast<int32_t*>( sBv + B_BYTES );          // [TPT][REGION]
  uint32_t*      sQ    = reinterpret_cast<uint32_t*>( sCoef + TPT * REGION );  // [TPT][N*N/2] int16 pairs (levels)
  int*           sRed  = reinterpret_cast<int*>( sQ + TPT * N * N / 2 );       // [TPT][8]

  const int tid = threadIdx.x;
  const int keepW = par.keepW, keepH = par.keepH;            // == KEEP for DCT-II; 16 for DST-VII/DCT-VIII at 32

  // ---- one-time set-up: matrices in canonical layout
  // B[chunk c][row j (0..31)][16 B] = T[j][16c .. 16c+15], zero beyond N (K padding) and beyond the kept rows
  for( int i = tid; i < NCH * 32 * 16; i += 128 )
  {
    const int c = i / ( 32 * 16 ), r = ( i / 16 ) % 32, b = i % 16, k = c * 16 + b;
    sBh[i] = ( r < keepW && k < N ) ? (unsigned char) trTable[par.offH + r * N + k] : 0;
    sBv[i] = ( r < keepH && k < N ) ? (unsigned char) trTable[par.offV + r * N + k] : 0;
  }
  __syncthreads();

  // the N operand is padded to 32 columns for every TU size (rows >= keep are zero)
  const uint32_t aAddr = smem_u32( sA ), bhAddr = smem_u32( sBh ), bvAddr = smem_u32( sBv );
  const int numTiles = ( n + TPT - 1 ) / TPT;
  const int r1 = par.s1 > 0 ? 1 << ( par.s1 - 1 ) : 0, r2 = 1 << ( par.s2 - 1 );
  const int tuInTile = tid / N, rowInTu = tid % N;
  const int32_t* inv = scanTab + par.scanOff;

  for( int tile = blockIdx.x; tile < numTiles; tile += gridDim.x )
  {
    const int tu = tile * TPT + tuInTile;
    const bool live = tu < n;
    // ---- stage-1 A operand: thread = stacked row; byte planes r0 = r & 127, r1 = r >> 7
    {
      uint32_t w0[KB / 4], w1[KB / 4];
#pragma unroll
      for( int i = 0; i < KB / 4; i++ ) { w0[i] = 0; w1[i] = 0; }
      if( live )
      {
        const uint4* src = reinterpret_cast<const uint4*>( resi + ( (size_t) tu * N + rowInTu ) * N );
#pragma unroll
        for( int v = 0; v < N / 8; v++ )
        {
          const uint4 q = __ldg( src + v );
          const uint32_t ww[4] = { q.x, q.y, q.z, q.w };
#pragma unroll
          for( int j = 0; j < 4; j++ )
          {
            const int e0 = lo16( ww[j] ), e1 = hi16( ww[j] );
            const int k = v * 8 + 2 * j;                     // element index of e0
            w0[k / 4] |= (uint32_t)( e0 & 127 ) << ( 8 * ( k & 3 ) );        w0[( k + 1 ) / 4] |= (uint32_t)( e1 & 127 ) << ( 8 * ( ( k + 1 ) & 3 ) );
            w1[k / 4] |= (uint32_t)( ( e0 >> 7 ) & 255 ) << ( 8 * ( k & 3 ) ); w1[( k + 1 ) / 4] |= (uint32_t)( ( e1 >> 7 ) & 255 ) << ( 8 * ( ( k + 1 ) & 3 ) );
          }
        }
      }
#pragma unroll
      for( int c = 0; c < NCH; c++ )
      {
        *reinterpret_cast<uint4*>( sA + 0 * A_BYTES + ( c * 128 + tid ) * 16 ) = make_uint4( w0[4*c], w0[4*c+1], w0[4*c+2], w0[4*c+3] );
        *reinterpret_cast<uint4*>( sA + 1 * A_BYTES + ( c * 128 + tid ) * 16 ) = make_uint4( w1[4*c], w1[4*c+1], w1[4*c+2], w1[4*c+3] );
      }
      for( int i = tid; i < TPT * 8; i += 128 ) sRed[i] = 0;
    }
    fence_async_smem();
    __syncthreads();
    // ---- stage-1 MMAs: D_p[128 x 32] (d[half][p]) = A_p[128 x KB] * Bh^T, p = 0,1
    int d[2][2][16];
    wg_hold( d[0][0] ); wg_hold( d[0][1] ); wg_hold( d[1][0] ); wg_hold( d[1][1] );
    wg_fence();
#pragma unroll
    for( int h = 0; h < 2; h++ )
#pragma unroll
      for( int p = 0; p < 2; p++ )
#pragma unroll
        for( int ks = 0; ks < KB / 32; ks++ )
        {
          const uint64_t da = gmma_desc_kmajor( aAddr + p * A_BYTES + h * 64 * 16 + ks * 2 * 128 * 16, 128 * 16, 128 );
          const uint64_t db = gmma_desc_kmajor( bhAddr + ks * 2 * 32 * 16, 32 * 16, 128 );
          wgmma_i8<32, true>( d[h][p], da, db, ks > 0 );
        }
    wg_commit();
    wg_wait0();
    wg_hold( d[0][0] ); wg_hold( d[0][1] ); wg_hold( d[1][0] ); wg_hold( d[1][1] );
    __syncthreads();                                     // every MMA has read its A rows
    // ---- stage-1 epilogue: tmp[i][j] = ((d1 << 7) + d0 + r1) >> s1 ; scatter three byte planes, transposed, as stage-2 A
    {
      // zero the three planes first (rows of TUs that keep fewer columns, K padding) -- each thread clears its own rows
#pragma unroll
      for( int p = 0; p < 3; p++ )
#pragma unroll
        for( int c = 0; c < NCH; c++ ) *reinterpret_cast<uint4*>( sA + p * A_BYTES + ( c * 128 + tid ) * 16 ) = make_uint4( 0, 0, 0, 0 );
      __syncthreads();
#pragma unroll
      for( int h = 0; h < 2; h++ )
#pragma unroll
        for( int i = 0; i < 16; i++ )
        {
          // stage-1 row = (TU row / N, row in TU) ; stage-2 stacked row = tuInTile * keepW + j ; K index = row in TU
          const int row = h * 64 + wg_row( i ), j = wg_col( i ), rt = row % N;
          if( j < keepW && tile * TPT + row / N < n )
          {
            const int t = ( ( d[h][1][i] << 7 ) + d[h][0][i] + r1 ) >> par.s1;
            unsigned char* dst = sA + ( ( rt >> 4 ) * 128 + ( row / N ) * keepW + j ) * 16 + ( rt & 15 );
            dst[0 * A_BYTES] = (unsigned char)( t & 127 );
            dst[1 * A_BYTES] = (unsigned char)( ( t >> 7 ) & 127 );
            dst[2 * A_BYTES] = (unsigned char)( ( t >> 14 ) & 255 );
          }
        }
    }
    fence_async_smem();
    __syncthreads();
    // ---- stage-2 MMAs: D_p[128 x 32] = A2_p * Bv^T, p = 0,1,2, one 64-row half at a time
    // ---- stage-2 epilogue: stacked row = (TU t2, column i') ; coef[j'][i'] = ((d2<<14) + (d1<<7) + d0 + r2) >> s2
    {
#pragma unroll
      for( int h = 0; h < 2; h++ )
      {
        int e[3][16];
        wg_hold( e[0] ); wg_hold( e[1] ); wg_hold( e[2] );
        wg_fence();
#pragma unroll
        for( int p = 0; p < 3; p++ )
#pragma unroll
          for( int ks = 0; ks < KB / 32; ks++ )
          {
            const uint64_t da = gmma_desc_kmajor( aAddr + p * A_BYTES + h * 64 * 16 + ks * 2 * 128 * 16, 128 * 16, 128 );
            const uint64_t db = gmma_desc_kmajor( bvAddr + ks * 2 * 32 * 16, 32 * 16, 128 );
            wgmma_i8<32, true>( e[p], da, db, ks > 0 );
          }
        wg_commit();
        wg_wait0();
        wg_hold( e[0] ); wg_hold( e[1] ); wg_hold( e[2] );
#pragma unroll
        for( int i = 0; i < 16; i++ )
        {
          const int row = h * 64 + wg_row( i ), jj = wg_col( i ), t2 = row / keepW, i2 = row - t2 * keepW;
          if( t2 < TPT && tile * TPT + t2 < n && jj < keepH ) sCoef[t2 * REGION + jj * KEEP + i2] = ( ( e[2][i] << 14 ) + ( e[1][i] << 7 ) + e[0][i] + r2 ) >> par.s2;
        }
      }
      // MTS at 32 keeps 16x16 of the 32x32 scan region: clear the rest
      if( keepW < KEEP || keepH < KEEP )
        for( int i = tid; i < TPT * REGION; i += 128 )
        {
          const int rr = ( i % REGION ) / KEEP, cc = i % KEEP;
          if( cc >= keepW || rr >= keepH ) sCoef[i] = 0;
        }
    }
    __syncthreads();

    // ---- quantiser: the same device function as the CUDA-core kernel, team of N threads per TU
    {
      const int tt = rowInTu; constexpr int T = N;
      int32_t*  myCoef = sCoef + tuInTile * REGION;
      int*      myRed  = sRed + tuInTile * 8;
      uint32_t* myQ    = sQ + tuInTile * ( N * N / 2 );
      const int pos = team_quantise<( N == 16 ? 4 : N == 32 ? 5 : 6 ), ( N == 16 ? 4 : N == 32 ? 5 : 6 ), N>( par, myCoef, myQ, myRed, inv, tt, live );
      if( live )
      {
        uint32_t* dst = reinterpret_cast<uint32_t*>( qOut + (size_t) tu * N * N );
        for( int i = tt; i < N * N / 2; i += T ) dst[i] = myQ[i];
        if( coefOut )
        {
          int32_t* cd = coefOut + (size_t) tu * N * N;
          for( int i = tt; i < N * N; i += T )
          {
            const int y = i / N, x = i - y * N;
            cd[i] = ( x < KEEP && y < KEEP ) ? myCoef[y * KEEP + x] : 0;
          }
        }
        if( tt == 0 )
        {
          const int sum = myRed[4];
          if( absSumOut )   absSumOut[tu]   = sum;
          if( lastPosOut )  lastPosOut[tu]  = sum ? myRed[5] - 1 : pos;
          if( needRdoqOut ) needRdoqOut[tu] = (uint8_t) myRed[6];
        }
      }
    }
    __syncthreads();
  }
}

template<int N> static inline size_t trquant_tc_smem()
{
  constexpr int KB = N < 32 ? 32 : N, NCH = KB / 16, TPT = 128 / N, KEEP = N > 32 ? 32 : N;
  return (size_t) 3 * NCH * 128 * 16 + 2 * (size_t) NCH * 32 * 16 + (size_t) TPT * KEEP * KEEP * 4 + (size_t) TPT * N * N * 2 + TPT * 8 * 4 + 256;
}

} // namespace vvb
