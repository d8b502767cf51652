// trquant_tc2_kernels.cuh -- forward 2-D integer transform + quantiser of square TUs 8x8 .. 64x64 on the wgmma tensor cores.
//
// The operands of the MMAs are the RAW little-endian bytes of the values, so no thread ever splits a number into planes:
//   stage 1:  A1[row (tu, y)][2x + b] = byte b of the int16 residual r[y][x]            (a plain 16-byte copy of the residual row)
//             B1lo[j][2x] = Th[j][x], B1lo[j][2x+1] = 0 ; B1hi[j][2x] = 0, B1hi[j][2x+1] = Th[j][x]
//             Dlo = A1(u8) x B1lo^T , Dhi = A1(s8) x B1hi^T : sum_x r * Th[j][x] = Dlo + 256 * Dhi      (low byte unsigned, high byte signed)
//   stage 2:  A2[row (tu, j)][4y + b] = byte b of the int32 tmp[y][j] = (stage 1 + rnd) >> s1   (one 32-bit store per value, transposed on the way)
//             B2p[i][4y + b] = ( b == p ) ? Tv[i][y] : 0 , p = 0, 1 (A read as u8), 2 (A read as s8: |tmp| < 2^23 for every int16 residual)
//             sum_y tmp * Tv[i][y] = D0 + 256 * D1 + 65536 * D2
// The zero entries of the B matrices cost tensor throughput only, which this path has to spare (the kernel is bound by instruction issue, DESIGN.md).
// All sums are int32 like the reference's TCoeff arithmetic (TrQuant_EMT.cpp:1973-2000), no value is rounded: bit exact for every int16 input.
//
// Tile = 128 stage-2 rows = TPT TUs (16 / 8 / 4 / 4 for 8 / 16 / 32 / 64): one CTA of 128 threads = one warpgroup, whose registers hold the accumulators
// (two m64 halves of every 128-row product):
//   A  copy residual rows (pool) or org - pred (planes) into A1            B  2 x M1 MMAs chains, commit, wait
//   C  tmp from the Dlo / Dhi registers -> transposed int32 stores to A2   D  3 MMA chains, commit, wait
//   E  coefficients from the D registers -> staging rows; thread = one coefficient column (tu, j) -> QuantCore (Quant.cpp:132-230) in registers:
//      the KEEP lanes of a TU reduce with redux.sync
//      (last significant position, coefficient-group masks, sums), levels go out as int16 with 2*KEEP-byte row segments per warp store.
// The quantiser restates team_quantise (trquant_kernels.cuh) for EXT = false: plain quantiser, no LFNST limit, no sign-bit hiding, no transform skip.
#pragma once
#include "wgmma.cuh"
#include "trquant_kernels.cuh"

namespace vvb {

// reductions over the KEEP lanes of one TU (aligned lane groups of 8 / 16 lanes, or the warp): xor butterflies for the partial groups so that every lane of the
// warp executes the same shuffles whatever its group does
template<int KEEP> __device__ __forceinline__ int team_max( int v )
{
  if( KEEP >= 32 ) return __reduce_max_sync( 0xffffffffu, v );
#pragma unroll
  for( int d = KEEP / 2; d >= 1; d >>= 1 ) v = max( v, __shfl_xor_sync( 0xffffffffu, v, d ) );
  return v;
}
template<int KEEP> __device__ __forceinline__ int team_sum( int v )
{
  if( KEEP >= 32 ) return __reduce_add_sync( 0xffffffffu, v );
#pragma unroll
  for( int d = KEEP / 2; d >= 1; d >>= 1 ) v += __shfl_xor_sync( 0xffffffffu, v, d );
  return v;
}

template<int N> struct Tc2Shape
{
  static constexpr int KEEP = N > 32 ? 32 : N;             // kept outputs per dimension (DCT-II zero-out at 64; MTS at 32 keeps 16: run-time, rows beyond are zero)
  static constexpr int NMMA = KEEP < 16 ? 16 : KEEP;       // N of the MMAs (M = 128 needs a multiple of 16)
  static constexpr int TPT  = 128 / KEEP;                  // TUs per tile: the stage-2 rows (tu, j) fill the 128 lanes
  static constexpr int ROWS1 = TPT * N, M1 = ROWS1 / 128;  // stage-1 rows (tu, y): 128, or 256 at 64x64 (two M tiles)
  static constexpr int K1 = 2 * N < 32 ? 32 : 2 * N, NCH1 = K1 / 16;
  // A1: one [16-byte K chunk][128 rows][16 B] block per M tile (K chunks 2048 bytes apart also at 64x64)
  static constexpr int LBO1 = 128 * 16, MT1 = NCH1 * LBO1, A1_BYTES = M1 * MT1;
  static constexpr int K2 = 4 * N, NCH2 = K2 / 16;
  // A2: 8-row groups 160 bytes apart, K chunks one group-stride + 16 bytes apart: the transposed 32-bit stores of a warp (32 different y, or TUs x y) hit 32 banks
  static constexpr int SBO2 = 160, LBO2 = 16 * SBO2 + 16, A2_BYTES = NCH2 * LBO2;
  static constexpr bool ALIAS = N >= 64;                   // 64x64: A2 reuses A1's bytes (A1 is dead once the stage-1 MMAs completed).  Smaller TUs keep A1 apart so that
                                                           // the next tile's rows can stream in (cp.async) while the rest of this tile runs; 8x8 also keeps its zero K padding
  static constexpr int A_BYTES = ALIAS ? ( A1_BYTES > A2_BYTES ? A1_BYTES : A2_BYTES ) : A1_BYTES + A2_BYTES;
  static constexpr int BCH = NMMA * 16;                    // K-chunk stride of the B operands
  static constexpr int B1_BYTES = NCH1 * BCH, B2_BYTES = NCH2 * BCH;
  // coefficient rows of phase E, int32, LDS words apart (16-byte aligned, the row reads of a quarter warp hit distinct banks); they reuse A2's bytes, which
  // are dead once the stage-2 MMAs completed, where those are enough (16 .. 64), else they follow the B operands
  static constexpr int LDS = KEEP + 4, STG_BYTES = 128 * LDS * 4;
  static constexpr bool STG_ALIAS = A2_BYTES >= STG_BYTES;
  static constexpr int STG_OFF = STG_ALIAS ? ( ALIAS ? 0 : A1_BYTES ) : A_BYTES + 2 * B1_BYTES + 3 * B2_BYTES;
  static constexpr int SMEM = A_BYTES + 2 * B1_BYTES + 3 * B2_BYTES + ( STG_ALIAS ? 0 : STG_BYTES );
};

// 8 pels of a row segment as 4 packed words, whatever the alignment of the segment (16-byte, 4-byte or odd pel)
__device__ __forceinline__ void tc2_load8( const int16_t* __restrict__ p, uint32_t (&a)[4] )
{
  if( ( reinterpret_cast<uintptr_t>( p ) & 15 ) == 0 ) { const uint4 v = __ldg( reinterpret_cast<const uint4*>( p ) ); a[0] = v.x; a[1] = v.y; a[2] = v.z; a[3] = v.w; }
  else if( ( reinterpret_cast<uintptr_t>( p ) & 3 ) == 0 ) { const uint32_t* w = reinterpret_cast<const uint32_t*>( p ); a[0] = __ldg( w ); a[1] = __ldg( w + 1 ); a[2] = __ldg( w + 2 ); a[3] = __ldg( w + 3 ); }
  else
  {
    const uint32_t* w = reinterpret_cast<const uint32_t*>( p + 1 );
    const uint32_t h0 = (uint16_t) __ldg( p ), w0 = __ldg( w ), w1 = __ldg( w + 1 ), w2 = __ldg( w + 2 ), h7 = (uint16_t) __ldg( p + 7 );
    a[0] = h0 | ( w0 << 16 ); a[1] = __funnelshift_r( w0, w1, 16 ); a[2] = __funnelshift_r( w1, w2, 16 ); a[3] = ( w2 >> 16 ) | ( h7 << 16 );
  }
}
// 8 residuals = org - pred of one row segment as 4 packed words; pred may sit at any pel offset
__device__ __forceinline__ uint4 tc2_resi8( const int16_t* __restrict__ o, const int16_t* __restrict__ p )
{
  uint32_t a[4], b[4];
  tc2_load8( o, a ); tc2_load8( p, b );
  return make_uint4( __vsub2( a[0], b[0] ), __vsub2( a[1], b[1] ), __vsub2( a[2], b[2] ), __vsub2( a[3], b[3] ) );
}

// Host side: the B operands of one (size, horizontal type, vertical type) in the canonical K-major layout [16-byte K chunk][row][16 B], rows >= keep zero.
// tab: the int8 transform table, offH / offV the offsets of the two N x N matrices (row = output index).  Layout of the image: B1lo | B1hi | B2p0 | B2p1 | B2p2.
template<int N> static void tc2_build_b_image( const int8_t* tab, int offH, int offV, int keepW, int keepH, unsigned char* out )
{
  using S = Tc2Shape<N>;
  for( int i = 0; i < S::B1_BYTES; i++ )
  {
    const int c = i / S::BCH, j = ( i / 16 ) % S::NMMA, kb = c * 16 + ( i & 15 ), x = kb >> 1;
    const unsigned char v = ( j < keepW && x < N ) ? (unsigned char) tab[offH + j * N + x] : 0;
    out[i] = ( kb & 1 ) ? 0 : v;
    out[S::B1_BYTES + i] = ( kb & 1 ) ? v : 0;
  }
  unsigned char* o2 = out + 2 * S::B1_BYTES;
  for( int i = 0; i < S::B2_BYTES; i++ )
  {
    const int c = i / S::BCH, r = ( i / 16 ) % S::NMMA, kb = c * 16 + ( i & 15 ), y = kb >> 2, b = kb & 3;
    const unsigned char v = r < keepH ? (unsigned char) tab[offV + r * N + y] : 0;
    o2[i] = b == 0 ? v : 0; o2[S::B2_BYTES + i] = b == 1 ? v : 0; o2[2 * S::B2_BYTES + i] = b == 2 ? v : 0;
  }
}

// MODE 0: compact residual pool (resi); 1: residual formed from resident planes at the block positions; 2: residual = resi[] - resi2[] of two compact pools (org, pred)
template<int N, int MODE>
__global__ void __launch_bounds__( 128, N >= 32 ? 3 : 4 ) fwd_trquant_tc2_kernel( const __grid_constant__ TuPar par, const uint4* __restrict__ bImage, const int32_t* __restrict__ scanTab,
                                                                    const int16_t* __restrict__ resi, const int16_t* __restrict__ resi2,
                                                                    const __grid_constant__ Plane orgPlane, const __grid_constant__ Plane predPlane, const vvb_block* __restrict__ blocks,
                                                                    int n, int32_t* __restrict__ coefOut, int16_t* __restrict__ qOut, int32_t* __restrict__ absSumOut,
                                                                    int32_t* __restrict__ lastPosOut, uint8_t* __restrict__ needRdoqOut )
{
  using S = Tc2Shape<N>;
  constexpr int KEEP = S::KEEP, NMMA = S::NMMA, TPT = S::TPT, M1 = S::M1;
  extern __shared__ __align__( 128 ) unsigned char smemTc2[];
  unsigned char* sA1 = smemTc2;
  unsigned char* sA2 = S::ALIAS ? smemTc2 : smemTc2 + S::A1_BYTES;
  unsigned char* sB1 = smemTc2 + S::A_BYTES;                // lo, hi
  unsigned char* sB2 = sB1 + 2 * S::B1_BYTES;               // p = 0, 1, 2
  int* sStg = reinterpret_cast<int*>( smemTc2 + S::STG_OFF );

  const int tid = threadIdx.x;

  // ---- one-time set-up
  // the five B operands (B1 lo, hi of the horizontal matrix; B2 p = 0, 1, 2 of the vertical one) as the host laid them out (tc2_build_b_image): a straight copy
  for( int i = tid; i < ( 2 * S::B1_BYTES + 3 * S::B2_BYTES ) / 16; i += 128 ) reinterpret_cast<uint4*>( sB1 )[i] = __ldg( bImage + i );
  if( N == 8 ) for( int i = tid; i < S::A1_BYTES / 16; i += 128 ) reinterpret_cast<uint4*>( sA1 )[i] = make_uint4( 0, 0, 0, 0 );    // K padding of the 8x8 rows stays zero
  // stage-2 role of this thread: row (t2, j2) of the tile = column j2 of TU t2.  Down a column the scan position grows with the row (diagonal scan inside a
  // coefficient group, groups in diagonal order), so "last significant position" is "highest significant row" + one table look-up; what stays in registers is the
  // coefficient-group index (scan position >> 4) of each group of four rows
  const int t2 = tid / KEEP, j2 = tid % KEEP;
  const int32_t* invCol = scanTab + par.scanOff + j2;
  int cgIdx[KEEP / 4];
#pragma unroll
  for( int g = 0; g < KEEP / 4; g++ ) cgIdx[g] = __ldg( invCol + 4 * g * KEEP ) >> 4;
  __syncthreads();
  const uint32_t a1Addr = smem_u32( sA1 ), a2Addr = smem_u32( sA2 ), b1Addr = smem_u32( sB1 ), b2Addr = smem_u32( sB2 );
  const int numTiles = ( n + TPT - 1 ) / TPT;
  const int r1 = par.s1 > 0 ? 1 << ( par.s1 - 1 ) : 0, r2 = 1 << ( par.s2 - 1 ), s1 = par.s1, s2 = par.s2;
  // shared-memory descriptors of the four operand families; inside the loops only the start-address field (16-byte units, low word) moves
  const uint64_t dA1 = gmma_desc_kmajor( a1Addr, S::LBO1, 128 ), dB1 = gmma_desc_kmajor( b1Addr, S::BCH, 128 );
  const uint64_t dA2 = gmma_desc_kmajor( a2Addr, S::LBO2, S::SBO2 ), dB2 = gmma_desc_kmajor( b2Addr, S::BCH, 128 );

  // ---- A: residual rows of one tile -> A1 (raw bytes).  Compact pools of TUs up to 32x32 stream in with cp.async (STREAM): the copy of tile k+1 is issued as soon as
  //      the stage-1 MMAs of tile k have consumed A1 and lands while the rest of tile k runs.
  constexpr bool PLANES = MODE == 1;
  constexpr bool STREAM = MODE == 0 && !S::ALIAS;
  auto load_tile = [&]( int tile )
  {
#pragma unroll
    for( int m = 0; m < M1; m++ )
    {
      const int r = m * 128 + tid, tl = r / N, y = r % N, tu = tile * TPT + tl;
      const bool live = tu < n;
      if( PLANES )
      {
        const vvb_block blk = blocks[live ? tu : 0];
        const int16_t* o = orgPlane.origin + (ptrdiff_t)( blk.y + y ) * orgPlane.stride + blk.x;
        const int16_t* p = predPlane.origin + (ptrdiff_t)( blk.y + blk.start_y + y ) * predPlane.stride + blk.x + blk.start_x;
#pragma unroll
        for( int c = 0; c < N / 8; c++ )
          *reinterpret_cast<uint4*>( sA1 + m * S::MT1 + c * S::LBO1 + tid * 16 ) = live ? tc2_resi8( o + 8 * c, p + 8 * c ) : make_uint4( 0, 0, 0, 0 );
      }
      else if( MODE == 2 )
      {
        const size_t off = ( (size_t)( live ? tu : 0 ) * N + y ) * N;
        const uint4* so = reinterpret_cast<const uint4*>( resi + off ); const uint4* sp = reinterpret_cast<const uint4*>( resi2 + off );
#pragma unroll
        for( int c = 0; c < N / 8; c++ )
        {
          uint4 d = make_uint4( 0, 0, 0, 0 );
          if( live ) { const uint4 a = __ldg( so + c ), b = __ldg( sp + c ); d = make_uint4( __vsub2( a.x, b.x ), __vsub2( a.y, b.y ), __vsub2( a.z, b.z ), __vsub2( a.w, b.w ) ); }
          *reinterpret_cast<uint4*>( sA1 + m * S::MT1 + c * S::LBO1 + tid * 16 ) = d;
        }
      }
      else if( STREAM )
      {
        const int16_t* src = resi + ( (size_t)( live ? tu : 0 ) * N + y ) * N;
        const uint32_t bytes = live ? 16u : 0u;                                  // 0: the 16 bytes are zero-filled
#pragma unroll
        for( int c = 0; c < N / 8; c++ )
          asm volatile( "cp.async.cg.shared.global [%0], [%1], 16, %2;" :: "r"( a1Addr + m * S::MT1 + c * S::LBO1 + tid * 16 ), "l"( src + 8 * c ), "r"( bytes ) : "memory" );
      }
      else
      {
        const uint4* src = reinterpret_cast<const uint4*>( resi + ( (size_t)( live ? tu : 0 ) * N + y ) * N );
#pragma unroll
        for( int c = 0; c < N / 8; c++ )
          *reinterpret_cast<uint4*>( sA1 + m * S::MT1 + c * S::LBO1 + tid * 16 ) = live ? __ldg( src + c ) : make_uint4( 0, 0, 0, 0 );
      }
    }
    if( STREAM ) asm volatile( "cp.async.commit_group;" ::: "memory" );
  };
  if( STREAM && (int) blockIdx.x < numTiles ) load_tile( blockIdx.x );

  for( int tile = blockIdx.x; tile < numTiles; tile += gridDim.x )
  {
    if( STREAM ) asm volatile( "cp.async.wait_group 0;" ::: "memory" );
    else load_tile( tile );
    fence_async_smem();
    __syncthreads();
    // ---- B: stage-1 MMAs, both 64-row halves of one M tile at a time (Dlo: A1 read as u8, Dhi: as s8); tmp = ( Dlo + 256 * Dhi + rnd ) >> s1 in registers
    // every M tile has accumulator arrays of its own: chains that rewrite the registers another chain's results were just read from lose the first
    // chain (ptxas drops it)
    int tv[M1][2][NMMA / 2];
#pragma unroll
    for( int m = 0; m < M1; m++ )
    {
      int lo[M1][2][NMMA / 2], hi[M1][2][NMMA / 2];
      wg_fence();
#pragma unroll
      for( int h = 0; h < 2; h++ )
#pragma unroll
        for( int ks = 0; ks < S::K1 / 32; ks++ )
        {
          const uint64_t da = dA1 + (uint64_t)( ( m * S::MT1 + h * 64 * 16 + ks * 2 * S::LBO1 ) >> 4 );
          wgmma_i8<NMMA, false>( lo[m][h], da, dB1 + (uint64_t)( ( ks * 2 * S::BCH ) >> 4 ), ks > 0 );
          wgmma_i8<NMMA, true>( hi[m][h], da, dB1 + (uint64_t)( ( S::B1_BYTES + ks * 2 * S::BCH ) >> 4 ), ks > 0 );
        }
      wg_commit();
      wg_wait0();
      wg_hold( lo[m][0] ); wg_hold( lo[m][1] ); wg_hold( hi[m][0] ); wg_hold( hi[m][1] );
#pragma unroll
      for( int h = 0; h < 2; h++ )
#pragma unroll
        for( int i = 0; i < NMMA / 2; i++ ) tv[m][h][i] = ( ( hi[m][h][i] << 8 ) + lo[m][h][i] + r1 ) >> s1;
    }
    __syncthreads();                                     // A1 is consumed: the next tile may stream in, A2 may overwrite it (64x64)
    if( STREAM && tile + (int) gridDim.x < numTiles ) load_tile( tile + gridDim.x );
    // ---- C: tmp of stage-1 row r = (tu, y), column j stored transposed as the raw int32 bytes of A2 row (tu, j), K bytes 4y .. 4y+3
#pragma unroll
    for( int m = 0; m < M1; m++ )
#pragma unroll
      for( int h = 0; h < 2; h++ )
#pragma unroll
        for( int i = 0; i < NMMA / 2; i++ )
        {
          const int r = m * 128 + h * 64 + wg_row( i ), j = wg_col( i ), tl = r / N, y = r % N;
          if( j < KEEP )
            *reinterpret_cast<int*>( sA2 + ( y >> 2 ) * S::LBO2 + ( tl * KEEP / 8 + ( j >> 3 ) ) * S::SBO2 + ( y & 3 ) * 4 + ( j & 7 ) * 16 ) = tv[m][h][i];
        }
    fence_async_smem();
    __syncthreads();
    // ---- D: stage-2 MMAs (D0, D1: A2 read as u8, D2: as s8); c = ( D0 + 256 * D1 + 65536 * D2 + rnd ) >> s2 -> staging row (t2, j2), column i
    {
      int d0[2][NMMA / 2], d1[2][NMMA / 2], d2[2][NMMA / 2];
      wg_hold( d0[0] ); wg_hold( d0[1] ); wg_hold( d1[0] ); wg_hold( d1[1] ); wg_hold( d2[0] ); wg_hold( d2[1] );
      wg_fence();
#pragma unroll
      for( int h = 0; h < 2; h++ )
#pragma unroll
        for( int ks = 0; ks < S::K2 / 32; ks++ )
        {
          const uint64_t da = dA2 + (uint64_t)( ( h * 8 * S::SBO2 + ks * 2 * S::LBO2 ) >> 4 );
          wgmma_i8<NMMA, false>( d0[h], da, dB2 + (uint64_t)( ( 0 * S::B2_BYTES + ks * 2 * S::BCH ) >> 4 ), ks > 0 );
          wgmma_i8<NMMA, false>( d1[h], da, dB2 + (uint64_t)( ( 1 * S::B2_BYTES + ks * 2 * S::BCH ) >> 4 ), ks > 0 );
          wgmma_i8<NMMA, true>( d2[h], da, dB2 + (uint64_t)( ( 2 * S::B2_BYTES + ks * 2 * S::BCH ) >> 4 ), ks > 0 );
        }
      wg_commit();
      wg_wait0();
      wg_hold( d0[0] ); wg_hold( d0[1] ); wg_hold( d1[0] ); wg_hold( d1[1] ); wg_hold( d2[0] ); wg_hold( d2[1] );
      if( S::STG_ALIAS ) __syncthreads();                // the staging rows overwrite A2
#pragma unroll
      for( int h = 0; h < 2; h++ )
#pragma unroll
        for( int i = 0; i < NMMA / 2; i++ )
        {
          const int r = h * 64 + wg_row( i ), c = wg_col( i );
          if( c < KEEP ) sStg[r * S::LDS + c] = ( ( d2[h][i] << 16 ) + ( d1[h][i] << 8 ) + d0[h][i] + r2 ) >> s2;
        }
    }
    __syncthreads();
    // ---- E: coefficient column (t2, j2) = staging row tid, then QuantCore in registers
    {
      const int tu = tile * TPT + t2;
      const bool live = tu < n;
      int cf[KEEP];
#pragma unroll
      for( int c = 0; c < KEEP / 4; c++ )
      {
        const int4 v = reinterpret_cast<const int4*>( sStg + tid * S::LDS )[c];
        cf[4 * c] = v.x; cf[4 * c + 1] = v.y; cf[4 * c + 2] = v.z; cf[4 * c + 3] = v.w;
      }
      // pass 1 (Quant.cpp:160-208) at coefficient-group granularity: the group of the last non-zero coefficient, the highest group above the threshold, the RDOQ
      // pre-check (largest magnitude).  The group index grows down the column, so the last assignment is the maximum.
      int amax = 0, cgMax = 0, initCg = 0;
      const int useThres = par.useThres;
#pragma unroll
      for( int g = 0; g < KEEP / 4; g++ )
      {
        const int m4 = max( max( abs( cf[4 * g] ), abs( cf[4 * g + 1] ) ), max( abs( cf[4 * g + 2] ), abs( cf[4 * g + 3] ) ) );
        amax = max( amax, m4 );
        if( m4 ) initCg = cgIdx[g];
        if( m4 > useThres ) cgMax = cgIdx[g];
      }
      initCg = team_max<KEEP>( initCg );
      cgMax  = team_max<KEEP>( cgMax );
      amax   = team_max<KEEP>( amax );
      // Quant.cpp:182-208: the groups above the threshold all hold a non-zero coefficient, hence lie at or below the last one: the highest of them decides.
      // Trimmed: the final position is the end of group cgMax (15 when cgMax == 0) and whole groups beyond it drop out (scan position <= pos <=> group <= pos >> 4).
      const bool trimmed = initCg >= 1 && cgMax != initCg;
      if( live && coefOut )                                 // the transform coefficients as xT leaves them (before the trimming below)
      {
        int32_t* cd = coefOut + (size_t) tu * N * N + j2;
#pragma unroll
        for( int i = 0; i < KEEP; i++ ) cd[i * N] = cf[i];
      }
      if( trimmed )
      {
#pragma unroll
        for( int g = 0; g < KEEP / 4; g++ )
          if( cgIdx[g] > cgMax ) { cf[4 * g] = 0; cf[4 * g + 1] = 0; cf[4 * g + 2] = 0; cf[4 * g + 3] = 0; }
      }
      // pass 2 (Quant.cpp:211-227)
      int sum = 0, hiQ = -1;
      const int qbits = par.qbits; const unsigned scale = (unsigned) par.scale, add32 = par.add32;
      int16_t* qd = qOut + (size_t)( live ? tu : 0 ) * N * N + j2;
      if( par.q32 && (unsigned) amax < 32768u && ( ( (unsigned) amax * scale + add32 ) >> qbits ) <= 32767u )
      {
        // -(( |c| * scale + add ) >> qbits) == ( c * scale + 2^qbits - 1 - add ) >> qbits for c < 0 (arithmetic shift): one multiply-add per level, no clipping needed
        const int addP = (int) add32, addN = (int)( ( 1u << qbits ) - 1u - add32 );
#pragma unroll
        for( int i = 0; i < KEEP; i++ )
        {
          const int c = cf[i];
          const int v = ( c * (int) scale + ( c < 0 ? addN : addP ) ) >> qbits;
          sum += abs( v );
          if( v ) hiQ = i;
          if( live ) qd[i * N] = (int16_t) v;
        }
      }
      else
      {
#pragma unroll
        for( int i = 0; i < KEEP; i++ )
        {
          const long long ac = (long long) abs( cf[i] );
          const int mag = (int)( ( ac * par.scale + par.add ) >> qbits );
          sum += mag;
          const int v = cf[i] < 0 ? max( -32768, -mag ) : min( 32767, mag );
          if( v ) hiQ = i;
          if( live ) qd[i * N] = (int16_t) v;
        }
      }
      int lastQ = hiQ >= 0 ? __ldg( invCol + hiQ * KEEP ) + 1 : 0;
      sum   = team_sum<KEEP>( sum );
      lastQ = team_max<KEEP>( lastQ );
      int pos = cgMax * 16 + 15;                            // the final scan position is only reported when every level is zero (Quant.cpp:830)
      const bool exact = sum == 0 && !trimmed;              // ... and then, untrimmed, it is the exact position of the last non-zero coefficient
      if( __any_sync( 0xffffffffu, exact ) )                // rare; the whole warp walks through so that the lane groups reduce together
      {
        int hiNZ = -1;
#pragma unroll
        for( int i = 0; i < KEEP; i++ ) if( cf[i] ) hiNZ = i;
        const int lastNZ = team_max<KEEP>( hiNZ >= 0 ? __ldg( invCol + hiNZ * KEEP ) : 0 );
        if( exact ) pos = lastNZ;
      }
      if( live )
      {
        if( j2 == 0 )
        {
          if( absSumOut )   absSumOut[tu]   = sum;
          if( lastPosOut )  lastPosOut[tu]  = sum ? lastQ - 1 : pos;          // Quant.cpp:806-816, :830
          if( needRdoqOut ) needRdoqOut[tu] = (uint8_t)( (unsigned) amax >= par.rdoqThr );
        }
      }
      if( N > KEEP )                                                            // 64x64: the zeroed-out three quarters of the level (and coefficient) blocks
      {
        // per TU: rows 0..31 columns 32..63 (4 x 16 B per row) and rows 32..63 (8 x 16 B per row) = 128 + 256 vectors; 128 threads x TPT TUs
        for( int t = 0; t < TPT; t++ )
        {
          const int tz = tile * TPT + t;
          if( tz >= n ) break;
          uint4* qz = reinterpret_cast<uint4*>( qOut + (size_t) tz * N * N );
          for( int v = tid; v < 384; v += 128 )
          {
            const int idx = v < 128 ? ( v >> 2 ) * 8 + 4 + ( v & 3 ) : 256 + ( v - 128 );
            qz[idx] = make_uint4( 0, 0, 0, 0 );
          }
          if( coefOut )
          {
            uint4* cz = reinterpret_cast<uint4*>( coefOut + (size_t) tz * N * N );
            for( int v = tid; v < 768; v += 128 )
            {
              const int idx = v < 256 ? ( v >> 3 ) * 16 + 8 + ( v & 7 ) : 512 + ( v - 256 );
              cz[idx] = make_uint4( 0, 0, 0, 0 );
            }
          }
        }
      }
    }
    __syncthreads();
  }
}

} // namespace vvb
