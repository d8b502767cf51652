// mctf_affine_kernels.cuh -- MCTF block-matching errors and the affine motion estimation's gradient step for sm_90a.
//
// MCTF: MCTF::motionErrorLuma (CommonLib/MCTF.cpp:1099-1164) -> motionErrorLumaInt (:122-145),
//       motionErrorLumaFrac6 (:147-203), motionErrorLumaFrac4 (:205-257); filter tables :72-110.
// Affine: xHorizontalSobelFilter / xVerticalSobelFilter / xEqualCoeffComputer (CommonLib/AffineGradientSearch.cpp:84-190), single-block
//         (sobel_kernel, equal_coeff_kernel) and one block per CTA over a list of blocks (affine_eq_batch_kernel, SURVEY row a16).
#pragma once
#include "common.cuh"
#include "packed_filter.cuh"

namespace vvb {

// MCTF interpolation filters (constants of the algorithm, CommonLib/MCTF.cpp:72-110): row = 1/16-pel phase
__device__ __constant__ short c_mctfF8[16][8] = {
  {0,0,0,64,0,0,0,0},{0,1,-3,64,4,-2,0,0},{0,1,-6,62,9,-3,1,0},{0,2,-8,60,14,-5,1,0},{0,2,-9,57,19,-7,2,0},{0,3,-10,53,24,-8,2,0},
  {0,3,-11,50,29,-9,2,0},{0,3,-11,44,35,-10,3,0},{0,1,-7,38,38,-7,1,0},{0,3,-10,35,44,-11,3,0},{0,2,-9,29,50,-11,3,0},{0,2,-8,24,53,-10,3,0},
  {0,2,-7,19,57,-9,2,0},{0,1,-5,14,60,-8,2,0},{0,1,-3,9,62,-6,1,0},{0,0,-2,4,64,-3,1,0} };
__device__ __constant__ short c_mctfF4[16][4] = {
  {0,64,0,0},{-2,62,4,0},{-2,58,10,-2},{-4,56,14,-2},{-4,54,16,-2},{-6,52,20,-2},{-6,46,28,-4},{-4,42,30,-4},
  {-4,36,36,-4},{-4,30,42,-4},{-4,28,46,-6},{-2,20,52,-6},{-2,16,54,-4},{-2,14,56,-4},{-2,10,58,-2},{0,4,62,-2} };

#define MCTF_WARPS 4

// ---------------------------------------------------------------------------------------------------------------------------------
// mctf_error_packed_kernel: one warp per candidate (int32 error exactly as the reference, no early exit: besterror = INT_MAX as in
// vvenc_unit_test.cpp:1552); the source region and the horizontally filtered rows live in the warp's slice of shared
// memory, both filter passes run on IDP.2A.  Pel pairs are packed along x for the horizontal pass and along y (row pairs) for the
// vertical pass; a 6-tap output whose first pel sits in the low half of a word takes 3 IDP.2A ("E"), one that starts in the high half
// takes 4 with zero-padded taps ("O").  The 4-tap filters are embedded as (0, t0, t1, t2, t3, 0): same pels, same sums.
// Taps fit int8 (|t| <= 64), pels and clipped intermediates fit int16.  A lane's partial sum covers at most 128 pels and fits int32; the warp sum is
// reduced unsigned, which is exact up to 64 x 64 pels at 10 bits (4096 * 1023^2 < 2^32), and the kernels saturate it to 0x7fffffff where they store int32.
// The reference's sums are int32 too, but its early exit (MCTF.cpp:138, 196, 250) returns before they can wrap; a saturated error loses every strict
// `error < best.error` against a finite best, as the reference's partial sum does.
struct MctfSmem { int regionPitch, regionWords, t2Words, warpWords; };
__host__ __device__ inline MctfSmem mctf_smem( int maxW, int maxH )
{
  MctfSmem m;
  m.regionPitch = maxW / 2 + 4;                                  // words per region row: w + 5 pels + alignment, rounded up
  m.regionWords = ( maxH + 6 ) * m.regionPitch;                  // h + 5 rows, + 1 so that the last row pair is addressable
  m.t2Words     = ( ( maxH + 6 ) / 2 ) * maxW;                   // row pairs x w
  m.warpWords   = m.regionWords + m.t2Words;
  return m;
}
__host__ __device__ inline MctfSmem mctf_smem( int maxDim ) { return mctf_smem( maxDim, maxDim ); }

__device__ __forceinline__ int32_t mctf_sat32( unsigned long long e ) { return (int32_t)( e < 0x7fffffffull ? e : 0x7fffffffull ); }

// the taps of 1/16-pel phase `phase` as a 6-tap filter over pels x-2 .. x+3, packed: the 8-tap set without its zero ends, or the 4-tap set
// embedded as (0, t0, t1, t2, t3, 0)
__device__ __forceinline__ PackedTaps<6> mctf_taps6( int tap4, int phase )
{
  int f[6];
#pragma unroll
  for( int t = 0; t < 6; t++ ) f[t] = tap4 ? ( t >= 1 && t <= 4 ? c_mctfF4[phase][t - 1] : 0 ) : c_mctfF8[phase][t + 1];
  return pack_taps<6>( f );
}

// a filter pass's rounding with the clip to the pel range (motionErrorLumaFrac6/4 after both passes, applyFrac after the second)
__device__ __forceinline__ int mctf_round_clip( int v, int maxv ) { return max( min( ( v + 32 ) >> 6, maxv ), 0 ); }

// motionErrorLuma of one candidate by one warp (no early exit, unsaturated); region / t2: the warp's slices of shared memory (mctf_smem); every lane returns the error
__device__ __forceinline__ unsigned mctf_warp_error( const Plane& orgPlane, const Plane& refPlane, const vvb_mctf_cand& c, int tap4, const MctfSmem& L, uint32_t* region, uint32_t* t2, int lane )
{
  const int PW = L.regionPitch;
  const int maxv = ( 1 << refPlane.bitDepth ) - 1;
  const int w = c.w, h = c.h;
  int dx = c.mvx, dy = c.mvy;
  const int fx = dx & 15, fy = dy & 15;
  const int16_t* org = orgPlane.origin + (ptrdiff_t) c.y * orgPlane.stride + c.x;
  const int hw = w >> 1;
  const float invHw = 1.0f / (float) hw, invW = 1.0f / (float) w;
  int err = 0;
  if( ( fx | fy ) == 0 )
  {
    dx /= 16; dy /= 16;                                  // MCTF.cpp:1121-1122 (C division, truncating)
    const int16_t* buf = refPlane.origin + (ptrdiff_t)( c.y + dy ) * refPlane.stride + c.x + dx;
    for( int i = lane; i < w * h; i += 32 )
    {
      const int y = div_rcp( i, invW ), x = i - y * w;
      const int d = (int) __ldg( org + (ptrdiff_t) y * orgPlane.stride + x ) - (int) __ldg( buf + (ptrdiff_t) y * refPlane.stride + x );
      err += d * d;
    }
  }
  else
  {
    dx >>= 4; dy >>= 4;                                  // MCTF.cpp:1136-1137 / :1151-1152 (arithmetic shift)
    const PackedTaps<6> X = mctf_taps6( tap4, fx ), Y = mctf_taps6( tap4, fy );
    // ---- stage the source region: rows y-2 .. y+h+3 (the last one only pairs up the row count), pels from the even pel at or below x-2
    const int rowsP = ( h + 6 ) & ~1;
    __syncwarp();
    const int o = stage_pel_pairs( region, PW, refPlane.origin + (ptrdiff_t)( c.y + dy - 2 ) * refPlane.stride + c.x + dx - 2, refPlane.stride, w + 5, rowsP, lane, 32 );
    __syncwarp();
    // ---- horizontal pass: item = (row pair rp, column pair cp) -> t2[rp][x], t2[rp][x+1] = packed ( row 2rp, row 2rp+1 )
    const int nRp = rowsP >> 1;
    for( int i = lane; i < nRp * hw; i += 32 )
    {
      const int rp = div_rcp( i, invHw ), cp = i - rp * hw;
      const uint32_t* ra = region + ( 2 * rp ) * PW + cp;
      int2 ha, hb;
      filter_row_pair<6>( ra, ra + PW, o, X, ha, hb );
      uint2 pk;
      pk.x = (uint32_t) mctf_round_clip( ha.x, maxv ) | ( (uint32_t) mctf_round_clip( hb.x, maxv ) << 16 );
      pk.y = (uint32_t) mctf_round_clip( ha.y, maxv ) | ( (uint32_t) mctf_round_clip( hb.y, maxv ) << 16 );
      *reinterpret_cast<uint2*>( t2 + rp * w + 2 * cp ) = pk;
    }
    __syncwarp();
    // ---- vertical pass + SSE: item = (output row pair yp, column x): rows 2yp (E on pairs yp..yp+2) and 2yp+1 (O on pairs yp..yp+3)
    for( int i = lane; i < ( h >> 1 ) * w; i += 32 )
    {
      const int yp = div_rcp( i, invW ), x = i - yp * w;
      const uint32_t* tp = t2 + yp * w + x;
      const uint32_t p[4] = { tp[0], tp[w], tp[2 * w], tp[3 * w] };
      const int2 v = filter_pair<6>( p, false, Y );
      const int16_t* op = org + (ptrdiff_t)( 2 * yp ) * orgPlane.stride + x;
      const int d0 = mctf_round_clip( v.x, maxv ) - (int) __ldg( op ), d1 = mctf_round_clip( v.y, maxv ) - (int) __ldg( op + orgPlane.stride );
      err += d0 * d0 + d1 * d1;
    }
  }
  return __reduce_add_sync( 0xffffffffu, (unsigned) err );
}

__global__ void __launch_bounds__( MCTF_WARPS * 32 ) mctf_error_packed_kernel( const __grid_constant__ Plane orgPlane, const __grid_constant__ Plane refPlane,
                                                                               const vvb_mctf_cand* __restrict__ cands, int n, int tap4, int maxDim, int32_t* __restrict__ out )
{
  extern __shared__ __align__( 16 ) uint32_t sMctf[];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const MctfSmem L = mctf_smem( maxDim );
  uint32_t* region = sMctf + warp * L.warpWords;
  uint32_t* t2     = region + L.regionWords;
  const int warpsPerGrid = gridDim.x * MCTF_WARPS;
  for( int ci = blockIdx.x * MCTF_WARPS + warp; ci < n; ci += warpsPerGrid )
  {
    const vvb_mctf_cand c = cands[ci];
    if( c.w > maxDim || c.h > maxDim || ( ( c.w | c.h ) & 1 ) ) { if( lane == 0 ) out[ci] = -1; continue; }     // outside the promised geometry
    const unsigned err = mctf_warp_error( orgPlane, refPlane, c, tap4, L, region, t2, lane );
    if( lane == 0 ) out[ci] = mctf_sat32( err );
  }
}

// ---------------------------------------------------------------------------------------------------------------------------------
// Grid search: all (2r+1)^2 candidates  centre + (i - r, j - r) * step  (1/16 pel) of one block in one CTA -- the loops of
// MCTF::estimateLumaLn (CommonLib/MCTF.cpp:1218-1287: integer grid step 16 range 5/8, then 7x7 step 4, 3x3 step 2, 3x3 step 1).
// The source window is staged once per block; for every distinct horizontal vector the horizontally filtered rows are computed once
// (packed as row pairs; as many grid columns per pass as fit 40 KB of shared memory) and shared by the 2r+1 candidates above it; a thread owns output positions (row pair, column), so the original
// pels are read once and each candidate's error is reduced with one REDUX + one shared atomic per warp.  Same arithmetic as
// mctf_error_packed_kernel (IDP.2A, int32 sums, clip after each pass): results equal motionErrorLuma for every candidate.
struct MctfGridSmem { int winPitch, winWords, colWords, G, hWords, orgWords, errWords, tapOff, tapWords, total; };
__host__ __device__ inline MctfGridSmem mctf_grid_smem( int maxDim, int step, int radius )
{
  const int span = ( ( 2 * radius * step + 15 ) >> 4 ) + 1;      // upper bound of (max - min) integer displacement
  const int K1 = 2 * radius + 1;
  MctfGridSmem m;
  const int rows = ( maxDim + 6 + span + 1 ) & ~1;
  m.winPitch = ( maxDim + 5 + span + 2 + 1 ) >> 1;
  m.winWords = rows * m.winPitch;
  m.colWords = ( rows >> 1 ) * maxDim;                           // filtered rows of one horizontal vector: row pairs x w
  m.G        = 10240 / m.colWords < 1 ? 1 : ( 10240 / m.colWords > K1 ? K1 : 10240 / m.colWords );   // grid columns per pass (up to 40 KB)
  m.hWords   = m.G * m.colWords;
  m.orgWords = ( maxDim >> 1 ) * maxDim;
  m.errWords = ( K1 * K1 + 1 ) & ~1;
  m.tapWords = 8 * K1;                                           // packed taps per grid column (x) and row (y)
  m.tapOff   = ( m.winWords + m.hWords + m.orgWords + m.errWords + 3 ) & ~3;   // PackedTaps<6> entries: 16-byte aligned
  m.total    = m.tapOff + m.tapWords;
  return m;
}

__global__ void __launch_bounds__( 256 ) mctf_grid_kernel( const __grid_constant__ Plane orgPlane, const __grid_constant__ Plane refPlane,
                                                           const vvb_mctf_cand* __restrict__ blocks, int n, int step, int radius, int tap4, int maxDim,
                                                           int32_t* __restrict__ out )
{
  extern __shared__ __align__( 16 ) uint32_t sGrid[];
  const MctfGridSmem L = mctf_grid_smem( maxDim, step, radius );
  uint32_t* win  = sGrid;
  uint32_t* hbuf = win + L.winWords;
  uint32_t* orgP = hbuf + L.hWords;
  unsigned* sErr = orgP + L.orgWords;                                       // exact up to 64 x 64 pels at 10 bits (4096 * 1023^2 < 2^32)
  PackedTaps<6>* sTap = reinterpret_cast<PackedTaps<6>*>( sGrid + L.tapOff );   // [2 * K1]: x columns, then y rows
  const int tid = threadIdx.x, T = blockDim.x;
  const int K1 = 2 * radius + 1, K = K1 * K1;
  const int maxv = ( 1 << refPlane.bitDepth ) - 1;
  const int PW = L.winPitch;

  for( int b = blockIdx.x; b < n; b += gridDim.x )
  {
    const vvb_mctf_cand blk = blocks[b];
    const int w = blk.w, h = blk.h;
    if( w > maxDim || h > maxDim || ( ( w | h ) & 1 ) ) { for( int k = tid; k < K; k += T ) out[(size_t) b * K + k] = -1; continue; }
    const int hw = w >> 1, hh = h >> 1;
    const float invHw = 1.0f / (float) hw, invW = 1.0f / (float) w;
    const int dxMin = ( blk.mvx - radius * step ) >> 4, dyMin = ( blk.mvy - radius * step ) >> 4;
    const int dxMax = ( blk.mvx + radius * step ) >> 4, dyMax = ( blk.mvy + radius * step ) >> 4;
    const int rowsP = ( h + 6 + ( dyMax - dyMin ) + 1 ) & ~1;
    // ---- stage the window (rows y+dyMin-2 .., pels from the even pel at or below x+dxMin-2), the original block as row pairs, clear the errors
    __syncthreads();
    const int o = stage_pel_pairs( win, PW, refPlane.origin + (ptrdiff_t)( blk.y + dyMin - 2 ) * refPlane.stride + blk.x + dxMin - 2, refPlane.stride,
                                   w + 5 + ( dxMax - dxMin ), rowsP, tid, T );
    {
      const int16_t* org = orgPlane.origin + (ptrdiff_t) blk.y * orgPlane.stride + blk.x;
      for( int i = tid; i < hh * w; i += T )
      {
        const int yp = div_rcp( i, invW ), x = i - yp * w;
        const int16_t* op = org + (ptrdiff_t)( 2 * yp ) * orgPlane.stride + x;
        orgP[i] = (uint32_t)(uint16_t) __ldg( op ) | ( (uint32_t)(uint16_t) __ldg( op + orgPlane.stride ) << 16 );
      }
    }
    for( int k = tid; k < K; k += T ) sErr[k] = 0;
    __syncthreads();
    // packed taps of every grid column / row (phase = vector & 15)
    for( int k = tid; k < 2 * K1; k += T )
    {
      const int mv = ( k < K1 ? blk.mvx : blk.mvy ) + ( ( k < K1 ? k : k - K1 ) - radius ) * step;
      sTap[k] = mctf_taps6( tap4, mv & 15 );
    }
    __syncthreads();
    const int perCol = ( rowsP >> 1 ) * hw;
    const float invPerCol = 1.0f / (float) perCol;
    for( int i0 = 0; i0 < K1; i0 += L.G )
    {
      const int gcount = min( L.G, K1 - i0 );
      // ---- horizontal pass for gcount grid columns: item = (column, row pair, column pair)
      for( int it = tid; it < gcount * perCol; it += T )
      {
        const int g = div_rcp( it, invPerCol ), rem = it - g * perCol;
        const int rp = div_rcp( rem, invHw ), cp = rem - rp * hw;
        const int mvx = blk.mvx + ( i0 + g - radius ) * step;
        const int e = ( mvx >> 4 ) - dxMin + o, eo = e & 1, ew = e >> 1;      // pel offset of this vector inside the window rows
        const PackedTaps<6> X = sTap[i0 + g];
        const uint32_t* ra = win + ( 2 * rp ) * PW + cp + ew;
        int2 ha, hb;
        filter_row_pair<6>( ra, ra + PW, eo, X, ha, hb );
        uint2 pk;
        pk.x = (uint32_t) mctf_round_clip( ha.x, maxv ) | ( (uint32_t) mctf_round_clip( hb.x, maxv ) << 16 );
        pk.y = (uint32_t) mctf_round_clip( ha.y, maxv ) | ( (uint32_t) mctf_round_clip( hb.y, maxv ) << 16 );
        *reinterpret_cast<uint2*>( hbuf + g * L.colWords + rp * w + 2 * cp ) = pk;
      }
      __syncthreads();
      // ---- vertical pass + SSE for the gcount * (2r+1) candidates of these columns; a thread keeps its output positions
      if( hh * w <= T )                // one position per thread (blocks up to 16x16): decode it and fetch the original pels once
      {
        const bool act = tid < hh * w;
        const int yp = div_rcp( tid, invW ), x = tid - yp * w;
        const uint32_t ow = act ? orgP[tid] : 0u;
        const int o0 = (int)( ow & 0xffffu ), o1 = (int)( ow >> 16 );
        const uint32_t* hx = hbuf + x;
        for( int g = 0; g < gcount; g++, hx += L.colWords )
        {
          for( int j = 0; j < K1; j++ )
          {
            const int q = ( ( blk.mvy + ( j - radius ) * step ) >> 4 ) - dyMin + 2 * yp;
            const PackedTaps<6> Y = sTap[K1 + j];
            unsigned err = 0;
            if( act )
            {
              const uint32_t* tp = hx + ( q >> 1 ) * w;
              const uint32_t p[4] = { tp[0], tp[w], tp[2 * w], tp[3 * w] };
              const int2 v = filter_pair<6>( p, q & 1, Y );
              const int d0 = mctf_round_clip( v.x, maxv ) - o0, d1 = mctf_round_clip( v.y, maxv ) - o1;
              err = d0 * d0 + d1 * d1;
            }
            err = __reduce_add_sync( 0xffffffffu, err );
            if( ( tid & 31 ) == 0 && err ) atomicAdd( &sErr[j * K1 + i0 + g], err );
          }
        }
      }
      else
      for( int g = 0; g < gcount; g++ )
      {
        const uint32_t* H = hbuf + g * L.colWords;
        for( int j = 0; j < K1; j++ )
        {
          const int mvy = blk.mvy + ( j - radius ) * step;
          const int q0 = ( mvy >> 4 ) - dyMin;                                 // first filtered row of output row 0
          const PackedTaps<6> Y = sTap[K1 + j];
          unsigned err = 0;
          for( int p = tid; p < hh * w; p += T )
          {
            const int yp = div_rcp( p, invW ), x = p - yp * w;
            const int q = q0 + 2 * yp;
            const uint32_t* tp = H + ( q >> 1 ) * w + x;
            const uint32_t pw[4] = { tp[0], tp[w], tp[2 * w], tp[3 * w] };
            const int2 v = filter_pair<6>( pw, q & 1, Y );
            const uint32_t ow = orgP[p];
            const int d0 = mctf_round_clip( v.x, maxv ) - (int)( ow & 0xffffu ), d1 = mctf_round_clip( v.y, maxv ) - (int)( ow >> 16 );
            err += d0 * d0 + d1 * d1;
          }
          err = __reduce_add_sync( 0xffffffffu, err );
          if( ( tid & 31 ) == 0 && err ) atomicAdd( &sErr[j * K1 + i0 + g], err );
        }
      }
      __syncthreads();               // the filtered rows are consumed before the next group of columns overwrites them
    }
    __syncthreads();
    for( int k = tid; k < K; k += T ) out[(size_t) b * K + k] = mctf_sat32( sErr[k] );
  }
}

// ---------------------------------------------------------------------------------------------------------------------------------
// MCTF apply stage (SURVEY 8f rank 3): the per-block body of MCTF::xFinalizeBlkLine (CommonLib/MCTF.cpp:1437-1483) for luma, one CTA per block:
//   for every reference picture: applyFrac8Core_6Tap / _4Tap (:259-357, first pass unclipped, second pass clipped) at the block's motion vector,
//   applyPlanarCorrectionCore (:372-420) when rmsme > 0, QP <= 32, square block <= 32; then applyBlockCore (:422-518): noise estimate per
//   reference, weights, per-pel bilateral blend with fastExp (:359-367).  Integer parts are exact; the float parts follow the C++ expression
//   types of the reference literally (float *= double goes through double, `newVal + 0.5` is a double add) and the library is built with
//   --fmad=false, so results equal the scalar and the AVX2 reference bit for bit.
struct MctfApplyPar
{
  int    numRefs, blockSize, tap4, planar, width, height, blocksX, bitDepth, orgPlane, outStride;
  int    refPlane[8];
  double weightScaling, sigmaSq, refStrength[8];
};
struct MctfApplySmem { int winPitch, winWords, hWords, corrWords, orgWords, total; };
__host__ __device__ inline MctfApplySmem mctf_apply_smem( int bs, int numRefs )
{
  MctfApplySmem m;
  m.winPitch  = bs / 2 + 4;
  m.winWords  = ( bs + 6 ) * m.winPitch;
  m.hWords    = ( ( bs + 6 ) / 2 ) * bs;
  m.corrWords = numRefs * bs * bs / 2;
  m.orgWords  = bs * bs / 2;
  m.total     = m.winWords + m.hWords + m.corrWords + m.orgWords + 64 + 8 * 6;      // + weights + 64-bit accumulators
  return m;
}

__device__ __forceinline__ float mctf_fast_exp( float n, float d )
{
  float x = 1.0f + n / ( d * 1024 );
  x *= x; x *= x; x *= x; x *= x; x *= x; x *= x; x *= x; x *= x; x *= x; x *= x;
  return x;
}

__global__ void __launch_bounds__( 256 ) mctf_apply_kernel( const __grid_constant__ PlaneTable planes, const __grid_constant__ MctfApplyPar par,
                                                            const int4* __restrict__ mvs, int nBlocks, int16_t* __restrict__ out )
{
  extern __shared__ __align__( 16 ) uint32_t sApply[];
  const int bs = par.blockSize;
  const MctfApplySmem L = mctf_apply_smem( bs, par.numRefs );
  uint32_t* win  = sApply;
  uint32_t* hbuf = win + L.winWords;
  int16_t*  corr = reinterpret_cast<int16_t*>( hbuf + L.hWords );                   // [numRefs][h][w]
  int16_t*  orgB = reinterpret_cast<int16_t*>( hbuf + L.hWords + L.corrWords );     // [h][w]
  float*    sW   = reinterpret_cast<float*>( hbuf + L.hWords + L.corrWords + L.orgWords );   // vww[8], vsw[8]
  int*      sI   = reinterpret_cast<int*>( sW + 16 );                                // [0..2] planar sums, [8..15] vnoise
  unsigned long long* sAcc = reinterpret_cast<unsigned long long*>( sW + 64 );      // [0] variance, [1] diffsum
  const int tid = threadIdx.x, T = blockDim.x;
  const Plane orgPlane = planes.p[par.orgPlane];
  const int maxv = ( 1 << par.bitDepth ) - 1;
  const int PW = L.winPitch;
  const int tap4 = par.tap4;

  for( int b = blockIdx.x; b < nBlocks; b += gridDim.x )
  {
    const int bxI = b % par.blocksX, byI = b / par.blocksX;
    const int bx = bxI * bs, by = byI * bs;
    const int w = min( bs, par.width - bx ), h = min( bs, par.height - by );
    const int hw = w >> 1, hh = h >> 1;
    const float invHw = 1.0f / (float) hw, invW = 1.0f / (float) w;
    __syncthreads();
    for( int i = tid; i < h * w; i += T )
    {
      const int y = div_rcp( i, invW ), x = i - y * w;
      orgB[i] = __ldg( orgPlane.origin + (ptrdiff_t)( by + y ) * orgPlane.stride + bx + x );
    }
    for( int r = 0; r < par.numRefs; r++ )
    {
      const Plane refPlane = planes.p[par.refPlane[r]];
      const int4 mv = __ldg( mvs + (size_t) r * nBlocks + b );                        // x, y, error, rmsme
      int16_t* cr = corr + r * h * w;
      // ---- window: rows by+yInt-2 .., pels from the even pel at or below bx+xInt-2
      const int rowsP = ( h + 6 ) & ~1;
      __syncthreads();                                   // previous reference's readers of win / hbuf are done
      const int o = stage_pel_pairs( win, PW, refPlane.origin + (ptrdiff_t)( by + ( mv.y >> 4 ) - 2 ) * refPlane.stride + bx + ( mv.x >> 4 ) - 2, refPlane.stride,
                                     w + 5, rowsP, tid, T );
      if( tid < 3 ) sI[tid] = 0;
      if( tid < 2 ) sAcc[tid] = 0ull;
      __syncthreads();
      const PackedTaps<6> X = mctf_taps6( tap4, mv.x & 15 );
      for( int it = tid; it < ( rowsP >> 1 ) * hw; it += T )
      {
        const int rp = div_rcp( it, invHw ), cp = it - rp * hw;
        const uint32_t* ra = win + ( 2 * rp ) * PW + cp;
        int2 ha, hb;
        filter_row_pair<6>( ra, ra + PW, o, X, ha, hb );
        uint2 pk;                                        // first pass is NOT clipped (MCTF.cpp:284): signed 16-bit halves
        pk.x = ( (uint32_t)( ( ha.x + 32 ) >> 6 ) & 0xffffu ) | ( (uint32_t)( ( hb.x + 32 ) >> 6 ) << 16 );
        pk.y = ( (uint32_t)( ( ha.y + 32 ) >> 6 ) & 0xffffu ) | ( (uint32_t)( ( hb.y + 32 ) >> 6 ) << 16 );
        *reinterpret_cast<uint2*>( hbuf + rp * w + 2 * cp ) = pk;
      }
      __syncthreads();
      const PackedTaps<6> Y = mctf_taps6( tap4, mv.y & 15 );
      const bool doPlanar = ( mv.w & 0xffff ) > 0 && par.planar && w == h && w <= 32;
      int s1 = 0, s2 = 0, s0 = 0;
      for( int p = tid; p < hh * w; p += T )
      {
        const int yp = div_rcp( p, invW ), x = p - yp * w;
        const uint32_t* tp = hbuf + yp * w + x;
        const uint32_t pw[4] = { tp[0], tp[w], tp[2 * w], tp[3 * w] };
        const int2 v = filter_pair<6>( pw, false, Y );
        const int v0 = mctf_round_clip( v.x, maxv ), v1 = mctf_round_clip( v.y, maxv );
        cr[( 2 * yp ) * w + x] = (int16_t) v0; cr[( 2 * yp + 1 ) * w + x] = (int16_t) v1;
        if( doPlanar )
        {
          const int z0 = v0 - orgB[( 2 * yp ) * w + x], z1 = v1 - orgB[( 2 * yp + 1 ) * w + x];
          s1 += x * ( z0 + z1 ); s2 += ( 2 * yp ) * z0 + ( 2 * yp + 1 ) * z1; s0 += z0 + z1;
        }
      }
      if( doPlanar )
      {
        s1 = __reduce_add_sync( 0xffffffffu, s1 ); s2 = __reduce_add_sync( 0xffffffffu, s2 ); s0 = __reduce_add_sync( 0xffffffffu, s0 );
        if( ( tid & 31 ) == 0 ) { atomicAdd( &sI[0], s1 ); atomicAdd( &sI[1], s2 ); atomicAdd( &sI[2], s0 ); }
      }
      __syncthreads();
      if( doPlanar )                                     // applyPlanarCorrectionCore, fixed-point plane fit (MCTF.cpp:395-418)
      {
        const int xSzm[6] = { 0, 1, 20, 336, 5440, 87296 };
        const int blockSize = w * h, log2W = 31 - __clz( w );
        const unsigned me = (unsigned)( mv.w & 0xffff );
        const int mWeight = (int) min( 512u, me * me );
        const int xSum = ( blockSize * ( w - 1 ) ) >> 1;
        const int x1yzm = sI[0], x2yzm = sI[1], ySum = sI[2];
        const long long denom = (long long) blockSize * xSzm[log2W];
        long long numer = (long long) mWeight * ( (long long) x1yzm * blockSize - (long long) xSum * ySum );
        int b1 = (int)( ( numer < 0 ? numer - ( denom >> 1 ) : numer + ( denom >> 1 ) ) / denom );
        b1 = max( -32768, min( 32767, b1 ) );
        numer = (long long) mWeight * ( (long long) x2yzm * blockSize - (long long) xSum * ySum );
        int b2 = (int)( ( numer < 0 ? numer - ( denom >> 1 ) : numer + ( denom >> 1 ) ) / denom );
        b2 = max( -32768, min( 32767, b2 ) );
        const int b0 = ( mWeight * ySum - ( b1 + b2 ) * xSum + ( blockSize >> 1 ) ) >> ( log2W << 1 );
        if( b0 | b1 | b2 )
          for( int i = tid; i < h * w; i += T )
          {
            const int y = div_rcp( i, invW ), x = i - y * w;
            const int pc = ( b0 + b1 * x + b2 * y + 256 ) >> 9;
            cr[i] = (int16_t) max( 0, min( maxv, (int) cr[i] - pc ) );
          }
        __syncthreads();
      }
      // ---- noise estimate of applyBlockCore (MCTF.cpp:442-472): variance and first-difference energy of (org - corrected)
      {
        unsigned long long var = 0, dsum = 0;
        for( int i = tid; i < h * w; i += T )
        {
          const int y = div_rcp( i, invW ), x = i - y * w;
          const int diff = (int) orgB[i] - (int) cr[i];
          var += (unsigned)( diff * diff );
          if( x != w - 1 ) { const int dR = (int) orgB[i + 1] - (int) cr[i + 1]; dsum += (unsigned)( ( dR - diff ) * ( dR - diff ) ); }
          if( y != h - 1 ) { const int dD = (int) orgB[i + w] - (int) cr[i + w]; dsum += (unsigned)( ( dD - diff ) * ( dD - diff ) ); }
        }
#pragma unroll
        for( int m = 16; m > 0; m >>= 1 ) { var += __shfl_xor_sync( 0xffffffffu, var, m ); dsum += __shfl_xor_sync( 0xffffffffu, dsum, m ); }
        if( ( tid & 31 ) == 0 ) { atomicAdd( &sAcc[0], var ); atomicAdd( &sAcc[1], dsum ); }
        __syncthreads();
        if( tid == 0 )
        {
          long long variance = (long long) sAcc[0], diffsum = (long long) sAcc[1];
          variance *= 1ll << ( 2 * ( 10 - par.bitDepth ) );
          diffsum  *= 1ll << ( 2 * ( 10 - par.bitDepth ) );
          const int cntV = w * h, cntD = 2 * cntV - w - h;
          sI[8 + r] = (int) round( ( 15.0 * cntD / cntV * (double) variance + 5.0 ) / ( (double) diffsum + 5.0 ) );
          sI[16 + r] = mv.z;                             // verror
        }
      }
    }
    __syncthreads();
    if( tid == 0 )                                       // weights (MCTF.cpp:474-489)
    {
      int minError = 0x7fffffff;
      for( int r = 0; r < par.numRefs; r++ ) minError = min( minError, sI[16 + r] );
      for( int r = 0; r < par.numRefs; r++ )
      {
        const int error = sI[16 + r], noise = sI[8 + r];
        float ww = 1, sw = 1;
        ww = (float)( (double) ww * ( ( noise < 25 ) ? 1.0 : 0.6 ) );
        sw = (float)( (double) sw * ( ( noise < 25 ) ? 1.0 : 0.8 ) );
        ww = (float)( (double) ww * ( ( error < 50 ) ? 1.2 : ( ( error > 100 ) ? 0.6 : 1.0 ) ) );
        sw = (float)( (double) sw * ( ( error < 50 ) ? 1.0 : 0.8 ) );
        ww = (float)( (double) ww * ( ( minError + 1.0 ) / ( error + 1.0 ) ) );
        sW[r]     = (float)( (double) ww * par.weightScaling * par.refStrength[r] );
        sW[8 + r] = (float)( (double)( sw * 2 ) * par.sigmaSq );
      }
    }
    __syncthreads();
    // ---- per-pel blend (MCTF.cpp:491-517)
    for( int i = tid; i < h * w; i += T )
    {
      const int y = div_rcp( i, invW ), x = i - y * w;
      const int orgVal = orgB[i];
      float temporalWeightSum = 1.0f;
      float newVal = (float) orgVal;
      for( int r = 0; r < par.numRefs; r++ )
      {
        const int refVal = corr[r * h * w + i];
        const int diff = refVal - orgVal;
        const float diffSq = (float)( diff * diff );
        const float weight = sW[r] * mctf_fast_exp( -diffSq, sW[8 + r] );
        newVal += weight * (float) refVal;
        temporalWeightSum += weight;
      }
      newVal /= temporalWeightSum;
      int sampleVal = (int)(short)(int)( (double) newVal + 0.5 );
      sampleVal = max( 0, min( maxv, sampleVal ) );
      out[(size_t)( by + y ) * par.outStride + bx + x] = (int16_t) sampleVal;
    }
  }
}

// calcVarCore (MCTF.cpp:520-546): 16 * variance of a block in 1/256 units, double result
__global__ void mctf_calc_var_kernel( const __grid_constant__ Plane plane, const vvb_mctf_cand* __restrict__ blocks, int n, double* __restrict__ out )
{
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int b = blockIdx.x * ( blockDim.x >> 5 ) + warp;
  if( b >= n ) return;
  const vvb_mctf_cand c = blocks[b];
  const int w = c.w, h = c.h;
  const int16_t* org = plane.origin + (ptrdiff_t) c.y * plane.stride + c.x;
  const float invW = 1.0f / (float) w;
  int avg = 0;
  for( int i = lane; i < w * h; i += 32 ) { const int y = div_rcp( i, invW ), x = i - y * w; avg += __ldg( org + (ptrdiff_t) y * plane.stride + x ); }
  avg = __reduce_add_sync( 0xffffffffu, avg );
  avg <<= 4;
  avg = avg / ( w * h );
  long long var = 0;
  for( int i = lane; i < w * h; i += 32 )
  {
    const int y = div_rcp( i, invW ), x = i - y * w;
    const int pix = (int) __ldg( org + (ptrdiff_t) y * plane.stride + x ) << 4;
    var += (long long)( ( pix - avg ) * ( pix - avg ) );
  }
#pragma unroll
  for( int m = 16; m > 0; m >>= 1 ) var += __shfl_xor_sync( 0xffffffffu, var, m );
  if( lane == 0 ) out[b] = (double) var / 256.0;
}

// ---- affine (AffineGradientSearch.cpp:84-190): the Sobel filters and the normal equations of xEqualCoeffComputer, written once and used by the
// single-block helpers (sobel_kernel, equal_coeff_kernel) and by the fused per-block form (affine_eq_batch_kernel)

// xHorizontalSobelFilter (vertical = false) / xVerticalSobelFilter at sample (x, y) of a w x h block with row stride ps.  Border samples copy the nearest
// interior result (edges: inner neighbour, corners: inner diagonal).
__device__ __forceinline__ int affine_sobel_at( const int16_t* p, int ps, int x, int y, int w, int h, bool vertical )
{
  const int yy = min( max( y, 1 ), h - 2 ), xx = min( max( x, 1 ), w - 2 );
  const int16_t* c = p + yy * ps + xx;
  if( !vertical ) return c[1 - ps] - c[-1 - ps] + ( c[1] << 1 ) - ( c[-1] << 1 ) + c[1 + ps] - c[-1 + ps];
  return c[ps - 1] - c[-ps - 1] + ( c[ps] << 1 ) - ( c[-ps] << 1 ) + c[ps + 1] - c[-ps + 1];
}

// the terms one sample adds to the 4- or 6-parameter normal equations: gradients a (x) and b (y) and residual r at (x, y), whose 4x4 sub-block centre
// gives the affine coordinates; acc[col][row] for row < NP is the matrix, acc[col][NP] the right-hand side
template<int NP>
__device__ __forceinline__ void affine_eq_terms( long long ( &acc )[NP][NP + 1], int a, int b, int r, int x, int y )
{
  const int cy = ( ( y >> 2 ) << 2 ) + 2, cx = ( ( x >> 2 ) << 2 ) + 2;
  int c[NP];
  if( NP == 4 ) { c[0] = a; c[1] = cx * a + cy * b; c[2] = b; c[3] = cy * a - cx * b; }
  else          { c[0] = a; c[1] = cx * a; c[2] = b; c[3] = cx * b; c[NP > 4 ? 4 : 0] = cy * a; c[NP > 4 ? 5 : 0] = cy * b; }
#pragma unroll
  for( int col = 0; col < NP; col++ )
  {
#pragma unroll
    for( int row = 0; row < NP; row++ ) acc[col][row] += (long long) c[col] * c[row];
    acc[col][NP] += ( (long long) c[col] * r ) * 8;
  }
}

// the CTA's sum of acc in sEq[49], laid out as pEqualCoeff: acc[col][row] goes to sEq[(col + 1) * 7 + row].  Every thread of the CTA calls it; sEq is
// complete on return.
template<int NP>
__device__ __forceinline__ void affine_eq_reduce( const long long ( &acc )[NP][NP + 1], unsigned long long* sEq )
{
  for( int i = threadIdx.x; i < 49; i += blockDim.x ) sEq[i] = 0;
  __syncthreads();
#pragma unroll
  for( int col = 0; col < NP; col++ )
#pragma unroll
    for( int row = 0; row <= NP; row++ )
    {
      long long v = acc[col][row];
#pragma unroll
      for( int m = 16; m > 0; m >>= 1 ) v += __shfl_xor_sync( 0xffffffffu, v, m );
      if( ( threadIdx.x & 31 ) == 0 && v ) atomicAdd( &sEq[( col + 1 ) * 7 + row], (unsigned long long) v );
    }
  __syncthreads();
}

// Sobel of one w x h block, grid-stride over its samples
__global__ void sobel_kernel( const int16_t* __restrict__ pred, int ps, int16_t* __restrict__ deriv, int ds, int w, int h, int vertical )
{
  for( int i = blockIdx.x * blockDim.x + threadIdx.x; i < w * h; i += gridDim.x * blockDim.x )
  {
    const int y = i / w, x = i - y * w;
    deriv[y * ds + x] = (int16_t) affine_sobel_at( pred, ps, x, y, w, h, vertical );
  }
}

// normal equations of one w x h block, grid-stride over its samples; each CTA adds its sums to eq[49] with global atomics
template<int NP>
__global__ void __launch_bounds__( 256 ) equal_coeff_kernel( const int16_t* __restrict__ resi, int rs, const int16_t* __restrict__ gx, const int16_t* __restrict__ gy, int ds,
                                                             int w, int h, long long* __restrict__ eq )
{
  long long acc[NP][NP + 1] = {};
  for( int i = blockIdx.x * blockDim.x + threadIdx.x; i < w * h; i += gridDim.x * blockDim.x )
  {
    const int y = i / w, x = i - y * w;
    affine_eq_terms<NP>( acc, gx[y * ds + x], gy[y * ds + x], resi[y * rs + x], x, y );
  }
  __shared__ unsigned long long sEq[49];
  affine_eq_reduce<NP>( acc, sEq );
  for( int i = threadIdx.x; i < 49; i += blockDim.x )
    if( sEq[i] ) atomicAdd( reinterpret_cast<unsigned long long*>( &eq[i] ), sEq[i] );
}

// xHorizontalSobelFilter + xVerticalSobelFilter + xEqualCoeffComputer of one block per CTA, the body of the affine motion-estimation iteration
// (InterSearch.cpp:5373-5387): pred, resi are compact [n][h][w]; the Sobel results live in shared memory (and go to derivX / derivY when those are given)
template<int NP>
__global__ void __launch_bounds__( 128 ) affine_eq_batch_kernel( const int16_t* __restrict__ pred, const int16_t* __restrict__ resi, int w, int h,
                                                                 int16_t* __restrict__ derivX, int16_t* __restrict__ derivY, long long* __restrict__ eq )
{
  extern __shared__ int16_t sm[];
  int16_t* sP = sm; int16_t* sX = sm + w * h; int16_t* sY = sX + w * h;
  const size_t off = (size_t) blockIdx.x * w * h;
  for( int i = threadIdx.x; i < w * h; i += blockDim.x ) sP[i] = pred[off + i];
  __syncthreads();
  for( int i = threadIdx.x; i < w * h; i += blockDim.x )
  {
    const int y = i / w, x = i - y * w;
    const int gx = affine_sobel_at( sP, w, x, y, w, h, false ), gy = affine_sobel_at( sP, w, x, y, w, h, true );
    sX[i] = (int16_t) gx; sY[i] = (int16_t) gy;
    if( derivX ) derivX[off + i] = (int16_t) gx;
    if( derivY ) derivY[off + i] = (int16_t) gy;
  }
  __syncthreads();
  long long acc[NP][NP + 1] = {};
  for( int i = threadIdx.x; i < w * h; i += blockDim.x )
  {
    const int y = i / w, x = i - y * w;
    affine_eq_terms<NP>( acc, sX[i], sY[i], resi[off + i], x, y );
  }
  __shared__ unsigned long long sEq[49];
  affine_eq_reduce<NP>( acc, sEq );
  for( int i = threadIdx.x; i < 49; i += blockDim.x ) eq[(size_t) blockIdx.x * 49 + i] = (long long) sEq[i];
}

} // namespace vvb
