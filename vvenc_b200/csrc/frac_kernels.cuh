// frac_kernels.cuh -- fractional-pel refinement feeding SATD (SURVEY 8f rank 2).
//
// frac_grid_kernel: for every block and its integer vector, the distortion (SAD or 8x8-tiled SATD) of all 49 quarter-pel offsets (-3..3)^2 -- every
// position InterSearch::xPatternRefinement (EncoderLib/InterSearch.cpp:760-972) can visit in its half-pel round (+-2) and its quarter-pel round
// around the best half-pel position (+-1 more).  The filtered blocks are produced as the reference produces them (xPatternRefinement :790-850,
// xExtDIFUpSamplingH/Q :2912-3040): TWO passes of the 8-tap luma filter for every position, InterpolationFilter::filterHor( frac_x, isLast = false )
// then filterVer( frac_y, isFirst = false, isLast = true ) (CommonLib/InterpolationFilter.cpp:357-455; phase 0 is filterCopy :258-340, identical to
// the filter with the single tap 64), 14-bit signed intermediates, clip after the second pass.  The filter set follows m_meReduceTap / useAltHpelIf.
//
// One CTA per block.  The window (h + 8 rows) is staged once; the horizontally filtered rows of one horizontal offset at a time (all seven at once for
// 8x8 blocks) are computed once (packed as row pairs, IDP.2A) and shared by the 7 vertical offsets; a lane owns one (vertical offset, 8x8 tile): it runs the vertical filter for its
// tile (IDP.2A on row pairs), forms the 64 differences in registers and either sums |d| or runs the 64-point 2-D Hadamard there (as had8_direct_kernel).
#pragma once
#include "common.cuh"
#include "dist_kernels.cuh"
#include "packed_filter.cuh"

namespace vvb {

// Quarter-pel phases as 8-tap rows over pels x-3 .. x+4, chosen by the host (frac_filter): m_meReduceTap 0 -> m_lumaFilter rows 0,4,8,12;
// 1 -> m_lumaFilter4x4 rows as 6 taps; 2 -> m_chromaFilter rows 8,16,24 as 4 taps (InterpolationFilter.cpp:64-142, 557-600; every preset's
// ReduceFilterME = 2); useAltHpelIf replaces the half-pel phase by m_lumaAltHpelIFilter.  Shorter filters are zero-padded: same pels, same sums.
struct FracFilter { signed char c[4][8]; };
static inline FracFilter frac_filter( int reduceTap, int altHpel )
{
  static const signed char sets[3][4][8] = {
    { { 0, 0, 0, 64, 0, 0, 0, 0 }, { -1, 4, -10, 58, 17, -5, 1, 0 }, { -1, 4, -11, 40, 40, -11, 4, -1 }, { 0, 1, -5, 17, 58, -10, 4, -1 } },
    { { 0, 0, 0, 64, 0, 0, 0, 0 }, {  0, 3, -10, 58, 17, -5, 1, 0 }, {  0, 3, -11, 40, 40, -11, 3,  0 }, { 0, 1, -5, 17, 58, -10, 3,  0 } },
    { { 0, 0, 0, 64, 0, 0, 0, 0 }, {  0, 0,  -4, 54, 16, -2, 0, 0 }, {  0, 0,  -4, 36, 36,  -4, 0,  0 }, { 0, 0, -2, 16, 54,  -4, 0,  0 } } };
  static const signed char alt[8] = { 0, 3, 9, 20, 20, 9, 3, 0 };
  FracFilter f;
  for( int p = 0; p < 4; p++ ) for( int t = 0; t < 8; t++ ) f.c[p][t] = ( altHpel && p == 2 ) ? alt[t] : sets[reduceTap][p][t];
  return f;
}

struct FracSmem { int winPitch, winWords, colWords, G, hWords, orgWords, total; };
__host__ __device__ inline FracSmem frac_smem( int w, int h )
{
  FracSmem m;
  m.winPitch = w / 2 + 6;                       // w + 8 pels + alignment + one word of slack for the zero-weighted tap
  m.winWords = ( h + 8 ) * m.winPitch;
  m.colWords = ( ( h + 8 ) / 2 ) * w;           // horizontally filtered rows of one horizontal offset: row pairs x w
  m.G        = w * h <= 64 ? 7 : 1;             // horizontal offsets per pass: all seven for 8x8 blocks (lane utilisation), one otherwise (measured faster)
  m.hWords   = m.G * m.colWords;
  m.orgWords = h * w / 2;
  m.total    = m.winWords + m.hWords + m.orgWords + 52 + 40;     // + table + packed taps of the 4 phases
  return m;
}

__device__ __forceinline__ PackedTaps<8> frac_taps( const FracFilter& flt, int phase )
{
  int f[8];
#pragma unroll
  for( int t = 0; t < 8; t++ ) f[t] = flt.c[phase][t];
  return pack_taps<8>( f );
}

// family: 1 = SAD, 2 = HAD (8x8 tiles: square blocks 8..64)
__global__ void __launch_bounds__( 128 ) frac_grid_kernel( const __grid_constant__ Plane orgPlane, const __grid_constant__ Plane refPlane,
                                                           const vvb_block* __restrict__ blocks, int n, int w, int h, int family, const __grid_constant__ FracFilter flt,
                                                           uint32_t* __restrict__ out )
{
  extern __shared__ __align__( 16 ) uint32_t sFrac[];
  const FracSmem L = frac_smem( w, h );
  uint32_t* win  = sFrac;
  uint32_t* hbuf = win + L.winWords;
  uint32_t* orgS = hbuf + L.hWords;                 // [h][w/2] words, rows 16-byte aligned (w multiple of 8)
  uint32_t* sOut = orgS + L.orgWords;               // [49]
  PackedTaps<8>* sTaps = reinterpret_cast<PackedTaps<8>*>( sOut + 52 );   // packed taps of the 4 phases (same for both passes)
  const int tid = threadIdx.x, T = blockDim.x;
  const int PW = L.winPitch, hw = w >> 1, rowsP = h + 8, tilesX = w >> 3, nTiles = tilesX * ( h >> 3 );
  const int bd = refPlane.bitDepth, maxv = ( 1 << bd ) - 1;
  const int headRoom = 14 - bd;                      // bit depths 8..12
  const int shift1 = 6 - headRoom, offset1 = -( 8192 << shift1 );
  const int shift2 = 6 + headRoom, offset2 = ( 1 << ( shift2 - 1 ) ) + ( 8192 << 6 );
  const float invHw = 1.0f / (float) hw, invNt = 1.0f / (float) nTiles, invTx = 1.0f / (float) tilesX;
  if( threadIdx.x < 4 ) sTaps[threadIdx.x] = frac_taps( flt, threadIdx.x );

  for( int b = blockIdx.x; b < n; b += gridDim.x )
  {
    const vvb_block blk = blocks[b];
    // ---- window: rows y+my-4 .. y+my+h+3, pels from the even pel at or below x+mx-4; original block; clear the table
    __syncthreads();
    const int o = stage_pel_pairs( win, PW, refPlane.origin + (ptrdiff_t)( blk.y + blk.start_y - 4 ) * refPlane.stride + blk.x + blk.start_x - 4, refPlane.stride,
                                   w + 8, rowsP, tid, T );
    {
      const int16_t* org = orgPlane.origin + (ptrdiff_t) blk.y * orgPlane.stride + blk.x;
      for( int i = tid; i < h * hw; i += T )
      {
        const int y = div_rcp( i, invHw ), c = i - y * hw;
        const int16_t* p = org + (ptrdiff_t) y * orgPlane.stride + 2 * c;
        orgS[i] = (uint32_t)(uint16_t) __ldg( p ) | ( (uint32_t)(uint16_t) __ldg( p + 1 ) << 16 );
      }
    }
    for( int k = tid; k < 49; k += T ) sOut[k] = 0u;
    __syncthreads();
    const int perCol = ( rowsP >> 1 ) * hw, jobsPerCol = 7 * nTiles;
    const float invPerCol = 1.0f / (float) perCol, invJobs = 1.0f / (float) jobsPerCol;
    for( int i0 = 0; i0 < 7; i0 += L.G )
    {
      const int gcount = min( L.G, 7 - i0 );
      // ---- horizontal pass (filterHor, isLast = false) for gcount horizontal offsets: item = (offset, row pair, column pair), results packed as row pairs
      for( int it = tid; it < gcount * perCol; it += T )
      {
        const int g = div_rcp( it, invPerCol ), rem = it - g * perCol;
        const int rp = div_rcp( rem, invHw ), cp = rem - rp * hw;
        const int qx = i0 + g - 3;
        const int e = ( qx >> 2 ) + 1 + o, eo = e & 1, ew = e >> 1;
        const PackedTaps<8> X = sTaps[qx & 3];
        const uint32_t* ra = win + ( 2 * rp ) * PW + cp + ew;
        int2 ha, hb;
        filter_row_pair<8>( ra, ra + PW, eo, X, ha, hb );
        uint2 pk;
        pk.x = ( (uint32_t)( ( ha.x + offset1 ) >> shift1 ) & 0xffffu ) | ( (uint32_t)( ( hb.x + offset1 ) >> shift1 ) << 16 );
        pk.y = ( (uint32_t)( ( ha.y + offset1 ) >> shift1 ) & 0xffffu ) | ( (uint32_t)( ( hb.y + offset1 ) >> shift1 ) << 16 );
        *reinterpret_cast<uint2*>( hbuf + g * L.colWords + rp * w + 2 * cp ) = pk;
      }
      __syncthreads();
      // ---- vertical pass (filterVer, isFirst = false, isLast = true) + distortion: lane = (horizontal offset, vertical offset j, 8x8 tile)
      for( int job = tid; job < gcount * jobsPerCol; job += T )
      {
        const int g = div_rcp( job, invJobs ), jr = job - g * jobsPerCol;
        const int i = i0 + g;
        const int j = div_rcp( jr, invNt ), t = jr - j * nTiles;
        const int ty = div_rcp( t, invTx ), tx = t - ty * tilesX;
        const int qy = j - 3;
        const PackedTaps<8> Y = sTaps[qy & 3];
        const int q = ( qy >> 2 ) + 1 + ty * 8;                                 // first filtered row of the tile's first output row
        const uint32_t* hp = hbuf + g * L.colWords + ( q >> 1 ) * w + tx * 8;
        const bool odd = ( q & 1 ) != 0;
        int d[64];
#pragma unroll
        for( int c = 0; c < 8; c++ )
        {
          uint32_t P[8];
#pragma unroll
          for( int k = 0; k < 8; k++ ) P[k] = hp[k * w + c];
#pragma unroll
          for( int m = 0; m < 4; m++ )
          {
            const int2 v = filter_pair<8>( P + m, odd, Y );
            d[8 * ( 2 * m ) + c]     = max( min( ( v.x + offset2 ) >> shift2, maxv ), 0 );
            d[8 * ( 2 * m + 1 ) + c] = max( min( ( v.y + offset2 ) >> shift2, maxv ), 0 );
          }
        }
#pragma unroll
        for( int r = 0; r < 8; r++ )
        {
          const uint4 ow = *reinterpret_cast<const uint4*>( orgS + ( ( ty * 8 + r ) * w + tx * 8 ) / 2 );
          d[8*r+0] = lo16( ow.x ) - d[8*r+0]; d[8*r+1] = hi16( ow.x ) - d[8*r+1];
          d[8*r+2] = lo16( ow.y ) - d[8*r+2]; d[8*r+3] = hi16( ow.y ) - d[8*r+3];
          d[8*r+4] = lo16( ow.z ) - d[8*r+4]; d[8*r+5] = hi16( ow.z ) - d[8*r+5];
          d[8*r+6] = lo16( ow.w ) - d[8*r+6]; d[8*r+7] = hi16( ow.w ) - d[8*r+7];
        }
        uint32_t s = 0;
        if( family == 2 ) s = had8<0, 1>( d );          // one abs-sum chain: with four, ptxas spills in this kernel
        else
        {
#pragma unroll
          for( int k = 0; k < 64; k++ ) s = __sad( d[k], 0, s );
        }
        atomicAdd( &sOut[j * 7 + i], s );
      }
      __syncthreads();               // the filtered rows are consumed before the next group of offsets overwrites them
    }
    for( int k = tid; k < 49; k += T ) out[(size_t) b * 49 + k] = sOut[k];
  }
}


// ---------------------------------------------------------------------------------------------------------------------------------------------
// Generic shapes (SURVEY 8f-2, the rest of the PU shapes xPatternRefinement meets): rectangular PUs (SATD on 16x8 / 8x16 / 8x4 / 4x8 tiles with the fp64
// normalisation, RdCost.cpp:1324-1766), DF_HAD_fast on square multiples of 32 (16x16_fast tiles: 2x2 rounded means of original and prediction, :1126-1223),
// blocks with a 4-pel side, and SAD on all of them.  Same interpolation as frac_grid_kernel (one horizontal offset at a time); the seven vertically filtered
// blocks of that offset are written to shared memory as pels and each warp evaluates whole blocks with the tile code of the pair-list kernels
// (had_tile_lanes: a tile row per lane, vertical Hadamard over shuffles).
struct FracGenSmem { int winPitch, winWords, hWords, orgWords, predWords, total; };
__host__ __device__ inline FracGenSmem frac_gen_smem( int w, int h )
{
  FracGenSmem m;
  m.winPitch  = w / 2 + 6;
  m.winWords  = ( h + 8 ) * m.winPitch;
  m.hWords    = ( ( h + 8 ) / 2 + 4 ) * w;          // + slack: the vertical pass always reads 8 row pairs
  m.orgWords  = h * w / 2;
  m.predWords = 7 * h * w / 2;
  m.total     = m.winWords + m.hWords + m.orgWords + m.predWords + 52 + 40;
  return m;
}

template<int TW>
__device__ __forceinline__ uint32_t frac_warp_had( const int16_t* __restrict__ org, const int16_t* __restrict__ pred, int w, int h, const HadShape& s, int lane )
{
  const int th = s.fast16 ? 8 : s.th;                 // lanes per tile
  const int tilesX = w / s.tw, nt = tilesX * ( h / s.th );
  const int tpi = 32 / th, row = lane % th, sub = lane / th;
  uint32_t acc = 0;
  for( int t0 = 0; t0 < nt; t0 += tpi )
  {
    const int t = t0 + sub;
    const bool active = t < nt;
    int d[TW];
#pragma unroll
    for( int i = 0; i < TW; i++ ) d[i] = 0;
    if( active )
    {
      const int ty = t / tilesX, tx = t - ty * tilesX;
      if( s.fast16 )
      {
        const int16_t* o = org  + ( ty * 16 + 2 * row ) * w + tx * 16;
        const int16_t* c = pred + ( ty * 16 + 2 * row ) * w + tx * 16;
#pragma unroll
        for( int x = 0; x < TW; x++ )
          d[x] = ( ( (int) o[2*x] + o[2*x + 1] + o[w + 2*x] + o[w + 2*x + 1] + 2 ) >> 2 ) - ( ( (int) c[2*x] + c[2*x + 1] + c[w + 2*x] + c[w + 2*x + 1] + 2 ) >> 2 );
      }
      else
      {
        const int16_t* o = org  + ( ty * s.th + row ) * w + tx * TW;
        const int16_t* c = pred + ( ty * s.th + row ) * w + tx * TW;
#pragma unroll
        for( int x = 0; x < TW; x++ ) d[x] = (int) o[x] - (int) c[x];
      }
    }
    const uint32_t v = had_tile_lanes<TW>( d, th, row, active, 0xffffffffu );
    acc += s.fast16 ? ( v << 2 ) : v;
  }
  return __reduce_add_sync( 0xffffffffu, acc );
}

// family: 1 = SAD, 2 = HAD, 3 = HAD_fast
__global__ void __launch_bounds__( 128 ) frac_grid_generic_kernel( const __grid_constant__ Plane orgPlane, const __grid_constant__ Plane refPlane,
                                                                   const vvb_block* __restrict__ blocks, int n, int w, int h, int family, const __grid_constant__ FracFilter flt,
                                                                   uint32_t* __restrict__ out )
{
  extern __shared__ __align__( 16 ) uint32_t sFrac[];
  const FracGenSmem L = frac_gen_smem( w, h );
  uint32_t* win  = sFrac;
  uint32_t* hbuf = win + L.winWords;
  uint32_t* orgW = hbuf + L.hWords;                 // [h][w] pels
  uint32_t* prdW = orgW + L.orgWords;               // [7][h][w] pels
  uint32_t* sOut = prdW + L.predWords;              // [49]
  PackedTaps<8>* sTaps = reinterpret_cast<PackedTaps<8>*>( sOut + 52 );
  const int16_t* orgS = reinterpret_cast<const int16_t*>( orgW );
  int16_t* pred = reinterpret_cast<int16_t*>( prdW );
  const int tid = threadIdx.x, T = blockDim.x, lane = tid & 31, warp = tid >> 5, nWarps = T >> 5;
  const int PW = L.winPitch, hw = w >> 1, rowsP = h + 8, cellsY = ( h + 7 ) >> 3;
  const int bd = refPlane.bitDepth, maxv = ( 1 << bd ) - 1;
  const int headRoom = 14 - bd;
  const int shift1 = 6 - headRoom, offset1 = -( 8192 << shift1 );
  const int shift2 = 6 + headRoom, offset2 = ( 1 << ( shift2 - 1 ) ) + ( 8192 << 6 );
  const float invHw = 1.0f / (float) hw, invW = 1.0f / (float) w;
  if( tid < 4 ) sTaps[tid] = frac_taps( flt, tid );
  HadShape hs; hs.tw = 8; hs.th = 8; hs.fast16 = 0;
  if( family >= 2 ) had_shape( w, h, family == 3, hs );

  for( int b = blockIdx.x; b < n; b += gridDim.x )
  {
    const vvb_block blk = blocks[b];
    __syncthreads();
    const int o = stage_pel_pairs( win, PW, refPlane.origin + (ptrdiff_t)( blk.y + blk.start_y - 4 ) * refPlane.stride + blk.x + blk.start_x - 4, refPlane.stride,
                                   w + 8, rowsP, tid, T );
    {
      const int16_t* org = orgPlane.origin + (ptrdiff_t) blk.y * orgPlane.stride + blk.x;
      for( int i = tid; i < h * hw; i += T )
      {
        const int y = div_rcp( i, invHw ), c = i - y * hw;
        const int16_t* p = org + (ptrdiff_t) y * orgPlane.stride + 2 * c;
        orgW[i] = (uint32_t)(uint16_t) __ldg( p ) | ( (uint32_t)(uint16_t) __ldg( p + 1 ) << 16 );
      }
    }
    for( int i = tid; i < L.hWords; i += T ) hbuf[i] = 0u;          // the slack rows stay defined
    __syncthreads();
    const int perCol = ( rowsP >> 1 ) * hw;
    for( int i = 0; i < 7; i++ )
    {
      // ---- horizontal pass for offset i (as frac_grid_kernel)
      const int qx = i - 3;
      const int e = ( qx >> 2 ) + 1 + o, eo = e & 1, ew = e >> 1;
      const PackedTaps<8> X = sTaps[qx & 3];
      for( int it = tid; it < perCol; it += T )
      {
        const int rp = div_rcp( it, invHw ), cp = it - rp * hw;
        const uint32_t* ra = win + ( 2 * rp ) * PW + cp + ew;
        int2 ha, hb;
        filter_row_pair<8>( ra, ra + PW, eo, X, ha, hb );
        hbuf[rp * w + 2 * cp]     = ( (uint32_t)( ( ha.x + offset1 ) >> shift1 ) & 0xffffu ) | ( (uint32_t)( ( hb.x + offset1 ) >> shift1 ) << 16 );
        hbuf[rp * w + 2 * cp + 1] = ( (uint32_t)( ( ha.y + offset1 ) >> shift1 ) & 0xffffu ) | ( (uint32_t)( ( hb.y + offset1 ) >> shift1 ) << 16 );
      }
      __syncthreads();
      // ---- vertical pass: item = (vertical offset j, cell row ty, column x) -> up to 8 prediction pels of column x
      for( int it = tid; it < 7 * cellsY * w; it += T )
      {
        const int jc = div_rcp( it, invW ), x = it - jc * w;
        const int j = jc / cellsY, ty = jc - j * cellsY;
        const int qy = j - 3;
        const PackedTaps<8> Y = sTaps[qy & 3];
        const int q = ( qy >> 2 ) + 1 + ty * 8;
        const uint32_t* hp = hbuf + ( q >> 1 ) * w + x;
        const bool odd = ( q & 1 ) != 0;
        uint32_t P[8];
#pragma unroll
        for( int k = 0; k < 8; k++ ) P[k] = hp[k * w];
        int16_t* pc = pred + ( j * h + ty * 8 ) * w + x;
        const int rows = min( 8, h - ty * 8 );
#pragma unroll
        for( int m = 0; m < 4; m++ )
        {
          const int2 v = filter_pair<8>( P + m, odd, Y );
          if( 2 * m < rows )     pc[( 2 * m ) * w]     = (int16_t) max( min( ( v.x + offset2 ) >> shift2, maxv ), 0 );
          if( 2 * m + 1 < rows ) pc[( 2 * m + 1 ) * w] = (int16_t) max( min( ( v.y + offset2 ) >> shift2, maxv ), 0 );
        }
      }
      __syncthreads();
      // ---- distortion of the seven blocks: one warp per block
      for( int j = warp; j < 7; j += nWarps )
      {
        const int16_t* pj = pred + j * h * w;
        uint32_t s = 0;
        if( family == 1 )
        {
          for( int k = lane; k < h * hw; k += 32 )
          {
            const uint32_t a = orgW[k], c = reinterpret_cast<const uint32_t*>( pj )[k];
            s += (uint32_t)( abs( lo16( a ) - lo16( c ) ) + abs( hi16( a ) - hi16( c ) ) );
          }
          s = __reduce_add_sync( 0xffffffffu, s );
        }
        else
        {
          const int tw = hs.fast16 ? 8 : hs.tw;
          if( tw == 16 )     s = frac_warp_had<16>( orgS, pj, w, h, hs, lane );
          else if( tw == 8 ) s = frac_warp_had<8>( orgS, pj, w, h, hs, lane );
          else               s = frac_warp_had<4>( orgS, pj, w, h, hs, lane );
        }
        if( lane == 0 ) sOut[j * 7 + i] = s;
      }
      __syncthreads();
    }
    for( int k = tid; k < 49; k += T ) out[(size_t) b * 49 + k] = sOut[k];
  }
}

} // namespace vvb
