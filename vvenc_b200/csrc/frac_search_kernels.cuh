// frac_search_kernels.cuh -- the fractional motion refinement, InterSearch::xPatternSearchFracDIF (EncoderLib/InterSearch.cpp:2678-2724), on the device.
//
// One CTA per PU, persistent CTAs over the PU list.  The reference window around the integer vector (h + 8 rows, w + 8 pels) and the original block
// are staged once.  Each round lists the quarter-pel offsets it needs, grouped by horizontal offset: per group the horizontal pass runs once over the
// window (filter_row_pair, as frac_grid_kernel) and the vertical pass writes one filtered block per listed offset into a shared-memory slot; the warps
// then sum the distortion of the filled slots (SAD, or the tiles of xGetHADs through frac_warp_had), a slot split into row bands when there are fewer
// slots than warps.  Large PUs hold fewer slots (three for 128x128), so their groups are evaluated one after the other.
//   half-pel round: all nine positions of s_acMvRefineH.  With m_fastSubPel = 1 the member stops early (:808-811); positions it never reaches are
//                   evaluated but not used, the selection below replays the member's order and its distH values.
//   quarter-pel round: the offsets of s_acMvRefineQ around the half-pel best that s_skipQpelPosition leaves for the pattern id (all nine with
//                   m_fastSubPel = 0); offset (0, 0) is the half-pel best itself, whose distortion the half-pel round already has.
// The selection of each round (strict `<` in the member's order, the starting uiDistBest of :769, the early stops, the pattern id of :886-969 in
// wrapping Distortion arithmetic) runs on one thread, the MV rate from the host-computed table (mv_cost, cost scale 1 and 0, :2696, :2714).
// Reads are not clamped: a PU is evaluated only when its window, columns x + mv - 5 .. x + mv + w + 4 (the filter reach of the +-1 pel refinement plus
// the pel-pair rounding of stage_pel_pairs) and rows y + mv - 4 .. y + mv + h + 3, lies inside the reference margin; any other PU gets cost ~0.
#pragma once
#include "common.cuh"
#include "frac_kernels.cuh"
#include "search_kernels.cuh"

namespace vvb {

struct FracSearchPar { int w, h, family /* 1 SAD, 2 HAD, 3 HAD_fast */, fast, quarter, slots; };

// dynamic shared memory of the largest PU: 128x128 holds its window, the filtered rows, the original and three filtered blocks (the static part stays below 1 KB)
#define FRAC_SEARCH_SMEM ( 226 * 1024 )

static_assert( sizeof( vvb_frac_best ) == 16, "vvb_frac_best layout" );

struct FracSearchSmem { int winPitch, winWords, hWords, orgWords, slotWords, base; };
__host__ __device__ inline FracSearchSmem frac_search_smem( int w, int h )
{
  FracSearchSmem m;
  m.winPitch  = w / 2 + 6;                       // as frac_smem: w + 8 pels, the pair alignment and one word of slack
  m.winWords  = ( h + 8 ) * m.winPitch;
  m.hWords    = ( ( h + 8 ) / 2 + 4 ) * w;       // + slack: the vertical pass always reads 8 row pairs
  m.orgWords  = h * w / 2;
  m.slotWords = h * w / 2;
  m.base      = m.winWords + m.hWords + m.orgWords;
  return m;
}

// whether the window of a PU at (x, y) with integer vector (mx, my) lies inside the reference plane's margin (the admission rule of the host call)
__host__ __device__ inline bool frac_search_admitted( const Plane& ref, long long x, long long y, long long mx, long long my, int w, int h )
{
  const long long m = ref.margin;
  return x + mx - 5 >= -m && x + mx + w + 4 <= ref.width + m - 1 && y + my - 4 >= -m && y + my + h + 3 <= ref.height + m - 1;
}

// s_acMvRefineH / s_acMvRefineQ (InterSearch.cpp:67-91) and s_skipQpelPosition (:93-137) as one 9-bit mask per pattern id, bit i = position i skipped
__constant__ signed char c_refineH[9][2] = { { 0, 0 }, { 0, -1 }, { 0, 1 }, { -1, 0 }, { 1, 0 }, { -1, -1 }, { 1, -1 }, { -1, 1 }, { 1, 1 } };
__constant__ signed char c_refineQ[9][2] = { { 0, 0 }, { 0, -1 }, { 0, 1 }, { -1, -1 }, { 1, -1 }, { -1, 0 }, { 1, 0 }, { -1, 1 }, { 1, 1 } };
__constant__ unsigned short c_skipQpel[42] = { 510, 479, 447, 509, 469, 429, 507, 347, 187, 123, 479, 347, 447, 187, 485, 479, 469, 447, 429, 175, 509,
                                               429, 507, 187, 343, 509, 469, 507, 347, 447, 507, 187, 479, 507, 347, 447, 509, 429, 479, 509, 469, 0 };

// the switch of InterSearch.cpp:886-969 after the half-pel round, in uint64 wrap-around arithmetic (Distortion; unvisited positions hold MAX_DISTORTION)
__device__ __forceinline__ int frac_pattern_id( unsigned long long* d, int dir )
{
  const unsigned long long TH = 17, TL = 15;
  auto ratio = [&]( int a, int b, int hi, int lo ) { d[a] <<= 4; return d[a] > TH * d[b] ? hi : ( d[a] < TL * d[b] ? lo : 0 ); };
  auto slope = [&]( int a, int c, int b ) { return d[a] - d[c] > d[c] - d[b] ? 1 : 0; };
  int p = 41;
  switch( dir )
  {
    case 0: p += ratio( 3, 4, 2, 1 ); p += ratio( 1, 2, 6, 3 ); return p;
    case 1: p += ratio( 5, 6, 4, 2 ); p += slope( 2, 0, 1 ); return p + ( p == 41 ? 0 : 8 );
    case 2: p += ratio( 7, 8, 4, 2 ); p += slope( 1, 0, 2 ); return p + ( p == 41 ? 0 : 13 );
    case 3: p += slope( 4, 0, 3 ); p += ratio( 5, 7, 4, 2 ); return p + ( p == 41 ? 0 : 18 );
    case 4: p += slope( 3, 0, 4 ); p += ratio( 6, 8, 4, 2 ); return p + ( p == 41 ? 0 : 23 );
    case 5: p += slope( 6, 1, 5 ); p += 2 * slope( 7, 3, 5 ); return p + ( p == 41 ? 0 : 28 );
    case 6: p += slope( 5, 1, 6 ); p += 2 * slope( 8, 4, 6 ); return p + ( p == 41 ? 0 : 31 );
    case 7: p += slope( 8, 2, 7 ); p += 2 * slope( 5, 3, 7 ); return p + ( p == 41 ? 0 : 34 );
    default: p += slope( 7, 2, 8 ); p += 2 * slope( 6, 4, 8 ); return p + ( p == 41 ? 0 : 37 );
  }
}

// a listed offset: quarter-pel qx, qy in -3..3 and the entry of sDist it fills
__device__ __forceinline__ int frac_item( int qx, int qy, int dst ) { return ( qx + 8 ) | ( ( qy + 8 ) << 8 ) | ( dst << 16 ); }

struct FracSearchCta
{
  const FracSearchPar& p;
  const uint32_t* win; uint32_t* hbuf; const int16_t* org; int16_t* slots;
  const PackedTaps<8>* taps; const int* list; uint32_t* dist;
  int o, tid, T, lane, warp, nWarps, maxv, shift1, offset1, shift2, offset2;
  HadShape hs;

  // distortion of the `count` filled slots, list entries first .. first + count - 1, summed into dist[]
  __device__ __forceinline__ void distortion( int first, int count )
  {
    const int w = p.w, h = p.h;
    const int tileRows = p.family == 1 ? min( 8, h ) : ( hs.fast16 ? 16 : hs.th );
    int bands = 1;
    while( 2 * bands <= h / tileRows && count * bands < nWarps ) bands *= 2;
    const int rows = h / bands;
    for( int it = warp; it < count * bands; it += nWarps )
    {
      const int s = it / bands, band = it - s * bands;
      const int16_t* ob = org + band * rows * w;
      const int16_t* pb = slots + (size_t) s * h * w + band * rows * w;
      uint32_t v = 0;
      if( p.family == 1 )
      {
        const uint32_t* a = reinterpret_cast<const uint32_t*>( ob );
        const uint32_t* c = reinterpret_cast<const uint32_t*>( pb );
        for( int k = lane; k < rows * w / 2; k += 32 ) v += (uint32_t)( abs( lo16( a[k] ) - lo16( c[k] ) ) + abs( hi16( a[k] ) - hi16( c[k] ) ) );
        v = __reduce_add_sync( 0xffffffffu, v );
      }
      else
      {
        const int tw = hs.fast16 ? 8 : hs.tw;
        if( tw == 16 )     v = frac_warp_had<16>( ob, pb, w, rows, hs, lane );
        else if( tw == 8 ) v = frac_warp_had<8>( ob, pb, w, rows, hs, lane );
        else               v = frac_warp_had<4>( ob, pb, w, rows, hs, lane );
      }
      if( lane == 0 ) atomicAdd( &dist[list[first + s] >> 16], v );
    }
  }

  // the filtered blocks of list[0 .. n - 1] (grouped by qx) and their distortions
  __device__ __forceinline__ void evaluate( int n )
  {
    const int w = p.w, h = p.h, hw = w >> 1;
    const int perCol = ( ( h + 8 ) >> 1 ) * hw, cellsY = ( h + 7 ) >> 3;
    const float invHw = 1.0f / (float) hw, invW = 1.0f / (float) w;
    int first = 0, filled = 0;
    for( int g = 0; g < n; )
    {
      const int qx = ( list[g] & 0xff ) - 8;
      int ge = g + 1;
      while( ge < n && ( list[ge] & 0xff ) - 8 == qx ) ge++;
      if( filled + ge - g > p.slots ) { distortion( first, filled ); __syncthreads(); first = g; filled = 0; }
      // horizontal pass (filterHor, isLast = false) for offset qx, as frac_grid_generic_kernel
      {
        const int e = ( qx >> 2 ) + 1 + o, eo = e & 1, ew = e >> 1;
        const PackedTaps<8> X = taps[qx & 3];
        for( int it = tid; it < perCol; it += T )
        {
          const int rp = div_rcp( it, invHw ), cp = it - rp * hw;
          const uint32_t* ra = win + ( 2 * rp ) * ( hw + 6 ) + cp + ew;
          int2 ha, hb;
          filter_row_pair<8>( ra, ra + hw + 6, eo, X, ha, hb );
          hbuf[rp * w + 2 * cp]     = ( (uint32_t)( ( ha.x + offset1 ) >> shift1 ) & 0xffffu ) | ( (uint32_t)( ( hb.x + offset1 ) >> shift1 ) << 16 );
          hbuf[rp * w + 2 * cp + 1] = ( (uint32_t)( ( ha.y + offset1 ) >> shift1 ) & 0xffffu ) | ( (uint32_t)( ( hb.y + offset1 ) >> shift1 ) << 16 );
        }
      }
      __syncthreads();
      // vertical pass (filterVer, isFirst = false, isLast = true): item = (listed offset, cell row, column) -> up to 8 pels of the column
      const int items = cellsY * w;
      for( int it = tid; it < ( ge - g ) * items; it += T )
      {
        const int k = it / items, r = it - k * items;
        const int ty = div_rcp( r, invW ), x = r - ty * w;
        const int qy = ( ( list[g + k] >> 8 ) & 0xff ) - 8;
        const PackedTaps<8> Y = taps[qy & 3];
        const int q = ( qy >> 2 ) + 1 + ty * 8;
        const uint32_t* hp = hbuf + ( q >> 1 ) * w + x;
        const bool odd = ( q & 1 ) != 0;
        uint32_t P[8];
#pragma unroll
        for( int j = 0; j < 8; j++ ) P[j] = hp[j * w];
        int16_t* pc = slots + (size_t)( filled + k ) * h * w + ty * 8 * w + x;
        const int rows = min( 8, h - ty * 8 );
#pragma unroll
        for( int m = 0; m < 4; m++ )
        {
          const int2 v = filter_pair<8>( P + m, odd, Y );
          if( 2 * m < rows )     pc[( 2 * m ) * w]     = (int16_t) max( min( ( v.x + offset2 ) >> shift2, maxv ), 0 );
          if( 2 * m + 1 < rows ) pc[( 2 * m + 1 ) * w] = (int16_t) max( min( ( v.y + offset2 ) >> shift2, maxv ), 0 );
        }
      }
      __syncthreads();                 // the slots are written, and hbuf is free for the next group
      filled += ge - g;
      g = ge;
    }
    if( filled ) distortion( first, filled );
    __syncthreads();
  }
};

// Where frac_search_kernel's PUs, original block and results come from.  FracOrgPlane: vvb_frac_search -- vvb_tz_search's PU list, the PU's block of the
// original plane, vvb_frac_best.  (bipred_kernels.cuh has the other source: the bi-prediction target 2 * org - pred.)
struct FracOrgPlane
{
  using Pu = vvb_tz_pu;
  using Out = vvb_frac_best;
  // the original pels ( 2 * i, 2 * i + 1 ) of PU b's compact block, q pointing at the first of them in the plane
  __device__ __forceinline__ uint32_t org_pair( const int16_t* q, int, int ) const { return (uint32_t)(uint16_t) __ldg( q ) | ( (uint32_t)(uint16_t) __ldg( q + 1 ) << 16 ); }
  __device__ __forceinline__ void fail( Out* out, int b ) const { vvb_frac_best r{}; r.cost = ~0ull; out[b] = r; }
  __device__ __forceinline__ void done( Out* out, int b, const Pu&, int, int, const vvb_frac_best& r ) const { out[b] = r; }
};

// Src: where the PUs, the original block and the results come from.  Extra: the kernel parameters Src is built from -- none for FracOrgPlane, so its
// instantiation keeps the parameter list and the code of the kernel before Src existed.
template<class Src, class... Extra>
__global__ void __launch_bounds__( 256, 2 ) frac_search_kernel( const __grid_constant__ Plane orgPlane, const __grid_constant__ Plane refPlane,
                                                             const typename Src::Pu* __restrict__ pus, const vvb_tz_best* __restrict__ intMv, int n,
                                                             const __grid_constant__ FracSearchPar p, const __grid_constant__ FracFilter flt,
                                                             const __grid_constant__ MePar mpHalf, const __grid_constant__ MePar mpQter, typename Src::Out* __restrict__ out,
                                                             Extra... extra )
{
  extern __shared__ __align__( 16 ) uint32_t sFs[];
  __shared__ uint32_t sMv[VVB_MVCOST_ENTRIES];
  __shared__ PackedTaps<8> sTaps[4];
  __shared__ uint32_t sDist[18];             // [0..8] half-pel positions, [9..17] quarter-pel positions
  __shared__ int sList[9], sCount, sHalf, sPattern;
  __shared__ unsigned long long sBest, sDistH[9];        // distH of the half-pel round (thread 0)
  const FracSearchSmem L = frac_search_smem( p.w, p.h );
  const int w = p.w, h = p.h, tid = threadIdx.x, T = blockDim.x;
  FracSearchCta C{ p };
  C.win = sFs; C.hbuf = sFs + L.winWords;
  C.org = reinterpret_cast<const int16_t*>( C.hbuf + L.hWords );
  C.slots = reinterpret_cast<int16_t*>( sFs + L.base );
  C.taps = sTaps; C.list = sList; C.dist = sDist;
  C.tid = tid; C.T = T; C.lane = tid & 31; C.warp = tid >> 5; C.nWarps = T >> 5;
  const int bd = refPlane.bitDepth, headRoom = 14 - bd;
  C.maxv = ( 1 << bd ) - 1;
  C.shift1 = 6 - headRoom; C.offset1 = -( 8192 << C.shift1 );
  C.shift2 = 6 + headRoom; C.offset2 = ( 1 << ( C.shift2 - 1 ) ) + ( 8192 << 6 );
  C.hs.tw = 8; C.hs.th = 8; C.hs.fast16 = 0;
  if( p.family >= 2 ) had_shape( w, h, p.family == 3, C.hs );
  for( int i = tid; i < VVB_MVCOST_ENTRIES; i += T ) sMv[i] = mpHalf.tab.cost[i];
  if( tid < 4 ) sTaps[tid] = frac_taps( flt, tid );
  for( int i = ( ( h + 8 ) / 2 ) * w + tid; i < L.hWords; i += T ) C.hbuf[i] = 0u;     // the slack rows stay defined
  uint32_t* orgW = C.hbuf + L.hWords;

  for( int b = blockIdx.x; b < n; b += gridDim.x )
  {
    const typename Src::Pu pu = pus[b];
    const int mx = intMv[b].mv_hor, my = intMv[b].mv_ver;
    if( pu.x < 0 || pu.y < 0 || pu.x > orgPlane.width - w || pu.y > orgPlane.height - h || !frac_search_admitted( refPlane, pu.x, pu.y, mx, my, w, h ) )
    {
      if( tid == 0 ) Src{ extra... }.fail( out, b );
      continue;
    }
    __syncthreads();                         // the previous PU is done with the shared buffers
    C.o = stage_pel_pairs( sFs, L.winPitch, refPlane.origin + (ptrdiff_t)( pu.y + my - 4 ) * refPlane.stride + pu.x + mx - 4, refPlane.stride, w + 8, h + 8, tid, T );
    {
      const int16_t* src = orgPlane.origin + (ptrdiff_t) pu.y * orgPlane.stride + pu.x;
      const int hw = w >> 1;
      const float invHw = 1.0f / (float) hw;
      for( int i = tid; i < h * hw; i += T )
      {
        const int y = div_rcp( i, invHw ), c = i - y * hw;
        const int16_t* q = src + (ptrdiff_t) y * orgPlane.stride + 2 * c;
        orgW[i] = Src{ extra... }.org_pair( q, b, i );
      }
    }
    if( tid < 18 ) sDist[tid] = 0u;
    if( tid < 9 )                            // the half-pel positions grouped by horizontal offset: -1 (3, 5, 7), 0 (0, 1, 2), +1 (4, 6, 8)
    {
      const int i = tid < 3 ? 3 + 2 * tid : tid < 6 ? tid - 3 : 4 + 2 * ( tid - 6 );
      sList[tid] = frac_item( 2 * c_refineH[i][0], 2 * c_refineH[i][1], i );
    }
    __syncthreads();
    C.evaluate( 9 );

    // half-pel round (xPatternRefinement with iFrac = 2, cost scale 1) and the quarter-pel list
    const int bx = mx * 2, by = my * 2;
    if( tid == 0 )
    {
      unsigned long long best = ~0ull, *distH = sDistH;
      int dir = 0;
      for( int i = 0; i < 9; i++ ) distH[i] = ~0ull;
      for( int i = 0; i < 9; i++ )
      {
        if( p.fast && ( ( i == 5 && dir == 0 ) || ( i == 7 && dir == 1 ) || ( i == 8 && ( dir == 1 || dir == 3 || dir == 5 ) ) ) ) break;
        const unsigned long long c = (unsigned long long) sDist[i] + mv_cost( mpHalf, sMv, bx + c_refineH[i][0], by + c_refineH[i][1], pu.pred_hor, pu.pred_ver );
        distH[i] = c;
        if( c < best ) { best = c; dir = i; }
      }
      const int pattern = p.fast ? frac_pattern_id( distH, dir ) - 41 : 41;
      int cnt = 0;
      if( p.quarter && pattern != 0 )
      {
        const unsigned skip = p.fast ? c_skipQpel[pattern] : 0u;
        for( int dx = -1; dx <= 1; dx++ )
          for( int i = 1; i < 9; i++ )
            if( c_refineQ[i][0] == dx && !( ( skip >> i ) & 1 ) )
              sList[cnt++] = frac_item( 2 * c_refineH[dir][0] + dx, 2 * c_refineH[dir][1] + c_refineQ[i][1], 9 + i );
        sDist[9] = sDist[dir];               // quarter-pel offset (0, 0) is the half-pel best
      }
      sCount = cnt; sBest = best; sHalf = dir; sPattern = pattern;
    }
    __syncthreads();
    const int cnt = sCount;
    if( cnt ) C.evaluate( cnt );

    // quarter-pel round (iFrac = 1, cost scale 0): uiDistBest starts from the half-pel best with m_fastSubPel = 1, from MAX_DISTORTION otherwise (:769)
    if( tid == 0 )
    {
      const int dir = sHalf, pattern = sPattern;
      unsigned long long best = sBest;
      int qdir = 0;
      if( p.quarter && pattern != 0 )
      {
        const unsigned skip = p.fast ? c_skipQpel[pattern] : 0u;
        if( !p.fast ) best = ~0ull;
        const int qbx = ( bx + c_refineH[dir][0] ) * 2, qby = ( by + c_refineH[dir][1] ) * 2;
        for( int i = 0; i < 9; i++ )
        {
          if( ( skip >> i ) & 1 ) continue;
          const unsigned long long c = (unsigned long long) sDist[9 + i] + mv_cost( mpQter, sMv, qbx + c_refineQ[i][0], qby + c_refineQ[i][1], pu.pred_hor, pu.pred_ver );
          if( c < best ) { best = c; qdir = i; }
        }
      }
      vvb_frac_best r;
      r.half_hor = c_refineH[dir][0]; r.half_ver = c_refineH[dir][1];
      r.qter_hor = c_refineQ[qdir][0]; r.qter_ver = c_refineQ[qdir][1];
      r.cost = best;
      Src{ extra... }.done( out, b, pu, mx, my, r );
    }
  }
}

} // namespace vvb
