// tz_kernels.cuh -- the TZ integer motion search, InterSearch::xTZSearch (EncoderLib/InterSearch.cpp:2297-2573), walked on the device.
//
// One warp per PU, persistent warps over the PU list.  The original block is staged in shared memory once per PU.  The walk's control
// (start vector, zero vector, extra start candidates, integer early termination, the doubling diamond with its first-search stop, the
// zero-neighbourhood test, the adaptive or fixed raster, star refinement with its stop rule) is held identically by every lane of the
// warp.  Each round's point set -- the 4..16 points of one xTZ8PointDiamondSearch, the 4 of xTZ4PointSquareSearch, the 2 of xTZ2PointSearch,
// up to 32 raster points at a time -- is listed in shared memory in the member's order, G-lane groups evaluate its SADs in parallel
// (group_sad, packed VIMNMX.S16x2 + IDP.2A), and then every lane applies xTZSearchHelp's update (:410-438) point by point in list order,
// so the strict `<`, uiBestRound, ucPointNr and uiBestDistance evolve exactly as in the member.  The full SAD is always summed: the
// member's early exit returns a partial sum only when it already exceeds the best cost, which is decision-equivalent.
//
// Clipping happens here too, because it depends on the best vector found so far: xClipMvSearch of the start vector and of every
// candidate with their precision changes (:2329-2331, :2357-2358), and xSetSearchRange around the best vector after the candidates
// (:2372-2377, :2183-2206).  Every position the walk reads lies in the box xClipMvSearch allows (the raster and the zero-neighbourhood
// test stay between the zero vector and the search range), so the host admits a call when the reference margin covers that box.
#pragma once
#include "common.cuh"
#include "dist_kernels.cuh"
#include "search_kernels.cuh"

namespace vvb {

// what one call shares: the walk's settings, the picture geometry of the clip rules and the MV rate
struct TzPar
{
  int searchRange, extended, fast, integerET, firstSearchStop, subShift;
  int picW, picH, ctuSize, ctuLog2, heightInCtus, ifpLines;
  int w, h, nCands;
};

static_assert( sizeof( vvb_tz_pu ) == 28 && sizeof( vvb_tz_best ) == 32, "vvb_tz_pu / vvb_tz_best layout" );

#define TZ_LIST 32          // points listed and evaluated together (a diamond round lists at most 16)

struct TzClip { int horMin, horMax, verMin, verMax; };

// clipMv (CommonLib/Mv.cpp:68-80) and xClipMvSearch (InterSearch.cpp:2134-2152): limits in 1/16 pel
__host__ __device__ __forceinline__ TzClip tz_clip_box( const TzPar& p, int x, int y, bool search )
{
  TzClip c;
  c.horMax = ( p.picW + 8 - x - 1 ) << 4;
  c.horMin = ( -p.ctuSize - 8 - x + 1 ) * 16;
  int maxLumaHeight = p.picH + 8;
  if( search && p.ifpLines && ( y >> p.ctuLog2 ) + p.ifpLines + 1 < p.heightInCtus )
    maxLumaHeight = ( ( ( y >> p.ctuLog2 ) + p.ifpLines + 1 ) << p.ctuLog2 ) - p.h - 4;
  c.verMax = ( maxLumaHeight - y - 1 ) << 4;
  c.verMin = ( -p.ctuSize - 8 - y + 1 ) * 16;
  return c;
}
__host__ __device__ __forceinline__ int tz_clamp( int v, int lo, int hi ) { return min( hi, max( lo, v ) ); }
// Mv::changePrecision to a coarser precision and Mv::divideByPowerOf2 (Mv.h:134-142, 189-203): the same rounding
__host__ __device__ __forceinline__ int tz_round_shift( int v, int s ) { const int o = 1 << ( s - 1 ); return v >= 0 ? ( v + o - 1 ) >> s : ( v + o ) >> s; }

// xSetSearchRange (InterSearch.cpp:2183-2206): the integer window of range rng around mv (1/16 pel), its top left clipped by clipMv, its bottom right
// by xClipMvSearch
__host__ __device__ __forceinline__ void tz_search_range( const TzPar& p, int x, int y, int mvHor, int mvVer, int rng, int& left, int& right, int& top, int& bottom )
{
  const TzClip cm = tz_clip_box( p, x, y, false ), cs = tz_clip_box( p, x, y, true );
  const int r = rng << 4;
  const int px = tz_clamp( mvHor, cm.horMin, cm.horMax ), py = tz_clamp( mvVer, cm.verMin, cm.verMax );
  left   = tz_round_shift( tz_clamp( px - r, cm.horMin, cm.horMax ), 4 );
  top    = tz_round_shift( tz_clamp( py - r, cm.verMin, cm.verMax ), 4 );
  right  = tz_round_shift( tz_clamp( px + r, cs.horMin, cs.horMax ), 4 );
  bottom = tz_round_shift( tz_clamp( py + r, cs.verMin, cs.verMax ), 4 );
}

struct TzState
{
  unsigned long long bestSad;
  int bestX, bestY;
  uint32_t bestDistance, bestRound;
  int pointNr;
  int left, right, top, bottom;     // TZSearchStruct::searchRange
};

// the start of a walk: no best cost yet, the zero vector, a zero search range
__device__ __forceinline__ void tz_reset( TzState& s )
{
  s.bestSad = ~0ull; s.bestX = 0; s.bestY = 0; s.bestDistance = 0; s.bestRound = 0; s.pointNr = 0;
  s.left = s.right = s.top = s.bottom = 0;
}

// one warp's view of the walk: the staged original, the point list, the SADs of the listed points
struct TzWarp
{
  int16_t* org;                     // shared, w x h compact
  int4* pts;                        // shared [TZ_LIST]: x, y, ucPointNr (-1: an extra start candidate), distance
  uint32_t* sad;                    // shared [TZ_LIST]
  const int16_t* ref;               // reference plane at the PU position
  int refStride, lane, cnt;
};

template<int G>
__device__ __forceinline__ void tz_flush( TzWarp& W, TzState& s, const TzPar& p, const MePar& mp, const uint32_t* tab, int predHor, int predVer )
{
  if( W.cnt == 0 ) return;
  __syncwarp();
  const int lg = W.lane & ( G - 1 ), grp = W.lane / G;
  for( int k = grp; k < W.cnt; k += 32 / G )
  {
    const int4 q = W.pts[k];
    const uint32_t v = group_sad<G, true>( W.org, p.w, W.ref + (ptrdiff_t) q.y * W.refStride + q.x, W.refStride, p.w, p.h, p.subShift, lg );
    if( lg == 0 ) W.sad[k] = v;
  }
  __syncwarp();
  for( int k = 0; k < W.cnt; k++ )          // xTZSearchHelp in list order, in every lane
  {
    const int4 q = W.pts[k];
    const unsigned long long c = (unsigned long long) W.sad[k] + mv_cost( mp, tab, q.x, q.y, predHor, predVer );
    if( c < s.bestSad )
    {
      s.bestSad = c; s.bestX = q.x; s.bestY = q.y;
      if( q.z >= 0 ) { s.bestDistance = (uint32_t) q.w; s.bestRound = 0; s.pointNr = q.z; }
    }
  }
  __syncwarp();                             // the list is rewritten next
  W.cnt = 0;
}

// the two untested neighbours of the best point per ucPointNr (:446-447)
__constant__ int c_tzOffX[2][9] = { {  0, -1, -1,  0, -1, +1, -1, -1, +1 }, {  0,  0, +1, +1, -1, +1,  0, +1,  0 } };
__constant__ int c_tzOffY[2][9] = { {  0,  0, -1, -1, +1, -1,  0, +1,  0 }, {  0, -1, -1,  0, -1, +1, +1, +1, +1 } };

template<int G> struct TzWalk
{
  TzWarp& W; TzState& s; const TzPar& p; const MePar& mp; const uint32_t* tab; int predHor, predVer;

  __device__ __forceinline__ void add( int x, int y, int nr, int dist )
  {
    if( W.lane == 0 ) W.pts[W.cnt] = make_int4( x, y, nr, dist );
    W.cnt++;
  }
  __device__ __forceinline__ void flush() { tz_flush<G>( W, s, p, mp, tab, predHor, predVer ); }
  __device__ __forceinline__ void help( int x, int y, int nr, int dist ) { add( x, y, nr, dist ); flush(); }

  // xTZ2PointSearch (:442-467)
  __device__ __forceinline__ void twoPoint()
  {
    const int n = s.pointNr;
    const int x1 = s.bestX + c_tzOffX[0][n], x2 = s.bestX + c_tzOffX[1][n];
    const int y1 = s.bestY + c_tzOffY[0][n], y2 = s.bestY + c_tzOffY[1][n];
    if( x1 >= s.left && x1 <= s.right && y1 >= s.top && y1 <= s.bottom ) add( x1, y1, 0, 2 );
    if( x2 >= s.left && x2 <= s.right && y2 >= s.top && y2 <= s.bottom ) add( x2, y2, 0, 2 );
    flush();
  }
  // xTZ4PointSquareSearch (:469-504)
  __device__ __forceinline__ void square4( int sx, int sy, int d )
  {
    const int top = sy - d, bottom = sy + d, left = sx - d, right = sx + d;
    s.bestRound += 1;
    if( top >= s.top ) { if( left >= s.left ) add( left, top, 1, d ); if( right <= s.right ) add( right, top, 3, d ); }
    if( bottom <= s.bottom ) { if( left >= s.left ) add( left, bottom, 6, d ); if( right <= s.right ) add( right, bottom, 8, d ); }
    flush();
  }
  // xTZ8PointDiamondSearch (:557-758)
  __device__ __forceinline__ void diamond( int sx, int sy, int d, bool corners1 )
  {
    const int top = sy - d, bottom = sy + d, left = sx - d, right = sx + d;
    s.bestRound += 1;
    if( d == 1 )
    {
      if( top >= s.top )
      {
        if( corners1 ) { if( left >= s.left ) add( left, top, 1, d ); add( sx, top, 2, d ); if( right <= s.right ) add( right, top, 3, d ); }
        else add( sx, top, 2, d );
      }
      if( left >= s.left ) add( left, sy, 4, d );
      if( right <= s.right ) add( right, sy, 5, d );
      if( bottom <= s.bottom )
      {
        if( corners1 ) { if( left >= s.left ) add( left, bottom, 6, d ); add( sx, bottom, 7, d ); if( right <= s.right ) add( right, bottom, 8, d ); }
        else add( sx, bottom, 7, d );
      }
    }
    else if( d <= 8 )                       // the border checks pass for every point when the square lies inside the range
    {
      const int h2 = d >> 1, top2 = sy - h2, bottom2 = sy + h2, left2 = sx - h2, right2 = sx + h2;
      if( top >= s.top ) add( sx, top, 2, d );
      if( top2 >= s.top ) { if( left2 >= s.left ) add( left2, top2, 1, h2 ); if( right2 <= s.right ) add( right2, top2, 3, h2 ); }
      if( left >= s.left ) add( left, sy, 4, d );
      if( right <= s.right ) add( right, sy, 5, d );
      if( bottom2 <= s.bottom ) { if( left2 >= s.left ) add( left2, bottom2, 6, h2 ); if( right2 <= s.right ) add( right2, bottom2, 8, h2 ); }
      if( bottom <= s.bottom ) add( sx, bottom, 7, d );
    }
    else
    {
      if( top >= s.top ) add( sx, top, 0, d );
      if( left >= s.left ) add( left, sy, 0, d );
      if( right <= s.right ) add( right, sy, 0, d );
      if( bottom <= s.bottom ) add( sx, bottom, 0, d );
      for( int index = 1; index < 4; index++ )
      {
        const int yt = top + ( d >> 2 ) * index, yb = bottom - ( d >> 2 ) * index;
        const int xl = sx - ( d >> 2 ) * index, xr = sx + ( d >> 2 ) * index;
        if( yt >= s.top ) { if( xl >= s.left ) add( xl, yt, 0, d ); if( xr <= s.right ) add( xr, yt, 0, d ); }
        if( yb <= s.bottom ) { if( xl >= s.left ) add( xl, yb, 0, d ); if( xr <= s.right ) add( xr, yb, 0, d ); }
      }
    }
    flush();
  }
  // the raster of :2477-2483 / :2491-2497
  __device__ __forceinline__ void raster( int top, int bottom, int left, int right, int step )
  {
    for( int y = top; y <= bottom; y += step )
      for( int x = left; x <= right; x += step ) { add( x, y, 0, step ); if( W.cnt == TZ_LIST ) flush(); }
    flush();
  }

};

// per warp: org block (w * h pels, rounded to 16 bytes), the point list and its SADs; pts is the point list's offset, bytes the warp's share.  The rounding is
// written out twice: with bytes = pts + ..., ptxas gives tz_search_kernel<8> 78 registers instead of 72.
struct TzWarpSmem { int pts, bytes; };
__host__ __device__ inline TzWarpSmem tz_warp_smem( int w, int h ) { return { ( w * h * 2 + 15 ) & ~15, ( ( w * h * 2 + 15 ) & ~15 ) + TZ_LIST * 16 + TZ_LIST * 4 }; }

// The PUs a walk refuses: outside the picture, or a candidate range outside cands.  vvb_tz_pu and vvb_bi_pu name these fields alike; both kernels give such a
// PU a sentinel and both host calls refuse it.  A macro rather than a bool function, because through a function ptxas gives tz_search_kernel<4> and <8> 78
// registers instead of 72.
#define TZ_PU_OUTSIDE( p, pu ) ( (pu).x < 0 || (pu).y < 0 || (pu).x > (p).picW - (p).w || (pu).y > (p).picH - (p).h || (pu).cand_first < 0 || (pu).cand_count < 0 || \
                                 (pu).cand_first > (p).nCands - (pu).cand_count )

// the prologue of a warp-per-PU kernel: the CTA copies the MV-rate table to sMv, and each warp takes its share of the dynamic shared memory
__device__ __forceinline__ TzWarp tz_warp_begin( uint8_t* smem, uint32_t* sMv, const TzPar& p, const MePar& mp, const Plane& refPlane )
{
  for( int i = threadIdx.x; i < VVB_MVCOST_ENTRIES; i += blockDim.x ) sMv[i] = mp.tab.cost[i];
  __syncthreads();
  const TzWarpSmem L = tz_warp_smem( p.w, p.h );
  const int warp = threadIdx.x >> 5;
  uint8_t* mine = smem + (size_t) warp * L.bytes;
  TzWarp W;
  W.org = reinterpret_cast<int16_t*>( mine );
  W.pts = reinterpret_cast<int4*>( mine + L.pts );
  W.sad = reinterpret_cast<uint32_t*>( W.pts + TZ_LIST );
  W.refStride = refPlane.stride; W.lane = threadIdx.x & 31; W.cnt = 0;
  return W;
}

// the result of a finished walk: its best vector and cost, and the SAD without the vector's MV rate
__device__ __forceinline__ vvb_tz_best tz_best( const TzState& s, const MePar& mp, const uint32_t* tab, int predHor, int predVer, uint32_t bestDistance )
{
  vvb_tz_best b;
  b.mv_hor = s.bestX; b.mv_ver = s.bestY;
  b.cost = s.bestSad;
  b.sad = s.bestSad - mv_cost( mp, tab, s.bestX, s.bestY, predHor, predVer );
  b.best_distance = bestDistance; b.pad = 0;
  return b;
}

template<int G>
__global__ void __launch_bounds__( 128 ) tz_search_kernel( const __grid_constant__ Plane orgPlane, const __grid_constant__ Plane refPlane,
                                                           const vvb_tz_pu* __restrict__ pus, int n, const int32_t* __restrict__ cands,
                                                           const __grid_constant__ TzPar p, const __grid_constant__ MePar mp, vvb_tz_best* __restrict__ out )
{
  extern __shared__ __align__( 16 ) uint8_t tzSmem[];
  __shared__ uint32_t sMv[VVB_MVCOST_ENTRIES];
  TzWarp W = tz_warp_begin( tzSmem, sMv, p, mp, refPlane );
  int16_t* org = W.org;
  const int lane = W.lane, warp = threadIdx.x >> 5, warpsPerGrid = gridDim.x * ( blockDim.x >> 5 );

  for( int i = blockIdx.x * ( blockDim.x >> 5 ) + warp; i < n; i += warpsPerGrid )     // persistent warps: PUs i, i + warps of the grid, ...
  {
    const vvb_tz_pu pu = pus[i];
    if( TZ_PU_OUTSIDE( p, pu ) )
    {
      if( lane == 0 ) { vvb_tz_best b{}; b.sad = ~0ull; b.cost = ~0ull; b.best_distance = 0xffffffffu; out[i] = b; }
      continue;
    }
    __syncwarp();                           // the previous PU's org block is no longer read
    const int16_t* src = orgPlane.origin + (ptrdiff_t) pu.y * orgPlane.stride + pu.x;
    if( ( ( (uintptr_t) src & 3 ) | ( orgPlane.stride & 1 ) ) == 0 )
      for( int k = lane; k < ( p.w * p.h ) >> 1; k += 32 )
      {
        const int e = k << 1, y = e / p.w, x = e - y * p.w;
        reinterpret_cast<uint32_t*>( org )[k] = *reinterpret_cast<const uint32_t*>( src + (ptrdiff_t) y * orgPlane.stride + x );
      }
    else
      for( int e = lane; e < p.w * p.h; e += 32 ) { const int y = e / p.w; org[e] = src[(ptrdiff_t) y * orgPlane.stride + e - y * p.w]; }
    __syncwarp();
    W.ref = refPlane.origin + (ptrdiff_t) pu.y * refPlane.stride + pu.x;

    TzState s;
    tz_reset( s );
    TzWalk<G> T{ W, s, p, mp, sMv, pu.pred_hor, pu.pred_ver };
    const TzClip cs = tz_clip_box( p, pu.x, pu.y, true );

    // start vector (:2329-2338) and the zero vector (:2341-2348)
    const int mvx = tz_round_shift( tz_round_shift( tz_clamp( pu.start_hor, cs.horMin, cs.horMax ), 2 ), 2 );
    const int mvy = tz_round_shift( tz_round_shift( tz_clamp( pu.start_ver, cs.verMin, cs.verMax ), 2 ), 2 );
    T.help( mvx, mvy, 0, 0 );
    if( !p.fast && ( mvx != 0 || mvy != 0 ) && ( s.bestX != 0 || s.bestY != 0 ) ) T.help( 0, 0, 0, 0 );

    // extra start candidates (:2352-2370): only cost and position change
    for( int c = 0; c < pu.cand_count; c++ )
    {
      const int j = pu.cand_first + c;
      if( W.cnt == TZ_LIST ) T.flush();
      T.add( tz_round_shift( tz_clamp( cands[2 * j], cs.horMin, cs.horMax ), 4 ), tz_round_shift( tz_clamp( cands[2 * j + 1], cs.verMin, cs.verMax ), 4 ), -1, 0 );
    }
    T.flush();

    // xSetSearchRange around the best vector (:2372-2377)
    tz_search_range( p, pu.x, pu.y, s.bestX * 16, s.bestY * 16, p.searchRange >> ( p.fast ? 1 : 0 ), s.left, s.right, s.top, s.bottom );

    const bool ext = p.extended != 0;
    bool done = false;
    int sx = s.bestX, sy = s.bestY;
    if( p.integerET )                       // :2385-2410
    {
      T.diamond( sx, sy, 1, false );
      if( s.bestX == sx && s.bestY == sy )
      {
        if( p.w * p.h > 64 ) { T.square4( sx, sy, 1 ); done = s.bestX == sx && s.bestY == sy; }
        else done = true;
      }
    }
    if( !done )
    {
      sx = s.bestX; sy = s.bestY;
      const bool bestCandidateZero = s.bestX == 0 && s.bestY == 0;
      for( int d = 1; d <= p.searchRange; d *= 2 )            // first search (:2421-2436), stop after 3 rounds without improvement
      {
        T.diamond( sx, sy, d, ext );
        if( p.firstSearchStop && s.bestRound >= 3 ) break;
      }
      if( ext && !bestCandidateZero )                          // zero-neighbourhood test (:2438-2451)
        for( int d = 1; d <= ( p.searchRange >> 1 ); d *= 2 ) T.diamond( 0, 0, d, false );
      if( s.bestDistance == 1 ) { s.bestDistance = 0; T.twoPoint(); }
      const int iRaster = p.fast ? 8 : 5;
      if( ext )                                                // adaptive raster (:2461-2484)
      {
        int win = iRaster, l = s.left, r = s.right, t = s.top, b = s.bottom;
        if( !( (int) s.bestDistance >= iRaster ) ) { win++; l /= 2; r /= 2; t /= 2; b /= 2; }
        s.bestDistance = win;
        T.raster( t, b, l, r, win );
      }
      else if( (int) s.bestDistance >= iRaster )              // fixed raster (:2487-2498)
      {
        s.bestDistance = iRaster;
        T.raster( s.top, s.bottom, s.left, s.right, iRaster );
      }
      while( s.bestDistance > 0 )                              // star refinement (:2535-2569)
      {
        sx = s.bestX; sy = s.bestY;
        s.bestDistance = 0; s.pointNr = 0;
        for( int d = 1; d < p.searchRange + 1; d *= 2 )
        {
          T.diamond( sx, sy, d, ext );
          if( p.fast && s.bestRound >= 2 ) break;
        }
        if( s.bestDistance == 1 ) { s.bestDistance = 0; if( s.pointNr != 0 ) T.twoPoint(); }
      }
    }
    if( lane == 0 ) out[i] = tz_best( s, mp, sMv, pu.pred_hor, pu.pred_ver, s.bestDistance );
  }
}

} // namespace vvb
