// dist_kernels.cuh -- SAD / SSE / SATD (Hadamard) cost kernels for sm_90a.
//
// Replaces the function-pointer surface RdCost::m_afpDistortFunc (CommonLib/RdCost.h:120, table filled at
// CommonLib/RdCost.cpp:85-131 and overwritten by CommonLib/x86/RdCostX86.h:3376-3425).  All results are exact
// integers identical to the reference (early exit is never taken: the full sum is always returned, which is
// decision-equivalent, SURVEY.md 7-2).
//
// Work decomposition: a *group* of G lanes (G = 4..32, power of two) evaluates one candidate; groups are packed
// into warps so that 4x4 blocks do not waste 28 lanes.  SAD runs on packed 16x2 halfwords (VIMNMX.S16x2 + IDP.2A),
// SATD keeps one tile row per lane (horizontal butterflies in registers, vertical butterflies over lane shuffles).
#pragma once
#include "common.cuh"

namespace vvb {

enum { FAM_SSE = 0, FAM_SAD = 1, FAM_HAD = 2, FAM_HAD_FAST = 3, FAM_HAD_2SAD = 4 };

// ---------------------------------------------------------------------------------------------------------------
// SAD: sum over rows y = 0, s, 2s.. (s = 1<<subShift) of sum_x |org - cur|, result << subShift
// (CommonLib/RdCost.cpp:300-335; every width-specialised variant computes the same value)
// ---------------------------------------------------------------------------------------------------------------
// SMEM: org points into shared memory (a block staged once and searched many times) and is read with plain loads
template<bool SMEM, class T> __device__ __forceinline__ T org_load( const T* p ) { if constexpr( SMEM ) return *p; else return __ldg( p ); }

template<int G, bool ORG_SMEM = false>
__device__ __forceinline__ uint32_t group_sad( const int16_t* __restrict__ org, int so, const int16_t* __restrict__ cur, int sc,
                                               int w, int h, int subShift, int lg )
{
  const int lw   = ilog2_dev( w );
  const int rows = ( h + ( 1 << subShift ) - 1 ) >> subShift;
  int acc = 0;
  const uintptr_t ao = (uintptr_t) org, ac = (uintptr_t) cur;
  if( w >= 8 && ( ( ao | ac ) & 15 ) == 0 && ( ( so | sc ) & 7 ) == 0 )
  {
    // 8 pels (16 B) per load
    const int cpr = w >> 3, total = rows * cpr, lc = lw - 3;
    for( int i = lg; i < total; i += G )
    {
      const int r = i >> lc, c = i & ( cpr - 1 ), y = r << subShift;
      const uint4 a = org_load<ORG_SMEM>( reinterpret_cast<const uint4*>( org + (size_t) y * so ) + c );
      const uint4 b = __ldg( reinterpret_cast<const uint4*>( cur + (size_t) y * sc ) + c );
      acc = sad2_acc( a.x, b.x, acc ); acc = sad2_acc( a.y, b.y, acc );
      acc = sad2_acc( a.z, b.z, acc ); acc = sad2_acc( a.w, b.w, acc );
    }
  }
  else if( w >= 2 && ( ( ao | ac ) & 3 ) == 0 && ( ( so | sc ) & 1 ) == 0 )
  {
    const int cpr = w >> 1, total = rows * cpr, lc = lw - 1;
    for( int i = lg; i < total; i += G )
    {
      const int r = i >> lc, c = i & ( cpr - 1 ), y = r << subShift;
      const uint32_t a = org_load<ORG_SMEM>( reinterpret_cast<const uint32_t*>( org + (size_t) y * so ) + c );
      const uint32_t b = __ldg( reinterpret_cast<const uint32_t*>( cur + (size_t) y * sc ) + c );
      acc = sad2_acc( a, b, acc );
    }
  }
  else
  {
    const int total = rows << lw;
    for( int i = lg; i < total; i += G )
    {
      const int r = i >> lw, x = i & ( w - 1 ), y = r << subShift;
      acc += abs( (int) org_load<ORG_SMEM>( org + (size_t) y * so + x ) - (int) __ldg( cur + (size_t) y * sc + x ) );
    }
  }
  return group_sum_u32<G>( (uint32_t) acc ) << subShift;
}

// SSE (CommonLib/RdCost.cpp:651-1000): 64-bit exact
template<int G, bool ORG_SMEM = false>
__device__ __forceinline__ unsigned long long group_sse( const int16_t* __restrict__ org, int so, const int16_t* __restrict__ cur, int sc,
                                                         int w, int h, int lg )
{
  const int lw = ilog2_dev( w );
  unsigned long long acc = 0;
  if( w >= 2 && ( ( (uintptr_t) org | (uintptr_t) cur ) & 3 ) == 0 && ( ( so | sc ) & 1 ) == 0 )
  {
    const int cpr = w >> 1, total = h * cpr, lc = lw - 1;
    for( int i = lg; i < total; i += G )
    {
      const int y = i >> lc, c = i & ( cpr - 1 );
      const uint32_t a = org_load<ORG_SMEM>( reinterpret_cast<const uint32_t*>( org + (size_t) y * so ) + c );
      const uint32_t b = __ldg( reinterpret_cast<const uint32_t*>( cur + (size_t) y * sc ) + c );
      const int d0 = lo16( a ) - lo16( b ), d1 = hi16( a ) - hi16( b );
      acc += (unsigned long long)( (long long) d0 * d0 ) + (unsigned long long)( (long long) d1 * d1 );
    }
  }
  else
  {
    const int total = h << lw;
    for( int i = lg; i < total; i += G )
    {
      const int y = i >> lw, x = i & ( w - 1 );
      const int d = (int) org_load<ORG_SMEM>( org + (size_t) y * so + x ) - (int) __ldg( cur + (size_t) y * sc + x );
      acc += (unsigned long long)( (long long) d * d );
    }
  }
  return group_sum_u64<G>( acc );
}

// ---------------------------------------------------------------------------------------------------------------
// SATD.  Tile rules and normalisations: CommonLib/RdCost.cpp:1818-1938 (dispatch), :1006-1766 (tiles).
// ---------------------------------------------------------------------------------------------------------------
struct HadShape { int tw, th, fast16; };

__device__ __forceinline__ bool had_shape( int w, int h, int fast, HadShape& s )
{
  s.fast16 = 0;
  if(      w > h && ( h & 7 ) == 0 && ( w & 15 ) == 0 ) { s.tw = 16; s.th = 8; }
  else if( w < h && ( w & 7 ) == 0 && ( h & 15 ) == 0 ) { s.tw = 8;  s.th = 16; }
  else if( w > h && ( h & 3 ) == 0 && ( w & 7 ) == 0 )  { s.tw = 8;  s.th = 4; }
  else if( w < h && ( w & 3 ) == 0 && ( h & 7 ) == 0 )  { s.tw = 4;  s.th = 8; }
  else if( fast && ( h & 31 ) == 0 && ( w & 31 ) == 0 && w == h ) { s.tw = 16; s.th = 16; s.fast16 = 1; }
  else if( ( h & 7 ) == 0 && ( w & 7 ) == 0 ) { s.tw = 8; s.th = 8; }
  else if( ( h & 3 ) == 0 && ( w & 3 ) == 0 ) { s.tw = 4; s.th = 4; }
  else if( ( h & 1 ) == 0 && ( w & 1 ) == 0 ) { s.tw = 2; s.th = 2; }
  else return false;
  return true;
}

template<int TW> __device__ __forceinline__ void wht_regs( int (&d)[TW] )
{
#pragma unroll
  for( int len = 1; len < TW; len <<= 1 )
  {
#pragma unroll
    for( int i = 0; i < TW; i += 2 * len )
    {
#pragma unroll
      for( int j = 0; j < len; j++ )
      {
        const int a = d[i + j], b = d[i + j + len];
        d[i + j] = a + b; d[i + j + len] = a - b;
      }
    }
  }
}

// loads TW differences org-cur of one tile row; also accumulates sum|d| for HAD_2SAD.  ORG_SMEM: org is read from shared memory (org_load)
template<int TW, bool ORG_SMEM = false> __device__ __forceinline__ void load_diff_row( const int16_t* __restrict__ o, const int16_t* __restrict__ c, int (&d)[TW], int& sadAcc )
{
  if( TW >= 8 && ( ( (uintptr_t) o | (uintptr_t) c ) & 15 ) == 0 )
  {
#pragma unroll
    for( int v = 0; v < TW / 8; v++ )
    {
      const uint4 a = org_load<ORG_SMEM>( reinterpret_cast<const uint4*>( o ) + v ), b = __ldg( reinterpret_cast<const uint4*>( c ) + v );
      d[8*v+0] = lo16( a.x ) - lo16( b.x ); d[8*v+1] = hi16( a.x ) - hi16( b.x );
      d[8*v+2] = lo16( a.y ) - lo16( b.y ); d[8*v+3] = hi16( a.y ) - hi16( b.y );
      d[8*v+4] = lo16( a.z ) - lo16( b.z ); d[8*v+5] = hi16( a.z ) - hi16( b.z );
      d[8*v+6] = lo16( a.w ) - lo16( b.w ); d[8*v+7] = hi16( a.w ) - hi16( b.w );
    }
  }
  else if( ( ( (uintptr_t) o | (uintptr_t) c ) & 3 ) == 0 )
  {
#pragma unroll
    for( int v = 0; v < TW / 2; v++ )
    {
      const uint32_t a = org_load<ORG_SMEM>( reinterpret_cast<const uint32_t*>( o ) + v ), b = __ldg( reinterpret_cast<const uint32_t*>( c ) + v );
      d[2*v] = lo16( a ) - lo16( b ); d[2*v+1] = hi16( a ) - hi16( b );
    }
  }
  else
  {
#pragma unroll
    for( int x = 0; x < TW; x++ ) d[x] = (int) org_load<ORG_SMEM>( o + x ) - (int) __ldg( c + x );
  }
#pragma unroll
  for( int x = 0; x < TW; x++ ) sadAcc += abs( d[x] );
}

// One tile per TH consecutive lanes.  Returns the normalised tile cost in the tile's row-0 lane, 0 elsewhere.
template<int TW> __device__ __forceinline__ uint32_t had_tile_lanes( int (&d)[TW], int th, int row, bool active, unsigned mk )
{
  wht_regs<TW>( d );
#pragma unroll 4
  for( int m = 1; m < th; m <<= 1 )
  {
    const bool up = ( row & m ) != 0;
#pragma unroll
    for( int i = 0; i < TW; i++ )
    {
      const int p = __shfl_xor_sync( mk, d[i], m );
      d[i] = up ? p - d[i] : d[i] + p;
    }
  }
  uint32_t s = 0;
#pragma unroll
  for( int i = 0; i < TW; i++ ) s += (uint32_t) abs( d[i] );
  const uint32_t dc = (uint32_t) abs( d[0] );                 // valid in row 0: the all-plus coefficient
  for( int m = 1; m < th; m <<= 1 ) s += __shfl_xor_sync( mk, s, m );
  if( !active || row != 0 ) return 0u;
  const int area = TW * th;
  if( area == 4 ) return s - dc + ( dc >> 2 );               // 2x2: RdCost.cpp:1020-1023
  s = s - dc + ( dc >> 2 );
  if( area == 16 ) return ( s + 1 ) >> 1;                    // 4x4: :1121
  if( area == 64 ) return ( s + 2 ) >> 2;                    // 8x8: :1319
  if( area == 128 ) return (uint32_t)(int)( __ddiv_rn( (double)(int) s, sqrt( 16.0 * 8 ) ) * 2.0 );   // 16x8 / 8x16: :1467,:1606
  return (uint32_t)(int)( __ddiv_rn( (double)(int) s, sqrt( 4.0 * 8 ) ) * 2.0 );                       // 8x4 / 4x8: :1682,:1763
}

template<int G, int TW, bool ORG_SMEM = false>
__device__ __forceinline__ void group_had_tw( const int16_t* __restrict__ org, int so, const int16_t* __restrict__ cur, int sc, int w, int h,
                                              const HadShape& s, int lg, uint32_t& hadSum, uint32_t& sadSum )
{
  const int th = s.fast16 ? 8 : s.th;                 // lanes per tile
  const int tilesX = w / s.tw, tilesY = h / s.th, nt = tilesX * tilesY;
  const int tpi = G / th;                             // tiles per iteration of this group
  const int row = lg % th, sub = lg / th;
  int sadAcc = 0;
  uint32_t acc = 0;
  for( int t0 = 0; t0 < nt; t0 += tpi )
  {
    const int t = t0 + sub;
    const bool active = t < nt && sub < tpi;
    int d[TW];
#pragma unroll
    for( int i = 0; i < TW; i++ ) d[i] = 0;
    if( active )
    {
      const int ty = t / tilesX, tx = t - ty * tilesX;
      if( s.fast16 )
      {
        // 2x2 rounded means of org and cur separately (RdCost.cpp:1132-1145); TW == 8 here
        const int16_t* o = org + (size_t)( ty * 16 + 2 * row ) * so + tx * 16;
        const int16_t* c = cur + (size_t)( ty * 16 + 2 * row ) * sc + tx * 16;
#pragma unroll
        for( int x = 0; x < TW; x++ )
        {
          const int ov = ( (int) org_load<ORG_SMEM>( o + 2*x ) + org_load<ORG_SMEM>( o + 2*x + 1 ) + org_load<ORG_SMEM>( o + so + 2*x ) + org_load<ORG_SMEM>( o + so + 2*x + 1 ) + 2 ) >> 2;
          const int cv = ( (int) __ldg( c + 2*x ) + __ldg( c + 2*x + 1 ) + __ldg( c + sc + 2*x ) + __ldg( c + sc + 2*x + 1 ) + 2 ) >> 2;
          d[x] = ov - cv;
        }
      }
      else
      {
        load_diff_row<TW, ORG_SMEM>( org + (size_t)( ty * s.th + row ) * so + tx * TW, cur + (size_t)( ty * s.th + row ) * sc + tx * TW, d, sadAcc );
      }
    }
    const uint32_t v = had_tile_lanes<TW>( d, th, row, active, gmask<G>() );
    acc += s.fast16 ? ( v << 2 ) : v;                 // 16x16_fast returns sad << 2 (:1222)
  }
  hadSum = group_sum_u32<G>( acc );
  sadSum = group_sum_u32<G>( (uint32_t) sadAcc );
}

// family dispatch for one candidate evaluated by a G-lane group; returns the cost in every lane of the group.  ORG_SMEM: org is a block staged in shared memory
template<int G, bool ORG_SMEM = false>
__device__ __forceinline__ unsigned long long group_dist( int fam, const int16_t* __restrict__ org, int so, const int16_t* __restrict__ cur, int sc,
                                                          int w, int h, int subShift, int lg )
{
  if( fam == FAM_SAD ) return group_sad<G, ORG_SMEM>( org, so, cur, sc, w, h, subShift, lg );
  if( fam == FAM_SSE ) return group_sse<G, ORG_SMEM>( org, so, cur, sc, w, h, lg );
  HadShape s;
  if( !had_shape( w, h, fam == FAM_HAD_FAST, s ) ) return ~0ull;
  uint32_t had = 0, sad = 0;
  const int tw = s.fast16 ? 8 : s.tw;
  if( G >= 16 && tw == 16 )     group_had_tw<G, 16, ORG_SMEM>( org, so, cur, sc, w, h, s, lg, had, sad );
  else if( tw == 8 )            group_had_tw<G, 8,  ORG_SMEM>( org, so, cur, sc, w, h, s, lg, had, sad );
  else if( tw == 4 )            group_had_tw<G, 4,  ORG_SMEM>( org, so, cur, sc, w, h, s, lg, had, sad );
  else if( tw == 2 )            group_had_tw<G, 2,  ORG_SMEM>( org, so, cur, sc, w, h, s, lg, had, sad );
  if( fam == FAM_HAD_2SAD ) return had < 2u * sad ? had : 2u * sad;       // RdCost.cpp:1815
  return had;
}

// smallest legal group size for a uniform (fam, w, h) batch
static inline int pick_group( int fam, int w, int h )
{
  int need;
  if( fam == FAM_SAD || fam == FAM_SSE ) need = ( w * h ) / 8;          // ~8 pels per lane
  else
  {
    // lanes per tile (th) times number of tiles, at least th
    int tw, th;
    if(      w > h && ( h & 7 ) == 0 && ( w & 15 ) == 0 ) { tw = 16; th = 8; }
    else if( w < h && ( w & 7 ) == 0 && ( h & 15 ) == 0 ) { tw = 8;  th = 16; }
    else if( w > h && ( h & 3 ) == 0 && ( w & 7 ) == 0 )  { tw = 8;  th = 4; }
    else if( w < h && ( w & 3 ) == 0 && ( h & 7 ) == 0 )  { tw = 4;  th = 8; }
    else if( fam == FAM_HAD_FAST && ( h & 31 ) == 0 && ( w & 31 ) == 0 && w == h ) { tw = 16; th = 8; }
    else if( ( h & 7 ) == 0 && ( w & 7 ) == 0 ) { tw = 8; th = 8; }
    else if( ( h & 3 ) == 0 && ( w & 3 ) == 0 ) { tw = 4; th = 4; }
    else { tw = 2; th = 2; }
    int tiles = ( w / tw ) * ( h / ( fam == FAM_HAD_FAST && tw == 16 && th == 8 && w == h && ( w & 31 ) == 0 ? 16 : th ) );
    need = th * tiles;
    if( need < th ) need = th;
    if( need < 4 ) need = 4;
    if( tw == 16 && need < 16 ) need = 16;
  }
  int g = 4;
  while( g < need && g < 32 ) g <<= 1;
  return g;
}

// ---------------------------------------------------------------------------------------------------------------
// kernels
// ---------------------------------------------------------------------------------------------------------------

// generic descriptor list: one warp per candidate (mixed shapes / families allowed)
__global__ void __launch_bounds__( 256 ) dist_list_kernel( const __grid_constant__ PlaneTable planes, const vvb_cand* __restrict__ cands, int n,
                                                           unsigned long long* __restrict__ out )
{
  const int lane = threadIdx.x & 31;
  const int warpsPerGrid = ( gridDim.x * blockDim.x ) >> 5;
  for( int i = ( blockIdx.x * blockDim.x + threadIdx.x ) >> 5; i < n; i += warpsPerGrid )
  {
    const vvb_cand c = cands[i];
    const Plane& po = planes.p[c.org_plane];
    const Plane& pc = planes.p[c.cur_plane];
    const int16_t* org = po.origin + (ptrdiff_t) c.org_y * po.stride + c.org_x;
    const int16_t* cur = pc.origin + (ptrdiff_t) c.cur_y * pc.stride + c.cur_x;
    const unsigned long long v = group_dist<32>( c.dfunc, org, po.stride, cur, pc.stride, c.w, c.h, c.sub_shift, lane );
    if( lane == 0 ) out[i] = v;
  }
}

// uint32 cost outputs saturate: the SSE of a 128x64 block at 10 bits or of a 32x32 block at 12 bits exceeds 32 bits and must not wrap to a small cost
__device__ __forceinline__ uint32_t sat_u32( unsigned long long v ) { return v < 0xffffffffull ? (uint32_t) v : 0xffffffffu; }

// candidate pool: candidate (b,k) = compact w*h block at pool + (b*K+k)*w*h against org block b of a plane
template<int G>
__global__ void __launch_bounds__( 256 ) dist_pool_kernel( const __grid_constant__ Plane orgPlane, const vvb_pos* __restrict__ blocks, int nBlocks,
                                                           int w, int h, int K, int fam, int subShift, const int16_t* __restrict__ pool,
                                                           uint32_t* __restrict__ out )
{
  const int lg = threadIdx.x & ( G - 1 );
  const long long groupsPerGrid = ( (long long) gridDim.x * blockDim.x ) / G;
  const long long total = (long long) nBlocks * K;
  const int area = w * h;
  for( long long i = ( (long long) blockIdx.x * blockDim.x + threadIdx.x ) / G; i < total; i += groupsPerGrid )
  {
    const int b = (int)( i / K );
    const vvb_pos p = blocks[b];
    const int16_t* org = orgPlane.origin + (ptrdiff_t) p.y * orgPlane.stride + p.x;
    const int16_t* cur = pool + (size_t) i * area;
    const unsigned long long v = group_dist<G>( fam, org, orgPlane.stride, cur, w, w, h, subShift, lg );   // shuffles use the group's own lane mask
    if( lg == 0 ) out[i] = sat_u32( v );
  }
}

// ---------------------------------------------------------------------------------------------------------------
// streaming fast paths for uniform candidate pools (HBM bound): many independent 16-byte loads in flight per lane,
// no shared memory, the original block is re-read through L1.
// ---------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ uint4 ld_stream( const uint4* p )
{
  uint4 r;
  asm volatile( "ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"( r.x ), "=r"( r.y ), "=r"( r.z ), "=r"( r.w ) : "l"( p ) );
  return r;
}

// SAD / SSE over a pool: G lanes per candidate, L = chunks (8 pels = 16 bytes) per lane per pass; the candidates of one block are walked
// by the same group.  SINGLE (chunks <= G*L, the common case): the original chunks are loaded once per block and stay in registers, the
// loop body is 4 independent streaming loads followed by arithmetic -- no branches between the loads.
// Requires w >= 8 (chunks never straddle rows) and 16-byte aligned original rows.
template<bool SSE> __device__ __forceinline__ void chunk_acc( const uint4& o, const uint4& c, int& acc, unsigned long long& acc64 )
{
  if( !SSE )
  {
    acc = sad2_acc( o.x, c.x, acc ); acc = sad2_acc( o.y, c.y, acc ); acc = sad2_acc( o.z, c.z, acc ); acc = sad2_acc( o.w, c.w, acc );
  }
  else
  {
    const uint32_t ow[4] = { o.x, o.y, o.z, o.w }, cw[4] = { c.x, c.y, c.z, c.w };
#pragma unroll
    for( int j = 0; j < 4; j++ )
    {
      const int d0 = lo16( ow[j] ) - lo16( cw[j] ), d1 = hi16( ow[j] ) - hi16( cw[j] );
      acc64 += (unsigned long long)( (unsigned) ( d0 * d0 ) ) + (unsigned long long)( (unsigned) ( d1 * d1 ) );
    }
  }
}

template<int G, int L, bool SSE, bool SINGLE>
__global__ void __launch_bounds__( 256, 3 ) sad_pool_stream_kernel( const __grid_constant__ Plane orgPlane, const vvb_pos* __restrict__ blocks, int nBlocks,
                                                                    int w, int h, int K, int kSplit, int subShift, const int16_t* __restrict__ pool,
                                                                    uint32_t* __restrict__ out )
{
  const int lg = threadIdx.x & ( G - 1 );
  const long long groupsPerGrid = ( (long long) gridDim.x * blockDim.x ) / G;
  const long long jobs = (long long) nBlocks * kSplit;                 // job = (block, slice of its K candidates)
  const int cpr = w >> 3, lcpr = ilog2_dev( cpr );                    // chunks per row (power of two)
  const int rows = h >> subShift;
  const int chunks = rows * cpr;                                       // visited chunks per candidate
  const int kPer = ( K + kSplit - 1 ) / kSplit;
  const unsigned mk = gmask<G>();
  const int area8 = ( w * h ) >> 3;                                    // uint4 units per candidate
  for( long long job = ( (long long) blockIdx.x * blockDim.x + threadIdx.x ) / G; job < jobs; job += groupsPerGrid )
  {
    const int b = (int)( job / kSplit ), ks = (int)( job - (long long) b * kSplit );
    const int k0 = ks * kPer, k1 = min( K, k0 + kPer );
    const vvb_pos p = blocks[b];
    const int16_t* org = orgPlane.origin + (ptrdiff_t) p.y * orgPlane.stride + p.x;
    if( SINGLE )
    {
      int offC[L]; uint4 o0[L];
#pragma unroll
      for( int i = 0; i < L; i++ )
      {
        const int ch = min( i * G + lg, chunks - 1 );                  // lanes past the end redo the last chunk with a zeroed original
        const int r = ch >> lcpr, cc = ch & ( cpr - 1 ), y = r << subShift;
        offC[i] = y * cpr + cc;
        o0[i] = __ldg( reinterpret_cast<const uint4*>( org + (ptrdiff_t) y * orgPlane.stride ) + cc );
      }
      const uint4* cur = reinterpret_cast<const uint4*>( pool ) + ( (size_t) b * K + k0 ) * area8;
      for( int k = k0; k < k1; k++, cur += area8 )
      {
        uint4 c[L];
#pragma unroll
        for( int i = 0; i < L; i++ ) c[i] = ld_stream( cur + offC[i] );
        int acc = 0; unsigned long long acc64 = 0;
#pragma unroll
        for( int i = 0; i < L; i++ ) if( i * G + lg < chunks ) chunk_acc<SSE>( o0[i], c[i], acc, acc64 );
        if( !SSE )
        {
          uint32_t v = (uint32_t) acc;
#pragma unroll
          for( int m = G >> 1; m > 0; m >>= 1 ) v += __shfl_xor_sync( mk, v, m );
          if( lg == 0 ) out[(size_t) b * K + k] = v << subShift;
        }
        else
        {
#pragma unroll
          for( int m = G >> 1; m > 0; m >>= 1 ) acc64 += __shfl_xor_sync( mk, acc64, m );
          if( lg == 0 ) out[(size_t) b * K + k] = sat_u32( acc64 );
        }
      }
    }
    else
    {
      const int passes = ( chunks + G * L - 1 ) / ( G * L );
      for( int k = k0; k < k1; k++ )
      {
        const uint4* cur = reinterpret_cast<const uint4*>( pool ) + ( (size_t) b * K + k ) * area8;
        int acc = 0; unsigned long long acc64 = 0;
        for( int ps = 0; ps < passes; ps++ )
        {
          uint4 c[L], o[L];
#pragma unroll
          for( int i = 0; i < L; i++ )
          {
            const int ch = min( ( ps * L + i ) * G + lg, chunks - 1 );
            const int r = ch >> lcpr, cc = ch & ( cpr - 1 ), y = r << subShift;
            c[i] = ld_stream( cur + y * cpr + cc );
            o[i] = __ldg( reinterpret_cast<const uint4*>( org + (ptrdiff_t) y * orgPlane.stride ) + cc );
          }
#pragma unroll
          for( int i = 0; i < L; i++ ) if( ( ps * L + i ) * G + lg < chunks ) chunk_acc<SSE>( o[i], c[i], acc, acc64 );
        }
        if( !SSE )
        {
          uint32_t v = (uint32_t) acc;
#pragma unroll
          for( int m = G >> 1; m > 0; m >>= 1 ) v += __shfl_xor_sync( mk, v, m );
          if( lg == 0 ) out[(size_t) b * K + k] = v << subShift;
        }
        else
        {
#pragma unroll
          for( int m = G >> 1; m > 0; m >>= 1 ) acc64 += __shfl_xor_sync( mk, acc64, m );
          if( lg == 0 ) out[(size_t) b * K + k] = sat_u32( acc64 );
        }
      }
    }
  }
}

// xCalcHADs8x8 (RdCost.cpp:1316-1319) of the 8x8 differences d[8 * row + col], all in registers; d is overwritten by its transform.
// 2-D Walsh-Hadamard: the index bits are butterflied one after another (order-free for sum|.| and for the DC term).  A caller that has already done the
// stages below bit BIT0 itself enters here with BIT0 > 0 (BIT0 = 6: d holds the transform).  The abs-sum runs as CHAINS VABSDIFF chains, four by
// default so that they can issue back to back; that is a scheduling choice, the integer sum is the same in any order.
template<int BIT0 = 0, int CHAINS = 4>
__device__ __forceinline__ uint32_t had8( int ( &d )[64] )
{
#pragma unroll
  for( int bit = BIT0; bit < 6; bit++ )
  {
#pragma unroll
    for( int i = 0; i < 64; i++ )
    {
      if( !( i & ( 1 << bit ) ) )
      {
        const int a = d[i], bb = d[i | ( 1 << bit )];
        d[i] = a + bb; d[i | ( 1 << bit )] = a - bb;
      }
    }
  }
  uint32_t acc[CHAINS] = {};
#pragma unroll
  for( int i = 0; i < 64; i++ ) acc[i % CHAINS] = __sad( d[i], 0, acc[i % CHAINS] );    // VABSDIFF: |d| + acc in one instruction
  const uint32_t dc = (uint32_t) abs( d[0] );
  uint32_t s = 0;
#pragma unroll
  for( int i = 0; i < CHAINS; i++ ) s += acc[i];
  s = s - dc + ( dc >> 2 );                                          // RdCost.cpp:1316-1318
  return ( s + 2 ) >> 2;                                             // :1319
}

// SATD with 8x8 tiles (every block whose dispatch lands on xCalcHADs8x8, RdCost.cpp:1894-1905): ONE LANE PER TILE, the whole 8x8
// Hadamard in registers (no shuffles); LPC = min(tiles, 32) lanes per candidate.  Also serves HAD_2SAD (min(SATD, 2 SAD)).
template<int LPC>
__global__ void __launch_bounds__( 128 ) had8_pool_stream_kernel( const __grid_constant__ Plane orgPlane, const vvb_pos* __restrict__ blocks, int nBlocks,
                                                                  int w, int h, int K, int with2Sad, const int16_t* __restrict__ pool, uint32_t* __restrict__ out )
{
  const int lg = threadIdx.x & ( LPC - 1 );
  const long long groupsPerGrid = ( (long long) gridDim.x * blockDim.x ) / LPC;
  const long long total = (long long) nBlocks * K;
  const int tilesX = w >> 3, T = tilesX * ( h >> 3 );
  const unsigned mk = gmask<LPC>();
  for( long long ci = ( (long long) blockIdx.x * blockDim.x + threadIdx.x ) / LPC; ci < total; ci += groupsPerGrid )
  {
    const int b = (int)( ci / K );
    const vvb_pos p = blocks[b];
    const int16_t* org = orgPlane.origin + (ptrdiff_t) p.y * orgPlane.stride + p.x;
    const int16_t* cur = pool + (size_t) ci * w * h;
    uint32_t hadSum = 0, sadSum = 0;
    for( int t = lg; t < T; t += LPC )
    {
      const int ty = t / tilesX, tx = t - ty * tilesX;
      uint4 c[8], o[8];
#pragma unroll
      for( int r = 0; r < 8; r++ ) c[r] = ld_stream( reinterpret_cast<const uint4*>( cur + ( ty * 8 + r ) * w + tx * 8 ) );
#pragma unroll
      for( int r = 0; r < 8; r++ ) o[r] = __ldg( reinterpret_cast<const uint4*>( org + (ptrdiff_t)( ty * 8 + r ) * orgPlane.stride + tx * 8 ) );
      int d[64];
#pragma unroll
      for( int r = 0; r < 8; r++ )
      {
        d[8*r+0] = lo16( o[r].x ) - lo16( c[r].x ); d[8*r+1] = hi16( o[r].x ) - hi16( c[r].x );
        d[8*r+2] = lo16( o[r].y ) - lo16( c[r].y ); d[8*r+3] = hi16( o[r].y ) - hi16( c[r].y );
        d[8*r+4] = lo16( o[r].z ) - lo16( c[r].z ); d[8*r+5] = hi16( o[r].z ) - hi16( c[r].z );
        d[8*r+6] = lo16( o[r].w ) - lo16( c[r].w ); d[8*r+7] = hi16( o[r].w ) - hi16( c[r].w );
      }
      if( with2Sad )
      {
#pragma unroll
        for( int i = 0; i < 64; i++ ) sadSum = __sad( d[i], 0, sadSum );
      }
      hadSum += had8( d );
    }
#pragma unroll
    for( int m = LPC >> 1; m > 0; m >>= 1 ) { hadSum += __shfl_xor_sync( mk, hadSum, m ); sadSum += __shfl_xor_sync( mk, sadSum, m ); }
    if( lg == 0 ) out[ci] = with2Sad ? min( hadSum, 2u * sadSum ) : hadSum;
  }
}

} // namespace vvb
