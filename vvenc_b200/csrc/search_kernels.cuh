// search_kernels.cuh -- integer motion-search SAD sweeps for sm_90a.
//
//  * sad_search_kernel : dense full search, InterSearch::xPatternSearch (EncoderLib/InterSearch.cpp:2209-2251).
//    One CTA per block; the (w + range) x (h + range) reference window and the original block are staged in shared
//    memory once, every thread then owns strips of 8 horizontally adjacent candidates and slides the original row over
//    a register-resident window row (packed 16x2 SAD: VIMNMX.S16x2 + IDP.2A), so each staged reference word is reused
//    for 8 candidates and each original word for 8 candidates x all strips.
//  * sad_pattern_kernel: the fixed TZ point pattern (xTZ8PointDiamondSearch / raster grid, InterSearch.cpp:557-758,
//    2491-2497) around a per-block start vector; candidates are read straight from the (L2-resident) reference plane.
//
// Both add the MV rate Distortion(sqrt(lambda)*bits) (CommonLib/RdCost.h:181-203) from a host-computed table and
// resolve the argmin with the reference's tie-break: first strictly smaller cost in evaluation order.
#pragma once
#include <cuda.h>            // CUtensorMap (type only; the encoder entry point is fetched at run time, libcuda is not linked)
#include "common.cuh"
#include "dist_kernels.cuh"

namespace vvb {

struct MePar { int costScale, imvShift, subShift, orderBits; MvCostTable tab; };   // orderBits: width of the raster-order field of 32-bit argmin keys (KEY32 kernels)

// tab: shared-memory copy of MePar::tab (dynamic indexing of the parameter bank would serialise per distinct address)
__device__ __forceinline__ uint32_t mv_cost( const MePar& p, const uint32_t* tab, int x, int y, int predHor, int predVer )
{
  const uint32_t bits = eg_bits( ( x * ( 1 << p.costScale ) - predHor ) >> p.imvShift ) + eg_bits( ( y * ( 1 << p.costScale ) - predVer ) >> p.imvShift );
  return tab[bits < VVB_MVCOST_ENTRIES ? bits : VVB_MVCOST_ENTRIES - 1];
}

// lexicographic (cost, order) minimum -> "first strictly smaller wins"
struct BestKey { unsigned long long cost; uint32_t order; };
__device__ __forceinline__ bool better( unsigned long long c, uint32_t o, unsigned long long bc, uint32_t bo ) { return c < bc || ( c == bc && o < bo ); }

// ---------------------------------------------------------------------------------------------------------------
// dense full search
// ---------------------------------------------------------------------------------------------------------------
#define SS_STRIP 8          // candidates per strip (consecutive dx)
#define SS_XCHUNK 16        // original pels consumed per inner step

// One CTA evaluates a MACRO block of nbx x nby adjacent blocks (1x1, or a z-order quad 2x2 whose members share range and
// predictor -- the encoder's quad-tree order): the staged window, the row sums and the column sums are shared by the members.
//
// smem layout: win[winH][ws] int16 | org[MH][MW] int16 | V[winH][nxpV] uint32 | bitsX[nxp], bitsY[ny] | per-member sumA / best keys
//
// SAD via  sum|a-b| = sum a + sum b - 2 sum min(a,b):
//   sum a           : once per member block
//   sum b (box sum) : V[cy'][cx'] = sum over a w x h box of the staged window, from row-sliding sums + in-place column sums
//                     (O(window) work, shared by all candidates and all members: member (bx,by) reads V[cy + by*h][cx + bx*w])
//   sum min(a,b)    : the only per-(candidate, pel) work: VIMNMX.S16x2 + IDP.2A per pel PAIR, i.e. one instruction per pel difference
// All three are exact integers, so the result is bit-identical to the direct sum.
struct SearchSmem { int ws, winH, nxp, nStrips, nxpV, nStripsV, vRows, offOrg, offV, offBits, offMisc, total; };

__host__ __device__ inline SearchSmem search_smem( int w, int h, int nx, int ny, int nbx, int nby )
{
  SearchSmem s;
  s.nStrips  = ( nx + SS_STRIP - 1 ) / SS_STRIP;
  s.nxp      = s.nStrips * SS_STRIP;
  s.nStripsV = ( nx + ( nbx - 1 ) * w + SS_STRIP - 1 ) / SS_STRIP;
  s.nxpV     = s.nStripsV * SS_STRIP;
  s.winH     = nby * h + ny - 1;
  s.vRows    = ny + ( nby - 1 ) * h;
  const int need = ( nbx * w + s.nxp + 8 + 7 ) & ~7;      // row pitch in pels, multiple of 8 -> every row 16-byte aligned
  // (A pitch with pitch*2 == 16*nStrips (mod 128) would make the row wrap of a warp's LDS.128 conflict-free, but the larger window costs
  //  more in occupancy than the conflicts do: measured 3.68 ms vs 3.14 ms on the 8x8 base level -- define SS_PAD_PITCH to try it again.)
#ifdef SS_PAD_PITCH
  const int padded = need + ( ( ( 8 * s.nStrips - need ) % 64 ) + 64 ) % 64;
#else
  const int padded = need;
#endif
  for( int attempt = 0; attempt < 2; attempt++ )
  {
    s.ws       = attempt == 0 ? padded : need;
    s.offOrg   = s.winH * s.ws * 2;                        // bytes
    s.offV     = s.offOrg + nbx * w * nby * h * 2;
    s.offBits  = s.offV + s.winH * s.nxpV * 4;
    s.offMisc  = s.offBits + 5 * ( s.nxp + ( ( ny + 3 ) & ~3 ) ) * 4;   // MV bits per member (4) + parent (pyramid mode), each set 16-byte aligned
    s.total    = s.offMisc + 64;
    if( s.total + 16 <= ( nbx * nby > 1 ? 100 * 1024 : 220 * 1024 ) && s.ws <= 256 ) break;
  }
  return s;
}

// TMA window staging: tmap describes the whole padded reference plane (uint16 elements), box = (ws x winH) of the launch's
// largest window; (tmaNx, tmaNy, tmaQuad) say which window geometry the box was built for -- blocks with another geometry
// use the load/store staging loop.  The copy is one cp.async.bulk.tensor.2d per CTA (any start alignment, zero fill outside).
struct TmaInfo { int enabled, nx, ny, quad, margin, pad[3]; };

__device__ __forceinline__ void mbar_init_s( uint32_t addr, uint32_t count ) { asm volatile( "mbarrier.init.shared::cta.b64 [%0], %1;" :: "r"( addr ), "r"( count ) : "memory" ); }
__device__ __forceinline__ void mbar_expect_tx_s( uint32_t addr, uint32_t bytes ) { asm volatile( "mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" :: "r"( addr ), "r"( bytes ) : "memory" ); }
__device__ __forceinline__ void mbar_wait_s( uint32_t addr, uint32_t parity )
{
  uint32_t done = 0;
  while( !done )
    asm volatile( "{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}\n" : "=r"( done ) : "r"( addr ), "r"( parity ) : "memory" );
}
__device__ __forceinline__ void tma_load_2d( uint32_t smemDst, const CUtensorMap* tmap, uint32_t mbar, int x, int y )
{
  asm volatile( "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
                :: "r"( smemDst ), "l"( (unsigned long long) tmap ), "r"( mbar ), "r"( x ), "r"( y ) : "memory" );
}

// - sum over the visited rows of min(org, ref) for a strip of 8 adjacent candidates: acc[k] = -sum min(o, r(k))
__device__ __forceinline__ void strip_min_sums( const int16_t* __restrict__ obase, const int16_t* __restrict__ rbase, int MW, int ws, int w, int h, int step, int (&acc)[SS_STRIP] )
{
#pragma unroll
  for( int k = 0; k < SS_STRIP; k++ ) acc[k] = 0;
  if( w >= SS_XCHUNK )
  {
    for( int y = 0; y < h; y += step )
    {
      const uint32_t* orow = reinterpret_cast<const uint32_t*>( obase + y * MW );
      const uint32_t* rrow = reinterpret_cast<const uint32_t*>( rbase + y * ws );
      for( int x = 0; x < w; x += SS_XCHUNK )
      {
        uint32_t o[SS_XCHUNK / 2], r[SS_XCHUNK / 2 + SS_STRIP / 2];
#pragma unroll
        for( int i = 0; i < SS_XCHUNK / 2; i += 4 ) *reinterpret_cast<uint4*>( &o[i] ) = *reinterpret_cast<const uint4*>( orow + x / 2 + i );
#pragma unroll
        for( int i = 0; i < SS_XCHUNK / 2 + SS_STRIP / 2; i += 4 ) *reinterpret_cast<uint4*>( &r[i] ) = *reinterpret_cast<const uint4*>( rrow + x / 2 + i );
#pragma unroll
        for( int k = 0; k < SS_STRIP; k++ )
        {
#pragma unroll
          for( int i = 0; i < SS_XCHUNK / 2; i++ )
          {
            const uint32_t rv = ( k & 1 ) ? __funnelshift_r( r[i + k / 2], r[i + k / 2 + 1], 16 ) : r[i + k / 2];
            acc[k] = __dp2a_lo( (int) __vmins2( o[i], rv ), (int) 0x0000ffffu, acc[k] );
          }
        }
      }
    }
  }
  else if( w == 8 )
  {
    for( int y = 0; y < h; y += step )
    {
      uint32_t o[4], r[8];
      *reinterpret_cast<uint4*>( &o[0] ) = *reinterpret_cast<const uint4*>( obase + y * MW );
      *reinterpret_cast<uint4*>( &r[0] ) = *reinterpret_cast<const uint4*>( rbase + y * ws );
      *reinterpret_cast<uint4*>( &r[4] ) = *reinterpret_cast<const uint4*>( rbase + y * ws + 8 );
#pragma unroll
      for( int k = 0; k < SS_STRIP; k++ )
      {
#pragma unroll
        for( int i = 0; i < 4; i++ )
        {
          const uint32_t rv = ( k & 1 ) ? __funnelshift_r( r[i + k / 2], r[i + k / 2 + 1], 16 ) : r[i + k / 2];
          acc[k] = __dp2a_lo( (int) __vmins2( o[i], rv ), (int) 0x0000ffffu, acc[k] );
        }
      }
    }
  }
  else      // w == 4 (single-block mode only)
  {
    for( int y = 0; y < h; y += step )
    {
      uint32_t o[2], r[8];
      *reinterpret_cast<uint2*>( &o[0] ) = *reinterpret_cast<const uint2*>( obase + y * MW );
      *reinterpret_cast<uint4*>( &r[0] ) = *reinterpret_cast<const uint4*>( rbase + y * ws );
      *reinterpret_cast<uint4*>( &r[4] ) = *reinterpret_cast<const uint4*>( rbase + y * ws + 8 );
#pragma unroll
      for( int k = 0; k < SS_STRIP; k++ )
      {
#pragma unroll
        for( int i = 0; i < 2; i++ )
        {
          const uint32_t rv = ( k & 1 ) ? __funnelshift_r( r[i + k / 2], r[i + k / 2 + 1], 16 ) : r[i + k / 2];
          acc[k] = __dp2a_lo( (int) __vmins2( o[i], rv ), (int) 0x0000ffffu, acc[k] );
        }
      }
    }
  }
}

template<bool K32> struct KeyType { typedef unsigned long long type; };
template<> struct KeyType<true> { typedef uint32_t type; };

template<bool USE_TMA, bool PARENT, bool KEY32 = false>
__global__ void __launch_bounds__( PARENT ? 256 : 384, PARENT ? 3 : 2 ) sad_search_kernel( const __grid_constant__ Plane orgPlane, const __grid_constant__ Plane refPlane,
                                                            const vvb_block* __restrict__ blocks, int nBlocks, int w, int h, int quadMode,
                                                            const __grid_constant__ MePar par, const __grid_constant__ CUtensorMap tmap, const __grid_constant__ TmaInfo tma,
                                                            uint32_t* __restrict__ sadTables, int tableStride, vvb_best* __restrict__ bestOut,
                                                            const vvb_block* __restrict__ parentBlocks, vvb_best* __restrict__ parentBest,
                                                            uint32_t* __restrict__ parentTables, int parentStride )
{
  extern __shared__ __align__( 128 ) unsigned char smemRaw[];
  __shared__ uint32_t sMv[VVB_MVCOST_ENTRIES];
  __shared__ __align__( 8 ) unsigned long long sTmaBar;
  const int tid = threadIdx.x, nthr = blockDim.x, lane = tid & 31;
  for( int i = tid; i < VVB_MVCOST_ENTRIES; i += nthr ) sMv[i] = par.tab.cost[i];
  const int step = 1 << par.subShift;
  const uint32_t tmaBar = (uint32_t) __cvta_generic_to_shared( &sTmaBar );
  uint32_t tmaPhase = 0;
  if( USE_TMA && tma.enabled && tid == 0 ) { mbar_init_s( tmaBar, 1 ); asm volatile( "fence.mbarrier_init.release.cluster;" ::: "memory" ); }

  // ---- which blocks does this CTA own, and are they a proper quad?
  const int first = quadMode ? blockIdx.x * 4 : blockIdx.x;
  const int owned = quadMode ? min( 4, nBlocks - first ) : 1;
  const vvb_block b0 = blocks[first];
  bool isQuad = false;
  if( quadMode && owned == 4 && w >= 8 )
  {
    const vvb_block b1 = blocks[first + 1], b2 = blocks[first + 2], b3 = blocks[first + 3];
    isQuad = b1.x == b0.x + w && b1.y == b0.y && b2.x == b0.x && b2.y == b0.y + h && b3.x == b0.x + w && b3.y == b0.y + h;
    const vvb_block* q[3] = { &b1, &b2, &b3 };
#pragma unroll
    for( int i = 0; i < 3; i++ )
      isQuad = isQuad && q[i]->left == b0.left && q[i]->right == b0.right && q[i]->top == b0.top && q[i]->bottom == b0.bottom;   // predictors may differ
  }
  const int nSub = isQuad ? 1 : owned;
  if( PARENT && !isQuad )
  {
    // pyramid launches handle proper quads only: a broken quad reports its members and its parent as invalid
    if( tid < owned ) { vvb_best b; b.dx = 0; b.dy = 0; b.sad = 0xffffffffu; b.cost = ~0ull; bestOut[first + tid] = b; }
    return;
  }

  for( int sub = 0; sub < nSub; sub++ )
  {
    const vvb_block blk = isQuad ? b0 : blocks[first + sub];
    const int nbx = isQuad ? 2 : 1, nby = isQuad ? 2 : 1, nMem = nbx * nby;
    const int nx = blk.right - blk.left + 1, ny = blk.bottom - blk.top + 1;
    const SearchSmem L = search_smem( w, h, nx, ny, nbx, nby );
    const int ws = L.ws, winH = L.winH, nxp = L.nxp, nStrips = L.nStrips, nxpV = L.nxpV;
    const int MW = nbx * w, MH = nby * h;
    int16_t*  win   = reinterpret_cast<int16_t*>( smemRaw );
    int16_t*  orgS  = reinterpret_cast<int16_t*>( smemRaw + L.offOrg );          // [MH][MW]
    uint32_t* V     = reinterpret_cast<uint32_t*>( smemRaw + L.offV );            // [winH][nxpV]
    int*      bitsAll = reinterpret_cast<int*>( smemRaw + L.offBits );            // per member m: X bits [nxp] then Y bits [ny] at m*(nxp+ny); set 4 = parent
    const int bitsSet = nxp + ( ( ny + 3 ) & ~3 );
    int*      sSumA = reinterpret_cast<int*>( smemRaw + L.offMisc );              // [4]
    unsigned long long* sKey = reinterpret_cast<unsigned long long*>( smemRaw + L.offMisc + 16 );   // [5] members + parent (cost << 16 | raster order)

    __syncthreads();                                      // previous sub-iteration fully consumed
    if( tid < 4 ) sSumA[tid] = 0;
    if( tid < 5 ) sKey[tid] = ~0ull;

    // ---- stage the window: TMA when the box matches this window, else 32-bit words (even start) / 16-bit, 16 loads in flight per thread
    {
      const int16_t* src = refPlane.origin + (ptrdiff_t)( blk.y + blk.top ) * refPlane.stride + blk.x + blk.left;
      const int validW = MW + nx - 1;
      const bool even = ( ( (uintptr_t) src & 3 ) == 0 ) && ( ( refPlane.stride & 1 ) == 0 );
      // cp.async.bulk.tensor with 16-bit elements needs the innermost start coordinate on a 16-byte boundary (multiple of 8 pels; measured with
      // tools/tma_probe.cu: any other start raises an illegal-instruction fault) -- windows that start elsewhere take the manual path below
      const bool viaTma = USE_TMA && tma.enabled && nx == tma.nx && ny == tma.ny && ( isQuad ? 1 : 0 ) == tma.quad && ( ( ( blk.x + blk.left + tma.margin ) & 7 ) == 0 );
      if( viaTma )
      {
        if( tid == 0 )
        {
          asm volatile( "fence.proxy.async.shared::cta;" ::: "memory" );      // earlier generic accesses to the window are ordered before the async write
          mbar_expect_tx_s( tmaBar, (uint32_t)( winH * ws * 2 ) );
          tma_load_2d( (uint32_t) __cvta_generic_to_shared( win ), &tmap, tmaBar, blk.x + blk.left + tma.margin, blk.y + blk.top + tma.margin );
        }
      }
      else if( even )
      {
        const int wpr = ws >> 1, total = winH * wpr, validWords = ( validW + 1 ) >> 1;
        const float inv = 1.0f / (float) wpr;
        uint32_t* win32 = reinterpret_cast<uint32_t*>( win );
        for( int i0 = tid; i0 < total; i0 += nthr * 16 )
        {
          uint32_t v[16];
#pragma unroll
          for( int u = 0; u < 16; u++ )
          {
            const int i = i0 + u * nthr;
            v[u] = 0u;
            if( i < total )
            {
              const int r = div_rcp( i, inv ), c = i - r * wpr;
              if( c < validWords ) v[u] = __ldg( reinterpret_cast<const uint32_t*>( src + (ptrdiff_t) r * refPlane.stride ) + c );
            }
          }
#pragma unroll
          for( int u = 0; u < 16; u++ ) { const int i = i0 + u * nthr; if( i < total ) win32[i] = v[u]; }
        }
      }
      else
      {
        const int total = winH * ws;
        const float inv = 1.0f / (float) ws;
        for( int i0 = tid; i0 < total; i0 += nthr * 16 )
        {
          int16_t v[16];
#pragma unroll
          for( int u = 0; u < 16; u++ )
          {
            const int i = i0 + u * nthr;
            v[u] = 0;
            if( i < total )
            {
              const int r = div_rcp( i, inv ), c = i - r * ws;
              if( c < validW ) v[u] = __ldg( src + (ptrdiff_t) r * refPlane.stride + c );
            }
          }
#pragma unroll
          for( int u = 0; u < 16; u++ ) { const int i = i0 + u * nthr; if( i < total ) win[i] = v[u]; }
        }
      }
      // original macro block (MW is a power of two or twice one -> shifts) and per-member sum a
      const int16_t* so = orgPlane.origin + (ptrdiff_t) blk.y * orgPlane.stride + blk.x;
      const int lMW = ilog2_dev( MW );
      int sumA[4] = { 0, 0, 0, 0 };
      for( int i = tid; i < MW * MH; i += nthr )
      {
        const int r = i >> lMW, c = i & ( MW - 1 );
        const int16_t v = __ldg( so + (ptrdiff_t) r * orgPlane.stride + c );
        orgS[i] = v;
        const int ry = r >= h ? r - h : r;                 // row inside the member
        if( ( ry & ( step - 1 ) ) == 0 ) sumA[( r >= h ? 2 : 0 ) + ( c >= w ? 1 : 0 )] += v;
      }
      if( viaTma ) { mbar_wait_s( tmaBar, tmaPhase ); tmaPhase ^= 1; }
      __syncthreads();                                     // sSumA / sKey initialised, window visible
#pragma unroll
      for( int m4 = 0; m4 < 4; m4++ )
      {
        int v = sumA[m4];
#pragma unroll
        for( int m = 16; m > 0; m >>= 1 ) v += __shfl_xor_sync( 0xffffffffu, v, m );
        if( lane == 0 && v ) atomicAdd( &sSumA[m4], v );
      }
      // MV-rate bit counts per column / row of the window (RdCost.h:183-203), one set per member (each keeps its own predictor)
      for( int mm = 0; mm < nMem; mm++ )
      {
        const vvb_block mb = isQuad ? blocks[first + mm] : blk;
        int* bx_ = bitsAll + mm * bitsSet; int* by_ = bx_ + nxp;
        for( int i = tid; i < nxp; i += nthr ) bx_[i] = (int) eg_bits( ( ( blk.left + i ) * ( 1 << par.costScale ) - mb.pred_hor ) >> par.imvShift );
        for( int i = tid; i < ny;  i += nthr ) by_[i] = (int) eg_bits( ( ( blk.top  + i ) * ( 1 << par.costScale ) - mb.pred_ver ) >> par.imvShift );
      }
    }
    // ---- row sums Hs[r][cx'] = sum_{x<w} win[r][cx'+x]: one task = (row, strip of 8 cx')
    {
      const int nTasks = winH * L.nStripsV;
      const float inv = 1.0f / (float) L.nStripsV;
      for( int t = tid; t < nTasks; t += nthr )
      {
        const int r = div_rcp( t, inv ), st = t - r * L.nStripsV;
        const int16_t* row = win + r * ws + st * SS_STRIP;
        int s = 0;
        for( int x = 0; x < w; x++ ) s += row[x];
        uint32_t* dst = V + r * nxpV + st * SS_STRIP;
        dst[0] = (uint32_t) s;
#pragma unroll
        for( int k = 1; k < SS_STRIP; k++ ) { s += row[w + k - 1] - row[k - 1]; dst[k] = (uint32_t) s; }
      }
    }
    __syncthreads();
    // ---- column sums in place: V[cy'][cx'] = sum_{k < h/step} Hs[cy' + k*step][cx']; rows of one phase (cy' mod step) only depend on that phase
    {
      const int m = h >> par.subShift;
      for( int t = tid; t < nxpV * step; t += nthr )
      {
        const int cx = t % nxpV, p = t / nxpV;
        if( p < L.vRows )
        {
          int cur = 0;
          for( int k = 0; k < m; k++ ) cur += (int) V[( p + k * step ) * nxpV + cx];
          int prevTop = (int) V[p * nxpV + cx];
          V[p * nxpV + cx] = (uint32_t) cur;
          for( int cy = p + step; cy < L.vRows; cy += step )
          {
            cur += (int) V[( cy + ( m - 1 ) * step ) * nxpV + cx] - prevTop;
            prevTop = (int) V[cy * nxpV + cx];
            V[cy * nxpV + cx] = (uint32_t) cur;
          }
        }
      }
    }
    __syncthreads();

    // ---- candidates
    const int perMem = ny * nStrips;
    const float invStr = 1.0f / (float) nStrips;
    if( !PARENT )
    {
      // item = (member, cy, strip of 8 cx); a thread walks items in increasing order, so members are visited in order
      const int items = nMem * perMem;
      const float invPer = 1.0f / (float) perMem;
      unsigned long long bestKey = ~0ull; int curMem = -1;
      for( int it = tid; it < items; it += nthr )
      {
        const int mem = div_rcp( it, invPer ), loc = it - mem * perMem;
        const int cy = div_rcp( loc, invStr ), st = loc - cy * nStrips;
        const int bx = mem & ( nbx - 1 ), by = mem >> ( nbx - 1 );
        const int cx0 = st * SS_STRIP;
        if( mem != curMem )
        {
          if( curMem >= 0 && bestKey != ~0ull ) atomicMin( &sKey[curMem], bestKey );
          curMem = mem; bestKey = ~0ull;
        }
        int acc[SS_STRIP];
        strip_min_sums( orgS + ( by * h ) * MW + bx * w, win + ( by * h + cy ) * ws + bx * w + cx0, MW, ws, w, h, step, acc );
        const int* bitsX = bitsAll + mem * bitsSet; const int* bitsY = bitsX + nxp;
        const int byBits = bitsY[cy];
        const int sumA = sSumA[( by << 1 ) | bx];
        const int gblk = first + ( isQuad ? mem : sub );
        // 8 consecutive words per thread: two LDS.128 each instead of 8 bank-conflicting LDS.32
        uint32_t vv[SS_STRIP]; int bxv[SS_STRIP];
        *reinterpret_cast<uint4*>( &vv[0] )  = *reinterpret_cast<const uint4*>( V + ( cy + by * h ) * nxpV + bx * w + cx0 );
        *reinterpret_cast<uint4*>( &vv[4] )  = *reinterpret_cast<const uint4*>( V + ( cy + by * h ) * nxpV + bx * w + cx0 + 4 );
        *reinterpret_cast<int4*>( &bxv[0] )  = *reinterpret_cast<const int4*>( bitsX + cx0 );
        *reinterpret_cast<int4*>( &bxv[4] )  = *reinterpret_cast<const int4*>( bitsX + cx0 + 4 );
#pragma unroll
        for( int k = 0; k < SS_STRIP; k++ )
        {
          const int cx = cx0 + k;
          if( cx < nx )
          {
            const uint32_t sad = (uint32_t)( sumA + (int) vv[k] + 2 * acc[k] ) << par.subShift;
            const uint32_t order = (uint32_t)( cy * nx + cx );
            if( sadTables ) sadTables[(size_t) gblk * tableStride + order] = sad;
            const uint32_t bits = (uint32_t)( bxv[k] + byBits );
            const unsigned long long c = (unsigned long long) sad + sMv[bits < VVB_MVCOST_ENTRIES ? bits : VVB_MVCOST_ENTRIES - 1];
            const unsigned long long key = ( c << 16 ) | order;          // lexicographic (cost, raster order): first strictly smaller wins
            bestKey = key < bestKey ? key : bestKey;
          }
        }
      }
      if( curMem >= 0 && bestKey != ~0ull ) atomicMin( &sKey[curMem], bestKey );
    }
    else
    {
      // SAD pyramid: item = (cy, strip); the thread evaluates the strip for all four members, so the parent block's SAD at the same
      // vector -- the exact sum of its children's SADs -- costs four additions instead of a second pass over the pels.
      const vvb_block pblk = parentBlocks[blockIdx.x];
      const bool parentOk = pblk.left == blk.left && pblk.right == blk.right && pblk.top == blk.top && pblk.bottom == blk.bottom;
      int* pBitsX = bitsAll + 4 * bitsSet;                // parent MV bits (its own predictor)
      int* pBitsY = pBitsX + nxp;
      for( int i = tid; i < nxp; i += nthr ) pBitsX[i] = (int) eg_bits( ( ( blk.left + i ) * ( 1 << par.costScale ) - pblk.pred_hor ) >> par.imvShift );
      for( int i = tid; i < ny;  i += nthr ) pBitsY[i] = (int) eg_bits( ( ( blk.top  + i ) * ( 1 << par.costScale ) - pblk.pred_ver ) >> par.imvShift );
      __syncthreads();
      // argmin keys (cost << ob | raster order): 64 bit with a 16-bit order field in general; KEY32 instantiations are launched when the host has
      // verified that every possible cost of the batch fits 32 - ob bits (half the epilogue arithmetic, REDUX instead of shuffle trees)
      typedef typename KeyType<KEY32>::type KT;
      const int ob = KEY32 ? par.orderBits : 16;
      const KT KMAX = ~(KT) 0;
      KT key4[4] = { KMAX, KMAX, KMAX, KMAX }, keyP = KMAX;
      for( int it = tid; it < perMem; it += nthr )
      {
        const int cy = div_rcp( it, invStr ), st = it - cy * nStrips;
        const int cx0 = st * SS_STRIP;
        const int pByBits = pBitsY[cy];
        uint32_t psad[SS_STRIP];
#pragma unroll
        for( int k = 0; k < SS_STRIP; k++ ) psad[k] = 0;
#pragma unroll 1
        for( int mem = 0; mem < 4; mem++ )       // not unrolled on purpose: one copy of the strip code, key4[] lives in local memory (2 accesses per member)
        {
          const int bx = mem & 1, by = mem >> 1;
          int acc[SS_STRIP];
          strip_min_sums( orgS + ( by * h ) * MW + bx * w, win + ( by * h + cy ) * ws + bx * w + cx0, MW, ws, w, h, step, acc );
          const int sumA = sSumA[mem];
          const int* bitsX = bitsAll + mem * bitsSet;
          const int byBits = bitsX[nxp + cy];
          KT bk = key4[mem];
          uint32_t vv[SS_STRIP]; int bxv[SS_STRIP];
          *reinterpret_cast<uint4*>( &vv[0] )  = *reinterpret_cast<const uint4*>( V + ( cy + by * h ) * nxpV + bx * w + cx0 );
          *reinterpret_cast<uint4*>( &vv[4] )  = *reinterpret_cast<const uint4*>( V + ( cy + by * h ) * nxpV + bx * w + cx0 + 4 );
          *reinterpret_cast<int4*>( &bxv[0] )  = *reinterpret_cast<const int4*>( bitsX + cx0 );
          *reinterpret_cast<int4*>( &bxv[4] )  = *reinterpret_cast<const int4*>( bitsX + cx0 + 4 );
#pragma unroll
          for( int k = 0; k < SS_STRIP; k++ )
          {
            const int cx = cx0 + k;
            if( cx < nx )
            {
              const uint32_t sad = (uint32_t)( sumA + (int) vv[k] + 2 * acc[k] ) << par.subShift;
              const uint32_t order = (uint32_t)( cy * nx + cx );
              psad[k] += sad;
              if( sadTables ) sadTables[(size_t)( first + mem ) * tableStride + order] = sad;
              const uint32_t bits = (uint32_t)( bxv[k] + byBits );
              const KT key = ( ( (KT) sad + sMv[bits < VVB_MVCOST_ENTRIES ? bits : VVB_MVCOST_ENTRIES - 1] ) << ob ) | order;
              bk = key < bk ? key : bk;
            }
          }
          key4[mem] = bk;
        }
        int pbx[SS_STRIP];
        *reinterpret_cast<int4*>( &pbx[0] ) = *reinterpret_cast<const int4*>( pBitsX + cx0 );
        *reinterpret_cast<int4*>( &pbx[4] ) = *reinterpret_cast<const int4*>( pBitsX + cx0 + 4 );
#pragma unroll
        for( int k = 0; k < SS_STRIP; k++ )
        {
          const int cx = cx0 + k;
          if( cx < nx )
          {
            const uint32_t order = (uint32_t)( cy * nx + cx );
            if( parentTables ) parentTables[(size_t) blockIdx.x * parentStride + order] = psad[k];
            const uint32_t bits = (uint32_t)( pbx[k] + pByBits );
            const KT key = ( ( (KT) psad[k] + sMv[bits < VVB_MVCOST_ENTRIES ? bits : VVB_MVCOST_ENTRIES - 1] ) << ob ) | order;
            keyP = key < keyP ? key : keyP;
          }
        }
      }
      // warp minimum first, then one atomic per warp and key
      unsigned long long k64[5];
      if( KEY32 )
      {
#pragma unroll
        for( int q = 0; q < 5; q++ )
        {
          const uint32_t k = __reduce_min_sync( 0xffffffffu, (uint32_t)( q < 4 ? key4[q] : keyP ) );
          k64[q] = k == 0xffffffffu ? ~0ull : ( ( (unsigned long long)( k >> ob ) << 16 ) | ( k & ( ( 1u << ob ) - 1u ) ) );
        }
      }
      else
      {
#pragma unroll
        for( int q = 0; q < 5; q++ ) k64[q] = (unsigned long long)( q < 4 ? key4[q] : keyP );
#pragma unroll
        for( int m = 16; m > 0; m >>= 1 )
        {
#pragma unroll
          for( int q = 0; q < 5; q++ ) { const unsigned long long o = __shfl_xor_sync( 0xffffffffu, k64[q], m ); k64[q] = o < k64[q] ? o : k64[q]; }
        }
      }
      if( lane == 0 )
      {
#pragma unroll
        for( int q = 0; q < 5; q++ ) if( k64[q] != ~0ull ) atomicMin( &sKey[q], k64[q] );
      }
      __syncthreads();
      if( tid == 0 )
      {
        vvb_best b;
        const unsigned long long key = sKey[4];
        if( !parentOk || key == ~0ull ) { b.dx = 0; b.dy = 0; b.sad = 0xffffffffu; b.cost = ~0ull; }
        else
        {
          const uint32_t order = (uint32_t)( key & 0xffffu );
          const int cy = order / nx, cx = order - cy * nx;
          const uint32_t bits = (uint32_t)( pBitsX[cx] + pBitsY[cy] );
          b.dx = (int16_t)( blk.left + cx ); b.dy = (int16_t)( blk.top + cy ); b.cost = key >> 16;
          b.sad = (uint32_t)( b.cost - sMv[bits < VVB_MVCOST_ENTRIES ? bits : VVB_MVCOST_ENTRIES - 1] );
        }
        parentBest[blockIdx.x] = b;
      }
    }
    __syncthreads();
    if( tid < nMem )
    {
      const unsigned long long key = sKey[tid];
      const uint32_t order = (uint32_t)( key & 0xffffu );
      const unsigned long long cost = key >> 16;
      const int cy = order / nx, cx = order - cy * nx;
      const int* bitsX = bitsAll + tid * bitsSet;
      const uint32_t bits = (uint32_t)( bitsX[cx] + bitsX[nxp + cy] );
      vvb_best b;
      b.dx = (int16_t)( blk.left + cx ); b.dy = (int16_t)( blk.top + cy ); b.cost = cost;
      b.sad = (uint32_t)( cost - sMv[bits < VVB_MVCOST_ENTRIES ? bits : VVB_MVCOST_ENTRIES - 1] );
      bestOut[first + ( isQuad ? tid : sub )] = b;
    }
  }
}

// Pyramid level >= 2: the SAD table of a parent block is the sum of its four children's tables (children 4p..4p+3 of the level below);
// argmin with the parent's own MV predictor; optional table output for the next level.  One CTA per parent.
__global__ void __launch_bounds__( 256 ) sad_table_sum_kernel( const vvb_block* __restrict__ parents, int nParents, int nx, int ny, const __grid_constant__ MePar par,
                                                               const uint32_t* __restrict__ childTables, int childStride, const vvb_best* __restrict__ childBest,
                                                               uint32_t* __restrict__ outTables, int outStride, vvb_best* __restrict__ bestOut )
{
  __shared__ uint32_t sMv[VVB_MVCOST_ENTRIES];
  __shared__ int sBitsX[512], sBitsY[512];
  __shared__ unsigned long long sKeyP;
  const int tid = threadIdx.x, nthr = blockDim.x, lane = tid & 31;
  const vvb_block blk = parents[blockIdx.x];
  for( int i = tid; i < VVB_MVCOST_ENTRIES; i += nthr ) sMv[i] = par.tab.cost[i];
  for( int i = tid; i < nx; i += nthr ) sBitsX[i] = (int) eg_bits( ( ( blk.left + i ) * ( 1 << par.costScale ) - blk.pred_hor ) >> par.imvShift );
  for( int i = tid; i < ny; i += nthr ) sBitsY[i] = (int) eg_bits( ( ( blk.top  + i ) * ( 1 << par.costScale ) - blk.pred_ver ) >> par.imvShift );
  if( tid == 0 ) sKeyP = ~0ull;
  __syncthreads();
  // a child reported invalid (broken quad below: its table row was never written) makes this parent invalid as well
  bool ok = ( blk.right - blk.left + 1 ) == nx && ( blk.bottom - blk.top + 1 ) == ny;
#pragma unroll
  for( int c = 0; c < 4; c++ ) ok = ok && childBest[4 * (size_t) blockIdx.x + c].cost != ~0ull;
  const uint32_t* c0 = childTables + (size_t)( 4 * blockIdx.x ) * childStride;
  const int total = nx * ny;
  const float inv = 1.0f / (float) nx;
  unsigned long long best = ~0ull;
  for( int o = tid; o < total; o += nthr )
  {
    const uint32_t s = __ldg( c0 + o ) + __ldg( c0 + childStride + o ) + __ldg( c0 + 2 * (size_t) childStride + o ) + __ldg( c0 + 3 * (size_t) childStride + o );
    if( outTables ) outTables[(size_t) blockIdx.x * outStride + o] = s;
    const int cy = div_rcp( o, inv ), cx = o - cy * nx;
    const uint32_t bits = (uint32_t)( sBitsX[cx] + sBitsY[cy] );
    const unsigned long long key = ( ( (unsigned long long) s + sMv[bits < VVB_MVCOST_ENTRIES ? bits : VVB_MVCOST_ENTRIES - 1] ) << 16 ) | (unsigned) o;
    best = key < best ? key : best;
  }
#pragma unroll
  for( int m = 16; m > 0; m >>= 1 ) { const unsigned long long o = __shfl_xor_sync( 0xffffffffu, best, m ); best = o < best ? o : best; }
  if( lane == 0 && best != ~0ull ) atomicMin( &sKeyP, best );
  __syncthreads();
  if( tid == 0 )
  {
    vvb_best b;
    const unsigned long long key = sKeyP;
    if( !ok || key == ~0ull ) { b.dx = 0; b.dy = 0; b.sad = 0xffffffffu; b.cost = ~0ull; }
    else
    {
      const uint32_t order = (uint32_t)( key & 0xffffu );
      const int cy = order / nx, cx = order - cy * nx;
      const uint32_t bits = (uint32_t)( sBitsX[cx] + sBitsY[cy] );
      b.dx = (int16_t)( blk.left + cx ); b.dy = (int16_t)( blk.top + cy ); b.cost = key >> 16;
      b.sad = (uint32_t)( b.cost - sMv[bits < VVB_MVCOST_ENTRIES ? bits : VVB_MVCOST_ENTRIES - 1] );
    }
    bestOut[blockIdx.x] = b;
  }
}

// ---------------------------------------------------------------------------------------------------------------
// fixed pattern around a start vector; one CTA per block, G-lane groups take candidates round-robin
// ---------------------------------------------------------------------------------------------------------------
template<int G>
__global__ void __launch_bounds__( 128 ) cost_pattern_kernel( const __grid_constant__ Plane orgPlane, const __grid_constant__ Plane refPlane,
                                                              const vvb_block* __restrict__ blocks, int w, int h, int fam, const vvb_mv* __restrict__ pattern, int K,
                                                              const __grid_constant__ MePar par, uint32_t* __restrict__ sadOut, vvb_best* __restrict__ bestOut )
{
  __shared__ uint32_t sMv[VVB_MVCOST_ENTRIES];
  for( int i = threadIdx.x; i < VVB_MVCOST_ENTRIES; i += blockDim.x ) sMv[i] = par.tab.cost[i];
  __syncthreads();
  const vvb_block blk = blocks[blockIdx.x];
  const int lg = threadIdx.x & ( G - 1 );
  const int group = threadIdx.x / G, nGroups = blockDim.x / G;
  const int16_t* org = orgPlane.origin + (ptrdiff_t) blk.y * orgPlane.stride + blk.x;
  unsigned long long bestCost = ~0ull; uint32_t bestOrder = 0xffffffffu, bestSad = 0;

  for( int k = group; k < K; k += nGroups )
  {
    const vvb_mv pm = pattern[k];
    const int mx = blk.start_x + pm.dx, my = blk.start_y + pm.dy;
    const bool inside = mx >= blk.left && mx <= blk.right && my >= blk.top && my <= blk.bottom;      // SearchRange clip, InterSearch.cpp:576-620
    uint32_t sad = 0xffffffffu;
    if( inside )        // uniform per group
    {
      // the decision uses the full 64-bit distortion (an SSE may exceed 32 bits); the uint32 outputs saturate below the "outside" marker
      const int16_t* cur = refPlane.origin + (ptrdiff_t)( blk.y + my ) * refPlane.stride + blk.x + mx;
      const unsigned long long dist = group_dist<G>( fam, org, orgPlane.stride, cur, refPlane.stride, w, h, par.subShift, lg );
      sad = dist < 0xfffffffeull ? (uint32_t) dist : 0xfffffffeu;
      const unsigned long long c = dist + mv_cost( par, sMv, mx, my, blk.pred_hor, blk.pred_ver );
      if( better( c, (uint32_t) k, bestCost, bestOrder ) ) { bestCost = c; bestOrder = (uint32_t) k; bestSad = sad; }
    }
    if( sadOut && lg == 0 ) sadOut[(size_t) blockIdx.x * K + k] = sad;
  }
  if( !bestOut ) return;
  __shared__ unsigned long long sCost[32];
  __shared__ uint32_t sOrder[32], sSad[32];
  if( lg == 0 ) { sCost[group] = bestCost; sOrder[group] = bestOrder; sSad[group] = bestSad; }
  __syncthreads();
  if( threadIdx.x == 0 )
  {
    for( int i = 1; i < nGroups; i++ )
      if( better( sCost[i], sOrder[i], bestCost, bestOrder ) ) { bestCost = sCost[i]; bestOrder = sOrder[i]; bestSad = sSad[i]; }
    vvb_best b;
    if( bestOrder == 0xffffffffu ) { b.dx = 0; b.dy = 0; b.sad = 0xffffffffu; b.cost = ~0ull; }
    else { const vvb_mv pm = pattern[bestOrder]; b.dx = (int16_t)( blk.start_x + pm.dx ); b.dy = (int16_t)( blk.start_y + pm.dy ); b.sad = bestSad; b.cost = bestCost; }
    bestOut[blockIdx.x] = b;
  }
}

// ---------------------------------------------------------------------------------------------------------------
// had8_ring_kernel: Hadamard refinement over a small pattern of K points around each block's start vector, for square power-of-two blocks whose SATD
// dispatch lands on 8x8 tiles (RdCost.cpp:1836-1905).  One lane owns one (block, 8x8 tile) and walks all K points: its original tile stays in 32
// registers, and the candidate tiles come from a reference window staged once per block in shared memory.  Every lane of a warp takes the same point
// at the same time; a block's tiles sit in adjacent lanes and are summed with x-or shuffles.
//
// Window of a block: rows start_y - RC ... start_y + w + RC - 1 and WPR words per row in two copies, win0 word m = pels (2m, 2m+1) and win1 word m =
// pels (2m+1, 2m+2), where pel 0 is plane column x + start_x - RC.  A candidate column of either parity therefore reads whole words, and the window
// position does not depend on the parity of the start vector.  RC (2 or 8) is the staged radius; points farther out read the plane directly.
//
// Banks: lane reads word i of a row at laneBase + U + ( i ^ xr ), where U is the same for the whole warp and laneBase = slot * S + 8 * ty * PITCH + 4 * tx.
// S = 4 mod 8, and PITCH is not a multiple of 4 for 32x32, so at most four lanes of a warp share laneBase / 4 mod 8; xr (0..3) is the lane's rank
// among them, and the 32 reads hit 32 banks.  Reading a row's words in the order i ^ xr x-ors the tile's column index with 2 * xr; the original tile
// is loaded in the same order, and an x-or permutation of the columns only flips signs of Hadamard coefficients, so the SATD is the same bit for bit.
// tools/had_ring_banks.py evaluates these addresses for every lane.
template<int W, int RC>
struct HadRingShape
{
  static constexpr int TX = W / 8, T = TX * TX, ROWS = W + 2 * RC, WPR = W / 2 + RC;
  static constexpr int PITCH = WPR + ( ( TX == 4 && WPR % 4 == 0 ) ? 1 : 0 );
  static constexpr int WIN1 = ROWS * PITCH;                          // offset of win1 in a slot
  static constexpr int S = ( ( 2 * WIN1 + 3 ) & ~7 ) + 4;            // slot stride in words, 4 mod 8
  static constexpr int CHUNKS = ( WPR + 7 ) / 4;                     // 16-byte chunks per staged row (start pel anywhere in the first one)
};

// shared memory after the windows: per-candidate costs (two halves for 64x64), argmin keys, block descriptors, pattern
struct HadRingSmem { int slots, kStride, costOff, keyOff, blkOff, patOff, total; };
__host__ __device__ inline HadRingSmem had_ring_smem( int threads, int T, int S, int K )
{
  HadRingSmem s;
  s.slots = threads / T; if( s.slots < 1 ) s.slots = 1;
  s.kStride = K | 1;
  s.costOff = s.slots * S;
  s.keyOff = ( s.costOff + ( T > 32 ? 2 : 1 ) * s.slots * s.kStride + 1 ) & ~1;
  s.blkOff = s.keyOff + 2 * s.slots; s.patOff = s.blkOff + 6 * s.slots; s.total = s.patOff + K;
  return s;
}

// dp2a with unsigned 16-bit halves against signed byte weights (the biased packed values of the PACKED path below)
__device__ __forceinline__ int dp2a_lo_us( uint32_t a, int b, int c ) { int d; asm( "dp2a.lo.u32.s32 %0, %1, %2, %3;" : "=r"( d ) : "r"( a ), "r"( b ), "r"( c ) ); return d; }

// SATD of one 8x8 tile (RdCost.cpp:1311-1319).  row( r, o, c ) gives the original and reference words of row r, o[m] and c[m] holding pels (2m, 2m+1).
// Each row is differenced as soon as row() returns it.  Gathering all 64 words first made ptxas issue every original load before the first reference load:
// had8_direct_kernel<true> took 0.107 ms instead of 0.101 for the 8x8 blocks of a 2160p picture (H100 80GB HBM3, 700 W).
// PACKED (planes of at most 10 bits): the difference lives in 32 registers as pairs of 16-bit values biased by 0x8000.  Difference and the five butterfly
// stages across registers are one IADD3 per register each: ( A + B - K ) and ( A - B + K ) with K = 0x80008000 keep both halves inside [0, 65535]
// (|value| <= 32 * 1023), so the carry between the halves cancels exactly.  The sixth stage (the two halves of a word against each other, results up to
// 64 * 1023) and the bias removal are two dp2a per word.  Otherwise the difference and the first stage come out of IDP.2A into 64 scalar values:
// (o0 - c0) + (o1 - c1) = dp2a( o, (1,1) ) + dp2a( c, (-1,-1) ), (o0 - c0) - (o1 - c1) = dp2a( o, (1,-1) ) + dp2a( c, (-1,1) ).
template<bool PACKED, class Row>
__device__ __forceinline__ uint32_t had8_tile_cost( Row row )
{
  int d[64];
  uint32_t u[32];
#pragma unroll
  for( int r = 0; r < 8; r++ )
  {
    uint32_t o[4], c[4];
    row( r, o, c );
#pragma unroll
    for( int m = 0; m < 4; m++ )
    {
      const int i = 4 * r + m;
      if( PACKED ) u[i] = o[m] - c[m] + 0x80008000u;
      else
      {
        d[2 * i]     = __dp2a_lo( (int) c[m], (int) 0x0000ffff, __dp2a_lo( (int) o[m], (int) 0x00000101, 0 ) );
        d[2 * i + 1] = __dp2a_lo( (int) c[m], (int) 0x000001ff, __dp2a_lo( (int) o[m], (int) 0x0000ff01, 0 ) );
      }
    }
  }
  if( PACKED )
  {
#pragma unroll
    for( int bit = 0; bit < 5; bit++ )
    {
#pragma unroll
      for( int i = 0; i < 32; i++ )
      {
        if( !( i & ( 1 << bit ) ) )
        {
          const uint32_t a = u[i], b = u[i | ( 1 << bit )];
          u[i] = a + b - 0x80008000u; u[i | ( 1 << bit )] = a - b + 0x80008000u;
        }
      }
    }
#pragma unroll
    for( int i = 0; i < 32; i++ ) { d[2 * i] = dp2a_lo_us( u[i], 0x00000101, -65536 ); d[2 * i + 1] = dp2a_lo_us( u[i], 0x0000ff01, 0 ); }
  }
  return had8<PACKED ? 6 : 1>( d );                          // the stages the two forms have done
}

// The shared tables of both Hadamard refinement kernels: the MV-rate table, the pattern, and for the current group of blocks their descriptors, argmin
// keys and costs (block j at point k in cost[j * kStride + k], 0xffffffff where the point is outside the block's range).
struct HadTables { uint32_t* mv; vvb_mv* pat; vvb_block* blk; unsigned long long* key; uint32_t* cost; int kStride; };

// once per CTA: the MV-rate table and the pattern
__device__ __forceinline__ void had_load_tables( const HadTables& S, const MePar& par, const vvb_mv* __restrict__ pattern, int K )
{
  for( int i = threadIdx.x; i < VVB_MVCOST_ENTRIES; i += blockDim.x ) S.mv[i] = par.tab.cost[i];
  for( int i = threadIdx.x; i < K; i += blockDim.x ) S.pat[i] = pattern[i];
}

// start of a group of blocks firstBlk ... firstBlk + nSlot - 1, once the previous group is done with the tables: descriptors in, keys at "none"
__device__ __forceinline__ void had_group_begin( const HadTables& S, const vvb_block* __restrict__ blocks, int firstBlk, int nSlot )
{
  __syncthreads();
  for( int i = threadIdx.x; i < nSlot * 6; i += blockDim.x ) reinterpret_cast<uint32_t*>( S.blk )[i] = __ldg( reinterpret_cast<const uint32_t*>( blocks + firstBlk ) + i );
  if( threadIdx.x < nSlot ) S.key[threadIdx.x] = ~0ull;
}

// end of a group, once its cost table is complete: the table goes out, and the argmin with MV rate is taken in list order on ( tot << 16 ) | k, so the
// first strict minimum wins.  FOLD: a second half of the table lies at foldOff (64x64 ring blocks span two warps) and is added first; "outside" stays.
template<bool FOLD>
__device__ __forceinline__ void had_group_end( const HadTables& S, int foldOff, const MePar& par, int K, int firstBlk, int nSlot,
                                               uint32_t* __restrict__ costOut, vvb_best* __restrict__ bestOut )
{
  for( int i = threadIdx.x; i < nSlot * K; i += blockDim.x )
  {
    const int j = i / K, k = i - j * K;
    uint32_t c = S.cost[j * S.kStride + k];
    if( FOLD && c != 0xffffffffu ) { c += S.cost[foldOff + j * S.kStride + k]; S.cost[j * S.kStride + k] = c; }
    if( costOut ) costOut[(size_t)( firstBlk + j ) * K + k] = c;
    if( bestOut && c != 0xffffffffu )
    {
      const vvb_block b = S.blk[j];
      const vvb_mv pm = S.pat[k];
      const unsigned long long tot = (unsigned long long) c + mv_cost( par, S.mv, b.start_x + pm.dx, b.start_y + pm.dy, b.pred_hor, b.pred_ver );
      atomicMin( &S.key[j], ( tot << 16 ) | (unsigned) k );
    }
  }
  if( !bestOut ) return;
  __syncthreads();
  if( threadIdx.x < nSlot )
  {
    const unsigned long long key = S.key[threadIdx.x];
    vvb_best b;
    if( key == ~0ull ) { b.dx = 0; b.dy = 0; b.sad = 0xffffffffu; b.cost = ~0ull; }
    else
    {
      const int k = (int)( key & 0xffffu );
      const vvb_block bb = S.blk[threadIdx.x];
      const vvb_mv pm = S.pat[k];
      b.dx = (int16_t)( bb.start_x + pm.dx ); b.dy = (int16_t)( bb.start_y + pm.dy ); b.sad = S.cost[threadIdx.x * S.kStride + k]; b.cost = key >> 16;
    }
    bestOut[firstBlk + threadIdx.x] = b;
  }
}

// Persistent CTAs walk groups of `slots` blocks.  Per group: stage the windows, one lane per (block, tile) walks the K points, then had_group_end.
template<bool PACKED, int W, int RC>
__global__ void __launch_bounds__( 128, PACKED ? 5 : 4 ) had8_ring_kernel( const __grid_constant__ Plane orgPlane, const __grid_constant__ Plane refPlane,
                                                           const vvb_block* __restrict__ blocks, int nBlocks, const vvb_mv* __restrict__ pattern, int K,
                                                           const __grid_constant__ MePar par, uint32_t* __restrict__ costOut, vvb_best* __restrict__ bestOut )
{
  using Sh = HadRingShape<W, RC>;
  constexpr int TX = Sh::TX, T = Sh::T, RED = T < 32 ? T : 32;
  extern __shared__ __align__( 16 ) uint32_t smemHr[];
  __shared__ uint32_t sMv[VVB_MVCOST_ENTRIES];
  const int tid = threadIdx.x, nthr = blockDim.x, lane = tid & 31;
  const HadRingSmem L = had_ring_smem( nthr, T, Sh::S, K );
  uint32_t* sWin = smemHr;
  const HadTables S = { sMv, reinterpret_cast<vvb_mv*>( smemHr + L.patOff ), reinterpret_cast<vvb_block*>( smemHr + L.blkOff ),
                        reinterpret_cast<unsigned long long*>( smemHr + L.keyOff ), smemHr + L.costOff, L.kStride };
  had_load_tables( S, par, pattern, K );

  const int slot = tid / T, t = tid % T, tx = t % TX, ty = t / TX, half = t / 32;
  const int laneBase = slot * Sh::S + 8 * ty * Sh::PITCH + 4 * tx;
  const unsigned peers = __match_any_sync( 0xffffffffu, ( laneBase >> 2 ) & 7 );
  const int xr = __popc( peers & ( ( 1u << lane ) - 1u ) ) & 3;
  int wofs[4];                                                // this lane's word i of a window row sits at wofs[i] + row offset
#pragma unroll
  for( int i = 0; i < 4; i++ ) wofs[i] = laneBase + ( i ^ xr );
  const int nGroups = ( nBlocks + L.slots - 1 ) / L.slots;
  constexpr int perSlot = Sh::ROWS * Sh::CHUNKS;
  const int xLo = -refPlane.margin, xHi = refPlane.width + refPlane.margin, yLo = -refPlane.margin, yHi = refPlane.height + refPlane.margin;

  for( int g = blockIdx.x; g < nGroups; g += gridDim.x )
  {
    const int firstBlk = g * L.slots, nSlot = min( L.slots, nBlocks - firstBlk );
    had_group_begin( S, blocks, firstBlk, nSlot );            // its barrier also frees the windows

    // ---- stage the windows: consecutive threads take consecutive 16-byte chunks of a row; each chunk (+ the next word) fills 4 words of both copies
    for( int it = tid; it < nSlot * perSlot; it += nthr )
    {
      const int j = it / perSlot, rem = it - j * perSlot, row = rem / Sh::CHUNKS, q = rem - row * Sh::CHUNKS;
      const vvb_block* bp = blocks + firstBlk + j;
      const int gx0 = __ldg( &bp->x ) + __ldg( &bp->start_x ) - RC, gy = __ldg( &bp->y ) + __ldg( &bp->start_y ) - RC + row;
      const int16_t* p = refPlane.origin + (ptrdiff_t) gy * refPlane.stride + gx0;
      const int s = (int)( ( (uintptr_t) p >> 1 ) & 7 );      // pel offset of the window's first pel in its 16-byte chunk
      const int X = gx0 - s + 8 * q;                          // plane column of this chunk's first pel
      const uint32_t* cp = reinterpret_cast<const uint32_t*>( p - s ) + 4 * q;
      const bool rowOk = gy >= yLo && gy < yHi;               // chunks that hold no pel of the allocation are not read
      uint4 a = make_uint4( 0u, 0u, 0u, 0u ); uint32_t a4 = 0u;
      if( rowOk && X + 8 > xLo && X < xHi ) a = __ldg( reinterpret_cast<const uint4*>( cp ) );
      if( rowOk && X + 8 >= xLo && X + 8 < xHi ) a4 = __ldg( cp + 4 );
      const uint32_t A[5] = { a.x, a.y, a.z, a.w, a4 };
      uint32_t* w0 = sWin + j * Sh::S + row * Sh::PITCH;
      uint32_t* w1 = w0 + Sh::WIN1;
      const int odd = s & 1, m0 = 4 * q - ( s >> 1 );
#pragma unroll
      for( int e = 0; e < 4; e++ )
      {
        const uint32_t F = __funnelshift_r( A[e], A[e + 1], 16 );
        const int m = m0 + e, m1 = m - odd;
        if( m >= 0 && m < Sh::WPR ) w0[m] = odd ? F : A[e];
        if( m1 >= 0 && m1 < Sh::WPR ) w1[m1] = odd ? A[e] : F;
      }
    }
    __syncthreads();

    // ---- one lane per (block, tile): original tile once, then every pattern point
    const bool live = slot < nSlot;
    vvb_block blk = {};
    uint32_t o[32];
#pragma unroll
    for( int i = 0; i < 32; i++ ) o[i] = 0u;
    if( live )
    {
      blk = S.blk[slot];
      const int16_t* op = orgPlane.origin + (ptrdiff_t)( blk.y + 8 * ty ) * orgPlane.stride + blk.x + 8 * tx;
      const bool oW = ( ( (uintptr_t) op & 3 ) == 0 ) && ( ( orgPlane.stride & 1 ) == 0 );
#pragma unroll
      for( int r = 0; r < 8; r++ )
      {
#pragma unroll
        for( int i = 0; i < 4; i++ )
        {
          const int16_t* q = op + (ptrdiff_t) r * orgPlane.stride + 2 * ( i ^ xr );
          o[4 * r + i] = oW ? __ldg( reinterpret_cast<const uint32_t*>( q ) ) : ( (uint32_t)(uint16_t) __ldg( q ) | ( (uint32_t)(uint16_t) __ldg( q + 1 ) << 16 ) );
        }
      }
    }
    for( int k = 0; k < K; k++ )
    {
      const vvb_mv pm = S.pat[k];
      const int mx = blk.start_x + pm.dx, my = blk.start_y + pm.dy;
      const bool inside = live && mx >= blk.left && mx <= blk.right && my >= blk.top && my <= blk.bottom;     // the same for the lanes of a block
      uint32_t tileCost = 0;
      if( inside )
      {
        uint32_t c[32];
        if( pm.dx >= -RC && pm.dx <= RC && pm.dy >= -RC && pm.dy <= RC )      // the same for the whole warp
        {
          const int cx = pm.dx + RC;
          const int off = ( pm.dy + RC ) * Sh::PITCH + ( cx >> 1 ) + ( cx & 1 ) * Sh::WIN1;
#pragma unroll
          for( int r = 0; r < 8; r++ )
#pragma unroll
            for( int i = 0; i < 4; i++ ) c[4 * r + i] = sWin[wofs[i] + off + r * Sh::PITCH];
        }
        else
        {
          const int16_t* rp = refPlane.origin + (ptrdiff_t)( blk.y + my + 8 * ty ) * refPlane.stride + blk.x + mx + 8 * tx;
          const int odd = (int)( ( (uintptr_t) rp >> 1 ) & 1 );     // plane rows keep the parity (even strides)
          const uint32_t* rw = reinterpret_cast<const uint32_t*>( rp - odd );
#pragma unroll
          for( int r = 0; r < 8; r++ )
#pragma unroll
            for( int i = 0; i < 4; i++ )
            {
              const uint32_t* a = rw + (ptrdiff_t) r * ( refPlane.stride >> 1 ) + ( i ^ xr );
              c[4 * r + i] = odd ? __funnelshift_r( __ldg( a ), __ldg( a + 1 ), 16 ) : __ldg( a );
            }
        }
        tileCost = had8_tile_cost<PACKED>( [&]( int r, uint32_t ( &ow )[4], uint32_t ( &cw )[4] ) {
#pragma unroll
          for( int i = 0; i < 4; i++ ) { ow[i] = o[4 * r + i]; cw[i] = c[4 * r + i]; }
        } );
      }
#pragma unroll
      for( int d = 1; d < RED; d <<= 1 ) tileCost += __shfl_xor_sync( 0xffffffffu, tileCost, d );
      if( live && ( t & ( RED - 1 ) ) == 0 ) S.cost[( half * L.slots + slot ) * L.kStride + k] = inside ? tileCost : 0xffffffffu;
    }
    __syncthreads();
    had_group_end<( T > 32 )>( S, L.slots * L.kStride, par, K, firstBlk, nSlot, costOut, bestOut );
  }
}

// had8_direct_kernel: the same refinement without staging, used for 8x8 blocks, where it measured faster than had8_ring_kernel (there every lane of the
// ring kernel belongs to another block: each original load touches 32 lines, and 32 windows per warp limit the resident warps).  Persistent CTAs walk
// groups of BPC blocks; a lane owns a (block, candidate, 8x8 tile), reads its 8 original rows (LDG.128) and 8 reference rows (5 aligned words,
// funnel-shifted for odd columns) straight from the L1/L2-resident planes -- the K candidates of a block overlap almost completely, so the reads hit L1 --
// and sums the tile with had8_tile_cost.  Vector loads of the original need 16-byte aligned rows (checked per block, scalar loads otherwise).
struct HadDirSmem { int costOff, keyOff, blkOff, patOff, total; };
__host__ __device__ inline HadDirSmem had_dir_smem( int K, int BPC )
{
  HadDirSmem s;
  s.costOff = 0; s.keyOff = ( BPC * K + 1 ) & ~1; s.blkOff = s.keyOff + 2 * BPC; s.patOff = s.blkOff + 6 * BPC; s.total = s.patOff + K;
  return s;
}

template<bool PACKED>
__global__ void __launch_bounds__( 256 ) had8_direct_kernel( const __grid_constant__ Plane orgPlane, const __grid_constant__ Plane refPlane,
                                                             const vvb_block* __restrict__ blocks, int nBlocks, int w, int h, int BPC,
                                                             const vvb_mv* __restrict__ pattern, int K, const __grid_constant__ MePar par,
                                                             uint32_t* __restrict__ costOut, vvb_best* __restrict__ bestOut )
{
  extern __shared__ __align__( 16 ) uint32_t smemHd[];
  __shared__ uint32_t sMv[VVB_MVCOST_ENTRIES];
  const int tid = threadIdx.x, nthr = blockDim.x;
  const HadDirSmem L = had_dir_smem( K, BPC );
  const HadTables S = { sMv, reinterpret_cast<vvb_mv*>( smemHd + L.patOff ), reinterpret_cast<vvb_block*>( smemHd + L.blkOff ),
                        reinterpret_cast<unsigned long long*>( smemHd + L.keyOff ), smemHd + L.costOff, K };
  had_load_tables( S, par, pattern, K );
  const int tilesX = w >> 3, T = tilesX * ( h >> 3 ), perSlot = K * T;
  const int nGroups = ( nBlocks + BPC - 1 ) / BPC;
  const float invPer = 1.0f / (float) perSlot, invT = 1.0f / (float) T, invTx = 1.0f / (float) tilesX;
  for( int g = blockIdx.x; g < nGroups; g += gridDim.x )
  {
    const int firstBlk = g * BPC, nSlot = min( BPC, nBlocks - firstBlk );
    had_group_begin( S, blocks, firstBlk, nSlot );
    for( int i = tid; i < nSlot * K; i += nthr ) S.cost[i] = 0u;
    __syncthreads();
    for( int it = tid; it < nSlot * perSlot; it += nthr )
    {
      const int j = div_rcp( it, invPer ), loc = it - j * perSlot;
      const int k = div_rcp( loc, invT ), t = loc - k * T;
      const int ty = div_rcp( t, invTx ), tx = t - ty * tilesX;
      const vvb_block blk = S.blk[j];
      const vvb_mv pm = S.pat[k];
      const int mx = blk.start_x + pm.dx, my = blk.start_y + pm.dy;
      if( !( mx >= blk.left && mx <= blk.right && my >= blk.top && my <= blk.bottom ) ) { if( t == 0 ) S.cost[j * K + k] = 0xffffffffu; continue; }
      const int16_t* op = orgPlane.origin + (ptrdiff_t)( blk.y + ty * 8 ) * orgPlane.stride + blk.x + tx * 8;
      const int16_t* rp = refPlane.origin + (ptrdiff_t)( blk.y + my + ty * 8 ) * refPlane.stride + blk.x + mx + tx * 8;
      const bool oVec = ( ( (uintptr_t) op & 15 ) == 0 ) && ( ( orgPlane.stride & 7 ) == 0 );
      const int odd = (int)( ( (uintptr_t) rp >> 1 ) & 1 );      // plane rows keep the parity (even strides)
      const uint32_t* rw = reinterpret_cast<const uint32_t*>( rp - odd );
      const uint32_t tileCost = had8_tile_cost<PACKED>( [&]( int r, uint32_t ( &o )[4], uint32_t ( &c )[4] ) {
        const int16_t* q = op + (ptrdiff_t) r * orgPlane.stride;
        if( oVec )
        {
          const uint4 v = __ldg( reinterpret_cast<const uint4*>( q ) );
          o[0] = v.x; o[1] = v.y; o[2] = v.z; o[3] = v.w;
        }
        else
        {
#pragma unroll
          for( int m = 0; m < 4; m++ ) o[m] = (uint32_t)(uint16_t) __ldg( q + 2 * m ) | ( (uint32_t)(uint16_t) __ldg( q + 2 * m + 1 ) << 16 );
        }
        const uint32_t* rr = rw + (ptrdiff_t) r * ( refPlane.stride >> 1 );
#pragma unroll
        for( int m = 0; m < 4; m++ ) c[m] = __ldg( rr + m );
        if( odd )
        {
          const uint32_t c4 = __ldg( rr + 4 );
#pragma unroll
          for( int m = 0; m < 4; m++ ) c[m] = __funnelshift_r( c[m], m < 3 ? c[m + 1] : c4, 16 );
        }
      } );
      if( T == 1 ) S.cost[j * K + k] = tileCost; else atomicAdd( &S.cost[j * K + k], tileCost );
    }
    __syncthreads();
    had_group_end<false>( S, 0, par, K, firstBlk, nSlot, costOut, bestOut );
  }
}

// chains device-resident stages: the best vector of a search becomes the start / prediction offset of the next stage
__global__ void blocks_set_start_kernel( vvb_block* __restrict__ blocks, const vvb_best* __restrict__ best, int n )
{
  for( int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x )
  {
    blocks[i].start_x = best[i].dx; blocks[i].start_y = best[i].dy;
  }
}

} // namespace vvb
