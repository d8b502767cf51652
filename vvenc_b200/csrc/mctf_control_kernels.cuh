// mctf_control_kernels.cuh -- the control of the MCTF motion search on the device: MCTF::motionEstimationLuma / estimateLumaLn (CommonLib/MCTF.cpp:1166-1397).
// The error tables come from mctf_error_packed_kernel / mctf_grid_kernel (mctf_affine_kernels.cuh); the kernels here build the candidate lists, replay the
// `error < best.error` chains in the reference's loop order and resolve the dependency on the upper and left neighbour (the prevLineX scheme of :1176, 1357-1386)
// with one warp per block row that waits for the row above, so that a whole pyramid level runs without the host looking at a number.
//   stage A  mctf_pred_cands_kernel + mctf_select_list_kernel : the 3x3 neighbourhood of the coarser level's field and the zero vector       (:1191-1214)
//   stage B  mctf_centre_kernel + grid + mctf_select_grid_kernel: integer grid around trunc(best / 16)                                      (:1216-1228)
//   stage C  the same pair, three times, around the running best with the centre skipped (doubleRes)                                        (:1229-1287)
//   stage D  mctf_wave_kernel: final vectors of the block above and of the block to the left                                                (:1288-1306)
//   stage E  mctf_final_kernel: error scaling with the block variance, rmsme (doubleRes)                                                    (:1308-1321)
// vvenc_b200/mctf_host.py holds the same replay on the host (the round-1 path, kept as the test oracle's driver).
#pragma once
#include "common.cuh"
#include "mctf_affine_kernels.cuh"

namespace vvb {

struct MctfGeom
{
  int width, height, bs, bxn, byn, n;      // level picture, block size, blocks per row / column (`blockX + 8 <= origWidth`, :1174, 1388)
  int prevW, prevH, factor;                // coarser level's field (0 x 0: none) and the vector scale between the levels
  int outW, outH;                          // field array the level writes into (entries no block writes keep the default vector 0,0)
};
struct MctfBest { int x, y, e; };

__device__ __forceinline__ void mctf_block_of( const MctfGeom& g, int i, int& X, int& Y, int& W, int& H )
{
  const int by = i / g.bxn, bx = i - by * g.bxn;
  X = bx * g.bs; Y = by * g.bs;
  W = min( g.bs, g.width - X ) & ~7; H = min( g.bs, g.height - Y ) & ~7;
}

__global__ void mctf_init_kernel( MctfGeom g, MctfBest* __restrict__ best, int* __restrict__ progress )
{
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if( i < g.n ) { best[i].x = 0; best[i].y = 0; best[i].e = 0x7fffffff; }          // MotionVector(): error = INT_LEAST32_MAX (MCTF.h:79)
  if( i <= g.byn ) progress[i] = 0;                                                 // [0] = row ticket, [1 + row] = blocks finished in that row
}

// candidate k of block i: k = 0..8 the coarser level's vector at (Y / 2bs + dy, X / 2bs + dx), dy outer, dx inner; k = 9 the zero vector.  Positions outside
// the coarser field are evaluated as the zero vector and ignored by the selection.
__global__ void mctf_pred_cands_kernel( MctfGeom g, const vvb_mctf_mv* __restrict__ prev, vvb_mctf_cand* __restrict__ cands )
{
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if( t >= g.n * 10 ) return;
  const int i = t / 10, k = t - i * 10;
  int X, Y, W, H; mctf_block_of( g, i, X, Y, W, H );
  vvb_mctf_cand c; c.x = X; c.y = Y; c.w = (uint16_t) W; c.h = (uint16_t) H; c.mvx = 0; c.mvy = 0;
  if( k < 9 )
  {
    const int ty = Y / ( 2 * g.bs ) + k / 3 - 1, tx = X / ( 2 * g.bs ) + k % 3 - 1;
    if( ty >= 0 && ty < g.prevH && tx >= 0 && tx < g.prevW ) { const vvb_mctf_mv p = prev[ty * g.prevW + tx]; c.mvx = p.x * g.factor; c.mvy = p.y * g.factor; }
  }
  cands[t] = c;
}

__global__ void mctf_select_list_kernel( MctfGeom g, const vvb_mctf_cand* __restrict__ cands, const int32_t* __restrict__ err, MctfBest* __restrict__ best )
{
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if( i >= g.n ) return;
  int X, Y, W, H; mctf_block_of( g, i, X, Y, W, H );
  MctfBest b = best[i];
  for( int k = 0; k < 10; k++ )
  {
    if( k < 9 )
    {
      const int ty = Y / ( 2 * g.bs ) + k / 3 - 1, tx = X / ( 2 * g.bs ) + k % 3 - 1;
      if( !( ty >= 0 && ty < g.prevH && tx >= 0 && tx < g.prevW ) ) continue;
    }
    const int e = err[i * 10 + k];
    if( e < b.e ) { b.e = e; b.x = cands[i * 10 + k].mvx; b.y = cands[i * 10 + k].mvy; }
  }
  best[i] = b;
}

// grid centre of every block: truncInt != 0 -> trunc( best / 16 ) * 16 (C division, `prevBest.x / m_motionVectorFactor`), else the running best; the block list
// handed to the grid kernel carries centre + shift (the lattice of the grid call may be offset against the offsets the selection visits)
__global__ void mctf_centre_kernel( MctfGeom g, const MctfBest* __restrict__ best, int truncInt, int shift, int2* __restrict__ centre, vvb_mctf_cand* __restrict__ blocks )
{
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if( i >= g.n ) return;
  int X, Y, W, H; mctf_block_of( g, i, X, Y, W, H );
  int cx = best[i].x, cy = best[i].y;
  if( truncInt ) { cx = ( cx / 16 ) * 16; cy = ( cy / 16 ) * 16; }
  centre[i] = make_int2( cx, cy );
  vvb_mctf_cand c; c.x = X; c.y = Y; c.w = (uint16_t) W; c.h = (uint16_t) H; c.mvx = cx + shift; c.mvy = cy + shift;
  blocks[i] = c;
}

// offsets o = off0 + k * delta (k = 0..count-1) in both directions, y outer, x inner, strictly smaller wins; the table holds the lattice (o - off0) / step
__global__ void mctf_select_grid_kernel( MctfGeom g, const int32_t* __restrict__ tab, int K1, int off0, int delta, int count, int step, int skipZero,
                                         const int2* __restrict__ centre, MctfBest* __restrict__ best )
{
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if( i >= g.n ) return;
  MctfBest b = best[i];
  const int2 c = centre[i];
  const int32_t* t = tab + (size_t) i * K1 * K1;
  const int stride = delta / step;
  for( int j = 0; j < count; j++ )
    for( int k = 0; k < count; k++ )
    {
      const int oy = off0 + j * delta, ox = off0 + k * delta;
      if( skipZero && ox == 0 && oy == 0 ) continue;
      const int e = t[j * stride * K1 + k * stride];
      if( e < b.e ) { b.e = e; b.x = c.x + ox; b.y = c.y + oy; }
    }
  best[i] = b;
}

// stage D: one CTA per block row (rows are claimed through a ticket, so a waiting row always has the row above already running or finished).  The two
// candidates of a block -- the final vector of the block above, then that of the block to the left -- are evaluated side by side: four warps each, a warp
// takes a horizontal quarter of the block (the error is a sum over pels, and a pel's interpolation only reads its own neighbourhood, so the quarters add up to
// motionErrorLuma of the block exactly).  A candidate whose vector equals the block's current vector (or the other candidate's) cannot win the strict
// `error < best.error` and is not evaluated -- on smooth fields that is most of them.  The four quarters add up in 64 bits and saturate to 0x7fffffff.
#define MCTF_WAVE_WARPS 8
// a warp's slice holds one quarter: up to maxDim x maxDim / 4 pels (8 warps of 64 x 64 regions would not fit the 100 KB the kernel is given)
__host__ __device__ inline MctfSmem mctf_wave_smem( int maxDim ) { return mctf_smem( maxDim, maxDim >> 2 ); }
__global__ void __launch_bounds__( MCTF_WAVE_WARPS * 32 ) mctf_wave_kernel( const __grid_constant__ Plane orgPlane, const __grid_constant__ Plane refPlane, MctfGeom g, int tap4, int maxDim,
                                                                            MctfBest* best, int* progress )
{
  extern __shared__ __align__( 16 ) uint32_t sWave[];
  __shared__ int sRow;
  __shared__ unsigned sErr[MCTF_WAVE_WARPS];
  const MctfSmem L = mctf_wave_smem( maxDim );
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  uint32_t* region = sWave + warp * L.warpWords; uint32_t* t2 = region + L.regionWords;
  if( threadIdx.x == 0 ) sRow = atomicAdd( &progress[0], 1 );
  __syncthreads();
  const int by = sRow;
  if( by >= g.byn ) return;
  volatile int* above = progress + by;                  // progress[1 + (by - 1)]
  MctfBest left = { 0, 0, 0 };
  for( int bx = 0; bx < g.bxn; bx++ )
  {
    const int i = by * g.bxn + bx;
    int X, Y, W, H; mctf_block_of( g, i, X, Y, W, H );
    MctfBest b;
    b.x = best[i].x; b.y = best[i].y; b.e = best[i].e;
    MctfBest up = { b.x, b.y, 0 };
    if( by > 0 )
    {
      if( threadIdx.x == 0 ) while( *above <= bx ) __nanosleep( 32 );
      __syncthreads();
      __threadfence();
      up.x = __ldcg( &best[i - g.bxn].x ); up.y = __ldcg( &best[i - g.bxn].y );
    }
    const bool needUp   = by > 0 && ( up.x != b.x || up.y != b.y );
    const bool needLeft = bx > 0 && ( left.x != b.x || left.y != b.y ) && !( by > 0 && left.x == up.x && left.y == up.y );
    const bool mine = warp < 4 ? needUp : needLeft;
    if( mine )
    {
      const int q = warp & 3, sh = H >> 2;                // H is a multiple of 8: quarters of an even number of rows
      vvb_mctf_cand c; c.x = X; c.y = Y + q * sh; c.w = (uint16_t) W; c.h = (uint16_t) sh;
      c.mvx = warp < 4 ? up.x : left.x; c.mvy = warp < 4 ? up.y : left.y;
      const unsigned e = mctf_warp_error( orgPlane, refPlane, c, tap4, L, region, t2, lane );
      if( lane == 0 ) sErr[warp] = e;
    }
    __syncthreads();
    if( needUp )   { const int e = mctf_sat32( (unsigned long long) sErr[0] + sErr[1] + sErr[2] + sErr[3] ); if( e < b.e ) { b.e = e; b.x = up.x; b.y = up.y; } }
    if( needLeft ) { const int e = mctf_sat32( (unsigned long long) sErr[4] + sErr[5] + sErr[6] + sErr[7] ); if( e < b.e ) { b.e = e; b.x = left.x; b.y = left.y; } }
    left = b;
    if( threadIdx.x == 0 )
    {
      best[i].x = b.x; best[i].y = b.y; best[i].e = b.e;
      __threadfence();
      atomicExch( &progress[1 + by], bx + 1 );
    }
    __syncthreads();                                      // sErr is rewritten by the next block
  }
}

// Integer search grid (stage B: step 16, centre on the integer grid): motionErrorLumaInt (MCTF.cpp:122-145) for all (2r+1)^2 integer displacements of one block
// in one CTA, without the interpolation machinery of mctf_grid_kernel.  SSE = sum o^2 + sum r^2 - 2 sum o r:
//   sum o r   pels are unsigned and below 2^10, so r = 256 r_hi + r_lo with both parts in a byte: the reference window is staged as words
//             ( r_lo[x], r_lo[x+1], r_hi[x], r_hi[x+1] ) -- once for even x, once for odd x -- and a pel pair of the original costs two IDP.2A
//             ( dp2a.lo against the low bytes, dp2a.hi against the high bytes );
//   sum r^2   box sums of the squared window by two sliding passes, shared by all candidates;
//   sum o^2   once per block.
// Same table layout as mctf_grid_kernel (out[b][j][i], displacement centre + (i - r, j - r) * 16); the exact 64-bit SSE saturates to 0x7fffffff.
struct MctfIntSmem { int orgWords, pitch, rows, planeWords, sqPitch, total; };
__host__ __device__ inline MctfIntSmem mctf_int_smem( int maxDim, int radius )
{
  MctfIntSmem m;
  m.orgWords = ( maxDim >> 1 ) * maxDim;
  m.pitch = ( ( maxDim + 2 * radius ) >> 1 ) + 1;               // words per window row of one parity plane
  m.rows = maxDim + 2 * radius;
  m.planeWords = m.rows * m.pitch;
  m.sqPitch = 2 * radius + 1;
  m.total = m.orgWords + 2 * m.planeWords + m.rows * m.sqPitch + m.sqPitch * m.sqPitch + 8;
  return m;
}

__global__ void __launch_bounds__( 128 ) mctf_int_grid_kernel( const __grid_constant__ Plane orgPlane, const __grid_constant__ Plane refPlane, const vvb_mctf_cand* __restrict__ blocks,
                                                               int n, int radius, int maxDim, int32_t* __restrict__ out )
{
  extern __shared__ __align__( 16 ) uint32_t sInt[];
  const MctfIntSmem L = mctf_int_smem( maxDim, radius );
  uint32_t* sOrg = sInt;                                        // [h][w/2] packed pel pairs
  uint32_t* sP0  = sOrg + L.orgWords;                           // window pairs starting at even window columns
  uint32_t* sP1  = sP0 + L.planeWords;                          // ... at odd window columns
  unsigned* sHs = sP1 + L.planeWords;                           // [rows][2r+1] horizontal sliding sums of r^2 (64 x 64 x 1023^2 still fits 32 bits unsigned)
  unsigned* sV  = sHs + L.rows * L.sqPitch;                          // [2r+1][2r+1] box sums of r^2
  __shared__ unsigned long long sOo;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, K1 = 2 * radius + 1;
  for( int b = blockIdx.x; b < n; b += gridDim.x )
  {
    const vvb_mctf_cand blk = blocks[b];
    const int w = blk.w, h = blk.h, hw = w >> 1;
    const int ww = w + 2 * radius, wr = h + 2 * radius;        // window size in pels
    const int16_t* org = orgPlane.origin + (ptrdiff_t) blk.y * orgPlane.stride + blk.x;
    const int16_t* ref = refPlane.origin + (ptrdiff_t)( blk.y + blk.mvy / 16 - radius ) * refPlane.stride + blk.x + blk.mvx / 16 - radius;
    __syncthreads();
    if( tid == 0 ) sOo = 0;
    for( int i = tid; i < wr * L.pitch; i += blockDim.x )
    {
      const int y = i / L.pitch, p = i - y * L.pitch, x = 2 * p;
      const int16_t* rp = ref + (ptrdiff_t) y * refPlane.stride + x;
      const unsigned a0 = x < ww ? (unsigned)(unsigned short) __ldg( rp ) : 0u, a1 = x + 1 < ww ? (unsigned)(unsigned short) __ldg( rp + 1 ) : 0u, a2 = x + 2 < ww ? (unsigned)(unsigned short) __ldg( rp + 2 ) : 0u;
      sP0[i] = ( a0 & 255u ) | ( ( a1 & 255u ) << 8 ) | ( ( a0 >> 8 ) << 16 ) | ( ( a1 >> 8 ) << 24 );
      sP1[i] = ( a1 & 255u ) | ( ( a2 & 255u ) << 8 ) | ( ( a1 >> 8 ) << 16 ) | ( ( a2 >> 8 ) << 24 );
    }
    unsigned long long oo = 0;
    for( int i = tid; i < h * hw; i += blockDim.x )
    {
      const int y = i / hw, p = i - y * hw;
      const unsigned o0 = (unsigned short) __ldg( org + (ptrdiff_t) y * orgPlane.stride + 2 * p ), o1 = (unsigned short) __ldg( org + (ptrdiff_t) y * orgPlane.stride + 2 * p + 1 );
      sOrg[i] = o0 | ( o1 << 16 );
      oo += (unsigned long long)( o0 * o0 + o1 * o1 );
    }
    for( int m = 16; m > 0; m >>= 1 ) oo += __shfl_xor_sync( 0xffffffffu, oo, m );
    __syncthreads();
    if( lane == 0 ) atomicAdd( &sOo, oo );
    // horizontal sliding sums of r^2: Hs[y][dx] = sum over x in [dx, dx + w) of r(y, x)^2
    for( int y = tid; y < wr; y += blockDim.x )
    {
      const int16_t* rp = ref + (ptrdiff_t) y * refPlane.stride;
      unsigned sacc = 0;
      for( int x = 0; x < w; x++ ) { const unsigned v = (unsigned short) __ldg( rp + x ); sacc += v * v; }
      sHs[y * L.sqPitch] = sacc;
      for( int dx = 1; dx < K1; dx++ ) { const unsigned v0 = (unsigned short) __ldg( rp + dx - 1 ), v1 = (unsigned short) __ldg( rp + dx - 1 + w ); sacc += v1 * v1 - v0 * v0; sHs[y * L.sqPitch + dx] = sacc; }
    }
    __syncthreads();
    for( int dx = tid; dx < K1; dx += blockDim.x )
    {
      unsigned sacc = 0;
      for( int y = 0; y < h; y++ ) sacc += sHs[y * L.sqPitch + dx];
      sV[dx] = sacc;
      for( int dy = 1; dy < K1; dy++ ) { sacc += sHs[( dy - 1 + h ) * L.sqPitch + dx] - sHs[( dy - 1 ) * L.sqPitch + dx]; sV[dy * L.sqPitch + dx] = sacc; }
    }
    __syncthreads();
    const unsigned long long ooAll = sOo;
    for( int c = warp; c < K1 * K1; c += ( blockDim.x >> 5 ) )
    {
      const int j = c / K1, i0 = c - j * K1;                    // displacement (i0 - r, j - r): window origin (i0, j)
      const uint32_t* plane = ( i0 & 1 ) ? sP1 : sP0;
      const int pw = i0 >> 1;
      unsigned lo = 0, hi = 0;
      if( ( hw & ( hw - 1 ) ) == 0 && hw <= 32 )
      {
        // w in {8, 16, 32, 64}: a lane keeps its column pair and walks down the rows (32 / hw rows per step) -- no index division in the loop
        const int p = lane & ( hw - 1 ), y0 = lane / hw, rowsPerStep = 32 / hw;
        const uint32_t* rp = plane + ( y0 + j ) * L.pitch + pw + p;
        const uint32_t* op = sOrg + lane;
        const int rstep = rowsPerStep * L.pitch;
#pragma unroll 4
        for( int y = y0; y < h; y += rowsPerStep, rp += rstep, op += 32 )
        {
          const unsigned o = *op, r = *rp;
          lo = __dp2a_lo( o, r, lo ); hi = __dp2a_hi( o, r, hi );
        }
      }
      else
        for( int t = lane; t < h * hw; t += 32 )
        {
          const int y = t / hw, p = t - y * hw;
          const unsigned o = sOrg[t], r = plane[( y + j ) * L.pitch + pw + p];
          lo = __dp2a_lo( o, r, lo ); hi = __dp2a_hi( o, r, hi );
        }
      unsigned long long cross = (unsigned long long) lo + 256ull * hi;
      for( int m = 16; m > 0; m >>= 1 ) cross += __shfl_xor_sync( 0xffffffffu, cross, m );
      if( lane == 0 ) out[(size_t) b * K1 * K1 + c] = mctf_sat32( ooAll + (unsigned long long) sV[j * L.sqPitch + i0] - 2ull * cross );
    }
  }
}

// stage E and the hand-over to the next level / the apply stage: field[by][bx] = { x, y, error, rmsme } for the blocks inside the out_w x out_h array
__global__ void mctf_final_kernel( MctfGeom g, const MctfBest* __restrict__ best, const double* __restrict__ var, int doubleRes, int bitDepth, vvb_mctf_mv* __restrict__ field )
{
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if( i >= g.n ) return;
  const int by = i / g.bxn, bx = i - by * g.bxn;
  if( bx >= g.outW || by >= g.outH ) return;
  int X, Y, W, H; mctf_block_of( g, i, X, Y, W, H );
  const MctfBest b = best[i];
  vvb_mctf_mv m; m.x = b.x; m.y = b.y; m.error = b.e; m.rmsme = 0xffff; m.pad = 0;
  if( doubleRes )
  {
    const double bdScale = (double)( 1 << ( 2 * ( 10 - bitDepth ) ) );
    const double wh = (double) W * (double) H;
    const double dvar = var[i] * bdScale;
    const double mse = (double) b.e * bdScale / wh;
    m.error = (int)( 20 * ( ( (double) b.e * bdScale + 5.0 ) / ( dvar + 5.0 ) ) + mse / 50.0 );
    m.rmsme = (uint16_t)(int)( 0.5 + sqrt( mse ) );
  }
  field[by * g.outW + bx] = m;
}

// MCTF::subsampleLuma (MCTF.cpp:1072-1097) with the border replication of PelStorage::extendBorderPel: dst(x, y) for x, y in [-margin, size + margin)
__global__ void mctf_subsample_kernel( const __grid_constant__ Plane src, int16_t* __restrict__ dstOrigin, int dstStride, int dw, int dh, int margin )
{
  const int x = blockIdx.x * blockDim.x + threadIdx.x - margin, y = blockIdx.y * blockDim.y + threadIdx.y - margin;
  if( x >= dw + margin || y >= dh + margin ) return;
  const int cx = min( max( x, 0 ), dw - 1 ), cy = min( max( y, 0 ), dh - 1 );
  const int16_t* p = src.origin + (ptrdiff_t)( 2 * cy ) * src.stride + 2 * cx;
  dstOrigin[(ptrdiff_t) y * dstStride + x] = (int16_t)( ( (int) p[0] + (int) p[src.stride] + (int) p[1] + (int) p[src.stride + 1] + 2 ) >> 2 );
}

} // namespace vvb
