// batch_kernels.cuh -- descriptor-list forms of the special distortions (SURVEY rows a7, a8, a9), also run by their single-call helpers:
//   sad_mask_batch_kernel  RdCost::xGetSADwMask (RdCost.cpp:2062-2093), GEO mask SAD
//   sad_x5_batch_kernel    RdCost::xGetSAD8X5 / xGetSAD16X5 (RdCost.cpp:1984-2034), DMVR's five horizontal positions
//   fix_wsse_batch_kernel  RdCost::fixWeightedSSE (RdCost.cpp:1948-1982)
// One warp per descriptor; the blocks sit in resident planes.  The affine step's list form is affine_eq_batch_kernel (mctf_affine_kernels.cuh).
#pragma once
#include "common.cuh"
#include "dist_kernels.cuh"

namespace vvb {

#define VVB_BATCH_WARPS 4

__global__ void __launch_bounds__( VVB_BATCH_WARPS * 32 ) sad_mask_batch_kernel( const __grid_constant__ PlaneTable planes, const vvb_mask_cand* __restrict__ cands, int n,
                                                                                 const int16_t* __restrict__ maskBuf, unsigned long long* __restrict__ out )
{
  const int i = blockIdx.x * VVB_BATCH_WARPS + ( threadIdx.x >> 5 ), lane = threadIdx.x & 31;
  if( i >= n ) return;
  const vvb_mask_cand d = cands[i];
  const Plane &po = planes.p[d.c.org_plane], &pc = planes.p[d.c.cur_plane];
  const int16_t* org = po.origin + (ptrdiff_t) d.c.org_y * po.stride + d.c.org_x;
  const int16_t* cur = pc.origin + (ptrdiff_t) d.c.cur_y * pc.stride + d.c.cur_x;
  const int16_t* mask = maskBuf + d.mask_offset;
  const int w = d.c.w, h = d.c.h, step = 1 << d.c.sub_shift, rows = h >> d.c.sub_shift;
  // RdCost.cpp:2062-2093: the mask pointer walks stepX per sample, then maskStride * step + maskStride2 per visited row
  const long long rowAdv = (long long) w * d.step_x + (long long) d.mask_stride * step + d.mask_stride2;
  unsigned long long acc = 0;
  for( int k = lane; k < rows * w; k += 32 )
  {
    const int r = k / w, x = k - r * w, y = r * step;
    acc += (unsigned long long)( abs( (int) org[(ptrdiff_t) y * po.stride + x] - (int) cur[(ptrdiff_t) y * pc.stride + x] ) * (int) mask[r * rowAdv + (long long) x * d.step_x] );
  }
  for( int m = 16; m > 0; m >>= 1 ) acc += __shfl_xor_sync( 0xffffffffu, acc, m );
  if( lane == 0 ) out[i] = acc << d.c.sub_shift;
}

__global__ void __launch_bounds__( VVB_BATCH_WARPS * 32 ) sad_x5_batch_kernel( const __grid_constant__ PlaneTable planes, const vvb_cand* __restrict__ cands, int n,
                                                                               unsigned long long* __restrict__ out5 )
{
  const int i = blockIdx.x * VVB_BATCH_WARPS + ( threadIdx.x >> 5 ), lane = threadIdx.x & 31;
  if( i >= n ) return;
  const vvb_cand d = cands[i];
  const Plane &po = planes.p[d.org_plane], &pc = planes.p[d.cur_plane];
  const int16_t* org = po.origin + (ptrdiff_t) d.org_y * po.stride + d.org_x;
  const int16_t* cur = pc.origin + (ptrdiff_t) d.cur_y * pc.stride + d.cur_x;
  // RdCost.cpp:1984-2034: position k compares org + k with cur - k, each SAD >> 1
  for( int k = 0; k < 5; k++ )
  {
    const uint32_t s = group_sad<32>( org + k, po.stride, cur - k, pc.stride, d.w, d.h, d.sub_shift, lane );      // reduced over the warp, scaled by the sub-sampling
    if( lane == 0 ) out5[(size_t) i * 5 + k] = s >> 1;
  }
}

__global__ void __launch_bounds__( VVB_BATCH_WARPS * 32 ) fix_wsse_batch_kernel( const __grid_constant__ PlaneTable planes, const vvb_cand* __restrict__ cands,
                                                                                 const uint32_t* __restrict__ weights, int n, unsigned long long* __restrict__ out )
{
  const int i = blockIdx.x * VVB_BATCH_WARPS + ( threadIdx.x >> 5 ), lane = threadIdx.x & 31;
  if( i >= n ) return;
  const vvb_cand d = cands[i];
  const Plane &po = planes.p[d.org_plane], &pc = planes.p[d.cur_plane];
  const int16_t* org = po.origin + (ptrdiff_t) d.org_y * po.stride + d.org_x;
  const int16_t* cur = pc.origin + (ptrdiff_t) d.cur_y * pc.stride + d.cur_x;
  const long long weight = weights[i];
  unsigned long long acc = 0;
  for( int k = lane; k < d.w * d.h; k += 32 )
  {
    const int y = k / d.w, x = k - y * d.w;
    const int df = (int) org[(ptrdiff_t) y * po.stride + x] - (int) cur[(ptrdiff_t) y * pc.stride + x];
    acc += (unsigned long long)(int)( ( weight * ( df * df ) + ( 1 << 15 ) ) >> 16 );              // RdCost.cpp:1942-1946
  }
  for( int m = 16; m > 0; m >>= 1 ) acc += __shfl_xor_sync( 0xffffffffu, acc, m );
  if( lane == 0 ) out[i] = acc;
}

// ---- levels trimmed to the last significant scan position (round 2, e2e): TU i contributes the levels at scan positions 0 .. lastPos[i], in scan order
__global__ void pack_sizes_kernel( const int32_t* __restrict__ lastPos, int n, uint32_t* __restrict__ sizes )
{
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if( i <= n ) sizes[i] = i < n ? (uint32_t) max( lastPos[i] + 1, 0 ) : 0u;
}
// warp per TU; fwd: scan position -> raster index inside the scanned region (row pitch 1 << lrw); q: compact [n][h][w]; out may be mapped host memory
__global__ void __launch_bounds__( 128 ) pack_levels_kernel( const int16_t* __restrict__ q, const int32_t* __restrict__ lastPos, const uint32_t* __restrict__ offsets,
                                                             const int32_t* __restrict__ fwd, int w, int area, int lrw, int n, int16_t* __restrict__ out )
{
  const int tu = blockIdx.x * 4 + ( threadIdx.x >> 5 ), lane = threadIdx.x & 31;
  if( tu >= n ) return;
  const int last = lastPos[tu];
  const uint32_t off = offsets[tu];
  const int16_t* qt = q + (size_t) tu * area;
  for( int s = lane; s <= last; s += 32 )
  {
    const int p = __ldg( fwd + s );
    out[off + s] = qt[( p >> lrw ) * w + ( p & ( ( 1 << lrw ) - 1 ) )];
  }
}

} // namespace vvb
