// common.cuh -- shared device helpers and the context object of the B200 cost path.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <string>
#include <vector>
#include "../../include/vvenc_b200.h"

#define VVB_MAX_PLANES 64

namespace vvb {

// A resident picture plane: origin points at sample (0,0) inside a buffer that carries `margin` samples on every side
// (mirrors PelStorage with extendBorderPel, CommonLib/Picture.cpp:461-501).
struct Plane
{
  const int16_t* origin;
  int stride, width, height, margin, bitDepth;
};

struct PlaneTable { Plane p[VVB_MAX_PLANES]; };

__device__ __forceinline__ int ilog2_dev( int v ) { return 31 - __clz( v ); }

// i / d for d > 0 given as inv = 1.0f / d: a float multiply instead of an integer division; exact for i < 2^20 and small divisors
__device__ __forceinline__ int div_rcp( int i, float inv ) { return __float2int_rz( ( (float) i + 0.5f ) * inv ); }

// ---- packed 16x2 arithmetic (SASS: VIMNMX.S16x2, IDP.2A) -------------------------------------------------------
// sum over both signed 16-bit halves of |a - b|, added to acc:  |a-b| = max(a,b) - min(a,b)
__device__ __forceinline__ int sad2_acc( uint32_t a, uint32_t b, int acc )
{
  const uint32_t mx = __vmaxs2( a, b );
  const uint32_t mn = __vmins2( a, b );
  acc = __dp2a_lo( (int) mx, 0x00000101, acc );          // + mx.lo + mx.hi
  acc = __dp2a_lo( (int) mn, (int) 0x0000ffffu, acc );   // - mn.lo - mn.hi   (bytes -1,-1)
  return acc;
}

__device__ __forceinline__ int lo16( uint32_t v ) { return (int)(short)( v & 0xffffu ); }
__device__ __forceinline__ int hi16( uint32_t v ) { return ( (int) v ) >> 16; }

// mask of the G-lane group this thread belongs to (groups are G-aligned inside a warp)
template<int G> __device__ __forceinline__ unsigned gmask()
{
  if( G == 32 ) return 0xffffffffu;
  unsigned lane;
  asm( "mov.u32 %0, %%laneid;" : "=r"( lane ) );
  return ( 0xffffffffu >> ( 32 - G ) ) << ( lane & ~( G - 1 ) );
}
template<int G> __device__ __forceinline__ uint32_t group_sum_u32( uint32_t v )
{
  const unsigned mk = gmask<G>();
#pragma unroll
  for( int m = G >> 1; m > 0; m >>= 1 ) v += __shfl_xor_sync( mk, v, m );
  return v;
}
template<int G> __device__ __forceinline__ unsigned long long group_sum_u64( unsigned long long v )
{
  const unsigned mk = gmask<G>();
#pragma unroll
  for( int m = G >> 1; m > 0; m >>= 1 ) v += __shfl_xor_sync( mk, v, m );
  return v;
}

// Exp-Golomb length used by the MV rate (CommonLib/RdCost.h:183-201)
__device__ __forceinline__ uint32_t eg_bits( int v )
{
  const uint32_t t = v <= 0 ? ( (uint32_t)( -v ) << 1 ) + 1u : (uint32_t) v << 1;
  return 1u + ( (uint32_t)( 31 - __clz( t ) ) << 1 );
}

#define VVB_MVCOST_ENTRIES 80
struct MvCostTable { uint32_t cost[VVB_MVCOST_ENTRIES]; };   // cost[bits] = Distortion( sqrt(lambda) * bits ), host-computed in IEEE double

enum class ScratchArena { Host, Work };                      // the two scratch arenas of a context (vvb_ctx::d_scratch)

} // namespace vvb

// ---- host side -------------------------------------------------------------------------------------------------
struct vvb_ctx
{
  int            device   = 0;
  cudaStream_t   stream   = nullptr;
  vvb::PlaneTable planes  {};
  void*          owned[VVB_MAX_PLANES] = {};
  size_t         ownedBytes[VVB_MAX_PLANES] = {};
  bool           bound[VVB_MAX_PLANES] = {};
  std::string    err;
  uint64_t       launches = 0;
  bool           poolBlocksAligned = false;   // see vvb_pool_hint
  void*          itcImage[36] = {};           // the same for the inverse tensor engine
  void*          tc2Image[36] = {};           // B operand images of the raw-byte tensor engine, index ((lw - 3) * 3 + trHor) * 3 + trVer
  bool           tensorTransform = true;      // see vvb_set_tensor_transform: on = raw-byte wgmma engines where they apply (tensorFwd, tensorInv in capi.cu), off = CUDA cores for every shape
  int            rdoqEngine = 1;              // see vvb_set_rdoq_engine: 1 = templates gathered per position (first engine, verified on hardware), 2 = accumulated templates + cost tables
  int            dqEngine = 1;                // see vvb_set_depquant_engine: 1 = four lanes per TU (one per trellis state), 0 = one thread per TU
  int            pyramidEngine = 1;           // see vvb_set_pyramid_engine: 1 = all pyramid levels inside one CTA per root block, 0 = per-quad kernel + table sums
  int            useTma = 2;                  // see vvb_set_tma_staging: 0 off, 1 on, 2 (default) on where measured faster (blocks up to 8 wide)
  void*          tmaEncode = nullptr;         // cuTensorMapEncodeTiled, resolved at vvb_create
  int            numSMs   = 132;
  // device-side constant data
  int8_t*        d_trTable   = nullptr;     // all transform matrices (vvc_tables.h)
  int8_t*        d_lfnst     = nullptr;     // LFNST forward kernels (vvc_lfnst_tables.h)
  int32_t*       d_scan      = nullptr;     // scan tables for all (log2w, log2h) in 2..6, 1024 entries each
  void*          d_dqScan    = nullptr;     // dependent quantisation: ScanInfo / NbInfoOut tables of the 25 shapes (built at the first vvb_dep_quant call)
  void*          d_dqNb      = nullptr;
  void*          dqShapes    = nullptr;     // host: vvbdq::DqShapeTables[25]
  int16_t*       d_mask      = nullptr;     // GEO weight masks (vvb_mask_upload)
  int            maskCount   = 0;
  int            mctfMaxDim = 64;      // largest MCTF block dimension in device-resident candidate lists (vvb_mctf_hint)
  bool           async = false;        // host-buffer calls enqueue only; vvb_synchronize() completes them (vvb_set_async)
  // Grow-only device scratch, indexed by vvb::ScratchArena.  Growing an arena synchronises the stream and frees the old buffer, so whoever holds an arena
  // must not call anything that takes the same one:
  //  - Host: the buffers of one host-buffer entry point or single-block helper, for the duration of that call; its _dev twin never takes Host.
  //  - Work: the temporaries of a _dev call.  A _dev call that holds Work never calls another entry point that takes Work.
  void*          d_scratch[2] = {};
  size_t         d_scratchSize[2] = {};
  std::vector<uint8_t> hostStage;      // host side of the single-call helpers' one upload (BlockCall in capi.cu)
};
