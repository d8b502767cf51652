// capi.cu -- C ABI (include/vvenc_b200.h) of the B200 block-cost path: context, plane residency, launch logic.
// There is deliberately no CPU fallback anywhere in this file: without a usable CUDA device every entry point fails.
#include <cstdio>
#include <cstring>
#include <cstdlib>
#include <cmath>
#include <algorithm>
#include <new>
#include "common.cuh"
#include <cub/device/device_scan.cuh>
#include "dist_kernels.cuh"
#include "search_kernels.cuh"
#include "pyramid_kernels.cuh"
#include "trquant_kernels.cuh"
#include "trquant_tc2_kernels.cuh"
#include "itrquant_kernels.cuh"
#include "itrquant_tc_kernels.cuh"
#include "mctf_affine_kernels.cuh"
#include "frac_kernels.cuh"
#include "depquant_kernels.cuh"
#include "rdoq_kernels.cuh"
#include "batch_kernels.cuh"
#include "mctf_control_kernels.cuh"
#include "depquant_host.h"
#include "rdoq_host.h"
#include "vvc_tables.h"
#include "vvc_lfnst_tables.h"

using namespace vvb;

namespace {

int fail( vvb_ctx* c, int code, const char* what, cudaError_t e = cudaSuccess )
{
  if( c )
  {
    c->err = what;
    if( e != cudaSuccess ) { c->err += ": "; c->err += cudaGetErrorString( e ); }
  }
  return code;
}

#define CU( call ) do { cudaError_t e_ = ( call ); if( e_ != cudaSuccess ) return fail( ctx, VVB_ERR_CUDA, #call, e_ ); } while( 0 )
#define CHECK_LAUNCH( name ) do { cudaError_t e_ = cudaGetLastError(); if( e_ != cudaSuccess ) return fail( ctx, VVB_ERR_CUDA, name, e_ ); ctx->launches++; } while( 0 )

bool isPow2( int v ) { return v > 0 && ( v & ( v - 1 ) ) == 0; }
int  ilog2h( int v ) { int r = 0; while( v > 1 ) { v >>= 1; r++; } return r; }

int scratch( vvb_ctx* ctx, ScratchArena which, size_t bytes, void** out )
{
  const int arena = (int) which;
  if( bytes == 0 ) bytes = 16;
  if( ctx->d_scratchSize[arena] < bytes )
  {
    if( ctx->d_scratch[arena] ) { cudaStreamSynchronize( ctx->stream ); cudaFree( ctx->d_scratch[arena] ); ctx->d_scratch[arena] = nullptr; ctx->d_scratchSize[arena] = 0; }
    const size_t cap = bytes + bytes / 4 + 4096;
    CU( cudaMalloc( &ctx->d_scratch[arena], cap ) );
    ctx->d_scratchSize[arena] = cap;
  }
  *out = ctx->d_scratch[arena];
  return VVB_OK;
}

// Buffers laid out back to back, each rounded up to 256 bytes.  A walk with a null base only adds up the total; the same walk over an allocation
// of that size hands out the pointers.
struct Layout
{
  uint8_t* base = nullptr;
  size_t total = 0;
  template<class T> T* take( size_t count )
  {
    T* p = base ? reinterpret_cast<T*>( base + total ) : nullptr;
    total += ( count * sizeof( T ) + 255 ) & ~(size_t) 255;
    return p;
  }
};

// sizes the buffers `carve( Layout& )` takes, allocates them in one arena and walks `carve` again to set its pointers
template<class F> int carveArena( vvb_ctx* ctx, ScratchArena arena, F&& carve )
{
  Layout size;
  carve( size );
  void* mem;
  const int rc = scratch( ctx, arena, size.total, &mem );
  if( rc ) return rc;
  Layout at{ (uint8_t*) mem };
  carve( at );
  return VVB_OK;
}

// End of a host-buffer entry point: blocking mode waits for the stream (results are in the caller's buffers on return); in asynchronous mode the
// call only enqueues (copies included) and vvb_synchronize() is the completion point.
inline cudaError_t endCall( vvb_ctx* ctx ) { return ctx->async ? cudaSuccess : cudaStreamSynchronize( ctx->stream ); }

// The protocol of a host-buffer entry point around its _dev twin: in() buffers are copied up before `call`, out() buffers copied down after it, then
// the call ends (endCall).  All of them live in the Host arena.  A null host pointer gives a null device pointer and no copy; `always` keeps the
// device buffer of an output the _dev twin needs even when the caller does not want it, and tmp() is a device buffer without a copy.
class HostCall
{
public:
  explicit HostCall( vvb_ctx* c ) : ctx( c ) {}
  template<class T> HostCall& in( const T*& dev, const T* host, size_t count ) { return add( dev, host, nullptr, count, false ); }
  template<class T> HostCall& out( T*& dev, T* host, size_t count, bool always = false ) { return add( dev, nullptr, host, count, always ); }
  template<class T> HostCall& tmp( T*& dev, size_t count ) { return add( dev, nullptr, nullptr, count, true ); }
  template<class F> int run( F&& call )
  {
    if( nb > MaxBufs ) return fail( ctx, VVB_ERR_ARG, "too many staged buffers" );
    const Buf* end = bufs + nb;
    int rc = carveArena( ctx, ScratchArena::Host, [&]( Layout& L ) { for( Buf* b = bufs; b < end; b++ ) b->set( b->slot, b->dev = b->in || b->out || b->always ? L.take<uint8_t>( b->bytes ) : nullptr ); } );
    if( rc ) return rc;
    for( const Buf* b = bufs; b < end; b++ ) if( b->in && b->bytes ) CU( cudaMemcpyAsync( b->dev, b->in, b->bytes, cudaMemcpyHostToDevice, ctx->stream ) );
    if( ( rc = call() ) ) return rc;
    for( const Buf* b = bufs; b < end; b++ ) if( b->out && b->bytes ) CU( cudaMemcpyAsync( b->out, b->dev, b->bytes, cudaMemcpyDeviceToHost, ctx->stream ) );
    CU( endCall( ctx ) );
    return VVB_OK;
  }
private:
  static constexpr int MaxBufs = 48;               // vvb_search_refine_tu stages the most: up to nine buffers per level for five levels, and the pattern
  struct Buf { void* slot; void ( *set )( void* slot, uint8_t* dev ); uint8_t* dev; const void* in; void* out; size_t bytes; bool always; };
  template<class T> HostCall& add( T*& dev, const void* in, void* out, size_t count, bool always )
  {
    if( nb < MaxBufs ) bufs[nb] = Buf{ &dev, []( void* slot, uint8_t* p ) { *static_cast<T**>( slot ) = reinterpret_cast<T*>( p ); }, nullptr, in, out, count * sizeof( T ), always };
    nb++;
    return *this;
  }
  vvb_ctx* ctx;
  Buf bufs[MaxBufs];
  int nb = 0;
};

// The single-block helpers that return their value: `body` checks the arguments, enqueues the work and points dOut at the 8-byte result.  The call
// always waits, asynchronous mode or not, because the value is returned.
template<class F> uint64_t blockValue( vvb_ctx* ctx, int* err, const char* readback, F&& body )
{
  uint64_t result = 0;
  unsigned long long* dOut = nullptr;
  int rc = body( dOut );
  if( !rc )
  {
    cudaError_t e = cudaMemcpyAsync( &result, dOut, 8, cudaMemcpyDeviceToHost, ctx->stream );
    if( e == cudaSuccess ) e = cudaStreamSynchronize( ctx->stream );
    if( e != cudaSuccess ) rc = fail( ctx, VVB_ERR_CUDA, readback, e );
  }
  if( err ) *err = rc;
  return result;
}

// QpParam (Quant.cpp:99-113): the QP with the bit-depth offset, clipped
int baseQp( const vvb_tu_par* par ) { return std::max( 0, std::min( 63 + 6 * ( par->bit_depth - 8 ), par->qp + 6 * ( par->bit_depth - 8 ) ) ); }

// scan position -> raster index inside the scanned region of a (1 << lw) x (1 << lh) TU, in scan tables laid out by buildScanTables
const int32_t* scanOrder( const int32_t* tables, int lw, int lh ) { return tables + 25 * 1024 + ( ( lw - 2 ) * 5 + ( lh - 2 ) ) * 1024; }

bool validPlane( const vvb_ctx* ctx, int id ) { return id >= 0 && id < VVB_MAX_PLANES - 2 && ctx->planes.p[id].origin != nullptr; }

// shape domain of the reference's distortion table: width a power of two (index = base + log2 w, RdCost.cpp:176-184)
int checkDistShape( vvb_ctx* ctx, int fam, int w, int h, int subShift )
{
  if( fam < 0 || fam > 4 ) return fail( ctx, VVB_ERR_ARG, "unknown dfunc" );
  if( !isPow2( w ) || w > 128 || h < 1 || h > 128 ) return fail( ctx, VVB_ERR_UNSUPPORTED, "block shape outside the reference's DFunc domain (w power of two <= 128, h <= 128)" );
  if( fam == FAM_SAD && subShift && ( h & ( ( 1 << subShift ) - 1 ) ) ) return fail( ctx, VVB_ERR_UNSUPPORTED, "subShift needs an even height" );
  if( fam >= FAM_HAD && ( w < 2 || ( h & 1 ) ) ) return fail( ctx, VVB_ERR_UNSUPPORTED, "Hadamard needs even dimensions (RdCost.cpp:1933 THROW)" );
  if( fam == FAM_HAD_2SAD && ( w < 4 || ( h & 3 ) ) ) return fail( ctx, VVB_ERR_UNSUPPORTED, "HAD_2SAD needs w >= 4 and h % 4 == 0 (RdCost.cpp:1783-1784)" );
  if( fam == FAM_SSE && w < 2 ) return fail( ctx, VVB_ERR_UNSUPPORTED, "SSE of width 1 is routed to the scalar xGetSSE by the reference (RdCost.cpp:275)" );
  return VVB_OK;
}

int makeMePar( vvb_ctx* ctx, const vvb_me_par* in, MePar& out )
{
  if( !in ) return fail( ctx, VVB_ERR_ARG, "null me_par" );
  out.costScale = in->cost_scale; out.imvShift = in->imv_shift; out.subShift = in->sub_shift; out.orderBits = 0;
  const double motionLambda = std::sqrt( in->lambda );                 // RdCost.cpp:77
  for( int b = 0; b < VVB_MVCOST_ENTRIES; b++ )
  {
    const uint64_t c = (uint64_t)( motionLambda * (uint32_t) b );       // RdCost.h:181 Distortion( m_motionLambda * b )
    if( c > 0xffffffffull ) return fail( ctx, VVB_ERR_UNSUPPORTED, "lambda too large for the 32-bit MV cost table" );
    out.tab.cost[b] = (uint32_t) c;
  }
  return VVB_OK;
}

void buildScanTables( std::vector<int32_t>& inv )
{
  // grouped 4x4 up-right diagonal scan (Rom.cpp:1098-1136, 1236-1284); inv[shape][y*regionW + x] = scan position
  inv.assign( 2 * 25 * 1024, 0 );                 // second half: scan position -> raster index inside the scanned region (sign-bit hiding walks groups in scan order)
  auto diag = []( int bw, int bh, std::vector<int>& xs, std::vector<int>& ys )
  {
    xs.resize( bw * bh ); ys.resize( bw * bh );
    int line = 0, col = 0;
    for( int i = 0; i < bw * bh; i++ )
    {
      xs[i] = col; ys[i] = line;
      if( col == bw - 1 || line == 0 ) { line += col + 1; col = 0; if( line >= bh ) { col += line - ( bh - 1 ); line = bh - 1; } }
      else { col++; line--; }
    }
  };
  std::vector<int> cx, cy, gx, gy;
  diag( 4, 4, cx, cy );
  for( int lw = 2; lw <= 6; lw++ )
    for( int lh = 2; lh <= 6; lh++ )
    {
      const int rw = std::min( 32, 1 << lw ), rh = std::min( 32, 1 << lh );
      diag( rw >> 2, rh >> 2, gx, gy );
      int32_t* t = inv.data() + ( ( lw - 2 ) * 5 + ( lh - 2 ) ) * 1024;
      for( int g = 0; g < ( rw >> 2 ) * ( rh >> 2 ); g++ )
        for( int c = 0; c < 16; c++ )
        {
          t[( gy[g] * 4 + cy[c] ) * rw + gx[g] * 4 + cx[c]] = g * 16 + c;
          t[25 * 1024 + g * 16 + c] = ( gy[g] * 4 + cy[c] ) * rw + gx[g] * 4 + cx[c];
        }
    }
}

// single-block helper kernels (FpDistFunc-shaped calls)
__global__ void sad_mask_kernel( const int16_t* org, int so, const int16_t* cur, int sc, int w, int h, const int16_t* mask, int maskStride, int stepX, int maskStride2,
                                 int subShift, unsigned long long* out )
{
  // RdCost.cpp:2062-2093: mask pointer walks stepX per sample, then maskStride*step + maskStride2 per visited row
  const int step = 1 << subShift;
  unsigned long long acc = 0;
  const int rows = h >> subShift;
  for( int i = threadIdx.x; i < rows * w; i += blockDim.x )
  {
    const int r = i / w, x = i - r * w, y = r * step;
    const long long mpos = (long long) r * ( (long long) w * stepX + (long long) maskStride * step + maskStride2 ) + (long long) x * stepX;
    acc += (unsigned long long)( abs( (int) org[y * so + x] - (int) cur[y * sc + x] ) * (int) mask[mpos] );
  }
  for( int m = 16; m > 0; m >>= 1 ) acc += __shfl_xor_sync( 0xffffffffu, acc, m );
  if( threadIdx.x == 0 ) *out = acc << subShift;
}

__global__ void sad_x5_kernel( const int16_t* org, int so, const int16_t* cur, int sc, int w, int h, int subShift, unsigned long long* out5 )
{
  // RdCost.cpp:1984-2034: position i compares org+i with cur-i, each SAD >> 1
  const int i5 = blockIdx.x;
  const uint32_t s = group_sad<32>( org + i5, so, cur - i5, sc, w, h, subShift, threadIdx.x );
  if( threadIdx.x == 0 ) out5[i5] = s >> 1;
}

__global__ void fix_wsse_kernel( const int16_t* org, int so, const int16_t* cur, int sc, int w, int h, uint32_t weight, unsigned long long* out )
{
  unsigned long long acc = 0;
  for( int i = threadIdx.x; i < w * h; i += blockDim.x )
  {
    const int y = i / w, x = i - y * w;
    const int d = (int) org[y * so + x] - (int) cur[y * sc + x];
    acc += (unsigned long long)(int)( ( (long long) weight * ( d * d ) + ( 1 << 15 ) ) >> 16 );     // RdCost.cpp:1942-1946
  }
  for( int m = 16; m > 0; m >>= 1 ) acc += __shfl_xor_sync( 0xffffffffu, acc, m );
  if( threadIdx.x == 0 ) *out = acc;
}

// Issue-rate probe for the packed-SAD instruction mix (2 x VIMNMX.S16x2 + 2 x IDP.2A per pel pair) on register operands:
// the measured ceiling the dense search kernel is compared against (bench.py "alu" roofline).
template<int MODE>
__global__ void __launch_bounds__( 256 ) alu_probe_kernel( int iters, uint32_t seed, uint32_t* out )
{
  uint32_t a[8], b[8]; int acc[8];
#pragma unroll
  for( int i = 0; i < 8; i++ ) { a[i] = seed * ( 2654435761u + i ) + threadIdx.x; b[i] = a[i] ^ ( 0x01230123u * ( i + 1 ) ); acc[i] = 0; }
  for( int it = 0; it < iters; it++ )
  {
#pragma unroll
    for( int i = 0; i < 8; i++ )
    {
      // exactly the 4 instructions of one packed SAD step; feeding max/min back keeps the loop body from being hoisted
      if( MODE == 0 )      // list / pattern kernels: |a-b| = max - min
      {
        const uint32_t mx = __vmaxs2( a[i], b[i] ), mn = __vmins2( a[i], b[i] );
        acc[i] = __dp2a_lo( (int) mx, 0x00000101, acc[i] );
        acc[i] = __dp2a_lo( (int) mn, (int) 0x0000ffffu, acc[i] );
        a[i] = mx; b[i] = mn;
      }
      else                 // dense search: only sum min(a,b) is per-candidate work
      {
        const uint32_t mn = __vmins2( a[i], b[i] );
        acc[i] = __dp2a_lo( (int) mn, (int) 0x0000ffffu, acc[i] );
        a[i] = b[i]; b[i] = mn;
      }
    }
  }
  int s = 0;
#pragma unroll
  for( int i = 0; i < 8; i++ ) s += acc[i];
  if( s == 0x7fffffff ) out[0] = (uint32_t) s;      // keeps the loop alive
}

// a kernel's dynamic shared memory limit, set in vvb_create
struct SmemLimit { const void* fn; int bytes; };
template<class K> SmemLimit smemLimit( K* kernel, int bytes ) { return { (const void*) kernel, bytes }; }

// a compact device copy of a strided host block, rows of pad + w samples: blockPels samples, filled by uploadBlock (padBefore of the pad samples come
// from the left of the block)
size_t blockPels( int w, int h, int pad = 0 ) { return (size_t)( w + pad ) * h + 32; }
int uploadBlock( vvb_ctx* ctx, int16_t* d, const int16_t* host, int stride, int w, int h, int padBefore = 0, int padAfter = 0 )
{
  const int rowPels = w + padBefore + padAfter;
  CU( cudaMemcpy2DAsync( d, (size_t) rowPels * 2, host - padBefore, (size_t) stride * 2, (size_t) rowPels * 2, h, cudaMemcpyHostToDevice, ctx->stream ) );
  return VVB_OK;
}

} // namespace

extern "C" {

int vvb_create( vvb_ctx** out, int device )
{
  if( !out ) return VVB_ERR_ARG;
  *out = nullptr;
  int count = 0;
  cudaError_t e = cudaGetDeviceCount( &count );
  if( e != cudaSuccess || count <= 0 || device < 0 || device >= count ) return VVB_ERR_CUDA;
  vvb_ctx* ctx = new( std::nothrow ) vvb_ctx;
  if( !ctx ) return VVB_ERR_NOMEM;
  ctx->device = device;
  cudaDeviceProp prop;
  if( cudaSetDevice( device ) != cudaSuccess || cudaGetDeviceProperties( &prop, device ) != cudaSuccess ) { delete ctx; return VVB_ERR_CUDA; }
  ctx->numSMs = prop.multiProcessorCount;
  if( cudaStreamCreateWithFlags( &ctx->stream, cudaStreamNonBlocking ) != cudaSuccess ) { delete ctx; return VVB_ERR_CUDA; }
  std::vector<int32_t> inv;
  buildScanTables( inv );
  if( cudaMalloc( &ctx->d_trTable, VVC_TR_TABLE_SIZE ) != cudaSuccess || cudaMalloc( &ctx->d_scan, inv.size() * sizeof( int32_t ) ) != cudaSuccess ||
      cudaMalloc( &ctx->d_lfnst, VVC_LFNST_BYTES ) != cudaSuccess ||
      cudaMemcpy( ctx->d_trTable, vvc_tr_table_host, VVC_TR_TABLE_SIZE, cudaMemcpyHostToDevice ) != cudaSuccess ||
      cudaMemcpy( ctx->d_scan, inv.data(), inv.size() * sizeof( int32_t ), cudaMemcpyHostToDevice ) != cudaSuccess ||
      cudaMemcpy( ctx->d_lfnst, vvc_lfnst_words, VVC_LFNST_BYTES, cudaMemcpyHostToDevice ) != cudaSuccess )
  {
    vvb_destroy( ctx );
    return VVB_ERR_CUDA;
  }
  // dynamic shared memory limits above the 48 KB default
#define VVB_FWD_TC_SMEM( Nv ) smemLimit( fwd_trquant_tc2_kernel<Nv, 0>, Tc2Shape<Nv>::SMEM ), smemLimit( fwd_trquant_tc2_kernel<Nv, 1>, Tc2Shape<Nv>::SMEM ), \
                              smemLimit( fwd_trquant_tc2_kernel<Nv, 2>, Tc2Shape<Nv>::SMEM )
#define VVB_ITC_SMEM( Nv ) smemLimit( inv_trquant_tc_kernel<Nv, false>, ItcShape<Nv>::SMEM ), smemLimit( inv_trquant_tc_kernel<Nv, true>, ItcShape<Nv>::SMEM )
#define VVB_RING_SMEM( W ) smemLimit( had8_ring_kernel<true, W, 2>, 220 * 1024 ), smemLimit( had8_ring_kernel<false, W, 2>, 220 * 1024 ), \
                           smemLimit( had8_ring_kernel<true, W, 8>, 220 * 1024 ), smemLimit( had8_ring_kernel<false, W, 8>, 220 * 1024 )
  const SmemLimit smemLimits[] = {
    smemLimit( sad_search_kernel<false, false>, 220 * 1024 ), smemLimit( sad_search_kernel<true, false>, 220 * 1024 ),
    smemLimit( sad_search_kernel<false, true>, 220 * 1024 ), smemLimit( sad_search_kernel<true, true>, 220 * 1024 ),
    smemLimit( sad_search_kernel<false, true, true>, 220 * 1024 ), smemLimit( sad_search_kernel<true, true, true>, 220 * 1024 ),
    smemLimit( sad_pyramid8_kernel<2>, 227 * 1024 ), smemLimit( sad_pyramid8_kernel<3>, 227 * 1024 ), smemLimit( sad_pyramid8_kernel<4>, 227 * 1024 ),
    smemLimit( affine_eq_batch_kernel<4>, 100 * 1024 ), smemLimit( affine_eq_batch_kernel<6>, 100 * 1024 ),
    VVB_RING_SMEM( 16 ), VVB_RING_SMEM( 32 ), VVB_RING_SMEM( 64 ),
    smemLimit( mctf_error_packed_kernel, 100 * 1024 ), smemLimit( mctf_grid_kernel, 200 * 1024 ), smemLimit( mctf_wave_kernel, 100 * 1024 ),
    smemLimit( mctf_int_grid_kernel, 100 * 1024 ), smemLimit( mctf_apply_kernel, 100 * 1024 ), smemLimit( frac_grid_kernel, 100 * 1024 ),
    smemLimit( frac_grid_generic_kernel, 100 * 1024 ),
    VVB_FWD_TC_SMEM( 8 ), VVB_FWD_TC_SMEM( 16 ), VVB_FWD_TC_SMEM( 32 ), VVB_FWD_TC_SMEM( 64 ), VVB_ITC_SMEM( 8 ), VVB_ITC_SMEM( 16 ), VVB_ITC_SMEM( 32 ), VVB_ITC_SMEM( 64 ) };
#undef VVB_FWD_TC_SMEM
#undef VVB_ITC_SMEM
#undef VVB_RING_SMEM
  for( const auto& s : smemLimits ) cudaFuncSetAttribute( s.fn, cudaFuncAttributeMaxDynamicSharedMemorySize, s.bytes );
  {
    // cuTensorMapEncodeTiled through the runtime's driver entry point lookup (no link-time dependency on libcuda)
    void* fn = nullptr; cudaDriverEntryPointQueryResult qres;
    if( cudaGetDriverEntryPoint( "cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &qres ) == cudaSuccess && qres == cudaDriverEntryPointSuccess ) ctx->tmaEncode = fn;
    cudaGetLastError();
  }
  *out = ctx;
  return VVB_OK;
}

void vvb_destroy( vvb_ctx* ctx )
{
  if( !ctx ) return;
  cudaSetDevice( ctx->device );
  if( ctx->stream ) cudaStreamSynchronize( ctx->stream );
  for( int i = 0; i < VVB_MAX_PLANES; i++ ) if( ctx->owned[i] ) cudaFree( ctx->owned[i] );
  for( void* s : ctx->d_scratch ) if( s ) cudaFree( s );
  if( ctx->d_trTable ) cudaFree( ctx->d_trTable );
  for( void*& im : ctx->tc2Image ) if( im ) { cudaFree( im ); im = nullptr; }
  for( void*& im : ctx->itcImage ) if( im ) { cudaFree( im ); im = nullptr; }
  if( ctx->d_scan ) cudaFree( ctx->d_scan );
  if( ctx->d_lfnst ) cudaFree( ctx->d_lfnst );
  if( ctx->d_mask ) cudaFree( ctx->d_mask );
  if( ctx->d_dqScan ) cudaFree( ctx->d_dqScan );
  if( ctx->d_dqNb ) cudaFree( ctx->d_dqNb );
  delete[] static_cast<vvbdq::DqShapeTables*>( ctx->dqShapes );
  if( ctx->stream ) cudaStreamDestroy( ctx->stream );
  delete ctx;
}

const char* vvb_last_error( const vvb_ctx* ctx ) { return ctx ? ctx->err.c_str() : "null context"; }

int vvb_synchronize( vvb_ctx* ctx )
{
  if( !ctx ) return VVB_ERR_ARG;
  CU( cudaStreamSynchronize( ctx->stream ) );
  return VVB_OK;
}

void* vvb_stream( vvb_ctx* ctx ) { return ctx ? (void*) ctx->stream : nullptr; }

int vvb_set_async( vvb_ctx* ctx, int enable ) { if( !ctx ) return VVB_ERR_ARG; ctx->async = enable != 0; return VVB_OK; }

int vvb_launch_count( const vvb_ctx* ctx, uint64_t* k ) { if( !ctx || !k ) return VVB_ERR_ARG; *k = ctx->launches; return VVB_OK; }

#ifdef VVB_PYR_PHASES
// phase-timing build only (tools/pyr_phases.py): copies the pyramid kernel's per-level phase sums (3 levels x (PYR_NPHASE spans in ns, root count)) out after
// the context's stream has finished, then clears them
int vvb_pyr_phases_read( vvb_ctx* ctx, unsigned long long* out )
{
  if( !ctx || !out ) return VVB_ERR_ARG;
  CU( cudaSetDevice( ctx->device ) );
  CU( cudaStreamSynchronize( ctx->stream ) );
  CU( cudaMemcpyFromSymbol( out, g_pyrPhaseNs, sizeof( g_pyrPhaseNs ) ) );
  static const unsigned long long zero[3][PYR_NPHASE + 1] = {};
  CU( cudaMemcpyToSymbol( g_pyrPhaseNs, zero, sizeof( zero ) ) );
  return VVB_OK;
}
#endif

// window staging of the dense search: 1 = TMA (cp.async.bulk.tensor.2d, default when available), 0 = load/store loop
int vvb_set_tma_staging( vvb_ctx* ctx, int enable )
{
  if( !ctx ) return VVB_ERR_ARG;
  ctx->useTma = enable;
  return VVB_OK;
}

// SAD pyramid engine: 1 (default) = all levels inside one CTA per root block (pyramid_kernels.cuh) where it applies, 0 = per-quad kernel + table sums
int vvb_set_pyramid_engine( vvb_ctx* ctx, int engine )
{
  if( !ctx ) return VVB_ERR_ARG;
  ctx->pyramidEngine = engine;
  return VVB_OK;
}

// transform engine (include/vvenc_b200.h): non-zero (default) = the raw-byte wgmma engines where they apply, 0 = IDP.2A CUDA-core kernels for every shape
int vvb_set_tensor_transform( vvb_ctx* ctx, int enable )
{
  if( !ctx ) return VVB_ERR_ARG;
  ctx->tensorTransform = enable != 0;
  return VVB_OK;
}

// launches the ALU probe: grid_ctas CTAs x 256 threads x iters iterations x 8 packed SADs (16 pel differences) each
int vvb_alu_probe_dev( vvb_ctx* ctx, int gridCtas, int iters, int mode )
{
  if( !ctx || gridCtas < 1 || iters < 1 ) return fail( ctx, VVB_ERR_ARG, "bad arguments" );
  CU( cudaSetDevice( ctx->device ) );
  void* d; int rc;
  if( ( rc = scratch( ctx, ScratchArena::Work, 64, &d ) ) ) return rc;
  if( mode == 0 ) alu_probe_kernel<0><<<gridCtas, 256, 0, ctx->stream>>>( iters, 12345u, (uint32_t*) d );
  else            alu_probe_kernel<1><<<gridCtas, 256, 0, ctx->stream>>>( iters, 12345u, (uint32_t*) d );
  CHECK_LAUNCH( "alu_probe_kernel" );
  return VVB_OK;
}

// ---- planes --------------------------------------------------------------------------------------------------
int vvb_plane_free( vvb_ctx* ctx, int id )
{
  if( !ctx || id < 0 || id >= VVB_MAX_PLANES - 2 ) return fail( ctx, VVB_ERR_ARG, "plane id out of range" );
  if( ctx->owned[id] ) { cudaStreamSynchronize( ctx->stream ); cudaFree( ctx->owned[id] ); ctx->owned[id] = nullptr; ctx->ownedBytes[id] = 0; }
  ctx->planes.p[id] = Plane{};
  return VVB_OK;
}

int vvb_plane_upload( vvb_ctx* ctx, int id, const int16_t* origin, int stride, int width, int height, int margin, int bitDepth )
{
  if( !ctx || !origin || id < 0 || id >= VVB_MAX_PLANES - 2 || width <= 0 || height <= 0 || margin < 0 || stride < width + 2 * margin )
    return fail( ctx, VVB_ERR_ARG, "bad plane arguments" );
  CU( cudaSetDevice( ctx->device ) );
  const int dw = width + 2 * margin, dh = height + 2 * margin;
  const int dstride = ( dw + 7 ) & ~7;                                 // rows 16-byte aligned
  const size_t bytes = (size_t) dstride * dh * sizeof( int16_t ) + 256;
  void* d = ctx->owned[id];
  if( !d || ctx->ownedBytes[id] < bytes )                              // a new picture of the same geometry re-uses the allocation
  {
    vvb_plane_free( ctx, id );
    CU( cudaMalloc( &d, bytes ) );
    ctx->ownedBytes[id] = bytes;
  }
  const int16_t* src = origin - (ptrdiff_t) margin * stride - margin;
  CU( cudaMemcpy2DAsync( d, (size_t) dstride * 2, src, (size_t) stride * 2, (size_t) dw * 2, dh, cudaMemcpyHostToDevice, ctx->stream ) );
  ctx->owned[id] = d;
  Plane p; p.origin = reinterpret_cast<int16_t*>( d ) + (size_t) margin * dstride + margin; p.stride = dstride; p.width = width; p.height = height; p.margin = margin; p.bitDepth = bitDepth;
  ctx->planes.p[id] = p;
  CU( endCall( ctx ) );                          // the host buffer is only borrowed for the call
  return VVB_OK;
}

int vvb_plane_bind_dev( vvb_ctx* ctx, int id, const int16_t* devOrigin, int stride, int width, int height, int margin, int bitDepth )
{
  if( !ctx || !devOrigin || id < 0 || id >= VVB_MAX_PLANES - 2 ) return fail( ctx, VVB_ERR_ARG, "bad plane arguments" );
  vvb_plane_free( ctx, id );
  Plane p; p.origin = devOrigin; p.stride = stride; p.width = width; p.height = height; p.margin = margin; p.bitDepth = bitDepth;
  ctx->planes.p[id] = p;
  return VVB_OK;
}

// ---- pair list -------------------------------------------------------------------------------------------------
int vvb_dist_batch_dev( vvb_ctx* ctx, const vvb_cand* dCands, int n, uint64_t* dOut )
{
  if( !ctx || !dCands || !dOut || n < 0 ) return fail( ctx, VVB_ERR_ARG, "bad arguments" );
  if( n == 0 ) return VVB_OK;
  CU( cudaSetDevice( ctx->device ) );
  const int warpsPerCta = 8;
  const int grid = std::min( ( n + warpsPerCta - 1 ) / warpsPerCta, ctx->numSMs * 16 );
  dist_list_kernel<<<grid, warpsPerCta * 32, 0, ctx->stream>>>( ctx->planes, dCands, n, reinterpret_cast<unsigned long long*>( dOut ) );
  CHECK_LAUNCH( "dist_list_kernel" );
  return VVB_OK;
}

int vvb_dist_batch( vvb_ctx* ctx, const vvb_cand* cands, int n, uint64_t* out )
{
  if( !ctx || !cands || !out || n < 0 ) return fail( ctx, VVB_ERR_ARG, "bad arguments" );
  for( int i = 0; i < n; i++ )
  {
    const vvb_cand& c = cands[i];
    if( !validPlane( ctx, c.org_plane ) || !validPlane( ctx, c.cur_plane ) ) return fail( ctx, VVB_ERR_ARG, "candidate refers to an unknown plane" );
    int rc = checkDistShape( ctx, c.dfunc, c.w, c.h, c.sub_shift );
    if( rc ) return rc;
  }
  if( n == 0 ) return VVB_OK;
  const vvb_cand* dC; uint64_t* dO;
  return HostCall( ctx ).in( dC, cands, n ).out( dO, out, n ).run( [&] { return vvb_dist_batch_dev( ctx, dC, n, dO ); } );
}

uint64_t vvb_dist_block( vvb_ctx* ctx, int dfunc, const int16_t* org, int orgStride, const int16_t* cur, int curStride, int w, int h, int bitDepth, int subShift, int* err )
{
  return blockValue( ctx, err, "dist_block readback", [&]( unsigned long long*& dOut )
  {
    if( !ctx || !org || !cur ) return fail( ctx, VVB_ERR_ARG, "null pointer" );
    int rc = checkDistShape( ctx, dfunc, w, h, subShift );
    if( rc ) return rc;
    if( cudaSetDevice( ctx->device ) != cudaSuccess ) return fail( ctx, VVB_ERR_CUDA, "cudaSetDevice" );
    int16_t *dO, *dC; vvb_cand* dCand;
    if( ( rc = carveArena( ctx, ScratchArena::Host, [&]( Layout& L ) { dO = L.take<int16_t>( blockPels( w, h ) ); dC = L.take<int16_t>( blockPels( w, h ) ); dCand = L.take<vvb_cand>( 1 ); dOut = L.take<unsigned long long>( 1 ); } ) ) ||
        ( rc = uploadBlock( ctx, dO, org, orgStride, w, h ) ) || ( rc = uploadBlock( ctx, dC, cur, curStride, w, h ) ) ) return rc;
    PlaneTable pt = ctx->planes;
    pt.p[VVB_MAX_PLANES - 2] = Plane{ dO, w, w, h, 0, bitDepth };
    pt.p[VVB_MAX_PLANES - 1] = Plane{ dC, w, w, h, 0, bitDepth };
    vvb_cand c{}; c.org_plane = VVB_MAX_PLANES - 2; c.cur_plane = VVB_MAX_PLANES - 1; c.w = (uint16_t) w; c.h = (uint16_t) h; c.dfunc = (uint8_t) dfunc; c.sub_shift = (uint8_t) subShift;
    if( cudaMemcpyAsync( dCand, &c, sizeof( c ), cudaMemcpyHostToDevice, ctx->stream ) != cudaSuccess ) return fail( ctx, VVB_ERR_CUDA, "memcpy cand" );
    dist_list_kernel<<<1, 32, 0, ctx->stream>>>( pt, dCand, 1, dOut );
    CHECK_LAUNCH( "dist_list_kernel" );
    return VVB_OK;
  } );
}

uint64_t vvb_sad_mask_block( vvb_ctx* ctx, const int16_t* org, int orgStride, const int16_t* cur, int curStride, int w, int h,
                             const int16_t* mask, int maskStride, int stepX, int maskStride2, int subShift, int* err )
{
  return blockValue( ctx, err, "sad_mask readback", [&]( unsigned long long*& dOut )
  {
    if( !ctx || !org || !cur || !mask || ( stepX != 1 && stepX != -1 ) ) return fail( ctx, VVB_ERR_ARG, "bad arguments" );
    if( w < 1 || h < 1 || w > 128 || h > 128 || ( h & ( ( 1 << subShift ) - 1 ) ) ) return fail( ctx, VVB_ERR_UNSUPPORTED, "bad mask-SAD shape" );
    cudaSetDevice( ctx->device );
    // the mask walk covers, per visited row r: start + r*rowAdv + x*stepX ; gather exactly those samples into a compact [rows][w] mask
    const int step = 1 << subShift, rows = h >> subShift;
    std::vector<int16_t> m( (size_t) rows * w );
    for( int r = 0; r < rows; r++ )
      for( int x = 0; x < w; x++ )
        m[(size_t) r * w + x] = mask[(ptrdiff_t) r * ( (ptrdiff_t) w * stepX + (ptrdiff_t) maskStride * step + maskStride2 ) + (ptrdiff_t) x * stepX];
    int16_t *dO, *dC, *dM; int rc;
    if( ( rc = carveArena( ctx, ScratchArena::Host, [&]( Layout& L ) { dO = L.take<int16_t>( blockPels( w, h ) ); dC = L.take<int16_t>( blockPels( w, h ) ); dM = L.take<int16_t>( m.size() ); dOut = L.take<unsigned long long>( 1 ); } ) ) ||
        ( rc = uploadBlock( ctx, dO, org, orgStride, w, h ) ) || ( rc = uploadBlock( ctx, dC, cur, curStride, w, h ) ) ) return rc;
    if( cudaMemcpyAsync( dM, m.data(), m.size() * 2, cudaMemcpyHostToDevice, ctx->stream ) != cudaSuccess ) return fail( ctx, VVB_ERR_CUDA, "mask upload" );
    // compact mask: stepX = +1, row advance = w  -> maskStride*step + maskStride2 = 0
    sad_mask_kernel<<<1, 32, 0, ctx->stream>>>( dO, w, dC, w, w, h, dM, 0, 1, 0, subShift, dOut );
    CHECK_LAUNCH( "sad_mask_kernel" );
    return VVB_OK;
  } );
}

int vvb_sad_x5_block( vvb_ctx* ctx, const int16_t* org, int orgStride, const int16_t* cur, int curStride, int w, int h, int subShift, int calcCentre, uint64_t cost5[5] )
{
  if( !ctx || !org || !cur || !cost5 ) return fail( ctx, VVB_ERR_ARG, "bad arguments" );
  if( ( w != 8 && w != 16 ) || h < 1 || h > 128 || ( h & ( ( 1 << subShift ) - 1 ) ) ) return fail( ctx, VVB_ERR_UNSUPPORTED, "SADX5 is defined for widths 8 and 16 (RdCost.cpp:131-132)" );
  CU( cudaSetDevice( ctx->device ) );
  int16_t *dO, *dC; unsigned long long* dOut; int rc;
  if( ( rc = carveArena( ctx, ScratchArena::Host, [&]( Layout& L ) { dO = L.take<int16_t>( blockPels( w, h, 4 ) ); dC = L.take<int16_t>( blockPels( w, h, 4 ) ); dOut = L.take<unsigned long long>( 5 ); } ) ) ||
      ( rc = uploadBlock( ctx, dO, org, orgStride, w, h, 0, 4 ) ) || ( rc = uploadBlock( ctx, dC, cur, curStride, w, h, 4, 0 ) ) ) return rc;
  sad_x5_kernel<<<5, 32, 0, ctx->stream>>>( dO, w + 4, dC + 4, w + 4, w, h, subShift, dOut );
  CHECK_LAUNCH( "sad_x5_kernel" );
  uint64_t tmp[5];
  CU( cudaMemcpyAsync( tmp, dOut, 40, cudaMemcpyDeviceToHost, ctx->stream ) );
  CU( cudaStreamSynchronize( ctx->stream ) );         // tmp is consumed right below: always wait, asynchronous mode or not
  for( int i = 0; i < 5; i++ ) if( i != 2 || calcCentre ) cost5[i] = tmp[i];
  return VVB_OK;
}

uint64_t vvb_fix_wsse_block( vvb_ctx* ctx, const int16_t* org, int orgStride, const int16_t* cur, int curStride, int w, int h, uint32_t weight, int* err )
{
  return blockValue( ctx, err, "fix_wsse readback", [&]( unsigned long long*& dOut )
  {
    if( !ctx || !org || !cur ) return fail( ctx, VVB_ERR_ARG, "null pointer" );
    if( w < 1 || h < 1 || w > 128 || h > 128 || ( ( w & 1 ) && w != 1 ) ) return fail( ctx, VVB_ERR_UNSUPPORTED, "width must be even or 1 (RdCost.cpp:1966)" );
    cudaSetDevice( ctx->device );
    int16_t *dO, *dC; int rc;
    if( ( rc = carveArena( ctx, ScratchArena::Host, [&]( Layout& L ) { dO = L.take<int16_t>( blockPels( w, h ) ); dC = L.take<int16_t>( blockPels( w, h ) ); dOut = L.take<unsigned long long>( 1 ); } ) ) ||
        ( rc = uploadBlock( ctx, dO, org, orgStride, w, h ) ) || ( rc = uploadBlock( ctx, dC, cur, curStride, w, h ) ) ) return rc;
    fix_wsse_kernel<<<1, 32, 0, ctx->stream>>>( dO, w, dC, w, w, h, weight, dOut );
    CHECK_LAUNCH( "fix_wsse_kernel" );
    return VVB_OK;
  } );
}

// ---- descriptor-list forms of the mask SAD, the five-position SAD and the weighted SSE -----------------------------------------------------------------------------
namespace {
int checkCandPlanes( vvb_ctx* ctx, const vvb_cand* c, int n )      // host lists only
{
  for( int i = 0; i < n; i++ )
    if( !validPlane( ctx, c[i].org_plane ) || !validPlane( ctx, c[i].cur_plane ) || c[i].w < 1 || c[i].h < 1 || c[i].w > 128 || c[i].h > 128 ) return fail( ctx, VVB_ERR_ARG, "bad descriptor" );
  return VVB_OK;
}
}

int vvb_mask_upload( vvb_ctx* ctx, const int16_t* mask, int count )
{
  if( !ctx || !mask || count < 1 ) return fail( ctx, VVB_ERR_ARG, "bad arguments" );
  CU( cudaSetDevice( ctx->device ) );
  CU( cudaStreamSynchronize( ctx->stream ) );
  if( ctx->d_mask ) { cudaFree( ctx->d_mask ); ctx->d_mask = nullptr; ctx->maskCount = 0; }
  CU( cudaMalloc( &ctx->d_mask, (size_t) count * 2 ) );
  CU( cudaMemcpy( ctx->d_mask, mask, (size_t) count * 2, cudaMemcpyHostToDevice ) );
  ctx->maskCount = count;
  return VVB_OK;
}

int vvb_sad_mask_batch_dev( vvb_ctx* ctx, const vvb_mask_cand* dCands, int n, uint64_t* dOut )
{
  if( !ctx || !dCands || !dOut || n < 0 ) return fail( ctx, VVB_ERR_ARG, "bad arguments" );
  if( !ctx->d_mask ) return fail( ctx, VVB_ERR_ARG, "no mask table (vvb_mask_upload)" );
  if( n == 0 ) return VVB_OK;
  CU( cudaSetDevice( ctx->device ) );
  sad_mask_batch_kernel<<<( n + VVB_BATCH_WARPS - 1 ) / VVB_BATCH_WARPS, VVB_BATCH_WARPS * 32, 0, ctx->stream>>>( ctx->planes, dCands, n, ctx->d_mask, (unsigned long long*) dOut );
  CHECK_LAUNCH( "sad_mask_batch_kernel" );
  return VVB_OK;
}

int vvb_sad_mask_batch( vvb_ctx* ctx, const vvb_mask_cand* cands, int n, uint64_t* out )
{
  if( !ctx || !cands || !out || n < 0 ) return fail( ctx, VVB_ERR_ARG, "bad arguments" );
  if( n == 0 ) return VVB_OK;
  for( int i = 0; i < n; i++ )
  {
    const vvb_mask_cand& d = cands[i];
    int rc = checkCandPlanes( ctx, &d.c, 1 );
    if( rc ) return rc;
    if( ( d.step_x != 1 && d.step_x != -1 ) || ( d.c.h & ( ( 1 << d.c.sub_shift ) - 1 ) ) ) return fail( ctx, VVB_ERR_ARG, "bad mask descriptor" );
    // every mask sample the walk touches must lie inside the uploaded table
    const long long rows = d.c.h >> d.c.sub_shift, rowAdv = (long long) d.c.w * d.step_x + (long long) d.mask_stride * ( 1 << d.c.sub_shift ) + d.mask_stride2;
    const long long a = d.mask_offset, b = a + ( rows - 1 ) * rowAdv, lo = std::min( a, b ) + ( d.step_x < 0 ? -( d.c.w - 1 ) : 0 ), hi = std::max( a, b ) + ( d.step_x > 0 ? d.c.w - 1 : 0 );
    if( lo < 0 || hi >= ctx->maskCount ) return fail( ctx, VVB_ERR_ARG, "mask walk leaves the uploaded table" );
  }
  const vvb_mask_cand* dC; uint64_t* dO;
  return HostCall( ctx ).in( dC, cands, n ).out( dO, out, n ).run( [&] { return vvb_sad_mask_batch_dev( ctx, dC, n, dO ); } );
}

int vvb_sad_x5_batch_dev( vvb_ctx* ctx, const vvb_cand* dCands, int n, uint64_t* dOut5 )
{
  if( !ctx || !dCands || !dOut5 || n < 0 ) return fail( ctx, VVB_ERR_ARG, "bad arguments" );
  if( n == 0 ) return VVB_OK;
  CU( cudaSetDevice( ctx->device ) );
  sad_x5_batch_kernel<<<( n + VVB_BATCH_WARPS - 1 ) / VVB_BATCH_WARPS, VVB_BATCH_WARPS * 32, 0, ctx->stream>>>( ctx->planes, dCands, n, (unsigned long long*) dOut5 );
  CHECK_LAUNCH( "sad_x5_batch_kernel" );
  return VVB_OK;
}

int vvb_sad_x5_batch( vvb_ctx* ctx, const vvb_cand* cands, int n, uint64_t* out5 )
{
  if( !ctx || !cands || !out5 || n < 0 ) return fail( ctx, VVB_ERR_ARG, "bad arguments" );
  if( n == 0 ) return VVB_OK;
  int rc = checkCandPlanes( ctx, cands, n );
  if( rc ) return rc;
  for( int i = 0; i < n; i++ )
    if( ( cands[i].w != 8 && cands[i].w != 16 ) || ( cands[i].h & ( ( 1 << cands[i].sub_shift ) - 1 ) ) ) return fail( ctx, VVB_ERR_UNSUPPORTED, "SADX5 is defined for widths 8 and 16 (RdCost.cpp:131-132)" );
  const vvb_cand* dC; uint64_t* dO;
  return HostCall( ctx ).in( dC, cands, n ).out( dO, out5, (size_t) n * 5 ).run( [&] { return vvb_sad_x5_batch_dev( ctx, dC, n, dO ); } );
}

int vvb_fix_wsse_batch_dev( vvb_ctx* ctx, const vvb_cand* dCands, const uint32_t* dWeights, int n, uint64_t* dOut )
{
  if( !ctx || !dCands || !dWeights || !dOut || n < 0 ) return fail( ctx, VVB_ERR_ARG, "bad arguments" );
  if( n == 0 ) return VVB_OK;
  CU( cudaSetDevice( ctx->device ) );
  fix_wsse_batch_kernel<<<( n + VVB_BATCH_WARPS - 1 ) / VVB_BATCH_WARPS, VVB_BATCH_WARPS * 32, 0, ctx->stream>>>( ctx->planes, dCands, dWeights, n, (unsigned long long*) dOut );
  CHECK_LAUNCH( "fix_wsse_batch_kernel" );
  return VVB_OK;
}

int vvb_fix_wsse_batch( vvb_ctx* ctx, const vvb_cand* cands, const uint32_t* weights, int n, uint64_t* out )
{
  if( !ctx || !cands || !weights || !out || n < 0 ) return fail( ctx, VVB_ERR_ARG, "bad arguments" );
  if( n == 0 ) return VVB_OK;
  int rc = checkCandPlanes( ctx, cands, n );
  if( rc ) return rc;
  for( int i = 0; i < n; i++ ) if( ( cands[i].w & 1 ) && cands[i].w != 1 ) return fail( ctx, VVB_ERR_UNSUPPORTED, "width must be even or 1 (RdCost.cpp:1966)" );
  const vvb_cand* dC; const uint32_t* dW; uint64_t* dO;
  return HostCall( ctx ).in( dC, cands, n ).in( dW, weights, n ).out( dO, out, n ).run( [&] { return vvb_fix_wsse_batch_dev( ctx, dC, dW, n, dO ); } );
}

// _dev callers state whether every block x position in their (device-resident) lists is a multiple of 8 pels; only then the
// 16-byte streaming kernels are used (default: not assumed).
int vvb_pool_hint( vvb_ctx* ctx, int blocksXAlignedTo8 )
{
  if( !ctx ) return VVB_ERR_ARG;
  ctx->poolBlocksAligned = blocksXAlignedTo8 != 0;
  return VVB_OK;
}

// ---- candidate pool ----------------------------------------------------------------------------------------------
int vvb_dist_pool_dev( vvb_ctx* ctx, int dfunc, int orgPlane, const vvb_pos* dBlocks, int nBlocks, int w, int h, int K, const int16_t* dPool, int subShift, uint32_t* dOut )
{
  if( !ctx || !dBlocks || !dPool || !dOut || nBlocks < 0 || K < 1 ) return fail( ctx, VVB_ERR_ARG, "bad arguments" );
  if( !validPlane( ctx, orgPlane ) ) return fail( ctx, VVB_ERR_ARG, "unknown plane" );
  int rc = checkDistShape( ctx, dfunc, w, h, subShift );
  if( rc ) return rc;
  if( nBlocks == 0 ) return VVB_OK;
  CU( cudaSetDevice( ctx->device ) );
  const long long total = (long long) nBlocks * K;
  const Plane& op = ctx->planes.p[orgPlane];
  // fast streaming paths need 16-byte aligned rows of the original (block x on a multiple of 8 is checked on the device side by
  // construction of the batch: callers with unaligned block positions get the generic kernel via the alignment test below)
  const bool planeAligned = ( ( (uintptr_t) op.origin & 15 ) == 0 ) && ( ( op.stride & 7 ) == 0 ) && ( ( (uintptr_t) dPool & 15 ) == 0 );
  const bool posAligned = ctx->poolBlocksAligned;     // set by the host entry point after inspecting the positions; _dev callers promise it via vvb_pool_hint
  bool launched = false;
  if( planeAligned && posAligned && w >= 8 && ( dfunc == FAM_SAD || dfunc == FAM_SSE ) )
  {
    const int rows = h >> ( dfunc == FAM_SAD ? subShift : 0 );
    const int chunks = rows * ( w >> 3 );
    int G = 4; while( G < 32 && chunks / G > 4 ) G <<= 1;             // aim at L = 4 chunks (64 bytes) per lane per pass
    const long long wantGroups = (long long) ctx->numSMs * 2048 / G * 2;
    int kSplit = 1; while( (long long) nBlocks * kSplit < wantGroups && kSplit < K ) kSplit <<= 1;
    if( kSplit > K ) kSplit = K;
    const long long threads = (long long) nBlocks * kSplit * G;
    const int grid = (int) std::min<long long>( ( threads + 255 ) / 256, (long long) ctx->numSMs * 32 );
    const int ss = dfunc == FAM_SAD ? subShift : 0;
    const bool single = chunks <= G * 4;
#define LAUNCH_SP2( GG, SS, SG ) sad_pool_stream_kernel<GG, 4, SS, SG><<<grid, 256, 0, ctx->stream>>>( op, dBlocks, nBlocks, w, h, K, kSplit, ss, dPool, dOut )
#define LAUNCH_SP( GG, SS ) do { if( single ) LAUNCH_SP2( GG, SS, true ); else LAUNCH_SP2( GG, SS, false ); } while( 0 )
    if( dfunc == FAM_SAD ) { switch( G ) { case 4: LAUNCH_SP( 4, false ); break; case 8: LAUNCH_SP( 8, false ); break; case 16: LAUNCH_SP( 16, false ); break; default: LAUNCH_SP( 32, false ); break; } }
    else                   { switch( G ) { case 4: LAUNCH_SP( 4, true ); break; case 8: LAUNCH_SP( 8, true ); break; case 16: LAUNCH_SP( 16, true ); break; default: LAUNCH_SP( 32, true ); break; } }
#undef LAUNCH_SP2
#undef LAUNCH_SP
    launched = true;
  }
  else if( planeAligned && posAligned && ( dfunc == FAM_HAD || dfunc == FAM_HAD_2SAD ) && ( w & 7 ) == 0 && isPow2( h ) && h >= 8 && w == h )
  {
    // tile dispatch lands on 8x8 (RdCost.cpp:1836-1905 with the rectangular 16x8 / 8x16 cases excluded above)
    const int T = ( w >> 3 ) * ( h >> 3 );
    const int LPC = T >= 32 ? 32 : T;
    const long long threads = total * LPC;
    const int grid = (int) std::min<long long>( ( threads + 127 ) / 128, (long long) ctx->numSMs * 32 );
    const int two = dfunc == FAM_HAD_2SAD ? 1 : 0;
#define LAUNCH_HP( LL ) had8_pool_stream_kernel<LL><<<grid, 128, 0, ctx->stream>>>( op, dBlocks, nBlocks, w, h, K, two, dPool, dOut )
    switch( LPC ) { case 1: LAUNCH_HP( 1 ); break; case 2: LAUNCH_HP( 2 ); break; case 4: LAUNCH_HP( 4 ); break; case 8: LAUNCH_HP( 8 ); break; case 16: LAUNCH_HP( 16 ); break; default: LAUNCH_HP( 32 ); break; }
#undef LAUNCH_HP
    launched = true;
  }
  if( !launched )
  {
    const int G = pick_group( dfunc, w, h );
    const long long threads = total * G;
    const int block = 256;
    const int grid = (int) std::min<long long>( ( threads + block - 1 ) / block, (long long) ctx->numSMs * 32 );
#define LAUNCH_POOL( GG ) dist_pool_kernel<GG><<<grid, block, 0, ctx->stream>>>( op, dBlocks, nBlocks, w, h, K, dfunc, subShift, dPool, dOut )
    switch( G ) { case 4: LAUNCH_POOL( 4 ); break; case 8: LAUNCH_POOL( 8 ); break; case 16: LAUNCH_POOL( 16 ); break; default: LAUNCH_POOL( 32 ); break; }
#undef LAUNCH_POOL
  }
  CHECK_LAUNCH( "dist_pool_kernel" );
  return VVB_OK;
}

int vvb_dist_pool( vvb_ctx* ctx, int dfunc, int orgPlane, const vvb_pos* blocks, int nBlocks, int w, int h, int K, const int16_t* pool, int subShift, uint32_t* out )
{
  if( !ctx || !blocks || !pool || !out || nBlocks < 0 || K < 1 ) return fail( ctx, VVB_ERR_ARG, "bad arguments" );
  if( nBlocks == 0 ) return VVB_OK;
  bool aligned = true;
  for( int i = 0; i < nBlocks && aligned; i++ ) aligned = ( blocks[i].x & 7 ) == 0;
  const size_t total = (size_t) nBlocks * K;
  const vvb_pos* dB; const int16_t* dP; uint32_t* dO;
  return HostCall( ctx ).in( dB, blocks, nBlocks ).in( dP, pool, total * w * h ).out( dO, out, total ).run( [&]
  {
    ctx->poolBlocksAligned = aligned;
    return vvb_dist_pool_dev( ctx, dfunc, orgPlane, dB, nBlocks, w, h, K, dP, subShift, dO );
  } );
}

// ---- motion search -----------------------------------------------------------------------------------------------
static int checkSearchShape( vvb_ctx* ctx, int orgPlane, int refPlane, int w, int h )
{
  if( !validPlane( ctx, orgPlane ) || !validPlane( ctx, refPlane ) ) return fail( ctx, VVB_ERR_ARG, "unknown plane" );
  if( !isPow2( w ) || !isPow2( h ) || w < 4 || h < 4 || w > 128 || h > 128 ) return fail( ctx, VVB_ERR_UNSUPPORTED, "search blocks are 4..128 powers of two" );
  return VVB_OK;
}

} // extern "C"

struct PyramidOut { const vvb_block* parents; vvb_best* best; uint32_t* tables; int stride; };

// host-known maximum window (nx, ny) variant used by both public entry points
static int sadSearchLaunch( vvb_ctx* ctx, int orgPlane, int refPlane, const vvb_block* dBlocks, int n, int w, int h, const vvb_me_par* par,
                            int maxNx, int maxNy, int quad, uint32_t* dTables, int tableStride, vvb_best* dBest, const PyramidOut* pyr = nullptr )
{
  int rc = checkSearchShape( ctx, orgPlane, refPlane, w, h );
  if( rc ) return rc;
  MePar mp;
  if( ( rc = makeMePar( ctx, par, mp ) ) ) return rc;
  if( mp.subShift && ( h & ( ( 1 << mp.subShift ) - 1 ) ) ) return fail( ctx, VVB_ERR_UNSUPPORTED, "subShift needs an even height" );
  if( maxNx * maxNy > 65536 ) return fail( ctx, VVB_ERR_UNSUPPORTED, "search window above 65536 positions" );
  if( n == 0 ) return VVB_OK;
  CU( cudaSetDevice( ctx->device ) );
  // z-order quads share one staged window; fall back to one block per CTA when the quad window does not fit
  int nb = ( quad && w >= 8 && n >= 4 ) ? 2 : 1;
  SearchSmem L = search_smem( w, h, maxNx, maxNy, nb, nb );
  if( nb == 2 && (size_t) L.total + 16 > 100 * 1024 && !pyr ) { nb = 1; L = search_smem( w, h, maxNx, maxNy, 1, 1 ); }
  if( pyr && nb != 2 ) return fail( ctx, VVB_ERR_UNSUPPORTED, "the SAD pyramid needs quads of blocks at least 8 wide" );
  const size_t smem = (size_t) L.total + 16;
  if( smem > 220 * 1024 ) return fail( ctx, VVB_ERR_UNSUPPORTED, "search window does not fit shared memory (reduce the range)" );
  // block size: the multiple of 32 in 64..384 that wastes the fewest thread slots on the (members x ny x strips) work items; ties -> larger
  const int items = ( pyr ? 1 : nb * nb ) * maxNy * ( ( maxNx + SS_STRIP - 1 ) / SS_STRIP );      // pyramid items cover all four members
  int bd = 256; double bestScore = -1.0;
  for( int cand = 64; cand <= ( pyr ? 256 : 384 ); cand += 32 )
  {
    const int rounds = ( items + cand - 1 ) / cand;
    const double eff = (double) items / ( (double) rounds * cand );
    const int ctasPerSM = (int) std::min<size_t>( std::min<size_t>( 32, ( 227 * 1024 ) / ( smem + 1024 ) ), 2048 / cand );
    const double occ = std::min( 1.0, ( ctasPerSM * cand / 32 ) / 24.0 );          // >= 24 resident warps hide the LDS latency
    const double score = eff * ( 0.5 + 0.5 * occ );
    if( score >= bestScore - 1e-9 ) { bestScore = std::max( bestScore, score ); bd = cand; }
  }
  const int grid = nb == 2 ? ( n + 3 ) / 4 : n;
  // TMA descriptor of the padded reference plane with a (ws x winH) box; needs a 16-byte aligned buffer start and row pitch
  CUtensorMap tmap; memset( &tmap, 0, sizeof( tmap ) );
  TmaInfo ti; memset( &ti, 0, sizeof( ti ) );
  const Plane& rp = ctx->planes.p[refPlane];
  if( ctx->tmaEncode && ( ctx->useTma == 1 || ( ctx->useTma == 2 && w <= 8 ) ) && L.ws <= 256 && L.winH <= 256 )
  {
    const int16_t* base = rp.origin - (ptrdiff_t) rp.margin * rp.stride - rp.margin;
    if( ( (uintptr_t) base & 15 ) == 0 && ( rp.stride & 7 ) == 0 )
    {
      typedef CUresult ( *EncodeFn )( CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*, const cuuint32_t*, const cuuint32_t*,
                                      CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill );
      const cuuint64_t gdim[2] = { (cuuint64_t) rp.stride, (cuuint64_t)( rp.height + 2 * rp.margin ) };
      const cuuint64_t gstr[1] = { (cuuint64_t) rp.stride * 2 };
      const cuuint32_t box[2]  = { (cuuint32_t) L.ws, (cuuint32_t) L.winH };
      const cuuint32_t estr[2] = { 1, 1 };
      const CUresult r = ( (EncodeFn) ctx->tmaEncode )( &tmap, CU_TENSOR_MAP_DATA_TYPE_UINT16, 2, (void*) base, gdim, gstr, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                                                       CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE );
      if( r == CUDA_SUCCESS ) { ti.enabled = 1; ti.nx = maxNx; ti.ny = maxNy; ti.quad = nb == 2 ? 1 : 0; ti.margin = rp.margin; }
    }
  }
#define LAUNCH_SS( T_, P_ ) LAUNCH_SS3( T_, P_, false )
#define LAUNCH_SS3( T_, P_, K_ ) sad_search_kernel<T_, P_, K_><<<grid, bd, smem, ctx->stream>>>( ctx->planes.p[orgPlane], rp, dBlocks, n, w, h, nb == 2 ? 1 : 0, mp, tmap, ti, dTables, tableStride, dBest, \
                                                                                    pyr ? pyr->parents : nullptr, pyr ? pyr->best : nullptr, pyr ? pyr->tables : nullptr, pyr ? pyr->stride : 0 )
  // 32-bit argmin keys in the pyramid base kernel when the largest possible parent cost (4 members' SAD + MV cost) leaves room for the raster order.
  // A pel difference is bounded by the wider of the two planes' bit depths.
  bool key32 = false;
  if( pyr )
  {
    int ob = 1; while( ( 1 << ob ) < maxNx * maxNy ) ob++;
    const int bd = std::max( ctx->planes.p[orgPlane].bitDepth, rp.bitDepth );
    const unsigned long long maxCost = 4ull * w * h * ( ( 1ull << bd ) - 1 ) + mp.tab.cost[VVB_MVCOST_ENTRIES - 1];
    if( ob <= 16 && maxCost < ( 1ull << ( 32 - ob ) ) - 1 ) { key32 = true; mp.orderBits = ob; }
  }
  if( pyr && key32 ) { if( ti.enabled ) LAUNCH_SS3( true, true, true ); else LAUNCH_SS3( false, true, true ); }
  else if( pyr ) { if( ti.enabled ) LAUNCH_SS( true, true ); else LAUNCH_SS( false, true ); }
  else      { if( ti.enabled ) LAUNCH_SS( true, false ); else LAUNCH_SS( false, false ); }
#undef LAUNCH_SS
#undef LAUNCH_SS3
  CHECK_LAUNCH( "sad_search_kernel" );
  return VVB_OK;
}

// In-CTA pyramid (pyramid_kernels.cuh): usable for 8x8 base blocks, no row sub-sampling, up to four levels, 32-bit keys at the 8x8 / 16x16 levels
template<int LV>
static int pyramidV2LaunchLevel( vvb_ctx* ctx, int orgPlane, int refPlane, const PyrLevels& lv, int rootFirst, int nRoots, int nx, int ny, const MePar& mp )
{
  const PyrSmem L = pyr_smem<LV>( nx, ny );
  const int NQ = ( 1 << ( 2 * ( LV - 1 ) ) ) / 4, maxT = pyr_max_threads<LV>();
  const int items = NQ * ( ( ny + 1 ) / 2 ) * ( nx >> 3 ) + NQ * ( nx & 7 ) * ( ( ny + 7 ) / 8 );      // the kernel's strip items + column items
  // CTA size: big grids take the largest CTA the instantiation allows (pyr_max_threads).  Small roots / ranges: fewest rounds of items per CTA (a CTA's rounds
  // run one after another, and a grid of fewer roots than SMs takes as long as one CTA), then fewest idle thread slots, ties -> more threads.
  int bd = maxT;
  if( items < 4 * maxT )
  {
    const int minRounds = ( items + maxT - 1 ) / maxT;
    double bestEff = -1.0;
    for( int cand = 128; cand <= maxT; cand += 32 )
    {
      const int rounds = ( items + cand - 1 ) / cand;
      const double eff = (double) items / ( (double) rounds * cand );
      if( rounds == minRounds && eff >= bestEff - 1e-9 ) { bestEff = std::max( bestEff, eff ); bd = cand; }
    }
  }
  static const int forced = []{ const char* e = getenv( "VVB_PYR_THREADS" ); return e ? atoi( e ) : 0; }();     // tuning aid: fixed CTA size
  if( forced >= 64 && forced <= maxT && ( forced & 31 ) == 0 ) bd = forced;
  // 64x64 roots fill an SM each: one CTA per SM walks a run of consecutive roots and carries the shared half of each window to its right neighbour.
  // Smaller roots share SMs and keep one CTA per root.
  const int runs = LV == 4 ? std::min( nRoots, ctx->numSMs ) : nRoots;
  sad_pyramid8_kernel<LV><<<runs, bd, (size_t) L.total, ctx->stream>>>( ctx->planes.p[orgPlane], ctx->planes.p[refPlane], lv, rootFirst, nRoots, nx, ny, mp, L, 1u, 8u );
  CHECK_LAUNCH( "sad_pyramid8_kernel" );
  return VVB_OK;
}

// The kernel keeps the reference window's 8x8 box sums as uint16 lanes (64 * 1023 fits, 64 * 2047 does not): planes above 10 bits take engine 0.  The cost
// bound takes the wider of the two bit depths, since a pel difference can reach either plane's maximum.
static bool pyramidV2Usable( const vvb_ctx* ctx, int orgPlane, int refPlane, int levels, int baseW, const vvb_me_par* par, int nx, int ny, MePar& mp )
{
  if( ctx->pyramidEngine != 1 || baseW != 8 || par->sub_shift != 0 || levels < 2 || levels > 4 ) return false;
  const int bd = std::max( ctx->planes.p[orgPlane].bitDepth, ctx->planes.p[refPlane].bitDepth );
  if( bd > 10 ) return false;
  int ob = 1; while( ( 1 << ob ) < nx * ny ) ob++;
  const unsigned long long maxCost16 = 4ull * 64 * ( ( 1ull << bd ) - 1 ) + mp.tab.cost[VVB_MVCOST_ENTRIES - 1];
  if( ob > 16 || maxCost16 >= ( 1ull << ( 32 - ob ) ) || maxCost16 >= PYR_NEVER / 4 ) return false;
  const int total = levels == 4 ? pyr_smem<4>( nx, ny ).total : ( levels == 3 ? pyr_smem<3>( nx, ny ).total : pyr_smem<2>( nx, ny ).total );
  if( total > 227 * 1024 ) return false;
  mp.orderBits = ob;
  return true;
}

// had8_ring_kernel: the CTA size (one to four warps, at least one block) that keeps the most warps resident, then as many persistent CTAs as fit
template<bool PACKED, int W, int RC>
static int hadRingLaunch( vvb_ctx* ctx, const Plane& op, const Plane& rp, const vvb_block* dBlocks, int n, const vvb_mv* dPattern, int K, const MePar& mp,
                          uint32_t* dCost, vvb_best* dBest )
{
  using Sh = HadRingShape<W, RC>;
  const auto kernel = had8_ring_kernel<PACKED, W, RC>;
  int threads = 0, perSM = 0;
  for( int t = 128; t >= std::max( 32, Sh::T ); t >>= 1 )
  {
    int b = 0;
    if( cudaOccupancyMaxActiveBlocksPerMultiprocessor( &b, kernel, t, (size_t) had_ring_smem( t, Sh::T, Sh::S, K ).total * 4 ) != cudaSuccess ) b = 0;
    if( b * t > perSM * threads ) { threads = t; perSM = b; }
  }
  cudaGetLastError();
  if( perSM < 1 ) return fail( ctx, VVB_ERR_ARG, "pattern too long for the Hadamard refinement's shared memory" );
  const HadRingSmem L = had_ring_smem( threads, Sh::T, Sh::S, K );
  const int groups = ( n + L.slots - 1 ) / L.slots;
  kernel<<<std::min( groups, perSM * ctx->numSMs ), threads, (size_t) L.total * 4, ctx->stream>>>( op, rp, dBlocks, n, dPattern, K, mp, dCost, dBest );
  CHECK_LAUNCH( "had8_ring_kernel" );
  return VVB_OK;
}

// B operand image of a tensor engine (table: vvb_ctx::tc2Image or itcImage) for the size and transform pair of p: build( std::integral_constant<int, N>, img )
// fills it on the host at the first use, then it stays on the device
template<class Build> static int bImage( vvb_ctx* ctx, const TuPar& p, void* ( &table )[36], const uint4** out, Build build )
{
  void*& slot = table[( ( p.lw - 3 ) * 3 + p.trHor ) * 3 + p.trVer];
  if( !slot )
  {
    std::vector<unsigned char> img;
    switch( p.w ) { case 8: build( std::integral_constant<int, 8>(), img ); break; case 16: build( std::integral_constant<int, 16>(), img ); break;
                    case 32: build( std::integral_constant<int, 32>(), img ); break; default: build( std::integral_constant<int, 64>(), img ); break; }
    void* d = nullptr;
    CU( cudaMalloc( &d, img.size() ) );
    CU( cudaMemcpyAsync( d, img.data(), img.size(), cudaMemcpyHostToDevice, ctx->stream ) );
    CU( cudaStreamSynchronize( ctx->stream ) );                // img is a local
    slot = d;
  }
  *out = (const uint4*) slot;
  return VVB_OK;
}

extern "C" {

// SAD pyramid (see include/vvenc_b200.h): pel work at the base level only, every higher level is the exact sum of its children's SADs
int vvb_sad_search_pyramid_dev( vvb_ctx* ctx, int orgPlane, int refPlane, int levels, const vvb_block* const* dBlocks, const int* counts, int baseW,
                                const vvb_me_par* par, int nx, int ny, vvb_best* const* dBest )
{
  if( !ctx || !dBlocks || !counts || !dBest || !par || levels < 2 || levels > 5 || nx < 1 || ny < 1 ) return fail( ctx, VVB_ERR_ARG, "bad arguments" );
  for( int l = 0; l < levels; l++ ) if( !dBlocks[l] || !dBest[l] || counts[l] < 0 ) return fail( ctx, VVB_ERR_ARG, "bad level arguments" );
  for( int l = 0; l + 1 < levels; l++ ) if( counts[l] < 4 * counts[l + 1] ) return fail( ctx, VVB_ERR_ARG, "a level is shorter than four times the next one" );
  if( ( baseW << ( levels - 1 ) ) > 128 ) return fail( ctx, VVB_ERR_UNSUPPORTED, "top level above 128" );
  if( nx > 512 || ny > 512 || (long long) nx * ny > 65536 ) return fail( ctx, VVB_ERR_UNSUPPORTED, "pyramid search range above 512 positions per axis / 65536 positions" );
  if( counts[0] == 0 ) return VVB_OK;
  CU( cudaSetDevice( ctx->device ) );
  const int T = nx * ny;
  uint32_t* tab[2] = { nullptr, nullptr };
  int rc;
  {
    MePar mp2;
    if( ( rc = makeMePar( ctx, par, mp2 ) ) ) return rc;
    if( ( rc = checkSearchShape( ctx, orgPlane, refPlane, baseW, baseW ) ) ) return rc;
    if( pyramidV2Usable( ctx, orgPlane, refPlane, levels, baseW, par, nx, ny, mp2 ) )
    {
      PyrLevels lv; memset( &lv, 0, sizeof( lv ) );
      for( int l = 0; l < levels; l++ ) { lv.blocks[l] = dBlocks[l]; lv.best[l] = dBest[l]; }
      for( int Ltop = levels - 1; Ltop >= 1; Ltop-- )                                   // roots of this level: the blocks no larger block covers
      {
        const int first = Ltop == levels - 1 ? 0 : 4 * counts[Ltop + 1], nRoots = counts[Ltop] - first;
        if( nRoots <= 0 ) continue;
        if( Ltop == 3 )      rc = pyramidV2LaunchLevel<4>( ctx, orgPlane, refPlane, lv, first, nRoots, nx, ny, mp2 );
        else if( Ltop == 2 ) rc = pyramidV2LaunchLevel<3>( ctx, orgPlane, refPlane, lv, first, nRoots, nx, ny, mp2 );
        else                 rc = pyramidV2LaunchLevel<2>( ctx, orgPlane, refPlane, lv, first, nRoots, nx, ny, mp2 );
        if( rc ) return rc;
      }
      if( counts[0] > 4 * counts[1] &&      // base-level blocks without a parent
          ( rc = sadSearchLaunch( ctx, orgPlane, refPlane, dBlocks[0] + 4 * counts[1], counts[0] - 4 * counts[1], baseW, baseW, par, nx, ny, 1, nullptr, 0, dBest[0] + 4 * counts[1] ) ) ) return rc;
      return VVB_OK;
    }
  }
  // two generations of cost tables: level l reads tab[(l - 1) & 1] and writes tab[l & 1]
  if( levels > 2 && ( rc = carveArena( ctx, ScratchArena::Work, [&]( Layout& L ) { tab[1] = L.take<uint32_t>( (size_t) counts[1] * T ); if( levels > 3 ) tab[0] = L.take<uint32_t>( (size_t) counts[2] * T ); } ) ) )
    return rc;
  CU( cudaMemsetAsync( dBest[1], 0xff, (size_t) counts[1] * sizeof( vvb_best ), ctx->stream ) );   // parents of broken quads stay "invalid" (cost = ~0)
  PyramidOut po{ dBlocks[1], dBest[1], tab[1], T };
  if( counts[1] > 0 && ( rc = sadSearchLaunch( ctx, orgPlane, refPlane, dBlocks[0], 4 * counts[1], baseW, baseW, par, nx, ny, 1, nullptr, 0, dBest[0], &po ) ) ) return rc;
  if( counts[0] > 4 * counts[1] &&      // base-level blocks without a parent
      ( rc = sadSearchLaunch( ctx, orgPlane, refPlane, dBlocks[0] + 4 * counts[1], counts[0] - 4 * counts[1], baseW, baseW, par, nx, ny, 1, nullptr, 0, dBest[0] + 4 * counts[1] ) ) ) return rc;
  MePar mp;
  if( ( rc = makeMePar( ctx, par, mp ) ) ) return rc;
  for( int l = 2; l < levels; l++ )
  {
    uint32_t* in  = tab[( l - 1 ) & 1];
    uint32_t* out = l + 1 < levels ? tab[l & 1] : nullptr;
    if( counts[l] == 0 ) continue;
    sad_table_sum_kernel<<<counts[l], 256, 0, ctx->stream>>>( dBlocks[l], counts[l], nx, ny, mp, in, T, dBest[l - 1], out, T, dBest[l] );
    CHECK_LAUNCH( "sad_table_sum_kernel" );
  }
  return VVB_OK;
}

// host-buffer twin of the pyramid: block lists up, best tables down, one synchronisation
int vvb_sad_search_pyramid( vvb_ctx* ctx, int orgPlane, int refPlane, int levels, const vvb_block* const* blocks, const int* counts, int baseW,
                            const vvb_me_par* par, int nx, int ny, vvb_best* const* best )
{
  if( !ctx || !blocks || !counts || !best || !par || levels < 2 || levels > 5 ) return fail( ctx, VVB_ERR_ARG, "bad arguments" );
  size_t total = 0;
  for( int l = 0; l < levels; l++ ) { if( !blocks[l] || !best[l] || counts[l] < 0 ) return fail( ctx, VVB_ERR_ARG, "bad level arguments" ); total += (size_t) counts[l]; }
  for( int l = 0; l < levels; l++ )
    for( int i = 0; i < counts[l]; i++ )
      if( blocks[l][i].right - blocks[l][i].left + 1 != nx || blocks[l][i].bottom - blocks[l][i].top + 1 != ny ) return fail( ctx, VVB_ERR_ARG, "pyramid blocks must share one nx x ny range" );
  if( total == 0 ) return VVB_OK;
  HostCall call( ctx );
  const vvb_block* pb[5]; vvb_best* po[5];
  for( int l = 0; l < levels; l++ ) call.in( pb[l], blocks[l], counts[l] ).out( po[l], best[l], counts[l] );
  return call.run( [&] { return vvb_sad_search_pyramid_dev( ctx, orgPlane, refPlane, levels, pb, counts, baseW, par, nx, ny, po ); } );
}

// device-resident variant: the host states the largest window (max_nx x max_ny positions) in the batch, it sizes shared memory
int vvb_sad_search_dev( vvb_ctx* ctx, int orgPlane, int refPlane, const vvb_block* dBlocks, int n, int w, int h, const vvb_me_par* par,
                        int maxNx, int maxNy, uint32_t* dTables, int tableStride, vvb_best* dBest )
{
  if( !ctx || !dBlocks || !dBest || !par || n < 0 || maxNx < 1 || maxNy < 1 ) return fail( ctx, VVB_ERR_ARG, "bad arguments" );
  return sadSearchLaunch( ctx, orgPlane, refPlane, dBlocks, n, w, h, par, maxNx, maxNy, par->quad_order, dTables, tableStride, dBest );
}

int vvb_sad_search( vvb_ctx* ctx, int orgPlane, int refPlane, const vvb_block* blocks, int n, int w, int h, const vvb_me_par* par,
                    uint32_t* tables, int tableStride, vvb_best* best )
{
  if( !ctx || !blocks || !best || n < 0 ) return fail( ctx, VVB_ERR_ARG, "bad arguments" );
  if( n == 0 ) return VVB_OK;
  int maxNx = 1, maxNy = 1;
  for( int i = 0; i < n; i++ )
  {
    const int nx = blocks[i].right - blocks[i].left + 1, ny = blocks[i].bottom - blocks[i].top + 1;
    if( nx < 1 || ny < 1 ) return fail( ctx, VVB_ERR_ARG, "empty search range" );
    if( tables && nx * ny > tableStride ) return fail( ctx, VVB_ERR_ARG, "table_stride smaller than the window" );
    maxNx = std::max( maxNx, nx ); maxNy = std::max( maxNy, ny );
  }
  const vvb_block* dB; vvb_best* dO; uint32_t* dT;
  return HostCall( ctx ).in( dB, blocks, n ).out( dO, best, n ).out( dT, tables, (size_t) n * tableStride ).run( [&]
  {
    return sadSearchLaunch( ctx, orgPlane, refPlane, dB, n, w, h, par, maxNx, maxNy, 1 /* quads are verified per CTA */, dT, tableStride, dO );
  } );
}

int vvb_cost_pattern_dev( vvb_ctx* ctx, int dfunc, int orgPlane, int refPlane, const vvb_block* dBlocks, int n, int w, int h, const vvb_mv* dPattern, int K,
                          const vvb_me_par* par, uint32_t* dCost, vvb_best* dBest )
{
  if( !ctx || !dBlocks || !dPattern || !par || n < 0 || K < 1 || ( !dCost && !dBest ) ) return fail( ctx, VVB_ERR_ARG, "bad arguments" );
  int rc = checkSearchShape( ctx, orgPlane, refPlane, w, h );
  if( rc ) return rc;
  MePar mp;
  if( ( rc = makeMePar( ctx, par, mp ) ) ) return rc;
  if( dfunc != FAM_SAD ) mp.subShift = 0;
  if( ( rc = checkDistShape( ctx, dfunc, w, h, mp.subShift ) ) ) return rc;
  if( n == 0 ) return VVB_OK;
  CU( cudaSetDevice( ctx->device ) );
  const Plane &op = ctx->planes.p[orgPlane], &rp = ctx->planes.p[refPlane];
  // small-radius Hadamard refinement of square power-of-two blocks up to 64x64: the dispatch lands on 8x8 tiles (RdCost.cpp:1836-1905)
  const int R = par->pattern_radius;
  if( dfunc == FAM_HAD && R > 0 && R <= 8 && K <= 1024 && w == h && w >= 8 && w <= 64 && isPow2( w ) )
  {
    const bool packed = op.bitDepth <= 10 && rp.bitDepth <= 10;
    if( w == 8 )      // one tile per block: candidates read through L1 (faster here than the staged windows)
    {
      const int bpc = std::max( 1, std::min( 32, 512 / K ) );
      const HadDirSmem LD = had_dir_smem( K, bpc );
      const int bd = std::min( 256, std::max( 64, ( bpc * K + 31 ) & ~31 ) );
      const int grid = std::min( ( n + bpc - 1 ) / bpc, ctx->numSMs * 8 );
      if( packed ) had8_direct_kernel<true><<<grid, bd, (size_t) LD.total * 4, ctx->stream>>>( op, rp, dBlocks, n, w, h, bpc, dPattern, K, mp, dCost, dBest );
      else         had8_direct_kernel<false><<<grid, bd, (size_t) LD.total * 4, ctx->stream>>>( op, rp, dBlocks, n, w, h, bpc, dPattern, K, mp, dCost, dBest );
      CHECK_LAUNCH( "had8_direct_kernel" );
      return VVB_OK;
    }
#define VVB_RING( W ) ( R <= 2 ? ( packed ? hadRingLaunch<true, W, 2> : hadRingLaunch<false, W, 2> ) : ( packed ? hadRingLaunch<true, W, 8> : hadRingLaunch<false, W, 8> ) )
    const auto launch = w == 16 ? VVB_RING( 16 ) : w == 32 ? VVB_RING( 32 ) : VVB_RING( 64 );
#undef VVB_RING
    return launch( ctx, op, rp, dBlocks, n, dPattern, K, mp, dCost, dBest );
  }
  const int G = dfunc == FAM_SAD ? pick_group( FAM_SAD, w, h >> mp.subShift ) : pick_group( dfunc, w, h );
#define LAUNCH_PAT( GG ) cost_pattern_kernel<GG><<<n, 128, 0, ctx->stream>>>( op, rp, dBlocks, w, h, dfunc, dPattern, K, mp, dCost, dBest )
  switch( G ) { case 4: LAUNCH_PAT( 4 ); break; case 8: LAUNCH_PAT( 8 ); break; case 16: LAUNCH_PAT( 16 ); break; default: LAUNCH_PAT( 32 ); break; }
#undef LAUNCH_PAT
  CHECK_LAUNCH( "cost_pattern_kernel" );
  return VVB_OK;
}

int vvb_cost_pattern( vvb_ctx* ctx, int dfunc, int orgPlane, int refPlane, const vvb_block* blocks, int n, int w, int h, const vvb_mv* pattern, int K,
                      const vvb_me_par* par, uint32_t* costOut, vvb_best* best )
{
  if( !ctx || !blocks || !pattern || !par || n < 0 || K < 1 || ( !costOut && !best ) ) return fail( ctx, VVB_ERR_ARG, "bad arguments" );
  if( n == 0 ) return VVB_OK;
  vvb_me_par hp = *par;                                   // the host sees the pattern: its radius selects the staged Hadamard kernel
  hp.pattern_radius = 0;
  for( int i = 0; i < K; i++ ) hp.pattern_radius = std::max( hp.pattern_radius, std::max( std::abs( (int) pattern[i].dx ), std::abs( (int) pattern[i].dy ) ) );
  const vvb_block* dB; const vvb_mv* dP; uint32_t* dS; vvb_best* dO;
  return HostCall( ctx ).in( dB, blocks, n ).in( dP, pattern, K ).out( dS, costOut, (size_t) n * K ).out( dO, best, n )
                        .run( [&] { return vvb_cost_pattern_dev( ctx, dfunc, orgPlane, refPlane, dB, n, w, h, dP, K, &hp, dS, dO ); } );
}

int vvb_sad_pattern_dev( vvb_ctx* ctx, int orgPlane, int refPlane, const vvb_block* dBlocks, int n, int w, int h, const vvb_mv* dPattern, int K,
                         const vvb_me_par* par, uint32_t* dSad, vvb_best* dBest )
{
  return vvb_cost_pattern_dev( ctx, FAM_SAD, orgPlane, refPlane, dBlocks, n, w, h, dPattern, K, par, dSad, dBest );
}

int vvb_sad_pattern( vvb_ctx* ctx, int orgPlane, int refPlane, const vvb_block* blocks, int n, int w, int h, const vvb_mv* pattern, int K,
                     const vvb_me_par* par, uint32_t* sadOut, vvb_best* best )
{
  return vvb_cost_pattern( ctx, FAM_SAD, orgPlane, refPlane, blocks, n, w, h, pattern, K, par, sadOut, best );
}

int vvb_blocks_set_start_dev( vvb_ctx* ctx, vvb_block* dBlocks, const vvb_best* dBest, int n )
{
  if( !ctx || !dBlocks || !dBest || n < 0 ) return fail( ctx, VVB_ERR_ARG, "bad arguments" );
  if( n == 0 ) return VVB_OK;
  CU( cudaSetDevice( ctx->device ) );
  blocks_set_start_kernel<<<std::min( ( n + 255 ) / 256, ctx->numSMs * 8 ), 256, 0, ctx->stream>>>( dBlocks, dBest, n );
  CHECK_LAUNCH( "blocks_set_start_kernel" );
  return VVB_OK;
}

// ---- transform + quantise ----------------------------------------------------------------------------------------
static int teamGrid( vvb_ctx* ctx, int n, int nTeams, size_t smem )
{
  const int ctasNeeded = ( n + nTeams - 1 ) / nTeams;
  const int perSM = (int) std::max<size_t>( 1, std::min<size_t>( 16, ( 200 * 1024 ) / ( smem + 1024 ) ) );
  return std::min( ctasNeeded, ctx->numSMs * perSM );
}

static int makeTuPar( vvb_ctx* ctx, const vvb_tu_par* in, TuPar& p )
{
  if( !in ) return fail( ctx, VVB_ERR_ARG, "null tu_par" );
  const int w = in->w, h = in->h;
  if( !isPow2( w ) || !isPow2( h ) || w < 4 || h < 4 || w > 64 || h > 64 ) return fail( ctx, VVB_ERR_UNSUPPORTED, "TU sizes are 4..64" );
  if( in->tr_hor < 0 || in->tr_hor > 2 || in->tr_ver < 0 || in->tr_ver > 2 ) return fail( ctx, VVB_ERR_ARG, "unknown transform type" );
  if( ( in->tr_hor && w > 32 ) || ( in->tr_ver && h > 32 ) ) return fail( ctx, VVB_ERR_UNSUPPORTED, "DST-VII/DCT-VIII exist for 4..32 only (TrQuant.cpp:76-81)" );
  if( in->bit_depth < 8 || in->bit_depth > 12 ) return fail( ctx, VVB_ERR_UNSUPPORTED, "bit depth 8..12" );
  p.w = w; p.h = h; p.lw = ilog2h( w ); p.lh = ilog2h( h );
  p.trHor = in->tr_hor; p.trVer = in->tr_ver;
  const int skipW = ( p.trHor != 0 && w == 32 ) ? 16 : ( w > 32 ? w - 32 : 0 );        // TrQuant.cpp:496
  const int skipH = ( p.trVer != 0 && h == 32 ) ? 16 : ( h > 32 ? h - 32 : 0 );        // TrQuant.cpp:497
  p.keepW = w - skipW; p.keepH = h - skipH;
  p.s1 = p.lw + in->bit_depth + 6 - 15;                                                 // TrQuant.cpp:544
  p.s2 = p.lh + 6;                                                                       // TrQuant.cpp:545
  if( p.s1 < 0 ) return fail( ctx, VVB_ERR_UNSUPPORTED, "negative first-stage shift (TrQuant.cpp:546 CHECK)" );
  p.offH = vvc_tr_offset_host[p.trHor][p.lw]; p.offV = vvc_tr_offset_host[p.trVer][p.lh];
  p.regionW = std::min( 32, w ); p.regionH = std::min( 32, h );
  p.scanOff = ( ( p.lw - 2 ) * 5 + ( p.lh - 2 ) ) * 1024;
  p.ts = in->transform_skip ? 1 : 0;
  if( p.ts )
  {
    if( w > 32 || h > 32 ) return fail( ctx, VVB_ERR_UNSUPPORTED, "transform skip exists up to 32 x 32 (log2MaxTransformSkipBlockSize)" );
    if( in->lfnst_idx ) return fail( ctx, VVB_ERR_UNSUPPORTED, "LFNST does not apply to skipped transforms" );
    if( in->input_bit_depth_delta < 0 || in->input_bit_depth_delta > 8 ) return fail( ctx, VVB_ERR_ARG, "input_bit_depth_delta 0..8" );
    p.keepW = w; p.keepH = h;
  }
  // QpParam (Quant.cpp:89-124): Qps[0] = clip( qp + qpBdOffset ), Qps[1] = max( Qps[0], 4 + 6 * internalMinusInputBitDepth ) for skipped transforms
  auto baseQpOf = [&]( bool tsQp ) { return tsQp ? std::max( baseQp( in ), 4 + 6 * in->input_bit_depth_delta ) : baseQp( in ); };
  const int sqrt2 = p.ts ? 0 : ( ( p.lw + p.lh ) & 1 );                                   // TU::needsSqrt2Scale, UnitTools.cpp:3616-3621
  const int trShift = 15 - in->bit_depth - ( ( p.lw + p.lh ) >> 1 ) - sqrt2;              // Quant.h:69-72, Quant.cpp:767
  {
    const int qp = baseQpOf( p.ts != 0 ), per = qp / 6, rem = qp % 6;
    p.scale = vvc_quant_scales_host[sqrt2][rem];
    p.qbits = 14 + per + ( p.ts ? 0 : trShift );                                          // Quant.cpp:772
    p.add   = (long long)( in->is_irap ? 171 : 85 ) << ( p.qbits - 9 );                   // :774
  }
  {
    // Quant::xNeedRDOQ (:852-879): the dependent-quantisation pre-check adds 1 AFTER the clip and only for non-skipped transforms; the transform shift stays in
    // its iQBits even for skipped transforms; chroma components round with 256
    const bool isDq = in->dep_quant && !p.ts;
    const int qp = isDq ? baseQpOf( false ) + 1 : baseQpOf( p.ts != 0 ), per = qp / 6, rem = qp % 6;
    p.scaleRdoq = vvc_quant_scales_host[sqrt2][rem];
    p.qbitsRdoq = 14 + per + trShift;
    p.addRdoq   = (long long)( in->is_chroma ? 256 : 171 ) << ( p.qbitsRdoq - 9 );
  }
  if( p.qbits < 9 || p.qbitsRdoq < 9 ) return fail( ctx, VVB_ERR_UNSUPPORTED, "quantiser shift below 9" );
  const int thrVal = 8;                                                                  // vvencCfg.cpp:971-973
  const int32_t thres = (int32_t)( (int64_t) thrVal << ( p.qbits - 1 ) );               // Quant.cpp:175-176 (TCoeff cast)
  p.useThres = thres / ( p.scale << 2 );                                                 // Quant.cpp:180
  int t = ( w * h ) / 4;
  p.team = std::max( 4, std::min( 128, t ) );
  {                                                                                      // Quant::dequant, Quant.cpp:554-607
    const int qp = baseQpOf( p.ts != 0 ), per = qp / 6, rem = qp % 6;
    static const int invScales[2][6] = { { 40, 45, 51, 57, 64, 72 }, { 57, 64, 72, 80, 90, 102 } };   // g_invQuantScales, Rom.cpp:1396-1400
    p.dqScale = invScales[sqrt2][rem];
    p.dqShift = 6 - ( ( p.ts ? 0 : trShift ) + per );                                    // IQUANT_SHIFT = 6 (CommonDef.h:370); :561
    const int tib = std::min( 16, 32 + p.dqShift - 7 );                                  // targetInputBitDepth, Quant.cpp:606
    p.dqInMax = ( 1 << ( tib - 1 ) ) - 1;
    p.s2Inv   = 20 - in->bit_depth;                                                      // TrQuant.cpp:609
    p.pelMax  = ( 1 << in->bit_depth ) - 1;
  }
  p.lKeepW = ilog2h( p.keepW ); p.lKeepH = ilog2h( p.keepH ); p.lRegW = ilog2h( p.regionW );
  p.signHiding = in->sign_hiding ? 1 : 0;
  p.lfnstIdx = 0; p.lfnstTranspose = 0; p.lfnstMat = nullptr; p.lfnstMaxScan = 0x7fffffff;
  if( in->lfnst_idx )
  {
    // TrQuant::xFwdLfnst applies to intra CUs, whose luma TUs use DCT-II when an LFNST index is set (MTS and LFNST exclude each other)
    if( in->lfnst_idx < 0 || in->lfnst_idx > 2 || in->lfnst_set < 0 || in->lfnst_set > 3 ) return fail( ctx, VVB_ERR_ARG, "lfnst_idx 0..2, lfnst_set 0..3" );
    if( in->tr_hor != 0 || in->tr_ver != 0 ) return fail( ctx, VVB_ERR_UNSUPPORTED, "LFNST goes with DCT-II" );
    const bool whge3 = w >= 8 && h >= 8;
    p.lfnstIdx = in->lfnst_idx; p.lfnstTranspose = in->lfnst_transpose ? 1 : 0;
    p.lfnstMat = ctx->d_lfnst + ( whge3 ? ( in->lfnst_set * 2 + in->lfnst_idx - 1 ) * 16 * 48 : VVC_LFNST_4X4_OFFSET + ( in->lfnst_set * 2 + in->lfnst_idx - 1 ) * 16 * 16 );
    p.lfnstMaxScan = ( ( w == 4 && h == 4 ) || ( w == 8 && h == 8 ) ) ? 7 : 15;                   // Quant.cpp:151-158
  }
  p.q32 = p.qbits <= 30 ? 1 : 0;
  p.add32 = (unsigned)( p.add & 0xffffffffll );
  {
    const long long num = ( 1ll << p.qbitsRdoq ) - p.addRdoq;                         // > 0: addRdoq = 171 << (qbits-9) < 2^(qbits-1)
    const long long thr = ( num + p.scaleRdoq - 1 ) / p.scaleRdoq;
    p.rdoqThr = thr > 0xffffffffll ? 0xffffffffu : (unsigned) thr;
  }
  return VVB_OK;
}

// forward tensor-core engine (trquant_tc2_kernels.cuh): square TUs 8..64 with the plain quantiser
static bool tc2Eligible( const vvb_ctx* ctx, const TuPar& p )
{
  return ctx->tensorTransform && !p.lfnstIdx && !p.ts && !p.signHiding && p.w == p.h && p.w >= 8 && p.w <= 64 && p.s1 >= 0;
}
// dResi alone: residual pool; dResi + dResi2: original and prediction pools; dBlocks: positions in the two planes
static int tc2Launch( vvb_ctx* ctx, const TuPar& p, const int16_t* dResi, int orgPlane, int predPlane, const vvb_block* dBlocks, int n,
                      int32_t* dCoef, int16_t* dQ, int32_t* dAbsSum, int32_t* dLastPos, uint8_t* dNeedRdoq, const int16_t* dResi2 = nullptr )
{
  const Plane po = dBlocks ? ctx->planes.p[orgPlane] : Plane{}, pp = dBlocks ? ctx->planes.p[predPlane] : Plane{};
  const uint4* dImg; int rc;
  if( ( rc = bImage( ctx, p, ctx->tc2Image, &dImg, [&]( auto nc, std::vector<unsigned char>& img ) {
          constexpr int N = decltype( nc )::value; using S = Tc2Shape<N>;
          img.resize( 2 * S::B1_BYTES + 3 * S::B2_BYTES ); tc2_build_b_image<N>( vvc_tr_table_host, p.offH, p.offV, p.keepW, p.keepH, img.data() ); } ) ) ) return rc;
#define VVB_FWD_TC_CALL( Nv ) { using S = Tc2Shape<Nv>; const int tiles = ( n + S::TPT - 1 ) / S::TPT; \
    static int perSm[3] = { 0, 0, 0 }; const int mode = dBlocks ? 1 : dResi2 ? 2 : 0; int& ps = perSm[mode]; \
    if( !ps ) { cudaFuncAttributes fa = {}; \
                if( mode == 1 ) cudaFuncGetAttributes( &fa, fwd_trquant_tc2_kernel<Nv, 1> ); else if( mode == 2 ) cudaFuncGetAttributes( &fa, fwd_trquant_tc2_kernel<Nv, 2> ); \
                else cudaFuncGetAttributes( &fa, fwd_trquant_tc2_kernel<Nv, 0> ); \
                const int regs = std::max( fa.numRegs, 32 ); \
                ps = std::min( 65536 / ( regs * 128 ), ( 227 * 1024 ) / ( (int) S::SMEM + (int) fa.sharedSizeBytes + 1024 ) ); ps = std::max( std::min( ps, Nv == 8 ? 6 : 8 ), 1 ); } \
    const int grid = std::min( tiles, ctx->numSMs * ps ); \
    if( mode == 1 )      fwd_trquant_tc2_kernel<Nv, 1><<<grid, 128, S::SMEM, ctx->stream>>>( p, dImg, ctx->d_scan, nullptr, nullptr, po, pp, dBlocks, n, dCoef, dQ, dAbsSum, dLastPos, dNeedRdoq ); \
    else if( mode == 2 ) fwd_trquant_tc2_kernel<Nv, 2><<<grid, 128, S::SMEM, ctx->stream>>>( p, dImg, ctx->d_scan, dResi, dResi2, po, pp, nullptr, n, dCoef, dQ, dAbsSum, dLastPos, dNeedRdoq ); \
    else                 fwd_trquant_tc2_kernel<Nv, 0><<<grid, 128, S::SMEM, ctx->stream>>>( p, dImg, ctx->d_scan, dResi, nullptr, po, pp, nullptr, n, dCoef, dQ, dAbsSum, dLastPos, dNeedRdoq ); }
  switch( p.w ) { case 8: VVB_FWD_TC_CALL( 8 ) break; case 16: VVB_FWD_TC_CALL( 16 ) break; case 32: VVB_FWD_TC_CALL( 32 ) break; default: VVB_FWD_TC_CALL( 64 ) break; }
#undef VVB_FWD_TC_CALL
  CHECK_LAUNCH( "fwd_trquant_tc2_kernel" );
  return VVB_OK;
}

// inverse tensor-core engine (itrquant_tc_kernels.cuh): square 8 / 16 / 32 TUs, plain or DepQuant dequantiser parameters in p, no LFNST / transform skip
static bool itcEligible( const vvb_ctx* ctx, const TuPar& p, const void* dQ )
{
  return ctx->tensorTransform && !p.lfnstIdx && !p.ts && p.w == p.h && p.w >= 8 && p.w <= 64 && ( ( (uintptr_t) dQ ) & 15 ) == 0;
}
// dResi != nullptr: levels -> residual.  Otherwise the second half of the TU round trip (reconstruction + distortions; dSum / dLast from the forward engine)
static int itcLaunch( vvb_ctx* ctx, const TuPar& p, const int16_t* dQ, int n, int16_t* dResi,
                      int orgPlane, int predPlane, const vvb_block* dBlocks, const int16_t* dOrg, const int16_t* dPred, int16_t* dReco, TuResult* dRes, const int32_t* dSum, const int32_t* dLast )
{
  const uint4* dImg; int rc;
  if( ( rc = bImage( ctx, p, ctx->itcImage, &dImg, [&]( auto nc, std::vector<unsigned char>& img ) {
          constexpr int N = decltype( nc )::value;
          img.resize( 4 * ItcShape<N>::B_BYTES ); itc_build_b_image<N>( vvc_tr_table_host, p.offH, p.offV, p.keepW, p.keepH, img.data() ); } ) ) ) return rc;
  const Plane po = dBlocks ? ctx->planes.p[orgPlane] : Plane{}, pp = dBlocks ? ctx->planes.p[predPlane] : Plane{};
#define VVB_ITC_CALL( Nv ) { using S = ItcShape<Nv>; const int tiles = ( n + S::TPT - 1 ) / S::TPT; const int grid = std::min( tiles, ctx->numSMs * std::min( 6, ( 227 * 1024 ) / ( S::SMEM + 1024 ) ) ); \
    if( dResi ) inv_trquant_tc_kernel<Nv, false><<<grid, 128, S::SMEM, ctx->stream>>>( p, dImg, dQ, n, dResi, 0, po, pp, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr ); \
    else        inv_trquant_tc_kernel<Nv, true><<<grid, 128, S::SMEM, ctx->stream>>>( p, dImg, dQ, n, nullptr, dBlocks ? 1 : 0, po, pp, dBlocks, dOrg, dPred, dReco, dRes, dSum, dLast ); }
  switch( p.w ) { case 8: VVB_ITC_CALL( 8 ) break; case 16: VVB_ITC_CALL( 16 ) break; case 32: VVB_ITC_CALL( 32 ) break; default: VVB_ITC_CALL( 64 ) break; }
#undef VVB_ITC_CALL
  CHECK_LAUNCH( "inv_trquant_tc_kernel" );
  return VVB_OK;
}

int vvb_fwd_trquant_dev( vvb_ctx* ctx, const vvb_tu_par* par, const int16_t* dResi, int n, int32_t* dCoef, int16_t* dQ, int32_t* dAbsSum, int32_t* dLastPos, uint8_t* dNeedRdoq )
{
  if( !ctx || !dResi || !dQ || n < 0 ) return fail( ctx, VVB_ERR_ARG, "bad arguments" );
  TuPar p;
  int rc = makeTuPar( ctx, par, p );
  if( rc ) return rc;
  if( n == 0 ) return VVB_OK;
  CU( cudaSetDevice( ctx->device ) );
  if( tc2Eligible( ctx, p ) ) return tc2Launch( ctx, p, dResi, 0, 0, nullptr, n, dCoef, dQ, dAbsSum, dLastPos, dNeedRdoq );
  const bool ext = p.lfnstIdx != 0 || p.signHiding != 0 || p.ts != 0;        // the plain instantiation carries neither the LFNST stage, the sign-bit hiding pass nor transform skip
#define VVB_FWD_CALL( LWv, LHv ) { using S = TuShape<LWv, LHv>; const size_t smem = (size_t)( S::MAT_WORDS + S::NTEAMS * S::TEAM_WORDS ) * 4; \
    if( ext ) fwd_trquant_kernel<LWv, LHv, true><<<teamGrid( ctx, n, S::NTEAMS, smem ), 128, smem, ctx->stream>>>( p, ctx->d_trTable, ctx->d_scan, dResi, n, dCoef, dQ, dAbsSum, dLastPos, dNeedRdoq ); \
    else      fwd_trquant_kernel<LWv, LHv, false><<<teamGrid( ctx, n, S::NTEAMS, smem ), 128, smem, ctx->stream>>>( p, ctx->d_trTable, ctx->d_scan, dResi, n, dCoef, dQ, dAbsSum, dLastPos, dNeedRdoq ); }
  VVB_TU_DISPATCH( p.lw, p.lh, VVB_FWD_CALL )
#undef VVB_FWD_CALL
  CHECK_LAUNCH( "fwd_trquant_kernel" );
  return VVB_OK;
}

int vvb_fwd_trquant( vvb_ctx* ctx, const vvb_tu_par* par, const int16_t* resi, int n, int32_t* coef, int16_t* q, int32_t* absSum, int32_t* lastPos, uint8_t* needRdoq )
{
  if( !ctx || !par || !resi || !q || n < 0 ) return fail( ctx, VVB_ERR_ARG, "bad arguments" );
  if( n == 0 ) return VVB_OK;
  const size_t samples = (size_t) n * par->w * par->h;
  const int16_t* dR; int16_t* dQ; int32_t *dC, *dSum, *dLast; uint8_t* dNr;
  return HostCall( ctx ).in( dR, resi, samples ).out( dQ, q, samples ).out( dC, coef, samples ).out( dSum, absSum, n, true ).out( dLast, lastPos, n, true ).out( dNr, needRdoq, n, true )
                        .run( [&] { return vvb_fwd_trquant_dev( ctx, par, dR, n, dC, dQ, dSum, dLast, dNr ); } );
}

int vvb_fwd_trquant_planes_dev( vvb_ctx* ctx, const vvb_tu_par* par, int orgPlane, int predPlane, const vvb_block* dBlocks, int n,
                                int32_t* dCoef, int16_t* dQ, int32_t* dAbsSum, int32_t* dLastPos, uint8_t* dNeedRdoq )
{
  if( !ctx || !par || !dBlocks || !dQ || n < 0 ) return fail( ctx, VVB_ERR_ARG, "bad arguments" );
  if( !validPlane( ctx, orgPlane ) || !validPlane( ctx, predPlane ) ) return fail( ctx, VVB_ERR_ARG, "unknown plane" );
  if( n == 0 ) return VVB_OK;
  CU( cudaSetDevice( ctx->device ) );
  TuPar p;
  int rc = makeTuPar( ctx, par, p );
  if( rc ) return rc;
  if( tc2Eligible( ctx, p ) ) return tc2Launch( ctx, p, nullptr, orgPlane, predPlane, dBlocks, n, dCoef, dQ, dAbsSum, dLastPos, dNeedRdoq );
  // CUDA-core engine: the residual is formed while the TU is loaded (one launch, no compact residual buffer)
  const Plane &po = ctx->planes.p[orgPlane], &pp = ctx->planes.p[predPlane];
  const bool ext = p.lfnstIdx != 0 || p.signHiding != 0 || p.ts != 0;
#define VVB_FWDP_CALL( LWv, LHv ) { using S = TuShape<LWv, LHv>; const size_t smem = (size_t)( S::MAT_WORDS + S::NTEAMS * S::TEAM_WORDS ) * 4; \
    if( ext ) fwd_trquant_planes_kernel<LWv, LHv, true><<<teamGrid( ctx, n, S::NTEAMS, smem ), 128, smem, ctx->stream>>>( p, ctx->d_trTable, ctx->d_scan, po, pp, dBlocks, n, dCoef, dQ, dAbsSum, dLastPos, dNeedRdoq ); \
    else      fwd_trquant_planes_kernel<LWv, LHv, false><<<teamGrid( ctx, n, S::NTEAMS, smem ), 128, smem, ctx->stream>>>( p, ctx->d_trTable, ctx->d_scan, po, pp, dBlocks, n, dCoef, dQ, dAbsSum, dLastPos, dNeedRdoq ); }
  VVB_TU_DISPATCH( p.lw, p.lh, VVB_FWDP_CALL )
#undef VVB_FWDP_CALL
  CHECK_LAUNCH( "fwd_trquant_planes_kernel" );
  return VVB_OK;
}

int vvb_fwd_trquant_planes( vvb_ctx* ctx, const vvb_tu_par* par, int orgPlane, int predPlane, const vvb_block* blocks, int n,
                            int32_t* coef, int16_t* q, int32_t* absSum, int32_t* lastPos, uint8_t* needRdoq )
{
  if( !ctx || !par || !blocks || !q || n < 0 ) return fail( ctx, VVB_ERR_ARG, "bad arguments" );
  if( n == 0 ) return VVB_OK;
  const size_t samples = (size_t) n * par->w * par->h;
  const vvb_block* dB; int16_t* dQ; int32_t *dC, *dSum, *dLast; uint8_t* dNr;
  return HostCall( ctx ).in( dB, blocks, n ).out( dQ, q, samples ).out( dC, coef, samples ).out( dSum, absSum, n, true ).out( dLast, lastPos, n, true ).out( dNr, needRdoq, n, true )
                        .run( [&] { return vvb_fwd_trquant_planes_dev( ctx, par, orgPlane, predPlane, dB, n, dC, dQ, dSum, dLast, dNr ); } );
}


// Whole per-picture chain in one call (include/vvenc_b200.h): search -> start = best -> pattern distortion -> TU, chained on the device
// ---- levels trimmed to lastPos, in scan order (the e2e download) --------------------------------------------------------------------------------------------
int vvb_pack_levels_dev( vvb_ctx* ctx, const vvb_tu_par* par, const int16_t* dQ, const int32_t* dLastPos, int n, int16_t* outPacked, uint32_t* dOffsets )
{
  if( !ctx || !par || !dQ || !dLastPos || !outPacked || !dOffsets || n < 0 ) return fail( ctx, VVB_ERR_ARG, "bad arguments" );
  if( !isPow2( par->w ) || !isPow2( par->h ) || par->w < 4 || par->h < 4 || par->w > 64 || par->h > 64 ) return fail( ctx, VVB_ERR_UNSUPPORTED, "TU sizes are 4..64" );
  if( n == 0 ) return VVB_OK;
  CU( cudaSetDevice( ctx->device ) );
  const int lw = ilog2h( par->w ), lh = ilog2h( par->h ), lrw = std::min( lw, 5 );
  const int32_t* fwd = scanOrder( ctx->d_scan, lw, lh );
  uint32_t* dSizes; uint8_t* dTmp; int rc;
  size_t tmpBytes = 0;
  cub::DeviceScan::ExclusiveSum( nullptr, tmpBytes, (uint32_t*) nullptr, (uint32_t*) nullptr, n + 1, ctx->stream );
  if( ( rc = carveArena( ctx, ScratchArena::Work, [&]( Layout& L ) { dSizes = L.take<uint32_t>( n + 1 ); dTmp = L.take<uint8_t>( tmpBytes ); } ) ) ) return rc;
  pack_sizes_kernel<<<( n + 1 + 255 ) / 256, 256, 0, ctx->stream>>>( dLastPos, n, dSizes );
  CHECK_LAUNCH( "pack_sizes_kernel" );
  CU( cub::DeviceScan::ExclusiveSum( dTmp, tmpBytes, dSizes, dOffsets, n + 1, ctx->stream ) );
  ctx->launches++;
  pack_levels_kernel<<<( n + 3 ) / 4, 128, 0, ctx->stream>>>( dQ, dLastPos, dOffsets, fwd, par->w, par->w * par->h, lrw, n, outPacked );
  CHECK_LAUNCH( "pack_levels_kernel" );
  return VVB_OK;
}

// scan position -> raster index (row pitch w) of the grouped 4x4 diagonal scan of a w x h TU (min(w,32) * min(h,32) entries): what unpacks vvb_pack_levels output
int vvb_scan_order( int w, int h, int32_t* out )
{
  if( !out || !isPow2( w ) || !isPow2( h ) || w < 4 || h < 4 || w > 64 || h > 64 ) return VVB_ERR_ARG;
  std::vector<int32_t> inv;
  buildScanTables( inv );
  const int lw = ilog2h( w ), lh = ilog2h( h ), rw = std::min( w, 32 ), rh = std::min( h, 32 );
  const int32_t* t = scanOrder( inv.data(), lw, lh );
  for( int s = 0; s < rw * rh; s++ ) out[s] = ( t[s] / rw ) * w + ( t[s] % rw );
  return VVB_OK;
}

int vvb_search_refine_tu( vvb_ctx* ctx, int orgPlane, int refPlane, int levels, const vvb_level_io* io, int baseW, const vvb_me_par* me, int nx, int ny,
                          int refineDfunc, const vvb_mv* pattern, int K )
{
  if( !ctx || !io || !me || levels < 2 || levels > 5 || nx < 1 || ny < 1 ) return fail( ctx, VVB_ERR_ARG, "bad arguments" );
  bool anyRefine = false;
  for( int l = 0; l < levels; l++ )
  {
    if( io[l].count < 0 || ( io[l].count && ( !io[l].blocks || !io[l].best ) ) ) return fail( ctx, VVB_ERR_ARG, "bad level arguments" );
    anyRefine = anyRefine || io[l].refine_cost;
  }
  if( anyRefine && ( !pattern || K < 1 ) ) return fail( ctx, VVB_ERR_ARG, "refinement needs a pattern" );
  HostCall call( ctx );
  const vvb_block* pb[5]; vvb_best* po[5]; int counts[5];
  uint32_t *cost[5], *offsets[5]; int16_t *q[5], *packed[5]; int32_t *sum[5], *last[5]; uint8_t* nr[5]; bool pageable[5];
  for( int l = 0; l < levels; l++ )
  {
    const vvb_level_io& L = io[l];
    if( L.packed_q && ( !L.packed_offsets || !L.last_pos ) ) return fail( ctx, VVB_ERR_ARG, "packed levels need packed_offsets and last_pos" );
    const size_t n = (size_t)( counts[l] = L.count ), side = (size_t) baseW << l, tuN = L.q || L.packed_q ? n : 0;
    packed[l] = nullptr; pageable[l] = false;
    if( L.packed_q && n )
    {
      // pinned host memory is visible to the device under UVA: the pack kernel then writes the trimmed levels straight into the caller's buffer (no size has to
      // come back first); a pageable destination gets a staging area in the arena
      cudaPointerAttributes at;
      if( cudaPointerGetAttributes( &at, L.packed_q ) == cudaSuccess && at.type == cudaMemoryTypeHost && at.devicePointer ) packed[l] = (int16_t*) at.devicePointer;
      else { cudaGetLastError(); pageable[l] = true; call.tmp( packed[l], n * side * side ).tmp( offsets[l], n + 1 ); }
    }
    if( n ) call.in( pb[l], L.blocks, n ); else call.tmp( pb[l], 0 );             // an empty level may come without a block list
    call.out( po[l], L.best, n, true ).out( cost[l], L.refine_cost, n * K ).out( q[l], L.q, tuN * side * side, tuN > 0 )
        .out( sum[l], L.abs_sum, tuN, tuN > 0 ).out( last[l], L.last_pos, tuN, tuN > 0 ).out( nr[l], L.need_rdoq, tuN, tuN > 0 );
    if( !pageable[l] ) call.out( offsets[l], L.packed_offsets, L.packed_q && n ? n + 1 : 0 );
  }
  const vvb_mv* dPattern;
  call.in( dPattern, anyRefine ? pattern : nullptr, K );
  return call.run( [&]
  {
    int rc = vvb_sad_search_pyramid_dev( ctx, orgPlane, refPlane, levels, pb, counts, baseW, me, nx, ny, po );
    if( rc ) return rc;
    vvb_me_par hp = *me;
    hp.pattern_radius = 0;
    for( int i = 0; anyRefine && i < K; i++ ) hp.pattern_radius = std::max( hp.pattern_radius, std::max( std::abs( (int) pattern[i].dx ), std::abs( (int) pattern[i].dy ) ) );
    for( int l = 0; l < levels; l++ )
    {
      const int n = counts[l], side = baseW << l;
      if( !n ) continue;
      vvb_block* dB = const_cast<vvb_block*>( pb[l] );                               // the start vectors are set in place
      if( ( rc = vvb_blocks_set_start_dev( ctx, dB, po[l], n ) ) ) return rc;
      if( io[l].refine_cost && ( rc = vvb_cost_pattern_dev( ctx, refineDfunc, orgPlane, refPlane, dB, n, side, side, dPattern, K, &hp, cost[l], nullptr ) ) ) return rc;
      if( !io[l].q && !io[l].packed_q ) continue;
      if( ( rc = vvb_fwd_trquant_planes_dev( ctx, &io[l].tu, orgPlane, refPlane, dB, n, nullptr, q[l], sum[l], last[l], nr[l] ) ) ) return rc;
      if( io[l].packed_q && ( rc = vvb_pack_levels_dev( ctx, &io[l].tu, q[l], last[l], n, packed[l], offsets[l] ) ) ) return rc;
    }
    for( int l = 0; l < levels; l++ )
      if( pageable[l] )
      {
        // pageable destination: the size has to come back before the exact copy can be issued
        CU( cudaMemcpyAsync( io[l].packed_offsets, offsets[l], ( (size_t) counts[l] + 1 ) * 4, cudaMemcpyDeviceToHost, ctx->stream ) );
        CU( cudaStreamSynchronize( ctx->stream ) );
        CU( cudaMemcpyAsync( io[l].packed_q, packed[l], (size_t) io[l].packed_offsets[counts[l]] * 2, cudaMemcpyDeviceToHost, ctx->stream ) );
      }
    return VVB_OK;
  } );
}

// ---- dependent quantisation (SURVEY 8f-4) --------------------------------------------------------------------------------------------------------------------
namespace {
int dqTables( vvb_ctx* ctx )
{
  if( ctx->dqShapes ) return VVB_OK;
  // two table sets: luma, then chroma (the context offsets of the next position differ per channel type, DepQuant.cpp:321-330)
  std::vector<vvbdq::DqScanInfo> si, siC; std::vector<vvbdq::DqNbOut> nb, nbC;
  vvbdq::DqShapeTables* shapes = new vvbdq::DqShapeTables[50];
  vvbdq::dq_build_tables( si, nb, shapes, false );
  vvbdq::dq_build_tables( siC, nbC, shapes + 25, true );
  for( int i = 0; i < 25; i++ ) shapes[25 + i].offset += si.size();
  si.insert( si.end(), siC.begin(), siC.end() ); nb.insert( nb.end(), nbC.begin(), nbC.end() );
  if( cudaMalloc( &ctx->d_dqScan, si.size() * sizeof( vvbdq::DqScanInfo ) ) != cudaSuccess || cudaMalloc( &ctx->d_dqNb, nb.size() * sizeof( vvbdq::DqNbOut ) ) != cudaSuccess ||
      cudaMemcpy( ctx->d_dqScan, si.data(), si.size() * sizeof( vvbdq::DqScanInfo ), cudaMemcpyHostToDevice ) != cudaSuccess ||
      cudaMemcpy( ctx->d_dqNb, nb.data(), nb.size() * sizeof( vvbdq::DqNbOut ), cudaMemcpyHostToDevice ) != cudaSuccess )
  {
    delete[] shapes;
    if( ctx->d_dqScan ) { cudaFree( ctx->d_dqScan ); ctx->d_dqScan = nullptr; }
    if( ctx->d_dqNb ) { cudaFree( ctx->d_dqNb ); ctx->d_dqNb = nullptr; }
    return fail( ctx, VVB_ERR_CUDA, "dependent quantisation tables", cudaGetLastError() );
  }
  ctx->dqShapes = shapes;
  return VVB_OK;
}
} // namespace

int vvb_dep_quant_dev( vvb_ctx* ctx, const vvb_tu_par* par, const vvb_dq_par* dq, const vvb_dq_rates* rates, const int32_t* dCoef, const uint8_t* dNeedRdoq, int n,
                       int16_t* dQ, int32_t* dAbsSum, int32_t* dLastPos )
{
  if( !ctx || !par || !dq || !rates || !dCoef || !dQ || n < 0 ) return fail( ctx, VVB_ERR_ARG, "bad arguments" );
  const int shapeIdx = vvbdq::dq_shape_index( par->w, par->h );
  if( shapeIdx < 0 ) return fail( ctx, VVB_ERR_UNSUPPORTED, "TU sides must be 4, 8, 16, 32 or 64" );
  if( par->bit_depth != 8 && par->bit_depth != 10 ) return fail( ctx, VVB_ERR_UNSUPPORTED, "bit depth 8 or 10" );
  if( !( dq->lambda > 0.0 ) ) return fail( ctx, VVB_ERR_ARG, "lambda must be greater than 0 (DepQuant.cpp:535)" );
  if( n == 0 ) return VVB_OK;
  CU( cudaSetDevice( ctx->device ) );
  int rc;
  if( ( rc = dqTables( ctx ) ) ) return rc;
  const vvbdq::DqShapeTables& st = static_cast<vvbdq::DqShapeTables*>( ctx->dqShapes )[shapeIdx + ( par->is_chroma ? 25 : 0 )];
  DqLaunch L = {};
  L.shape.width = st.width; L.shape.height = st.height; L.shape.numCoeff = st.numCoeff; L.shape.numSbb = st.numSbb;
  L.shape.scanInfo = static_cast<vvbdq::DqScanInfo*>( ctx->d_dqScan ) + st.offset;
  L.shape.nbOut    = static_cast<vvbdq::DqNbOut*>( ctx->d_dqNb ) + st.offset;
  L.quant = vvbdq::dq_init_quant( par->w, par->h, par->bit_depth, par->qp + 6 * ( par->bit_depth - 8 ), dq->lambda, dq->dq_thr_val );
  L.zeroOutMts = par->is_chroma ? 0 : dq->zero_out;      // the zero-out of :1155 is a luma rule
  L.lfnst = par->lfnst_idx > 0; L.capSum = dq->scalar_members ? 0 : 1;
  L.ctxBytes  = (uint32_t)( ( 8 * ( st.numSbb + st.numCoeff ) + 15 ) & ~15 );
  L.slotBytes = (uint32_t)( ( L.ctxBytes + (size_t) st.numCoeff * 2 * sizeof( vvbdq::DqTrellis ) + 15 ) & ~(size_t) 15 );
  vvbdq::DqRates r;
  static_assert( sizeof( vvbdq::DqRates ) == sizeof( vvb_dq_rates ), "vvb_dq_rates mirrors DqRates" );
  memcpy( &r, rates, sizeof( r ) );
  void* arena;
  if( ctx->dqEngine == 1 )
  {
    // four lanes per TU, 32 TUs per CTA; beyond a few resident waves the quads stride over the TU list and reuse their arena slot
    const int perCta = VVB_DQQ_THREADS / 4;
    const int blocks = std::min( ( n + perCta - 1 ) / perCta, ctx->numSMs * 16 );
    if( ( rc = scratch( ctx, ScratchArena::Work, (size_t) blocks * perCta * L.slotBytes, &arena ) ) ) return rc;
    dep_quant_quad_kernel<<<blocks, VVB_DQQ_THREADS, 0, ctx->stream>>>( L, r, dCoef, dNeedRdoq, n, dQ, dAbsSum, dLastPos, (uint8_t*) arena );
    CHECK_LAUNCH( "dep_quant_quad_kernel" );
    return VVB_OK;
  }
  // one thread per TU up to a few resident waves; beyond that the threads stride over the TU list and reuse their arena slot
  const int maxBlocks = ctx->numSMs * 8;
  const int blocks = std::min( ( n + VVB_DQ_THREADS - 1 ) / VVB_DQ_THREADS, maxBlocks );
  if( ( rc = scratch( ctx, ScratchArena::Work, (size_t) blocks * VVB_DQ_THREADS * L.slotBytes, &arena ) ) ) return rc;
  dep_quant_kernel<<<blocks, VVB_DQ_THREADS, 0, ctx->stream>>>( L, r, dCoef, dNeedRdoq, n, dQ, dAbsSum, dLastPos, (uint8_t*) arena );
  CHECK_LAUNCH( "dep_quant_kernel" );
  return VVB_OK;
}

int vvb_set_depquant_engine( vvb_ctx* ctx, int engine )
{
  if( !ctx || engine < 0 || engine > 1 ) return VVB_ERR_ARG;
  ctx->dqEngine = engine;
  return VVB_OK;
}

int vvb_dep_quant( vvb_ctx* ctx, const vvb_tu_par* par, const vvb_dq_par* dq, const vvb_dq_rates* rates, const int32_t* coef, const uint8_t* needRdoq, int n,
                   int16_t* q, int32_t* absSum, int32_t* lastPos )
{
  if( !ctx || !par || !coef || !q || n < 0 ) return fail( ctx, VVB_ERR_ARG, "bad arguments" );
  if( n == 0 ) return VVB_OK;
  const size_t samples = (size_t) n * par->w * par->h;
  const int32_t* dC; const uint8_t* dNr; int16_t* dQ; int32_t *dSum, *dLast;
  return HostCall( ctx ).in( dC, coef, samples ).in( dNr, needRdoq, n ).out( dQ, q, samples ).out( dSum, absSum, n, true ).out( dLast, lastPos, n, true )
                        .run( [&] { return vvb_dep_quant_dev( ctx, par, dq, rates, dC, dNr, n, dQ, dSum, dLast ); } );
}

// Quantizer::initQuantBlock as the device call derives it (for bindings / tests that want to inspect the constants): out[9] = qShift, maxQIdx, thresLast, distShift,
// qAdd, qScale, distAdd, distStepAdd, distOrgFact
int vvb_dep_quant_constants( const vvb_tu_par* par, const vvb_dq_par* dq, int64_t out[9] )
{
  if( !par || !dq || !out || vvbdq::dq_shape_index( par->w, par->h ) < 0 || !( dq->lambda > 0.0 ) ) return VVB_ERR_ARG;
  const vvbdq::DqQuant q = vvbdq::dq_init_quant( par->w, par->h, par->bit_depth, par->qp + 6 * ( par->bit_depth - 8 ), dq->lambda, dq->dq_thr_val );
  out[0] = q.qShift; out[1] = q.maxQIdx; out[2] = q.thresLast; out[3] = q.distShift; out[4] = q.qAdd; out[5] = q.qScale; out[6] = q.distAdd; out[7] = q.distStepAdd; out[8] = q.distOrgFact;
  return VVB_OK;
}

// ---- fast RDOQ (SURVEY 8f-4): QuantRDOQ2::xRateDistOptQuantFast, one TU per thread ---------------------------------------------------------------------------
namespace {
int rqPar( vvb_ctx* ctx, const vvb_tu_par* par, const vvb_rdoq_par* rq, vvbrq::RqPar& p )
{
  if( !par || !rq ) return fail( ctx, VVB_ERR_ARG, "null parameters" );
  if( !vvbrq::rq_shape_ok( par->w, par->h ) ) return fail( ctx, VVB_ERR_UNSUPPORTED, "TU sides must be 4, 8, 16, 32 or 64" );
  if( par->bit_depth != 8 && par->bit_depth != 10 ) return fail( ctx, VVB_ERR_UNSUPPORTED, "bit depth 8 or 10" );
  if( par->transform_skip ) return fail( ctx, VVB_ERR_UNSUPPORTED, "transform-skipped TUs go through vvb_rdoq_ts" );
  if( !( rq->lambda > 0.0 ) ) return fail( ctx, VVB_ERR_ARG, "lambda must be greater than 0" );
  if( rq->thr_val < 1 || rq->thr_val > 64 ) return fail( ctx, VVB_ERR_ARG, "thr_val 1..64" );
  p = vvbrq::rq_init_par( par->w, par->h, par->bit_depth, baseQp( par ), par->lfnst_idx > 0, rq->sbt_zero_out, par->sign_hiding, par->is_chroma, rq->lambda, rq->thr_val );
  if( p.qBits < 1 || p.qBits > 30 ) return fail( ctx, VVB_ERR_UNSUPPORTED, "quantiser shift outside 1..30" );
  return VVB_OK;
}
} // namespace

int vvb_rdoq_dev( vvb_ctx* ctx, const vvb_tu_par* par, const vvb_rdoq_par* rq, const vvb_rdoq_rates* rates, const int32_t* dCoef, const uint8_t* dNeedRdoq, int n,
                  int16_t* dQ, int32_t* dAbsSum, int32_t* dLastPos )
{
  if( !ctx || !par || !rq || !rates || !dCoef || !dQ || n < 0 ) return fail( ctx, VVB_ERR_ARG, "bad arguments" );
  RqLaunch L = {};
  int rc = rqPar( ctx, par, rq, L.par );
  if( rc ) return rc;
  if( n == 0 ) return VVB_OK;
  CU( cudaSetDevice( ctx->device ) );
  L.scan = scanOrder( ctx->d_scan, ilog2h( par->w ), ilog2h( par->h ) );
  L.numScan = std::min( 32, par->w ) * std::min( 32, par->h );
  vvbrq::RqRates r;
  static_assert( sizeof( vvbrq::RqRates ) == sizeof( vvb_rdoq_rates ) && sizeof( vvb_rdoq_rates ) == 760, "vvb_rdoq_rates mirrors RqRates" );
  memcpy( &r, rates, sizeof( r ) );
  const int blocks = std::min( ( n + VVB_RQ_THREADS - 1 ) / VVB_RQ_THREADS, ctx->numSMs * 16 );
  if( ctx->rdoqEngine == 2 )
  {
    const vvbrq::RqCost c = vvbrq::rq_init_cost( L.par, r );
    rdoq_v2_kernel<<<blocks, VVB_RQ_THREADS, 0, ctx->stream>>>( L, r, c, dCoef, dNeedRdoq, n, dQ, dAbsSum, dLastPos );
    CHECK_LAUNCH( "rdoq_v2_kernel" );
    return VVB_OK;
  }
  rdoq_kernel<<<blocks, VVB_RQ_THREADS, 0, ctx->stream>>>( L, r, dCoef, dNeedRdoq, n, dQ, dAbsSum, dLastPos );
  CHECK_LAUNCH( "rdoq_kernel" );
  return VVB_OK;
}

int vvb_set_rdoq_engine( vvb_ctx* ctx, int engine )
{
  if( !ctx || engine < 1 || engine > 2 ) return VVB_ERR_ARG;
  ctx->rdoqEngine = engine;
  return VVB_OK;
}

int vvb_rdoq( vvb_ctx* ctx, const vvb_tu_par* par, const vvb_rdoq_par* rq, const vvb_rdoq_rates* rates, const int32_t* coef, const uint8_t* needRdoq, int n,
              int16_t* q, int32_t* absSum, int32_t* lastPos )
{
  if( !ctx || !par || !rq || !rates || !coef || !q || n < 0 ) return fail( ctx, VVB_ERR_ARG, "bad arguments" );
  if( n == 0 ) return VVB_OK;
  const size_t samples = (size_t) n * par->w * par->h;
  const int32_t* dC; const uint8_t* dNr; int16_t* dQ; int32_t *dSum, *dLast;
  return HostCall( ctx ).in( dC, coef, samples ).in( dNr, needRdoq, n ).out( dQ, q, samples ).out( dSum, absSum, n, true ).out( dLast, lastPos, n, true )
                        .run( [&] { return vvb_rdoq_dev( ctx, par, rq, rates, dC, dNr, n, dQ, dSum, dLast ); } );
}

// transform-skipped TUs: QuantRDOQ::rateDistOptQuantTS
int vvb_rdoq_ts_dev( vvb_ctx* ctx, const vvb_tu_par* par, double lambda, const vvb_rdoq_ts_rates* rates, const int32_t* dCoef, const uint8_t* dNeedRdoq, int n, int16_t* dQ, int32_t* dAbsSum )
{
  if( !ctx || !par || !rates || !dCoef || !dQ || n < 0 ) return fail( ctx, VVB_ERR_ARG, "bad arguments" );
  if( !vvbrq::rq_ts_shape_ok( par->w, par->h ) ) return fail( ctx, VVB_ERR_UNSUPPORTED, "transform skip: TU sides 4, 8, 16 or 32" );
  if( par->bit_depth != 8 && par->bit_depth != 10 ) return fail( ctx, VVB_ERR_UNSUPPORTED, "bit depth 8 or 10" );
  if( par->input_bit_depth_delta < 0 || par->input_bit_depth_delta > 8 ) return fail( ctx, VVB_ERR_ARG, "input_bit_depth_delta 0..8" );
  if( !( lambda > 0.0 ) ) return fail( ctx, VVB_ERR_ARG, "lambda must be greater than 0" );
  if( n == 0 ) return VVB_OK;
  CU( cudaSetDevice( ctx->device ) );
  const int qp = std::max( baseQp( par ), 4 + 6 * par->input_bit_depth_delta );                                           // Quant.cpp:117-124: the QP of skipped transforms
  RqTsLaunch L = {};
  L.par = vvbrq::rq_ts_init_par( par->w, par->h, par->bit_depth, qp, lambda );
  L.scan = scanOrder( ctx->d_scan, ilog2h( par->w ), ilog2h( par->h ) );
  L.numScan = par->w * par->h;
  vvbrq::RqTsRates r;
  static_assert( sizeof( vvbrq::RqTsRates ) == sizeof( vvb_rdoq_ts_rates ) && sizeof( vvb_rdoq_ts_rates ) == 176, "vvb_rdoq_ts_rates mirrors RqTsRates" );
  memcpy( &r, rates, sizeof( r ) );
  const int blocks = std::min( ( n + VVB_RQ_THREADS - 1 ) / VVB_RQ_THREADS, ctx->numSMs * 16 );
  rdoq_ts_kernel<<<blocks, VVB_RQ_THREADS, 0, ctx->stream>>>( L, r, dCoef, dNeedRdoq, n, dQ, dAbsSum );
  CHECK_LAUNCH( "rdoq_ts_kernel" );
  return VVB_OK;
}

int vvb_rdoq_ts( vvb_ctx* ctx, const vvb_tu_par* par, double lambda, const vvb_rdoq_ts_rates* rates, const int32_t* coef, const uint8_t* needRdoq, int n, int16_t* q, int32_t* absSum )
{
  if( !ctx || !par || !rates || !coef || !q || n < 0 ) return fail( ctx, VVB_ERR_ARG, "bad arguments" );
  if( n == 0 ) return VVB_OK;
  const size_t samples = (size_t) n * par->w * par->h;
  const int32_t* dC; const uint8_t* dNr; int16_t* dQ; int32_t* dSum;
  return HostCall( ctx ).in( dC, coef, samples ).in( dNr, needRdoq, n ).out( dQ, q, samples ).out( dSum, absSum, n, true )
                        .run( [&] { return vvb_rdoq_ts_dev( ctx, par, lambda, rates, dC, dNr, n, dQ, dSum ); } );
}

// BDPCM TUs: QuantRDOQ::forwardRDPCM
int vvb_rdoq_bdpcm_dev( vvb_ctx* ctx, const vvb_tu_par* par, double lambda, int dirMode, const vvb_rdoq_ts_rates* rates, const int32_t* dCoef, const uint8_t* dNeedRdoq, int n, int16_t* dQ,
                        int32_t* dAbsSum )
{
  if( !ctx || !par || !rates || !dCoef || !dQ || n < 0 ) return fail( ctx, VVB_ERR_ARG, "bad arguments" );
  if( dirMode < 1 || dirMode > 2 ) return fail( ctx, VVB_ERR_ARG, "dir_mode 1 (horizontal) or 2 (vertical)" );
  if( !vvbrq::rq_ts_shape_ok( par->w, par->h ) ) return fail( ctx, VVB_ERR_UNSUPPORTED, "BDPCM: TU sides 4, 8, 16 or 32" );
  if( par->bit_depth != 8 && par->bit_depth != 10 ) return fail( ctx, VVB_ERR_UNSUPPORTED, "bit depth 8 or 10" );
  if( par->input_bit_depth_delta < 0 || par->input_bit_depth_delta > 8 ) return fail( ctx, VVB_ERR_ARG, "input_bit_depth_delta 0..8" );
  if( !( lambda > 0.0 ) ) return fail( ctx, VVB_ERR_ARG, "lambda must be greater than 0" );
  if( n == 0 ) return VVB_OK;
  CU( cudaSetDevice( ctx->device ) );
  const int qp = std::max( baseQp( par ), 4 + 6 * par->input_bit_depth_delta );
  RqTsLaunch L = {};
  L.par = vvbrq::rq_ts_init_par( par->w, par->h, par->bit_depth, qp, lambda );
  const vvbrq::RqBdpcmPar B = vvbrq::rq_bdpcm_init_par( dirMode, qp );
  L.scan = scanOrder( ctx->d_scan, ilog2h( par->w ), ilog2h( par->h ) );
  L.numScan = par->w * par->h;
  vvbrq::RqTsRates r;
  memcpy( &r, rates, sizeof( r ) );
  const int blocks = std::min( ( n + VVB_RQ_THREADS - 1 ) / VVB_RQ_THREADS, ctx->numSMs * 8 );
  void* arena; int rc;
  if( ( rc = scratch( ctx, ScratchArena::Work, (size_t) blocks * VVB_RQ_THREADS * par->w * par->h * sizeof( int32_t ), &arena ) ) ) return rc;
  rdoq_bdpcm_kernel<<<blocks, VVB_RQ_THREADS, 0, ctx->stream>>>( L, B, r, dCoef, dNeedRdoq, n, dQ, dAbsSum, (int32_t*) arena );
  CHECK_LAUNCH( "rdoq_bdpcm_kernel" );
  return VVB_OK;
}

int vvb_rdoq_bdpcm( vvb_ctx* ctx, const vvb_tu_par* par, double lambda, int dirMode, const vvb_rdoq_ts_rates* rates, const int32_t* coef, const uint8_t* needRdoq, int n, int16_t* q,
                    int32_t* absSum )
{
  if( !ctx || !par || !rates || !coef || !q || n < 0 ) return fail( ctx, VVB_ERR_ARG, "bad arguments" );
  if( n == 0 ) return VVB_OK;
  const size_t samples = (size_t) n * par->w * par->h;
  const int32_t* dC; const uint8_t* dNr; int16_t* dQ; int32_t* dSum;
  return HostCall( ctx ).in( dC, coef, samples ).in( dNr, needRdoq, n ).out( dQ, q, samples ).out( dSum, absSum, n, true )
                        .run( [&] { return vvb_rdoq_bdpcm_dev( ctx, par, lambda, dirMode, rates, dC, dNr, n, dQ, dSum ); } );
}

// the per-call constants as the device call derives them (for bindings / tests): quantScale, errScale, qBits, useThres, remRegBins, numCG, firstScanPos
int vvb_rdoq_constants( const vvb_tu_par* par, const vvb_rdoq_par* rq, int32_t out[7] )
{
  if( !par || !rq || !out || !vvbrq::rq_shape_ok( par->w, par->h ) || ( par->bit_depth != 8 && par->bit_depth != 10 ) ) return VVB_ERR_ARG;
  const vvbrq::RqPar p = vvbrq::rq_init_par( par->w, par->h, par->bit_depth, baseQp( par ), par->lfnst_idx > 0, rq->sbt_zero_out, par->sign_hiding, par->is_chroma, rq->lambda, rq->thr_val );
  out[0] = p.quantScale; out[1] = p.errScale; out[2] = p.qBits; out[3] = p.useThres; out[4] = p.remRegBins; out[5] = p.numCG; out[6] = p.firstScanPos;
  return VVB_OK;
}

// ---- inverse path + fused TU round trip ------------------------------------------------------------------------------
int vvb_inv_trquant_dev( vvb_ctx* ctx, const vvb_tu_par* par, const int16_t* dQ, int n, int16_t* dResi )
{
  if( !ctx || !dQ || !dResi || n < 0 ) return fail( ctx, VVB_ERR_ARG, "bad arguments" );
  TuPar p;
  int rc = makeTuPar( ctx, par, p );
  if( rc ) return rc;
  if( n == 0 ) return VVB_OK;
  CU( cudaSetDevice( ctx->device ) );
  if( par->dep_quant && !p.ts )
  {
    // DepQuant::dequant (DepQuant.cpp:1492-1514 -> Quantizer::dequantBlock :574-629): the state machine turns the levels into qIdx values, which the inverse kernel
    // then dequantises with the DepQuant scale and shift at QP + 1 -- the same ( v * scale + add ) >> shift it applies to plain levels; no input clipping there
    const int qp = baseQp( par ) + 1;
    const int per = qp / 6, rem = qp - 6 * per, sqrt2 = ( p.lw + p.lh ) & 1;
    const int trShift = 15 - par->bit_depth - ( ( p.lw + p.lh ) >> 1 ) - sqrt2;
    static const int invScales[2][6] = { { 40, 45, 51, 57, 64, 72 }, { 57, 64, 72, 80, 90, 102 } };
    p.dqScale = invScales[sqrt2][rem]; p.dqShift = 6 + 1 - per - trShift; p.dqInMax = 32767;
    void* dIdx;
    if( ( rc = scratch( ctx, ScratchArena::Work, (size_t) n * p.w * p.h * 2, &dIdx ) ) ) return rc;
    const int lrw = std::min( p.lw, 5 ), nScan = std::min( p.w, 32 ) * std::min( p.h, 32 );
    dq_levels_to_qidx_kernel<<<( n + 3 ) / 4, 128, 0, ctx->stream>>>( dQ, scanOrder( ctx->d_scan, p.lw, p.lh ), p.w, p.h, lrw, nScan, n, (int16_t*) dIdx );
    CHECK_LAUNCH( "dq_levels_to_qidx_kernel" );
    dQ = (const int16_t*) dIdx;
  }
  if( itcEligible( ctx, p, dQ ) && ( ( (uintptr_t) dResi ) & 15 ) == 0 ) return itcLaunch( ctx, p, dQ, n, dResi, 0, 0, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr );
#define VVB_INV_CALL( LWv, LHv ) { using S = TuShape<LWv, LHv>; const size_t smem = inv_trquant_smem<LWv, LHv>(); \
    if( p.lfnstIdx ) inv_trquant_kernel<LWv, LHv, true><<<teamGrid( ctx, n, S::NTEAMS, smem ), 128, smem, ctx->stream>>>( p, ctx->d_trTable, ctx->d_scan, dQ, n, dResi ); \
    else             inv_trquant_kernel<LWv, LHv, false><<<teamGrid( ctx, n, S::NTEAMS, smem ), 128, smem, ctx->stream>>>( p, ctx->d_trTable, ctx->d_scan, dQ, n, dResi ); }
  VVB_TU_DISPATCH( p.lw, p.lh, VVB_INV_CALL )
#undef VVB_INV_CALL
  CHECK_LAUNCH( "inv_trquant_kernel" );
  return VVB_OK;
}

int vvb_inv_trquant( vvb_ctx* ctx, const vvb_tu_par* par, const int16_t* q, int n, int16_t* resi )
{
  if( !ctx || !par || !q || !resi || n < 0 ) return fail( ctx, VVB_ERR_ARG, "bad arguments" );
  if( n == 0 ) return VVB_OK;
  const size_t samples = (size_t) n * par->w * par->h;
  const int16_t* dQ; int16_t* dR;
  return HostCall( ctx ).in( dQ, q, samples ).out( dR, resi, samples ).run( [&] { return vvb_inv_trquant_dev( ctx, par, dQ, n, dR ); } );
}

static_assert( sizeof( vvb_tu_result ) == sizeof( TuResult ) && sizeof( TuResult ) == 32, "vvb_tu_result layout" );

static int tuRoundtripLaunch( vvb_ctx* ctx, const vvb_tu_par* par, int orgPlane, int predPlane, const vvb_block* dBlocks, const int16_t* dOrg, const int16_t* dPred,
                              int n, int16_t* dQ, int16_t* dReco, vvb_tu_result* dRes, uint8_t* dNeedRdoq )
{
  TuPar p;
  int rc = makeTuPar( ctx, par, p );
  if( rc ) return rc;
  if( n == 0 ) return VVB_OK;
  CU( cudaSetDevice( ctx->device ) );
  const Plane po = dBlocks ? ctx->planes.p[orgPlane] : Plane{}, pp = dBlocks ? ctx->planes.p[predPlane] : Plane{};
  const bool ext = p.signHiding != 0 || p.ts != 0 || p.lfnstIdx != 0;
  // square 8..64 TUs with the plain quantiser: the forward half on the tensor-core engine (levels, absSum, lastPos, RDOQ flag), then the inverse half from the levels
  if( tc2Eligible( ctx, p ) && ( dBlocks || ( ( ( (uintptr_t) dOrg | (uintptr_t) dPred ) & 15 ) == 0 ) ) )
  {
    int32_t *dSum, *dLast;
    if( ( rc = carveArena( ctx, ScratchArena::Work, [&]( Layout& L ) { dSum = L.take<int32_t>( n ); dLast = L.take<int32_t>( n ); } ) ) ) return rc;
    if( ( rc = tc2Launch( ctx, p, dBlocks ? nullptr : dOrg, orgPlane, predPlane, dBlocks, n, nullptr, dQ, dSum, dLast, dNeedRdoq, dBlocks ? nullptr : dPred ) ) ) return rc;
    if( itcEligible( ctx, p, dQ ) && ( !dReco || ( ( (uintptr_t) dReco ) & 15 ) == 0 ) )
      return itcLaunch( ctx, p, dQ, n, nullptr, orgPlane, predPlane, dBlocks, dOrg, dPred, dReco, (TuResult*) dRes, dSum, dLast );
#define VVB_RTQ_CALL( LWv, LHv ) { using S = TuShape<LWv, LHv>; const size_t smem = tu_roundtrip_smem<LWv, LHv>(); \
      tu_roundtrip_kernel<LWv, LHv, false, true><<<teamGrid( ctx, n, S::NTEAMS, smem ), 128, smem, ctx->stream>>>( p, ctx->d_trTable, ctx->d_scan, dBlocks ? 1 : 0, po, pp, dBlocks, dOrg, dPred, n, \
                                                                                              dQ, dReco, (TuResult*) dRes, dNeedRdoq, dSum, dLast ); }
    switch( p.lw ) { case 3: VVB_RTQ_CALL( 3, 3 ) break; case 4: VVB_RTQ_CALL( 4, 4 ) break; case 5: VVB_RTQ_CALL( 5, 5 ) break; default: VVB_RTQ_CALL( 6, 6 ) break; }
#undef VVB_RTQ_CALL
    CHECK_LAUNCH( "tu_roundtrip_kernel (from levels)" );
    return VVB_OK;
  }
#define VVB_RT_CALL( LWv, LHv ) { using S = TuShape<LWv, LHv>; const size_t smem = tu_roundtrip_smem<LWv, LHv>(); \
    if( ext ) tu_roundtrip_kernel<LWv, LHv, true><<<teamGrid( ctx, n, S::NTEAMS, smem ), 128, smem, ctx->stream>>>( p, ctx->d_trTable, ctx->d_scan, dBlocks ? 1 : 0, po, pp, dBlocks, dOrg, dPred, n, \
                                                                                              dQ, dReco, (TuResult*) dRes, dNeedRdoq ); \
    else      tu_roundtrip_kernel<LWv, LHv, false><<<teamGrid( ctx, n, S::NTEAMS, smem ), 128, smem, ctx->stream>>>( p, ctx->d_trTable, ctx->d_scan, dBlocks ? 1 : 0, po, pp, dBlocks, dOrg, dPred, n, \
                                                                                              dQ, dReco, (TuResult*) dRes, dNeedRdoq ); }
  VVB_TU_DISPATCH( p.lw, p.lh, VVB_RT_CALL )
#undef VVB_RT_CALL
  CHECK_LAUNCH( "tu_roundtrip_kernel" );
  return VVB_OK;
}

int vvb_tu_roundtrip_dev( vvb_ctx* ctx, const vvb_tu_par* par, const int16_t* dOrg, const int16_t* dPred, int n, int16_t* dQ, int16_t* dReco, vvb_tu_result* dRes, uint8_t* dNeedRdoq )
{
  if( !ctx || !dOrg || !dPred || !dQ || !dRes || n < 0 ) return fail( ctx, VVB_ERR_ARG, "bad arguments" );
  return tuRoundtripLaunch( ctx, par, -1, -1, nullptr, dOrg, dPred, n, dQ, dReco, dRes, dNeedRdoq );
}

int vvb_tu_roundtrip_planes_dev( vvb_ctx* ctx, const vvb_tu_par* par, int orgPlane, int predPlane, const vvb_block* dBlocks, int n,
                                 int16_t* dQ, int16_t* dReco, vvb_tu_result* dRes, uint8_t* dNeedRdoq )
{
  if( !ctx || !dBlocks || !dQ || !dRes || n < 0 ) return fail( ctx, VVB_ERR_ARG, "bad arguments" );
  if( !validPlane( ctx, orgPlane ) || !validPlane( ctx, predPlane ) ) return fail( ctx, VVB_ERR_ARG, "unknown plane" );
  return tuRoundtripLaunch( ctx, par, orgPlane, predPlane, dBlocks, nullptr, nullptr, n, dQ, dReco, dRes, dNeedRdoq );
}

int vvb_tu_roundtrip( vvb_ctx* ctx, const vvb_tu_par* par, const int16_t* org, const int16_t* pred, int n, int16_t* q, int16_t* reco, vvb_tu_result* res, uint8_t* needRdoq )
{
  if( !ctx || !par || !org || !pred || !q || !res || n < 0 ) return fail( ctx, VVB_ERR_ARG, "bad arguments" );
  if( n == 0 ) return VVB_OK;
  const size_t samples = (size_t) n * par->w * par->h;
  const int16_t *dO, *dP; int16_t *dQ, *dR; vvb_tu_result* dRes; uint8_t* dNr;
  return HostCall( ctx ).in( dO, org, samples ).in( dP, pred, samples ).out( dQ, q, samples ).out( dR, reco, samples ).out( dRes, res, n ).out( dNr, needRdoq, n, true )
                        .run( [&] { return vvb_tu_roundtrip_dev( ctx, par, dO, dP, n, dQ, dR, dRes, dNr ); } );
}

// ---- MCTF ----------------------------------------------------------------------------------------------------------
static int mctfLaunch( vvb_ctx* ctx, const Plane& po, const Plane& pr, const vvb_mctf_cand* dCands, int n, int lowRes, int maxDim, int32_t* dErr )
{
  CU( cudaSetDevice( ctx->device ) );
  maxDim = std::max( 8, std::min( 64, ( maxDim + 7 ) & ~7 ) );
  const MctfSmem L = mctf_smem( maxDim );
  const size_t smem = (size_t) MCTF_WARPS * L.warpWords * 4;
  const int perSM = (int) std::max<size_t>( 1, std::min<size_t>( 12, ( 220 * 1024 ) / ( smem + 1024 ) ) );
  const int grid = std::min( ( n + MCTF_WARPS - 1 ) / MCTF_WARPS, ctx->numSMs * perSM );
  mctf_error_packed_kernel<<<grid, MCTF_WARPS * 32, smem, ctx->stream>>>( po, pr, dCands, n, lowRes ? 1 : 0, maxDim, dErr );
  CHECK_LAUNCH( "mctf_error_packed_kernel" );
  return VVB_OK;
}

// the MCTF filters and errors are defined up to 10 bits (MCTF.cpp:1313 CHECKD; 64 x 64 SSEs above it leave 32 bits): the wider of the two planes decides
static int mctfBitDepthOk( vvb_ctx* ctx, int orgPlane, int refPlane )
{
  if( std::max( ctx->planes.p[orgPlane].bitDepth, ctx->planes.p[refPlane].bitDepth ) > 10 ) return fail( ctx, VVB_ERR_UNSUPPORTED, "MCTF supports up to 10 bit (MCTF.cpp:1313 CHECKD)" );
  return VVB_OK;
}

int vvb_mctf_hint( vvb_ctx* ctx, int maxBlockDim )
{
  if( !ctx || maxBlockDim < 8 || maxBlockDim > 64 ) return fail( ctx, VVB_ERR_ARG, "MCTF block dimension hint must be 8..64" );
  ctx->mctfMaxDim = maxBlockDim;
  return VVB_OK;
}

int vvb_mctf_error_batch_dev( vvb_ctx* ctx, int orgPlane, int refPlane, const vvb_mctf_cand* dCands, int n, int lowRes, int32_t* dErr )
{
  if( !ctx || !dCands || !dErr || n < 0 ) return fail( ctx, VVB_ERR_ARG, "bad arguments" );
  if( !validPlane( ctx, orgPlane ) || !validPlane( ctx, refPlane ) ) return fail( ctx, VVB_ERR_ARG, "unknown plane" );
  if( int rc = mctfBitDepthOk( ctx, orgPlane, refPlane ) ) return rc;
  if( n == 0 ) return VVB_OK;
  return mctfLaunch( ctx, ctx->planes.p[orgPlane], ctx->planes.p[refPlane], dCands, n, lowRes, ctx->mctfMaxDim, dErr );
}

int vvb_mctf_error_batch( vvb_ctx* ctx, int orgPlane, int refPlane, const vvb_mctf_cand* cands, int n, int lowRes, int32_t* err )
{
  if( !ctx || !cands || !err || n < 0 ) return fail( ctx, VVB_ERR_ARG, "bad arguments" );
  for( int i = 0; i < n; i++ )
    if( cands[i].w < 8 || cands[i].h < 8 || cands[i].w > 64 || cands[i].h > 64 || ( cands[i].w & 7 ) || ( cands[i].h & 7 ) )
      return fail( ctx, VVB_ERR_UNSUPPORTED, "MCTF blocks are multiples of 8 up to 64 (MCTF.cpp:1113-1118)" );
  if( n == 0 ) return VVB_OK;
  if( !validPlane( ctx, orgPlane ) || !validPlane( ctx, refPlane ) ) return fail( ctx, VVB_ERR_ARG, "unknown plane" );
  if( int rc = mctfBitDepthOk( ctx, orgPlane, refPlane ) ) return rc;
  int maxDim = 8;
  for( int i = 0; i < n; i++ ) maxDim = std::max( maxDim, (int) std::max( cands[i].w, cands[i].h ) );
  const vvb_mctf_cand* dC; int32_t* dE;
  return HostCall( ctx ).in( dC, cands, n ).out( dE, err, n )
                        .run( [&] { return mctfLaunch( ctx, ctx->planes.p[orgPlane], ctx->planes.p[refPlane], dC, n, lowRes, maxDim, dE ); } );
}

// ---- fractional-pel refinement grid (xPatternRefinement's filtered blocks + distFunc) -----------------------------------------------
static int fracGridArgs( vvb_ctx* ctx, int dfunc, int orgPlane, int refPlane, int n, int w, int h )
{
  if( n < 0 ) return fail( ctx, VVB_ERR_ARG, "bad arguments" );
  if( !validPlane( ctx, orgPlane ) || !validPlane( ctx, refPlane ) ) return fail( ctx, VVB_ERR_ARG, "unknown plane" );
  if( dfunc != VVB_DF_SAD && dfunc != VVB_DF_HAD && dfunc != VVB_DF_HAD_FAST ) return fail( ctx, VVB_ERR_UNSUPPORTED, "fractional grid: SAD, HAD or HAD_fast" );
  if( !isPow2( w ) || !isPow2( h ) || w < 4 || h < 4 || w > 64 || h > 64 ) return fail( ctx, VVB_ERR_UNSUPPORTED, "fractional grid: PU sides 4..64, powers of two" );
  if( ctx->planes.p[refPlane].bitDepth > 12 ) return fail( ctx, VVB_ERR_UNSUPPORTED, "bit depth above 12" );
  return VVB_OK;
}

int vvb_frac_cost_grid_dev( vvb_ctx* ctx, int dfunc, int orgPlane, int refPlane, const vvb_block* dBlocks, int n, int w, int h, int reduceTap, int altHpel, uint32_t* dCost )
{
  if( !ctx || !dBlocks || !dCost ) return fail( ctx, VVB_ERR_ARG, "bad arguments" );
  int rc = fracGridArgs( ctx, dfunc, orgPlane, refPlane, n, w, h );
  if( rc ) return rc;
  if( reduceTap < 0 || reduceTap > 2 ) return fail( ctx, VVB_ERR_ARG, "reduce_tap is 0, 1 or 2 (ReduceFilterME, vvencCfg.cpp:2058)" );
  if( n == 0 ) return VVB_OK;
  CU( cudaSetDevice( ctx->device ) );
  const FracFilter flt = frac_filter( reduceTap, altHpel );
  // square blocks of 8 and more whose SATD lands on 8x8 tiles (and their SAD) take the register-tile kernel; every other shape of xPatternRefinement -- rectangular
  // PUs, 4-pel sides, DF_HAD_fast on multiples of 32 -- the generic one
  const bool fast16 = dfunc == VVB_DF_HAD_FAST && w == h && ( w & 31 ) == 0;
  if( w != h || w < 8 || fast16 )
  {
    const FracGenSmem G = frac_gen_smem( w, h );
    if( (size_t) G.total * 4 > 100 * 1024 ) return fail( ctx, VVB_ERR_UNSUPPORTED, "fractional grid: block too large for shared memory" );
    frac_grid_generic_kernel<<<std::min( n, ctx->numSMs * 16 ), 128, (size_t) G.total * 4, ctx->stream>>>( ctx->planes.p[orgPlane], ctx->planes.p[refPlane], dBlocks, n, w, h,
                                                                                                       dfunc == VVB_DF_SAD ? 1 : ( fast16 ? 3 : 2 ), flt, dCost );
    CHECK_LAUNCH( "frac_grid_generic_kernel" );
    return VVB_OK;
  }
  const FracSmem L = frac_smem( w, h );
  const int jobs = L.G * 7 * ( w / 8 ) * ( h / 8 );                                   // (horizontal offsets per pass) x vertical offsets x tiles
  const int threads = std::max( 32, std::min( 128, ( jobs + 31 ) & ~31 ) );
  frac_grid_kernel<<<std::min( n, ctx->numSMs * 32 ), threads, (size_t) L.total * 4, ctx->stream>>>( ctx->planes.p[orgPlane], ctx->planes.p[refPlane], dBlocks, n, w, h,
                                                                                                  dfunc == VVB_DF_SAD ? 1 : 2, flt, dCost );
  CHECK_LAUNCH( "frac_grid_kernel" );
  return VVB_OK;
}

int vvb_frac_cost_grid( vvb_ctx* ctx, int dfunc, int orgPlane, int refPlane, const vvb_block* blocks, int n, int w, int h, int reduceTap, int altHpel, uint32_t* cost )
{
  if( !ctx || !blocks || !cost ) return fail( ctx, VVB_ERR_ARG, "bad arguments" );
  int rc = fracGridArgs( ctx, dfunc, orgPlane, refPlane, n, w, h );
  if( rc || n == 0 ) return rc;
  const vvb_block* dB; uint32_t* dC;
  return HostCall( ctx ).in( dB, blocks, n ).out( dC, cost, (size_t) n * 49 )
                        .run( [&] { return vvb_frac_cost_grid_dev( ctx, dfunc, orgPlane, refPlane, dB, n, w, h, reduceTap, altHpel, dC ); } );
}

// ---- MCTF apply stage (xFinalizeBlkLine body per block) ---------------------------------------------------------------------
static_assert( sizeof( vvb_mctf_mv ) == 16, "vvb_mctf_mv layout" );

static int mctfApplyPar( vvb_ctx* ctx, int orgPlane, const vvb_mctf_apply_par* in, MctfApplyPar& p, int& nBlocks )
{
  if( !in ) return fail( ctx, VVB_ERR_ARG, "null apply parameters" );
  if( !validPlane( ctx, orgPlane ) ) return fail( ctx, VVB_ERR_ARG, "unknown plane" );
  if( in->num_refs < 1 || in->num_refs > 8 ) return fail( ctx, VVB_ERR_ARG, "1..8 reference pictures (2 * VVENC_MCTF_RANGE, MCTF.cpp:430)" );
  if( in->block_size != 4 && in->block_size != 8 && in->block_size != 16 && in->block_size != 32 ) return fail( ctx, VVB_ERR_UNSUPPORTED, "MCTF unit size 4 (chroma of unit 8), 8, 16 or 32" );
  const Plane& o = ctx->planes.p[orgPlane];
  // trailing partial units (h = min(blkSizeY, height - by), MCTF.cpp:1427-1431) are filtered like full ones; the packed two-pass filter walks pel / row pairs
  if( ( o.width & 1 ) || ( o.height & 1 ) ) return fail( ctx, VVB_ERR_UNSUPPORTED, "picture dimensions must be even" );
  if( o.bitDepth > 10 ) return fail( ctx, VVB_ERR_UNSUPPORTED, "MCTF supports up to 10 bit (MCTF.cpp:1313 CHECKD)" );
  memset( &p, 0, sizeof( p ) );
  p.numRefs = in->num_refs; p.blockSize = in->block_size; p.tap4 = in->low_res_filter ? 1 : 0; p.planar = in->planar_correction ? 1 : 0;
  p.width = o.width; p.height = o.height; p.blocksX = ( o.width + in->block_size - 1 ) / in->block_size; p.bitDepth = o.bitDepth; p.orgPlane = orgPlane;
  p.weightScaling = in->weight_scaling; p.sigmaSq = in->sigma_sq;
  for( int i = 0; i < in->num_refs; i++ )
  {
    if( !validPlane( ctx, in->ref_plane[i] ) ) return fail( ctx, VVB_ERR_ARG, "unknown reference plane" );
    p.refPlane[i] = in->ref_plane[i]; p.refStrength[i] = in->ref_strength[i];
  }
  nBlocks = p.blocksX * ( ( o.height + in->block_size - 1 ) / in->block_size );
  return VVB_OK;
}

int vvb_mctf_apply_dev( vvb_ctx* ctx, int orgPlane, const vvb_mctf_apply_par* par, const vvb_mctf_mv* dMvs, int16_t* dOut, int outStride )
{
  if( !ctx || !dMvs || !dOut ) return fail( ctx, VVB_ERR_ARG, "bad arguments" );
  MctfApplyPar p; int nBlocks = 0;
  int rc = mctfApplyPar( ctx, orgPlane, par, p, nBlocks );
  if( rc ) return rc;
  if( outStride < p.width ) return fail( ctx, VVB_ERR_ARG, "output stride below the picture width" );
  p.outStride = outStride;
  CU( cudaSetDevice( ctx->device ) );
  const MctfApplySmem L = mctf_apply_smem( p.blockSize, p.numRefs );
  const size_t smem = (size_t) L.total * 4;
  const int threads = std::max( 32, std::min( 256, ( ( p.blockSize / 2 ) * p.blockSize + 31 ) & ~31 ) );
  mctf_apply_kernel<<<std::min( nBlocks, ctx->numSMs * 16 ), threads, smem, ctx->stream>>>( ctx->planes, p, (const int4*) dMvs, nBlocks, dOut );
  CHECK_LAUNCH( "mctf_apply_kernel" );
  return VVB_OK;
}

int vvb_mctf_apply( vvb_ctx* ctx, int orgPlane, const vvb_mctf_apply_par* par, const vvb_mctf_mv* mvs, int16_t* out, int outStride )
{
  if( !ctx || !mvs || !out ) return fail( ctx, VVB_ERR_ARG, "bad arguments" );
  MctfApplyPar p; int nBlocks = 0;
  int rc = mctfApplyPar( ctx, orgPlane, par, p, nBlocks );
  if( rc ) return rc;
  if( outStride < p.width ) return fail( ctx, VVB_ERR_ARG, "output stride below the picture width" );
  const vvb_mctf_mv* dM; int16_t* dO;
  return HostCall( ctx ).in( dM, mvs, (size_t) p.numRefs * nBlocks ).tmp( dO, (size_t) p.width * p.height ).run( [&]
  {
    const int r = vvb_mctf_apply_dev( ctx, orgPlane, par, dM, dO, p.width );
    if( r ) return r;
    CU( cudaMemcpy2DAsync( out, (size_t) outStride * 2, dO, (size_t) p.width * 2, (size_t) p.width * 2, p.height, cudaMemcpyDeviceToHost, ctx->stream ) );
    return VVB_OK;
  } );
}

int vvb_mctf_calc_var_dev( vvb_ctx* ctx, int plane, const vvb_mctf_cand* dBlocks, int n, double* dVar )
{
  if( !ctx || !dBlocks || !dVar || n < 0 ) return fail( ctx, VVB_ERR_ARG, "bad arguments" );
  if( !validPlane( ctx, plane ) ) return fail( ctx, VVB_ERR_ARG, "unknown plane" );
  if( int rc = mctfBitDepthOk( ctx, plane, plane ) ) return rc;
  if( n == 0 ) return VVB_OK;
  CU( cudaSetDevice( ctx->device ) );
  mctf_calc_var_kernel<<<( n + 3 ) / 4, 128, 0, ctx->stream>>>( ctx->planes.p[plane], dBlocks, n, dVar );
  CHECK_LAUNCH( "mctf_calc_var_kernel" );
  return VVB_OK;
}

int vvb_mctf_calc_var( vvb_ctx* ctx, int plane, const vvb_mctf_cand* blocks, int n, double* var )
{
  if( !ctx || !blocks || !var || n < 0 ) return fail( ctx, VVB_ERR_ARG, "bad arguments" );
  if( n == 0 ) return VVB_OK;
  const vvb_mctf_cand* dB; double* dV;
  return HostCall( ctx ).in( dB, blocks, n ).out( dV, var, n ).run( [&] { return vvb_mctf_calc_var_dev( ctx, plane, dB, n, dV ); } );
}

// MCTF grid search: all (2r+1)^2 candidates around each block's centre vector in one CTA (estimateLumaLn loops, MCTF.cpp:1218-1287)
static int mctfGridLaunch( vvb_ctx* ctx, const Plane& po, const Plane& pr, const vvb_mctf_cand* dBlocks, int n, int step, int radius, int lowRes, int maxDim, int32_t* dErr )
{
  CU( cudaSetDevice( ctx->device ) );
  maxDim = std::max( 8, std::min( 64, ( maxDim + 7 ) & ~7 ) );
  const MctfGridSmem L = mctf_grid_smem( maxDim, step, radius );
  const size_t smem = (size_t) L.total * 4;
  if( smem > 200 * 1024 ) return fail( ctx, VVB_ERR_UNSUPPORTED, "MCTF grid too large for shared memory" );
  const int threads = std::max( 32, std::min( 256, ( ( maxDim / 2 ) * maxDim + 31 ) & ~31 ) );
  mctf_grid_kernel<<<std::min( n, ctx->numSMs * 32 ), threads, smem, ctx->stream>>>( po, pr, dBlocks, n, step, radius, lowRes ? 1 : 0, maxDim, dErr );
  CHECK_LAUNCH( "mctf_grid_kernel" );
  return VVB_OK;
}

static int mctfGridArgs( vvb_ctx* ctx, int orgPlane, int refPlane, int n, int step, int radius )
{
  if( n < 0 || step < 1 || step > 16 || radius < 0 || radius > 8 ) return fail( ctx, VVB_ERR_ARG, "MCTF grid: step 1..16 (1/16 pel), radius 0..8 steps" );
  if( !validPlane( ctx, orgPlane ) || !validPlane( ctx, refPlane ) ) return fail( ctx, VVB_ERR_ARG, "unknown plane" );
  return mctfBitDepthOk( ctx, orgPlane, refPlane );
}

int vvb_mctf_search_grid_dev( vvb_ctx* ctx, int orgPlane, int refPlane, const vvb_mctf_cand* dBlocks, int n, int step, int radius, int lowRes, int32_t* dErr )
{
  if( !ctx || !dBlocks || !dErr ) return fail( ctx, VVB_ERR_ARG, "bad arguments" );
  int rc = mctfGridArgs( ctx, orgPlane, refPlane, n, step, radius );
  if( rc || n == 0 ) return rc;
  return mctfGridLaunch( ctx, ctx->planes.p[orgPlane], ctx->planes.p[refPlane], dBlocks, n, step, radius, lowRes, ctx->mctfMaxDim, dErr );
}

int vvb_mctf_search_grid( vvb_ctx* ctx, int orgPlane, int refPlane, const vvb_mctf_cand* blocks, int n, int step, int radius, int lowRes, int32_t* err )
{
  if( !ctx || !blocks || !err ) return fail( ctx, VVB_ERR_ARG, "bad arguments" );
  int rc = mctfGridArgs( ctx, orgPlane, refPlane, n, step, radius );
  if( rc || n == 0 ) return rc;
  int maxDim = 8;
  for( int i = 0; i < n; i++ )
  {
    if( blocks[i].w < 8 || blocks[i].h < 8 || blocks[i].w > 64 || blocks[i].h > 64 || ( blocks[i].w & 7 ) || ( blocks[i].h & 7 ) )
      return fail( ctx, VVB_ERR_UNSUPPORTED, "MCTF blocks are multiples of 8 up to 64 (MCTF.cpp:1113-1118)" );
    maxDim = std::max( maxDim, (int) std::max( blocks[i].w, blocks[i].h ) );
  }
  const size_t K = (size_t)( 2 * radius + 1 ) * ( 2 * radius + 1 );
  const vvb_mctf_cand* dB; int32_t* dE;
  return HostCall( ctx ).in( dB, blocks, n ).out( dE, err, n * K )
                        .run( [&] { return mctfGridLaunch( ctx, ctx->planes.p[orgPlane], ctx->planes.p[refPlane], dB, n, step, radius, lowRes, maxDim, dE ); } );
}

// ---- MCTF motion search with the control on the device (MCTF::motionEstimationMCTF, MCTF.cpp:666-724 -> motionEstimationLuma :1329-1397) ---------------------------
namespace {
struct MctfArena { MctfBest* best; int2* centre; vvb_mctf_cand* cands; int32_t* err; double* var; int* progress; };

// the temporaries of mctfLevel for up to n blocks in byn block rows
MctfArena mctfCarve( Layout& L, int n, int byn )
{
  MctfArena a;
  a.best = L.take<MctfBest>( n ); a.centre = L.take<int2>( n ); a.cands = L.take<vvb_mctf_cand>( (size_t) n * 10 );
  a.err = L.take<int32_t>( (size_t) n * 289 ); a.var = L.take<double>( n ); a.progress = L.take<int>( byn + 2 );
  return a;
}

// offsets off0 + k * delta (k < count) -> the smallest lattice the grid kernel can evaluate that contains them (step <= 16): vvenc_b200/mctf_host.py _offset_table
struct MctfOffs { int off0, delta, count, step, radius, shift; };
MctfOffs mctfOffsets( int first, int last, int delta )
{
  MctfOffs o; o.off0 = first; o.delta = delta; o.count = ( last - first ) / delta + 1;
  if( o.count == 1 ) { o.delta = 16; o.step = 16; o.radius = 0; o.shift = first; return o; }
  o.step = delta;
  while( o.step > 16 ) o.step /= 2;
  o.radius = ( ( last - first ) + 2 * o.step - 1 ) / ( 2 * o.step );
  o.shift = first + o.radius * o.step;
  return o;
}

// one level for the whole picture; every stage is enqueued on the context stream, nothing returns to the host
int mctfLevel( vvb_ctx* ctx, const Plane& po, const Plane& pr, int width, int height, int bs, const vvb_mctf_mv* dPrev, int prevW, int prevH, int factor, bool doubleRes,
               int bitDepth, int searchPattern, int lowRes, vvb_mctf_mv* dOut, int outW, int outH, const MctfArena& a )
{
  MctfGeom g;
  g.width = width; g.height = height; g.bs = bs;
  g.bxn = width >= 8 ? ( width - 8 ) / bs + 1 : 0; g.byn = height >= 8 ? ( height - 8 ) / bs + 1 : 0; g.n = g.bxn * g.byn;
  g.prevW = dPrev ? prevW : 0; g.prevH = dPrev ? prevH : 0; g.factor = factor; g.outW = outW; g.outH = outH;
  CU( cudaMemsetAsync( dOut, 0, (size_t) outW * outH * sizeof( vvb_mctf_mv ), ctx->stream ) );
  if( g.n == 0 ) return VVB_OK;
  const int T = 128, nb = ( g.n + T - 1 ) / T;
  int rc;
  mctf_init_kernel<<<( std::max( g.n, g.byn + 1 ) + T - 1 ) / T, T, 0, ctx->stream>>>( g, a.best, a.progress );
  CHECK_LAUNCH( "mctf_init_kernel" );
  int searchRange = 8;
  if( dPrev )
  {
    searchRange = doubleRes ? 0 : ( searchPattern == 2 ? 3 : 5 );
    mctf_pred_cands_kernel<<<( g.n * 10 + T - 1 ) / T, T, 0, ctx->stream>>>( g, dPrev, a.cands );
    CHECK_LAUNCH( "mctf_pred_cands_kernel" );
    if( ( rc = mctfLaunch( ctx, po, pr, a.cands, g.n * 10, lowRes, bs, a.err ) ) ) return rc;
    mctf_select_list_kernel<<<nb, T, 0, ctx->stream>>>( g, a.cands, a.err, a.best );
    CHECK_LAUNCH( "mctf_select_list_kernel" );
  }
  auto gridStage = [&]( const MctfOffs& o, int truncInt, int skipZero ) -> int
  {
    mctf_centre_kernel<<<nb, T, 0, ctx->stream>>>( g, a.best, truncInt, o.shift, a.centre, a.cands );
    CHECK_LAUNCH( "mctf_centre_kernel" );
    if( truncInt && o.step == 16 && ( o.shift & 15 ) == 0 )
    {
      // stage B: every candidate sits on the integer grid -> the SSE-only grid kernel
      const int maxDim = std::max( 8, std::min( 64, ( bs + 7 ) & ~7 ) );
      const MctfIntSmem LI = mctf_int_smem( maxDim, o.radius );
      mctf_int_grid_kernel<<<std::min( g.n, ctx->numSMs * 16 ), 128, (size_t) LI.total * 4, ctx->stream>>>( po, pr, a.cands, g.n, o.radius, maxDim, a.err );
      CHECK_LAUNCH( "mctf_int_grid_kernel" );
    }
    else
    {
      int r = mctfGridLaunch( ctx, po, pr, a.cands, g.n, o.step, o.radius, lowRes, bs, a.err );
      if( r ) return r;
    }
    mctf_select_grid_kernel<<<nb, T, 0, ctx->stream>>>( g, a.err, 2 * o.radius + 1, o.off0, o.delta, o.count, o.step, skipZero, a.centre, a.best );
    CHECK_LAUNCH( "mctf_select_grid_kernel" );
    return VVB_OK;
  };
  const int d = ( !dPrev && searchPattern == 2 ) ? 2 : 1;                                                     // :1217
  if( ( rc = gridStage( mctfOffsets( -16 * searchRange, -16 * searchRange + 16 * d * ( 2 * searchRange / d ), 16 * d ), 1, 0 ) ) ) return rc;
  if( doubleRes )
  {
    const int rng = searchPattern == 0 ? 12 : 6, d1 = searchPattern == 2 ? 6 : 4;
    if( ( rc = gridStage( mctfOffsets( -rng, -rng + d1 * ( 2 * rng / d1 ), d1 ), 0, 1 ) ) ) return rc;
    if( ( rc = gridStage( mctfOffsets( -2, 2, 2 ), 0, 1 ) ) ) return rc;
    if( ( rc = gridStage( mctfOffsets( -1, 1, 1 ), 0, 1 ) ) ) return rc;
  }
  {
    const int maxDim = std::max( 8, std::min( 64, ( bs + 7 ) & ~7 ) );
    const MctfSmem L = mctf_wave_smem( maxDim );
    mctf_wave_kernel<<<g.byn, MCTF_WAVE_WARPS * 32, (size_t) MCTF_WAVE_WARPS * L.warpWords * 4, ctx->stream>>>( po, pr, g, lowRes ? 1 : 0, maxDim, a.best, a.progress );
    CHECK_LAUNCH( "mctf_wave_kernel" );
  }
  if( doubleRes )
  {
    mctf_centre_kernel<<<nb, T, 0, ctx->stream>>>( g, a.best, 0, 0, a.centre, a.cands );                      // the block list (x, y, w, h) for calcVar
    CHECK_LAUNCH( "mctf_centre_kernel" );
    mctf_calc_var_kernel<<<( g.n + 3 ) / 4, 128, 0, ctx->stream>>>( po, a.cands, g.n, a.var );
    CHECK_LAUNCH( "mctf_calc_var_kernel" );
  }
  mctf_final_kernel<<<nb, T, 0, ctx->stream>>>( g, a.best, a.var, doubleRes ? 1 : 0, bitDepth, dOut );
  CHECK_LAUNCH( "mctf_final_kernel" );
  return VVB_OK;
}
} // namespace

int vvb_mctf_estimate_level_dev( vvb_ctx* ctx, int orgPlane, int refPlane, const vvb_mctf_level_par* lp, const vvb_mctf_mv* dPrev, vvb_mctf_mv* dOut )
{
  if( !ctx || !lp || !dOut ) return fail( ctx, VVB_ERR_ARG, "bad arguments" );
  if( !validPlane( ctx, orgPlane ) || !validPlane( ctx, refPlane ) ) return fail( ctx, VVB_ERR_ARG, "unknown plane" );
  if( ( lp->block_size != 8 && lp->block_size != 16 && lp->block_size != 32 && lp->block_size != 64 ) || lp->search_pattern < 0 || lp->search_pattern > 2 || lp->out_w < 1 || lp->out_h < 1 )
    return fail( ctx, VVB_ERR_ARG, "bad level parameters" );
  if( int rc = mctfBitDepthOk( ctx, orgPlane, refPlane ) ) return rc;
  const Plane& po = ctx->planes.p[orgPlane];
  CU( cudaSetDevice( ctx->device ) );
  const int bxn = ( po.width - 8 ) / lp->block_size + 1, byn = ( po.height - 8 ) / lp->block_size + 1;
  MctfArena a;
  const int rc = carveArena( ctx, ScratchArena::Work, [&]( Layout& L ) { a = mctfCarve( L, std::max( 1, bxn * byn ), byn ); } );
  if( rc ) return rc;
  return mctfLevel( ctx, po, ctx->planes.p[refPlane], po.width, po.height, lp->block_size, dPrev, lp->prev_w, lp->prev_h, lp->factor, lp->double_res != 0, po.bitDepth,
                    lp->search_pattern, lp->low_res_filter, dOut, lp->out_w, lp->out_h, a );
}

int vvb_mctf_estimate_level( vvb_ctx* ctx, int orgPlane, int refPlane, const vvb_mctf_level_par* lp, const vvb_mctf_mv* prev, vvb_mctf_mv* out )
{
  if( !ctx || !lp || !out ) return fail( ctx, VVB_ERR_ARG, "bad arguments" );
  const vvb_mctf_mv* dPrev; vvb_mctf_mv* dOut;
  return HostCall( ctx ).in( dPrev, prev, (size_t) lp->prev_w * lp->prev_h ).out( dOut, out, (size_t) lp->out_w * lp->out_h )
                        .run( [&] { return vvb_mctf_estimate_level_dev( ctx, orgPlane, refPlane, lp, dPrev, dOut ); } );
}

// whole pyramid of one neighbour picture: the subsampled pictures (MCTF::subsampleLuma, border replication 128) are produced into context-owned memory, the four
// (five with add_level) levels chain through device-resident fields; the final field has ceil(W / unit) x ceil(H / unit) entries
int vvb_mctf_estimate_pyramid_dev( vvb_ctx* ctx, int orgPlane, int refPlane, const vvb_mctf_pyr_par* pp, vvb_mctf_mv* dOut )
{
  if( !ctx || !pp || !dOut ) return fail( ctx, VVB_ERR_ARG, "bad arguments" );
  if( !validPlane( ctx, orgPlane ) || !validPlane( ctx, refPlane ) ) return fail( ctx, VVB_ERR_ARG, "unknown plane" );
  if( ( pp->unit_size != 8 && pp->unit_size != 16 && pp->unit_size != 32 ) || pp->search_pattern < 0 || pp->search_pattern > 2 ) return fail( ctx, VVB_ERR_ARG, "bad pyramid parameters" );
  if( int rc = mctfBitDepthOk( ctx, orgPlane, refPlane ) ) return rc;
  CU( cudaSetDevice( ctx->device ) );
  const Plane po0 = ctx->planes.p[orgPlane], pr0 = ctx->planes.p[refPlane];
  const int W = po0.width, H = po0.height, u = pp->unit_size, nSub = pp->add_level ? 3 : 2, margin = 128;
  if( pr0.width != W || pr0.height != H ) return fail( ctx, VVB_ERR_ARG, "picture sizes differ" );
  if( po0.margin < 128 || pr0.margin < 128 ) return fail( ctx, VVB_ERR_ARG, "the MCTF search needs planes with a margin of at least 128 pels (MCTF_PADDING): vectors reach that far" );
  Plane po[4], pr[4]; po[0] = po0; pr[0] = pr0;
  int lw[4] = { W, 0, 0, 0 }, lh[4] = { H, 0, 0, 0 }, strideOf[4] = { 0, 0, 0, 0 };
  for( int l = 1; l <= nSub; l++ )
  {
    lw[l] = lw[l - 1] / 2; lh[l] = lh[l - 1] / 2;
    if( lw[l] < 8 || lh[l] < 8 ) return fail( ctx, VVB_ERR_UNSUPPORTED, "picture too small for the MCTF pyramid" );
    strideOf[l] = ( lw[l] + 2 * margin + 7 ) & ~7;
  }
  // intermediate fields (sized as the reference sizes them: width / (unit * k) + 1)
  const int fw[4] = { W / ( u * 2 ) + 1, W / ( u * 4 ) + 1, W / ( u * 8 ) + 1, W / ( u * 16 ) + 1 }, fh[4] = { H / ( u * 2 ) + 1, H / ( u * 4 ) + 1, H / ( u * 8 ) + 1, H / ( u * 16 ) + 1 };
  // Work holds the subsampled planes, the fields and the temporaries of mctfLevel, sized for the final level, which has the most blocks
  int16_t* planeMem[4][2]; vvb_mctf_mv* field[4]; MctfArena arena;
  int rc = carveArena( ctx, ScratchArena::Work, [&]( Layout& L )
  {
    for( int l = 1; l <= nSub; l++ ) for( int which = 0; which < 2; which++ ) planeMem[l][which] = L.take<int16_t>( (size_t) strideOf[l] * ( lh[l] + 2 * margin ) );
    for( int k = 0; k < 4; k++ ) field[k] = L.take<vvb_mctf_mv>( (size_t) fw[k] * fh[k] );
    arena = mctfCarve( L, std::max( 1, ( ( W - 8 ) / u + 1 ) * ( ( H - 8 ) / u + 1 ) ), ( H - 8 ) / u + 1 );
  } );
  if( rc ) return rc;
  for( int l = 1; l <= nSub; l++ )
    for( int which = 0; which < 2; which++ )
    {
      Plane& dst = which ? pr[l] : po[l];
      const Plane& src = which ? pr[l - 1] : po[l - 1];
      dst.origin = planeMem[l][which] + (size_t) margin * strideOf[l] + margin; dst.stride = strideOf[l]; dst.width = lw[l]; dst.height = lh[l]; dst.margin = margin; dst.bitDepth = src.bitDepth;
      dim3 blk( 32, 8 ), grd( ( lw[l] + 2 * margin + 31 ) / 32, ( lh[l] + 2 * margin + 7 ) / 8 );
      mctf_subsample_kernel<<<grd, blk, 0, ctx->stream>>>( src, const_cast<int16_t*>( dst.origin ), dst.stride, lw[l], lh[l], margin );
      CHECK_LAUNCH( "mctf_subsample_kernel" );
    }
  const vvb_mctf_mv* prev = nullptr; int prevW = 0, prevH = 0;
  const int bd = po0.bitDepth, sp = pp->search_pattern, low = pp->low_res_filter;
  if( pp->add_level )
  {
    if( ( rc = mctfLevel( ctx, po[3], pr[3], lw[3], lh[3], 2 * u, nullptr, 0, 0, 2, false, bd, sp, low, field[3], fw[3], fh[3], arena ) ) ) return rc;
    prev = field[3]; prevW = fw[3]; prevH = fh[3];
  }
  if( ( rc = mctfLevel( ctx, po[2], pr[2], lw[2], lh[2], 2 * u, prev, prevW, prevH, 2, false, bd, sp, low, field[2], fw[2], fh[2], arena ) ) ) return rc;
  if( ( rc = mctfLevel( ctx, po[1], pr[1], lw[1], lh[1], 2 * u, field[2], fw[2], fh[2], 2, false, bd, sp, low, field[1], fw[1], fh[1], arena ) ) ) return rc;
  if( ( rc = mctfLevel( ctx, po[0], pr[0], W, H, 2 * u, field[1], fw[1], fh[1], 2, false, bd, sp, low, field[0], fw[0], fh[0], arena ) ) ) return rc;
  return mctfLevel( ctx, po[0], pr[0], W, H, u, field[0], fw[0], fh[0], 1, true, bd, sp, low, dOut, ( W + u - 1 ) / u, ( H + u - 1 ) / u, arena );
}

int vvb_mctf_estimate_pyramid( vvb_ctx* ctx, int orgPlane, int refPlane, const vvb_mctf_pyr_par* pp, vvb_mctf_mv* out )
{
  if( !ctx || !pp || !out ) return fail( ctx, VVB_ERR_ARG, "bad arguments" );
  if( !validPlane( ctx, orgPlane ) ) return fail( ctx, VVB_ERR_ARG, "unknown plane" );
  const Plane& po = ctx->planes.p[orgPlane];
  const size_t count = (size_t)( ( po.width + pp->unit_size - 1 ) / std::max( 1, pp->unit_size ) ) * ( ( po.height + pp->unit_size - 1 ) / std::max( 1, pp->unit_size ) );
  vvb_mctf_mv* dOut;
  return HostCall( ctx ).out( dOut, out, count ).run( [&] { return vvb_mctf_estimate_pyramid_dev( ctx, orgPlane, refPlane, pp, dOut ); } );
}

// ---- affine ---------------------------------------------------------------------------------------------------------
int vvb_affine_sobel( vvb_ctx* ctx, int vertical, const int16_t* pred, int predStride, int16_t* deriv, int derivStride, int w, int h )
{
  if( !ctx || !pred || !deriv ) return fail( ctx, VVB_ERR_ARG, "null pointer" );
  if( w < 4 || h < 4 || w > 128 || h > 128 ) return fail( ctx, VVB_ERR_UNSUPPORTED, "affine blocks are 4..128" );
  CU( cudaSetDevice( ctx->device ) );
  int16_t *dP, *dD;
  return HostCall( ctx ).tmp( dP, blockPels( w, h ) ).tmp( dD, (size_t) w * h ).run( [&]
  {
    const int rc = uploadBlock( ctx, dP, pred, predStride, w, h );
    if( rc ) return rc;
    sobel_kernel<<<( w * h + 255 ) / 256, 256, 0, ctx->stream>>>( dP, w, dD, w, w, h, vertical );
    CHECK_LAUNCH( "sobel_kernel" );
    CU( cudaMemcpy2DAsync( deriv, (size_t) derivStride * 2, dD, (size_t) w * 2, (size_t) w * 2, h, cudaMemcpyDeviceToHost, ctx->stream ) );
    return VVB_OK;
  } );
}

int vvb_affine_equal_coeff( vvb_ctx* ctx, int sixParam, const int16_t* resi, int resiStride, const int16_t* gx, const int16_t* gy, int derivStride, int w, int h, int64_t eq[49] )
{
  if( !ctx || !resi || !gx || !gy || !eq ) return fail( ctx, VVB_ERR_ARG, "null pointer" );
  if( w < 4 || h < 4 || w > 128 || h > 128 ) return fail( ctx, VVB_ERR_UNSUPPORTED, "affine blocks are 4..128" );
  CU( cudaSetDevice( ctx->device ) );
  int16_t *dR, *dX, *dY; long long* dE; int rc;
  if( ( rc = carveArena( ctx, ScratchArena::Host, [&]( Layout& L ) { dR = L.take<int16_t>( blockPels( w, h ) ); dX = L.take<int16_t>( blockPels( w, h ) ); dY = L.take<int16_t>( blockPels( w, h ) ); dE = L.take<long long>( 49 ); } ) ) ||
      ( rc = uploadBlock( ctx, dR, resi, resiStride, w, h ) ) || ( rc = uploadBlock( ctx, dX, gx, derivStride, w, h ) ) || ( rc = uploadBlock( ctx, dY, gy, derivStride, w, h ) ) ) return rc;
  CU( cudaMemsetAsync( dE, 0, 49 * 8, ctx->stream ) );
  const int grid = std::min( 16, ( w * h + 255 ) / 256 );
  if( sixParam ) equal_coeff_kernel<6><<<grid, 256, 0, ctx->stream>>>( dR, w, dX, dY, w, w, h, dE );
  else           equal_coeff_kernel<4><<<grid, 256, 0, ctx->stream>>>( dR, w, dX, dY, w, w, h, dE );
  CHECK_LAUNCH( "equal_coeff_kernel" );
  int64_t tmp[49];
  CU( cudaMemcpyAsync( tmp, dE, 49 * 8, cudaMemcpyDeviceToHost, ctx->stream ) );
  CU( cudaStreamSynchronize( ctx->stream ) );         // tmp is consumed right below: always wait, asynchronous mode or not
  for( int i = 0; i < 49; i++ ) eq[i] += tmp[i];
  return VVB_OK;
}

int vvb_affine_eq_batch_dev( vvb_ctx* ctx, int sixParam, const int16_t* dPred, const int16_t* dResi, int n, int w, int h, int16_t* dDerivX, int16_t* dDerivY, int64_t* dEq )
{
  if( !ctx || !dPred || !dResi || !dEq || n < 0 ) return fail( ctx, VVB_ERR_ARG, "bad arguments" );
  if( w < 4 || h < 4 || w > 128 || h > 128 ) return fail( ctx, VVB_ERR_UNSUPPORTED, "affine blocks are 4..128" );
  if( n == 0 ) return VVB_OK;
  CU( cudaSetDevice( ctx->device ) );
  const size_t smem = (size_t) w * h * 6;
  if( sixParam ) affine_eq_batch_kernel<6><<<n, 128, smem, ctx->stream>>>( dPred, dResi, w, h, dDerivX, dDerivY, (long long*) dEq );
  else           affine_eq_batch_kernel<4><<<n, 128, smem, ctx->stream>>>( dPred, dResi, w, h, dDerivX, dDerivY, (long long*) dEq );
  CHECK_LAUNCH( "affine_eq_batch_kernel" );
  return VVB_OK;
}

int vvb_affine_eq_batch( vvb_ctx* ctx, int sixParam, const int16_t* pred, const int16_t* resi, int n, int w, int h, int16_t* derivX, int16_t* derivY, int64_t* eq )
{
  if( !ctx || !pred || !resi || !eq || n < 0 ) return fail( ctx, VVB_ERR_ARG, "bad arguments" );
  if( n == 0 ) return VVB_OK;
  const size_t samples = (size_t) n * w * h;
  const int16_t *dP, *dR; int16_t *dX, *dY; int64_t* dE;
  return HostCall( ctx ).in( dP, pred, samples ).in( dR, resi, samples ).out( dE, eq, (size_t) n * 49 ).out( dX, derivX, samples ).out( dY, derivY, samples )
                        .run( [&] { return vvb_affine_eq_batch_dev( ctx, sixParam, dP, dR, n, w, h, dX, dY, dE ); } );
}

} // extern "C"
