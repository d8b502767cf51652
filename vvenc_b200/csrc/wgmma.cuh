// wgmma.cuh -- the Hopper wgmma primitives of the tensor-core transform engines (trquant_tc2_kernels.cuh, itrquant_tc_kernels.cuh): shared-memory
// descriptors of K-major no-swizzle operands ([16-byte K chunk][row][16 B]), the s8 / u8 x s8 -> s32 MMAs of one warpgroup with register accumulators,
// the accumulator layout of a thread, and the fences that order them.
#pragma once
#include <stdint.h>

namespace vvb {

__device__ __forceinline__ uint32_t smem_u32( const void* p ) { return (uint32_t) __cvta_generic_to_shared( p ); }

// wgmma shared-memory descriptor, K-major, no swizzle (PTX ISA, "Matrix Descriptor Format"): start address, leading byte offset = stride between the
// 16-byte K chunks of a k32 step, stride byte offset = stride between 8-row groups; base offset 0, layout type 0
__device__ __forceinline__ uint64_t gmma_desc_kmajor( uint32_t smemAddr, uint32_t lboBytes, uint32_t sboBytes )
{
  uint64_t d = 0;
  d |= (uint64_t)( ( smemAddr >> 4 ) & 0x3fffu );           // start address, bits [0,14)
  d |= (uint64_t)( ( lboBytes >> 4 ) & 0x3fffu ) << 16;     // leading byte offset, bits [16,30)
  d |= (uint64_t)( ( sboBytes >> 4 ) & 0x3fffu ) << 32;     // stride byte offset, bits [32,46)
  return d;
}

// D[64 x NN] (+)= A[64 x 32 B] * B[NN x 32 B]^T, A read as u8 (AS = false) or s8 (AS = true), B as s8, s32 accumulators; issued by the whole warpgroup
// (the 128 threads of the CTA).  accumulate = 0 starts the chain.  Register i of a thread holds row wg_row( i ), column wg_col( i ) of D.
template<int NN, bool AS> __device__ __forceinline__ void wgmma_i8( int (&d)[NN / 2], uint64_t descA, uint64_t descB, int accumulate );
template<> __device__ __forceinline__ void wgmma_i8<16, false>( int (&d)[8], uint64_t descA, uint64_t descB, int accumulate )
{
  asm volatile( "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %10, 0;\n\t"
                "wgmma.mma_async.sync.aligned.m64n16k32.s32.u8.s8 {%0,%1,%2,%3,%4,%5,%6,%7}, %8, %9, p;\n\t}\n"
                : "+r"( d[0] ), "+r"( d[1] ), "+r"( d[2] ), "+r"( d[3] ), "+r"( d[4] ), "+r"( d[5] ), "+r"( d[6] ), "+r"( d[7] )
                : "l"( descA ), "l"( descB ), "r"( accumulate ) : "memory" );
}
template<> __device__ __forceinline__ void wgmma_i8<16, true>( int (&d)[8], uint64_t descA, uint64_t descB, int accumulate )
{
  asm volatile( "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %10, 0;\n\t"
                "wgmma.mma_async.sync.aligned.m64n16k32.s32.s8.s8 {%0,%1,%2,%3,%4,%5,%6,%7}, %8, %9, p;\n\t}\n"
                : "+r"( d[0] ), "+r"( d[1] ), "+r"( d[2] ), "+r"( d[3] ), "+r"( d[4] ), "+r"( d[5] ), "+r"( d[6] ), "+r"( d[7] )
                : "l"( descA ), "l"( descB ), "r"( accumulate ) : "memory" );
}
template<> __device__ __forceinline__ void wgmma_i8<32, false>( int (&d)[16], uint64_t descA, uint64_t descB, int accumulate )
{
  asm volatile( "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %18, 0;\n\t"
                "wgmma.mma_async.sync.aligned.m64n32k32.s32.u8.s8 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15}, %16, %17, p;\n\t}\n"
                : "+r"( d[0] ), "+r"( d[1] ), "+r"( d[2] ), "+r"( d[3] ), "+r"( d[4] ), "+r"( d[5] ), "+r"( d[6] ), "+r"( d[7] ), "+r"( d[8] ), "+r"( d[9] ), "+r"( d[10] ), "+r"( d[11] ), "+r"( d[12] ), "+r"( d[13] ), "+r"( d[14] ), "+r"( d[15] )
                : "l"( descA ), "l"( descB ), "r"( accumulate ) : "memory" );
}
template<> __device__ __forceinline__ void wgmma_i8<32, true>( int (&d)[16], uint64_t descA, uint64_t descB, int accumulate )
{
  asm volatile( "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %18, 0;\n\t"
                "wgmma.mma_async.sync.aligned.m64n32k32.s32.s8.s8 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15}, %16, %17, p;\n\t}\n"
                : "+r"( d[0] ), "+r"( d[1] ), "+r"( d[2] ), "+r"( d[3] ), "+r"( d[4] ), "+r"( d[5] ), "+r"( d[6] ), "+r"( d[7] ), "+r"( d[8] ), "+r"( d[9] ), "+r"( d[10] ), "+r"( d[11] ), "+r"( d[12] ), "+r"( d[13] ), "+r"( d[14] ), "+r"( d[15] )
                : "l"( descA ), "l"( descB ), "r"( accumulate ) : "memory" );
}
template<> __device__ __forceinline__ void wgmma_i8<64, false>( int (&d)[32], uint64_t descA, uint64_t descB, int accumulate )
{
  asm volatile( "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
                "wgmma.mma_async.sync.aligned.m64n64k32.s32.u8.s8 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31}, %32, %33, p;\n\t}\n"
                : "+r"( d[0] ), "+r"( d[1] ), "+r"( d[2] ), "+r"( d[3] ), "+r"( d[4] ), "+r"( d[5] ), "+r"( d[6] ), "+r"( d[7] ), "+r"( d[8] ), "+r"( d[9] ), "+r"( d[10] ), "+r"( d[11] ), "+r"( d[12] ), "+r"( d[13] ), "+r"( d[14] ), "+r"( d[15] ), "+r"( d[16] ), "+r"( d[17] ), "+r"( d[18] ), "+r"( d[19] ), "+r"( d[20] ), "+r"( d[21] ), "+r"( d[22] ), "+r"( d[23] ), "+r"( d[24] ), "+r"( d[25] ), "+r"( d[26] ), "+r"( d[27] ), "+r"( d[28] ), "+r"( d[29] ), "+r"( d[30] ), "+r"( d[31] )
                : "l"( descA ), "l"( descB ), "r"( accumulate ) : "memory" );
}
template<> __device__ __forceinline__ void wgmma_i8<64, true>( int (&d)[32], uint64_t descA, uint64_t descB, int accumulate )
{
  asm volatile( "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
                "wgmma.mma_async.sync.aligned.m64n64k32.s32.s8.s8 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31}, %32, %33, p;\n\t}\n"
                : "+r"( d[0] ), "+r"( d[1] ), "+r"( d[2] ), "+r"( d[3] ), "+r"( d[4] ), "+r"( d[5] ), "+r"( d[6] ), "+r"( d[7] ), "+r"( d[8] ), "+r"( d[9] ), "+r"( d[10] ), "+r"( d[11] ), "+r"( d[12] ), "+r"( d[13] ), "+r"( d[14] ), "+r"( d[15] ), "+r"( d[16] ), "+r"( d[17] ), "+r"( d[18] ), "+r"( d[19] ), "+r"( d[20] ), "+r"( d[21] ), "+r"( d[22] ), "+r"( d[23] ), "+r"( d[24] ), "+r"( d[25] ), "+r"( d[26] ), "+r"( d[27] ), "+r"( d[28] ), "+r"( d[29] ), "+r"( d[30] ), "+r"( d[31] )
                : "l"( descA ), "l"( descB ), "r"( accumulate ) : "memory" );
}


__device__ __forceinline__ int wg_row( int i ) { return ( ( threadIdx.x >> 5 ) << 4 ) + ( ( threadIdx.x & 31 ) >> 2 ) + ( i & 2 ) * 4; }
__device__ __forceinline__ int wg_col( int i ) { return ( i >> 2 ) * 8 + ( threadIdx.x & 3 ) * 2 + ( i & 1 ); }
__device__ __forceinline__ void wg_fence()  { asm volatile( "wgmma.fence.sync.aligned;" ::: "memory" ); }
__device__ __forceinline__ void wg_commit() { asm volatile( "wgmma.commit_group.sync.aligned;" ::: "memory" ); }
__device__ __forceinline__ void wg_wait0()  { asm volatile( "wgmma.wait_group.sync.aligned 0;" ::: "memory" ); }
// the compiler does not know that wgmma writes its accumulator registers asynchronously: pinning every register here (before the first MMA of a group
// and after wgmma.wait_group) keeps it from reading, moving or reusing them while MMAs are in flight
template<int R> __device__ __forceinline__ void wg_hold( int (&d)[R] )
{
#pragma unroll
  for( int i = 0; i < R; i++ ) asm volatile( "" : "+r"( d[i] ) :: "memory" );
}
__device__ __forceinline__ void fence_async_smem() { asm volatile( "fence.proxy.async.shared::cta;" ::: "memory" ); }

} // namespace vvb
