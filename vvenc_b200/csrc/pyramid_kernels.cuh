// pyramid_kernels.cuh -- SAD pyramid of the dense integer search with every level formed inside one CTA (sm_90a).
//
// Replaces, for 8x8 base blocks without row sub-sampling, the pair sad_search_kernel<.., PARENT> + sad_table_sum_kernel: one CTA owns one ROOT block of
// 16x16, 32x32 or 64x64 pels (LV = 2, 3, 4 levels) together with all of its quad-tree descendants, stages the reference window of the whole root once and
// produces the InterSearch::xPatternSearch result (EncoderLib/InterSearch.cpp:2209-2251: every vector of the range, MV rate of the block's own predictor,
// first strictly smaller cost in raster order) of EVERY block of every level.  Pel work happens once, at the 8x8 level; a 16x16 cost is the sum of its
// four children's SADs in registers; 32x32 tables are accumulated in shared memory and the 64x64 table is their sum -- no cost table ever leaves the SM
// (the previous design moved about 1.2 GB of 16x16 / 32x32 tables through HBM per 2160p picture).
//
// Arithmetic per (8x8 block, candidate):  SAD = sum a - sum b + 2 sum max(b - a, 0)
//   sum a : per block, once;  sum b : 8x8 box sums of the window (uint16 table V);  sum max : HFMA2.RELU (fma pipe; pels up to 1023 are exact fp16
//   subnormals) per pel pair, and per two pel pairs one IADD3 (alu pipe) into two uint16 lanes.  That is 1.5 instructions per pel pair where a min
//   (VIMNMX.S16x2, alu) + dot product (IDP.2A, fma) took 2, and the alu pipe carries half an instruction per pair instead of one.  Everything else is kept
//   off the alu pipe where possible:
//   * odd-offset candidates read a second, one-pel-shifted copy of the window (no funnel shifts),
//   * a thread evaluates TWO vertically adjacent candidate rows for a strip of 8 vectors: the nine window rows they need are loaded once (LDS.128) and
//     every original row serves both (shared-memory traffic per candidate halves),
//   * the epilogue per candidate is IDP.4A (shared address of the rate entry: table base + row bits, plus column bits), LDS (rate table pre-multiplied
//     by 8, one table per strip slot so that the slot index is part of the entry), IDP.2A (sum a + 2 * the two uint16 lanes), IDP.2A (unpack the box sum
//     and subtract it), IMAD (parent sum), IMAD (key) on the fma pipe and half a VIMNMX3.
//   * strip slots past the end of the range carry MV-bit count 250 and read rate-table entries that can never win; no predicate per candidate.
//   * the item keeps its base addresses and the four members step through fixed offsets.  For 32x32 and 64x64 roots the CTA has at most 512 threads so
//     that ptxas may keep them in 128 registers (at 640 threads the 96-register cap forced their recomputation in every member).
//
// Row walk (64x64 roots only; one such CTA fills an SM, so nothing hides its set-up): the host launches min(roots, SMs) CTAs and each walks a run of
// consecutive roots.  When the next root of the run lies one root width to the right with the same rows and range, and the window source is 4-byte aligned,
// the CTA copies the next window's new R pels of every row into a staging area with cp.async behind its own candidate loop (L2 prefetches cover the next
// root's descriptors and originals), then shifts the kept half of its window left and drops the staged columns in instead of restaging it from global
// memory.  The rate tables are staged once per CTA.  Any other next root (new row, other range, broken quad tree, 16-bit staging path, a staging area
// that does not fit) is restaged in full, so every result is the one a CTA per root would give.  The next root's originals are copied the same way into a
// second originals buffer where it fits (16-byte aligned rows), whether or not the window carries.  The 32x32 tables are zeroed once per CTA and the argmin
// pass clears each entry as it reads it, so no root spends a pass and a barrier on zeroing them; the prologue's row sums live in win1 until the shifted copy
// is formed after the box sums.
//
// Geometry: sad_pyramid8_kernel<LV, 0> takes the range and the shared-memory layout from the launch; sad_pyramid8_kernel<4, PYR_FIXED_N> is compiled for a
// 65 x 65 range (+-32, unclipped), where the window pitch, the table strides and the item counts are constants: row offsets fold into LDS immediates and the
// item decode divides by constants instead of float reciprocals.
#pragma once
#include "search_kernels.cuh"

namespace vvb {

// CTA size bound per root size.  A 64x64 root fills an SM's shared memory on its own; 512 threads leave 128 registers for the item loop.  16x16 roots need
// about 64 KB, so several CTAs share an SM and registers set how many: the 640-thread bound (96 registers) lets two CTAs of the 320 threads that a
// +-32 range picks run on one SM, where 120 registers would allow only one.
template<int LV> constexpr int pyr_max_threads() { return LV == 2 ? 640 : 512; }
#define PYR_MVN         296                      // rate-table entries per strip slot: 0..79 real, the rest "never wins" (padded columns index 250 + row bits)
#define PYR_PAD_BITS    250
#define PYR_NEVER       ( 1u << 26 )             // cost no real candidate reaches; 4 * PYR_NEVER * 8 still fits 32 bits
#define PYR_FIXED_N     65                       // range with a fixed-geometry instantiation of the 64x64 kernel: +-32, the encoder's default search range

struct PyrLevels { const vvb_block* blocks[4]; vvb_best* best[4]; };

struct PyrSmem
{
  int nStrips, nxp, nyp, bStride, ws, winH, winWords, vRows, vPitch, nT, tStride;
  int offWin0, offWin1, offV, offOrg, offBits, offPred, offSumA, offKey32, offKey64, offMv8, offMvRaw, offT, offStage, total;   // bytes
  int stageWords;                                        // words of the row walk's staging area (winH rows of R / 2 words); 0: every root restages in full
  int offOrgNext;                                        // bytes: second originals buffer the row walk fills for the next root behind the loop; 0: none
};

template<int LV>
__host__ __device__ constexpr PyrSmem pyr_smem( int nx, int ny )
{
  constexpr int R = 8 << ( LV - 1 ), NB0 = 1 << ( 2 * ( LV - 1 ) ), NBLK = ( 4 * NB0 - 1 ) / 3;
  PyrSmem s{};
  s.nStrips = ( nx + 7 ) >> 3;
  s.nxp     = s.nStrips * 8;
  s.nyp     = ( ny + 1 + 7 ) & ~7;                       // row B of the last pair may be one past the range
  s.bStride = s.nxp + s.nyp;                             // per block: column bits [nxp] (raw), row bits [nyp] (times 4); multiple of 8
  // row pitch: multiple of 8 pels (16-byte rows); pitch/8 == nStrips (mod 8) makes a warp's LDS.128 walk consecutive 16-byte chunks across rows
  int ws = R + s.nxp;
  const int want = ( ( s.nStrips - ( ws >> 3 ) ) % 8 + 8 ) % 8;
  if( want <= 2 ) ws += 8 * want;
  s.ws      = ws;
  s.winH    = R + ny - 1;
  s.winWords = ( s.winH * s.ws + 16 ) >> 1;              // + overrun for the shifted copy
  s.vRows   = s.winH - 7;
  s.vPitch  = R - 8 + s.nxp;
  s.nT      = LV == 4 ? 4 : ( LV == 3 ? 1 : 0 );
  s.tStride = ny * s.nxp;
  // fixed-size tables first: their offsets do not depend on the range
  int o = 0;
  s.offMv8  = o;   o += 8 * PYR_MVN * 4;
  s.offMvRaw = o;  o += VVB_MVCOST_ENTRIES * 4;
  s.offKey64 = o;  o += 8 * 8;
  s.offKey32 = o;  o += ( ( NB0 + NB0 / 4 ) * 4 + 15 ) & ~15;
  s.offSumA = o;   o += ( NB0 * 4 + 15 ) & ~15;
  s.offPred = o;   o += ( NBLK * 8 + 15 ) & ~15;
  s.offWin0 = o;   o += s.winWords * 4;
  s.offWin1 = o;   o += s.winWords * 4;
  s.offV    = o;   o += ( ( s.vRows * s.vPitch * 2 ) + 15 ) & ~15;
  s.offOrg  = o;   o += R * R * 2;
  s.offBits = o;   o += NBLK * s.bStride;
  s.offT    = ( o + 15 ) & ~15;
  s.total   = s.offT + s.nT * s.tStride * 4 + 16;        // the prologue's row-sum scratch lives in win1 (ws > vPitch), which is written after it
  // row walk of 64x64 roots: the next root's new R pels of every window row are copied behind the candidate loop into the shared memory the rest leaves
  // free.  Where that does not fit (larger ranges), or a row holds more words than the carry's 4 per lane, the walk restages every root in full.
  s.offStage   = ( s.total + 15 ) & ~15;
  s.stageWords = 0;
  if( LV == 4 && ( ( R + nx ) >> 1 ) <= 128 && s.offStage + s.winH * ( R / 2 ) * 4 <= 227 * 1024 )
  {
    s.stageWords = s.winH * ( R / 2 );
    s.total      = s.offStage + s.stageWords * 4;
  }
  // and the next root's originals go to a second buffer where that fits (at +-32 it does, next to the staging area)
  if( LV == 4 && ( ( s.total + 15 ) & ~15 ) + R * R * 2 <= 227 * 1024 )
  {
    s.offOrgNext = ( s.total + 15 ) & ~15;
    s.total      = s.offOrgNext + R * R * 2;
  }
  return s;
}

// Phase-timing build (-DVVB_PYR_PHASES, tools/pyr_phases.py; never the shipped library): thread 0 of every CTA adds the %globaltimer span of each phase of
// its root to g_pyrPhaseNs[LV - 2][phase] and counts the root in [LV - 2][PYR_NPHASE].  Phases: geometry, staging, prologue compute, candidate loop, argmin,
// results.  The results phase gets a barrier of its own in that build so that its span covers every thread's stores.
#define PYR_NPHASE 6
#ifdef VVB_PYR_PHASES
__device__ unsigned long long g_pyrPhaseNs[3][PYR_NPHASE + 1];
__device__ __forceinline__ unsigned long long pyr_now() { unsigned long long t; asm volatile( "mov.u64 %0, %%globaltimer;" : "=l"( t ) ); return t; }
#define PYR_MARK( k ) do { if( threadIdx.x == 0 ) { const unsigned long long t_ = pyr_now(); atomicAdd( &g_pyrPhaseNs[LV - 2][k], t_ - pyrT ); pyrT = t_; } } while( 0 )
#else
#define PYR_MARK( k ) do {} while( 0 )
#endif

__device__ __forceinline__ int pyr_compact( int v ) { v &= 0x55555555; v = ( v | ( v >> 1 ) ) & 0x33333333; v = ( v | ( v >> 2 ) ) & 0x0f0f0f0f; return ( v | ( v >> 4 ) ) & 0xff; }

__device__ __forceinline__ void pyr_cp_async16( void* s, const void* g ) { asm volatile( "cp.async.cg.shared.global [%0], [%1], 16;" :: "r"( (uint32_t) __cvta_generic_to_shared( s ) ), "l"( g ) : "memory" ); }
__device__ __forceinline__ void pyr_cp_async4( void* s, const void* g ) { asm volatile( "cp.async.ca.shared.global [%0], [%1], 4;" :: "r"( (uint32_t) __cvta_generic_to_shared( s ) ), "l"( g ) : "memory" ); }
__device__ __forceinline__ void pyr_cp_async_wait_all() { asm volatile( "cp.async.wait_all;" ::: "memory" ); }
__device__ __forceinline__ void pyr_prefetch_l2( const void* g ) { asm volatile( "prefetch.global.L2 [%0];" :: "l"( g ) ); }

// rate-table entry at a 32-bit shared-memory address: the table base rides in the IDP.4A accumulator and the slot offset becomes the LDS immediate
__device__ __forceinline__ uint32_t pyr_lds( uint32_t addr ) { uint32_t v; asm volatile( "ld.shared.u32 %0, [%1];" : "=r"( v ) : "r"( addr ) ); return v; }

// max(w - o, 0) per 16-bit half.  Pels up to 1023 are fp16 subnormals (or zero) as they stand, and fp16 arithmetic keeps subnormals, so the difference of
// two of them and its clamp are exact: the result's bits are the integer max(w - o, 0).
__device__ __forceinline__ uint32_t pyr_relu_diff( uint32_t o, uint32_t w )
{
  uint32_t d;
  asm( "fma.rn.relu.f16x2 %0, %1, %2, %3;" : "=r"( d ) : "r"( o ), "r"( 0xbc00bc00u ), "r"( w ) );
  return d;
}

// box sums of two candidates (uint16 lanes of v) times the signed bytes of w, plus c
__device__ __forceinline__ int pyr_dp2a_us( uint32_t v, uint32_t w, int c ) { int d; asm( "dp2a.lo.u32.s32 %0, %1, %2, %3;" : "=r"( d ) : "r"( v ), "r"( w ), "r"( c ) ); return d; }

// one candidate row of one member: box sum + MV rate -> 8 packed (cost * 8 + slot) keys, running minimum; the SAD goes into the parent's sum.
// acc[k] = sum a + 2 sum max(b - a, 0); mvRow = shared address of the rate tables + 4 * row bits
__device__ __forceinline__ uint32_t pyr_finish_row( const int (&acc)[8], const uint16_t* __restrict__ vrow, uint2 bw, uint32_t mvRow, uint32_t one, uint32_t eight,
                                                    uint32_t (&ps)[8] )
{
  const uint4 vw = *reinterpret_cast<const uint4*>( vrow );
  const uint32_t v[4] = { vw.x, vw.y, vw.z, vw.w };
  uint32_t bk = 0xffffffffu;
#pragma unroll
  for( int k = 0; k < 8; k++ )
  {
    const uint32_t a    = __dp4a( k < 4 ? bw.x : bw.y, 4u << ( 8 * ( k & 3 ) ), mvRow );                  // + 4 * column bits
    const uint32_t mvk  = pyr_lds( a + k * ( PYR_MVN * 4 ) );                                             // rate * 8 + k
    const uint32_t sad  = (uint32_t) pyr_dp2a_us( v[k >> 1], ( k & 1 ) ? 0xff00u : 0x00ffu, acc[k] );  // - box sum: sum |a - b| = sum a - sum b + 2 sum max(b - a, 0)
    ps[k] = sad * one + ps[k];                                                                             // IMAD: keeps the add off the alu pipe
    const uint32_t key = sad * eight + mvk;
    bk = min( bk, key );
  }
  return bk;
}

// a / d for a >= 0, d >= 1: with the geometry fixed at compile time d is a constant and this is an integer division by a constant (a multiply-high); otherwise
// the float reciprocal inv = 1 / d of the runtime count
template<int NXY>
__device__ __forceinline__ int pyr_div( int a, int d, float inv ) { return NXY ? (int)( (unsigned) a / (unsigned) d ) : div_rcp( a, inv ); }

// NXY = 0: the range nx x ny and the layout L come from the launch.  NXY > 0: nx = ny = NXY, and the layout and every count derived from it are compile-time
// constants, so window, box-sum and MV-bit offsets fold into the LDS immediates and the item decode needs no float reciprocals (the host checks that the
// launch's range is NXY x NXY).
template<int LV, int NXY>
__global__ void __launch_bounds__( pyr_max_threads<LV>(), 1 ) sad_pyramid8_kernel( const __grid_constant__ Plane orgPlane, const __grid_constant__ Plane refPlane,
                                                                             const __grid_constant__ PyrLevels lv, int rootFirst, int nRoots, int nxArg, int nyArg,
                                                                             const __grid_constant__ MePar par, const __grid_constant__ PyrSmem LArg,   // pyr_smem<LV>( nx, ny )
                                                                             uint32_t one, uint32_t eight )
{
  constexpr int R = 8 << ( LV - 1 ), NB0 = 1 << ( 2 * ( LV - 1 ) ), NQ = NB0 / 4, NBLK = ( 4 * NB0 - 1 ) / 3, LTOP = LV - 1;
  constexpr int OFF1 = NB0, OFF2 = NB0 + NQ, OFF3 = NB0 + NQ + NQ / 4, NT = LV == 4 ? 4 : ( LV == 3 ? 1 : 0 );
  constexpr PyrSmem LF = pyr_smem<LV>( NXY ? NXY : 1, NXY ? NXY : 1 );
  const int nx = NXY ? NXY : nxArg, ny = NXY ? NXY : nyArg;
  const PyrSmem L = NXY ? LF : LArg;
  extern __shared__ __align__( 128 ) unsigned char smemRaw[];
  uint32_t* win0w = reinterpret_cast<uint32_t*>( smemRaw + L.offWin0 );
  uint32_t* win1w = reinterpret_cast<uint32_t*>( smemRaw + L.offWin1 );
  uint16_t* V     = reinterpret_cast<uint16_t*>( smemRaw + L.offV );
  int16_t*  orgS  = reinterpret_cast<int16_t*>( smemRaw + L.offOrg );
  int16_t*  orgN  = reinterpret_cast<int16_t*>( smemRaw + L.offOrgNext );      // the other originals buffer (L.offOrgNext > 0)
  unsigned char* bitsS = smemRaw + L.offBits;
  int2*     sPred = reinterpret_cast<int2*>( smemRaw + L.offPred );
  int*      sSumA = reinterpret_cast<int*>( smemRaw + L.offSumA );
  uint32_t* sKey32 = reinterpret_cast<uint32_t*>( smemRaw + L.offKey32 );
  unsigned long long* sKey64 = reinterpret_cast<unsigned long long*>( smemRaw + L.offKey64 );
  unsigned char* sMv8 = smemRaw + L.offMv8;
  uint32_t* sMvRaw = reinterpret_cast<uint32_t*>( smemRaw + L.offMvRaw );
  uint32_t* T     = reinterpret_cast<uint32_t*>( smemRaw + L.offT );
  uint16_t* Hs    = reinterpret_cast<uint16_t*>( smemRaw + L.offWin1 );         // row sums: prologue scratch in win1, which is formed after the box sums

#ifdef VVB_PYR_PHASES
  unsigned long long pyrT = threadIdx.x == 0 ? pyr_now() : 0ull;
#endif
  const int tid = threadIdx.x, nthr = blockDim.x, lane = tid & 31;
  const int nxp = L.nxp, nStrips = L.nStrips, ws = L.ws, wsw = ws >> 1, winH = L.winH;
  const int ob = par.orderBits;
  const int validW = R + nx - 1, validWords = ( validW + 1 ) >> 1, keepWords = validWords - R / 2;   // a carried window keeps keepWords words of a row
  uint32_t* stage = reinterpret_cast<uint32_t*>( smemRaw + L.offStage );

  // rate tables: the same for every root of the launch
  for( int i = tid; i < VVB_MVCOST_ENTRIES; i += nthr ) sMvRaw[i] = par.tab.cost[i];
  for( int i = tid; i < 8 * PYR_MVN; i += nthr )
  {
    const int k = i / PYR_MVN, b = i - k * PYR_MVN;
    reinterpret_cast<uint32_t*>( sMv8 )[i] = ( b < VVB_MVCOST_ENTRIES ? par.tab.cost[b] : PYR_NEVER ) * 8u + (uint32_t) k;
  }
  // the 32x32 tables start zeroed; the argmin pass clears every entry it reads, and a root that skips its candidates leaves them untouched, so every root
  // finds them zeroed (the first barrier of the root loop publishes this)
  if( LV >= 3 ) { for( int i = tid; i < L.nT * L.tStride; i += nthr ) T[i] = 0u; }

  // A 64x64 CTA walks a run of consecutive roots (gridDim.x runs of balanced length); smaller roots take one CTA each.  carry: the window in shared memory is
  // the previous root's, this root lies one root width to its right with the same rows and range, and the staging area holds this root's new R pels of
  // every window row.
  constexpr bool WALK = LV == 4;
  const int rBeg = WALK ? rootFirst + (int)( (long long) blockIdx.x * nRoots / gridDim.x ) : rootFirst + (int) blockIdx.x;
  const int rEnd = WALK ? rootFirst + (int)( (long long)( blockIdx.x + 1 ) * nRoots / gridDim.x ) : rBeg + 1;
  bool carry = false;
  bool orgStaged = false;                 // orgN holds this root's originals, copied behind the previous root's loop
#pragma unroll 1
  for( int root = rBeg; root < rEnd; root++ )
  {
    const vvb_block rb = lv.blocks[LTOP][root];

    // ---- the root's descendants: positions must be the z-order tiling of the root, ranges must equal the launch's range
    int geomOk = ( rb.right - rb.left + 1 == nx ) && ( rb.bottom - rb.top + 1 == ny );
    for( int t = tid; t < NBLK; t += nthr )
    {
      const int l = t < OFF1 ? 0 : ( t < OFF2 ? 1 : ( t < OFF3 ? 2 : 3 ) );
      const int i = t - ( l == 0 ? 0 : ( l == 1 ? OFF1 : ( l == 2 ? OFF2 : OFF3 ) ) );
      const vvb_block b = lv.blocks[l][( (size_t) root << ( 2 * ( LTOP - l ) ) ) + i];
      const int s = 8 << l;
      geomOk &= ( b.x == rb.x + pyr_compact( i ) * s ) && ( b.y == rb.y + pyr_compact( i >> 1 ) * s ) &&
                ( b.left == rb.left ) && ( b.right == rb.right ) && ( b.top == rb.top ) && ( b.bottom == rb.bottom );
      sPred[t] = make_int2( b.pred_hor, b.pred_ver );
    }
    geomOk = __syncthreads_and( geomOk );
    PYR_MARK( 0 );
    if( !geomOk )
    {
      // not a proper quad tree (or a block with another range): everything below this root is reported invalid, as the header promises
      for( int t = tid; t < NBLK; t += nthr )
      {
        const int l = t < OFF1 ? 0 : ( t < OFF2 ? 1 : ( t < OFF3 ? 2 : 3 ) );
        const int i = t - ( l == 0 ? 0 : ( l == 1 ? OFF1 : ( l == 2 ? OFF2 : OFF3 ) ) );
        vvb_best b; b.dx = 0; b.dy = 0; b.sad = 0xffffffffu; b.cost = ~0ull;
        lv.best[l][( (size_t) root << ( 2 * ( LTOP - l ) ) ) + i] = b;
      }
      carry = false;                      // this root's staged columns and originals are dropped; the next root restages in full
      orgStaged = false;
      continue;
    }

    // ---- stage the window (zero beyond the valid columns) and the original root block
    const int16_t* src = refPlane.origin + (ptrdiff_t)( rb.y + rb.top ) * refPlane.stride + rb.x + rb.left;
    const bool src32 = ( ( (uintptr_t) src & 3 ) == 0 ) && ( ( refPlane.stride & 1 ) == 0 );
    {
      if( WALK && carry )
      {
        // the window moves R pels left: a warp rebuilds whole rows from the kept words of the row and the staged new ones; the words past validWords and the
        // overrun words stay zero
        for( int r = tid >> 5; r < winH; r += nthr >> 5 )
        {
          uint32_t* row = win0w + r * wsw;
          const uint32_t* st = stage + r * ( R / 2 );
          uint32_t v[4];
#pragma unroll
          for( int j = 0; j < 4; j++ ) { const int c = lane + 32 * j; v[j] = c < keepWords ? row[c + R / 2] : ( c < validWords ? st[c - keepWords] : 0u ); }
          __syncwarp();
#pragma unroll
          for( int j = 0; j < 4; j++ ) { const int c = lane + 32 * j; if( c < validWords ) row[c] = v[j]; }
        }
      }
      else if( src32 )
      {
        const int total = winH * wsw;
        const float inv = 1.0f / (float) wsw;
        for( int i0 = tid; i0 < total; i0 += nthr * 8 )
        {
          uint32_t v[8];
#pragma unroll
          for( int u = 0; u < 8; u++ )
          {
            const int i = i0 + u * nthr;
            v[u] = 0u;
            if( i < total )
            {
              const int r = pyr_div<NXY>( i, wsw, inv ), c = i - r * wsw;
              if( c < validWords ) v[u] = __ldg( reinterpret_cast<const uint32_t*>( src + (ptrdiff_t) r * refPlane.stride ) + c );
            }
          }
#pragma unroll
          for( int u = 0; u < 8; u++ ) { const int i = i0 + u * nthr; if( i < total ) win0w[i] = v[u]; }
        }
      }
      else
      {
        int16_t* win0 = reinterpret_cast<int16_t*>( win0w );
        const int total = winH * ws;
        const float inv = 1.0f / (float) ws;
        for( int i0 = tid; i0 < total; i0 += nthr * 8 )
        {
          int16_t v[8];
#pragma unroll
          for( int u = 0; u < 8; u++ )
          {
            const int i = i0 + u * nthr;
            v[u] = 0;
            if( i < total )
            {
              const int r = pyr_div<NXY>( i, ws, inv ), c = i - r * ws;
              if( c < validW ) v[u] = __ldg( src + (ptrdiff_t) r * refPlane.stride + c );
            }
          }
#pragma unroll
          for( int u = 0; u < 8; u++ ) { const int i = i0 + u * nthr; if( i < total ) win0[i] = v[u]; }
        }
      }
      if( tid < 8 ) win0w[winH * wsw + tid] = 0u;                                   // overrun words read by the shifted copy
      if( WALK && orgStaged ) { int16_t* t = orgS; orgS = orgN; orgN = t; }
      else
      {
        const int16_t* so = orgPlane.origin + (ptrdiff_t) rb.y * orgPlane.stride + rb.x;
        for( int i = tid; i < R * R; i += nthr )
        {
          const int r = i / R, c = i - r * R;
          orgS[i] = __ldg( so + (ptrdiff_t) r * orgPlane.stride + c );
        }
      }
      for( int i = tid; i < NB0 + NQ; i += nthr ) sKey32[i] = 0xffffffffu;
      if( tid < 8 ) sKey64[tid] = ~0ull;
    }
    __syncthreads();
    PYR_MARK( 1 );

    // ---- per-block sum a, row sums Hs[r][c] = sum_{x<8} win[r][c+x], MV bit counts
    {
      for( int b = tid; b < NB0; b += nthr )
      {
        const int bx = pyr_compact( b ), by = pyr_compact( b >> 1 );
        int s = 0;
        for( int y = 0; y < 8; y++ )
        {
          const uint4 o = *reinterpret_cast<const uint4*>( orgS + ( by * 8 + y ) * R + bx * 8 );
          s = __dp2a_lo( (int) o.x, 0x0101, s ); s = __dp2a_lo( (int) o.y, 0x0101, s ); s = __dp2a_lo( (int) o.z, 0x0101, s ); s = __dp2a_lo( (int) o.w, 0x0101, s );
        }
        sSumA[b] = s;
      }
      const int cStrips = L.vPitch >> 3, nTasks = winH * cStrips;
      const float inv = 1.0f / (float) cStrips;
      for( int t = tid; t < nTasks; t += nthr )
      {
        const int r = pyr_div<NXY>( t, cStrips, inv ), st = t - r * cStrips;
        const uint32_t* row = win0w + r * wsw + st * 4;
        const uint4 a = *reinterpret_cast<const uint4*>( row ), b = *reinterpret_cast<const uint4*>( row + 4 );
        const uint32_t w[8] = { a.x, a.y, a.z, a.w, b.x, b.y, b.z, b.w };
        int p[16];
#pragma unroll
        for( int i = 0; i < 8; i++ ) { p[2 * i] = (int)( w[i] & 0xffffu ); p[2 * i + 1] = (int)( w[i] >> 16 ); }
        int s = p[0] + p[1] + p[2] + p[3] + p[4] + p[5] + p[6] + p[7];
        uint32_t o[4];
#pragma unroll
        for( int k = 0; k < 8; k++ )
        {
          if( k ) s += p[k + 7] - p[k - 1];
          if( k & 1 ) o[k >> 1] |= (uint32_t) s << 16; else o[k >> 1] = (uint32_t) s;
        }
        *reinterpret_cast<uint4*>( Hs + r * L.vPitch + st * 8 ) = make_uint4( o[0], o[1], o[2], o[3] );
      }
      // a thread per (block, 8 entries): nxp and bStride are multiples of 8, so the 8 entries are all column bits or all row bits
      const int bChunks = L.bStride >> 3;
      const float invB = 1.0f / (float) bChunks;
      for( int t = tid; t < NBLK * bChunks; t += nthr )
      {
        const int bid = pyr_div<NXY>( t, bChunks, invB ), e0 = 8 * ( t - bid * bChunks );
        const int2 pr = sPred[bid];
        uint32_t w[2] = { 0u, 0u };
#pragma unroll
        for( int k = 0; k < 8; k++ )
        {
          const int e = e0 + k;
          uint32_t v;
          if( e0 < nxp ) v = e < nx ? eg_bits( ( ( rb.left + e ) * ( 1 << par.costScale ) - pr.x ) >> par.imvShift ) : (uint32_t) PYR_PAD_BITS;
          else           v = 4u * eg_bits( ( ( rb.top + ( e - nxp ) ) * ( 1 << par.costScale ) - pr.y ) >> par.imvShift );
          w[k >> 2] |= ( v & 0xffu ) << ( 8 * ( k & 3 ) );
        }
        *reinterpret_cast<uint2*>( bitsS + bid * L.bStride + e0 ) = make_uint2( w[0], w[1] );
      }
    }
    __syncthreads();
    // ---- box sums V[r][c] = sum_{y<8} Hs[r+y][c]  (uint16: 64 * 1023 fits; pyramidV2Usable sends planes above 10 bits to engine 0); a thread slides down
    // a chunk of rows of one column pair
    {
      const int cPairs = L.vPitch >> 1, chunk = 16, nChunks = ( L.vRows + chunk - 1 ) / chunk;
      const uint32_t* Hs32 = reinterpret_cast<const uint32_t*>( Hs );
      uint32_t* V32 = reinterpret_cast<uint32_t*>( V );
      for( int t = tid; t < cPairs * nChunks; t += nthr )
      {
        const int ch = t / cPairs, c = t - ch * cPairs;
        const int r0 = ch * chunk, r1 = min( L.vRows, r0 + chunk );
        uint32_t s = 0;                                                           // two uint16 lanes, no carry: each lane stays below 2^16
        for( int y = 0; y < 8; y++ ) s += Hs32[( r0 + y ) * cPairs + c];
        V32[r0 * cPairs + c] = s;
        for( int r = r0 + 1; r < r1; r++ ) { s += Hs32[( r + 7 ) * cPairs + c] - Hs32[( r - 1 ) * cPairs + c]; V32[r * cPairs + c] = s; }
      }
    }
    __syncthreads();
    // ---- one-pel-shifted copy of the window, over the row sums
    for( int i = tid; i < winH * wsw; i += nthr ) win1w[i] = __funnelshift_r( win0w[i], win0w[i + 1], 16 );
    __syncthreads();
    PYR_MARK( 2 );

    // ---- next root of the run: L2 prefetches of its descriptors, cp.async copies of its originals into the other originals buffer (L2 prefetches where the
    // buffer does not fit or the rows are not 16-byte aligned), and, when it can carry this window, cp.async copies of its new window columns into the staging
    // area.  They complete behind this root's candidate loop; the wait comes after the results, the next root's first barrier publishes them.
    bool carryNext = false, orgNext = false;
    if( WALK && root + 1 < rEnd )
    {
      const vvb_block nb = lv.blocks[LTOP][root + 1];
      for( int t = tid; t < NBLK; t += nthr )
      {
        const int l = t < OFF1 ? 0 : ( t < OFF2 ? 1 : ( t < OFF3 ? 2 : 3 ) );
        const int i = t - ( l == 0 ? 0 : ( l == 1 ? OFF1 : ( l == 2 ? OFF2 : OFF3 ) ) );
        pyr_prefetch_l2( &lv.blocks[l][( (size_t)( root + 1 ) << ( 2 * ( LTOP - l ) ) ) + i] );
      }
      const int16_t* so = orgPlane.origin + (ptrdiff_t) nb.y * orgPlane.stride + nb.x;
      orgNext = L.offOrgNext > 0 && ( ( (uintptr_t) so & 15 ) == 0 ) && ( ( orgPlane.stride & 7 ) == 0 );
      if( orgNext )
      {
        for( int i = tid; i < R * ( R / 8 ); i += nthr )
        {
          const int r = i / ( R / 8 ), c = i - r * ( R / 8 );
          pyr_cp_async16( orgN + r * R + 8 * c, so + (ptrdiff_t) r * orgPlane.stride + 8 * c );
        }
      }
      else if( tid < 2 * R ) pyr_prefetch_l2( so + (ptrdiff_t)( tid >> 1 ) * orgPlane.stride + ( tid & 1 ) * ( R - 1 ) );     // first and last pel of every row
      carryNext = L.stageWords > 0 && src32 && nb.x == rb.x + R && nb.y == rb.y && nb.left == rb.left && nb.right == rb.right && nb.top == rb.top &&
                  nb.bottom == rb.bottom;
      if( carryNext )
      {
        const int16_t* sn = src + R + 2 * keepWords;                      // the next window's first new word (its window starts R pels to the right)
        if( ( ( (uintptr_t) sn & 15 ) == 0 ) && ( ( refPlane.stride & 7 ) == 0 ) )
        {
          for( int i = tid; i < winH * ( R / 8 ); i += nthr )
          {
            const int r = i / ( R / 8 ), c = i - r * ( R / 8 );
            pyr_cp_async16( stage + r * ( R / 2 ) + 4 * c, sn + (ptrdiff_t) r * refPlane.stride + 8 * c );
          }
        }
        else
        {
          for( int i = tid; i < winH * ( R / 2 ); i += nthr )
          {
            const int r = i / ( R / 2 ), c = i - r * ( R / 2 );
            pyr_cp_async4( stage + i, sn + (ptrdiff_t) r * refPlane.stride + 2 * c );
          }
        }
      }
    }

    // ---- candidates.  Strip item = (quad of four 8x8 members, pair of candidate rows, strip of 8 vectors); column item = (quad, one of the nx % 8 rightmost
    // columns, group of 8 vertically adjacent vectors).  Both kinds share one item space, so the column items run in the short last round of the strip items
    // instead of a round of their own.
    {
      // Lane mapping.  A quarter warp's LDS.128 is one wavefront when its 8 lanes read 8 consecutive 16-byte chunks: main items are groups of 8 adjacent strips
      // of one row pair (it = ((q * nPairs + pr) * nMain + st), st fastest); the strips left over when the range is not a multiple of 64 vectors follow as
      // tail items with the row pair as the fast index.
      const int nFull = nx >> 3, nCols = nx & 7;                // full strips of 8 vectors; the nx % 8 columns left of them are column items
      const int nPairs = ( ny + 1 ) >> 1, nMain = nFull & ~7, nTail = nFull - nMain;
      const int perQm = nPairs * nMain, itemsMain = NQ * perQm, perQt = nPairs * nTail, itemsStrip = itemsMain + NQ * perQt;
      const int nV = ( ny + 7 ) >> 3, perQc = nCols * nV, items = itemsStrip + NQ * perQc;
      const float invPerQm = 1.0f / (float) max( 1, perQm ), invMain = 1.0f / (float) max( 1, nMain ), invPerQt = 1.0f / (float) max( 1, perQt ), invPairs = 1.0f / (float) nPairs;
      const float invPerQc = 1.0f / (float) max( 1, perQc ), invNv = 1.0f / (float) nV;
      const uint32_t* org32 = reinterpret_cast<const uint32_t*>( orgS );
      const uint32_t mvBase = (uint32_t) __cvta_generic_to_shared( sMv8 );
      const int vPitch = L.vPitch, bStride = L.bStride;
      for( int base = 0; base < items; base += nthr )
      {
        const int it = base + tid;
        const bool isStrip = it < itemsStrip, isCol = !isStrip && it < items;
        const unsigned maskS = __ballot_sync( 0xffffffffu, isStrip ), maskC = __ballot_sync( 0xffffffffu, isCol );
        if( isStrip )
        {
          const unsigned mask = maskS;
          int q, pr, st;
          if( it < itemsMain ) { q = pyr_div<NXY>( it, max( 1, perQm ), invPerQm ); const int rem = it - q * perQm; pr = pyr_div<NXY>( rem, max( 1, nMain ), invMain ); st = rem - pr * nMain; }
          else
          {
            const int i2 = it - itemsMain; q = pyr_div<NXY>( i2, max( 1, perQt ), invPerQt ); const int rem = i2 - q * perQt;
            const int ts = pyr_div<NXY>( rem, nPairs, invPairs ); pr = rem - ts * nPairs; st = nMain + ts;
          }
          const int cy = 2 * pr, cx0 = 8 * st;
          const bool validB = cy + 1 < ny;
          const int lead = __ffs( mask ) - 1;
          const bool uni = __all_sync( mask, q == __shfl_sync( mask, q, lead ) );
          const int qx = ( q & 1 ) | ( ( q >> 1 ) & 2 ), qy = ( ( q >> 1 ) & 1 ) | ( ( q >> 2 ) & 2 );     // z-order position of the quad (q < 16)
          uint32_t psA[8], psB[8];
#pragma unroll
          for( int k = 0; k < 8; k++ ) { psA[k] = 0u; psB[k] = 0u; }
          // member 0 of the quad; member m lies (m & 1) * 8 pels right and (m >> 1) * 8 rows down of it in the originals, the window and V
          const uint32_t* op = org32 + ( qy * 16 ) * ( R / 2 ) + qx * 8;
          const int wofs = ( qy * 16 + cy ) * wsw + qx * 8 + ( cx0 >> 1 );
          const uint32_t* w0 = win0w + wofs;
          const uint32_t* w1 = win1w + wofs;
          const uint16_t* vrow = V + ( qy * 16 + cy ) * vPitch + qx * 16 + cx0;
          const unsigned char* bb = bitsS + 4 * q * bStride;
#pragma unroll 1
          for( int m = 0; m < 4; m++ )
          {
            const int b0 = 4 * q + m;
            const int sumA = sSumA[b0];
            // per slot and row, max(b - a, 0) of the 32 pel-pair words (HFMA2.RELU, fma pipe) summed as two uint16 lanes: 32 * 1023 leaves no carry, and one
            // IADD3 (alu pipe) adds two words
            uint32_t pA[8], pB[8];
#pragma unroll
            for( int k = 0; k < 8; k++ ) { pA[k] = 0u; pB[k] = 0u; }
            uint4 oPrev = make_uint4( 0, 0, 0, 0 );
#pragma unroll
            for( int y = 0; y < 9; y++ )
            {
              const uint4 e0 = *reinterpret_cast<const uint4*>( w0 + y * wsw ), e1 = *reinterpret_cast<const uint4*>( w0 + y * wsw + 4 );
              const uint4 d0 = *reinterpret_cast<const uint4*>( w1 + y * wsw ), d1 = *reinterpret_cast<const uint4*>( w1 + y * wsw + 4 );
              const uint32_t e[8] = { e0.x, e0.y, e0.z, e0.w, e1.x, e1.y, e1.z, e1.w };
              const uint32_t d[8] = { d0.x, d0.y, d0.z, d0.w, d1.x, d1.y, d1.z, d1.w };
              uint4 oCur = oPrev;
              if( y < 8 )
              {
                oCur = *reinterpret_cast<const uint4*>( op + y * ( R / 2 ) );
                const uint32_t o[4] = { oCur.x, oCur.y, oCur.z, oCur.w };
#pragma unroll
                for( int k = 0; k < 8; k++ )
#pragma unroll
                  for( int i = 0; i < 4; i += 2 )
                  {
                    const uint32_t wa = ( k & 1 ) ? d[i + ( k >> 1 )] : e[i + ( k >> 1 )], wb = ( k & 1 ) ? d[i + 1 + ( k >> 1 )] : e[i + 1 + ( k >> 1 )];
                    pA[k] += pyr_relu_diff( o[i], wa ) + pyr_relu_diff( o[i + 1], wb );
                  }
              }
              if( y > 0 )
              {
                const uint32_t o[4] = { oPrev.x, oPrev.y, oPrev.z, oPrev.w };
#pragma unroll
                for( int k = 0; k < 8; k++ )
#pragma unroll
                  for( int i = 0; i < 4; i += 2 )
                  {
                    const uint32_t wa = ( k & 1 ) ? d[i + ( k >> 1 )] : e[i + ( k >> 1 )], wb = ( k & 1 ) ? d[i + 1 + ( k >> 1 )] : e[i + 1 + ( k >> 1 )];
                    pB[k] += pyr_relu_diff( o[i], wa ) + pyr_relu_diff( o[i + 1], wb );
                  }
              }
              oPrev = oCur;
            }
            int accA[8], accB[8];
#pragma unroll
            for( int k = 0; k < 8; k++ ) { accA[k] = __dp2a_lo( (int) pA[k], 0x0202, sumA ); accB[k] = __dp2a_lo( (int) pB[k], 0x0202, sumA ); }
            // member epilogue
            const uint2 bw = *reinterpret_cast<const uint2*>( bb + cx0 );
            uint32_t bk = pyr_finish_row( accA, vrow, bw, mvBase + bb[nxp + cy], one, eight, psA );
            uint32_t key = ( ( bk >> 3 ) << ob ) + (uint32_t)( cy * nx + cx0 ) + ( bk & 7u );
            if( validB )
            {
              bk = pyr_finish_row( accB, vrow + vPitch, bw, mvBase + bb[nxp + cy + 1], one, eight, psB );
              key = min( key, ( ( bk >> 3 ) << ob ) + (uint32_t)( ( cy + 1 ) * nx + cx0 ) + ( bk & 7u ) );
            }
            if( uni ) { key = __reduce_min_sync( mask, key ); if( lane == lead ) atomicMin( &sKey32[b0], key ); }
            else atomicMin( &sKey32[b0], key );
            const bool right = !( m & 1 );                        // next member: one to the right, or back left and one down
            op   += right ? 4 : 8 * ( R / 2 ) - 4;
            w0   += right ? 4 : 8 * wsw - 4;
            w1   += right ? 4 : 8 * wsw - 4;
            vrow += right ? 8 : 8 * vPitch - 8;
            bb   += bStride;
          }
          // the 16x16 parent of the quad: its SAD at a vector is the sum of the members' SADs
          {
            const unsigned char* pb = bitsS + ( OFF1 + q ) * bStride;
            const uint2 bw = *reinterpret_cast<const uint2*>( pb + cx0 );
            uint32_t* trow = LV >= 3 ? T + ( LV == 4 ? ( q >> 2 ) : 0 ) * L.tStride + cy * nxp + st : nullptr;      // table layout [cy][slot k][strip]: a warp's atomics spread over the banks
            uint32_t key = 0xffffffffu;
#pragma unroll
            for( int rowB = 0; rowB < 2; rowB++ )
            {
              if( rowB && !validB ) break;
              const uint32_t mvRow = mvBase + pb[nxp + cy + rowB];
              uint32_t bk = 0xffffffffu;
#pragma unroll
              for( int k = 0; k < 8; k++ )
              {
                const uint32_t ps  = rowB ? psB[k] : psA[k];
                const uint32_t a   = __dp4a( k < 4 ? bw.x : bw.y, 4u << ( 8 * ( k & 3 ) ), mvRow );
                const uint32_t mvk = pyr_lds( a + k * ( PYR_MVN * 4 ) );
                bk = min( bk, ps * eight + mvk );
                if( LV >= 3 ) atomicAdd( trow + rowB * nxp + k * nStrips, ps );
              }
              key = min( key, ( ( bk >> 3 ) << ob ) + (uint32_t)( ( cy + rowB ) * nx + cx0 ) + ( bk & 7u ) );
            }
            if( uni ) { key = __reduce_min_sync( mask, key ); if( lane == lead ) atomicMin( &sKey32[OFF1 + q], key ); }
            else atomicMin( &sKey32[OFF1 + q], key );
          }
        }
        else if( isCol )
        {
          // A strip item would spend a full strip of work on one column; here the thread keeps the member's eight original rows in registers and walks the
          // 15 window rows its 8 vectors touch: window row r meets original row r - c for vector c.
          const unsigned mask = maskC;
          const int ic = it - itemsStrip;
          const int q = pyr_div<NXY>( ic, max( 1, perQc ), invPerQc ), rem = ic - q * perQc;
          const int ci = pyr_div<NXY>( rem, nV, invNv ), g = rem - ci * nV;
          const int cx = 8 * nFull + ci, cy0 = 8 * g;
          const int lead = __ffs( mask ) - 1;
          const bool uni = __all_sync( mask, q == __shfl_sync( mask, q, lead ) );
          const int qx = ( q & 1 ) | ( ( q >> 1 ) & 2 ), qy = ( ( q >> 1 ) & 1 ) | ( ( q >> 2 ) & 2 );
          const uint32_t* wsrc = ( cx & 1 ) ? win1w : win0w;      // odd columns read the one-pel-shifted copy
          const int cw = cx >> 1;                                 // word offset of the column inside a window row
          uint32_t ps[8];
#pragma unroll
          for( int c = 0; c < 8; c++ ) ps[c] = 0u;
#pragma unroll 1
          for( int m = 0; m < 4; m++ )
          {
            const int bx8 = 2 * qx + ( m & 1 ), by8 = 2 * qy + ( m >> 1 ), b0 = 4 * q + m;
            const int sumA = sSumA[b0];
            uint32_t o[8][4];
#pragma unroll
            for( int y = 0; y < 8; y++ )
            {
              const uint4 ov = *reinterpret_cast<const uint4*>( org32 + ( by8 * 8 + y ) * ( R / 2 ) + bx8 * 4 );
              o[y][0] = ov.x; o[y][1] = ov.y; o[y][2] = ov.z; o[y][3] = ov.w;
            }
            int acc[8];
#pragma unroll
            for( int c = 0; c < 8; c++ ) acc[c] = sumA;
            const uint32_t* wp = wsrc + ( by8 * 8 + cy0 ) * wsw + bx8 * 4 + cw;
#pragma unroll
            for( int r = 0; r < 15; r++ )
            {
              uint32_t w[4];
              if( ( cw & 3 ) == 0 ) { const uint4 wv = *reinterpret_cast<const uint4*>( wp + r * wsw ); w[0] = wv.x; w[1] = wv.y; w[2] = wv.z; w[3] = wv.w; }
              else { w[0] = wp[r * wsw]; w[1] = wp[r * wsw + 1]; w[2] = wp[r * wsw + 2]; w[3] = wp[r * wsw + 3]; }
#pragma unroll
              for( int c = 0; c < 8; c++ )
              {
                if( r - c >= 0 && r - c < 8 )
                {
#pragma unroll
                  for( int i = 0; i < 4; i++ ) acc[c] = __dp2a_lo( (int) __vmins2( o[r - c][i], w[i] ), (int) 0x0000fefeu, acc[c] );
                }
              }
            }
            const unsigned char* bb = bitsS + b0 * bStride;
            const uint32_t mvCol = mvBase + 4u * bb[cx];
            const uint2 byw = *reinterpret_cast<const uint2*>( bb + nxp + cy0 );
            const uint16_t* vcol = V + ( by8 * 8 + cy0 ) * vPitch + bx8 * 8 + cx;
            uint32_t bk = 0xffffffffu;
#pragma unroll
            for( int c = 0; c < 8; c++ )
            {
              const uint32_t a   = __dp4a( c < 4 ? byw.x : byw.y, 1u << ( 8 * ( c & 3 ) ), mvCol );           // row bits are stored times 4
              const uint32_t mvk = pyr_lds( a + c * ( PYR_MVN * 4 ) );
              const uint32_t sad = (uint32_t)( (int) vcol[c * vPitch] + acc[c] );
              ps[c] += sad;
              const uint32_t key = cy0 + c < ny ? sad * eight + mvk : 0xffffffffu;
              bk = min( bk, key );
            }
            uint32_t key = ( ( bk >> 3 ) << ob ) + (uint32_t)( ( cy0 + (int)( bk & 7u ) ) * nx + cx );
            if( uni ) { key = __reduce_min_sync( mask, key ); if( lane == lead ) atomicMin( &sKey32[b0], key ); }
            else atomicMin( &sKey32[b0], key );
          }
          {
            const unsigned char* bb = bitsS + ( OFF1 + q ) * bStride;
            const uint32_t mvCol = mvBase + 4u * bb[cx];
            const uint2 byw = *reinterpret_cast<const uint2*>( bb + nxp + cy0 );
            uint32_t* tcol = LV >= 3 ? T + ( LV == 4 ? ( q >> 2 ) : 0 ) * L.tStride + cy0 * nxp + ( cx & 7 ) * nStrips + ( cx >> 3 ) : nullptr;
            uint32_t bk = 0xffffffffu;
#pragma unroll
            for( int c = 0; c < 8; c++ )
            {
              const uint32_t a   = __dp4a( c < 4 ? byw.x : byw.y, 1u << ( 8 * ( c & 3 ) ), mvCol );
              const uint32_t mvk = pyr_lds( a + c * ( PYR_MVN * 4 ) );
              if( cy0 + c < ny )
              {
                bk = min( bk, ps[c] * eight + mvk );
                if( LV >= 3 ) atomicAdd( tcol + c * nxp, ps[c] );
              }
            }
            uint32_t key = ( ( bk >> 3 ) << ob ) + (uint32_t)( ( cy0 + (int)( bk & 7u ) ) * nx + cx );
            if( uni ) { key = __reduce_min_sync( mask, key ); if( lane == lead ) atomicMin( &sKey32[OFF1 + q], key ); }
            else atomicMin( &sKey32[OFF1 + q], key );
          }
        }
      }
    }
    __syncthreads();
    PYR_MARK( 3 );

    // ---- 32x32 blocks from their tables and the 64x64 root from the sum of the four, in one pass: every table entry is read once
    if( LV >= 3 )
    {
      constexpr int NTOP = LV == 4 ? NT + 1 : 1;
      const float invNx = 1.0f / (float) nx;
      unsigned long long best[NTOP];
#pragma unroll
      for( int j = 0; j < NTOP; j++ ) best[j] = ~0ull;
      for( int o = tid; o < nx * ny; o += nthr )
      {
        const int cy = pyr_div<NXY>( o, nx, invNx ), cx = o - cy * nx;
        const int ti = cy * nxp + ( cx & 7 ) * nStrips + ( cx >> 3 );
        uint32_t sum = 0u;
#pragma unroll
        for( int j = 0; j < NTOP; j++ )
        {
          uint32_t s;
          if( j < NT ) { s = T[j * L.tStride + ti]; T[j * L.tStride + ti] = 0u; sum += s; }      // cleared for the next root
          else         s = sum;
          const unsigned char* bb = bitsS + ( j < NT ? OFF2 + j : OFF3 ) * L.bStride;
          const uint32_t bits = (uint32_t) bb[cx] + ( (uint32_t) bb[nxp + cy] >> 2 );
          const unsigned long long key = ( ( (unsigned long long) s + sMvRaw[bits < VVB_MVCOST_ENTRIES ? bits : VVB_MVCOST_ENTRIES - 1] ) << 16 ) | (unsigned) o;
          best[j] = key < best[j] ? key : best[j];
        }
      }
#pragma unroll
      for( int j = 0; j < NTOP; j++ )
      {
#pragma unroll
        for( int mm = 16; mm > 0; mm >>= 1 ) { const unsigned long long o2 = __shfl_xor_sync( 0xffffffffu, best[j], mm ); best[j] = o2 < best[j] ? o2 : best[j]; }
        if( lane == 0 && best[j] != ~0ull ) atomicMin( &sKey64[j], best[j] );
      }
      __syncthreads();
    }
    PYR_MARK( 4 );

    // ---- results
    for( int t = tid; t < NBLK; t += nthr )
    {
      const int l = t < OFF1 ? 0 : ( t < OFF2 ? 1 : ( t < OFF3 ? 2 : 3 ) );
      const int i = t - ( l == 0 ? 0 : ( l == 1 ? OFF1 : ( l == 2 ? OFF2 : OFF3 ) ) );
      unsigned long long cost; uint32_t order;
      if( l < 2 ) { const uint32_t k = sKey32[t]; cost = k >> ob; order = k & ( ( 1u << ob ) - 1u ); }
      else        { const unsigned long long k = sKey64[l == 2 ? i : L.nT]; cost = k >> 16; order = (uint32_t)( k & 0xffffu ); }
      const int cy = order / nx, cx = order - cy * nx;
      const unsigned char* bb = bitsS + t * L.bStride;
      const uint32_t bits = (uint32_t) bb[cx] + ( (uint32_t) bb[nxp + cy] >> 2 );
      vvb_best b;
      b.dx = (int16_t)( rb.left + cx ); b.dy = (int16_t)( rb.top + cy ); b.cost = cost;
      b.sad = (uint32_t)( cost - sMvRaw[bits < VVB_MVCOST_ENTRIES ? bits : VVB_MVCOST_ENTRIES - 1] );
      lv.best[l][( (size_t) root << ( 2 * ( LTOP - l ) ) ) + i] = b;
    }
    if( carryNext || orgNext ) pyr_cp_async_wait_all();
    carry = carryNext;
    orgStaged = orgNext;
#ifdef VVB_PYR_PHASES
    __syncthreads();
    PYR_MARK( 5 );
    if( tid == 0 ) atomicAdd( &g_pyrPhaseNs[LV - 2][PYR_NPHASE], 1ull );
#endif
  }
}

} // namespace vvb
