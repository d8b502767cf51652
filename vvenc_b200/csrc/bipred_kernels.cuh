// bipred_kernels.cuh -- the bi-predictive branch of InterSearch::xMotionEstimation (EncoderLib/InterSearch.cpp:1994-2005, 2046-2094, 2110-2125) on the device.
//
// Two launches per call.  bipred_int_kernel gives each PU one persistent warp, as tz_search_kernel does: the warp forms the search target 2 * org - pred
// (AreaBuf::removeHighFreq, Buffer.h:448-480) once in shared memory from the original plane and the other list's prediction, lists the start vector and the
// candidates that do not repeat an earlier one (:2051-2090), then the xPatternSearch window around the winner (:2092-2093, :2209-2251), and evaluates each list
// with tz_flush: G-lane groups sum the SADs (group_sad, target read from shared memory), every lane applies the strict `<` in list order.  The target spans
// -(2^bd - 1) .. 2^(bd + 1) - 2 and fits int16 for bd <= 12; group_sad's packed arithmetic (VIMNMX.S16x2, IDP.2A) is signed, so it takes the target as it is.
// frac_search_kernel<FracOrgTarget> then runs xPatternSearchFracDIF on the same target (formed again from the plane and the pool while the window is staged)
// and ends with the final cost of :2117-2124 (bi_finish).  With m_fastSubPel == 2 there is no fractional stage and bipred_int_kernel ends with bi_finish.
#pragma once
#include "common.cuh"
#include "tz_kernels.cuh"
#include "frac_search_kernels.cuh"

namespace vvb {

static_assert( sizeof( vvb_bi_pu ) == 36 && sizeof( vvb_bi_best ) == 56 && sizeof( vvb_bi_par ) == 56, "vvb_bi_pu / vvb_bi_best / vvb_bi_par layout" );

// what the target and the final cost need: ClipPel of the target, the MV rate of the final vector, the BCW weight of the list
struct BiPar { int clip, maxv, imvShift, refList; double motionLambda; };

__device__ __forceinline__ int bi_target( int o, int p, const BiPar& bp ) { const int t = 2 * o - p; return bp.clip ? min( max( t, 0 ), bp.maxv ) : t; }

// (Distortion) of a double as the x86-64 encoder converts it (InterSearch.cpp:2123 in the reference build: comisd against 2^63, then cvttsd2si below, or
// cvttsd2si of v - 2^63 with the top bit flipped at or above).  cvttsd2si gives 0x8000000000000000 for NaN and for values outside the int64 range, so a
// negative value -k becomes 2^64 - k, a value below -2^63 or a NaN becomes 2^63, and a value at or above 2^64 becomes 0.
__device__ __forceinline__ unsigned long long x86_cvttsd2si( double v ) { return v >= -9223372036854775808.0 && v < 9223372036854775808.0 ? (unsigned long long) __double2ll_rz( v ) : 0x8000000000000000ull; }
__device__ __forceinline__ unsigned long long x86_double_to_u64( double v )
{
  const double two63 = 9223372036854775808.0;
  return v >= two63 ? x86_cvttsd2si( __dsub_rn( v, two63 ) ) ^ 0x8000000000000000ull : x86_cvttsd2si( v );
}

// RdCost::getCost( b ) = Distortion( m_motionLambda * b ) (RdCost.h:181)
__device__ __forceinline__ unsigned long long motion_cost( double motionLambda, uint32_t b ) { return x86_double_to_u64( __dmul_rn( motionLambda, (double) b ) ); }
__device__ __forceinline__ unsigned long long bi_get_cost( const BiPar& bp, uint32_t b ) { return motion_cost( bp.motionLambda, b ); }

// xGetMEDistortionWeight (InterSearch.cpp:4257-4267): | getBcwWeight( bcw_idx, refList ) | / 8, or 0.5 for BCW_DEFAULT
__device__ __forceinline__ double bcw_me_weight( int bcwIdx, int refList )
{
  const int bw = bcwIdx == 0 ? -2 : bcwIdx == 1 ? 3 : bcwIdx == 3 ? 5 : 10;        // g_BcwWeights (Rom.cpp:1152)
  return bcwIdx == 2 ? 0.5 : fabs( (double)( refList == 0 ? 8 - bw : bw ) * 0.125 );      // = / 8.0 exactly
}

// :2117-2124: the final vector in internal units, ruiBits and the BCW-weighted ruiCost; cost is ruiCost after the fractional stage
__device__ __forceinline__ void bi_finish( const BiPar& bp, const vvb_bi_pu& pu, int mx, int my, int halfH, int halfV, int qterH, int qterV,
                                           unsigned long long cost, vvb_bi_best& r )
{
  const int qx = mx * 4 + halfH * 2 + qterH, qy = my * 4 + halfV * 2 + qterV;
  const uint32_t mvBits = eg_bits( ( qx - pu.pred_hor ) >> bp.imvShift ) + eg_bits( ( qy - pu.pred_ver ) >> bp.imvShift );
  const uint32_t bits = pu.bits + mvBits;
  const double weight = bcw_me_weight( pu.bcw_idx, bp.refList );
  const double d = __dsub_rn( __ull2double_rn( cost ), __ull2double_rn( bi_get_cost( bp, mvBits ) ) );
  r.frac_cost = cost;
  r.half_hor = (int16_t) halfH; r.half_ver = (int16_t) halfV; r.qter_hor = (int16_t) qterH; r.qter_ver = (int16_t) qterV;
  r.mv_hor = qx * 4; r.mv_ver = qy * 4;
  r.bits = bits; r.pad = 0;
  r.cost = x86_double_to_u64( __dadd_rn( floor( __dmul_rn( weight, d ) ), __ull2double_rn( bi_get_cost( bp, bits ) ) ) );
}

__device__ __forceinline__ vvb_bi_best bi_sentinel() { vvb_bi_best r{}; r.int_best = ~0ull; r.frac_cost = ~0ull; r.cost = ~0ull; return r; }

// The read box of a PU (the header's rule): the blocks at its clipped start and candidate vectors, and the fractional stage's box (frac_search_admitted) around the
// corners of the window centred on each of them, or around the zero vector when that window is empty.  Every lane of a warp evaluates it alike.
__host__ __device__ inline bool bi_admitted( const TzPar& p, const Plane& ref, const vvb_bi_pu& pu, const int32_t* cands )
{
  const TzClip cs = tz_clip_box( p, pu.x, pu.y, true );
  const long long m = ref.margin;
  for( int c = -1; c < pu.cand_count; c++ )
  {
    const int h = c < 0 ? pu.start_hor : cands[2 * ( pu.cand_first + c )], v = c < 0 ? pu.start_ver : cands[2 * ( pu.cand_first + c ) + 1];
    const long long sx = pu.x + tz_round_shift( tz_clamp( h, cs.horMin, cs.horMax ), 4 ), sy = pu.y + tz_round_shift( tz_clamp( v, cs.verMin, cs.verMax ), 4 );
    if( sx < -m || sx + p.w > ref.width + m || sy < -m || sy + p.h > ref.height + m ) return false;
    int l, r, t, b;
    tz_search_range( p, pu.x, pu.y, h, v, p.searchRange, l, r, t, b );
    if( l > r || t > b ) { l = r = t = b = 0; }
    if( !frac_search_admitted( ref, pu.x, pu.y, l, t, p.w, p.h ) || !frac_search_admitted( ref, pu.x, pu.y, r, b, p.w, p.h ) ) return false;
  }
  return true;
}

// frac_search_kernel's source for the bi branch: vvb_bi_pu, the target formed from the original plane and pred, vvb_bi_best with bi_finish
struct FracOrgTarget
{
  using Pu = vvb_bi_pu;
  using Out = vvb_bi_best;
  const int16_t* pred;              // [n][h][w]
  int wh;
  BiPar bp;
  __device__ __forceinline__ uint32_t org_pair( const int16_t* q, int b, int i ) const
  {
    const int16_t* pp = pred + (size_t) b * wh + 2 * i;
    return (uint32_t)(uint16_t) bi_target( __ldg( q ), __ldg( pp ), bp ) | ( (uint32_t)(uint16_t) bi_target( __ldg( q + 1 ), __ldg( pp + 1 ), bp ) << 16 );
  }
  // the fractional stage leaves the integer fields to bipred_int_kernel; a PU that the integer stage refused arrives here with an inadmissible vector
  __device__ __forceinline__ void fail( Out* out, int b ) const { out[b].frac_cost = ~0ull; out[b].cost = ~0ull; }
  __device__ __forceinline__ void done( Out* out, int b, const Pu& pu, int mx, int my, const vvb_frac_best& f ) const
  {
    vvb_bi_best r = out[b];
    bi_finish( bp, pu, mx, my, f.half_hor, f.half_ver, f.qter_hor, f.qter_ver, f.cost, r );
    out[b] = r;
  }
};

// integer vector of a refused PU: no reference margin admits it, so the fractional stage refuses it without reading
#define BI_REFUSED_MV ( -( 1 << 30 ) )

template<int G>
__global__ void __launch_bounds__( 128, 1 ) bipred_int_kernel( const __grid_constant__ Plane orgPlane, const __grid_constant__ Plane refPlane,
                                                            const vvb_bi_pu* __restrict__ pus, int n, const int32_t* __restrict__ cands,
                                                            const int16_t* __restrict__ pred, const __grid_constant__ TzPar p, const __grid_constant__ MePar mp,
                                                            const __grid_constant__ BiPar bp, int finish, vvb_tz_best* __restrict__ intOut, vvb_bi_best* __restrict__ out )
{
  extern __shared__ __align__( 16 ) uint8_t biSmem[];
  __shared__ uint32_t sMv[VVB_MVCOST_ENTRIES];
  TzWarp W = tz_warp_begin( biSmem, sMv, p, mp, refPlane );
  int16_t* tgt = W.org;
  const int lane = W.lane, warp = threadIdx.x >> 5, warpsPerGrid = gridDim.x * ( blockDim.x >> 5 );

  for( int i = blockIdx.x * ( blockDim.x >> 5 ) + warp; i < n; i += warpsPerGrid )     // persistent warps, as tz_search_kernel
  {
    const vvb_bi_pu pu = pus[i];
    if( TZ_PU_OUTSIDE( p, pu ) || pu.bcw_idx < 0 || pu.bcw_idx > 4 || !bi_admitted( p, refPlane, pu, cands ) )
    {
      if( lane == 0 ) { vvb_tz_best t{}; t.mv_hor = t.mv_ver = BI_REFUSED_MV; intOut[i] = t; out[i] = bi_sentinel(); }
      continue;
    }
    __syncwarp();                           // the previous PU's target is no longer read
    {
      const int16_t* src = orgPlane.origin + (ptrdiff_t) pu.y * orgPlane.stride + pu.x;
      const int16_t* pp = pred + (size_t) i * p.w * p.h;
      for( int e = lane; e < p.w * p.h; e += 32 ) { const int y = e / p.w; tgt[e] = (int16_t) bi_target( __ldg( src + (ptrdiff_t) y * orgPlane.stride + e - y * p.w ), __ldg( pp + e ), bp ); }
    }
    __syncwarp();
    W.ref = refPlane.origin + (ptrdiff_t) pu.y * refPlane.stride + pu.x;

    TzState s;
    tz_reset( s );
    TzWalk<G> T{ W, s, p, mp, sMv, pu.pred_hor, pu.pred_ver };
    const TzClip cs = tz_clip_box( p, pu.x, pu.y, true );

    // the start vector and the candidates that do not repeat an earlier one (:2051-2090); the entry's distance field holds its index (0: the start vector)
    T.add( tz_round_shift( tz_clamp( pu.start_hor, cs.horMin, cs.horMax ), 4 ), tz_round_shift( tz_clamp( pu.start_ver, cs.verMin, cs.verMax ), 4 ), 0, 0 );
    for( int c = 0; c < pu.cand_count; c++ )
    {
      const int j = pu.cand_first + c, ch = cands[2 * j], cv = cands[2 * j + 1];
      bool repeat = false;
      for( int k = pu.cand_first; k < j && !repeat; k++ ) repeat = cands[2 * k] == ch && cands[2 * k + 1] == cv;
      if( repeat ) continue;
      if( W.cnt == TZ_LIST ) T.flush();
      T.add( tz_round_shift( tz_clamp( ch, cs.horMin, cs.horMax ), 4 ), tz_round_shift( tz_clamp( cv, cs.verMin, cs.verMax ), 4 ), 0, c + 1 );
    }
    T.flush();
    const int win = (int) s.bestDistance;
    const int initH = win ? cands[2 * ( pu.cand_first + win - 1 )] : pu.start_hor, initV = win ? cands[2 * ( pu.cand_first + win - 1 ) + 1] : pu.start_ver;

    // xSetSearchRange around the unclipped winner, then xPatternSearch from uiSadBest = MAX_DISTORTION and (0, 0)
    int l, r, t, b;
    tz_search_range( p, pu.x, pu.y, initH, initV, p.searchRange, l, r, t, b );
    tz_reset( s );
    T.raster( t, b, l, r, 1 );
    if( lane == 0 )
    {
      const vvb_tz_best ib = tz_best( s, mp, sMv, pu.pred_hor, pu.pred_ver, 0 );
      intOut[i] = ib;
      vvb_bi_best o = bi_sentinel();
      o.int_hor = s.bestX; o.int_ver = s.bestY; o.int_best = s.bestSad;
      if( finish ) bi_finish( bp, pu, s.bestX, s.bestY, 0, 0, 0, 0, ib.sad, o );
      out[i] = o;
    }
  }
}

} // namespace vvb
