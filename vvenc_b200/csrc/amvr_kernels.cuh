// amvr_kernels.cuh -- InterSearch::xPatternSearchIntRefine (EncoderLib/InterSearch.cpp:2576-2676), the AMVR end of xMotionEstimation, on the device.
//
// One persistent warp per PU, as tz_search_kernel and bipred_int_kernel (tz_warp_begin, launchWalk).  The warp stages the key once in shared memory: the
// original block on the uni branch, the target 2 * org - pred on the bi branch (bi_target).  Every lane builds the member's 9 x numCand test vectors in its
// order (rounding, xClipMvToFppLine and clipMv included), the distinct ones are listed in shared memory, G-lane groups sum their distortion (group_dist with
// the key read from shared memory: xGetSAD / xGetHADs tile rules), and every lane then applies the member's update in loop order, so the strict `<` and the
// reuse of candidate 0's distortion for an equal candidate 1 (:2626-2637) hold exactly.  The sums are full: setDistParam resets the early-exit threshold
// (RdCost.cpp:172).  The target spans -(2^bd - 1) .. 2^(bd + 1) - 2; group_dist takes it in signed arithmetic (lo16 / hi16, IDP.2A), as bipred_int_kernel does.
#pragma once
#include "common.cuh"
#include "tz_kernels.cuh"
#include "bipred_kernels.cuh"

namespace vvb {

static_assert( sizeof( vvb_amvp ) == 24 && sizeof( vvb_amvr_best ) == 32 && sizeof( vvb_amvr_par ) == 40, "vvb_amvp / vvb_amvr_best / vvb_amvr_par layout" );

// what one call shares: the distortion family, the shift from internal units to the AMVR precision, m_auiMVPIdxCost[c][AMVP_MAX_NUM_CANDS], sqrt( lambda )
struct AmvrPar { int fam, shift; uint32_t mvpBits[2]; double motionLambda; };

// The member's CHECKs (:2579-2580, :2601-2602) and cBaseMvd rounded to the AMVR precision and back (roundTransPrecInternal2Amvr, :2604-2605); false where the
// member throws.  mvHor / mvVer: the integer vector (rcMv before changePrecision to internal units, :2128).
__host__ __device__ inline bool amvr_base( const vvb_amvp& a, int predHor, int predVer, int mvHor, int mvVer, int shift, int ( &base )[2][2] )
{
  if( a.num_cand < 1 || a.num_cand > 2 || a.mvp_idx < 0 || a.mvp_idx >= a.num_cand ) return false;
  if( ( a.mvp_idx ? a.cand_hor[1] : a.cand_hor[0] ) != 4 * predHor || ( a.mvp_idx ? a.cand_ver[1] : a.cand_ver[0] ) != 4 * predVer ) return false;
#ifdef __CUDA_ARCH__
#pragma unroll
#endif
  for( int c = 0; c < 2; c++ )
  {
    const int bh = mvHor * 16 - a.cand_hor[c], bv = mvVer * 16 - a.cand_ver[c];
    if( ( bh | bv ) & 3 ) return false;
    base[c][0] = tz_round_shift( bh, shift ) * ( 1 << shift );
    base[c][1] = tz_round_shift( bv, shift ) * ( 1 << shift );
  }
  return true;
}

// the vertical component of a test vector after CU::isMvInRangeFPP (UnitTools.cpp:3526-3535), xClipMvToFppLine (:2154-2163) and
// roundTransPrecInternal2AmvrVertical (Mv.h:227-234)
__device__ __forceinline__ int amvr_fpp( const TzPar& p, int y, int ver, int shift )
{
  const int yBMax = ( p.heightInCtus - 1 - p.ifpLines ) * ( 1 << p.ctuLog2 );
  const int yRefMax = ( ( ( y >> p.ctuLog2 ) + p.ifpLines + 1 ) << p.ctuLog2 ) - 1;
  const int yRefMv = y + p.h + 4 + ( ver >> 4 ) - 1;
  if( !p.ifpLines || y >= yBMax || yRefMv <= yRefMax ) return ver;
  return tz_round_shift( ver - ( yRefMv - yRefMax ) * 16, shift ) * ( 1 << shift );
}

// cTestMv[c] of position pos (:2614-2624): testPos (0,0) (-1,-1) (-1,0) (-1,1) (0,-1) (0,1) (1,-1) (1,0) (1,1) as (hor, ver).  Selections rather than indexed
// arrays, so that nothing goes to local memory.
__device__ __forceinline__ void amvr_point( const TzPar& p, const AmvrPar& ap, const vvb_amvp& a, const int ( &base )[2][2], int y, int pos, int c, int& th, int& tv )
{
  const int ph = pos == 0 ? 0 : pos <= 3 ? -1 : pos <= 5 ? 0 : 1;
  const int pv = pos == 0 ? 0 : pos <= 3 ? pos - 2 : pos == 4 ? -1 : pos == 5 ? 1 : pos - 7;
  th = ph * ( 1 << ap.shift ) + ( c ? base[1][0] + a.cand_hor[1] : base[0][0] + a.cand_hor[0] );
  tv = amvr_fpp( p, y, pv * ( 1 << ap.shift ) + ( c ? base[1][1] + a.cand_ver[1] : base[0][1] + a.cand_ver[0] ), ap.shift );
}

// the uni branch: vvb_tz_pu, the original block as the key, ruiBits from bits[], fWeight 1.0
struct AmvrOrgPlane
{
  using Pu = vvb_tz_pu;
  const uint32_t* bits;
  __device__ __forceinline__ int key( int o, int, int ) const { return o; }
  __device__ __forceinline__ bool refused( const vvb_tz_best& ) const { return false; }
  __device__ __forceinline__ uint32_t entryBits( const Pu&, int i ) const { return __ldg( bits + i ); }
  __device__ __forceinline__ double weight( const Pu& ) const { return 1.0; }
};

// the bi branch: vvb_bi_pu, the target formed from the original plane and pred[n][h][w], ruiBits from the PU, the BCW weight; a PU the integer stage refused
// arrives with BI_REFUSED_MV
struct AmvrTarget
{
  using Pu = vvb_bi_pu;
  const int16_t* pred;
  int wh;
  BiPar bp;
  __device__ __forceinline__ int key( int o, int i, int e ) const { return bi_target( o, __ldg( pred + (size_t) i * wh + e ), bp ); }
  __device__ __forceinline__ bool refused( const vvb_tz_best& im ) const { return im.mv_hor == BI_REFUSED_MV; }
  __device__ __forceinline__ uint32_t entryBits( const Pu& pu, int ) const { return pu.bits; }
  __device__ __forceinline__ double weight( const Pu& pu ) const { return bcw_me_weight( pu.bcw_idx, bp.refList ); }
};

// __launch_bounds__( 128, 1 ) as bipred_int_kernel: with the thread bound alone ptxas stops at 56-64 registers and spills for G = 4 and 8.
// p: the refinement's geometry (subShift 0); mp only feeds tz_warp_begin's MV-rate copy, which the refinement does not use (getCost is computed directly)
template<int G, class Src>
__global__ void __launch_bounds__( 128, 1 ) amvr_refine_kernel( const __grid_constant__ Plane orgPlane, const __grid_constant__ Plane refPlane,
                                                             const typename Src::Pu* __restrict__ pus, const vvb_tz_best* __restrict__ intMv,
                                                             const vvb_amvp* __restrict__ amvp, int n, const __grid_constant__ TzPar p,
                                                             const __grid_constant__ MePar mp, const __grid_constant__ AmvrPar ap, const __grid_constant__ Src src,
                                                             vvb_amvr_best* __restrict__ out )
{
  extern __shared__ __align__( 16 ) uint8_t amvrSmem[];
  __shared__ uint32_t sMv[VVB_MVCOST_ENTRIES];
  TzWarp W = tz_warp_begin( amvrSmem, sMv, p, mp, refPlane );
  const int lane = W.lane, warp = threadIdx.x >> 5, warpsPerGrid = gridDim.x * ( blockDim.x >> 5 ), wh = p.w * p.h;

  for( int i = blockIdx.x * ( blockDim.x >> 5 ) + warp; i < n; i += warpsPerGrid )     // persistent warps, as tz_search_kernel
  {
    const typename Src::Pu pu = pus[i];
    const vvb_tz_best im = intMv[i];
    const vvb_amvp a = amvp[i];
    int base[2][2];
    if( pu.x < 0 || pu.y < 0 || pu.x > p.picW - p.w || pu.y > p.picH - p.h || src.refused( im ) ||
        !amvr_base( a, pu.pred_hor, pu.pred_ver, im.mv_hor, im.mv_ver, ap.shift, base ) )
    {
      if( lane == 0 ) { vvb_amvr_best r{}; r.mvp_idx = -1; r.dist = r.cost = ~0ull; out[i] = r; }
      continue;
    }
    __syncwarp();                           // the previous PU's key and list are no longer read
    const int16_t* o = orgPlane.origin + (ptrdiff_t) pu.y * orgPlane.stride + pu.x;
    for( int e = lane; e < wh; e += 32 ) { const int y = e / p.w; W.org[e] = (int16_t) src.key( __ldg( o + (ptrdiff_t) y * orgPlane.stride + e - y * p.w ), i, e ); }
    W.ref = refPlane.origin + (ptrdiff_t) pu.y * refPlane.stride + pu.x;

    // the distinct test vectors, clipMv'd (:2629-2631), in loop order
    const TzClip cm = tz_clip_box( p, pu.x, pu.y, false );
    W.cnt = 0;
    for( int pos = 0; pos < 9; pos++ )
    {
      int h0 = 0, v0 = 0;
      for( int c = 0; c < a.num_cand; c++ )
      {
        int th, tv;
        amvr_point( p, ap, a, base, pu.y, pos, c, th, tv );
        if( c == 0 ) { h0 = th; v0 = tv; }
        else if( th == h0 && tv == v0 ) continue;
        if( lane == 0 ) W.pts[W.cnt] = make_int4( tz_clamp( th, cm.horMin, cm.horMax ) >> 4, tz_clamp( tv, cm.verMin, cm.verMax ) >> 4, 0, 0 );
        W.cnt++;
      }
    }
    __syncwarp();
    const int lg = lane & ( G - 1 ), grp = lane / G;
    for( int k = grp; k < W.cnt; k += 32 / G )
    {
      const int4 q = W.pts[k];
      const unsigned long long v = group_dist<G, true>( ap.fam, W.org, p.w, W.ref + (ptrdiff_t) q.y * W.refStride + q.x, W.refStride, p.w, p.h, 0, lg );
      if( lg == 0 ) W.sad[k] = (uint32_t) v;
    }
    __syncwarp();

    // the member's update in loop order, in every lane (:2633-2652)
    const double fWeight = src.weight( pu );
    unsigned long long bestDist = ~0ull, dist = 0;
    int bestH = im.mv_hor * 16, bestV = im.mv_ver * 16, bestIdx = a.mvp_idx, k = 0;
    uint32_t bestBits = 0;
    for( int pos = 0; pos < 9; pos++ )
    {
      int h0 = 0, v0 = 0;
      for( int c = 0; c < a.num_cand; c++ )
      {
        int th, tv;
        amvr_point( p, ap, a, base, pu.y, pos, c, th, tv );
        if( c == 0 ) { h0 = th; v0 = tv; }
        if( c == 0 || th != h0 || tv != v0 ) dist = x86_double_to_u64( __dmul_rn( (double) W.sad[k++], fWeight ) );
        const uint32_t bits = ( c ? ap.mvpBits[1] : ap.mvpBits[0] ) + eg_bits( tz_round_shift( th, ap.shift ) - tz_round_shift( c ? a.cand_hor[1] : a.cand_hor[0], ap.shift ) )
                                                                   + eg_bits( tz_round_shift( tv, ap.shift ) - tz_round_shift( c ? a.cand_ver[1] : a.cand_ver[0], ap.shift ) );
        const unsigned long long d = dist + motion_cost( ap.motionLambda, bits );
        if( d < bestDist ) { bestDist = d; bestH = th; bestV = tv; bestIdx = c; bestBits = bits; }
      }
    }
    if( lane == 0 )
    {
      vvb_amvr_best r;
      r.bits = src.entryBits( pu, i ) - ( a.mvp_idx ? ap.mvpBits[1] : ap.mvpBits[0] );
      r.dist = bestDist;
      if( bestDist == ~0ull ) { r.mv_hor = im.mv_hor * 16; r.mv_ver = im.mv_ver * 16; r.mvp_idx = a.mvp_idx; r.cost = ~0ull; }      // :2655-2659
      else
      {
        r.mv_hor = bestH; r.mv_ver = bestV; r.mvp_idx = bestIdx;
        r.bits += bestBits;
        r.cost = bestDist - motion_cost( ap.motionLambda, bestBits ) + motion_cost( ap.motionLambda, r.bits );
      }
      out[i] = r;
    }
  }
}

} // namespace vvb
