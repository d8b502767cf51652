/*
 * vvenc_b200.h -- C ABI of the B200-native block-cost path (drop-in boundary, SURVEY.md section 8b).
 *
 * Every entry point replaces one seam of the reference (fraunhoferhhi/vvenc); citations are
 * /root/reference-relative file:line.  Conventions: int return (0 = VVB_OK), no exceptions across the ABI,
 * plain pointers and sizes, no torch types.  A context owns one CUDA stream; calls on one context are
 * serialised on that stream, different contexts may be driven from different encoder worker threads
 * (the reference gives every worker its own RdCost/TrQuant, EncoderLib/EncSlice.cpp:142-147).
 * There is no CPU fallback: every call fails with VVB_ERR_CUDA if no sm_90 device is usable.
 *
 * Entry points without suffix take HOST buffers and copy in/out inside the call (the end-to-end path);
 * `_dev` twins take DEVICE pointers, enqueue on the context stream and return without synchronising.
 */
#ifndef VVENC_B200_H
#define VVENC_B200_H

#include <stdint.h>
#include <stddef.h>

#ifdef __cplusplus
extern "C" {
#endif

#define VVB_OK               0
#define VVB_ERR_ARG         -1   /* malformed argument (null pointer, negative size, unknown plane id)          */
#define VVB_ERR_UNSUPPORTED -2   /* shape outside the reference's own domain (e.g. width not a power of two)    */
#define VVB_ERR_CUDA        -3   /* CUDA runtime error, text in vvb_last_error()                                 */
#define VVB_ERR_NOMEM       -4

typedef struct vvb_ctx vvb_ctx;

/* Distortion function family == reference enum DFunc base (CommonLib/TypeDef.h:339-382); the per-width slot
 * (DF_SAD + log2 w etc.) is implied by the candidate's width exactly as RdCost::setDistParam does
 * (CommonLib/RdCost.cpp:158-226). */
enum vvb_dfunc
{
  VVB_DF_SSE      = 0,    /* xGetSSE*      CommonLib/RdCost.cpp:651-1000                        */
  VVB_DF_SAD      = 1,    /* xGetSAD*      CommonLib/RdCost.cpp:300-644 (subShift honoured)     */
  VVB_DF_HAD      = 2,    /* xGetHADs<0>   CommonLib/RdCost.cpp:1818-1938                       */
  VVB_DF_HAD_FAST = 3,    /* xGetHADs<1>   (16x16_fast tiles for square multiples of 32)       */
  VVB_DF_HAD_2SAD = 4     /* xGetHAD2SADs  CommonLib/RdCost.cpp:1768-1816                       */
};

/* ---- lifetime / errors -------------------------------------------------------------------------------- */
int         vvb_create     ( vvb_ctx** out, int device );   /* replaces RdCost::create(true) + initRdCostX86 (RdCost.cpp:82-148), TCoeffOps::initTCoeffOps (TrQuant_EMT.cpp:2028) */
void        vvb_destroy    ( vvb_ctx* ctx );
const char* vvb_last_error ( const vvb_ctx* ctx );
int         vvb_synchronize( vvb_ctx* ctx );
void*       vvb_stream     ( vvb_ctx* ctx );                /* cudaStream_t of the context, for event timing / interop */
int         vvb_launch_count( const vvb_ctx* ctx, uint64_t* kernels_launched );
/* Asynchronous mode (default off).  When on, the host-buffer entry points below (batch / search / pattern / trquant / roundtrip / plane upload)
 * only ENQUEUE their copies and kernels on the context's stream and return; vvb_synchronize() is the completion point.  Host input buffers
 * stay borrowed and host output buffers undefined until then; use page-locked host memory, otherwise the copies degrade to blocking ones.
 * Work of one context stays ordered; independent contexts (one per worker, EncSlice.cpp:142-147) overlap each other's copies and kernels.
 * The single-call helpers on borrowed host blocks (vvb_dist_block, vvb_sad_mask_block, vvb_sad_x5_block, vvb_fix_wsse_block, vvb_affine_sobel,
 * vvb_affine_equal_coeff) always block: their results are in place when they return, in either mode. */
int         vvb_set_async  ( vvb_ctx* ctx, int enable );   /* kernels this context has launched so far */

/* measurement aid (bench.py): issue-rate probe of the packed-SAD instruction mix; no reference counterpart */
int         vvb_alu_probe_dev( vvb_ctx* ctx, int grid_ctas, int iters, int mode /* 0: max-min SAD mix, 1: min-only mix of the dense search, 2: the SAD pyramid's tensor-core mix (min + relu + HMMA), 3: min + HMMA, 4: HMMA alone */ );

/* ---- pictures ("planes") ---------------------------------------------------------------------------------
 * int16 sample planes (Pel, CommonLib/TypeDef.h:181) with a margin on all sides, like the encoder's padded
 * reference pictures (CommonLib/Picture.cpp:461-501).  `origin` points at sample (0,0); rows -margin..height+margin-1
 * and columns -margin..width+margin-1 must be readable.  Uploaded once per picture, referenced by id afterwards.
 * Kernels do not clamp addresses: as in the encoder (Picture::extendPicBorder, MCTF_PADDING = 128) the margin has to cover the largest displacement
 * plus the filter reach -- search range for vvb_sad_search*, |vector| + 4 pels for vvb_frac_cost_grid, |vector|/16 + 4 pels for the MCTF calls. */
int vvb_plane_upload  ( vvb_ctx* ctx, int plane_id, const int16_t* origin, int stride, int width, int height, int margin, int bit_depth );
int vvb_plane_bind_dev( vvb_ctx* ctx, int plane_id, const int16_t* dev_origin, int stride, int width, int height, int margin, int bit_depth );
int vvb_plane_free    ( vvb_ctx* ctx, int plane_id );

/* ---- pair-list regime: one cost per descriptor (FpDistFunc, CommonLib/RdCost.h:74) ------------------------- */
typedef struct
{
  int32_t  org_plane, org_x, org_y;   /* DistParam::org (RdCost.h:85)                      */
  int32_t  cur_plane, cur_x, cur_y;   /* DistParam::cur                                    */
  uint16_t w, h;                      /* org.width / org.height                            */
  uint8_t  dfunc;                     /* enum vvb_dfunc                                    */
  uint8_t  sub_shift;                 /* DistParam::subShift (SAD only)                    */
  uint8_t  pad[2];
} vvb_cand;                           /* 32 bytes */

int vvb_dist_batch    ( vvb_ctx* ctx, const vvb_cand* cands, int n, uint64_t* cost_out );
int vvb_dist_batch_dev( vvb_ctx* ctx, const vvb_cand* dev_cands, int n, uint64_t* dev_cost_out );

/* Single synchronous call with borrowed HOST blocks: the exact shape of FpDistFunc for parity tests and for a
 * reference-side `RdCost::_initRdCostB200()` (see INTEGRATION.md).  Returns the cost; *err receives VVB_*. */
uint64_t vvb_dist_block( vvb_ctx* ctx, int dfunc, const int16_t* org, int org_stride, const int16_t* cur, int cur_stride,
                         int w, int h, int bit_depth, int sub_shift, int* err );

/* xGetSADwMask (RdCost.cpp:2062-2093), xGetSAD8X5/16X5 (RdCost.cpp:1984-2034), fixWeightedSSE (RdCost.cpp:1948-1982) */
uint64_t vvb_sad_mask_block( vvb_ctx* ctx, const int16_t* org, int org_stride, const int16_t* cur, int cur_stride, int w, int h,
                             const int16_t* mask, int mask_stride, int step_x, int mask_stride2, int sub_shift, int* err );
int      vvb_sad_x5_block  ( vvb_ctx* ctx, const int16_t* org, int org_stride, const int16_t* cur, int cur_stride, int w, int h,
                             int sub_shift, int calc_centre, uint64_t cost5[5] );
uint64_t vvb_fix_wsse_block( vvb_ctx* ctx, const int16_t* org, int org_stride, const int16_t* cur, int cur_stride, int w, int h,
                             uint32_t fixed_weight, int* err );

/* Descriptor-list forms of the three (SURVEY rows a7, a8, a9): the blocks sit in resident planes, one launch per list.
 * a7 GEO: the weight masks (g_globalGeoEncSADmask, Rom.cpp) are uploaded once with vvb_mask_upload; mask_offset is the sample the reference's mask pointer starts at
 *    (it may walk backwards from there with step_x = -1), mask_stride / mask_stride2 / step_x as DistParam carries them (RdCost.h:95-98).
 * a8 DMVR: cost5[i][k] = SAD( org + k, cur - k ) >> 1 for k = 0..4 (all five are written; the reference skips k = 2 unless asked for it).
 * a9: weights[i] = the fixed-point chroma weight of fixWeightedSSE. */
typedef struct { vvb_cand c; int32_t mask_offset, mask_stride, mask_stride2, step_x; } vvb_mask_cand;      /* 48 bytes; c.dfunc ignored */
int vvb_mask_upload       ( vvb_ctx* ctx, const int16_t* mask, int count );
int vvb_sad_mask_batch    ( vvb_ctx* ctx, const vvb_mask_cand* cands, int n, uint64_t* cost_out );
int vvb_sad_mask_batch_dev( vvb_ctx* ctx, const vvb_mask_cand* dev_cands, int n, uint64_t* dev_cost_out );
int vvb_sad_x5_batch      ( vvb_ctx* ctx, const vvb_cand* cands, int n, uint64_t* cost5_out /* [n][5] */ );
int vvb_sad_x5_batch_dev  ( vvb_ctx* ctx, const vvb_cand* dev_cands, int n, uint64_t* dev_cost5_out );
int vvb_fix_wsse_batch    ( vvb_ctx* ctx, const vvb_cand* cands, const uint32_t* weights, int n, uint64_t* cost_out );
int vvb_fix_wsse_batch_dev( vvb_ctx* ctx, const vvb_cand* dev_cands, const uint32_t* dev_weights, int n, uint64_t* dev_cost_out );

/* ---- candidate-pool regime (RDO style): K candidate predictions per original block, each with its own
 * compact w x h buffer: pool[(b*K + k)*w*h ...].  One cost per (block, candidate); HBM streaming.  Costs above 32 bits
 * (SSE of 128x64 blocks at 10 bits, of 32x32 at 12 bits) saturate at 0xffffffff; vvb_dist_batch returns them exactly. ---------- */
typedef struct { int32_t x, y; } vvb_pos;
int vvb_dist_pool    ( vvb_ctx* ctx, int dfunc, int org_plane, const vvb_pos* blocks, int n_blocks, int w, int h, int K,
                       const int16_t* pool, int sub_shift, uint32_t* cost_out /* n_blocks*K */ );
int vvb_dist_pool_dev( vvb_ctx* ctx, int dfunc, int org_plane, const vvb_pos* dev_blocks, int n_blocks, int w, int h, int K,
                       const int16_t* dev_pool, int sub_shift, uint32_t* dev_cost_out );
/* promise for the _dev variant: every block x in the device-resident lists is a multiple of 8 pels (enables 16-byte streaming loads) */
int vvb_pool_hint    ( vvb_ctx* ctx, int blocks_x_aligned_to_8 );

/* ---- motion-search regimes (EncoderLib/InterSearch.cpp) ----------------------------------------------------
 * MV rate: cost += Distortion( sqrt(lambda) * bits ), bits = EG((x<<cost_scale) - pred_hor >> imv_shift) + EG(y...)
 * (CommonLib/RdCost.h:181-203, RdCost.cpp:73-78). */
typedef struct
{
  int32_t x, y;                        /* block position in the original plane                    */
  int16_t left, right, top, bottom;    /* SearchRange (InterSearch.h:441-447), integer offsets    */
  int16_t pred_hor, pred_ver;          /* RdCost::setPredictor, units of 1/(1<<cost_scale) pel    */
  int16_t start_x, start_y;            /* pattern regime: centre of the fixed pattern              */
} vvb_block;                           /* 24 bytes */

typedef struct { int16_t dx, dy; uint32_t sad; uint64_t cost; } vvb_best;   /* 16 bytes; cost = sad + mv cost */

/* quad_order (dense search, _dev only): the block list is in quad-tree z-order (x,y),(x+w,y),(x,y+h),(x+w,y+h); quads whose members share
 * range and predictor are evaluated by one CTA on a shared window (verified per quad on the device, results identical either way) */
/* pattern_radius (pattern regime, _dev only; the host-buffer calls derive it): max |dx|,|dy| of the pattern, 0 = unknown */
typedef struct { double lambda; int32_t cost_scale, imv_shift, sub_shift, quad_order, pattern_radius, pad; } vvb_me_par;

/* Dense full search = InterSearch::xPatternSearch (InterSearch.cpp:2209-2251): every (dx,dy) in
 * [left..right]x[top..bottom], raster order, first strictly smaller total cost wins.  Optional SAD table
 * (uint32, row-major over the window, table_stride entries per block). */
int vvb_sad_search    ( vvb_ctx* ctx, int org_plane, int ref_plane, const vvb_block* blocks, int n, int w, int h, const vvb_me_par* par,
                        uint32_t* sad_tables, int table_stride, vvb_best* best_out );
/* max_nx / max_ny: largest (right-left+1) / (bottom-top+1) in the batch; the host sizes shared memory from them */
int vvb_sad_search_dev( vvb_ctx* ctx, int org_plane, int ref_plane, const vvb_block* dev_blocks, int n, int w, int h, const vvb_me_par* par,
                        int max_nx, int max_ny, uint32_t* dev_sad_tables, int table_stride, vvb_best* dev_best_out );

/* SAD pyramid over a quad-tree: level 0 holds blocks of base_w x base_w, level l blocks of (base_w << l); block p of level l+1 is the
 * parent of blocks 4p..4p+3 of level l (z-order: (x,y),(x+s,y),(x,y+s),(x+s,y+s)); a level may carry extra blocks after its 4*count[l+1]
 * children-of-parents.  Every block of every level gets the result InterSearch::xPatternSearch would give it over the SAME search range
 * (nx x ny positions, identical for all blocks; each block keeps its own MV predictor): pel work happens once, at level 0, and the SAD of a
 * larger block at a vector is the exact sum of its four children's SADs at that vector.  Parents whose children are not a proper quad or
 * whose range differs are reported with cost = ~0. */
int vvb_sad_search_pyramid_dev( vvb_ctx* ctx, int org_plane, int ref_plane, int levels, const vvb_block* const* dev_blocks /* [levels] */,
                                const int* counts /* [levels] */, int base_w, const vvb_me_par* par, int nx, int ny, vvb_best* const* dev_best_out /* [levels] */ );

int vvb_sad_search_pyramid    ( vvb_ctx* ctx, int org_plane, int ref_plane, int levels, const vvb_block* const* blocks /* [levels], host */,
                                const int* counts, int base_w, const vvb_me_par* par, int nx, int ny, vvb_best* const* best_out /* [levels], host */ );

/* Engine of vvb_sad_search_pyramid*: 1 (default) = one CTA per root block keeps every level on the SM (8x8 base blocks, no row sub-sampling, up to four
 * levels, planes of at most 10 bits, window within shared memory; other cases use engine 0 automatically), 0 = one CTA per quad + cost-table sums through
 * device memory.  Results are identical. */
int vvb_set_pyramid_engine( vvb_ctx* ctx, int engine );

/* Fixed candidate set = the static point pattern of xTZ8PointDiamondSearch / raster scan
 * (InterSearch.cpp:557-758, 2491-2497) around (start_x,start_y): pattern[k] = (dx,dy) offsets, clipped against the
 * block's SearchRange (points outside are reported as UINT32_MAX and never win).  costs are SAD only;
 * best_out applies the MV rate in list order (first strictly smaller wins). */
typedef struct { int16_t dx, dy; } vvb_mv;
int vvb_sad_pattern    ( vvb_ctx* ctx, int org_plane, int ref_plane, const vvb_block* blocks, int n, int w, int h, const vvb_mv* pattern, int K,
                         const vvb_me_par* par, uint32_t* sad_out /* n*K, nullable */, vvb_best* best_out /* nullable */ );
int vvb_sad_pattern_dev( vvb_ctx* ctx, int org_plane, int ref_plane, const vvb_block* dev_blocks, int n, int w, int h, const vvb_mv* dev_pattern, int K,
                         const vvb_me_par* par, uint32_t* dev_sad_out, vvb_best* dev_best_out );

/* Dense-search window staging: 1 = TMA (cp.async.bulk.tensor.2d; needs cuTensorMapEncodeTiled and a 16-byte aligned reference plane buffer) for every
 * window whose first column sits on a 16-byte boundary (8 pels), the load/store loop for the others; 0 = load/store loop only;
 * 2 (default) = TMA where it is measured faster (blocks up to 8 pels wide, i.e. the base level of the SAD pyramid).  Results are identical. */
int vvb_set_tma_staging( vvb_ctx* ctx, int enable );

/* Same candidate pattern with any distortion family (e.g. Hadamard integer refinement, InterSearch.cpp:2582,2630 and
 * xPatternRefinement :760-972, which add the MV rate the same way); cost_out holds the distortion only.  A distortion above 32 bits (SSE of large
 * blocks) is reported as 0xfffffffe in cost_out and best_out->sad; best_out->cost and the choice of the best point use the exact 64-bit value. */
int vvb_cost_pattern    ( vvb_ctx* ctx, int dfunc, int org_plane, int ref_plane, const vvb_block* blocks, int n, int w, int h, const vvb_mv* pattern, int K,
                          const vvb_me_par* par, uint32_t* cost_out /* n*K, nullable */, vvb_best* best_out /* nullable */ );
int vvb_cost_pattern_dev( vvb_ctx* ctx, int dfunc, int org_plane, int ref_plane, const vvb_block* dev_blocks, int n, int w, int h, const vvb_mv* dev_pattern, int K,
                          const vvb_me_par* par, uint32_t* dev_cost_out, vvb_best* dev_best_out );
/* device-side chaining: blocks[i].start = best[i].(dx,dy) (start of a refinement pattern / offset of the prediction block) */
int vvb_blocks_set_start_dev( vvb_ctx* ctx, vvb_block* dev_blocks, const vvb_best* dev_best, int n );

/* TZ integer motion search on the device = InterSearch::xTZSearch (EncoderLib/InterSearch.cpp:2297-2573) for every PU of a call, one PU shape per call
 * (w, h in 4..128, powers of two, no larger than tz->ctu_size).  The whole walk runs per PU: start vector and zero vector, the extra start candidates, the search range around the best
 * vector after them, integer early termination, the doubling diamond with its first-search stop, the zero-neighbourhood test, the adaptive or fixed raster,
 * star refinement with its stop rule -- with xTZSearchHelp's strict `<` and its uiBestRound / ucPointNr / uiBestDistance bookkeeping, so the results equal
 * the member's bit for bit.  The clipping that depends on the walk happens on the device: xClipMvSearch of the start vector and of every candidate
 * (:2329-2331, :2357-2358) and xSetSearchRange around the best vector (:2372-2377).  Costs are 64-bit; the MV rate is the table of `me` (lambda, cost_scale,
 * imv_shift); me->sub_shift is ignored, tz->sub_shift_mode selects the row sub-sampling per shape as RdCost::setDistParam does (RdCost.cpp:185-200).
 * Reads are not clamped: every position the walk can read lies in the box xClipMvSearch allows, i.e. columns -(ctu_size + 7) .. pic_w + w + 6 and rows
 * -(ctu_size + 7) .. pic_h + h + 6 around sample (0, 0), and a call whose ref_plane margin does not cover that box returns VVB_ERR_UNSUPPORTED.
 * Errors: null pointers, negative counts, settings out of range, and (host-buffer call) PUs outside the picture or candidate ranges outside cands: VVB_ERR_ARG;
 * shapes outside the domain (a PU larger than the CTU included), planes above 12 bits, an original plane smaller than the picture or a too small reference margin: VVB_ERR_UNSUPPORTED.
 * The _dev twin cannot check PU positions and candidate ranges on the host: such a PU gets cost = sad = ~0 and best_distance = 0xffffffff. */
typedef struct
{
  int32_t x, y;                    /* PU position in the original plane (inside the picture)                                                           */
  int32_t start_hor, start_ver;    /* rcMv as xTZSearch receives it: internal units (1/16 pel), not clipped                                            */
  int16_t pred_hor, pred_ver;      /* RdCost::setPredictor, quarter pel (as vvb_block.pred_*)                                                          */
  int32_t cand_first, cand_count;  /* extra start candidates cands[cand_first .. +cand_count): m_BlkUniMvInfoBuffer's uniMvs[refPicList][iRefIdxPred]
                                      in the buffer's order (:2352-2370), internal units, not clipped                                                   */
} vvb_tz_pu;                       /* 28 bytes */
typedef struct
{
  int32_t search_range;            /* m_iSearchRange                                                                                                   */
  int32_t extended, fast;          /* bExtendedSettings, bFastSettings                                                                                 */
  int32_t integer_et;              /* m_pcEncCfg->m_bIntegerET                                                                                         */
  int32_t first_search_stop;       /* m_pcEncCfg->m_bFastMEAssumingSmootherMVEnabled                                                                   */
  int32_t sub_shift_mode;          /* TZSearchStruct::subShiftMode: 0, 1 or 2                                                                          */
  int32_t pic_w, pic_h, ctu_size, ifp_lines;   /* pcv.lumaWidth, pcv.lumaHeight, pcv.maxCUSize (16..128), m_pcEncCfg->m_ifpLines                    */
} vvb_tz_par;
/* mv = rcMv as written out (integer pel); sad = ruiSAD (best cost minus its MV rate); cost = uiBestSad; best_distance = uiBestDistance at the end */
typedef struct { int32_t mv_hor, mv_ver; uint64_t sad, cost; uint32_t best_distance, pad; } vvb_tz_best;   /* 32 bytes */
int vvb_tz_search    ( vvb_ctx* ctx, int org_plane, int ref_plane, const vvb_tz_pu* pus, int n, int w, int h, const vvb_me_par* me, const vvb_tz_par* tz,
                       const int32_t* cands /* [n_cands][2] hor, ver; nullable when n_cands == 0 */, int n_cands, vvb_tz_best* out );
int vvb_tz_search_dev( vvb_ctx* ctx, int org_plane, int ref_plane, const vvb_tz_pu* dev_pus, int n, int w, int h, const vvb_me_par* me, const vvb_tz_par* tz,
                       const int32_t* dev_cands, int n_cands, vvb_tz_best* dev_out );

/* ---- forward transform + quantise (TrQuant::transformNxN; luma and chroma TUs with sides 4..64, transform skip included; ---------------
 * CommonLib/TrQuant.cpp:688-736 -> xT :481-564 -> Quant::quant CommonLib/Quant.cpp:735-833 -> QuantCore :132-230,
 * and Quant::xNeedRDOQ :835-891 -> needRdoqCore :264-278).  All TUs of a call share shape and transform types.
 * With lfnst_idx set (DCT-II only) the forward calls restate transformNxN's LFNST branch: transform zero-out to the top-left 4x4 / 8x8, the 16x16 / 16x48 int8
 * kernel, quantisation of coefficient group 0; `coef` returns the buffer xFwdLfnst leaves.  vvb_inv_trquant / vvb_tu_roundtrip restate invTransformNxN's LFNST branch
 * (TrQuant::xInvLfnst, TrQuant.cpp:838-940: the first 16 scan positions through the transposed kernel, then xIT over the top-left 8x8 / 4x4, :590-602); the levels
 * are expected as a bitstream carries them, zero beyond scan position 7 (4x4, 8x8) or 15.
 * deltaU (Quant.cpp:221), whose only consumer is the sign-bit hiding of the same call, stays on the device: with sign_hiding set the returned levels are the
 * ones Quant::quant leaves after xSignBitHidingHDQ (abs_sum stays QuantCore's sum, as uiAbsSum does; last_pos follows the hiding step).
 * Levels are clipped to -32768..32767; abs_sum is QuantCore's int32 sum of the unclipped magnitudes, so it may exceed the sum of the returned levels.
 * The results equal the reference for residuals within +-(2^bit_depth - 1) (org - pred of in-range pels) at any QP, where abs_sum stays below 2^24.  Beyond that
 * range (int16 residuals above the bit depth) the reference's own int32 transform sums can overflow (64 x 64 at 8 bits: 64 * 90 * 2^22 > 2^31 in the second
 * stage), so it has no defined result there.  The dequantiser of dependent quantisation (vvb_inv_trquant with dep_quant) forms qIdx = 2 * level -+ (state >> 1) in 32 bits
 * and the coefficient in 64 bits before the 16-bit clip, as DepQuant.cpp:616-618 does, so levels at the int16 extremes dequantise exactly. */
typedef struct
{
  int32_t w, h;                /* TU size, each in {4,8,16,32,64}                               */
  int32_t tr_hor, tr_ver;      /* 0 DCT-II, 1 DCT-VIII, 2 DST-VII (enum TransType)                */
  int32_t bit_depth;           /* 8..12 for vvb_fwd_trquant*, vvb_inv_trquant*, vvb_tu_roundtrip* and vvb_search_refine_tu; 8 or 10 for vvb_dep_quant and the
                                  vvb_rdoq* entries.  Anything else: VVB_ERR_UNSUPPORTED                                                                            */
  int32_t qp;                  /* CU QP (cu.qp); +6*(bit_depth-8) applied inside (Quant.cpp:99)   */
  int32_t is_irap;             /* slice->isIRAP(): rounding offset 171 vs 85 (Quant.cpp:772)      */
  int32_t dep_quant;           /* slice->depQuantEnabled: the QP of need_rdoq (Quant.cpp:852-855); vvb_inv_trquant then dequantises as DepQuant::dequant does
                                  (state machine + qIdx at QP + 1, DepQuant.cpp:574-629).  The forward calls and the round trip keep the plain quantiser pair */
  int32_t sign_hiding;         /* slice->signDataHidingEnabled: the levels pass through Quant::xSignBitHidingHDQ (Quant.cpp:817-826, 377-518) */
  int32_t lfnst_idx;           /* cu.lfnstIdx of an intra CU: 0 off, 1 / 2 = TrQuant::xFwdLfnst between the transform and the quantiser (TrQuant.cpp:942-1048) */
  int32_t lfnst_set;           /* g_lfnstLut[ xGetLFNSTIntraMode( intra mode ) ], 0..3 (Rom.cpp:95, TrQuant.cpp:806-828)                                     */
  int32_t lfnst_transpose;     /* xGetTransposeFlag of that mode (TrQuant.cpp:831-835)                                                                           */
  int32_t transform_skip;      /* tu.mtsIdx == MTS_SKIP (sides up to 32): xTransformSkip / xITransformSkip instead of the transforms (TrQuant.cpp:1050, 659), quantiser and
                                  dequantiser without the transform shift at max( QP, 4 + 6 * input_bit_depth_delta ) (Quant.cpp:117-124, 772, 561); tr_hor / tr_ver ignored */
  int32_t input_bit_depth_delta; /* sps.internalMinusInputBitDepth (transform skip only)                                                                               */
  int32_t is_chroma;           /* the TU belongs to a chroma component: `qp` is then the mapped chroma QP minus qpBdOffset (the mapping of QpParam, Quant.cpp:96-101, is
                                  host work) and Quant::xNeedRDOQ rounds with 256 instead of 171 (Quant.cpp:877).  Everything else is the luma arithmetic              */
} vvb_tu_par;

/* resi: n compact residual blocks [n][h][w] (Pel); outputs (each nullable except q):
 * coef [n][h][w] TCoeff (int32), q [n][h][w] TCoeffSig (int16), abs_sum[n], last_pos[n], need_rdoq[n] (0/1) */
int vvb_fwd_trquant    ( vvb_ctx* ctx, const vvb_tu_par* par, const int16_t* resi, int n,
                         int32_t* coef, int16_t* q, int32_t* abs_sum, int32_t* last_pos, uint8_t* need_rdoq );
int vvb_fwd_trquant_dev( vvb_ctx* ctx, const vvb_tu_par* par, const int16_t* dev_resi, int n,
                         int32_t* dev_coef, int16_t* dev_q, int32_t* dev_abs_sum, int32_t* dev_last_pos, uint8_t* dev_need_rdoq );
/* Transform engine of vvb_fwd_trquant*, vvb_inv_trquant* and vvb_tu_roundtrip*: 0 = CUDA-core IDP.2A kernels for every shape; any other value (default) = the
 * raw-byte wgmma engines (the MMAs read the bytes of the int16 residual / int32 stage-1 values as u8 / s8 against zero-interleaved matrices, quantiser in
 * registers) where they apply: square 8..64 TUs without LFNST or transform skip (forward: also without sign-bit hiding); CUDA cores elsewhere.
 * The raw-byte engines move TU data in 16-byte units, so a _dev call takes them only when every TU buffer it is given (residual, original and prediction
 * pools, levels, coefficients, residual and reconstruction outputs; null ones aside) is 16-byte aligned.  Buffers that are only 8-byte aligned run on the
 * CUDA-core kernels, which need no more than that.  Both settings are bit-exact. */
int vvb_set_tensor_transform( vvb_ctx* ctx, int enable );
/* Residual formed on the device: resi = org(x,y) - pred(x+start_x, y+start_y) for each TU position (PelBuf::subtract, IntraSearch.cpp:1328) */
int vvb_fwd_trquant_planes    ( vvb_ctx* ctx, const vvb_tu_par* par, int org_plane, int pred_plane, const vvb_block* blocks, int n,
                         int32_t* coef, int16_t* q, int32_t* abs_sum, int32_t* last_pos, uint8_t* need_rdoq );
int vvb_fwd_trquant_planes_dev( vvb_ctx* ctx, const vvb_tu_par* par, int org_plane, int pred_plane, const vvb_block* dev_blocks, int n,
                         int32_t* dev_coef, int16_t* dev_q, int32_t* dev_abs_sum, int32_t* dev_last_pos, uint8_t* dev_need_rdoq );

/* ---- one call for the whole per-picture chain (host buffers; the production shape of "batch the per-CTU candidate evaluations into CUDA launches") -------------
 * For a quad-tree of block lists (as vvb_sad_search_pyramid: level 0 = base_w, block p of level l+1 is the parent of blocks 4p..4p+3 of level l):
 *   1. dense search of every block (vvb_sad_search_pyramid)                                   -> best[l]
 *   2. blocks[l][i].start = best vector (on the device), distortion `refine_dfunc` over the fixed pattern around it (vvb_cost_pattern) -> refine_cost[l][i][K]
 *   3. residual org - pred(best vector), forward transform + quantiser (vvb_fwd_trquant_planes) -> q[l], abs_sum[l], last_pos[l], need_rdoq[l]
 * Nothing returns to the host between the stages; in asynchronous mode the call only enqueues (one upload, the launches, the downloads).  Results are those of
 * the three calls made one after the other with the host patching start_x / start_y in between.  Nullable outputs: refine_cost, q (with abs_sum...), need_rdoq. */
typedef struct
{
  const vvb_block* blocks; int32_t count;        /* in: block list of the level (start_x / start_y ignored)                        */
  vvb_best*  best;                               /* out [count]                                                                    */
  uint32_t*  refine_cost;                        /* out [count][K], nullable                                                       */
  int16_t*   q;                                  /* out [count][h][w] levels, nullable (then no transform stage for this level)    */
  int32_t*   abs_sum; int32_t* last_pos; uint8_t* need_rdoq;   /* out [count], each nullable                                       */
  vvb_tu_par tu;                                 /* TU parameters of the level (w = h = base_w << l)                               */
  int16_t*   packed_q;                           /* out, nullable: the levels of TU i at scan positions 0 .. last_pos[i], in scan order, TU after TU (capacity count * h * w);
                                                    with it packed_offsets [count + 1] (entry i = first level of TU i, entry count = total) and last_pos are required.  When the
                                                    buffer is page-locked (device-visible under UVA) the device writes it directly and only the used part crosses PCIe */
  uint32_t*  packed_offsets;
} vvb_level_io;
int vvb_search_refine_tu( vvb_ctx* ctx, int org_plane, int ref_plane, int levels, const vvb_level_io* io, int base_w, const vvb_me_par* me, int nx, int ny,
                          int refine_dfunc, const vvb_mv* pattern, int K );
/* the trimming on its own: out_packed (device-visible) receives the levels up to last_pos of every TU in scan order, dev_offsets [n + 1] their positions;
 * vvb_scan_order gives scan position -> raster index (row pitch w) for unpacking (grouped 4x4 diagonal scan, Rom.cpp:1098-1136; min(w,32) * min(h,32) entries) */
int vvb_pack_levels_dev( vvb_ctx* ctx, const vvb_tu_par* par, const int16_t* dev_q, const int32_t* dev_last_pos, int n, int16_t* out_packed, uint32_t* dev_offsets );
int vvb_scan_order( int w, int h, int32_t* out );

/* ---- dependent quantisation (SURVEY 8f-4): DepQuant::quant -> xQuantDQ (CommonLib/DepQuant.cpp:1462-1490, 1129-1264), luma and chroma TUs (par->is_chroma
 * selects the chroma context offsets of the scan tables; qp and the rate tables are then the chroma ones), without scaling lists --------
 * The 4-state trellis over the scan positions of each TU (xDecide / xDecideAndUpdate :1266-1414, the rate-distortion checks :697-888, the state updates
 * :907-1110, CommonCtx::update :473-531) runs on the device, one TU per thread, all TUs of the call sharing shape, QP, lambda and the rate tables.
 * What the caller supplies is what depends on the encoder's entropy-coding state at that point of the CTU:
 *   vvb_dq_rates -- the tables RateEstimator::initCtx (:344-471) derives from the CABAC contexts (public accessors of DQIntern::RateEstimator, DepQuant.h:161-170):
 *                   last_bits_x/y[pos] (xSetLastCoeffOffset; lastOffset( scan ) = x + y part), sig_sbb_bits[ctx][bin] (sigSbbFracBits), sig_bits[set][ctx][bin]
 *                   (m_sigFracBits; state k reads set max( k - 1, 0 )), gtx_bits[ctx][0..5] (gtxFracBits).
 *   vvb_dq_par   -- lambda (Quant::m_dLambda), dq_thr_val (Quant::init thrVal, 8), zero_out = the condition of :1155 evaluated by the caller
 *                   ( mtsIdx > MTS_SKIP || ( sps.MTS && cu.sbtInfo && w <= 32 && h <= 32 ) ): coefficients beyond 16 of a 32-sided TU are skipped.
 *                   scalar_members: the reference's scalar and x86 state updates differ for levels above 127 (update1State adds uint8_t( level ) to the template sum,
 *                   DepQuant.cpp:956-966; DepQuantX86.h:86-93, 163-166 adds the level capped to 126 / 127).  0 (default) follows the x86 members the encoder
 *                   installs on this platform, 1 the scalar ones of --SIMD=SCALAR.  Below 128 they agree.
 * The quantiser constants of Quantizer::initQuantBlock (:533-572) are derived inside from (w, h, bit_depth, qp, lambda) in the same double-precision steps.
 * Any par->qp is accepted: the internal QP qp + 6 * (bit_depth - 8) is clipped to 0..63 + 6 * (bit_depth - 8) as QpParam does (Quant.cpp:109) and as the other
 * entries and the dequantiser of dep_quant do, so the trellis runs at that clipped QP + 1.  Lambdas for which the reference's (uint32_t)( nomDistFactor * qScale2 )
 * (DepQuant.cpp:566, = 2^nomDShift / lambda) reaches 2^32 have no defined result there, and none here.
 * par->lfnst_idx > 0 restricts the first tested position to 7 / 15 (:1164-1167).  need_rdoq (nullable, [n]): TUs with need_rdoq[i] == 0 return all-zero levels and
 * last_pos -1 (picture->useSelectiveRdoq, :1464-1468).  coef: [n][h][w] TCoeff as vvb_fwd_trquant returns them; q: [n][h][w] levels; abs_sum, last_pos nullable. */
typedef struct { int32_t last_bits_x[32], last_bits_y[32], sig_sbb_bits[2][2], sig_bits[3][12][2], gtx_bits[21][6]; } vvb_dq_rates;   /* 1064 bytes */
typedef struct { double lambda; int32_t dq_thr_val, zero_out, scalar_members, pad; } vvb_dq_par;
int vvb_dep_quant    ( vvb_ctx* ctx, const vvb_tu_par* par, const vvb_dq_par* dq, const vvb_dq_rates* rates, const int32_t* coef, const uint8_t* need_rdoq, int n,
                       int16_t* q, int32_t* abs_sum, int32_t* last_pos );
int vvb_dep_quant_dev( vvb_ctx* ctx, const vvb_tu_par* par, const vvb_dq_par* dq, const vvb_dq_rates* rates, const int32_t* dev_coef, const uint8_t* dev_need_rdoq, int n,
                       int16_t* dev_q, int32_t* dev_abs_sum, int32_t* dev_last_pos );
/* kernel shape of the trellis: 1 (default) = four lanes per TU, one per trellis state, eight TUs per warp in lock step; 0 = one thread per TU.  Same results. */
int vvb_set_depquant_engine( vvb_ctx* ctx, int engine );
/* the constants the call derives (no device needed): out = qShift, maxQIdx, thresLast, distShift, qAdd, qScale, distAdd, distStepAdd, distOrgFact (Quantizer, DepQuant.h:220-231) */
int vvb_dep_quant_constants( const vvb_tu_par* par, const vvb_dq_par* dq, int64_t out[9] );

/* ---- fast rate-distortion optimised quantisation (SURVEY 8f-4): QuantRDOQ2::quant -> xRateDistOptQuant -> xRateDistOptQuantFast<bSBH, false>
 * (CommonLib/QuantRDOQ2.cpp:247-301, 1283-1296, 475-1281), what Quant::m_RDOQ == 2 (presets faster and fast, vvencCfg.cpp:2675, 2737) runs for every TU that is not
 * transform skipped and what DepQuant::quant falls back to in slices without dependent quantisation (DepQuant.cpp:1486-1489).  Luma and chroma components, sides 4..64,
 * with and without sign-bit hiding (par->sign_hiding = slice->signDataHidingEnabled), no scaling lists; transform-skipped TUs: vvb_rdoq_ts below; BDPCM stays on the host.
 * Per coefficient group, from the last scan position down: level decision between floor and ceil of |c| * scale >> qBits by distortion + lambda * bits (:697-969, bits
 * from the context the template of already-decided neighbours selects, ContextModelling.h:158-269), group zero-out (:971-1036), last-position optimisation (:1038-1095),
 * parity adjustment for sign-bit hiding (:1097-1167), coded-block-flag decision (:1185-1233), signs (:1251-1257).  One TU per thread, all TUs of a call sharing shape,
 * QP, lambda and the rate tables.  The caller supplies what depends on the encoder's entropy-coding state at that point of the CTU:
 *   vvb_rdoq_rates -- BinFracBits::intBits of the contexts the routine reads (FracBitsAccess::getFracBitsArray): sig_bits[ctxOfs] = Ctx::SigFlag[chType]( ctxOfs ),
 *                     par_bits[o] = Ctx::ParFlag[chType]( o ), gt1_bits[o] = Ctx::GtxFlag[chType + 2]( o ), gt2_bits[o] = Ctx::GtxFlag[chType]( o ),
 *                     sig_group_bits[i] = Ctx::SigCoeffGroup[chType]( i ); last_bits_x / last_bits_y = m_lastBitsX / m_lastBitsY[chType] as xInitLastPosBitsTab (:408-434)
 *                     leaves them (for Cr after a coded Cb the table of the Cb call, :490); cbf_bits = the context of :1185-1226 (QtRootCbf for the luma component of an
 *                     inter CU, QtCbf[compID]( CtxQtCbf(...) ) otherwise; zeros when the flag is inferred -- the last ISP partition after uncoded ones).
 *   vvb_rdoq_par   -- lambda (Quant::m_dLambda), thr_val (Quant::init thrVal, 8), sbt_zero_out = the condition of TransformUnit::getTbAreaAfterCoefZeroOut
 *                     (Unit.cpp:580: sps.MTS && cu.sbtInfo && w <= 32 && h <= 32 && luma) for the budget of context-coded bins.
 * Uses par->{w, h, bit_depth, qp, is_chroma, sign_hiding, lfnst_idx}: lfnst_idx > 0 (the CU's index, whatever the component: :552-559) limits the scan to group 0 and,
 * for 4x4 / 8x8, to position 7.  The error scale of xSetErrScaleCoeffNoScalingList (:203-219) is derived inside in the same double-precision steps.
 * need_rdoq (nullable, [n]): TUs with need_rdoq[i] == 0 return all-zero levels (picture->useSelectiveRdoq, :273, 291-295).  coef: [n][h][w] TCoeff as vvb_fwd_trquant
 * returns them; q: [n][h][w] levels; abs_sum / last_pos (nullable) as uiAbsSum / tu.lastPos are left (last_pos -1 where the routine does not write it: nothing coded).
 * Levels above 32767 (reachable at the lowest QPs: up to 104858 in a 64-sided TU at internal QP 0) are stored into q as the member stores them into TCoeffSig
 * (:942), i.e. as their low 16 bits, and the context templates read them as the member does.  One known difference remains, in engine 1 only, for levels from
 * 65533 up (lowest QP of 64-sided TUs): the member adds a neighbour's template term from the full level and removes it (group zero-out, last-position choice,
 * sign hiding) from abs() of the stored TCoeffSig, so a level whose low 16 bits are 0..3 or 65533..65535 leaves a term engine 1, which reads the stored levels
 * only, cannot reconstruct.  Engine 2 keeps the member's add / remove bookkeeping and agrees there too. */
typedef struct { int32_t sig_bits[12][2], par_bits[21][2], gt1_bits[21][2], gt2_bits[21][2], sig_group_bits[2][2], last_bits_x[16], last_bits_y[16], cbf_bits[2], pad[2]; } vvb_rdoq_rates;   /* 760 bytes */
typedef struct { double lambda; int32_t thr_val, sbt_zero_out, pad[2]; } vvb_rdoq_par;
int vvb_rdoq    ( vvb_ctx* ctx, const vvb_tu_par* par, const vvb_rdoq_par* rq, const vvb_rdoq_rates* rates, const int32_t* coef, const uint8_t* need_rdoq, int n,
                  int16_t* q, int32_t* abs_sum, int32_t* last_pos );
int vvb_rdoq_dev( vvb_ctx* ctx, const vvb_tu_par* par, const vvb_rdoq_par* rq, const vvb_rdoq_rates* rates, const int32_t* dev_coef, const uint8_t* dev_need_rdoq, int n,
                  int16_t* dev_q, int32_t* dev_abs_sum, int32_t* dev_last_pos );
/* kernel of vvb_rdoq: 1 (default) = the template of a position is gathered from its five neighbours when the position is visited; 2 = the templates are accumulated in the level slots of the
 * positions not visited yet (what the reference's m_tplBuf bookkeeping does) and lambda * bits of the frequent cases comes from per-call tables.  Same results, but for
 * the levels from 65533 up described above. */
int vvb_set_rdoq_engine( vvb_ctx* ctx, int engine );
/* the constants the call derives (no device needed): out = quantScale, errScale, qBits, useThres, remRegBins, numCG, firstScanPos (QuantRDOQ2.cpp:518-559, 573-583) */
int vvb_rdoq_constants( const vvb_tu_par* par, const vvb_rdoq_par* rq, int32_t out[7] );

/* Transform-skipped TUs: QuantRDOQ::rateDistOptQuantTS (CommonLib/QuantRDOQ.cpp:1124-1336; xGetCodedLevelTSPred :1578-1661, xGetICRateTS :1663-1807), what QuantRDOQ2::quant
 * runs for a TU with mtsIdx == MTS_SKIP and no BDPCM when Quant::m_useRDOQTS is set (QuantRDOQ2.cpp:263, 275-285).  Forward scan, contexts from the left and upper neighbour,
 * up to three candidate levels per coefficient priced in double precision (distortion = err * err * errorScale, rate = lambda * bits, summed in the member's order), group
 * zero-out, the budget of context-coded bins ( w * h * 7 ) >> 2.  Sides 4..32 (transform skip exists up to 32 x 32); coef = the residual as TrQuant::xTransformSkip copies it
 * (vvb_fwd_trquant with par->transform_skip returns it); uses par->{w, h, bit_depth, qp, input_bit_depth_delta}; forwardRDPCM (BDPCM) stays on the host.
 *   vvb_rdoq_ts_rates -- BinFracBits::intBits of the transform-skip context sets: sig_bits[numPos] = Ctx::TsSigFlag, par_bits = Ctx::TsParFlag( 0 ), gtx_bits[i] = Ctx::TsGtxFlag( i ),
 *                        lrg1_bits[numPos] = Ctx::TsLrg1Flag, sign_bits[ctx] = Ctx::TsResidualSign, sig_group_bits[sigLeft + sigAbove] = Ctx::TsSigCoeffGroup.
 * q: [n][h][w] signed levels; abs_sum (nullable) as the member leaves uiAbsSum (tu.lastPos is not touched by the member).  need_rdoq as for vvb_rdoq. */
typedef struct { int32_t sig_bits[3][2], par_bits[2], gtx_bits[5][2], lrg1_bits[4][2], sign_bits[6][2], sig_group_bits[3][2]; } vvb_rdoq_ts_rates;   /* 176 bytes */
int vvb_rdoq_ts    ( vvb_ctx* ctx, const vvb_tu_par* par, double lambda, const vvb_rdoq_ts_rates* rates, const int32_t* coef, const uint8_t* need_rdoq, int n, int16_t* q, int32_t* abs_sum );
int vvb_rdoq_ts_dev( vvb_ctx* ctx, const vvb_tu_par* par, double lambda, const vvb_rdoq_ts_rates* rates, const int32_t* dev_coef, const uint8_t* dev_need_rdoq, int n, int16_t* dev_q,
                     int32_t* dev_abs_sum );

/* BDPCM TUs: QuantRDOQ::forwardRDPCM (CommonLib/QuantRDOQ.cpp:1338-1562), what QuantRDOQ2::quant runs for a transform-skipped TU whose CU carries a block-DPCM direction
 * (dir_mode = cu.bdpcmM[chType]: 1 horizontal, 2 vertical).  As vvb_rdoq_ts, but each position quantises the residual minus the reconstructed left / upper neighbour
 * (xDequantSample :1564-1576 of the level just chosen plus its own prediction), with the BDPCM variants of the greater-1 and sign contexts and two candidate levels.
 * The inverse needs no entry point of its own: Quant::dequant undoes the DPCM on the levels (invResDPCM, Quant.cpp:298-340: clipped prefix sums along the direction)
 * before the ordinary dequantiser of skipped transforms -- the binding forms the sums and calls vvb_inv_trquant with par->transform_skip. */
int vvb_rdoq_bdpcm    ( vvb_ctx* ctx, const vvb_tu_par* par, double lambda, int dir_mode, const vvb_rdoq_ts_rates* rates, const int32_t* coef, const uint8_t* need_rdoq, int n, int16_t* q,
                        int32_t* abs_sum );
int vvb_rdoq_bdpcm_dev( vvb_ctx* ctx, const vvb_tu_par* par, double lambda, int dir_mode, const vvb_rdoq_ts_rates* rates, const int32_t* dev_coef, const uint8_t* dev_need_rdoq, int n,
                        int16_t* dev_q, int32_t* dev_abs_sum );

/* ---- inverse path of the TU loop (SURVEY 8f-1) -------------------------------------------------------------------
 * vvb_inv_trquant: TrQuant::invTransformNxN (TrQuant.cpp:318-348) = Quant::dequant (Quant.cpp:520-609, DeQuantCore :232) + TrQuant::xIT
 * (:567-660).  q: n compact level blocks [n][h][w] (TCoeffSig); resi: [n][h][w] Pel.  Uses par->{w,h,tr_hor,tr_ver,bit_depth,qp,transform_skip,...}; with par->dep_quant
 * (and no transform skip) the dequantiser is DepQuant::dequant's. */
int vvb_inv_trquant    ( vvb_ctx* ctx, const vvb_tu_par* par, const int16_t* q, int n, int16_t* resi );
int vvb_inv_trquant_dev( vvb_ctx* ctx, const vvb_tu_par* par, const int16_t* dev_q, int n, int16_t* dev_resi );

/* One luma TU candidate end to end in one kernel -- the loop body of IntraSearch::xIntraCodingTUBlock (IntraSearch.cpp:1328-1429) and of
 * InterSearch::xEstimateInterResidualQT (InterSearch.cpp:3659-3714):  residual = org - pred (PelBuf::subtract), TrQuant::transformNxN,
 * abs_sum > 0 ? TrQuant::invTransformNxN : zero residual, PelBuf::reconstruct (Buffer.cpp:719, clip to [0, 2^bitDepth - 1]), then
 *   dist_reco = SSE(org, reco)                 (intra: IntraSearch.cpp:1429)
 *   dist_resi = SSE(org - pred, rec. residual) (inter: InterSearch.cpp:3714)
 *   dist_zero = SSE(0, org - pred)             (inter zero-residual alternative: InterSearch.cpp:3670)
 * org / pred: n compact blocks [n][h][w]; q (levels) required, reco and need_rdoq nullable. */
typedef struct { uint64_t dist_reco, dist_resi, dist_zero; int32_t abs_sum, last_pos; } vvb_tu_result;   /* 32 bytes */
int vvb_tu_roundtrip    ( vvb_ctx* ctx, const vvb_tu_par* par, const int16_t* org, const int16_t* pred, int n,
                          int16_t* q, int16_t* reco, vvb_tu_result* res, uint8_t* need_rdoq );
int vvb_tu_roundtrip_dev( vvb_ctx* ctx, const vvb_tu_par* par, const int16_t* dev_org, const int16_t* dev_pred, int n,
                          int16_t* dev_q, int16_t* dev_reco, vvb_tu_result* dev_res, uint8_t* dev_need_rdoq );
/* same with org / pred taken from resident planes: TU i sits at (blocks[i].x, blocks[i].y), its prediction at (+start_x, +start_y) in pred_plane */
int vvb_tu_roundtrip_planes_dev( vvb_ctx* ctx, const vvb_tu_par* par, int org_plane, int pred_plane, const vvb_block* dev_blocks, int n,
                          int16_t* dev_q, int16_t* dev_reco, vvb_tu_result* dev_res, uint8_t* dev_need_rdoq );

/* The same TU candidate with the quantiser the slice runs for it, in one call: what DepQuant::quant / QuantRDOQ2::quant (DepQuant.cpp:1462-1490,
 * QuantRDOQ2.cpp:247-301) do inside TrQuant::transformNxN, then the round trip above.  Per TU:
 *   1. residual = org - pred; the forward transform (with LFNST when par->lfnst_idx is set) and need_rdoq (Quant::xNeedRDOQ) exactly as vvb_fwd_trquant;
 *   2. the levels: zero (abs_sum 0, last_pos -1) where `selective` (picture->useSelectiveRdoq) is set and need_rdoq is 0, otherwise those of vvb_rdoq (quantiser 1,
 *      QuantRDOQ2::xRateDistOptQuantFast, m_RDOQ == 2: presets faster and fast) or of vvb_dep_quant (quantiser 2, DepQuant::xQuantDQ: presets medium to slower) with
 *      the same parameters and rates, on the context's current RDOQ / DepQuant engine;
 *   3. abs_sum > 0: the dequantiser that belongs to the quantiser (Quant::dequant after fast RDOQ, DepQuant::dequant at QP + 1 after the trellis) and the inverse
 *      transform as vvb_inv_trquant; otherwise the residual is zero;
 *   4. reco = clip( pred + residual ) and dist_reco / dist_resi / dist_zero as vvb_tu_result defines them.  abs_sum and last_pos are the quantiser's.
 * need_rdoq (nullable) is returned whether or not `selective` is set.  The chroma distortion weight of getDistPart stays with the caller.  Luma and chroma
 * (par->is_chroma) TUs with sides 4..64 and every MTS pair the forward transform takes; bit depth 8 or 10.
 * Errors: quantiser other than 1 or 2, par->dep_quant set for quantiser 1 or clear for quantiser 2 (the dequantiser would not match), sign_hiding with quantiser 2
 * (a slice cannot signal both), null quantiser parameters or rates: VVB_ERR_ARG; the parameter errors of vvb_rdoq / vvb_dep_quant as those calls give them;
 * transform_skip (skipped and BDPCM TUs go through vvb_rdoq_ts / vvb_rdoq_bdpcm) and bit depths other than 8 or 10: VVB_ERR_UNSUPPORTED.
 * Engines: the forward and the inverse each follow the rule of vvb_set_tensor_transform over org, pred, q and reco (the quantiser's sign-bit hiding does not keep
 * the forward off the tensor engine); the intermediates live in the context's work arena. */
typedef struct
{
  int32_t quantiser;                                          /* 1 = fast RDOQ (as vvb_rdoq), 2 = dependent quantisation (as vvb_dep_quant)  */
  int32_t selective;                                          /* picture->useSelectiveRdoq: TUs whose need_rdoq is 0 get no levels           */
  const vvb_rdoq_par* rq; const vvb_rdoq_rates* rq_rates;     /* quantiser 1                                                                 */
  const vvb_dq_par*   dq; const vvb_dq_rates*   dq_rates;     /* quantiser 2                                                                 */
} vvb_tu_quant;
int vvb_tu_roundtrip_rdo    ( vvb_ctx* ctx, const vvb_tu_par* par, const vvb_tu_quant* quant, const int16_t* org, const int16_t* pred, int n,
                              int16_t* q, int16_t* reco, vvb_tu_result* res, uint8_t* need_rdoq );
int vvb_tu_roundtrip_rdo_dev( vvb_ctx* ctx, const vvb_tu_par* par, const vvb_tu_quant* quant, const int16_t* dev_org, const int16_t* dev_pred, int n,
                              int16_t* dev_q, int16_t* dev_reco, vvb_tu_result* dev_res, uint8_t* dev_need_rdoq );
int vvb_tu_roundtrip_rdo_planes_dev( vvb_ctx* ctx, const vvb_tu_par* par, const vvb_tu_quant* quant, int org_plane, int pred_plane, const vvb_block* dev_blocks, int n,
                              int16_t* dev_q, int16_t* dev_reco, vvb_tu_result* dev_res, uint8_t* dev_need_rdoq );

/* ---- MCTF block matching (CommonLib/MCTF.cpp:122-257 via MCTF::motionErrorLuma :1099-1164) -----------------
 * Every MCTF entry (error batch, search grid, calc_var, estimate_level, estimate_pyramid, apply) takes planes of up to 10 bits and returns
 * VVB_ERR_UNSUPPORTED when the original or the reference is wider (MCTF.cpp:1313 CHECKD).  Errors are exact SSEs while they fit int32 and saturate to
 * 0x7fffffff above it (a 64x64 block at 10 bits reaches 4096 * 1023^2): the reference stops summing as soon as its sum passes the best error, so a
 * saturated candidate never beats a finite best under the strict `error < best.error` chains, which is the reference's decision. */
typedef struct { int32_t x, y; int32_t mvx, mvy; /* 1/16 pel */ uint16_t w, h; } vvb_mctf_cand;   /* 20 bytes */
int vvb_mctf_error_batch    ( vvb_ctx* ctx, int org_plane, int ref_plane, const vvb_mctf_cand* cands, int n, int low_res_filter /* 4-tap */, int32_t* err_out );
int vvb_mctf_error_batch_dev( vvb_ctx* ctx, int org_plane, int ref_plane, const vvb_mctf_cand* dev_cands, int n, int low_res_filter, int32_t* dev_err_out );
/* promise for the _dev variant: no candidate in the device-resident lists is wider or taller than max_block_dim (8..64, default 64; sizes the per-warp
 * shared-memory window -- MCTF uses 8/16/32, vvencCfg.cpp:1495).  A candidate that breaks the promise gets error -1. */
int vvb_mctf_hint( vvb_ctx* ctx, int max_block_dim );

/* Grid search of MCTF::estimateLumaLn (MCTF.cpp:1218-1287): for every block (x, y, w, h) all (2*radius+1)^2 vectors  (mvx, mvy) + (i - radius, j - radius) * step,
 * step in 1/16 pel (16 = the integer grid with range 5/8, then 4, 2, 1 for the doubleRes refinements).  err_out[n][j][i] = motionErrorLuma of that vector
 * (no early exit).  One CTA per block: the window is staged once and the horizontally filtered rows are shared by the candidates of a column.
 * The `error < best.error` chain, the predictor candidates and the final error scaling (:1308-1321) replay on the host from these tables. */
int vvb_mctf_search_grid    ( vvb_ctx* ctx, int org_plane, int ref_plane, const vvb_mctf_cand* blocks, int n, int step, int radius, int low_res_filter, int32_t* err_out );
int vvb_mctf_search_grid_dev( vvb_ctx* ctx, int org_plane, int ref_plane, const vvb_mctf_cand* dev_blocks, int n, int step, int radius, int low_res_filter, int32_t* dev_err_out );

/* ---- fractional-pel refinement feeding SATD (SURVEY 8f-2) -------------------------------------------------------------------------------
 * For every block (x, y; integer vector start_x/start_y; PU sides 4..64, powers of two, square or rectangular) the distortion dfunc -- VVB_DF_SAD, VVB_DF_HAD or
 * VVB_DF_HAD_FAST, i.e. what setDistParam( ..., m_bUseHADME ? ( m_fastHad ? 2 : 1 ) : 0 ) selects (InterSearch.cpp:775), with the tile rules of xGetHADs -- between the original and
 * the filtered block at every quarter-pel offset (i, j), i, j = -3..3: cost_out[n][j+3][i+3] -- every position InterSearch::xPatternRefinement
 * (InterSearch.cpp:760-972) can visit in its half-pel round and in its quarter-pel round around the best half-pel position.  The filtered blocks are
 * produced exactly as there: InterpolationFilter::filterHor(frac_x, isLast=false) then filterVer(frac_y, isFirst=false, isLast=true) with the 8-tap
 * luma filter family of InterpolationFilter.cpp:557-600: reduce_tap = m_meReduceTap (0: 8-tap m_lumaFilter, 1: 6-tap m_lumaFilter4x4, 2: 4-tap
 * m_chromaFilter[frac<<1], the value every preset sets), alt_hpel = useAltHpelIf (half-pel phase from m_lumaAltHpelIFilter).  The MV rate and the
 * two-round selection replay on the host from the table: m_fastSubPel = 0 and 1 (early stops, pattern id, skip table) in integration/InterSearchB200.h
 * (xPatternSearchFracDIFB200) and vvenc_b200/candidates.py (subpel_refinement, subpel_refinement_fast); m_fastSubPel = 2 has no fractional search. */
int vvb_frac_cost_grid    ( vvb_ctx* ctx, int dfunc, int org_plane, int ref_plane, const vvb_block* blocks, int n, int w, int h, int reduce_tap, int alt_hpel, uint32_t* cost_out );
int vvb_frac_cost_grid_dev( vvb_ctx* ctx, int dfunc, int org_plane, int ref_plane, const vvb_block* dev_blocks, int n, int w, int h, int reduce_tap, int alt_hpel, uint32_t* dev_cost_out );

/* Fractional motion refinement on the device = InterSearch::xPatternSearchFracDIF (EncoderLib/InterSearch.cpp:2678-2724) for every PU of a call, one PU shape per call
 * (w, h in 4..128, powers of two, not 4x4): the half-pel round and the quarter-pel round of xPatternRefinement (:760-972) with their selection on the device, so the
 * results equal the member's bit for bit -- the strict `<` in the order of s_acMvRefineH / s_acMvRefineQ, the uiDistBest each round starts from (:769) and the distH
 * values, and with fast_sub_pel = 1 the early stops (:808-811), the pattern id in wrapping Distortion arithmetic (:886-969) and the s_skipQpelPosition masks; pattern 0
 * ends the search after the half-pel round (qter stays 0, 0).  The filtered blocks and the distortion are those of vvb_frac_cost_grid.  MV rate: Distortion( sqrt(lambda)
 * * bits ) as for vvb_tz_search, cost scale 1 in the half-pel round and 0 in the quarter-pel round, imvShift 0 (:2696, :2714, :873).
 * Inputs are the arrays of vvb_tz_search: pus[i] gives the position (x, y) and the quarter-pel predictor (pred_hor, pred_ver; the other fields are ignored), int_mv[i]
 * the integer vector (mv_hor, mv_ver; the other fields are ignored), so vvb_tz_search_dev followed by vvb_frac_search_dev chains without a copy.
 * Reads are not clamped: a PU reads reference columns x + mv_hor - 5 .. x + mv_hor + w + 4 and rows y + mv_ver - 4 .. y + mv_ver + h + 3 (the +-1 pel of the
 * refinement, the 8-tap reach, and one column on each side for the pel-pair alignment of the window load).  Every vector vvb_tz_search can return is covered by a
 * reference margin of tz->ctu_size + 12 pels.
 * Errors: null pointers, negative n, fast_sub_pel outside 0..1 (m_fastSubPel = 2 never calls the member, :2113), reduce_tap outside 0..2, a negative or non-finite lambda,
 * and (host-buffer call) a PU outside the original plane: VVB_ERR_ARG; shapes outside the domain, a dfunc other than SAD / HAD / HAD_FAST, planes above 12 bits and
 * (host-buffer call) a PU whose read box leaves the reference margin: VVB_ERR_UNSUPPORTED.  n == 0 returns VVB_OK without a launch.
 * The _dev twin checks the position and the read box per PU on the device before any read: a PU that fails gets cost = UINT64_MAX and offsets 0 (a real result is
 * never that value: the half-pel round always evaluates its position 0). */
typedef struct
{
  double  lambda;                  /* RdCost::setLambda                                                                                    */
  int32_t dfunc;                   /* VVB_DF_SAD / VVB_DF_HAD / VVB_DF_HAD_FAST: m_bUseHADME ? ( m_fastHad ? 2 : 1 ) : 0 (:775)               */
  int32_t reduce_tap;              /* m_meReduceTap, 0..2                                                                                  */
  int32_t alt_hpel;                /* cStruct.useAltHpelIf; implies imvShift == IMV_HPEL, i.e. no quarter-pel round (:2711)                */
  int32_t fast_sub_pel;            /* m_fastSubPel, 0 or 1                                                                                 */
} vvb_frac_par;
/* rcMvHalf, rcMvQter (offsets in half / quarter pel) and ruiCost as the member returns them */
typedef struct { int16_t half_hor, half_ver, qter_hor, qter_ver; uint64_t cost; } vvb_frac_best;   /* 16 bytes */
int vvb_frac_search    ( vvb_ctx* ctx, int org_plane, int ref_plane, const vvb_tz_pu* pus, const vvb_tz_best* int_mv, int n, int w, int h,
                         const vvb_frac_par* par, vvb_frac_best* out );
int vvb_frac_search_dev( vvb_ctx* ctx, int org_plane, int ref_plane, const vvb_tz_pu* dev_pus, const vvb_tz_best* dev_int_mv, int n, int w, int h,
                         const vvb_frac_par* par, vvb_frac_best* dev_out );

/* Bi-predictive motion refinement on the device = the bBi branch of InterSearch::xMotionEstimation (EncoderLib/InterSearch.cpp:1976-2132) with cu.imv IMV_OFF or
 * IMV_HPEL, for every PU of a call, one PU shape per call (w, h in 4..128, powers of two, no larger than par->ctu_size, not 4x4 / 4x8 / 8x4: CU::isBipredRestriction).
 *   target   the search key is 2 * org - pred (AreaBuf::removeHighFreq, Buffer.h:448-480), ClipPel( 2 * org - pred ) with par->clip; pred is the other list's
 *            prediction, passed per PU as a compact w x h block of pred[n][h][w] in the original's bit depth.  The target spans -(2^bd - 1) .. 2^(bd + 1) - 2 and is
 *            held as int16 (bd <= 12); the distortion takes it in signed arithmetic, no packed format that assumes samples in 0 .. 2^bd - 1.
 *   start    (:2051-2090) the SAD + MV rate of the start vector (start_hor / ver, xClipMvSearch with ifp_lines, then changePrecision to integer pel), then of every
 *            candidate cands[cand_first .. +cand_count) that does not repeat an earlier one of the list, clipped the same way; strict `<`; the window is centred
 *            on the unclipped winner.
 *   integer  xSetSearchRange( bestInitMv, search_range ) and xPatternSearch (:2209-2251): SAD over the window in raster order, first strictly smaller cost wins; MV
 *            rate at cost scale 2 and imvShift (1 with IMV_HPEL); row sub-sampling from sub_shift_mode as RdCost::setDistParam (RdCost.cpp:185-200).  The full SAD
 *            is always summed: the member's early exit is decision-equivalent.
 *   fraction xPatternSearchFracDIF (:2678-2724) on the target, exactly as vvb_frac_search (dfunc, reduce_tap, fast_sub_pel; IMV_HPEL: the alternative half-pel
 *            filter and no quarter-pel round).  fast_sub_pel == 2 has no fractional stage: frac_cost is xPatternSearch's ruiSAD (the SAD without the rate).
 *   final    (:2117-2124) rcMv = ( int << 2 ) + ( half << 1 ) + qter in quarter pel; uiMvBits at cost scale 0 and imvShift; bits = ruiBits + uiMvBits (uint32);
 *            cost = (Distortion)( floor( fWeight * ( (double) frac_cost - (double) getCost( uiMvBits ) ) ) + (double) getCost( bits ) ) in IEEE double without
 *            contraction, getCost( b ) = Distortion( sqrt( lambda ) * b ), fWeight = | getBcwWeight( bcw_idx, ref_list ) | / 8 ({ -2, 3, 4, 5, 10 }, Rom.cpp:1152-1163)
 *            or 0.5 for bcw_idx 2 (BCW_DEFAULT).  The (Distortion) conversion is the x86-64 one the encoder is built with (cvttsd2si below 2^63, cvttsd2si of
 *            v - 2^63 with the top bit flipped at or above; cvttsd2si yields 2^63 outside the int64 range): a negative value -k becomes 2^64 - k, as happens with
 *            fast_sub_pel == 2, a SAD of 0, weight 1.25 and few bits; a value at or above 2^64 becomes 0, as happens with fast_sub_pel == 2 and weight 1.25 when the
 *            search window is empty (xPatternSearch's cost is then MAX_DISTORTION).
 *            mv = rcMv in internal units (1/16 pel).
 * Domain: bit depths 8..12; search_range 0..VVB_BIPRED_MAX_RANGE; dfunc SAD with fast_sub_pel 1 only for w < 64 (for wider PUs the member's AVX2 SAD returns
 * early-exit partial sums, RdCostX86.h:372-405, which xPatternRefinement keeps in distH and turns into its pattern id); imv 1 (IMV_FPEL) and 2 (IMV_4PEL) go to xPatternSearchIntRefine in the encoder and are VVB_ERR_UNSUPPORTED here: vvb_bipred_amvr_search runs that branch.
 * Reads are not clamped.  A PU reads the blocks at its clipped start and candidate vectors, the blocks of the window around each of them (the zero vector when a
 * window is empty) and the fractional stage's box around the winner (columns mv - 5 .. mv + w + 4, rows mv - 4 .. mv + h + 3, as vvb_frac_search).  Every vector
 * the clip rules allow is covered by a reference margin of ctu_size + 12 pels (beyond the picture's right and bottom edges w + 12 columns and h + 11 rows suffice).
 * Errors: null pointers, negative counts, settings out of range, a negative or non-finite lambda and (host-buffer call) PUs outside the picture, candidate ranges
 * outside cands or a bcw_idx outside 0..4: VVB_ERR_ARG; shapes, imv or dfunc / fast_sub_pel outside the domain, planes above 12 bits, an original plane smaller than the picture and
 * (host-buffer call) a PU whose read box leaves the reference margin: VVB_ERR_UNSUPPORTED.  n == 0 returns VVB_OK without a launch.
 * The _dev twin checks each PU on the device before any read: a PU that fails gets cost = frac_cost = int_best = UINT64_MAX and zero vectors and bits. */
#define VVB_BIPRED_MAX_RANGE 8
typedef struct
{
  int32_t x, y;                    /* PU position in the original plane (inside the picture)                                                             */
  int32_t start_hor, start_ver;    /* rcMv on entry: internal units (1/16 pel), not clipped                                                              */
  int16_t pred_hor, pred_ver;      /* RdCost::setPredictor, quarter pel (as vvb_tz_pu)                                                                   */
  int32_t cand_first, cand_count;  /* m_BlkUniMvInfoBuffer's uniMvs[refPicList][iRefIdxPred] as cands[cand_first .. +cand_count), buffer order, internal units */
  uint32_t bits;                   /* ruiBits on entry                                                                                                   */
  int32_t bcw_idx;                 /* cu.BcwIdx, 0..4                                                                                                    */
} vvb_bi_pu;                       /* 36 bytes */
typedef struct
{
  double  lambda;                  /* RdCost::setLambda                                                                                                  */
  int32_t search_range;            /* m_bipredSearchRange, 0..VVB_BIPRED_MAX_RANGE                                                                      */
  int32_t sub_shift_mode;          /* TZSearchStruct::subShiftMode, 0..2                                                                                 */
  int32_t pic_w, pic_h, ctu_size, ifp_lines;   /* pcv.lumaWidth, pcv.lumaHeight, pcv.maxCUSize (16..128), m_pcEncCfg->m_ifpLines                      */
  int32_t ref_list;                /* refPicList being refined, 0 or 1                                                                                  */
  int32_t clip;                    /* m_bClipForBiPredMeEnabled                                                                                         */
  int32_t imv;                     /* cu.imv: 0 IMV_OFF or 3 IMV_HPEL (vvb_bipred_amvr_search: 1 IMV_FPEL or 2 IMV_4PEL)                                  */
  int32_t fast_sub_pel;            /* m_fastSubPel, 0..2                                                                                                 */
  int32_t dfunc;                   /* fractional stage: VVB_DF_SAD / VVB_DF_HAD / VVB_DF_HAD_FAST                                                        */
  int32_t reduce_tap;              /* m_meReduceTap, 0..2                                                                                                */
} vvb_bi_par;                      /* 56 bytes */
typedef struct
{
  int32_t int_hor, int_ver;        /* xPatternSearch's rcMv, integer pel                                                                                 */
  uint64_t int_best;               /* cStruct.uiBestSad                                                                                                  */
  uint64_t frac_cost;              /* ruiCost after xPatternSearchFracDIF (xPatternSearch's ruiSAD with fast_sub_pel == 2)                               */
  int16_t half_hor, half_ver, qter_hor, qter_ver;   /* rcMvHalf, rcMvQter                                                                            */
  int32_t mv_hor, mv_ver;          /* final rcMv, internal units                                                                                         */
  uint32_t bits, pad;              /* final ruiBits                                                                                                      */
  uint64_t cost;                   /* final ruiCost                                                                                                      */
} vvb_bi_best;                     /* 56 bytes */
int vvb_bipred_search    ( vvb_ctx* ctx, int org_plane, int ref_plane, const vvb_bi_pu* pus, int n, int w, int h, const vvb_bi_par* par,
                           const int32_t* cands /* [n_cands][2]; nullable when n_cands == 0 */, int n_cands, const int16_t* pred /* [n][h][w] */, vvb_bi_best* out );
int vvb_bipred_search_dev( vvb_ctx* ctx, int org_plane, int ref_plane, const vvb_bi_pu* dev_pus, int n, int w, int h, const vvb_bi_par* par,
                           const int32_t* dev_cands, int n_cands, const int16_t* dev_pred, vvb_bi_best* dev_out );

/* AMVR integer refinement on the device = InterSearch::xPatternSearchIntRefine (EncoderLib/InterSearch.cpp:2576-2676), the end of xMotionEstimation for cu.imv
 * 1 (IMV_FPEL) and 2 (IMV_4PEL) (:2126-2130), for every PU of a call, one PU shape per call (w, h in 4..128, powers of two, no larger than ctu_size).  Per PU, in
 * internal units (1/16 pel), with s = 4 (IMV_FPEL) or 6 (IMV_4PEL) the shift from internal units to the AMVR precision (Mv.cpp:57):
 *   entry    rcMv = 16 * the integer vector; bits = ruiBits - mvp_bits[mvp_idx] (uint32).  cBaseMvd[c] = rcMv - cand[c] for c = 0 and 1 (both, as the member),
 *            rounded to the AMVR precision and back (changePrecision's rounding: (v + 2^(s-1) - 1) >> s for v >= 0, (v + 2^(s-1)) >> s below, Mv.h:189-203).
 *   points   position-major, testPos (0,0) (-1,-1) (-1,0) (-1,1) (0,-1) (0,1) (1,-1) (1,0) (1,1) as (hor, ver), then c = 0 .. num_cand - 1:
 *            t = ( testPos << s ) + cBaseMvd[c] + cand[c].  With ifp_lines, a vertical component outside CU::isMvInRangeFPP (UnitTools.cpp:3526-3535, PUs above row
 *            yBMax only) is clipped by xClipMvToFppLine (:2154-2163) and rounded to the AMVR precision again (roundTransPrecInternal2AmvrVertical, Mv.h:227-234).
 *   distortion  dfunc (VVB_DF_SAD / VVB_DF_HAD / VVB_DF_HAD_FAST, what setDistParam( ..., m_bUseHADME ? ( m_fastHad ? 2 : 1 ) : 0 ) selects, no row sub-sampling)
 *            of the key against the reference block at clipMv( t ) >> 4 (Mv.cpp:68-80), full sums; computed for c = 0 and where t differs from candidate 0's t, else
 *            candidate 0's value; dist = (Distortion)( sum * fWeight ) in IEEE double with the x86-64 conversion of vvb_bipred_search.
 *   rate     bits = mvp_bits[c] + getBitsOfVectorWithPredictor at cost scale 0 of t and cand[c], both changed to the AMVR precision first (uint32); cost = dist +
 *            getCost( bits ) (uint64 wrapping), getCost( b ) = Distortion( sqrt( lambda ) * b ) computed directly (no 32-bit table, so any lambda and any bits).
 *   result   the first strictly smaller cost wins in that order: mv = its t, mvp_idx = its c, dist = uiBestDist, bits += its bits, cost = dist - getCost( its bits )
 *            + getCost( bits ) (uint64 wrapping).  If no cost is below UINT64_MAX the member's :2655-2659 holds: cost = dist = UINT64_MAX, mv = rcMv and the entry
 *            mvp_idx, bits as decremented (finite distortions never get there).
 * Reads are not clamped: every block the refinement reads lies in the box clipMv allows, columns -(ctu_size + 7) .. pic_w + w + 6 and rows -(ctu_size + 7) ..
 * pic_h + h + 6 around sample (0, 0) -- the box of vvb_tz_search -- and a call whose ref_plane margin does not cover it returns VVB_ERR_UNSUPPORTED.
 * Inputs on which the member throws (CHECK, :2579-2580, :2601-2602) are refused: num_cand outside 1..2, mvp_idx outside 0..num_cand - 1, 4 * (pred_hor, pred_ver)
 * != cand[mvp_idx], or a cBaseMvd component that is not a multiple of 4.  The host-buffer calls return VVB_ERR_ARG for them; the _dev twins check each PU on
 * the device before any read and give such a PU (and a PU outside the picture) the sentinel cost = dist = UINT64_MAX, mv = 0, bits = 0, mvp_idx = -1. */
typedef struct
{
  int32_t cand_hor[2], cand_ver[2];  /* amvpInfo.mvCand, internal units                                                                                    */
  int32_t num_cand;                  /* amvpInfo.numCand, 1..2                                                                                             */
  int32_t mvp_idx;                   /* riMVPIdx on entry                                                                                                  */
} vvb_amvp;                          /* 24 bytes */
typedef struct
{
  int32_t mv_hor, mv_ver;            /* final rcMv, internal units                                                                                         */
  int32_t mvp_idx;                   /* final riMVPIdx                                                                                                     */
  uint32_t bits;                     /* final ruiBits                                                                                                      */
  uint64_t dist;                     /* uiBestDist: weighted distortion plus the winner's MV and MVP-index rate                                            */
  uint64_t cost;                     /* final ruiCost                                                                                                      */
} vvb_amvr_best;                     /* 32 bytes */
typedef struct
{
  double   lambda;                   /* RdCost::setLambda                                                                                                  */
  int32_t  dfunc;                    /* VVB_DF_SAD / VVB_DF_HAD / VVB_DF_HAD_FAST                                                                          */
  int32_t  imv;                      /* cu.imv: 1 IMV_FPEL or 2 IMV_4PEL (0 and 3 refine with vvb_frac_search: VVB_ERR_UNSUPPORTED)                        */
  uint32_t mvp_bits[2];              /* m_auiMVPIdxCost[0|1][AMVP_MAX_NUM_CANDS] (InterSearch.cpp:241-253)                                                */
  int32_t  pic_w, pic_h, ctu_size, ifp_lines;   /* pcv.lumaWidth, pcv.lumaHeight, pcv.maxCUSize (16..128), m_pcEncCfg->m_ifpLines                        */
} vvb_amvr_par;                      /* 40 bytes */
/* The uni-prediction branch (fWeight 1.0, the key is the original block).  Inputs are the arrays of vvb_tz_search: pus[i] gives the position (x, y) and the
 * quarter-pel predictor (pred_hor, pred_ver; the other fields are ignored), int_mv[i] the integer vector (mv_hor, mv_ver; the other fields are ignored), so
 * vvb_tz_search_dev (imv_shift 2 or 4) followed by vvb_amvr_refine_dev chains without a copy.  amvp[i] is the PU's amvpInfo and riMVPIdx, bits[i] its ruiBits.
 * Errors: null pointers, negative n, settings out of range (picture sides 1..16384, ctu_size a power of two 16..128, ifp_lines 0..1024, imv 0..3), a negative
 * or non-finite lambda and (host-buffer call) PUs outside the picture or the member's CHECK inputs: VVB_ERR_ARG; shapes outside the domain, imv 0 or 3, a dfunc
 * other than SAD / HAD / HAD_FAST, planes above 12 bits, an original plane smaller than the picture or a too small reference margin: VVB_ERR_UNSUPPORTED.
 * n == 0 returns VVB_OK without a launch. */
int vvb_amvr_refine    ( vvb_ctx* ctx, int org_plane, int ref_plane, const vvb_tz_pu* pus, const vvb_tz_best* int_mv, const vvb_amvp* amvp, const uint32_t* bits,
                         int n, int w, int h, const vvb_amvr_par* par, vvb_amvr_best* out );
int vvb_amvr_refine_dev( vvb_ctx* ctx, int org_plane, int ref_plane, const vvb_tz_pu* dev_pus, const vvb_tz_best* dev_int_mv, const vvb_amvp* dev_amvp,
                         const uint32_t* dev_bits, int n, int w, int h, const vvb_amvr_par* par, vvb_amvr_best* dev_out );
/* The bi-predictive branch of xMotionEstimation for cu.imv 1 and 2 in one call: the integer stage of vvb_bipred_search (target, start selection and window, MV
 * rate at cost scale 2 and imvShift = imv << 1, :2020) into int_out (vvb_tz_search's layout: mv in integer pel, sad = ruiSAD, cost = uiBestSad), then
 * xPatternSearchIntRefine on the target 2 * org - pred with fWeight = xGetMEDistortionWeight( bcw_idx, ref_list ) (:2004, the weight of vvb_bipred_search's final
 * cost), pus[i].bits as ruiBits and pus[i].pred_hor / pred_ver as the predictor.  par is vvb_bipred_search's with imv 1 or 2 (0 and 3 belong to vvb_bipred_search:
 * VVB_ERR_UNSUPPORTED); fast_sub_pel and reduce_tap are ignored; mvp_bits as vvb_amvr_par's.
 * Reads: the integer stage keeps vvb_bipred_search's per-PU rule (a PU whose read box leaves the reference margin: VVB_ERR_UNSUPPORTED from the host-buffer call,
 * the sentinel from the _dev twin), the refinement needs the margin of vvb_amvr_refine for the call (VVB_ERR_UNSUPPORTED otherwise).
 * Errors as vvb_bipred_search and vvb_amvr_refine; the _dev twin gives a PU that the integer stage refuses int_out mv = (-2^30, -2^30), sad = cost = 0, and
 * the sentinel of vvb_amvr_refine in out. */
int vvb_bipred_amvr_search    ( vvb_ctx* ctx, int org_plane, int ref_plane, const vvb_bi_pu* pus, const vvb_amvp* amvp, int n, int w, int h, const vvb_bi_par* par,
                                const uint32_t mvp_bits[2], const int32_t* cands /* [n_cands][2]; nullable when n_cands == 0 */, int n_cands,
                                const int16_t* pred /* [n][h][w] */, vvb_tz_best* int_out /* nullable */, vvb_amvr_best* out );
int vvb_bipred_amvr_search_dev( vvb_ctx* ctx, int org_plane, int ref_plane, const vvb_bi_pu* dev_pus, const vvb_amvp* dev_amvp, int n, int w, int h,
                                const vvb_bi_par* par, const uint32_t mvp_bits[2], const int32_t* dev_cands, int n_cands, const int16_t* dev_pred,
                                vvb_tz_best* dev_int_out, vvb_amvr_best* dev_out );

/* ---- MCTF apply stage (SURVEY 8f-3): the per-block body of MCTF::xFinalizeBlkLine (MCTF.cpp:1437-1483) for the luma plane, fused:
 * per reference picture applyFrac (m_applyFrac, :259-357) at the block's vector, applyPlanarCorrection (:372-420) when rmsme > 0 and
 * planar_correction (the caller passes m_QP <= 32) and the block is square <= 32, then applyBlock (:422-518: noise estimate, weights, bilateral
 * blend with fastExp).  mvs[r][block] in raster order of block_size x block_size units; out is the filtered luma plane (newOrgPic).
 * Float results equal the reference's scalar and AVX2 kernels bit for bit. */
typedef struct { int32_t x, y; int32_t error; uint16_t rmsme, pad; } vvb_mctf_mv;                       /* 16 bytes; MotionVector (MCTF.h:72-82), 1/16 pel */
typedef struct { int32_t num_refs, block_size, low_res_filter /* 4-tap */, planar_correction; double weight_scaling /* overallStrength * 0.4 */, sigma_sq;
                 double ref_strength[8]; int32_t ref_plane[8]; } vvb_mctf_apply_par;
int vvb_mctf_apply    ( vvb_ctx* ctx, int org_plane, const vvb_mctf_apply_par* par, const vvb_mctf_mv* mvs, int16_t* out, int out_stride );
int vvb_mctf_apply_dev( vvb_ctx* ctx, int org_plane, const vvb_mctf_apply_par* par, const vvb_mctf_mv* dev_mvs, int16_t* dev_out, int out_stride );
/* MCTF::m_calcVar (calcVarCore, MCTF.cpp:520-546) for a list of blocks (x, y, w, h of vvb_mctf_cand; vectors ignored) */
int vvb_mctf_calc_var    ( vvb_ctx* ctx, int plane, const vvb_mctf_cand* blocks, int n, double* var_out );
int vvb_mctf_calc_var_dev( vvb_ctx* ctx, int plane, const vvb_mctf_cand* dev_blocks, int n, double* dev_var_out );

/* MCTF motion search with the control on the device (SURVEY a5; MCTF::motionEstimationLuma, MCTF.cpp:1329-1397 -> estimateLumaLn :1166-1327).  One call runs a whole
 * level for the whole picture: predictor candidates from the coarser level's field, the integer grid, the three sub-pel grids of the final level, the
 * `error < best.error` chains in the reference's loop order, the candidates of the block above and the block to the left (one warp per block row that waits for
 * the row above -- the prevLineX scheme of :1176, 1357-1386) and the final error scaling; the host sees no number in between.  The field is an array of
 * out_w x out_h vvb_mctf_mv in raster order (entries no block writes keep the default vector 0, 0, as the reference's field arrays do); it is what
 * vvb_mctf_apply_dev takes.  prev: field of the coarser level (prev_w x prev_h), null for the first level.  factor: m_motionVectorFactor scale between levels.
 * search_pattern: 0 / 1 / 2 as MCTFSpeed 0 / 1-2 / 3-4 select (:598-599).  Block sizes: multiples of 8 up to 64. */
typedef struct { int32_t block_size, factor, double_res, search_pattern, low_res_filter, prev_w, prev_h, out_w, out_h; } vvb_mctf_level_par;
int vvb_mctf_estimate_level    ( vvb_ctx* ctx, int org_plane, int ref_plane, const vvb_mctf_level_par* par, const vvb_mctf_mv* prev, vvb_mctf_mv* field_out );
int vvb_mctf_estimate_level_dev( vvb_ctx* ctx, int org_plane, int ref_plane, const vvb_mctf_level_par* par, const vvb_mctf_mv* dev_prev, vvb_mctf_mv* dev_field_out );
/* MCTF::motionEstimationMCTF (MCTF.cpp:666-724) for one neighbour picture: MCTF::subsampleLuma twice (three times with add_level) into context-owned planes with
 * 128 pels of border replication, then the levels 2u / 2u / 2u (/ 2u) / u chained through device-resident fields.  field_out: ceil(W / unit) x ceil(H / unit)
 * entries.  Both planes need a margin that covers the vectors (MCTF_PADDING = 128). */
typedef struct { int32_t unit_size, add_level, search_pattern, low_res_filter; } vvb_mctf_pyr_par;
int vvb_mctf_estimate_pyramid    ( vvb_ctx* ctx, int org_plane, int ref_plane, const vvb_mctf_pyr_par* par, vvb_mctf_mv* field_out );
int vvb_mctf_estimate_pyramid_dev( vvb_ctx* ctx, int org_plane, int ref_plane, const vvb_mctf_pyr_par* par, vvb_mctf_mv* dev_field_out );

/* ---- affine gradient helpers (CommonLib/AffineGradientSearch.cpp:84-190) ---------------------------------- */
int vvb_affine_sobel      ( vvb_ctx* ctx, int vertical, const int16_t* pred, int pred_stride, int16_t* deriv, int deriv_stride, int w, int h );
int vvb_affine_equal_coeff( vvb_ctx* ctx, int six_param, const int16_t* resi, int resi_stride, const int16_t* deriv_x, const int16_t* deriv_y,
                            int deriv_stride, int w, int h, int64_t eq_out[49] /* accumulated into, row stride 7 */ );

/* a16, batched: for n blocks of one shape (pred, resi compact [n][h][w]) the horizontal and vertical Sobel of the prediction and the normal-equation sums of
 * xEqualCoeffComputer in one launch -- the per-iteration body of the affine motion estimation (InterSearch.cpp:5373-5387).  eq_out [n][49] (row stride 7, rows 1..np,
 * written, not accumulated); deriv_x / deriv_y [n][h][w] nullable. */
int vvb_affine_eq_batch    ( vvb_ctx* ctx, int six_param, const int16_t* pred, const int16_t* resi, int n, int w, int h, int16_t* deriv_x, int16_t* deriv_y, int64_t* eq_out );
int vvb_affine_eq_batch_dev( vvb_ctx* ctx, int six_param, const int16_t* dev_pred, const int16_t* dev_resi, int n, int w, int h, int16_t* dev_deriv_x, int16_t* dev_deriv_y,
                             int64_t* dev_eq_out );

#ifdef __cplusplus
}
#endif
#endif
