"""Host-side mirror of the reference's cost interfaces on top of the C ABI (include/vvenc_b200.h).

`CostEngine` plays the role one `RdCost` + `TrQuant` pair plays for an encoder worker
(EncoderLib/EncCu.h:265-272): it owns a context (one CUDA stream), resident pictures and exposes

  getDistPart-like single calls .... dist_block / sad_mask_block / sad_x5_block / fix_wsse_block   (RdCost.h:74-75,117)
  batched candidate evaluation ..... dist_batch (descriptor list), dist_pool (RDO candidate pools)
  motion search .................... sad_search (xPatternSearch), sad_pattern (fixed TZ point set), tz_search (xTZSearch walk), frac_search (xPatternSearchFracDIF),
                                     bipred_search (the bi-predictive branch of xMotionEstimation)
  TU coding ........................ fwd_trquant (TrQuant::transformNxN: xT + Quant::quant + xNeedRDOQ)
  pre-analysis ..................... mctf_error_batch (MCTF::motionErrorLuma)
  affine ME ........................ affine_sobel / affine_equal_coeff

numpy arrays are host buffers (copied inside the call: the end-to-end path).  The *_dev methods take raw device
pointers (e.g. torch tensors' data_ptr()) and only enqueue work on the context stream.
Errors surface as VvbError carrying the reference-style reason; nothing falls back to the CPU.
"""
import ctypes
import numpy as np
from . import _lib as L

DF_SSE, DF_SAD, DF_HAD, DF_HAD_FAST, DF_HAD_2SAD = range(5)
DCT2, DCT8, DST7 = 0, 1, 2


class VvbError(RuntimeError):
    def __init__(self, code, msg):
        super().__init__('vvenc_b200 error %d: %s' % (code, msg))
        self.code = code


def _p(a):
    return None if a is None else a.ctypes.data_as(ctypes.c_void_p)


def _po(a, off):
    return ctypes.c_void_p(a.ctypes.data + off * a.itemsize)


class CostEngine:
    def __init__(self, device=0):
        self.lib = L.load()
        h = ctypes.c_void_p()
        rc = self.lib.vvb_create(ctypes.byref(h), device)
        if rc != L.VVB_OK:
            raise VvbError(rc, 'vvb_create failed (no usable CUDA device?)')
        self.h = h
        self._planes = {}

    # ---- lifetime
    def close(self):
        if self.h:
            self.lib.vvb_destroy(self.h); self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _chk(self, rc):
        if rc != L.VVB_OK:
            raise VvbError(rc, self.lib.vvb_last_error(self.h).decode())

    def synchronize(self):
        self._chk(self.lib.vvb_synchronize(self.h))

    def set_async(self, enable=True):
        """host-buffer calls only enqueue; synchronize() completes them (buffers should be page-locked)"""
        self._chk(self.lib.vvb_set_async(self.h, int(enable)))

    @property
    def stream(self):
        return self.lib.vvb_stream(self.h)

    @property
    def launches(self):
        n = ctypes.c_uint64()
        self._chk(self.lib.vvb_launch_count(self.h, ctypes.byref(n)))
        return n.value

    # ---- pictures
    def upload_plane(self, plane_id, padded, width, height, margin, bit_depth=10):
        """padded: 2-D int16 array of shape (>= height + 2*margin, stride) whose sample (0,0) sits at [margin, margin]"""
        assert padded.dtype == np.int16 and padded.ndim == 2 and padded.flags['C_CONTIGUOUS']
        stride = padded.shape[1]
        self._chk(self.lib.vvb_plane_upload(self.h, plane_id, _po(padded, margin * stride + margin), stride, width, height, margin, bit_depth))
        self._planes[plane_id] = (width, height, margin, bit_depth)

    def bind_plane_dev(self, plane_id, dev_origin_ptr, stride, width, height, margin, bit_depth=10):
        self._chk(self.lib.vvb_plane_bind_dev(self.h, plane_id, ctypes.c_void_p(dev_origin_ptr), stride, width, height, margin, bit_depth))
        self._planes[plane_id] = (width, height, margin, bit_depth)

    def free_plane(self, plane_id):
        self._chk(self.lib.vvb_plane_free(self.h, plane_id)); self._planes.pop(plane_id, None)

    # ---- distortion
    def dist_batch(self, cands):
        cands = np.ascontiguousarray(cands, dtype=L.CAND_DT)
        out = np.zeros(len(cands), dtype=np.uint64)
        self._chk(self.lib.vvb_dist_batch(self.h, _p(cands), len(cands), _p(out)))
        return out

    def dist_block(self, dfunc, org, org_stride, cur, cur_stride, w, h, bit_depth=10, sub_shift=0):
        err = ctypes.c_int(0)
        v = self.lib.vvb_dist_block(self.h, dfunc, _p(org), org_stride, _p(cur), cur_stride, w, h, bit_depth, sub_shift, ctypes.byref(err))
        self._chk(err.value)
        return int(v)

    def sad_mask_block(self, org, org_stride, cur, cur_stride, w, h, mask, mask_off, mask_stride, step_x, mask_stride2, sub_shift=0):
        err = ctypes.c_int(0)
        v = self.lib.vvb_sad_mask_block(self.h, _p(org), org_stride, _p(cur), cur_stride, w, h, _po(mask, mask_off), mask_stride, step_x, mask_stride2,
                                        sub_shift, ctypes.byref(err))
        self._chk(err.value)
        return int(v)

    def sad_x5_block(self, org, org_off, org_stride, cur, cur_off, cur_stride, w, h, sub_shift=1, calc_centre=True):
        out = np.zeros(5, dtype=np.uint64)
        self._chk(self.lib.vvb_sad_x5_block(self.h, _po(org, org_off), org_stride, _po(cur, cur_off), cur_stride, w, h, sub_shift, int(calc_centre), _p(out)))
        return out

    def fix_wsse_block(self, org, org_stride, cur, cur_stride, w, h, weight):
        err = ctypes.c_int(0)
        v = self.lib.vvb_fix_wsse_block(self.h, _p(org), org_stride, _p(cur), cur_stride, w, h, weight, ctypes.byref(err))
        self._chk(err.value)
        return int(v)

    # ---- descriptor-list forms of the mask SAD (GEO), the five-position SAD (DMVR) and the weighted SSE; blocks in resident planes
    def mask_upload(self, mask):
        mask = np.ascontiguousarray(mask, dtype=np.int16)
        self._chk(self.lib.vvb_mask_upload(self.h, _p(mask), mask.size))

    def sad_mask_batch(self, cands):
        cands = np.ascontiguousarray(cands, dtype=L.MASK_CAND_DT)
        out = np.zeros(len(cands), dtype=np.uint64)
        self._chk(self.lib.vvb_sad_mask_batch(self.h, _p(cands), len(cands), _p(out)))
        return out

    def sad_x5_batch(self, cands):
        cands = np.ascontiguousarray(cands, dtype=L.CAND_DT)
        out = np.zeros((len(cands), 5), dtype=np.uint64)
        self._chk(self.lib.vvb_sad_x5_batch(self.h, _p(cands), len(cands), _p(out)))
        return out

    def fix_wsse_batch(self, cands, weights):
        cands = np.ascontiguousarray(cands, dtype=L.CAND_DT); weights = np.ascontiguousarray(weights, dtype=np.uint32)
        out = np.zeros(len(cands), dtype=np.uint64)
        self._chk(self.lib.vvb_fix_wsse_batch(self.h, _p(cands), _p(weights), len(cands), _p(out)))
        return out

    def affine_eq_batch(self, six_param, pred, resi, want_derivs=False):
        """pred, resi: int16 [n][h][w] -> eq int64 [n][7][7] (rows 1..np filled) and, on request, the two Sobel planes [n][h][w]"""
        pred = np.ascontiguousarray(pred, dtype=np.int16); resi = np.ascontiguousarray(resi, dtype=np.int16)
        n, h, w = pred.shape
        eq = np.zeros((n, 7, 7), dtype=np.int64)
        gx = np.zeros_like(pred) if want_derivs else None; gy = np.zeros_like(pred) if want_derivs else None
        self._chk(self.lib.vvb_affine_eq_batch(self.h, int(six_param), _p(pred), _p(resi), n, w, h, _p(gx), _p(gy), _p(eq)))
        return (eq, gx, gy) if want_derivs else eq

    def dist_pool(self, dfunc, org_plane, blocks, w, h, K, pool, sub_shift=0):
        blocks = np.ascontiguousarray(blocks, dtype=L.POS_DT)
        pool = np.ascontiguousarray(pool, dtype=np.int16)
        assert pool.size == len(blocks) * K * w * h
        out = np.zeros(len(blocks) * K, dtype=np.uint32)
        self._chk(self.lib.vvb_dist_pool(self.h, dfunc, org_plane, _p(blocks), len(blocks), w, h, K, _p(pool), sub_shift, _p(out)))
        return out.reshape(len(blocks), K)

    # ---- motion search
    @staticmethod
    def me_par(lam, cost_scale=2, imv_shift=0, sub_shift=0, quad_order=0, pattern_radius=0):
        return L.vvb_me_par(float(lam), cost_scale, imv_shift, sub_shift, quad_order, pattern_radius, 0)

    def sad_search(self, org_plane, ref_plane, blocks, w, h, par, want_tables=False):
        blocks = np.ascontiguousarray(blocks, dtype=L.BLOCK_DT)
        n = len(blocks)
        best = np.zeros(n, dtype=L.BEST_DT)
        ts = 0; tab = None
        if want_tables and n:
            ts = int(((blocks['right'].astype(np.int64) - blocks['left'] + 1) * (blocks['bottom'].astype(np.int64) - blocks['top'] + 1)).max())
            tab = np.zeros((n, ts), dtype=np.uint32)
        self._chk(self.lib.vvb_sad_search(self.h, org_plane, ref_plane, _p(blocks), n, w, h, ctypes.byref(par), _p(tab), ts, _p(best)))
        return (best, tab) if want_tables else best

    def sad_search_pyramid(self, org_plane, ref_plane, level_blocks, base_w, par, nx, ny):
        """level_blocks: list of BLOCK_DT arrays (level 0 = base size).  Device-resident call wrapped with torch buffers; returns [BEST_DT array] per level."""
        import torch
        levels = len(level_blocks)
        d_blk = [torch.from_numpy(np.frombuffer(np.ascontiguousarray(b, dtype=L.BLOCK_DT).tobytes(), dtype=np.uint8).copy()).cuda() for b in level_blocks]
        d_best = [torch.empty(max(1, len(b)) * 16, dtype=torch.uint8, device='cuda') for b in level_blocks]
        pb = (ctypes.c_void_p * levels)(*[t.data_ptr() for t in d_blk])
        po = (ctypes.c_void_p * levels)(*[t.data_ptr() for t in d_best])
        cnt = (ctypes.c_int * levels)(*[len(b) for b in level_blocks])
        torch.cuda.synchronize()
        self._chk(self.lib.vvb_sad_search_pyramid_dev(self.h, org_plane, ref_plane, levels, pb, cnt, base_w, ctypes.byref(par), nx, ny, po))
        self.synchronize()
        return [np.frombuffer(t.cpu().numpy().tobytes(), dtype=L.BEST_DT)[:len(b)].copy() for t, b in zip(d_best, level_blocks)]

    def sad_pattern(self, org_plane, ref_plane, blocks, w, h, pattern, par, want_sad=True, want_best=True):
        blocks = np.ascontiguousarray(blocks, dtype=L.BLOCK_DT)
        pattern = np.ascontiguousarray(pattern, dtype=L.MV_DT)
        n, K = len(blocks), len(pattern)
        sad = np.zeros((n, K), dtype=np.uint32) if want_sad else None
        best = np.zeros(n, dtype=L.BEST_DT) if want_best else None
        self._chk(self.lib.vvb_sad_pattern(self.h, org_plane, ref_plane, _p(blocks), n, w, h, _p(pattern), K, ctypes.byref(par), _p(sad), _p(best)))
        return sad, best

    @staticmethod
    def tz_par(search_range, pic_w, pic_h, ctu_size, extended=False, fast=False, integer_et=False, first_search_stop=False, sub_shift_mode=0, ifp_lines=0):
        return L.vvb_tz_par(search_range, int(extended), int(fast), int(integer_et), int(first_search_stop), sub_shift_mode, pic_w, pic_h, ctu_size, ifp_lines)

    def tz_search(self, org_plane, ref_plane, pus, w, h, me, tz, cands=None):
        """InterSearch::xTZSearch for every PU of one shape.  pus: TZ_PU_DT array; cands: int32 [n_cands][2] (hor, ver, 1/16 pel) the PUs' cand_first /
        cand_count index into.  Returns a TZ_BEST_DT array (mv in integer pels, sad = ruiSAD, cost = uiBestSad, best_distance = uiBestDistance)."""
        pus = np.ascontiguousarray(pus, dtype=L.TZ_PU_DT)
        cands = np.zeros((0, 2), dtype=np.int32) if cands is None else np.ascontiguousarray(cands, dtype=np.int32).reshape(-1, 2)
        out = np.zeros(len(pus), dtype=L.TZ_BEST_DT)
        self._chk(self.lib.vvb_tz_search(self.h, org_plane, ref_plane, _p(pus), len(pus), w, h, ctypes.byref(me), ctypes.byref(tz),
                                         _p(cands) if len(cands) else None, len(cands), _p(out)))
        return out

    def cost_pattern(self, dfunc, org_plane, ref_plane, blocks, w, h, pattern, par, want_cost=True, want_best=True):
        """any distortion family over the fixed pattern (e.g. DF_HAD integer refinement around blocks['start_*'])"""
        blocks = np.ascontiguousarray(blocks, dtype=L.BLOCK_DT)
        pattern = np.ascontiguousarray(pattern, dtype=L.MV_DT)
        n, K = len(blocks), len(pattern)
        cost = np.zeros((n, K), dtype=np.uint32) if want_cost else None
        best = np.zeros(n, dtype=L.BEST_DT) if want_best else None
        self._chk(self.lib.vvb_cost_pattern(self.h, dfunc, org_plane, ref_plane, _p(blocks), n, w, h, _p(pattern), K, ctypes.byref(par), _p(cost), _p(best)))
        return cost, best

    # ---- transform + quantise
    @staticmethod
    def tu_par(w, h, tr_hor=DCT2, tr_ver=DCT2, bit_depth=10, qp=32, is_irap=False, dep_quant=False, sign_hiding=False, lfnst_idx=0, lfnst_set=0, lfnst_transpose=False,
               transform_skip=False, input_bit_depth_delta=0, is_chroma=False):
        return L.vvb_tu_par(w, h, tr_hor, tr_ver, bit_depth, qp, int(is_irap), int(dep_quant), int(sign_hiding), int(lfnst_idx), int(lfnst_set), int(lfnst_transpose),
                            int(transform_skip), int(input_bit_depth_delta), int(is_chroma))

    def set_tma_staging(self, enable):
        self._chk(self.lib.vvb_set_tma_staging(self.h, int(enable)))

    def set_pyramid_engine(self, engine):
        self._chk(self.lib.vvb_set_pyramid_engine(self.h, int(engine)))

    def set_tensor_transform(self, enable):
        self._chk(self.lib.vvb_set_tensor_transform(self.h, int(enable)))

    def fwd_trquant(self, par, resi, want_coef=True):
        """resi: int16 [n][h][w] compact.  Returns dict(coef, q, abs_sum, last_pos, need_rdoq)."""
        resi = np.ascontiguousarray(resi, dtype=np.int16)
        n = resi.shape[0]
        coef = np.zeros((n, par.h, par.w), dtype=np.int32) if want_coef else None
        q = np.zeros((n, par.h, par.w), dtype=np.int16)
        s = np.zeros(n, dtype=np.int32); lp = np.zeros(n, dtype=np.int32); nr = np.zeros(n, dtype=np.uint8)
        self._chk(self.lib.vvb_fwd_trquant(self.h, ctypes.byref(par), _p(resi), n, _p(coef), _p(q), _p(s), _p(lp), _p(nr)))
        return dict(coef=coef, q=q, abs_sum=s, last_pos=lp, need_rdoq=nr)

    def fwd_trquant_planes(self, par, org_plane, pred_plane, blocks, want_coef=False):
        """residual = org(x,y) - pred(x+start_x, y+start_y) formed on the device, then transformNxN"""
        blocks = np.ascontiguousarray(blocks, dtype=L.BLOCK_DT)
        n = len(blocks)
        coef = np.zeros((n, par.h, par.w), dtype=np.int32) if want_coef else None
        q = np.zeros((n, par.h, par.w), dtype=np.int16)
        s = np.zeros(n, dtype=np.int32); lp = np.zeros(n, dtype=np.int32); nr = np.zeros(n, dtype=np.uint8)
        self._chk(self.lib.vvb_fwd_trquant_planes(self.h, ctypes.byref(par), org_plane, pred_plane, _p(blocks), n, _p(coef), _p(q), _p(s), _p(lp), _p(nr)))
        return dict(coef=coef, q=q, abs_sum=s, last_pos=lp, need_rdoq=nr)

    def frac_cost_grid(self, dfunc, org_plane, ref_plane, blocks, w, h, reduce_tap=2, alt_hpel=False):
        """distortion of the filtered block at every quarter-pel offset (-3..3)^2 around each block's integer vector (start_x, start_y):
        uint32 [n][7 (dy)][7 (dx)] -- the positions of InterSearch::xPatternRefinement"""
        blocks = np.ascontiguousarray(blocks, dtype=L.BLOCK_DT)
        out = np.zeros((len(blocks), 7, 7), dtype=np.uint32)
        self._chk(self.lib.vvb_frac_cost_grid(self.h, dfunc, org_plane, ref_plane, _p(blocks), len(blocks), w, h, int(reduce_tap), int(alt_hpel), _p(out)))
        return out

    @staticmethod
    def frac_par(lambda_, dfunc, reduce_tap=2, alt_hpel=False, fast_sub_pel=1):
        return L.vvb_frac_par(float(lambda_), dfunc, reduce_tap, int(alt_hpel), fast_sub_pel)

    def frac_search(self, org_plane, ref_plane, pus, int_mv, w, h, par):
        """InterSearch::xPatternSearchFracDIF for every PU of one shape.  pus: TZ_PU_DT array (x, y, pred_hor, pred_ver used); int_mv: TZ_BEST_DT array
        (mv_hor, mv_ver used), e.g. what tz_search returned.  Returns a FRAC_BEST_DT array (rcMvHalf, rcMvQter, ruiCost)."""
        pus = np.ascontiguousarray(pus, dtype=L.TZ_PU_DT)
        int_mv = np.ascontiguousarray(int_mv, dtype=L.TZ_BEST_DT)
        assert len(pus) == len(int_mv)
        out = np.zeros(len(pus), dtype=L.FRAC_BEST_DT)
        self._chk(self.lib.vvb_frac_search(self.h, org_plane, ref_plane, _p(pus), _p(int_mv), len(pus), w, h, ctypes.byref(par), _p(out)))
        return out

    @staticmethod
    def bi_par(lambda_, search_range, pic_w, pic_h, ctu_size, dfunc, ref_list=0, clip=False, imv=0, fast_sub_pel=1, reduce_tap=2, sub_shift_mode=1, ifp_lines=0):
        return L.vvb_bi_par(float(lambda_), search_range, sub_shift_mode, pic_w, pic_h, ctu_size, ifp_lines, ref_list, int(clip), imv, fast_sub_pel, dfunc, reduce_tap)

    def bipred_search(self, org_plane, ref_plane, pus, w, h, par, pred, cands=None):
        """The bi-predictive branch of InterSearch::xMotionEstimation for every PU of one shape.  pus: BI_PU_DT array; pred: int16 [n][h][w], the other list's
        prediction per PU; cands: int32 [n_cands][2] (hor, ver, 1/16 pel) the PUs' cand_first / cand_count index into.  Returns a BI_BEST_DT array (each stage's
        result: integer vector and uiBestSad, rcMvHalf / rcMvQter and the fractional ruiCost, the final rcMv, ruiBits and ruiCost)."""
        pus = np.ascontiguousarray(pus, dtype=L.BI_PU_DT)
        pred = np.ascontiguousarray(pred, dtype=np.int16)
        assert pred.shape == (len(pus), h, w)
        cands = np.zeros((0, 2), dtype=np.int32) if cands is None else np.ascontiguousarray(cands, dtype=np.int32).reshape(-1, 2)
        out = np.zeros(len(pus), dtype=L.BI_BEST_DT)
        self._chk(self.lib.vvb_bipred_search(self.h, org_plane, ref_plane, _p(pus), len(pus), w, h, ctypes.byref(par),
                                             _p(cands) if len(cands) else None, len(cands), _p(pred), _p(out)))
        return out

    @staticmethod
    def amvr_par(lambda_, dfunc, imv, mvp_bits, pic_w, pic_h, ctu_size, ifp_lines=0):
        """settings of amvr_refine: imv 1 (IMV_FPEL) or 2 (IMV_4PEL); mvp_bits = (m_auiMVPIdxCost[0][2], m_auiMVPIdxCost[1][2])"""
        return L.vvb_amvr_par(float(lambda_), dfunc, imv, (ctypes.c_uint32 * 2)(*[int(b) & 0xffffffff for b in mvp_bits]), pic_w, pic_h, ctu_size, ifp_lines)

    def amvr_refine(self, org_plane, ref_plane, pus, int_mv, amvp, bits, w, h, par):
        """InterSearch::xPatternSearchIntRefine (uni-prediction, fWeight 1.0) for every PU of one shape.  pus: TZ_PU_DT (x, y, pred_hor, pred_ver used);
        int_mv: TZ_BEST_DT (mv_hor, mv_ver used), e.g. what tz_search returned with imv_shift 2 or 4; amvp: AMVP_DT; bits: uint32 ruiBits per PU.
        Returns an AMVR_BEST_DT array (final rcMv in 1/16 pel, riMVPIdx, ruiBits, uiBestDist, ruiCost)."""
        pus = np.ascontiguousarray(pus, dtype=L.TZ_PU_DT)
        int_mv = np.ascontiguousarray(int_mv, dtype=L.TZ_BEST_DT)
        amvp = np.ascontiguousarray(amvp, dtype=L.AMVP_DT)
        bits = np.ascontiguousarray(bits, dtype=np.uint32)
        assert len(pus) == len(int_mv) == len(amvp) == len(bits)
        out = np.zeros(len(pus), dtype=L.AMVR_BEST_DT)
        self._chk(self.lib.vvb_amvr_refine(self.h, org_plane, ref_plane, _p(pus), _p(int_mv), _p(amvp), _p(bits), len(pus), w, h, ctypes.byref(par), _p(out)))
        return out

    def bipred_amvr_search(self, org_plane, ref_plane, pus, amvp, w, h, par, mvp_bits, pred, cands=None):
        """The bi-predictive branch of InterSearch::xMotionEstimation for cu.imv 1 and 2 (par.imv) for every PU of one shape: the integer stage of
        bipred_search, then xPatternSearchIntRefine on the target with the BCW weight.  pus: BI_PU_DT; amvp: AMVP_DT; mvp_bits as amvr_par's; pred: int16
        [n][h][w].  Returns (TZ_BEST_DT integer stage, AMVR_BEST_DT result)."""
        pus = np.ascontiguousarray(pus, dtype=L.BI_PU_DT)
        amvp = np.ascontiguousarray(amvp, dtype=L.AMVP_DT)
        pred = np.ascontiguousarray(pred, dtype=np.int16)
        assert pred.shape == (len(pus), h, w) and len(amvp) == len(pus)
        cands = np.zeros((0, 2), dtype=np.int32) if cands is None else np.ascontiguousarray(cands, dtype=np.int32).reshape(-1, 2)
        mb = np.array([int(b) & 0xffffffff for b in mvp_bits], dtype=np.uint32)
        int_out = np.zeros(len(pus), dtype=L.TZ_BEST_DT)
        out = np.zeros(len(pus), dtype=L.AMVR_BEST_DT)
        self._chk(self.lib.vvb_bipred_amvr_search(self.h, org_plane, ref_plane, _p(pus), _p(amvp), len(pus), w, h, ctypes.byref(par), _p(mb),
                                                  _p(cands) if len(cands) else None, len(cands), _p(pred), _p(int_out), _p(out)))
        return int_out, out

    # ---- dependent quantisation
    def set_depquant_engine(self, engine):
        self._chk(self.lib.vvb_set_depquant_engine(self.h, int(engine)))

    @staticmethod
    def dq_rates(flat):
        """vvb_dq_rates from 266 int32 in declaration order (last_bits_x[32], last_bits_y[32], sig_sbb_bits[2][2], sig_bits[3][12][2], gtx_bits[21][6])"""
        flat = np.ascontiguousarray(flat, dtype=np.int32)
        assert flat.size == 266
        r = L.vvb_dq_rates()
        ctypes.memmove(ctypes.byref(r), flat.ctypes.data, 266 * 4)
        return r

    def dep_quant(self, par, rates, coef, lam, dq_thr_val=8, zero_out=False, scalar_members=False, need_rdoq=None):
        """DepQuant::quant for n TUs of one shape: coef int32 [n][h][w] (as fwd_trquant returns them) -> dict(q, abs_sum, last_pos).
        rates: vvb_dq_rates (RateEstimator tables of the caller's CABAC state), lam: Quant::m_dLambda."""
        coef = np.ascontiguousarray(coef, dtype=np.int32)
        n = coef.shape[0]
        q = np.zeros((n, par.h, par.w), dtype=np.int16)
        s = np.zeros(n, dtype=np.int32); lp = np.zeros(n, dtype=np.int32)
        dq = L.vvb_dq_par(float(lam), int(dq_thr_val), int(zero_out), int(scalar_members), 0)
        nr = None if need_rdoq is None else np.ascontiguousarray(need_rdoq, dtype=np.uint8)
        self._chk(self.lib.vvb_dep_quant(self.h, ctypes.byref(par), ctypes.byref(dq), ctypes.byref(rates), _p(coef), _p(nr), n, _p(q), _p(s), _p(lp)))
        return dict(q=q, abs_sum=s, last_pos=lp)

    def set_rdoq_engine(self, engine):
        """1 (default): templates gathered per position; 2: accumulated templates + cost tables (same results)"""
        self._chk(self.lib.vvb_set_rdoq_engine(self.h, int(engine)))

    @staticmethod
    def rdoq_rates(flat):
        """vvb_rdoq_rates from 190 int32 in declaration order (sig_bits[12][2], par_bits[21][2], gt1_bits[21][2], gt2_bits[21][2], sig_group_bits[2][2],
        last_bits_x[16], last_bits_y[16], cbf_bits[2], pad[2])"""
        flat = np.ascontiguousarray(flat, dtype=np.int32)
        assert flat.size == 190
        r = L.vvb_rdoq_rates()
        ctypes.memmove(ctypes.byref(r), flat.ctypes.data, 190 * 4)
        return r

    def rdoq(self, par, rates, coef, lam, thr_val=8, sbt_zero_out=False, need_rdoq=None):
        """QuantRDOQ2::quant (m_RDOQ == 2) for n TUs of one shape: coef int32 [n][h][w] (as fwd_trquant returns them) -> dict(q, abs_sum, last_pos).
        rates: vvb_rdoq_rates (fractional bits of the caller's CABAC contexts), lam: Quant::m_dLambda; par.sign_hiding / par.lfnst_idx / par.is_chroma apply."""
        coef = np.ascontiguousarray(coef, dtype=np.int32)
        n = coef.shape[0]
        q = np.zeros((n, par.h, par.w), dtype=np.int16)
        s = np.zeros(n, dtype=np.int32); lp = np.zeros(n, dtype=np.int32)
        rq = L.vvb_rdoq_par(float(lam), int(thr_val), int(sbt_zero_out))
        nr = None if need_rdoq is None else np.ascontiguousarray(need_rdoq, dtype=np.uint8)
        self._chk(self.lib.vvb_rdoq(self.h, ctypes.byref(par), ctypes.byref(rq), ctypes.byref(rates), _p(coef), _p(nr), n, _p(q), _p(s), _p(lp)))
        return dict(q=q, abs_sum=s, last_pos=lp)

    @staticmethod
    def rdoq_ts_rates(flat):
        """vvb_rdoq_ts_rates from 44 int32 in declaration order (sig_bits[3][2], par_bits[2], gtx_bits[5][2], lrg1_bits[4][2], sign_bits[6][2], sig_group_bits[3][2])"""
        flat = np.ascontiguousarray(flat, dtype=np.int32)
        assert flat.size == 44
        r = L.vvb_rdoq_ts_rates()
        ctypes.memmove(ctypes.byref(r), flat.ctypes.data, 44 * 4)
        return r

    def rdoq_ts(self, par, rates, coef, lam, need_rdoq=None):
        """QuantRDOQ::rateDistOptQuantTS for n transform-skipped TUs of one shape: coef int32 [n][h][w] (the residual as xTransformSkip copies it) -> dict(q, abs_sum)"""
        coef = np.ascontiguousarray(coef, dtype=np.int32)
        n = coef.shape[0]
        q = np.zeros((n, par.h, par.w), dtype=np.int16)
        s = np.zeros(n, dtype=np.int32)
        nr = None if need_rdoq is None else np.ascontiguousarray(need_rdoq, dtype=np.uint8)
        self._chk(self.lib.vvb_rdoq_ts(self.h, ctypes.byref(par), float(lam), ctypes.byref(rates), _p(coef), _p(nr), n, _p(q), _p(s)))
        return dict(q=q, abs_sum=s)

    def rdoq_bdpcm(self, par, rates, coef, lam, dir_mode, need_rdoq=None):
        """QuantRDOQ::forwardRDPCM for n BDPCM TUs of one shape (dir_mode 1 horizontal, 2 vertical): coef int32 [n][h][w] (the residual) -> dict(q, abs_sum)"""
        coef = np.ascontiguousarray(coef, dtype=np.int32)
        n = coef.shape[0]
        q = np.zeros((n, par.h, par.w), dtype=np.int16)
        s = np.zeros(n, dtype=np.int32)
        nr = None if need_rdoq is None else np.ascontiguousarray(need_rdoq, dtype=np.uint8)
        self._chk(self.lib.vvb_rdoq_bdpcm(self.h, ctypes.byref(par), float(lam), int(dir_mode), ctypes.byref(rates), _p(coef), _p(nr), n, _p(q), _p(s)))
        return dict(q=q, abs_sum=s)

    # ---- inverse path / fused TU round trip
    def inv_trquant(self, par, q):
        """TrQuant::invTransformNxN for n compact level blocks q [n][h][w] -> residual int16 [n][h][w]"""
        q = np.ascontiguousarray(q, dtype=np.int16)
        n = q.shape[0]
        resi = np.zeros((n, par.h, par.w), dtype=np.int16)
        self._chk(self.lib.vvb_inv_trquant(self.h, ctypes.byref(par), _p(q), n, _p(resi)))
        return resi

    def tu_roundtrip(self, par, org, pred, want_reco=True):
        """org, pred: int16 [n][h][w] compact.  residual -> transformNxN -> invTransformNxN -> reconstruct -> SSE in one kernel.
        Returns dict(q, reco, res (TU_RESULT_DT: dist_reco, dist_resi, dist_zero, abs_sum, last_pos), need_rdoq)."""
        org = np.ascontiguousarray(org, dtype=np.int16); pred = np.ascontiguousarray(pred, dtype=np.int16)
        n = org.shape[0]
        q = np.zeros((n, par.h, par.w), dtype=np.int16)
        reco = np.zeros((n, par.h, par.w), dtype=np.int16) if want_reco else None
        res = np.zeros(n, dtype=L.TU_RESULT_DT); nr = np.zeros(n, dtype=np.uint8)
        self._chk(self.lib.vvb_tu_roundtrip(self.h, ctypes.byref(par), _p(org), _p(pred), n, _p(q), _p(reco), _p(res), _p(nr)))
        return dict(q=q, reco=reco, res=res, need_rdoq=nr)

    def tu_roundtrip_planes(self, par, org_plane, pred_plane, blocks, want_reco=True):
        """same round trip with org / pred taken from resident planes (blocks: BLOCK_DT, prediction displaced by start_x/start_y).
        Device-resident entry point wrapped with torch buffers."""
        import torch
        blocks = np.ascontiguousarray(blocks, dtype=L.BLOCK_DT)
        n = len(blocks); area = par.w * par.h
        d_blk = torch.from_numpy(np.frombuffer(blocks.tobytes(), dtype=np.uint8).copy()).cuda()
        d_q = torch.empty(n * area, dtype=torch.int16, device='cuda')
        d_reco = torch.empty(n * area, dtype=torch.int16, device='cuda') if want_reco else None
        d_res = torch.empty(n * 32, dtype=torch.uint8, device='cuda'); d_nr = torch.empty(n, dtype=torch.uint8, device='cuda')
        torch.cuda.synchronize()
        self._chk(self.lib.vvb_tu_roundtrip_planes_dev(self.h, ctypes.byref(par), org_plane, pred_plane, d_blk.data_ptr(), n, d_q.data_ptr(),
                                                       d_reco.data_ptr() if want_reco else None, d_res.data_ptr(), d_nr.data_ptr()))
        self.synchronize()
        return dict(q=d_q.cpu().numpy().reshape(n, par.h, par.w), reco=d_reco.cpu().numpy().reshape(n, par.h, par.w) if want_reco else None,
                    res=np.frombuffer(d_res.cpu().numpy().tobytes(), dtype=L.TU_RESULT_DT).copy(), need_rdoq=d_nr.cpu().numpy())

    def _tu_quant(self, quantiser, rates, lam, thr_val, sbt_zero_out, dq_thr_val, zero_out, scalar_members, selective):
        """vvb_tu_quant of quantiser 1 (fast RDOQ: rates as rdoq_rates takes them) or 2 (dependent quantisation: rates as dq_rates takes them), and the
        structures it points to (kept alive by the caller while the call runs)"""
        tq = L.vvb_tu_quant(int(quantiser), int(selective))
        keep = []
        if quantiser == 1:
            r = rates if isinstance(rates, L.vvb_rdoq_rates) else self.rdoq_rates(rates)
            rq = L.vvb_rdoq_par(float(lam), int(thr_val), int(sbt_zero_out))
            tq.rq = ctypes.pointer(rq); tq.rq_rates = ctypes.pointer(r); keep += [r, rq]
        elif quantiser == 2:
            r = rates if isinstance(rates, L.vvb_dq_rates) else self.dq_rates(rates)
            dq = L.vvb_dq_par(float(lam), int(dq_thr_val), int(zero_out), int(scalar_members), 0)
            tq.dq = ctypes.pointer(dq); tq.dq_rates = ctypes.pointer(r); keep += [r, dq]
        return tq, keep

    def tu_roundtrip_rdo(self, par, org, pred, quantiser, rates, lam, *, thr_val=8, sbt_zero_out=False, dq_thr_val=8, zero_out=False, scalar_members=False,
                         selective=True, want_reco=True):
        """org, pred: int16 [n][h][w] compact.  residual -> transform -> fast RDOQ (quantiser 1) or dependent quantisation (quantiser 2) -> the matching
        dequantiser and inverse when abs_sum > 0 -> reconstruct -> SSE, in one call.  par.dep_quant must be set exactly for quantiser 2.
        Returns dict(q, reco, res (TU_RESULT_DT), need_rdoq) as tu_roundtrip does."""
        org = np.ascontiguousarray(org, dtype=np.int16); pred = np.ascontiguousarray(pred, dtype=np.int16)
        n = org.shape[0]
        tq, keep = self._tu_quant(quantiser, rates, lam, thr_val, sbt_zero_out, dq_thr_val, zero_out, scalar_members, selective)
        q = np.zeros((n, par.h, par.w), dtype=np.int16)
        reco = np.zeros((n, par.h, par.w), dtype=np.int16) if want_reco else None
        res = np.zeros(n, dtype=L.TU_RESULT_DT); nr = np.zeros(n, dtype=np.uint8)
        self._chk(self.lib.vvb_tu_roundtrip_rdo(self.h, ctypes.byref(par), ctypes.byref(tq), _p(org), _p(pred), n, _p(q), _p(reco), _p(res), _p(nr)))
        return dict(q=q, reco=reco, res=res, need_rdoq=nr)

    def tu_roundtrip_rdo_planes(self, par, org_plane, pred_plane, blocks, quantiser, rates, lam, *, thr_val=8, sbt_zero_out=False, dq_thr_val=8, zero_out=False,
                                scalar_members=False, selective=True, want_reco=True):
        """tu_roundtrip_rdo with org / pred taken from resident planes (blocks: BLOCK_DT, prediction displaced by start_x/start_y).
        Device-resident entry point wrapped with torch buffers."""
        import torch
        blocks = np.ascontiguousarray(blocks, dtype=L.BLOCK_DT)
        n = len(blocks); area = par.w * par.h
        tq, keep = self._tu_quant(quantiser, rates, lam, thr_val, sbt_zero_out, dq_thr_val, zero_out, scalar_members, selective)
        d_blk = torch.from_numpy(np.frombuffer(blocks.tobytes(), dtype=np.uint8).copy()).cuda()
        d_q = torch.empty(max(1, n * area), dtype=torch.int16, device='cuda')
        d_reco = torch.empty(max(1, n * area), dtype=torch.int16, device='cuda') if want_reco else None
        d_res = torch.empty(max(1, n * 32), dtype=torch.uint8, device='cuda'); d_nr = torch.empty(max(1, n), dtype=torch.uint8, device='cuda')
        torch.cuda.synchronize()
        self._chk(self.lib.vvb_tu_roundtrip_rdo_planes_dev(self.h, ctypes.byref(par), ctypes.byref(tq), org_plane, pred_plane, d_blk.data_ptr(), n, d_q.data_ptr(),
                                                           d_reco.data_ptr() if want_reco else None, d_res.data_ptr(), d_nr.data_ptr()))
        self.synchronize()
        return dict(q=d_q.cpu().numpy()[:n * area].reshape(n, par.h, par.w), reco=d_reco.cpu().numpy()[:n * area].reshape(n, par.h, par.w) if want_reco else None,
                    res=np.frombuffer(d_res.cpu().numpy().tobytes(), dtype=L.TU_RESULT_DT)[:n].copy(), need_rdoq=d_nr.cpu().numpy()[:n])

    # ---- MCTF
    def mctf_error_batch(self, org_plane, ref_plane, cands, low_res_filter=False):
        cands = np.ascontiguousarray(cands, dtype=L.MCTF_DT)
        out = np.zeros(len(cands), dtype=np.int32)
        self._chk(self.lib.vvb_mctf_error_batch(self.h, org_plane, ref_plane, _p(cands), len(cands), int(low_res_filter), _p(out)))
        return out

    def mctf_search_grid(self, org_plane, ref_plane, blocks, step, radius, low_res_filter=False):
        """blocks: MCTF_DT (x, y, centre mvx/mvy in 1/16 pel, w, h) -> errors int32 [n][2r+1 (dy)][2r+1 (dx)] of centre + (i-r, j-r)*step"""
        blocks = np.ascontiguousarray(blocks, dtype=L.MCTF_DT)
        k1 = 2 * radius + 1
        out = np.zeros((len(blocks), k1, k1), dtype=np.int32)
        self._chk(self.lib.vvb_mctf_search_grid(self.h, org_plane, ref_plane, _p(blocks), len(blocks), step, radius, int(low_res_filter), _p(out)))
        return out

    def mctf_apply(self, org_plane, ref_planes, mvs, block_size, ref_strengths, weight_scaling, sigma_sq, width, height, planar=True, low_res_filter=False):
        """xFinalizeBlkLine for the luma plane: mvs MCTF_MV_DT [num_refs][blocks]; returns the filtered picture int16 [height][width]"""
        par = L.vvb_mctf_apply_par()
        par.num_refs = len(ref_planes); par.block_size = block_size; par.low_res_filter = int(low_res_filter); par.planar_correction = int(planar)
        par.weight_scaling = weight_scaling; par.sigma_sq = sigma_sq
        for i, (pl, st) in enumerate(zip(ref_planes, ref_strengths)):
            par.ref_plane[i] = pl; par.ref_strength[i] = st
        mvs = np.ascontiguousarray(mvs, dtype=L.MCTF_MV_DT)
        out = np.zeros((height, width), dtype=np.int16)
        self._chk(self.lib.vvb_mctf_apply(self.h, org_plane, ctypes.byref(par), _p(mvs), _p(out), width))
        return out

    def mctf_calc_var(self, plane, blocks):
        blocks = np.ascontiguousarray(blocks, dtype=L.MCTF_DT)
        out = np.zeros(len(blocks), dtype=np.float64)
        self._chk(self.lib.vvb_mctf_calc_var(self.h, plane, _p(blocks), len(blocks), _p(out)))
        return out

    # ---- affine
    def mctf_estimate_level(self, org_plane, ref_plane, width, height, block_size, prev=None, factor=2, double_res=False, search_pattern=0, low_res_filter=False, out_shape=None):
        """MCTF::motionEstimationLuma for the whole picture with the control on the device.  prev: None or a MCTF_MV_DT array [prevH][prevW] (field of the coarser
        level).  Returns a MCTF_MV_DT array [out_h][out_w] (default: one entry per block)."""
        bxn, byn = (width - 8) // block_size + 1, (height - 8) // block_size + 1
        oh, ow = out_shape if out_shape is not None else (byn, bxn)
        out = np.zeros((oh, ow), dtype=L.MCTF_MV_DT)
        if prev is not None:
            prev = np.ascontiguousarray(prev, dtype=L.MCTF_MV_DT)
        par = L.vvb_mctf_level_par(block_size, factor, int(double_res), search_pattern, int(low_res_filter), 0 if prev is None else prev.shape[1], 0 if prev is None else prev.shape[0], ow, oh)
        self._chk(self.lib.vvb_mctf_estimate_level(self.h, org_plane, ref_plane, ctypes.byref(par), _p(prev), _p(out)))
        return out

    def mctf_estimate_pyramid(self, org_plane, ref_plane, width, height, unit_size=16, add_level=False, search_pattern=0, low_res_filter=False):
        """MCTF::motionEstimationMCTF for one neighbour picture, everything on the device (subsampling, 4 / 5 chained levels).  Planes: margin >= 128.
        Returns a MCTF_MV_DT array [ceil(H / unit)][ceil(W / unit)] -- the input of mctf_apply."""
        out = np.zeros(((height + unit_size - 1) // unit_size, (width + unit_size - 1) // unit_size), dtype=L.MCTF_MV_DT)
        par = L.vvb_mctf_pyr_par(unit_size, int(add_level), search_pattern, int(low_res_filter))
        self._chk(self.lib.vvb_mctf_estimate_pyramid(self.h, org_plane, ref_plane, ctypes.byref(par), _p(out)))
        return out

    def affine_sobel(self, vertical, pred, pred_stride, deriv_stride, w, h):
        d = np.zeros((h, deriv_stride), dtype=np.int16)
        self._chk(self.lib.vvb_affine_sobel(self.h, int(vertical), _p(pred), pred_stride, _p(d), deriv_stride, w, h))
        return d

    def affine_equal_coeff(self, six_param, resi, resi_stride, gx, gy, deriv_stride, w, h, eq=None):
        if eq is None:
            eq = np.zeros(49, dtype=np.int64)
        self._chk(self.lib.vvb_affine_equal_coeff(self.h, int(six_param), _p(resi), resi_stride, _p(gx), _p(gy), deriv_stride, w, h, _p(eq)))
        return eq
