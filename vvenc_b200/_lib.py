"""ctypes binding of the C-ABI shared library (include/vvenc_b200.h).  Fails loudly when the library is missing:
there is no Python or CPU fallback for any entry point."""
import ctypes, os

HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get('VVENC_B200_LIB') or os.path.join(HERE, 'csrc', 'libvvenc_b200.so')   # override: A/B builds of the same ABI

VVB_OK, VVB_ERR_ARG, VVB_ERR_UNSUPPORTED, VVB_ERR_CUDA, VVB_ERR_NOMEM = 0, -1, -2, -3, -4

c_p = ctypes.c_void_p
c_i = ctypes.c_int


class vvb_cand(ctypes.Structure):
    _fields_ = [('org_plane', ctypes.c_int32), ('org_x', ctypes.c_int32), ('org_y', ctypes.c_int32),
                ('cur_plane', ctypes.c_int32), ('cur_x', ctypes.c_int32), ('cur_y', ctypes.c_int32),
                ('w', ctypes.c_uint16), ('h', ctypes.c_uint16), ('dfunc', ctypes.c_uint8), ('sub_shift', ctypes.c_uint8), ('pad', ctypes.c_uint8 * 2)]


class vvb_mctf_apply_par(ctypes.Structure):
    _fields_ = [('num_refs', ctypes.c_int32), ('block_size', ctypes.c_int32), ('low_res_filter', ctypes.c_int32), ('planar_correction', ctypes.c_int32),
                ('weight_scaling', ctypes.c_double), ('sigma_sq', ctypes.c_double), ('ref_strength', ctypes.c_double * 8), ('ref_plane', ctypes.c_int32 * 8)]


class vvb_me_par(ctypes.Structure):
    _fields_ = [('lam', ctypes.c_double), ('cost_scale', ctypes.c_int32), ('imv_shift', ctypes.c_int32), ('sub_shift', ctypes.c_int32), ('quad_order', ctypes.c_int32), ('pattern_radius', ctypes.c_int32), ('pad', ctypes.c_int32)]


class vvb_tz_par(ctypes.Structure):
    _fields_ = [(k, ctypes.c_int32) for k in ('search_range', 'extended', 'fast', 'integer_et', 'first_search_stop', 'sub_shift_mode', 'pic_w', 'pic_h', 'ctu_size', 'ifp_lines')]


class vvb_frac_par(ctypes.Structure):
    _fields_ = [('lam', ctypes.c_double), ('dfunc', ctypes.c_int32), ('reduce_tap', ctypes.c_int32), ('alt_hpel', ctypes.c_int32), ('fast_sub_pel', ctypes.c_int32)]


FRAC_PAR = vvb_frac_par


class vvb_bi_par(ctypes.Structure):
    _fields_ = [('lam', ctypes.c_double)] + [(k, ctypes.c_int32) for k in ('search_range', 'sub_shift_mode', 'pic_w', 'pic_h', 'ctu_size', 'ifp_lines', 'ref_list',
                                                                          'clip', 'imv', 'fast_sub_pel', 'dfunc', 'reduce_tap')]


class vvb_amvr_par(ctypes.Structure):
    _fields_ = [('lam', ctypes.c_double), ('dfunc', ctypes.c_int32), ('imv', ctypes.c_int32), ('mvp_bits', ctypes.c_uint32 * 2)] + \
               [(k, ctypes.c_int32) for k in ('pic_w', 'pic_h', 'ctu_size', 'ifp_lines')]


AMVR_PAR = vvb_amvr_par


class vvb_tu_par(ctypes.Structure):
    _fields_ = [('w', ctypes.c_int32), ('h', ctypes.c_int32), ('tr_hor', ctypes.c_int32), ('tr_ver', ctypes.c_int32), ('bit_depth', ctypes.c_int32),
                ('qp', ctypes.c_int32), ('is_irap', ctypes.c_int32), ('dep_quant', ctypes.c_int32), ('sign_hiding', ctypes.c_int32), ('lfnst_idx', ctypes.c_int32), ('lfnst_set', ctypes.c_int32), ('lfnst_transpose', ctypes.c_int32),
                ('transform_skip', ctypes.c_int32), ('input_bit_depth_delta', ctypes.c_int32), ('is_chroma', ctypes.c_int32)]


class vvb_mctf_level_par(ctypes.Structure):
    _fields_ = [(k, ctypes.c_int32) for k in ('block_size', 'factor', 'double_res', 'search_pattern', 'low_res_filter', 'prev_w', 'prev_h', 'out_w', 'out_h')]


class vvb_mctf_pyr_par(ctypes.Structure):
    _fields_ = [(k, ctypes.c_int32) for k in ('unit_size', 'add_level', 'search_pattern', 'low_res_filter')]


class vvb_dq_rates(ctypes.Structure):
    _fields_ = [('last_bits_x', ctypes.c_int32 * 32), ('last_bits_y', ctypes.c_int32 * 32), ('sig_sbb_bits', ctypes.c_int32 * 4), ('sig_bits', ctypes.c_int32 * 72),
                ('gtx_bits', ctypes.c_int32 * 126)]


class vvb_dq_par(ctypes.Structure):
    _fields_ = [('lam', ctypes.c_double), ('dq_thr_val', ctypes.c_int32), ('zero_out', ctypes.c_int32), ('scalar_members', ctypes.c_int32), ('pad', ctypes.c_int32)]


class vvb_rdoq_rates(ctypes.Structure):
    _fields_ = [('sig_bits', ctypes.c_int32 * 24), ('par_bits', ctypes.c_int32 * 42), ('gt1_bits', ctypes.c_int32 * 42), ('gt2_bits', ctypes.c_int32 * 42), ('sig_group_bits', ctypes.c_int32 * 4),
                ('last_bits_x', ctypes.c_int32 * 16), ('last_bits_y', ctypes.c_int32 * 16), ('cbf_bits', ctypes.c_int32 * 2), ('pad', ctypes.c_int32 * 2)]


class vvb_rdoq_ts_rates(ctypes.Structure):
    _fields_ = [('sig_bits', ctypes.c_int32 * 6), ('par_bits', ctypes.c_int32 * 2), ('gtx_bits', ctypes.c_int32 * 10), ('lrg1_bits', ctypes.c_int32 * 8), ('sign_bits', ctypes.c_int32 * 12),
                ('sig_group_bits', ctypes.c_int32 * 6)]


class vvb_rdoq_par(ctypes.Structure):
    _fields_ = [('lam', ctypes.c_double), ('thr_val', ctypes.c_int32), ('sbt_zero_out', ctypes.c_int32), ('pad', ctypes.c_int32 * 2)]


class vvb_tu_quant(ctypes.Structure):
    _fields_ = [('quantiser', ctypes.c_int32), ('selective', ctypes.c_int32), ('rq', ctypes.POINTER(vvb_rdoq_par)), ('rq_rates', ctypes.POINTER(vvb_rdoq_rates)),
                ('dq', ctypes.POINTER(vvb_dq_par)), ('dq_rates', ctypes.POINTER(vvb_dq_rates))]


class vvb_level_io(ctypes.Structure):
    _fields_ = [('blocks', ctypes.c_void_p), ('count', ctypes.c_int32), ('best', ctypes.c_void_p), ('refine_cost', ctypes.c_void_p), ('q', ctypes.c_void_p),
                ('abs_sum', ctypes.c_void_p), ('last_pos', ctypes.c_void_p), ('need_rdoq', ctypes.c_void_p), ('tu', vvb_tu_par), ('packed_q', ctypes.c_void_p), ('packed_offsets', ctypes.c_void_p)]


# numpy dtypes mirroring the packed C structs
import numpy as np
MASK_CAND_DT = np.dtype([('org_plane', '<i4'), ('org_x', '<i4'), ('org_y', '<i4'), ('cur_plane', '<i4'), ('cur_x', '<i4'), ('cur_y', '<i4'),
                         ('w', '<u2'), ('h', '<u2'), ('dfunc', 'u1'), ('sub_shift', 'u1'), ('pad', 'u1', (2,)),
                         ('mask_offset', '<i4'), ('mask_stride', '<i4'), ('mask_stride2', '<i4'), ('step_x', '<i4')])
CAND_DT = np.dtype([('org_plane', '<i4'), ('org_x', '<i4'), ('org_y', '<i4'), ('cur_plane', '<i4'), ('cur_x', '<i4'), ('cur_y', '<i4'),
                    ('w', '<u2'), ('h', '<u2'), ('dfunc', 'u1'), ('sub_shift', 'u1'), ('pad', 'u1', (2,))])
POS_DT = np.dtype([('x', '<i4'), ('y', '<i4')])
BLOCK_DT = np.dtype([('x', '<i4'), ('y', '<i4'), ('left', '<i2'), ('right', '<i2'), ('top', '<i2'), ('bottom', '<i2'),
                     ('pred_hor', '<i2'), ('pred_ver', '<i2'), ('start_x', '<i2'), ('start_y', '<i2')])
BEST_DT = np.dtype([('dx', '<i2'), ('dy', '<i2'), ('sad', '<u4'), ('cost', '<u8')])
MV_DT = np.dtype([('dx', '<i2'), ('dy', '<i2')])
TU_RESULT_DT = np.dtype([('dist_reco', '<u8'), ('dist_resi', '<u8'), ('dist_zero', '<u8'), ('abs_sum', '<i4'), ('last_pos', '<i4')])
MCTF_MV_DT = np.dtype([('x', '<i4'), ('y', '<i4'), ('error', '<i4'), ('rmsme', '<u2'), ('pad', '<u2')])
MCTF_DT = np.dtype([('x', '<i4'), ('y', '<i4'), ('mvx', '<i4'), ('mvy', '<i4'), ('w', '<u2'), ('h', '<u2')])
TZ_PU_DT = np.dtype([('x', '<i4'), ('y', '<i4'), ('start_hor', '<i4'), ('start_ver', '<i4'), ('pred_hor', '<i2'), ('pred_ver', '<i2'), ('cand_first', '<i4'), ('cand_count', '<i4')])
TZ_BEST_DT = np.dtype([('mv_hor', '<i4'), ('mv_ver', '<i4'), ('sad', '<u8'), ('cost', '<u8'), ('best_distance', '<u4'), ('pad', '<u4')])
assert TZ_PU_DT.itemsize == 28 and TZ_BEST_DT.itemsize == 32
FRAC_BEST_DT = np.dtype([('half_hor', '<i2'), ('half_ver', '<i2'), ('qter_hor', '<i2'), ('qter_ver', '<i2'), ('cost', '<u8')])
assert FRAC_BEST_DT.itemsize == 16 and ctypes.sizeof(vvb_frac_par) == 24
BI_PU_DT = np.dtype([('x', '<i4'), ('y', '<i4'), ('start_hor', '<i4'), ('start_ver', '<i4'), ('pred_hor', '<i2'), ('pred_ver', '<i2'), ('cand_first', '<i4'), ('cand_count', '<i4'),
                     ('bits', '<u4'), ('bcw_idx', '<i4')])
BI_BEST_DT = np.dtype([('int_hor', '<i4'), ('int_ver', '<i4'), ('int_best', '<u8'), ('frac_cost', '<u8'), ('half_hor', '<i2'), ('half_ver', '<i2'), ('qter_hor', '<i2'),
                       ('qter_ver', '<i2'), ('mv_hor', '<i4'), ('mv_ver', '<i4'), ('bits', '<u4'), ('pad', '<u4'), ('cost', '<u8')])
BI_PAR = vvb_bi_par
assert BI_PU_DT.itemsize == 36 and BI_BEST_DT.itemsize == 56 and ctypes.sizeof(vvb_bi_par) == 56
AMVP_DT = np.dtype([('cand_hor', '<i4', (2,)), ('cand_ver', '<i4', (2,)), ('num_cand', '<i4'), ('mvp_idx', '<i4')])
AMVR_BEST_DT = np.dtype([('mv_hor', '<i4'), ('mv_ver', '<i4'), ('mvp_idx', '<i4'), ('bits', '<u4'), ('dist', '<u8'), ('cost', '<u8')])
assert AMVP_DT.itemsize == 24 and AMVR_BEST_DT.itemsize == 32 and ctypes.sizeof(vvb_amvr_par) == 40
assert CAND_DT.itemsize == 32 and BLOCK_DT.itemsize == 24 and BEST_DT.itemsize == 16 and MCTF_DT.itemsize == 20

# every symbol include/vvenc_b200.h declares: name -> (restype, argtypes)
SYMBOLS = {
    'vvb_create': (c_i, [ctypes.POINTER(c_p), c_i]),
    'vvb_destroy': (None, [c_p]),
    'vvb_last_error': (ctypes.c_char_p, [c_p]),
    'vvb_synchronize': (c_i, [c_p]),
    'vvb_stream': (c_p, [c_p]),
    'vvb_set_async': (c_i, [c_p, c_i]),
    'vvb_launch_count': (c_i, [c_p, ctypes.POINTER(ctypes.c_uint64)]),
    'vvb_alu_probe_dev': (c_i, [c_p, c_i, c_i, c_i]),
    'vvb_plane_upload': (c_i, [c_p, c_i, c_p, c_i, c_i, c_i, c_i, c_i]),
    'vvb_plane_bind_dev': (c_i, [c_p, c_i, c_p, c_i, c_i, c_i, c_i, c_i]),
    'vvb_plane_free': (c_i, [c_p, c_i]),
    'vvb_dist_batch': (c_i, [c_p, c_p, c_i, c_p]),
    'vvb_dist_batch_dev': (c_i, [c_p, c_p, c_i, c_p]),
    'vvb_dist_block': (ctypes.c_uint64, [c_p, c_i, c_p, c_i, c_p, c_i, c_i, c_i, c_i, c_i, ctypes.POINTER(c_i)]),
    'vvb_sad_mask_block': (ctypes.c_uint64, [c_p, c_p, c_i, c_p, c_i, c_i, c_i, c_p, c_i, c_i, c_i, c_i, ctypes.POINTER(c_i)]),
    'vvb_sad_x5_block': (c_i, [c_p, c_p, c_i, c_p, c_i, c_i, c_i, c_i, c_i, c_p]),
    'vvb_fix_wsse_block': (ctypes.c_uint64, [c_p, c_p, c_i, c_p, c_i, c_i, c_i, ctypes.c_uint32, ctypes.POINTER(c_i)]),
    'vvb_dist_pool': (c_i, [c_p, c_i, c_i, c_p, c_i, c_i, c_i, c_i, c_p, c_i, c_p]),
    'vvb_dist_pool_dev': (c_i, [c_p, c_i, c_i, c_p, c_i, c_i, c_i, c_i, c_p, c_i, c_p]),
    'vvb_pool_hint': (c_i, [c_p, c_i]),
    'vvb_sad_search': (c_i, [c_p, c_i, c_i, c_p, c_i, c_i, c_i, ctypes.POINTER(vvb_me_par), c_p, c_i, c_p]),
    'vvb_sad_search_dev': (c_i, [c_p, c_i, c_i, c_p, c_i, c_i, c_i, ctypes.POINTER(vvb_me_par), c_i, c_i, c_p, c_i, c_p]),
    'vvb_sad_search_pyramid': (c_i, [c_p, c_i, c_i, c_i, c_p, c_p, c_i, ctypes.POINTER(vvb_me_par), c_i, c_i, c_p]),
    'vvb_sad_search_pyramid_dev': (c_i, [c_p, c_i, c_i, c_i, c_p, c_p, c_i, ctypes.POINTER(vvb_me_par), c_i, c_i, c_p]),
    'vvb_set_tma_staging': (c_i, [c_p, c_i]),
    'vvb_set_pyramid_engine': (c_i, [c_p, c_i]),
    'vvb_sad_pattern': (c_i, [c_p, c_i, c_i, c_p, c_i, c_i, c_i, c_p, c_i, ctypes.POINTER(vvb_me_par), c_p, c_p]),
    'vvb_sad_pattern_dev': (c_i, [c_p, c_i, c_i, c_p, c_i, c_i, c_i, c_p, c_i, ctypes.POINTER(vvb_me_par), c_p, c_p]),
    'vvb_cost_pattern': (c_i, [c_p, c_i, c_i, c_i, c_p, c_i, c_i, c_i, c_p, c_i, ctypes.POINTER(vvb_me_par), c_p, c_p]),
    'vvb_cost_pattern_dev': (c_i, [c_p, c_i, c_i, c_i, c_p, c_i, c_i, c_i, c_p, c_i, ctypes.POINTER(vvb_me_par), c_p, c_p]),
    'vvb_blocks_set_start_dev': (c_i, [c_p, c_p, c_p, c_i]),
    'vvb_tz_search': (c_i, [c_p, c_i, c_i, c_p, c_i, c_i, c_i, ctypes.POINTER(vvb_me_par), ctypes.POINTER(vvb_tz_par), c_p, c_i, c_p]),
    'vvb_tz_search_dev': (c_i, [c_p, c_i, c_i, c_p, c_i, c_i, c_i, ctypes.POINTER(vvb_me_par), ctypes.POINTER(vvb_tz_par), c_p, c_i, c_p]),
    'vvb_fwd_trquant': (c_i, [c_p, ctypes.POINTER(vvb_tu_par), c_p, c_i, c_p, c_p, c_p, c_p, c_p]),
    'vvb_fwd_trquant_dev': (c_i, [c_p, ctypes.POINTER(vvb_tu_par), c_p, c_i, c_p, c_p, c_p, c_p, c_p]),
    'vvb_set_tensor_transform': (c_i, [c_p, c_i]),
    'vvb_pack_levels_dev': (c_i, [c_p, ctypes.POINTER(vvb_tu_par), c_p, c_p, c_i, c_p, c_p]),
    'vvb_scan_order': (c_i, [c_i, c_i, c_p]),
    'vvb_search_refine_tu': (c_i, [c_p, c_i, c_i, c_i, c_p, c_i, ctypes.POINTER(vvb_me_par), c_i, c_i, c_i, c_p, c_i]),
    'vvb_fwd_trquant_planes': (c_i, [c_p, ctypes.POINTER(vvb_tu_par), c_i, c_i, c_p, c_i, c_p, c_p, c_p, c_p, c_p]),
    'vvb_fwd_trquant_planes_dev': (c_i, [c_p, ctypes.POINTER(vvb_tu_par), c_i, c_i, c_p, c_i, c_p, c_p, c_p, c_p, c_p]),
    'vvb_mctf_estimate_level': (c_i, [c_p, c_i, c_i, ctypes.POINTER(vvb_mctf_level_par), c_p, c_p]),
    'vvb_mctf_estimate_level_dev': (c_i, [c_p, c_i, c_i, ctypes.POINTER(vvb_mctf_level_par), c_p, c_p]),
    'vvb_mctf_estimate_pyramid': (c_i, [c_p, c_i, c_i, ctypes.POINTER(vvb_mctf_pyr_par), c_p]),
    'vvb_mctf_estimate_pyramid_dev': (c_i, [c_p, c_i, c_i, ctypes.POINTER(vvb_mctf_pyr_par), c_p]),
    'vvb_mask_upload': (c_i, [c_p, c_p, c_i]),
    'vvb_sad_mask_batch': (c_i, [c_p, c_p, c_i, c_p]),
    'vvb_sad_mask_batch_dev': (c_i, [c_p, c_p, c_i, c_p]),
    'vvb_sad_x5_batch': (c_i, [c_p, c_p, c_i, c_p]),
    'vvb_sad_x5_batch_dev': (c_i, [c_p, c_p, c_i, c_p]),
    'vvb_fix_wsse_batch': (c_i, [c_p, c_p, c_p, c_i, c_p]),
    'vvb_fix_wsse_batch_dev': (c_i, [c_p, c_p, c_p, c_i, c_p]),
    'vvb_affine_eq_batch': (c_i, [c_p, c_i, c_p, c_p, c_i, c_i, c_i, c_p, c_p, c_p]),
    'vvb_affine_eq_batch_dev': (c_i, [c_p, c_i, c_p, c_p, c_i, c_i, c_i, c_p, c_p, c_p]),
    'vvb_dep_quant': (c_i, [c_p, ctypes.POINTER(vvb_tu_par), ctypes.POINTER(vvb_dq_par), ctypes.POINTER(vvb_dq_rates), c_p, c_p, c_i, c_p, c_p, c_p]),
    'vvb_dep_quant_dev': (c_i, [c_p, ctypes.POINTER(vvb_tu_par), ctypes.POINTER(vvb_dq_par), ctypes.POINTER(vvb_dq_rates), c_p, c_p, c_i, c_p, c_p, c_p]),
    'vvb_set_depquant_engine': (c_i, [c_p, c_i]),
    'vvb_dep_quant_constants': (c_i, [ctypes.POINTER(vvb_tu_par), ctypes.POINTER(vvb_dq_par), c_p]),
    'vvb_rdoq': (c_i, [c_p, ctypes.POINTER(vvb_tu_par), ctypes.POINTER(vvb_rdoq_par), ctypes.POINTER(vvb_rdoq_rates), c_p, c_p, c_i, c_p, c_p, c_p]),
    'vvb_rdoq_dev': (c_i, [c_p, ctypes.POINTER(vvb_tu_par), ctypes.POINTER(vvb_rdoq_par), ctypes.POINTER(vvb_rdoq_rates), c_p, c_p, c_i, c_p, c_p, c_p]),
    'vvb_rdoq_ts': (c_i, [c_p, ctypes.POINTER(vvb_tu_par), ctypes.c_double, ctypes.POINTER(vvb_rdoq_ts_rates), c_p, c_p, c_i, c_p, c_p]),
    'vvb_rdoq_ts_dev': (c_i, [c_p, ctypes.POINTER(vvb_tu_par), ctypes.c_double, ctypes.POINTER(vvb_rdoq_ts_rates), c_p, c_p, c_i, c_p, c_p]),
    'vvb_rdoq_bdpcm': (c_i, [c_p, ctypes.POINTER(vvb_tu_par), ctypes.c_double, c_i, ctypes.POINTER(vvb_rdoq_ts_rates), c_p, c_p, c_i, c_p, c_p]),
    'vvb_rdoq_bdpcm_dev': (c_i, [c_p, ctypes.POINTER(vvb_tu_par), ctypes.c_double, c_i, ctypes.POINTER(vvb_rdoq_ts_rates), c_p, c_p, c_i, c_p, c_p]),
    'vvb_set_rdoq_engine': (c_i, [c_p, c_i]),
    'vvb_rdoq_constants': (c_i, [ctypes.POINTER(vvb_tu_par), ctypes.POINTER(vvb_rdoq_par), c_p]),
    'vvb_inv_trquant': (c_i, [c_p, ctypes.POINTER(vvb_tu_par), c_p, c_i, c_p]),
    'vvb_inv_trquant_dev': (c_i, [c_p, ctypes.POINTER(vvb_tu_par), c_p, c_i, c_p]),
    'vvb_tu_roundtrip': (c_i, [c_p, ctypes.POINTER(vvb_tu_par), c_p, c_p, c_i, c_p, c_p, c_p, c_p]),
    'vvb_tu_roundtrip_dev': (c_i, [c_p, ctypes.POINTER(vvb_tu_par), c_p, c_p, c_i, c_p, c_p, c_p, c_p]),
    'vvb_tu_roundtrip_planes_dev': (c_i, [c_p, ctypes.POINTER(vvb_tu_par), c_i, c_i, c_p, c_i, c_p, c_p, c_p, c_p]),
    'vvb_tu_roundtrip_rdo': (c_i, [c_p, ctypes.POINTER(vvb_tu_par), ctypes.POINTER(vvb_tu_quant), c_p, c_p, c_i, c_p, c_p, c_p, c_p]),
    'vvb_tu_roundtrip_rdo_dev': (c_i, [c_p, ctypes.POINTER(vvb_tu_par), ctypes.POINTER(vvb_tu_quant), c_p, c_p, c_i, c_p, c_p, c_p, c_p]),
    'vvb_tu_roundtrip_rdo_planes_dev': (c_i, [c_p, ctypes.POINTER(vvb_tu_par), ctypes.POINTER(vvb_tu_quant), c_i, c_i, c_p, c_i, c_p, c_p, c_p, c_p]),
    'vvb_mctf_error_batch': (c_i, [c_p, c_i, c_i, c_p, c_i, c_i, c_p]),
    'vvb_mctf_search_grid': (c_i, [c_p, c_i, c_i, c_p, c_i, c_i, c_i, c_i, c_p]),
    'vvb_mctf_search_grid_dev': (c_i, [c_p, c_i, c_i, c_p, c_i, c_i, c_i, c_i, c_p]),
    'vvb_frac_cost_grid': (c_i, [c_p, c_i, c_i, c_i, c_p, c_i, c_i, c_i, c_i, c_i, c_p]),
    'vvb_frac_cost_grid_dev': (c_i, [c_p, c_i, c_i, c_i, c_p, c_i, c_i, c_i, c_i, c_i, c_p]),
    'vvb_frac_search': (c_i, [c_p, c_i, c_i, c_p, c_p, c_i, c_i, c_i, ctypes.POINTER(vvb_frac_par), c_p]),
    'vvb_frac_search_dev': (c_i, [c_p, c_i, c_i, c_p, c_p, c_i, c_i, c_i, ctypes.POINTER(vvb_frac_par), c_p]),
    'vvb_bipred_search': (c_i, [c_p, c_i, c_i, c_p, c_i, c_i, c_i, ctypes.POINTER(vvb_bi_par), c_p, c_i, c_p, c_p]),
    'vvb_bipred_search_dev': (c_i, [c_p, c_i, c_i, c_p, c_i, c_i, c_i, ctypes.POINTER(vvb_bi_par), c_p, c_i, c_p, c_p]),
    'vvb_amvr_refine': (c_i, [c_p, c_i, c_i, c_p, c_p, c_p, c_p, c_i, c_i, c_i, ctypes.POINTER(vvb_amvr_par), c_p]),
    'vvb_amvr_refine_dev': (c_i, [c_p, c_i, c_i, c_p, c_p, c_p, c_p, c_i, c_i, c_i, ctypes.POINTER(vvb_amvr_par), c_p]),
    'vvb_bipred_amvr_search': (c_i, [c_p, c_i, c_i, c_p, c_p, c_i, c_i, c_i, ctypes.POINTER(vvb_bi_par), c_p, c_p, c_i, c_p, c_p, c_p]),
    'vvb_bipred_amvr_search_dev': (c_i, [c_p, c_i, c_i, c_p, c_p, c_i, c_i, c_i, ctypes.POINTER(vvb_bi_par), c_p, c_p, c_i, c_p, c_p, c_p]),
    'vvb_mctf_apply': (c_i, [c_p, c_i, ctypes.POINTER(vvb_mctf_apply_par), c_p, c_p, c_i]),
    'vvb_mctf_apply_dev': (c_i, [c_p, c_i, ctypes.POINTER(vvb_mctf_apply_par), c_p, c_p, c_i]),
    'vvb_mctf_calc_var': (c_i, [c_p, c_i, c_p, c_i, c_p]),
    'vvb_mctf_calc_var_dev': (c_i, [c_p, c_i, c_p, c_i, c_p]),
    'vvb_mctf_hint': (c_i, [c_p, c_i]),
    'vvb_mctf_error_batch_dev': (c_i, [c_p, c_i, c_i, c_p, c_i, c_i, c_p]),
    'vvb_affine_sobel': (c_i, [c_p, c_i, c_p, c_i, c_p, c_i, c_i, c_i]),
    'vvb_affine_equal_coeff': (c_i, [c_p, c_i, c_p, c_i, c_p, c_p, c_i, c_i, c_i, c_p]),
}

_lib = None


def load():
    """dlopen the in-tree CUDA library and bind every declared symbol; raises if it is absent (no fallback)."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise RuntimeError('vvenc_b200: %s is missing -- run `python -c "import __graft_entry__ as g; g.build()"` '
                               '(nvcc, sm_90a); there is no CPU fallback' % LIB_PATH)
        lib = ctypes.CDLL(LIB_PATH)
        for name, (res, args) in SYMBOLS.items():
            f = getattr(lib, name)          # AttributeError if the export is missing
            f.restype = res
            f.argtypes = args
        _lib = lib
    return _lib
