"""vvenc_b200 -- H100-native (sm_90a) implementation of VVenC's block-cost hot path:
SAD / SATD / SSE distortion kernels, fixed-pattern and full-search motion sweeps, forward DCT-II/DST-VII/DCT-VIII +
quantisation, MCTF block matching and the affine gradient helpers, behind a C ABI (include/vvenc_b200.h).

The Python layer is plumbing only (ctypes + numpy / torch device pointers); the product is csrc/*.cu."""
from .api import CostEngine, VvbError, DF_SSE, DF_SAD, DF_HAD, DF_HAD_FAST, DF_HAD_2SAD, DCT2, DCT8, DST7
from . import candidates
from ._lib import CAND_DT, POS_DT, BLOCK_DT, BEST_DT, MV_DT, MCTF_DT, MCTF_MV_DT, TU_RESULT_DT, TZ_PU_DT, TZ_BEST_DT, FRAC_BEST_DT, FRAC_PAR, BI_PU_DT, BI_BEST_DT, BI_PAR, AMVP_DT, AMVR_BEST_DT, AMVR_PAR, LIB_PATH

__all__ = ['CostEngine', 'VvbError', 'candidates', 'DF_SSE', 'DF_SAD', 'DF_HAD', 'DF_HAD_FAST', 'DF_HAD_2SAD', 'DCT2', 'DCT8', 'DST7',
           'CAND_DT', 'POS_DT', 'BLOCK_DT', 'BEST_DT', 'MV_DT', 'MCTF_DT', 'MCTF_MV_DT', 'TU_RESULT_DT', 'TZ_PU_DT', 'TZ_BEST_DT', 'FRAC_BEST_DT', 'FRAC_PAR', 'BI_PU_DT', 'BI_BEST_DT', 'BI_PAR', 'AMVP_DT', 'AMVR_BEST_DT', 'AMVR_PAR', 'LIB_PATH']
