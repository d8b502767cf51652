"""The instruction-mix probes behind bench.py's alu roofline and tools/mma_probe.py: every mode of vvb_alu_probe_dev launches and completes."""
import pytest

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("mode", [0, 1, 2, 3, 4])
def test_alu_probe_modes_run(mode):
    import torch
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    import vvenc_b200 as V
    eng = V.CostEngine(0)
    try:
        assert eng.lib.vvb_alu_probe_dev(eng.h, 4, 64, mode) == 0, eng.lib.vvb_last_error(eng.h)
        eng.synchronize()
    finally:
        eng.close()
