"""-m gpu, needs >= 2 GPUs on the box (skipped otherwise): the SHARDED product path on hardware.
  * bench.py's N-rank run: CTU-row bands of one picture (bands.split_ctu_rows), NCCL all-gather of the result tables (bands.BandGather), gathered tables ==
    the tables one GPU computes alone; and BASELINE configs[4] (one 7680x4320 picture, strong scaling) with the same check.
  * BASELINE configs[3]: MCTF, 8 neighbour pictures dealt over the ranks (bands.split_refs), all-gather of the motion fields, apply stage on every rank;
    fields and filtered picture == single GPU, first field == the reference's own motionEstimationMCTF."""
import json
import os
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
pytestmark = pytest.mark.gpu


def _ngpu():
    import torch
    return torch.cuda.device_count() if torch.cuda.is_available() else 0


def _torchrun(n, script_args, timeout):
    port = 29500 + (os.getpid() % 400)
    cmd = [sys.executable, '-m', 'torch.distributed.run', '--nnodes=1', '--nproc-per-node', str(n), '--master-addr', '127.0.0.1', '--master-port', str(port)] + script_args
    return subprocess.run(cmd, capture_output=True, text=True, timeout=timeout, cwd=ROOT)


def test_sharded_search_parity_on_gpus():
    n = min(_ngpu(), 4)
    if n < 2:
        pytest.skip('needs at least 2 GPUs')
    out = _torchrun(n, ['bench.py', '--gpus', str(n), '--steps', '1', '--warmup', '3', '--pictures-per-step', '2', '--skip-e2e', '--skip-cpu'], 900)
    assert out.returncode == 0, out.stderr[-3000:]
    line = json.loads([l for l in out.stdout.splitlines() if l.startswith('{')][-1])
    assert line['n_gpus'] == n
    sp = line['extra']['sharded_parity']
    assert sp['gathered_equals_single_gpu'] and sp['bands'] == n and sp['blocks_checked'] > 100000
    st = line['extra']['strong_4320p']
    assert st['parity']['gathered_equals_single_gpu'] and st['parity']['whole_picture_vs_bands_sampled']['equal'] and st['parity']['whole_picture_vs_bands_sampled']['blocks'] > 1000
    assert st['strong_efficiency'] > 0.5


def test_mctf_refs_over_gpus():
    n = min(_ngpu(), 4)
    if n < 2:
        pytest.skip('needs at least 2 GPUs')
    out = _torchrun(n, [os.path.join('tests', '_mctf_multigpu_run.py'), '832', '480'], 900)
    assert out.returncode == 0, (out.stdout[-2000:], out.stderr[-3000:])
    r = json.loads([l for l in out.stdout.splitlines() if l.startswith('RESULT ')][-1][len('RESULT '):])
    assert r['fields_equal_single_gpu'] and r['filtered_equal_single_gpu'] and r['filtered_equal_on_all_ranks']
    assert r.get('field0_equals_reference_motionEstimationMCTF', True)
    assert r['fractional_vectors'] > 0
