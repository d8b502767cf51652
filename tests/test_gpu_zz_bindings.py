"""-m gpu: the batched reference-side bindings of integration/ (InterSearchB200.h, MCTFB200.h, TrQuantB200.h, plus RdCostB200.h once more) bound to the REAL
libvvenc_b200.so and run next to the reference's own member functions -- the comparison tests/test_integration_host.py makes on the CPU with the oracle-backed
mock, with the kernels answering instead.  Runs in a process of its own (the probe binds one library per process) and last in the suite.

First ran on hardware at the end of round 1; the xfail guard is gone since."""
import json
import os
import subprocess
import sys

import pytest

from _libs import have_ref

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
pytestmark = [pytest.mark.gpu, pytest.mark.skipif(not have_ref(), reason='oracle/_ref not built')]


def test_batched_bindings_on_the_real_library():
    import vvenc_b200._lib as VL
    out = subprocess.run([sys.executable, os.path.join(ROOT, 'tests', '_integration_host_run.py'), VL.LIB_PATH], capture_output=True, text=True, timeout=400)
    assert out.returncode == 0, out.stderr[-3000:]
    line = [ln for ln in out.stdout.splitlines() if ln.startswith('RESULT ')]
    assert line, out.stdout[-2000:]
    r = json.loads(line[-1][len('RESULT '):])
    assert r['dist_mismatches'] == 0 and r['affine']['bad'] == 0
    for s in r['search']:
        assert s['rc'] == [0, 0] and s['member_eq_b200'] and s['member_eq_rows'], s
    for t in r['tz']:
        assert t['rc'] == [0, 0] and t['eq'], t
    for f in r['frac']:
        assert f['rc'] == 0 and f['eq'], f
    for m in r['mctf']:
        assert m['rc'] == [0] * 6 and all(m['eq']), m
    for a in r['mctf_apply']:
        assert a['rc'] == 0 and a['eq'], a
    for a in r['mctf_apply420']:
        assert a['rc'] == [0, 0] and a['eq_luma'] and a['eq_chroma'], a
    assert r['tu_fwd_lfnst']['cases'] == 288 and r['tu_fwd_lfnst']['bad'] == []
    assert r['tu_ts_chroma']['cases'] == 220 and r['tu_ts_chroma']['bad'] == []
    assert r['tu_inv_dq']['cases'] == 168 and r['tu_inv_dq']['bad'] == []
    assert r['tu_inv_lfnst']['cases'] == 288 and r['tu_inv_lfnst']['bad'] == []
    assert r['dep_quant_chroma']['cases'] == 72 and r['dep_quant_chroma']['bad'] == []
    assert r['dep_quant']['cases'] == 216 and r['dep_quant']['non_empty'] > 100 and r['dep_quant']['bad'] == []
    assert r['tu_fwd']['bad'] == [] and r['tu_inv']['bad'] == [] and r['tu_fwd_sdh']['bad'] == [] and r['tu_fwd_sdh']['levels_changed_by_hiding'] > 60
