"""The TU round trip with the slice's quantiser, pinned on the CPU: the oracle composition (tests/tu_rdo_cases.py) against the golden vectors the reference
wrote (tests/golden/golden_v8_tu_rdo.npz), and against the reference's own members, live, in its scalar and AVX2 builds where oracle/_ref exists."""
import os
import numpy as np
import pytest
import tu_rdo_cases as T
from _libs import have_ref

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'golden_v8_tu_rdo.npz')


@pytest.fixture(scope='module')
def golden_v8():
    return np.load(GOLDEN)


def golden_case(g, i):
    """(row, org, pred, rates, lfnst (set, transpose), expected q, reco, [dist_reco, dist_resi, dist_zero, abs_sum, last_pos], need_rdoq) of golden case i"""
    row = g['cases'][i]
    org, pred = T.inputs(row)
    assert T.inputs_crc(org[0], pred[0]) == int(g['inputs_crc'][i]), 'tu_rdo_cases.inputs() no longer regenerates the inputs of golden case %d' % i
    m = [int(v) for v in g['meta'][i]]
    return row, org[0], pred[0], g['rates_%d' % i], tuple(int(v) for v in g['lfnst'][i]), g['q_%d' % i], (pred[0] + g['dreco_%d' % i]).astype(np.int16), m[:5], m[5]


def test_golden_covers_the_issue_space(golden_v8):
    rows = [T.row_dict(r) for r in golden_v8['cases']]
    meta = golden_v8['meta']
    assert len(rows) >= 300
    assert {(r['w'], r['h']) for r in rows} == set(T.SHAPES)
    assert {r['quantiser'] for r in rows} == {1, 2} and {r['comp'] for r in rows} == {0, 1} and {r['bd'] for r in rows} == {8, 10}
    assert {r['lfnst'] for r in rows} == {0, 1, 2} and {(r['th'], r['tv']) for r in rows} == set(T.MTS_IDX)
    assert {r['sh'] for r in rows if r['quantiser'] == 1} == {0, 1} and {r['sel'] for r in rows} == {0, 1}
    assert any(T.zero_out(r) for r in rows)
    assert min(r['qp'] for r in rows) == 17 and max(r['qp'] for r in rows) == 51
    assert (meta[:, 3] > 0).any() and (meta[:, 3] == 0).any() and set(meta[:, 5].tolist()) == {0, 1}


def test_oracle_composition_equals_golden(golden_v8):
    bad = []
    for i in range(len(golden_v8['cases'])):
        row, org, pred, rates, st, eq, ereco, em, en = golden_case(golden_v8, i)
        q, reco, m, need = T.oracle_roundtrip_rdo(row, org, pred, rates, st)
        if not (np.array_equal(q, eq) and np.array_equal(reco, ereco) and m == em and need == en):
            bad.append((i, T.row_dict(row), m, em, need, en))
    assert bad == [], (len(bad), bad[:3])


@pytest.mark.skipif(not have_ref(), reason='oracle/_ref (the reference probe) is built only where the reference sources are available')
@pytest.mark.parametrize('simd', [b'SCALAR', b'AVX2'])
def test_oracle_composition_equals_reference(simd):
    """fresh seeded cases (not the golden rows) through the reference's members and through the oracle, with the rates the reference read"""
    rows = T.cases(120, seed=9301)
    bad = []
    for row in rows:
        org, pred = T.inputs(row)
        q, reco, m, need, rates, st = T.ref_roundtrip_rdo(row, org[0], pred[0], simd)
        oq, oreco, om, oneed = T.oracle_roundtrip_rdo(row, org[0], pred[0], rates, st)
        if not (np.array_equal(q, oq) and np.array_equal(reco, oreco) and m == om and need == oneed):
            bad.append((T.row_dict(row), m, om))
    assert bad == [], (len(bad), bad[:3])
