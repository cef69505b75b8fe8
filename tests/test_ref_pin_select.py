"""CPU tier of dmv_ct_make_new_traces' oracle: the restatement of PixelSelector::makeMaps + makeNewTraces (oracle/orc_select.cpp) against the
reference's own compiled code (oracle/_ref/libselect_ref.so) and against the golden fixture made from it."""
import os
import subprocess
import sys

import numpy as np
import pytest

from oracle import orc
from oracle import select as S

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "golden_select.npz")
needs_ref = pytest.mark.skipif(not S.ref_available(), reason="oracle/_ref/libselect_ref.so not built (no reference sources)")


def _same(a, b):
    assert a["numPointsTotal"] == b["numPointsTotal"]
    assert a["potential"] == b["potential"]
    for k in S.POINT_KEYS:
        assert np.array_equal(a["points"][k], b["points"][k]), k


def _golden(G, key):
    return dict(points={k: G[f"{key}/{k}"] for k in S.POINT_KEYS}, numPointsTotal=int(G[f"{key}/numPointsTotal"]), potential=int(G[f"{key}/potential"]))


def _restate_case(name):
    w, h, lv, kind, seed, args = S.CASES[name]
    a = S.case_args(args)
    img = S.image(kind, w, h, seed)
    return S.restate(orc.make_images(img, S.K_of(w, h), lv)[:3], **a), img, a


@needs_ref
@pytest.mark.parametrize("name", sorted(S.CASES))
def test_restatement_equals_reference(name):
    w, h, lv, kind, seed, args = S.CASES[name]
    o, img, a = _restate_case(name)
    R = S.Ref(w, h)
    R.potential = a.pop("potential", 3)
    r = R.new_traces(img, S.K_of(w, h), **a)
    R.close()
    assert np.array_equal(r["map"], o["map"])
    _same(r, o)


@needs_ref
def test_sequence_on_one_selector_equals_reference():
    w, h = S.SEQ[0][:2]
    R = S.Ref(w, h)
    pot = 3
    for w_, h_, lv, kind, seed in S.SEQ:
        img = S.image(kind, w, h, seed)
        r = R.new_traces(img, S.K_of(w, h))
        o = S.restate(orc.make_images(img, S.K_of(w, h), lv)[:3], potential=pot)
        assert np.array_equal(r["map"], o["map"])
        _same(r, o)
        pot = o["potential"]
    R.close()


@needs_ref
def test_golden_fixture_is_the_reference():
    G = np.load(GOLDEN)
    for name, (w, h, lv, kind, seed, args) in S.CASES.items():
        a = S.case_args(args)
        R = S.Ref(w, h)
        R.potential = a.pop("potential", 3)
        _same(R.new_traces(S.image(kind, w, h, seed), S.K_of(w, h), **a), _golden(G, name))
        R.close()


@pytest.mark.parametrize("name", sorted(S.CASES))
def test_restatement_equals_golden(name):
    _same(_restate_case(name)[0], _golden(np.load(GOLDEN), name))


def test_sequence_restatement_equals_golden():
    G = np.load(GOLDEN)
    pot = 3
    for i, (w, h, lv, kind, seed) in enumerate(S.SEQ):
        o = S.restate(orc.make_images(S.image(kind, w, h, seed), S.K_of(w, h), lv)[:3], potential=pot)
        _same(o, _golden(G, f"seq{i}"))
        pot = o["potential"]


def test_cases_cover_the_branches():
    """the cases reach both recursion directions, sub-selection, the potential clamp, picks on row h-4, a flat frame and mixed blocks"""
    R = {name: _restate_case(name)[0] for name in S.CASES}
    pot0 = {name: S.case_args(a[5]).get("potential", 3) for name, a in S.CASES.items()}
    assert any(R[n]["potential"] < pot0[n] and pot0[n] > 1 and S.CASES[n][3] == "low" for n in R)        # quotia > 1.25: fewer points wanted
    assert any(R[n]["potential"] > pot0[n] and S.CASES[n][3] == "high" for n in R)                       # quotia < 0.25
    assert any(0.25 <= R[n]["quotia"] < 0.95 and R[n]["numPointsTotal"] > 0 for n in R)                   # sub-selection
    assert R["low512_l5_pot1"]["potential"] == 1
    assert R["flat640_l4"]["numPointsTotal"] == 0 and len(R["flat640_l4"]["points"]["u"]) == 0
    assert any((R[n]["map"][S.CASES[n][1] - 4] != 0).any() for n in R)                                   # row h-4: counted, no point
    for n in R:
        assert not (R[n]["points"]["v"] >= S.CASES[n][1] - 4).any()
    assert R["stripe640_l4"]["n_mixed"] > 0 and R["stair512_l5"]["n_mixed"] > 0
    assert R["stair512_l5"]["numPointsTotal"] > 0


def test_random_pattern_is_glibc_rand():
    n = 640 * 480
    code = ("import ctypes, sys; L = ctypes.CDLL('libc.so.6'); L.srand(3141592); n = int(sys.argv[1]);"
            "sys.stdout.buffer.write(bytes(L.rand() & 0xFF for _ in range(n)))")
    out = subprocess.run([sys.executable, "-c", code, str(n)], capture_output=True, check=True).stdout
    assert np.array_equal(np.frombuffer(out, np.uint8), S.random_pattern(n))
