"""CPU tier of dmv_ba_select_activation's oracle: the restatement of makeDistanceMap, growDistBFS, addIntoDistFinal and activatePointsMT's
selection loop (oracle/orc_activation.cpp) against the reference's own compiled CoarseDistanceMap (oracle/_ref/libactivation_ref.so) and
against the golden fixture made from it.  Bit equality of the actions, toOptimize and the map."""
import os

import numpy as np
import pytest

from oracle import activation as A

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "golden_activation.npz")
needs_ref = pytest.mark.skipif(not A.ref_available(), reason="oracle/_ref/libactivation_ref.so not built (no reference sources)")


def _golden(name):
    G = np.load(GOLDEN)
    return G[f"{name}/tab"], G[f"{name}/action"], G[f"{name}/opt"], G[f"{name}/map"]


@pytest.mark.parametrize("name", sorted(A.CASES))
def test_restatement_equals_golden(name):
    tab, act, opt, m = _golden(name)
    a, o, mm = A.restate(A.make_case(**A.CASES[name]), tab)
    assert np.array_equal(a, act) and np.array_equal(o, opt) and np.array_equal(mm, m)


@needs_ref
@pytest.mark.parametrize("name", sorted(A.CASES))
def test_reference_equals_restatement_and_golden(name):
    case = A.make_case(**A.CASES[name])
    act, opt, m, tab = A.reference(case)
    a, o, mm = A.restate(case, tab)
    assert np.array_equal(a, act) and np.array_equal(o, opt) and np.array_equal(mm, m)
    g = _golden(name)
    assert np.array_equal(g[0], tab) and np.array_equal(g[1], act) and np.array_equal(g[2], opt) and np.array_equal(g[3], m)


def _project(tab, u, v, x):
    """the projection in float32 (numpy's scalar float32 arithmetic rounds every operation, as the reference's SSE code does)"""
    T = tab.reshape(-1, 12)
    with np.errstate(all="ignore"):
        ptp = [((T[:, 3 * k] * u + T[:, 3 * k + 1] * v) + T[:, 3 * k + 2] * np.float32(1)) + T[:, 9 + k] * x for k in range(3)]
        return ptp[0], ptp[1], ptp[2], ptp[0] / ptp[2] + np.float32(0.5)


def test_cases_reach_every_branch():
    seen = {k: False for k in ("del_nonfinite", "del_outlier", "del_notready_flagged", "del_notready_oob", "del_outside", "keep_notready", "keep_map",
                               "opt", "fail_status", "fail_interval", "fail_quality", "fail_depth", "type1", "type2", "type4", "mad0", "mad4",
                               "act_behind", "act_nan", "act_huge", "cand_behind", "cand_nan", "cand_huge", "newest_skipped", "empty_host",
                               "empty_active", "active_all_outside", "opt_border_ring", "opt_inside_ring")}
    for name, kw in A.CASES.items():
        case = A.make_case(**kw)
        tab, act, opt, m = _golden(name)
        I, off, nf, newest = case["imm"], case["off"], case["nf"], case["newest"]
        host = np.repeat(np.arange(nf), np.diff(off))
        other = host != newest
        st, imax, imin = I["status"], I["idepth_max"], I["idepth_min"]
        with np.errstate(invalid="ignore", over="ignore"):
            c_status = np.isin(st, (0, 1, 3, 4))
            c_int, c_q, c_d = I["interval"] < 8, I["quality"] > np.float32(A.MIN_TRACE_QUALITY), (imax + imin) > 0
        alive = other & np.isfinite(imax) & (st != 2)
        can = c_status & c_int & c_q & c_d
        seen["del_nonfinite"] |= bool(np.any(other & ~np.isfinite(imax) & (act == 1)))
        seen["del_outlier"] |= bool(np.any(other & np.isfinite(imax) & (st == 2) & (act == 1)))
        seen["del_notready_flagged"] |= bool(np.any(alive & ~can & (st != 1) & (case["flagged"][host] == 1) & (act == 1)))
        seen["del_notready_oob"] |= bool(np.any(alive & ~can & (st == 1) & (case["flagged"][host] == 0) & (act == 1)))
        seen["keep_notready"] |= bool(np.any(alive & ~can & (act == 0)))
        seen["del_outside"] |= bool(np.any(alive & can & (act == 1)))
        seen["keep_map"] |= bool(np.any(alive & can & (act == 0)))
        seen["opt"] |= len(opt) > 0
        for key, fails in (("fail_status", ~c_status), ("fail_interval", ~c_int), ("fail_quality", ~c_q), ("fail_depth", ~c_d)):
            alone = fails & (c_status | (key == "fail_status")) & (c_int | (key == "fail_interval")) & (c_q | (key == "fail_quality")) & (c_d | (key == "fail_depth"))
            seen[key] |= bool(np.any(alive & alone))
        for t in (1, 2, 4):
            seen[f"type{t}"] |= bool(np.any(alive & can & (I["type"] == t)))
        seen["mad0"] |= case["min_act_dist"] == 0 and len(opt) > 0
        seen["mad4"] |= case["min_act_dist"] == 4 and len(opt) > 0
        seen["newest_skipped"] |= bool(off[newest + 1] > off[newest] and np.all(act[off[newest]:off[newest + 1]] == 0))
        seen["empty_host"] |= bool(np.any(np.diff(off)[:newest] == 0))
        w1, h1 = case["w"] // 2, case["h"] // 2
        seen["empty_active"] |= len(case["act_u"]) == 0
        ah = case["act_host"]
        if len(ah):
            T = tab.reshape(-1, 12)[ah].reshape(-1)
            _, p1, p2, q = _project(T, case["act_u"], case["act_v"], case["act_id"])
            with np.errstate(all="ignore"):
                qv = p1 / p2 + np.float32(0.5)
                inside = (q >= 1) & (q < w1) & (qv >= 1) & (qv < h1) & (ah != newest)
            seen["act_behind"] |= bool(np.any((p2 <= 0) & (ah != newest)))
            seen["act_nan"] |= bool(np.any(np.isnan(q) & (ah != newest)))
            seen["act_huge"] |= bool(np.any(np.isfinite(q) & (np.abs(q) > 2.0 ** 31) & (ah != newest)))
            seen["active_all_outside"] |= not bool(np.any(inside))
        cand = alive & can
        if np.any(cand):
            T = tab.reshape(-1, 12)[host[cand]].reshape(-1)
            with np.errstate(over="ignore"):
                x = np.float32(0.5) * (imax[cand] + imin[cand])
            _, _, p2, q = _project(T, I["u"][cand], I["v"][cand], x)
            seen["cand_behind"] |= bool(np.any(p2 <= 0))
            seen["cand_nan"] |= bool(np.any(np.isnan(q)))
            seen["cand_huge"] |= bool(np.any(np.isfinite(q) & (np.abs(q) > 2.0 ** 31)))
        if len(opt) and kw.get("border"):
            p0, p1, p2, q = _project(tab.reshape(-1, 12)[host[opt]].reshape(-1), I["u"][opt], I["v"][opt], np.float32(0.5) * (imax[opt] + imin[opt]))
            cu, cv = q.astype(np.int64), (p1 / p2 + np.float32(0.5)).astype(np.int64)
            seen["opt_border_ring"] |= bool(np.any((cu == w1 - 1) | (cv == h1 - 1)))
            seen["opt_inside_ring"] |= bool(np.any((cu == w1 - 2) | (cv == 1)))
    missing = [k for k, v in seen.items() if not v]
    assert not missing, missing


def test_candidate_order_matters_in_a_cluster():
    """dense clusters: reversing the order of the candidates changes which points are accepted (and the map)"""
    case = A.make_case(**A.CASES["cluster"])
    tab = _golden("cluster")[0]
    a0, o0, m0 = A.restate(case, tab)
    n0 = int(case["off"][1])
    for k in A.IMM_KEYS:
        case["imm"][k][:n0] = case["imm"][k][:n0][::-1].copy()
    a1, o1, m1 = A.restate(case, tab)
    assert not np.array_equal(a0[:n0], a1[:n0][::-1]) or not np.array_equal(m0, m1)


@needs_ref
def test_flood_matches_reference_and_is_not_a_per_seed_minimum():
    """addIntoDistFinal sequences on random and border-hugging seed sets: the restatement equals the reference's own BFS; the map after
    several floods is neither the per-seed minimum nor independent of the order of the seeds, which is why the device runs them in order"""
    w, h = 320, 240
    w1, h1 = w // 2, h // 2
    rng = np.random.default_rng(7)
    not_min = order_dep = 0
    for trial in range(60):
        m0 = np.full(w1 * h1, 1000, np.float32) if trial % 2 == 0 else rng.choice([0, 1, 2, 3, 5, 1000], w1 * h1).astype(np.float32)
        pick = lambda lo, hi: int(rng.integers(lo, hi)) if rng.random() < 0.6 else int(rng.choice([1, 2, hi - 2, hi - 1]))
        seeds = [(pick(1, w1), pick(1, h1)) for _ in range(int(rng.integers(2, 8)))]
        if trial % 3 == 0:   # a tight cluster
            x, y = pick(1, w1), pick(1, h1)
            seeds = [(min(w1 - 1, max(1, x + int(rng.integers(-6, 7)))), min(h1 - 1, max(1, y + int(rng.integers(-6, 7))))) for _ in range(6)]
        seq = A.flood("orc", w, h, m0, seeds)
        assert np.array_equal(seq, A.flood("ref", w, h, m0, seeds))
        per = np.minimum(m0, np.min([A.flood("orc", w, h, np.full_like(m0, 1000), [s]) for s in seeds], axis=0))
        not_min += not np.array_equal(seq, per)
        order_dep += not np.array_equal(seq, A.flood("orc", w, h, m0, seeds[::-1]))
    assert not_min > 0 and order_dep > 0
