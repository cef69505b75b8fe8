"""ci_res_gs_kernel + dmv_ci_calc_res_and_gs (CoarseInitializer::calcResAndGS, DESIGN.md §5c) against the fp64 reference
tests/helpers.ci_calc_ref at DSO's point densities, with every comparison made on every evaluation.

Scenes: dense_640x480 (setFirst's densities 0.03 / 0.05 of w0 h0 at levels 0 and 1: two trips of the kernel's grid-stride loop on an H100),
euroc_752x480 (5 levels, coarsest 47x30, 18 048 points at level 1), tumvi_512x512 (4 levels), trip_edges (one level with n at and around
multiples of one trip, 2 SMs x 32 points, and n = 1, 7) and edges (points that leave the image, idepth_new < 0, one NaN in each plane).
Each level is evaluated fresh, after a small motion (alphaOpt = alphaW), after a snapped motion (alphaOpt = 0, iR != idepth_new) and with
~10 % of the points !isGood.

Exact: the verdict of every point that is not ambiguous, energies carried by points that are not good, energy_new[1] = (id - 1)^2, zero
Jb rows and maxstep = 1e10 where the input is !isGood, res3[1] and alphaOpt (the reference's rounding), res3[2] = 2n, n_good_new, symmetry
of H and Hsc, and the same bits from two launches on one handle.  Bounded (ci_calc_ref's first-order fp32 bound with the kernel's summation
depth): every other per-point output, res3[0], H, b, Hsc, bsc.  The largest |err|/bound of each is printed (pytest -s)."""
import numpy as np
import pytest

from helpers import (CI_ALPHA_K, CI_ALPHA_W, CI_STATES, alpha_cases, alpha_restatement, ci_bound_ratio, ci_calc_ref, ci_kernel_depth, ci_operands,
                     ci_points, ci_poison, ci_state)

pytestmark = pytest.mark.gpu

CI_OUTLIER_TH = np.float32(8 * 12 * 12)   # patternNum * setting_outlierTH (setFirst, CoarseInitializer.cpp:L857)
SCENES = dict(dense_640x480=(640, 480, (9216, 15360, 12000, 3000), 77),
              euroc_752x480=(752, 480, (10829, 18048, 12000, 3000, 600), 20),
              tumvi_512x512=(512, 512, (7864, 13107, 8000, 2000), 15))
OUTPUTS = ("isGood_new", "energy_new", "maxstep", "lastHessian_new", "Jb", "H", "b", "Hsc", "bsc", "res", "alphaOpt", "n_good_new")


def _sms():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


class Level:
    """one level of a handle: its planes, intrinsics and static point fields"""

    def __init__(self, g, lvl, first, new, k4, pts):
        self.g, self.lvl, self.first, self.new, self.k4 = g, lvl, first, new, k4
        self.u, self.v = pts["u"], pts["v"]
        self.n = len(self.u)
        self.th = np.full(self.n, CI_OUTLIER_TH, np.float32)
        g.set_K(lvl, *[float(x) for x in k4])
        g.upload_first(lvl, first)
        g.upload_new(lvl, new)
        g.set_points(lvl, self.u, self.v, self.th)


def _eval(L, st, synth, sms, worst, tag, wzp=(0.0, 0.0), huber=9.0):
    """one launch against ci_calc_ref at the Huber threshold `huber`: every exact check and every bounded one; worst collects the largest
    |err|/bound per quantity"""
    R, t, RKi, tlog = ci_operands(synth, L.k4, st)
    aff = (np.float32(np.exp(st["a"])), np.float32(st["b"]))
    n = L.n
    sg = L.g.calc_res_and_gs(L.lvl, RKi, t, tlog, aff, st["idepth_new"], st["isGood"], st["energy"], st["iR"], huberTH=huber, wzpx=wzp[0],
                             wzpy=wzp[1])
    good = sg["isGood_new"] != 0
    ref = ci_calc_ref(L.first, L.new, L.k4, L.u, L.v, L.th, st["idepth_new"], st["isGood"], st["energy"], st["iR"], RKi, t, tlog, aff,
                      huber=huber, wzp=wzp, depth=ci_kernel_depth(n, sms), verdict=good)
    sure = ~ref["amb"]
    assert np.array_equal(good[sure], ref["isGood_new"][sure]), (tag, np.nonzero(good[sure] != ref["isGood_new"][sure])[0][:10])
    np.testing.assert_array_equal(sg["energy_new"][~good], st["energy"][~good], err_msg=tag)
    id1 = st["idepth_new"] - np.float32(1)
    np.testing.assert_array_equal(sg["energy_new"][good, 1], (id1 * id1)[good], err_msg=tag)
    was = st["isGood"] != 0
    assert not sg["Jb"][~good].any() and not sg["lastHessian_new"][~good].any(), tag
    assert np.all(sg["maxstep"][~was] == np.float32(1e10)), tag
    aE, aO = alpha_restatement(CI_ALPHA_W, CI_ALPHA_K, t, n)
    assert sg["res"][1] == aE and np.float32(sg["alphaOpt"]) == aO, (tag, sg["res"][1], aE, sg["alphaOpt"], aO)
    assert sg["res"][2] == 2 * n and sg["n_good_new"] == int(good.sum()), tag
    assert np.array_equal(sg["H"], sg["H"].T) and np.array_equal(sg["Hsc"], sg["Hsc"].T), tag
    g = good & sure
    q = dict(E0=ci_bound_ratio(sg["energy_new"][g, 0], ref["energy_new"][g, 0], ref["dE0"][g]),
             maxstep=ci_bound_ratio(sg["maxstep"][g], ref["maxstep"][g], ref["dmaxstep"][g]),
             lastH=ci_bound_ratio(sg["lastHessian_new"][g], ref["lastHessian_new"][g], ref["dlastH"][g]),
             Jb=ci_bound_ratio(sg["Jb"][g], ref["Jb"][g], ref["dJb"][g]),
             res0=ci_bound_ratio(sg["res"][0], ref["res3"][0], ref["dres0"]))
    for k in ("H", "b", "Hsc", "bsc"):
        q[k] = ci_bound_ratio(sg[k], ref[k], ref["d" + k])
    for k, x in q.items():
        worst[k] = max(worst.get(k, 0.0), x)
    assert max(q.values()) <= 1.0, (tag, q)
    return sg, ref


def _same_bits(a, b, tag):
    for k in OUTPUTS:
        assert np.array_equal(np.asarray(a[k]), np.asarray(b[k])), (tag, k)


def _report(name, worst, extra=""):
    print(f"\n{name}: worst |err|/bound " + " ".join(f"{k}={x:.3g}" for k, x in worst.items()) + extra)


@pytest.mark.parametrize("scene", list(SCENES))
def test_calc_res_and_gs_vs_ref(synth, scene):
    import dmvio_b200.capi as capi
    w, h, counts, seed = SCENES[scene]
    T = synth.make_tracking_pair(w=w, h=h, seed=seed, trans=0.02, rot=0.005)
    nl = T["levels"]
    assert nl == len(counts)
    pts = ci_points(np.random.default_rng(seed), w, h, nl, counts)
    assert [len(p["u"]) for p in pts] == list(counts)
    sms = _sms()
    g = capi.CI(w, h, nl, max_points=max(counts))
    levels = [Level(g, l, T["pyr_ref"][l], T["pyr_new"][l], synth.level_K(T["K"], l), pts[l]) for l in range(nl)]
    worst, first_runs, branches, ngood = {}, {}, set(), []
    for lvl in range(nl - 1, -1, -1):
        for s, kind in enumerate(CI_STATES):
            st = ci_state(kind, counts[lvl], 1000 * lvl + s)
            sg, ref = _eval(levels[lvl], st, synth, sms, worst, f"{scene} lvl{lvl} {kind}")
            branches.add(float(ref["alphaOpt"]))
            ngood.append(sg["n_good_new"] / counts[lvl])
            if kind == "motion":
                first_runs[lvl] = (st, sg)
    assert branches == {0.0, CI_ALPHA_W}
    assert min(ngood) > 0.3, ngood
    # the same bits again: level 0 after the coarsest level, then the coarsest (small) level after level 0 (the ticket and the per-CTA
    # partials are reused)
    for lvl in (0, nl - 1):
        st, sg = first_runs[lvl]
        _same_bits(_eval(levels[lvl], st, synth, sms, {}, f"{scene} repeat lvl{lvl}")[0], sg, f"{scene} repeat lvl{lvl}")
    if scene == "dense_640x480":
        assert min(counts[:2]) > 2 * sms * 32   # levels 0 and 1 take two trips of the grid-stride loop
    _report(scene, worst, f"  (good fraction {min(ngood):.2f} .. {max(ngood):.2f})")
    g.close()


def test_calc_res_and_gs_vs_ref_trip_edges(synth):
    """one 640x480 level with n = k * (2 SMs * 32) + {-1, 0, +1} for k = 1, 2 (the grid-stride loop's trip boundaries) and n = 1, 7"""
    import dmvio_b200.capi as capi
    sms = _sms()
    trip = 2 * sms * 32
    ns = [k * trip + d for k in (1, 2) for d in (-1, 0, 1)] + [1, 7]
    T = synth.make_tracking_pair(w=640, h=480, seed=41, trans=0.02, rot=0.005, levels=1)
    g = capi.CI(640, 480, 1, max_points=max(ns))
    k4 = synth.level_K(T["K"], 0)
    worst, runs = {}, {}
    for i, n in enumerate(ns):
        pts = ci_points(np.random.default_rng(n), 640, 480, 1, (n,))[0]
        assert len(pts["u"]) == n
        L = Level(g, 0, T["pyr_ref"][0], T["pyr_new"][0], k4, pts)
        kind = CI_STATES[1 + i % 3]
        st = ci_state(kind, n, i)
        runs[n] = (L, st, _eval(L, st, synth, sms, worst, f"trip n={n} {kind}")[0])
    for n in (ns[-1], ns[5], ns[-2]):   # the same bits again, each after a launch of another size on the handle
        L, st, sg = runs[n]
        L = Level(g, 0, T["pyr_ref"][0], T["pyr_new"][0], k4, dict(u=L.u, v=L.v))
        _same_bits(_eval(L, st, synth, sms, {}, f"trip repeat n={n}")[0], sg, f"trip repeat n={n}")
    _report(f"trip_edges (SMs={sms}, n={ns})", worst)
    g.close()


def test_calc_res_and_gs_vs_ref_edges(synth):
    """a large motion that takes part of the points out of the image, a few idepth_new < 0, one NaN in each plane at a tap some points
    read; 4999 points, not a multiple of a warp's 4"""
    import dmvio_b200.capi as capi
    T = synth.make_tracking_pair(seed=31, trans=0.02, rot=0.005)
    pts = ci_points(np.random.default_rng(8), T["w"], T["h"], 1, (4999,))[0]
    n = len(pts["u"])
    k4 = synth.level_K(T["K"], 0)
    st_edge = ci_state("edge", n, 3)
    first, new = ci_poison(T["pyr_ref"][0], T["pyr_new"][0], pts, st_edge, k4, synth)
    sms = _sms()
    g = capi.CI(T["w"], T["h"], 1, max_points=n)
    L = Level(g, 0, first, new, k4, pts)
    worst = {}
    sg, ref = _eval(L, st_edge, synth, sms, worst, "edges")
    bad = sg["isGood_new"] == 0
    assert 0.1 < bad.mean() < 0.9 and bad[st_edge["idepth_new"] < 0].all() and bad[0]
    for s, kind in enumerate(CI_STATES):
        _eval(L, ci_state(kind, n, 10 + s), synth, sms, worst, f"edges {kind}")
    _report("edges", worst, f"  (edge state: {int(bad.sum())} of {n} not good, {ref['n_amb']} ambiguous)")
    g.close()


def _dense_level(synth, capi, lvl):
    """level lvl of dense_640x480 on a handle of its own"""
    w, h, counts, seed = SCENES["dense_640x480"]
    T = synth.make_tracking_pair(w=w, h=h, seed=seed, trans=0.02, rot=0.005)
    pts = ci_points(np.random.default_rng(seed), w, h, lvl + 1, counts)[lvl]
    g = capi.CI(w, h, lvl + 1, max_points=counts[lvl])
    return g, Level(g, lvl, T["pyr_ref"][lvl], T["pyr_new"][lvl], synth.level_K(T["K"], lvl), pts)


def test_alpha_energy_rounding(synth):
    """t = (0, 0, s) with s where the reference's rounding of alphaEnergy (double, once) and a float product of float(|t|^2 n) disagree:
    on alphaOpt in both directions and on the caller's `res3[1] == alphaK n` snap test in both directions (levels 0 and 2 of dense_640x480,
    9216 and 12000 points, between them have all four).  res3[1] and alphaOpt must be the reference's bit for bit (checked in _eval) and the
    system within the bound of ci_calc_ref, which takes the reference's alphaOpt."""
    import dmvio_b200.capi as capi
    sms, worst, found = _sms(), {}, set()
    for lvl in (0, 2):
        g, L = _dense_level(synth, capi, lvl)
        cases = alpha_cases(L.n)
        found |= set(cases)
        for kind, s in cases.items():
            st = ci_state("motion", L.n, 7)
            st["xi"] = np.array([0.0, 0.0, s, 0.0, 0.0, 0.0])
            _eval(L, st, synth, sms, worst, f"alpha n={L.n} {kind} s={s!r}")
        g.close()
    assert {"cap_ref_only", "cap_old_only", "eq_ref_only", "eq_old_only"} <= found, found
    _report(f"alphaEnergy (cases {sorted(found)})", worst)


def test_zero_prior(synth):
    """setting_weightZeroPriorDSOInitX/Y = 5e9 (DM-VIO's 4seasons configuration) against 0: H[0,0], H[1,1], b[0], b[1] are the zero-prior-free
    values plus the prior in double, rounded once; every other entry is identical"""
    import dmvio_b200.capi as capi
    g, L = _dense_level(synth, capi, 0)
    sms = _sms()
    for kind in ("motion", "snapped"):
        st = ci_state(kind, L.n, 21)
        _, t, _, _ = ci_operands(synth, L.k4, st)
        s0, _ = _eval(L, st, synth, sms, {}, f"zero prior 0 {kind}")
        s1, _ = _eval(L, st, synth, sms, {}, f"zero prior 5e9 {kind}", wzp=(5e9, 5e9))
        H, b = s0["H"].copy(), s0["b"].copy()
        H[0, 0] = np.float32(np.float64(H[0, 0]) + 5e9)
        H[1, 1] = np.float32(np.float64(H[1, 1]) + 5e9)
        b[0] = np.float32(np.float64(b[0]) + 5e9 * t[0])
        b[1] = np.float32(np.float64(b[1]) + 5e9 * t[1])
        np.testing.assert_array_equal(s1["H"], H)
        np.testing.assert_array_equal(s1["b"], b)
        for k in ("Hsc", "bsc", "res", "Jb", "energy_new", "isGood_new", "maxstep", "lastHessian_new"):
            np.testing.assert_array_equal(s1[k], s0[k], err_msg=k)
    g.close()
