"""dmv_ba_edit_window against a twin: a second BA handle with the same images that gets dmv_ba_set_window + dmv_ba_set_points +
dmv_ba_set_residuals from lists built by a numpy restatement of the header's rules (replay below), whose inputs are the twin's own read-backs
and the same activation outputs.  Both handles then get the same adjoints and state, and everything that follows must agree bit for bit:
linearize, gn_step with and without x, residual / point / target-energy outputs, idepth, accumulate, resubstitute, marginalize_points,
reset_oob, drop_residuals, the batched step, and launch counts."""
import numpy as np
import pytest

from dmvio_b200.capi import DMV_ERR_INVALID, DMV_ERR_STATE
from gpu_harness import assert_same, bits, capi, close, gpu  # noqa: F401
from helpers import edge_window, prior_f
from test_gpu_activate_store import Win, fill


# ---------------------------------------------------------------------------------------------------------------------------------
# the host's view of a window, the tables of a frame subset, and the restatement of the edit
# ---------------------------------------------------------------------------------------------------------------------------------
class Seq:
    """one synthetic sequence: every frame's image in slot = frame id, and the oracle's pair tables of all frames, sliced per window"""

    def __init__(self, W, ow):
        self.W, self.ow, self.nfa = W, ow, W["nf"]
        n = self.nfa
        self.P = ow.precalc().reshape(n, n, -1)                   # [h][t]
        adH, adT = ow.adjoints()
        self.adH, self.adT = adH.reshape(n, n, 8, 8), adT.reshape(n, n, 8, 8)   # [t][h]
        self.RT = ow.RT().reshape(n, n, 12)                       # [h][t]
        self.adD = ow.adHTdeltaF().reshape(n, n, 8)              # [t][h]
        self.TH = ow.frame_tables()["frameEnergyTH"]
        cal = ow.calib()
        self.k8, self.cD = cal["k8"], cal["cDeltaF"]

    def state(self, fr):
        ix = np.ix_(fr, fr)
        return self.k8, self.P[ix].reshape(len(fr) ** 2, -1), self.TH[list(fr)]

    def adjoints(self, fr):
        ix = np.ix_(fr, fr)
        return self.adH[ix].reshape(-1, 8, 8), self.adT[ix].reshape(-1, 8, 8)

    def rt(self, fr):
        return self.RT[np.ix_(fr, fr)].reshape(-1, 12)

    def adDelta(self, fr):
        return self.adD[np.ix_(fr, fr)].reshape(-1, 8)


class Mirror:
    """what the host keeps of a window: frames (ids of the sequence), points (host index in the window, read-only fields) and residuals
    with the input state the next linearisation reads"""

    def __init__(self, fr, host, u, v, color, weights, priorF, rp, rt, st, en):
        self.fr = list(fr)
        self.host, self.u, self.v = np.asarray(host, np.int32), np.asarray(u, np.float32), np.asarray(v, np.float32)
        self.color, self.weights = np.asarray(color, np.float32).reshape(-1, 8), np.asarray(weights, np.float32).reshape(-1, 8)
        self.priorF = np.asarray(priorF, np.float32)
        self.rp, self.rt = np.asarray(rp, np.int32), np.asarray(rt, np.int32)
        self.st, self.en = np.asarray(st, np.int32), np.asarray(en, np.float32)


def window_from(W, fr):
    """the window of frames fr (sequence ids): the points hosted there, by window host, and their residuals into fr in W's order"""
    fr = list(fr)
    pos = {f: i for i, f in enumerate(fr)}
    hw = np.array([pos.get(int(h), -1) for h in W["host"]])
    pts = np.array([p for p in np.lexsort((np.arange(len(hw)), hw)) if hw[p] >= 0], np.int64)
    newi = -np.ones(len(hw), np.int64)
    newi[pts] = np.arange(len(pts))
    tw = np.array([pos.get(int(t), -1) for t in W["res_target"]])
    keep = (newi[W["res_point"]] >= 0) & (tw >= 0)
    n = len(W["res_point"])
    st = W.get("res_state", np.zeros(n, np.int32))
    en = W.get("res_energy", np.zeros(n, np.float32))
    m = Mirror(fr, hw[pts], W["u"][pts], W["v"][pts], np.asarray(W["color"]).reshape(-1, 8)[pts], np.asarray(W["weights"]).reshape(-1, 8)[pts],
               prior_f(W)[pts], newi[W["res_point"][keep]], tw[keep], np.asarray(st)[keep], np.asarray(en)[keep])
    return m, np.asarray(W["idepth"], np.float32)[pts], np.asarray(W["idepth_zero"], np.float32)[pts]


def replay(m, idd, idz, fr_new, frame_src, point_src, nrt, act):
    """the header's rules on the host's lists: the new window's set_points / set_residuals arguments"""
    fnew = {int(s): f for f, s in enumerate(frame_src) if s >= 0}
    nf = len(fr_new)
    n = len(point_src)
    host = np.zeros(n, np.int32)
    u, v, pf, i1, z1 = (np.zeros(n, np.float32) for _ in range(5))
    col, wgt = np.zeros((n, 8), np.float32), np.zeros((n, 8), np.float32)
    pnew = {}
    for j, s in enumerate(point_src):
        if s >= 0:
            pnew[int(s)] = j
            host[j], u[j], v[j], col[j], wgt[j], pf[j], i1[j], z1[j] = fnew[int(m.host[s])], m.u[s], m.v[s], m.color[s], m.weights[s], m.priorF[s], idd[s], idz[s]
        else:
            k = -1 - s
            host[j], u[j], v[j], col[j], wgt[j], i1[j], z1[j] = fnew[int(act["host"][k])], act["u"][k], act["v"][k], act["color"][k], act["weights"][k], act["idepth"][k], act["idepth"][k]
    rp, rt, st, en = [], [], [], []
    for i in range(len(m.rp)):
        p, t = int(m.rp[i]), int(m.rt[i])
        if p in pnew and t in fnew:
            rp.append(pnew[p]); rt.append(fnew[t]); st.append(m.st[i]); en.append(m.en[i])
    if nrt >= 0:
        for j, s in enumerate(point_src):
            if s >= 0:
                rp.append(j); rt.append(nrt); st.append(0); en.append(0.0)
    for j, s in enumerate(point_src):
        if s < 0:
            for t in range(nf):
                if frame_src[t] >= 0 and act["rs"][-1 - s, frame_src[t]] == 0:
                    rp.append(j); rt.append(t); st.append(0); en.append(0.0)
    return Mirror(fr_new, host, u, v, col, wgt, pf, rp, rt, st, en), i1, z1


def upload(ba, m, idd, idz):
    ba.set_window(len(m.fr), m.fr)
    ba.set_points(m.host, m.u, m.v, idd, idz, m.color, m.weights, priorF=m.priorF)
    ba.set_residuals(m.rp, m.rt, m.st, m.en)


# ---------------------------------------------------------------------------------------------------------------------------------
# the pair: the handle that is edited and its twin that is re-uploaded
# ---------------------------------------------------------------------------------------------------------------------------------
class Pair:
    def __init__(self, capi, seq, m, idd, idz, chunk_points=0, max_points=None, bas=None):
        W = seq.W
        self.seq, self.m = seq, m
        if bas is None:
            bas = []
            for _ in range(2):
                b = capi.BA(W["w"], W["h"], max_frames=8, max_points=max_points or len(W["host"]), chunk_points=chunk_points)
                for k in range(seq.nfa):
                    b.upload_frame(k, W["dI"][k])
                upload(b, m, idd, idz)
                bas.append(b)
        self.ba, self.tw = bas
        self.act = None

    def both(self, fn, what):
        r = [fn(b) for b in (self.ba, self.tw)]
        if isinstance(r[0], dict) and "JpJdF" in r[0]:
            # JpJdF is written for residuals that come out IN; elsewhere its buffer holds whatever was there before
            assert np.array_equal(r[0]["newState"], r[1]["newState"]), what
            live = r[0]["newState"] == 0
            r = [dict(o, JpJdF=o["JpJdF"][live]) for o in r]
        if isinstance(r[0], dict):
            assert_same({k: x for k, x in r[0].items() if x is not None}, {k: x for k, x in r[1].items() if x is not None}, what)
        elif isinstance(r[0], tuple):
            for a, b in zip(*r):
                assert np.array_equal(bits(a), bits(b)), what
        elif r[0] is not None:
            assert np.array_equal(bits(r[0]), bits(r[1])), what
        return r[0]

    def prep(self):
        fr = self.m.fr
        adH, adT = self.seq.adjoints(fr)
        for b in (self.ba, self.tw):
            b.set_adjoints(adH, adT)
            b.set_state(*self.seq.state(fr))

    def edit(self, fr_new, point_src, nrt=-1, what=""):
        """dmv_ba_edit_window on ba, the replay re-uploaded to tw"""
        idd, idz = self.both(lambda b: b.get_idepth(), f"{what}: idepth before")
        frame_src = np.array([self.m.fr.index(f) if f in self.m.fr else -1 for f in fr_new], np.int32)
        point_src = np.asarray(point_src, np.int32)
        new, i1, z1 = replay(self.m, idd, idz, list(fr_new), frame_src, point_src, nrt, self.act)
        lc = self.ba.launch_count(), self.tw.launch_count()
        self.ba.edit_window(len(fr_new), list(fr_new), frame_src, point_src, nrt, nres=len(new.rp))
        upload(self.tw, new, i1, z1)
        assert self.ba.launch_count() - lc[0] == 1 and self.tw.launch_count() == lc[1], what
        self.m, self.act = new, None
        return new

    def commit(self, what):
        """apply_res on both; the committed states become the inputs the next linearisation (and edit) reads"""
        for b in (self.ba, self.tw):
            b.apply_res()
        o = self.both(lambda b: b.residual_outputs(), f"{what}: committed residual outputs")
        self.m.st, self.m.en = o["newState"].copy(), o["newEnergy"].copy()

    def check(self, what, seed=0):
        """adjoints + state, then every output of a linearisation, a commit, a resubstitution and two steps, bit for bit"""
        self.prep()
        lc = self.ba.launch_count(), self.tw.launch_count()
        fr, nf = self.m.fr, len(self.m.fr)
        self.both(lambda b: b.linearize(), f"{what}: linearize")
        self.both(lambda b: b.residual_outputs(), f"{what}: residual outputs")
        self.both(lambda b: b.point_outputs(), f"{what}: point outputs")
        for t in range(nf):
            self.both(lambda b: b.target_energies(t), f"{what}: target energies {t}")
        self.both(lambda b: b.get_idepth(), f"{what}: idepth")
        self.commit(what)
        self.both(lambda b: b.accumulate(), f"{what}: accumulate")
        x = np.random.default_rng(seed).normal(0, 1e-4, 8 * nf + 4)
        self.both(lambda b: b.resubstitute(x, apply=False), f"{what}: resubstitute")
        self.both(lambda b: b.gn_step(x, *self.seq.state(fr)), f"{what}: gn_step x")
        self.both(lambda b: b.gn_step(None, *self.seq.state(fr)), f"{what}: gn_step")
        self.both(lambda b: b.target_energies(nf - 1), f"{what}: newest target energies")
        self.both(lambda b: b.get_idepth(), f"{what}: idepth after the steps")
        self.commit(what)
        assert self.ba.launch_count() - lc[0] == self.tw.launch_count() - lc[1], what

    def optimize(self, its, what):
        """its Gauss-Newton iterations with the host solve (damped Schur system), the same x on both"""
        fr, nf = self.m.fr, len(self.m.fr)
        self.prep()
        self.both(lambda b: b.linearize(), f"{what}: linearize")
        self.commit(what)
        for i in range(its):
            s = self.both(lambda b: b.accumulate(), f"{what}: accumulate {i}")
            H, g = s["HA"] - s["Hsc"], s["bA"] - s["bsc"]
            x = -np.linalg.solve(H + np.diag(np.diag(H) * 0.1 + 1e-3), g)
            self.both(lambda b: b.gn_step(x, *self.seq.state(fr)), f"{what}: gn_step {i}")
            self.commit(f"{what} {i}")

    def activate(self, P, host, minObs=1):
        """dmv_ba_activate_points on both (the same entries); the entries become point_src's -1 - k"""
        st, idp, rs = self.both(lambda b: b.activate_points(host, P, self.seq.rt(self.m.fr), minObs), "activation")
        self.act = dict(host=np.asarray(host, np.int32), u=P["u"], v=P["v"], color=P["color"].reshape(-1, 8), weights=P["weights"].reshape(-1, 8),
                        idepth=idp, rs=rs, status=st)
        return st

    def close(self):
        close(self.ba, self.tw)


def new_order(m, keep, fr_new, act=None, ks=()):
    """point_src of carried points `keep` and activation entries ks, ordered by new host (activated after the carried ones of a host)"""
    pos = {f: i for i, f in enumerate(fr_new)}
    items = [(pos[m.fr[m.host[s]]], 0, int(s)) for s in keep] + [(pos[m.fr[act["host"][k]]], 1, int(k)) for k in ks]
    items.sort()
    return np.array([s if kind == 0 else -1 - s for _, kind, s in items], np.int32)


def immature(orc, seq, m, rng, n, frames):
    """n immature points hosted on window frames `frames` (host index), depth intervals around the scene's"""
    W = seq.W
    w, h = W["w"], W["h"]
    host = np.sort(rng.choice(frames, n)).astype(np.int32)
    u, v = rng.integers(10, w - 10, n), rng.integers(10, h - 10, n)
    parts = [orc.ip_init(W["dI"][m.fr[f]], w, h, u[host == f], v[host == f]) for f in sorted(set(host.tolist()))]
    P = {k: np.concatenate([p[k] for p in parts]) for k in parts[0]}
    idt = (0.5 * (1 + 0.02 * rng.standard_normal(n))).astype(np.float32)
    wide = rng.random(n) < 0.5
    P["idepth_min"] = (idt * np.where(wide, 0.7, 0.97)).astype(np.float32)
    P["idepth_max"] = (idt * np.where(wide, 1.4, 1.03)).astype(np.float32)
    return host, P


def sequence(orc, synth, seed, npts=1500, nf=8):
    W = edge_window(synth, dict(nf=nf, npts=npts, seed=seed, trans=0.06, rot=0.01))
    return Seq(W, orc.Window(W))


def pair(capi, seq, fr, **kw):
    m, idd, idz = window_from(seq.W, fr)
    return Pair(capi, seq, m, idd, idz, **kw)


# ---------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("chunk_points", [0, 16, 32])
def test_erase(capi, gpu, orc, synth, chunk_points):
    """the first point, the last, runs, a whole host's points, and none (the identity edit), each followed by the whole comparison"""
    seq = sequence(orc, synth, 11)
    pr = pair(capi, seq, range(7), chunk_points=chunk_points)
    pr.check("start")
    fr = pr.m.fr
    n = lambda: len(pr.m.host)   # noqa: E731
    for what, drop in (("first", [0]), ("last", [n() - 1]), ("runs", list(range(100, 180)) + [400, 401, 402, 900]),
                       ("host 2", np.nonzero(pr.m.host == 2)[0]), ("identity", [])):
        keep = np.setdiff1d(np.arange(n()), drop)
        pr.edit(fr, keep, what=what)
        pr.check(what)
    pr.close()


@pytest.mark.gpu
def test_frames(capi, gpu, orc, synth):
    """the oldest frame leaves, a frame joins with new_res_target (up to nf = 8), a middle frame leaves; and the first-keyframes window"""
    seq = sequence(orc, synth, 12)
    pr = pair(capi, seq, range(7))
    pr.check("start")
    for what, fr_new, nrt in (("oldest leaves", [1, 2, 3, 4, 5, 6], -1), ("7 joins", [1, 2, 3, 4, 5, 6, 7], 6),
                              ("0 joins: nf = 8", [1, 2, 3, 4, 5, 6, 7, 0], 7), ("middle leaves", [1, 2, 4, 5, 6, 7, 0], -1),
                              ("joins with no residuals", [1, 2, 4, 5, 6, 7, 0, 3], -1)):
        keep = [p for p in range(len(pr.m.host)) if pr.m.fr[pr.m.host[p]] in fr_new]
        pr.edit(fr_new, keep, nrt, what=what)
        pr.check(what)
    pr.close()
    pr = pair(capi, seq, [0, 1])
    pr.edit([0, 1], np.arange(len(pr.m.host)), what="first keyframes: identity")
    pr.check("first keyframes")
    pr.edit([0, 1, 2], np.arange(len(pr.m.host)), 2, what="first keyframes: 2 joins")
    pr.check("first keyframes + 1")
    pr.close()


@pytest.mark.gpu
def test_carried_state(capi, gpu, orc, synth):
    """the states an edit carries: the inputs of a fresh handle (OOB / OUTLIER with energies, idepth_zero apart from idepth), a tentative
    linearisation only (discarded), a committed one (aliased idepth_zero after a step), a committed one under a tentative one with other
    states, after reset_oob, drop_residuals and marginalize_points"""
    seq = sequence(orc, synth, 13)
    pr = pair(capi, seq, range(7))
    assert np.isin(pr.m.st, [1, 2]).any() and (pr.m.en != 0).any()
    n = len(pr.m.host)
    pr.edit(pr.m.fr, np.setdiff1d(np.arange(n), [3, 4, 50]), what="fresh")
    pr.prep()
    pr.both(lambda b: b.linearize(), "tentative")
    pr.edit(pr.m.fr, np.arange(len(pr.m.host) - 1), what="tentative only")
    pr.check("after tentative")             # ends committed, after a step
    pr.edit(pr.m.fr, np.arange(1, len(pr.m.host)), what="committed")
    pr.check("after committed")
    # a committed linearisation under a tentative one with other states: the edit carries the committed states
    # (a linearisation reads only which inputs are OOB, and their energies: a rejected step, as FullSystem::optimize's loadSateBackup
    # undoes it, leaves OOB residuals in the tentative states that the restored depths would not make)
    x = np.random.default_rng(13).normal(0, 5e-2, 8 * len(pr.m.fr) + 4)
    for b in (pr.ba, pr.tw):
        b.backup_points()
    pr.both(lambda b: b.gn_step(x, *seq.state(pr.m.fr)), "large step")
    o = pr.both(lambda b: b.residual_outputs(), "tentative outputs")
    assert ((o["newState"] == 1) != (pr.m.st == 1)).any()
    for b in (pr.ba, pr.tw):
        b.restore_points()
    pr.edit(pr.m.fr, np.arange(len(pr.m.host) - 2), what="committed under a tentative")
    pr.check("after committed under a tentative")
    for b in (pr.ba, pr.tw):
        b.reset_oob()
    pr.m.st[:], pr.m.en[:] = 0, 0
    pr.edit(pr.m.fr, np.arange(len(pr.m.host)), what="reset_oob")
    pr.check("after reset_oob")
    drop = np.arange(0, len(pr.m.rp), 7).astype(np.int32)
    for b in (pr.ba, pr.tw):
        b.drop_residuals(drop)
    keep = np.setdiff1d(np.arange(len(pr.m.rp)), drop)
    for k in ("rp", "rt", "st", "en"):
        setattr(pr.m, k, getattr(pr.m, k)[keep])
    pr.edit(pr.m.fr, np.arange(len(pr.m.host)), what="drop_residuals")
    pr.check("after drop_residuals")
    pr.prep()
    pr.both(lambda b: b.linearize(), "linearize before marginalisation")
    pr.commit("before marginalisation")
    marg = np.nonzero(pr.m.host == 1)[0][::2].astype(np.int32)
    pr.both(lambda b: b.marginalize_points(marg, seq.adDelta(pr.m.fr), seq.cD), "marginalize_points")
    pr.edit(pr.m.fr, np.setdiff1d(np.arange(len(pr.m.host)), marg), what="marginalised points erased")
    pr.check("after marginalize_points")
    pr.close()


@pytest.mark.gpu
def test_activated_points(capi, gpu, orc, synth):
    """activated points inserted mid-list on older hosts (only status-1 entries named, from an activation with every status); then every
    kind in one call: a frame leaves, a frame joins, points are erased and activated points inserted"""
    seq = sequence(orc, synth, 14)
    rng = np.random.default_rng(14)
    pr = pair(capi, seq, range(7), max_points=2400)
    pr.check("start")
    host, P = immature(orc, seq, pr.m, rng, 400, [0, 1, 2, 3, 4, 5])
    st = pr.activate(P, host)
    assert (st == 1).any() and (st != 1).any(), np.unique(st)
    ks = np.nonzero(st == 1)[0][::2]
    pr.edit(pr.m.fr, new_order(pr.m, range(len(pr.m.host)), pr.m.fr, pr.act, ks), what="insert")
    pr.check("after insert")
    host, P = immature(orc, seq, pr.m, rng, 300, [1, 2, 3, 4, 5, 6])
    st = pr.activate(P, host)
    fr_new = [1, 2, 3, 4, 5, 6, 7]
    keep = [p for p in range(len(pr.m.host)) if pr.m.host[p] != 0 and p % 5 != 2]
    ks = [k for k in np.nonzero(st == 1)[0] if k % 3 != 1]
    pr.edit(fr_new, new_order(pr.m, keep, fr_new, pr.act, ks), 6, what="all kinds")
    pr.check("after all kinds")
    pr.close()


@pytest.mark.gpu
def test_activate_store(capi, gpu, orc, synth):
    """entries of dmv_ba_activate_store inserted (the twin ran the five steps on host arrays), with points of one host erased in the same
    call"""
    win = Win(capi, synth, orc, 21, nf=7, npts=2000)
    slot = [5, 2, 9, 0, 3, 7, -1]
    fill(win, slot, 600)
    for t in (6, 5):
        win.trace(t)
    copies = {k: dict(P) for k, P in win.copies.items()}
    r, _ = win.turnover(slot, mad=2.0, what="turnover")
    seq = Seq(win.W, win.ow)
    m, idd, idz = window_from(win.W, range(7))
    pr = Pair(capi, seq, m, idd, idz, bas=win.bas)
    of, oi = r["opt_frame"], r["opt_index"]
    pick = lambda key, w: np.array([copies[slot[f]][key].reshape(len(copies[slot[f]]["u"]), -1)[i] for f, i in zip(of, oi)]).reshape(len(of), w)  # noqa: E731
    pr.act = dict(host=of, u=pick("u", 1)[:, 0], v=pick("v", 1)[:, 0], color=pick("color", 8), weights=pick("weights", 8), idepth=r["idepth"],
                  rs=r["res_state"], status=r["status"])
    keep = np.nonzero(m.host != 1)[0]
    ks = np.nonzero(r["status"] == 1)[0][: len(m.host) - len(keep) - 1]   # within the handles' max_points
    assert len(ks) > 0
    pr.edit(m.fr, new_order(m, keep, m.fr, pr.act, ks), what="store entries")
    pr.check("after store entries")
    win.close()


@pytest.mark.gpu
def test_chunk_threshold(capi, gpu, orc, synth):
    """an edit that takes the window below 16 x SMs points (P 32 -> 16) and one that takes it back above (16 -> 32)"""
    import torch
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    T = 16 * sms
    seq = sequence(orc, synth, 15, npts=T + 200)
    rng = np.random.default_rng(15)
    pr = pair(capi, seq, range(7), max_points=T + 800)
    n = len(pr.m.host)
    assert n > T, (n, T)
    pr.check("above")
    keep = np.arange(n)[: T - 30] if n > T - 30 else np.arange(n)
    pr.edit(pr.m.fr, keep, what="down")
    pr.check("below")
    host, P = immature(orc, seq, pr.m, rng, 600, [0, 1, 2, 3, 4, 5])
    st = pr.activate(P, host)
    ks = np.nonzero(st == 1)[0]
    assert len(ks) > 40, len(ks)
    pr.edit(pr.m.fr, new_order(pr.m, range(len(pr.m.host)), pr.m.fr, pr.act, ks), what="up")
    assert len(pr.m.host) > T
    pr.check("above again")
    pr.close()


@pytest.mark.gpu
def test_keyframe_cycles(capi, gpu, orc, synth):
    """three keyframes of makeKeyFrame's window flow, each step against the re-upload: the new frame joins (edit 1), activation and the
    inserting edit, a few Gauss-Newton steps with the host solve, marginalisation and the erasing edit, the oldest frame leaves"""
    seq = sequence(orc, synth, 16, npts=1800)
    rng = np.random.default_rng(16)
    pr = pair(capi, seq, [0, 1, 2, 3], max_points=2600)
    pr.optimize(2, "start")
    for kf in (4, 5, 6):
        fr_new = pr.m.fr + [kf]
        pr.edit(fr_new, np.arange(len(pr.m.host)), len(fr_new) - 1, what=f"kf {kf}: joins")
        pr.prep()
        host, P = immature(orc, seq, pr.m, rng, 250, list(range(len(fr_new) - 1)))
        st = pr.activate(P, host)
        ks = np.nonzero(st == 1)[0]
        pr.edit(pr.m.fr, new_order(pr.m, range(len(pr.m.host)), pr.m.fr, pr.act, ks), what=f"kf {kf}: insert")
        pr.optimize(3, f"kf {kf}")
        marg = np.nonzero(pr.m.host == 0)[0][::3].astype(np.int32)
        pr.both(lambda b: b.marginalize_points(marg, seq.adDelta(pr.m.fr), seq.cD), f"kf {kf}: marginalize_points")
        pr.edit(pr.m.fr, np.setdiff1d(np.arange(len(pr.m.host)), marg), what=f"kf {kf}: erase")
        if len(pr.m.fr) > 4:
            fr_new = pr.m.fr[1:]
            keep = np.nonzero(pr.m.host != 0)[0]
            pr.edit(fr_new, keep, what=f"kf {kf}: oldest leaves")
        pr.check(f"kf {kf}")
    pr.close()


@pytest.mark.gpu
def test_batch_after_edit(capi, gpu, orc, synth):
    """an edited handle in a dmv_ba_batch steps as its re-uploaded twin does"""
    seq = sequence(orc, synth, 17)
    pr = pair(capi, seq, range(7))
    pr.check("start")
    fr_new = [1, 2, 3, 4, 5, 6, 7]
    pr.edit(fr_new, np.nonzero(pr.m.host != 0)[0], 6, what="edit")
    pr.prep()
    st = [seq.state(fr_new)]
    r = [capi.BABatch([b]).gn_step(None, st) for b in (pr.ba, pr.tw)]
    assert_same(r[0][0], r[1][0], "batched step")
    pr.both(lambda b: b.residual_outputs(), "batched residual outputs")
    pr.close()


def nrt_refusal(m, nrt):
    """the first of the identity edit's points whose new_res_target residual is refused, in the call's order of checks"""
    has = set(zip(m.rp.tolist(), m.rt.tolist()))
    for j in range(len(m.host)):
        if m.host[j] == nrt:
            return f"new_res_target {nrt} is the host frame of point {j}"
        if (j, nrt) in has:
            return f"new_res_target {nrt}: point {j} already has a residual into it"
    raise AssertionError("no refusal")


def _raw_edit(capi, ba, nf, slots, frame_src, point_src, nrt=-1):
    import ctypes as C
    L = capi.lib()
    arrs = [None if a is None else np.ascontiguousarray(a, np.int32) for a in (slots, frame_src, point_src)]
    a = capi.BAEditArgs(nf, *(None if x is None else x.ctypes.data for x in arrs[:2]), 0 if arrs[2] is None else len(arrs[2]),
                        None if arrs[2] is None else arrs[2].ctypes.data, nrt)
    rc = L.dmv_ba_edit_window(ba.h if ba is not None else None, C.byref(a))
    return rc, L.dmv_last_error().decode()


@pytest.mark.gpu
def test_refusals(capi, gpu, orc, synth):
    """every refusal with its message; the handle is unchanged afterwards (its linearisation equals the untouched twin's, launch counts
    and the pinned outputs of the last linearisation too)"""
    import ctypes as C
    seq = sequence(orc, synth, 18, npts=600)
    rng = np.random.default_rng(18)
    pr = pair(capi, seq, range(5), max_points=700)
    pr.check("start")
    host, P = immature(orc, seq, pr.m, rng, 120, [0, 1, 2, 3])
    st = pr.activate(P, host)
    one, other = int(np.nonzero(st == 1)[0][0]), int(np.nonzero(st != 1)[0][0])
    n, m = len(pr.m.host), pr.m
    ident = np.arange(n)
    fr = list(range(5))
    fs = np.arange(5)
    ins = new_order(m, ident, fr, pr.act, [one])
    at = int(np.nonzero(ins == -1 - one)[0][0])
    cases = [
        ((5, fr, fs, ident, 6), DMV_ERR_INVALID, "new_res_target = 6: expected -1 to 4"),
        ((1, fr, fs, ident), DMV_ERR_INVALID, "nf out of range"),
        ((9, list(range(9)), np.arange(9), ident), DMV_ERR_INVALID, "nf out of range"),
        ((5, [0, 1, 2, 3, 8], fs, ident), DMV_ERR_INVALID, "slot out of range"),
        ((5, fr, [0, 1, 2, 3, 5], ident), DMV_ERR_INVALID, "frame_src[4] = 5: expected -1 to 4"),
        ((5, fr, [0, 1, 2, 3, -2], ident), DMV_ERR_INVALID, "frame_src[4] = -2: expected -1 to 4"),
        ((5, fr, [0, 1, 2, 3, 1], ident), DMV_ERR_INVALID, "frame_src[1] and frame_src[4] are both 1"),
        ((5, fr, fs, np.zeros(0, np.int32)), DMV_ERR_INVALID, "npts = 0: expected 1 to 700"),
        ((5, fr, fs, np.arange(701) % n), DMV_ERR_INVALID, "npts = 701: expected 1 to 700"),
        ((5, fr, fs, np.r_[ident[:-1], n]), DMV_ERR_INVALID, f"point_src[{n - 1}] = {n}: the window has {n} points"),
        ((5, fr, fs, np.r_[ident[:-1], 0]), DMV_ERR_INVALID, f"point_src[0] and point_src[{n - 1}] are both 0"),
        ((5, fr, fs, np.r_[ident, -1 - len(st)]), DMV_ERR_INVALID, f"point_src[{n}] = {-1 - len(st)}: the last activation has {len(st)} entries"),
        ((5, fr, fs, np.r_[ident, -1 - other]), DMV_ERR_INVALID, f"point_src[{n}] = {-1 - other}: activation entry {other} has status {st[other]}, not 1"),
        ((5, fr, fs, np.insert(ins, at, -1 - one)), DMV_ERR_INVALID, f"point_src[{at}] and point_src[{at + 1}] are both {-1 - one}"),
        ((4, [1, 2, 3, 4], [1, 2, 3, 4], ident), DMV_ERR_INVALID, "point 0: its host frame 0 leaves the window"),
        ((5, fr, fs, ident[::-1]), DMV_ERR_INVALID, "points must be ordered by host frame (EnergyFunctional::allPoints order)"),
        ((5, fr, fs, ident, 0), DMV_ERR_INVALID, "new_res_target 0 is the host frame of point 0"),
        ((5, fr, fs, ident, 3), DMV_ERR_INVALID, nrt_refusal(m, 3)),
    ]
    lc = pr.ba.launch_count()
    for args, code, msg in cases:
        rc, err = _raw_edit(capi, pr.ba, *args)
        assert (rc, err) == (code, msg), (args[0], rc, err, msg)
    L = capi.lib()
    a = capi.BAEditArgs(5, None, None, 1, None, -1)
    assert L.dmv_ba_edit_window(None, C.byref(a)) == DMV_ERR_INVALID and L.dmv_last_error().decode() == "null argument"
    assert L.dmv_ba_edit_window(pr.ba.h, None) == DMV_ERR_INVALID
    rc, err = _raw_edit(capi, pr.ba, 5, fr, None, ident)
    assert (rc, err) == (DMV_ERR_INVALID, "null argument")
    assert pr.ba.launch_count() == lc
    # unchanged: the pinned newest-frame energies and the per-residual outputs of the last linearisation, then a linearisation
    pr.both(lambda b: b.target_energies(len(fr) - 1), "after refusals: newest energies")
    pr.both(lambda b: b.residual_outputs(), "after refusals: residual outputs")
    pr.both(lambda b: b.linearize(), "after refusals: linearize")
    pr.both(lambda b: b.residual_outputs(), "after refusals: residual outputs of the linearisation")
    pr.edit(fr, new_order(m, ident, fr, pr.act, [one]), what="accepted after the refusals")
    pr.check("after the refusals")
    # an edit consumes the activation; a window without residuals set refuses
    rc, err = _raw_edit(capi, pr.ba, 5, fr, fs, np.r_[np.arange(len(pr.m.host)), -1])
    assert (rc, err) == (DMV_ERR_INVALID, f"point_src[{len(pr.m.host)}] = -1: no activation ran on this window")
    b = pr.tw
    b.set_window(5, fr)
    rc, err = _raw_edit(capi, b, 5, fr, fs, [0])
    assert (rc, err) == (DMV_ERR_STATE, "dmv_ba_set_window + dmv_ba_set_points + dmv_ba_set_residuals first")
    b.set_points(m.host, m.u, m.v, np.ones(n, np.float32), None, m.color, m.weights)
    rc, err = _raw_edit(capi, b, 5, fr, fs, [0])
    assert (rc, err) == (DMV_ERR_STATE, "dmv_ba_set_window + dmv_ba_set_points + dmv_ba_set_residuals first")
    pr.close()


def test_binding_declares_edit_window(capi):
    """the binding knows the entry point and its argument block (no device needed)"""
    assert "dmv_ba_edit_window" in capi.SYMBOLS
    names = [f[0] for f in capi.BAEditArgs._fields_]
    assert names == ["nf", "slots", "frame_src", "npts", "point_src", "new_res_target"]
    with pytest.raises(TypeError):
        capi.BA.edit_window(None, 2, None, [0, 1], [0])   # nres is keyword-only and required
