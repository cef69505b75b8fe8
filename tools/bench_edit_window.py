"""One change of the BA window's membership at a keyframe: the re-upload path (dmv_ba_get_idepth + dmv_ba_get_residual_outputs of the
states + dmv_ba_set_window + dmv_ba_set_points + dmv_ba_set_residuals, with the new lists built by numpy glue issued from Python) against
one dmv_ba_edit_window.
Edit kinds: erase (5 % of the points leave), frame leaves (the oldest, with its points), frame joins (with every old point's residual into it)
and insert (the status-1 entries of an activation of 300 immature points, staged by dmv_ba_activate_points).  Windows: the C3-like window
(7 keyframes, 2000 points, 640x480) and one past the P = 32 threshold (16 x SMs + 900 points).  Before each call both handles are reset
outside the timing to the same window with a committed linearisation (and, for insert, the same activation).  The arms alternate
(benchkit.alternate).  Reported per arm: median / p10 / p90 wall time per edit, the bytes each way computed from the layouts, and the
synchronisations per edit.  Outside the timed loop both arms' handles are linearised and compared bit for bit (idepth, energies, residual
outputs); the run exits non-zero if any bit differs.  The card's name, power limit and maximum SM clock are read in the same run.  Prints
one JSON line and writes it to --out."""
import argparse
import json
import os
import types

import numpy as np

import benchkit as K

MAXF = 8


def glue(m, idd, idz, st, en, frame_src, point_src, nrt, act):
    """the header's rules in vectorised numpy: set_points / set_residuals arguments of the new window"""
    nf0, np0 = len(m.fr), len(m.host)
    fnew = -np.ones(nf0, np.int64)
    fnew[frame_src[frame_src >= 0]] = np.nonzero(frame_src >= 0)[0]
    car = point_src >= 0
    cs, ak = point_src[car], -1 - point_src[~car]
    pnew = -np.ones(np0, np.int64)
    pnew[cs] = np.nonzero(car)[0]
    n = len(point_src)
    host = np.zeros(n, np.int32)
    host[car] = fnew[m.host[cs]]
    u, v, i1, z1, pf = (np.zeros(n, np.float32) for _ in range(5))
    col, wgt = np.zeros((n, 8), np.float32), np.zeros((n, 8), np.float32)
    u[car], v[car], i1[car], z1[car], pf[car], col[car], wgt[car] = m.u[cs], m.v[cs], idd[cs], idz[cs], m.priorF[cs], m.color[cs], m.weights[cs]
    if len(ak):
        host[~car] = fnew[act["host"][ak]]
        u[~car], v[~car], i1[~car], z1[~car], col[~car], wgt[~car] = act["u"][ak], act["v"][ak], act["idepth"][ak], act["idepth"][ak], act["color"][ak], act["weights"][ak]
    keep = (pnew[m.rp] >= 0) & (fnew[m.rt] >= 0)
    rp, rt, rs, re = [pnew[m.rp[keep]]], [fnew[m.rt[keep]]], [st[keep]], [en[keep]]
    if nrt >= 0:
        j = np.nonzero(car)[0]
        rp.append(j); rt.append(np.full(len(j), nrt)); rs.append(np.zeros(len(j), np.int32)); re.append(np.zeros(len(j), np.float32))
    if len(ak):
        ok = (frame_src[None, :] >= 0) & (act["rs"][ak][:, np.maximum(frame_src, 0)] == 0)
        jj, tt = np.nonzero(ok)
        rp.append(np.nonzero(~car)[0][jj]); rt.append(tt); rs.append(np.zeros(len(jj), np.int32)); re.append(np.zeros(len(jj), np.float32))
    cat = lambda a, t: np.ascontiguousarray(np.concatenate(a), t)  # noqa: E731
    return host, u, v, i1, z1, col, wgt, pf, cat(rp, np.int32), cat(rt, np.int32), cat(rs, np.int32), cat(re, np.float32)


def traffic(np0, npts, nres0, ncarry, mp):
    """bytes up / down and synchronisations of both arms per edit (ba_api.cu, ba_edit.cu), without the phase-D table both arms upload"""
    ns = MAXF * mp
    reup = dict(up_bytes=84 * npts + 5 * ns, down_bytes=8 * np0 + 5 * ns, syncs=7)
    edit = dict(up_bytes=8 * npts, down_bytes=5 * ncarry, syncs=1)
    return reup, edit


def workload(capi, orc, synth, T, npts, warmup, reps, seed):
    L = capi.lib()
    seq = T.sequence(orc, synth, seed, npts=npts)
    rng = np.random.default_rng(seed)
    out = {}
    kinds = {
        "erase": (list(range(7)), lambda m: (m.fr, np.sort(rng.permutation(len(m.host))[: int(0.95 * len(m.host))]), -1)),
        "frame_leaves": (list(range(7)), lambda m: (m.fr[1:], np.nonzero(m.host != 0)[0], -1)),
        "frame_joins": (list(range(6)), lambda m: (m.fr + [6], np.arange(len(m.host)), 6)),
        "insert": (list(range(7)), None),
    }
    for kind, (fr0, make) in kinds.items():
        m0, idd0, idz0 = T.window_from(seq.W, fr0)
        pr = T.Pair(capi, seq, m0, idd0, idz0, max_points=npts + 400)
        imm = T.immature(orc, seq, m0, rng, 300, list(range(len(fr0) - 1))) if kind == "insert" else None

        def reset(b):
            T.upload(b, m0, idd0, idz0)
            adH, adT = seq.adjoints(fr0)
            b.set_adjoints(adH, adT)
            b.set_state(*seq.state(fr0))
            b.linearize()
            b.apply_res()
            if imm is not None:
                return b.activate_points(imm[0], imm[1], seq.rt(fr0))
            return None

        r = reset(pr.ba)
        act = None
        if kind == "insert":
            st, idp, rs = r
            P = imm[1]
            act = dict(host=imm[0], u=P["u"], v=P["v"], color=P["color"].reshape(-1, 8), weights=P["weights"].reshape(-1, 8), idepth=idp, rs=rs)
            fr_new, point_src, nrt = fr0, T.new_order(m0, range(len(m0.host)), fr0, act, np.nonzero(st == 1)[0]), -1
        else:
            fr_new, point_src, nrt = make(m0)
        fr_new, point_src = list(fr_new), np.asarray(point_src, np.int32)
        frame_src = np.array([fr0.index(f) if f in fr0 else -1 for f in fr_new], np.int32)
        nres0 = len(m0.rp)
        stb, enb = np.zeros(nres0, np.int32), np.zeros(nres0, np.float32)
        new_nres = [0]

        def reupload():
            b = pr.tw
            idd, idz = b.get_idepth()
            rc = L.dmv_ba_get_residual_outputs(b.h, stb.ctypes.data, enb.ctypes.data, None, None, None)
            if rc:
                return rc
            host, u, v, i1, z1, col, wgt, pf, rp, rt, rs_, re = glue(m0, idd, idz, stb, enb, frame_src, point_src, nrt, act)
            b.set_window(len(fr_new), fr_new)
            b.set_points(host, u, v, i1, z1, col, wgt, priorF=pf)
            b.set_residuals(rp, rt, rs_, re)
            new_nres[0] = len(rp)
            return 0

        def edit():
            pr.ba.edit_window(len(fr_new), fr_new, frame_src, point_src, nrt, nres=new_nres[0])
            return 0

        reset(pr.tw)
        reupload()
        edit()
        check(pr, seq, fr_new, f"{kind} {npts}")
        t = K.alternate({"reupload": reupload, "edit_window": edit}, warmup, reps, f"{kind} {npts}", {"reupload": L, "edit_window": L},
                        resets={"reupload": lambda: reset(pr.tw), "edit_window": lambda: reset(pr.ba)})
        check(pr, seq, fr_new, f"{kind} {npts} after the timed loop")
        car = point_src[point_src >= 0]
        keepc = np.isin(m0.rp, car) & np.isin(m0.rt, frame_src[frame_src >= 0])
        s_re, s_ed = traffic(len(m0.host), len(point_src), nres0, int(keepc.sum()), (npts + 400 + 31) // 32 * 32)
        out[kind] = dict(points_before=len(m0.host), points_after=len(point_src), residuals_before=nres0, residuals_after=new_nres[0],
                         reupload=dict(K.stats(t["reupload"]), **s_re), edit_window=dict(K.stats(t["edit_window"]), **s_ed))
        out[kind]["ratio_of_medians"] = out[kind]["edit_window"]["median_ms"] / out[kind]["reupload"]["median_ms"]
        pr.close()
    return out


def check(pr, seq, fr, what):
    """both arms' handles: idepth, then a linearisation and its outputs, bit for bit"""
    try:
        pr.m = types.SimpleNamespace(fr=list(fr))   # what prep reads; the window's own mirror stays as the resets need it
        pr.both(lambda b: b.get_idepth(), f"{what}: idepth")
        pr.prep()
        pr.both(lambda b: b.linearize(), f"{what}: linearize")
        pr.both(lambda b: b.residual_outputs(), f"{what}: residual outputs")
        pr.both(lambda b: b.point_outputs(), f"{what}: point outputs")
    except AssertionError as e:
        raise SystemExit(f"the arms differ: {e}")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--reps", type=int, default=200)
    ap.add_argument("--out", default=os.path.join(K.ROOT, "records", "h100_edit_window.json"))
    a = ap.parse_args()
    import dmvio_b200.capi as capi
    import dmvio_b200.synth as synth
    from oracle import orc
    import test_gpu_edit_window as T
    K.device_lib("bench_edit_window")
    orc.build()
    import torch
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    res = dict(card=K.card(), sms=sms, warmup=a.warmup, reps=a.reps,
               timing="wall clock per edit, each call ending in a synchronisation; both handles reset outside the timed call to the same window "
                      "with a committed linearisation; the re-upload path is issued from Python with vectorised numpy glue")
    for name, npts, seed in (("c3_640x480", 2000, 31), ("p32_640x480", 16 * sms + 900, 32)):
        res[name] = dict(npts=npts, **workload(capi, orc, synth, T, npts, a.warmup, a.reps, seed))
    res["bit_identical"] = True   # check() exits before here on any differing bit
    line = json.dumps(res)
    print(line)
    os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
    open(a.out, "w").write(line + "\n")


if __name__ == "__main__":
    main()
