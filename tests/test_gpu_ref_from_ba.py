"""GPU tests of the keyframe hand-off from the BA window to the coarse tracker on the device: dmv_ct_set_ref_from_ba
(setCoarseTrackingRef + makeCoarseDepthL0 read straight from the BA handle), its adapter CoarseTracker::setCoarseTrackingRefFromWindow and
the Python bindings.  Windows go through the adapter's makeKeyFrame flow (optimize -> finishOptimize, which deletes the residuals that did
not end IN).  The lists must equal, bit for bit, dmv_ct_make_coarse_depth fed on the host with the same window's downloads and the oracle's
makeCoarseDepthL0."""
import numpy as np
import pytest

from gpu_harness import device_capi  # noqa: F401  (the "capi" fixture: every test that takes it needs the device)

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def hostapi(capi):
    import dmvio_b200.hostapi as h
    return h


def _residuals(host, nf):
    """every point -> every other frame, point-major, target ascending (synth.make_window's rule)"""
    npts = len(host)
    p = np.repeat(np.arange(npts, dtype=np.int32), nf)
    t = np.tile(np.arange(nf, dtype=np.int32), npts)
    keep = t != host[p]
    return p[keep].astype(np.int32), t[keep].astype(np.int32)


def _collide(W, seed, groups=((2, 60), (3, 40), (4, 30)), outliers=0.04):
    """Splat collisions: copies of a point (same host, pixel, pattern) with depths 1e-4 apart land in one pixel of the newest frame, 2-, 3- and
    4-way; the copies sit next to each other, so the point list stays ordered by host.  A few points get a far-off depth: their residuals end
    OUTLIER (or OOB) and the tail deletes them.
    FullSystem::removeOutliers: in every host frame the last `tail` points are 3-way collisions (depths 2e-3 apart) and 3 * tail / 2 points in
    the first half of the host's list have no residual, so the removal's swap-with-back pulls the last copies, in reverse, in front of their
    partners: half of those collisions are folded in reverse order by the reference."""
    rng = np.random.default_rng(seed)
    npts = len(W["host"])
    host = np.asarray(W["host"])
    tail = 8
    last = np.concatenate([np.nonzero(host == h)[0][-tail:] for h in np.unique(host) if np.count_nonzero(host == h) >= 5 * tail])
    mult = np.ones(npts, np.int64)
    pick = rng.choice(np.setdiff1d(np.arange(npts), last), sum(n for _, n in groups), replace=False)
    o = 0
    for k, n in groups:
        mult[pick[o:o + n]] = k
        o += n
    mult[last] = 3
    idx = np.repeat(np.arange(npts), mult)
    rank = np.concatenate([np.arange(m) for m in mult]).astype(np.float32)
    step = np.where(np.isin(idx, last), np.float32(2e-3), np.float32(1e-4)).astype(np.float32)
    for key in ("host", "u", "v", "idepth", "idepth_zero", "color", "weights", "hasDepthPrior"):
        W[key] = np.ascontiguousarray(np.asarray(W[key])[idx])
    W["idepth"] = (W["idepth"] * (1 + step * rank)).astype(np.float32)
    bad = (rng.random(len(idx)) < outliers) & ~np.isin(idx, last)
    W["idepth"][bad] *= np.float32(4.0)
    rp, rt = _residuals(W["host"], W["nf"])
    dead = []
    for h in np.unique(W["host"]):
        ii = np.nonzero(W["host"] == h)[0]
        if np.isin(idx[ii], last).any():
            dead += list(ii[len(ii) // 4 + 2 * np.arange(3 * tail // 2)])
    keep = ~np.isin(rp, dead)
    W["res_point"], W["res_target"] = rp[keep], rt[keep]
    W["no_residuals"] = np.asarray(dead, np.int32)
    return W


def _remove_outliers_order(host, alive):
    """FullSystem::removeOutliers (FullSystemOptimize.cpp:L680-697) replayed on point indices: per host frame, a point without residuals
    leaves by swap-with-back; returns the surviving points in the order makeCoarseDepthL0 then visits them"""
    out = []
    for h in np.unique(host):
        lst = list(np.nonzero(host == h)[0])
        i = 0
        while i < len(lst):
            if not alive[lst[i]]:
                lst[i] = lst[-1]
                lst.pop()
                i -= 1
            i += 1
        out += lst
    return np.asarray(out, np.int64)


def _adapter_window(hostapi, W):
    """WindowBA with the makeKeyFrame bookkeeping (lastResiduals[0] = the residual into the newest keyframe) through optimize -> finishOptimize"""
    hw = hostapi.WindowBA(W)
    nf, npts = W["nf"], len(W["host"])
    fid = np.asarray(W["frameID"])
    t = np.full((npts, 2), -1, np.int32)
    to_newest = np.zeros(npts, bool)
    to_newest[W["res_point"][W["res_target"] == nf - 1]] = True
    t[:, 0] = np.where(to_newest, fid[nf - 1], -1)
    t[:, 1] = np.where(W["host"] != nf - 2, fid[nf - 2], -1)
    hw.set_last_residuals(t, np.zeros((npts, 2), np.int32))
    hw.optimize(3)
    _, removed = hw.finish_optimize()
    return hw, removed


def _planes(ct, w, h, levels):
    return [ct.download_frame(l, w, h) for l in range(levels)]


def _lists(ct, levels):
    return [ct.get_ref(l) for l in range(levels)]


def _assert_lists_equal(a, b, what):
    for l, (x, y) in enumerate(zip(a, b)):
        for k in ("u", "v", "idepth", "color"):
            assert len(x[k]) == len(y[k]), f"{what}: level {l} {k}: {len(x[k])} vs {len(y[k])} entries"
            np.testing.assert_array_equal(np.asarray(x[k], np.float32).view(np.uint32), np.asarray(y[k], np.float32).view(np.uint32),
                                          err_msg=f"{what}: level {l} {k}")


def _fold_order_matters(Ku, Kv, nid, HdiF, w):
    """group sizes of the colliding splats, and how many pixels fold to another float value in reverse input order"""
    pix = np.trunc(Ku + np.float32(0.5)).astype(np.int64) + w * np.trunc(Kv + np.float32(0.5)).astype(np.int64)
    wgt = np.sqrt((1e-3 / (HdiF.astype(np.float64) + 1e-12)).astype(np.float32))
    term = (nid * wgt).astype(np.float32)
    sizes, differ = {}, 0
    for p in np.unique(pix):
        ii = np.nonzero(pix == p)[0]
        if len(ii) < 2:
            continue
        sizes[len(ii)] = sizes.get(len(ii), 0) + 1
        fwd, rev = np.float32(0), np.float32(0)
        for i in ii:
            fwd = np.float32(fwd + term[i])
        for i in ii[::-1]:
            rev = np.float32(rev + term[i])
        fw, rw = np.float32(0), np.float32(0)
        for i in ii:
            fw = np.float32(fw + wgt[i])
        for i in ii[::-1]:
            rw = np.float32(rw + wgt[i])
        differ += int(fwd.view(np.uint32) != rev.view(np.uint32) or fw.view(np.uint32) != rw.view(np.uint32))
    return sizes, differ


SCENES = {
    "c1": dict(nf=2, npts=200, seed=1234, hosts="first"),
    "c3": dict(nf=7, npts=2000, seed=1234),
    "s512_l4": dict(nf=5, npts=1500, w=512, h=512, seed=77, hosts="all", levels=4),
    "s512_l5": dict(nf=6, npts=1800, w=512, h=512, seed=78, hosts="all", levels=5),
}


@pytest.fixture(scope="module", params=list(SCENES), ids=list(SCENES))
def scene(request, synth, hostapi):
    cfg = dict(SCENES[request.param])
    levels = cfg.pop("levels", None)
    W = _collide(synth.make_window(state_noise=1e-3, **cfg), seed=cfg["seed"] + 5)
    levels = levels or synth.pyr_levels(W["w"], W["h"])
    hw, removed = _adapter_window(hostapi, W)
    yield dict(name=request.param, W=W, levels=levels, hw=hw, removed=removed)
    hw.close()


def test_lists_bit_identical(capi, orc, scene):
    """(1) every level's pc_u / pc_v / pc_idepth / pc_color, values and order: the device hand-off == dmv_ct_make_coarse_depth fed on the host
    from the window's downloads and its lastResiduals == the oracle's makeCoarseDepthL0.  The scene has 2-, 3- and 4-way collisions whose
    fold order changes the float result, residuals into the newest frame that the tail deleted, and (c3, 512x512) points of every host."""
    W, L, hw = scene["W"], scene["levels"], scene["hw"]
    w, h, nf = W["w"], W["h"], W["nf"]
    gone = scene["removed"]
    assert np.count_nonzero(W["res_target"][gone] == nf - 1) > 0, "no residual into the newest frame was deleted by the tail"
    if scene["name"] != "c1":
        assert set(np.unique(W["host"])) >= set(range(nf - 1))
    ct = capi.CT(w, h, L, max_points=65536)
    pc_n = ct.set_ref_from_ba(hw.ba_handle())
    got = _lists(ct, L)
    assert [len(x["u"]) for x in got] == list(pc_n[:L]) and pc_n[0] > 100
    planes = _planes(ct, w, h, L)
    Ku, Kv, nid, HdiF, pts = hw.coarse_ref_inputs(with_points=True)
    # the fold order is makeCoarseDepthL0's after removeOutliers: replayed here independently of the adapter
    left = np.setdiff1d(np.arange(len(W["res_point"])), gone)
    rp, rt = W["res_point"][left], W["res_target"][left]
    alive = np.zeros(len(W["host"]), bool)
    alive[rp] = True
    assert not alive[W["no_residuals"]].any() and len(W["no_residuals"]) > 0
    in_newest = np.zeros(len(W["host"]), bool)
    in_newest[rp[rt == nf - 1]] = True
    order = _remove_outliers_order(W["host"], alive)
    np.testing.assert_array_equal(pts, order[in_newest[order]])
    assert np.any(pts != np.sort(pts)), "removeOutliers moved no point that has an IN residual into the newest frame"
    sizes, differ = _fold_order_matters(Ku, Kv, nid, HdiF, w)
    assert all(sizes.get(k, 0) > 0 for k in (2, 3, 4)), sizes
    assert differ > 0, "no collision whose fold order changes the float result: the scene cannot tell the orders apart"
    # (a) host-fed path on the same planes
    ch = capi.CT(w, h, L, max_points=65536)
    for l in range(L):
        ch.upload_new(l, planes[l])
    np.testing.assert_array_equal(ch.make_coarse_depth(Ku, Kv, nid, HdiF)[:L], pc_n[:L])
    _assert_lists_equal(got, _lists(ch, L), "host-fed dmv_ct_make_coarse_depth")
    # (b) the oracle's makeCoarseDepthL0 in the swap-reordered order ...
    oc = orc.CoarseTracker(w, h, W["K"], L)
    oc.make_coarse_depth(Ku, Kv, nid, HdiF, planes)
    _assert_lists_equal(got, [oc.ref_points(l) for l in range(L)], "oracle makeCoarseDepthL0")
    # ... and the order matters on this scene: the oracle fed in the order before removeOutliers gives other lists
    s = np.argsort(pts, kind="stable")
    ob = orc.CoarseTracker(w, h, W["K"], L)
    ob.make_coarse_depth(Ku[s], Kv[s], nid[s], HdiF[s], planes)
    before = [ob.ref_points(l) for l in range(L)]
    assert any(not np.array_equal(g["idepth"].view(np.uint32), b["idepth"].view(np.uint32)) for g, b in zip(got, before)), \
        "the removeOutliers reorder changes no list entry: the scene cannot tell the fold orders apart"
    ct.close(); ch.close()


def test_tracking_after_handoff(capi, synth, scene):
    """(2) dmv_ct_track against the handed-off reference == the same track against the host-built reference"""
    W, L, hw = scene["W"], scene["levels"], scene["hw"]
    w, h = W["w"], W["h"]
    ct, ch = capi.CT(w, h, L, max_points=65536), capi.CT(w, h, L, max_points=65536)
    ct.set_ref_from_ba(hw.ba_handle())
    planes = _planes(ct, w, h, L)
    for l in range(L):
        ch.upload_new(l, planes[l])
    ch.make_coarse_depth(*hw.coarse_ref_inputs())
    new = W["images"][max(0, W["nf"] - 2)]
    for c in (ct, ch):
        for l in range(L):
            c.set_K(l, *synth.level_K(W["K"], l))
        c.upload_new_image(new)
    r1, r2 = ct.track(np.eye(3), np.zeros(3), 0.0, 0.0), ch.track(np.eye(3), np.zeros(3), 0.0, 0.0)
    assert r1["evaluations"] > 0
    for k in r1:
        np.testing.assert_array_equal(r1[k], r2[k], err_msg=k)
    ct.close(); ch.close()


def test_adapter_and_python_path(capi, hostapi, synth, scene):
    """(6) CoarseTracker::setCoarseTrackingRefFromWindow (hostapi) gives the ABI's counts and the same track; a window whose lastResiduals
    disagree with its residuals into the newest frame is refused"""
    W, L, hw = scene["W"], scene["levels"], scene["hw"]
    w, h = W["w"], W["h"]
    if L != synth.pyr_levels(w, h):
        pytest.skip("the adapter's tracker uses the calibration's pyramid depth")
    ct = capi.CT(w, h, L, max_points=65536)
    pc_abi = ct.set_ref_from_ba(hw.ba_handle())
    hc = hostapi.CoarseTracker(w, h, W["K"], L)
    assert hc.set_ref_from_ba(hw, 0.0, 0.0, 1.0) == list(pc_abi[:L])
    new = W["images"][max(0, W["nf"] - 2)]
    for l in range(L):
        ct.set_K(l, *synth.level_K(W["K"], l))
    ct.upload_new_image(new)
    hc.set_new_image(new)
    r1, r2 = ct.track(np.eye(3), np.zeros(3), 0.0, 0.0), hc.track(np.eye(3), np.zeros(3), 0.0, 0.0)
    for k in ("R", "t", "a", "b", "lastResiduals", "flow", "iterations"):
        np.testing.assert_array_equal(r1[k], r2[k], err_msg=k)
    t, s = hw.last_residuals()
    bad = t.copy()
    i = int(np.nonzero(t[:, 0] >= 0)[0][0])
    bad[i, 0] = -1
    hw.set_last_residuals(bad, s)
    with pytest.raises(capi.DmvError, match="lastResiduals"):
        hc.set_ref_from_ba(hw)
    hw.set_last_residuals(t, s)
    assert hc.set_ref_from_ba(hw) == list(pc_abi[:L])
    hc.close(); ct.close()


def _abi_window(capi, hm, W, adopt=None):
    ba = capi.BA(W["w"], W["h"], max_frames=W["nf"], max_points=len(W["host"]))
    for k in range(W["nf"]):
        if adopt is not None and k == W["nf"] - 1:
            ba.adopt_frame(k, adopt)
        else:
            ba.upload_frame(k, W["dI"][k])
    ba.set_window(W["nf"])
    ba.set_points(W["host"], W["u"], W["v"], W["idepth"], W["idepth_zero"], W["color"], W["weights"])
    ba.set_residuals(W["res_point"], W["res_target"])
    ba.set_adjoints(*hm.adjoints(W))
    st = (hm.calib8(W["K"]), hm.precalc_table(W), W["frameEnergyTH"])
    ba.set_state(*st)
    return ba, st


def _host_inputs(capi, ba, host, res_point, res_target, nf):
    """the host path's inputs from the handle's downloads: IN residuals into the newest frame in makeCoarseDepthL0's order (points after
    removeOutliers), with the last solve's HdiF"""
    o = ba.residual_outputs()
    hdi = np.zeros(ba.npts, np.float32)
    capi.check(ba.L.dmv_ba_get_solve_HdiF(ba.h, hdi))
    alive = np.zeros(ba.npts, bool)
    alive[res_point] = True
    res_of = np.full(ba.npts, -1)
    sel = np.nonzero((res_target == nf - 1) & (o["newState"] == 0))[0]
    res_of[res_point[sel]] = sel
    order = _remove_outliers_order(host, alive)
    sel = res_of[order[res_of[order] >= 0]]
    c = o["centerProjectedTo"][sel]
    return c[:, 0].copy(), c[:, 1].copy(), c[:, 2].copy(), hdi[res_point[sel]]


def test_pyramid_from_adopted_frame(capi, synth):
    """(3) every level after the hand-off == what dmv_ct_upload_new_image builds from the keyframe image, the BA slot having been filled by
    dmv_ba_adopt_frame; the tracker that takes the hand-off had another frame resident before"""
    import dmvio_b200.hostmath as hm
    W = synth.make_window(nf=4, npts=600, seed=21)
    w, h, L = W["w"], W["h"], 5
    src = capi.CT(w, h, L)
    src.upload_new_image(W["images"][-1])
    ba, _ = _abi_window(capi, hm, W, adopt=src)
    ba.linearize(); ba.apply_res(); ba.accumulate()
    dst = capi.CT(w, h, L)
    dst.upload_new_image(W["images"][0])
    dst.set_ref_from_ba(ba)
    for l in range(L):
        a, b = dst.download_frame(l, w, h), src.download_frame(l, w, h)
        np.testing.assert_array_equal(a.view(np.uint32), b.view(np.uint32), err_msg=f"level {l}")
    src.close(); dst.close(); ba.close()


def test_stream_order_and_repeat(capi, synth):
    """(4) right behind dmv_ba_gn_step + apply_res + dmv_ba_accumulate (whose HdiF copy is still queued on the BA stream, no synchronisation in
    between) the lists equal the host-fed ones; residuals that did not end IN were dropped first; repeated calls give identical lists"""
    import dmvio_b200.hostmath as hm
    W = _collide(synth.make_window(nf=6, npts=1500, seed=5, hosts="all"), seed=9)
    w, h, nf, L = W["w"], W["h"], W["nf"], 5
    ba, st = _abi_window(capi, hm, W)
    ba.linearize(); ba.apply_res(); ba.accumulate()
    ns = ba.residual_outputs()["newState"]
    drop = np.nonzero(ns != 0)[0].astype(np.int32)
    assert np.count_nonzero(W["res_target"][drop] == nf - 1) > 0
    ba.drop_residuals(drop)
    keep = np.setdiff1d(np.arange(len(ns)), drop)
    rp, rt = W["res_point"][keep], W["res_target"][keep]
    alive = np.zeros(len(W["host"]), bool)
    alive[rp] = True
    assert np.any(_remove_outliers_order(W["host"], alive) != np.nonzero(alive)[0])
    ct = capi.CT(w, h, L, max_points=65536)
    ba.gn_step(np.zeros(8 * nf + 4), *st)
    ba.apply_res()
    ba.accumulate()
    pc_n = ct.set_ref_from_ba(ba)
    first = _lists(ct, L)
    planes = _planes(ct, w, h, L)
    ch = capi.CT(w, h, L, max_points=65536)
    for l in range(L):
        ch.upload_new(l, planes[l])
    np.testing.assert_array_equal(ch.make_coarse_depth(*_host_inputs(capi, ba, W["host"], rp, rt, nf))[:L], pc_n[:L])
    _assert_lists_equal(first, _lists(ch, L), "host-fed after gn_step")
    for _ in range(3):
        np.testing.assert_array_equal(ct.set_ref_from_ba(ba), pc_n)
        _assert_lists_equal(_lists(ct, L), first, "repeated call")
    ct.close(); ch.close(); ba.close()


def test_errors(capi, synth):
    """(5) DMV_ERR_STATE before any accumulate and after dmv_ba_set_points; DMV_ERR_INVALID for another image size; the capacity error of the
    host path; a one-rank peer exchange is not a sharded handle"""
    import dmvio_b200.hostmath as hm
    W = synth.make_window(nf=3, npts=400, seed=3)
    w, h, L = W["w"], W["h"], 4
    ba, _ = _abi_window(capi, hm, W)
    ct = capi.CT(w, h, L)

    def rc_of(fn):
        with pytest.raises(capi.DmvError) as e:
            fn()
        return str(e.value)
    assert "error -4" in rc_of(lambda: ct.set_ref_from_ba(ba))          # nothing linearised
    ba.linearize(); ba.apply_res()
    assert "error -4" in rc_of(lambda: ct.set_ref_from_ba(ba))          # committed, but no accumulate
    ba.accumulate()
    pc_n = ct.set_ref_from_ba(ba)
    ba.set_points(W["host"], W["u"], W["v"], W["idepth"], W["idepth_zero"], W["color"], W["weights"])
    assert "error -4" in rc_of(lambda: ct.set_ref_from_ba(ba))          # the window was re-uploaded: HdiF of the last solve is gone
    ba.set_residuals(W["res_point"], W["res_target"])
    ba.linearize(); ba.apply_res(); ba.accumulate()
    other = capi.CT(w // 2, h // 2, 3)
    assert "error -1" in rc_of(lambda: other.set_ref_from_ba(ba))       # image size mismatch
    small = capi.CT(w, h, L, max_points=int(pc_n[0]) - 1)
    m_dev = rc_of(lambda: small.set_ref_from_ba(ba))
    for l in range(L):
        small.upload_new(l, ct.download_frame(l, w, h))
    m_host = rc_of(lambda: small.make_coarse_depth(*_host_inputs(capi, ba, W["host"], W["res_point"], W["res_target"], W["nf"])))
    assert "error -1" in m_dev and m_dev == m_host and "exceed max_points" in m_dev
    ba.p2p_export()
    ba.p2p_import(1, 0, [ba.p2p_export()])                               # nranks = 1: not sharded
    np.testing.assert_array_equal(ct.set_ref_from_ba(ba), pc_n)
    ct.close(); other.close(); small.close(); ba.close()


def _sharded_worker(rank, world, port, q):
    import os
    import sys
    sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
    import torch.distributed as dist
    import dmvio_b200.capi as capi
    import dmvio_b200.hostmath as hm
    import dmvio_b200.synth as synth
    from dmvio_b200.sharding import shard_window
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    W = synth.make_window(nf=4, npts=801, seed=17)
    S = shard_window(W, rank, world)
    ba = capi.BA(W["w"], W["h"], max_frames=W["nf"], max_points=len(S["host"]), device=rank)
    for k in range(W["nf"]):
        ba.upload_frame(k, S["dI"][k])
    ba.set_window(W["nf"])
    ba.set_points(S["host"], S["u"], S["v"], S["idepth"], S["idepth_zero"], S["color"], S["weights"])
    ba.set_residuals(S["res_point"], S["res_target"])
    ba.set_adjoints(*hm.adjoints(S))
    handles = [None] * world
    dist.all_gather_object(handles, ba.p2p_export())
    ba.p2p_import(world, rank, handles)
    ba.set_state(hm.calib8(S["K"]), hm.precalc_table(S), S["frameEnergyTH"])
    ba.linearize(); ba.apply_res(); ba.accumulate()
    ct = capi.CT(W["w"], W["h"], 4, device=rank)
    try:
        ct.set_ref_from_ba(ba)
        out = "accepted"
    except capi.DmvError as e:
        out = str(e)
    dist.barrier()
    q.put((rank, out))
    ct.close(); ba.close()
    dist.destroy_process_group()


def test_sharded_handle_refused(capi):
    """(5) a sharded handle holds one rank's share of the points: DMV_ERR_STATE on every rank"""
    world = 2
    if capi.lib().dmv_device_count() < world:
        pytest.skip(f"needs {world} GPUs for a sharded BA handle")
    import socket
    import torch.multiprocessing as mp
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_sharded_worker, args=(r, world, port, q)) for r in range(world)]
    try:
        for p in procs:
            p.start()
        res = dict(q.get(timeout=300) for _ in range(world))
        for p in procs:
            p.join(timeout=60)
            assert p.exitcode == 0
    finally:
        for p in procs:
            if p.is_alive():
                p.terminate()
            if p.pid is not None:
                p.join(timeout=30)
    for r in range(world):
        assert "error -4" in res[r] and "sharded" in res[r], res[r]
