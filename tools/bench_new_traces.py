"""Wall time per keyframe of FullSystem::makeNewTraces: dmv_ct_make_new_traces on the resident frame (device path) against the path an integrator
ran before it (read back levels 0-2 with dmv_ct_download_frame, PixelSelector::makeMaps on the CPU — the oracle restatement, built -O3 single-
threaded with the reference's flags — then dmv_ct_init_points for the selected pixels).  Seeded 640x480 and 512x512 keyframes at 4 and 5 levels;
each timed call ends in a synchronise.  Bytes each way come from the shapes and the point counts.  The adversarial stripe frame (every textured
pot-block mixed) gives the worst case of the serial chain, at the default arguments and at potential 1 without recursion; mean_mixed_blocks is
the chain length of the ordinary keyframes (from the CPU restatement).  Prints one JSON line, with the card's name and power limit read in the
same run, and writes it to --out if given.  --profile DIR instead times each kernel of the device path with torch.profiler (a run of its own)
and writes the table to DIR/new_traces_kernels.txt.
    python tools/bench_new_traces.py [--keyframes 40] [--out records/h100_new_traces.json] [--profile DIR]"""
import argparse
import ctypes as C
import json
import os
import time

import numpy as np

import benchkit  # first: it puts the repository root on sys.path
import dmvio_b200.capi as capi  # noqa: E402
from oracle import select as S  # noqa: E402

SHAPES = [(640, 480, 4), (640, 480, 5), (512, 512, 4), (512, 512, 5)]
POINT_BYTES = 4 * (2 + 1 + 8 + 8 + 4 + 1)   # u, v, type, color[8], weights[8], gradH[4], energyTH


def host_path(ct, w, h, pot):
    """download levels 0-2, makeMaps + the raster loop on the CPU, the constructor on the device"""
    pyr = [ct.download_frame(l, w, h) for l in range(3)]
    L = S.orc_lib()
    sf, si = S._settings(None)
    p, mixed, quot = C.c_int(pot), C.c_longlong(0), C.c_float(0)
    m = np.zeros(w * h, np.float32)
    c = lambda a: np.ascontiguousarray(a, np.float32).reshape(-1)
    npt = L.orc_sel_make_maps(w, h, c(pyr[0]), c(pyr[1]), c(pyr[2]), S.identity_B(), sf, si, 1500.0, 1, 1.0, C.byref(p), m, C.byref(mixed), C.byref(quot))
    u = np.zeros(w * h, np.int32); v = np.zeros(w * h, np.int32); t = np.zeros(w * h, np.float32)
    n = L.orc_sel_trace_pixels(w, h, m, u, v, t)
    P = ct.init_points(u[:n], v[:n])
    ok = P["ok"].astype(bool)
    pts = dict(u=u[:n][ok], v=v[:n][ok], type=t[:n][ok], color=P["color"][ok], weights=P["weights"][ok], gradH=P["gradH"][ok], energyTH=P["energyTH"][ok])
    return dict(points=pts, numPointsTotal=int(npt), potential=p.value), n, int(mixed.value)


def same(a, b):
    return (a["numPointsTotal"] == b["numPointsTotal"] and a["potential"] == b["potential"]
            and all(np.array_equal(np.asarray(a["points"][k], np.float32).view(np.uint32), np.asarray(b["points"][k], np.float32).view(np.uint32))
                    for k in S.POINT_KEYS))


def profile(outdir):
    import torch
    from torch.profiler import ProfilerActivity
    w, h, lv = 640, 480, 5
    imgs = [S.image("tex", w, h, 100 + k) for k in range(1, 11)]
    ct = capi.CT(w, h, lv)
    ct.upload_new_image(imgs[0])
    ct.make_new_traces(3)
    with torch.profiler.profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        for img in imgs:
            ct.upload_new_image(img)
            ct.make_new_traces(3)
    ct.close()
    table = prof.key_averages().table(sort_by="cuda_time_total", row_limit=40)
    os.makedirs(outdir, exist_ok=True)
    open(os.path.join(outdir, "new_traces_kernels.txt"), "w").write(benchkit.card() + "\n" + table + "\n")
    print(table)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--keyframes", type=int, default=40)
    ap.add_argument("--out", default=None)
    ap.add_argument("--profile", default=None)
    a = ap.parse_args()
    benchkit.device_lib("bench_new_traces")
    if a.profile:
        return profile(a.profile)
    res = dict(card=benchkit.card(), keyframes=a.keyframes, density=1500, shapes=[])
    identical = True
    for w, h, lv in SHAPES:
        imgs = [S.image("tex" if k % 3 else "high", w, h, 100 + k) for k in range(a.keyframes)]
        ct = capi.CT(w, h, lv)
        ct.upload_new_image(imgs[0])
        ct.make_new_traces(3)          # warm-up: scratch, random pattern, modules
        host_path(ct, w, h, 3)
        nmixed = 0
        t_dev = t_host = 0.0
        pot_d = pot_h = 3
        npts = ncand = 0
        for img in imgs:
            ct.upload_new_image(img)
            ct.download_frame(2, w, h)  # the upload has landed (synchronises the stream)
            t0 = time.perf_counter()
            g = ct.make_new_traces(pot_d)
            t1 = time.perf_counter()
            r, n, mx = host_path(ct, w, h, pot_h)
            t2 = time.perf_counter()
            t_dev += t1 - t0
            t_host += t2 - t1
            identical &= same(g, r)
            pot_d, pot_h = g["potential"], r["potential"]
            npts += len(g["points"]["u"])
            ncand += n
            nmixed += mx
        K = a.keyframes
        res["shapes"].append(dict(w=w, h=h, levels=lv, device_ms=1e3 * t_dev / K, host_path_ms=1e3 * t_host / K, mean_points=npts / K, mean_mixed_blocks=nmixed / K,
                                  d2h_bytes_device=int(POINT_BYTES * npts / K), h2d_bytes_device=256 * 4,
                                  d2h_bytes_host_path=sum((w >> l) * (h >> l) * 12 for l in range(3)) + int(4 * 22 * ncand / K),
                                  h2d_bytes_host_path=int(8 * ncand / K)))
        ct.close()
    # the serial chain's worst case: stripes, dx == 0 everywhere
    w, h, lv = 640, 480, 5
    img = S.image("stripe", w, h, 12)
    ct = capi.CT(w, h, lv)
    ct.upload_new_image(img)
    stripe = []
    for pot, rec in ((3, 1), (1, 0)):
        o = S.restate(ct_pyr := [ct.download_frame(l, w, h) for l in range(3)], potential=pot, recursionsLeft=rec)
        ct.make_new_traces(pot, recursionsLeft=rec)
        reps = 10
        t0 = time.perf_counter()
        for _ in range(reps):
            g = ct.make_new_traces(pot, recursionsLeft=rec)
        t = (time.perf_counter() - t0) / reps
        identical &= same(g, o)
        del ct_pyr
        stripe.append(dict(potential=pot, recursionsLeft=rec, mixed_blocks=o["n_mixed"], points=len(g["points"]["u"]), device_ms=1e3 * t))
    ct.close()
    res["stripe_640x480"] = stripe
    res["bit_identical"] = bool(identical)
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        open(a.out, "w").write(line + "\n")


if __name__ == "__main__":
    main()
