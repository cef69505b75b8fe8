"""Per-frame cost of getting a camera frame into the tracker's pyramid, two ways:
  raw    dmv_ct_upload_raw_image: the raw 8/16-bit frame goes up, undistortion + photometric map + pyramid run on the device
  float  the host undistorts (the CPU restatement of Undistort::undistort<T>, oracle/orc_undistort.cpp, -O3 single thread, the reference's
         flags) and dmv_ct_upload_new_image uploads 4-byte floats
Wall time per frame: N back-to-back frames and one final read-back (dmv_ct_download_frame of the coarsest level) that waits for the last,
divided by N.  H2D bytes come from the shapes.  Prints one JSON line, with the card's name and power limit read in the same run, and writes it
to --out if given.
    python tools/bench_ingest.py [--frames 300] [--out records/h100_ingest.json]"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import dmvio_b200.capi as capi  # noqa: E402
from oracle import undistort as U  # noqa: E402

SHAPES = [("euroc_radtan_752x480_to_640x480_u8", 752, 480, 640, 480, 1), ("tumvi_512x512_u16", 512, 512, 512, 512, 2)]
LEVELS = 5


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout
        return q.strip().splitlines()[0]
    except Exception as e:  # noqa: BLE001
        return f"unknown ({e})"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=300)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if capi.lib().dmv_device_count() < 1:
        raise SystemExit("bench_ingest needs a CUDA device")
    res = dict(card=card(), frames=a.frames, levels=LEVELS, photometric_mode=2, shapes=[])
    for name, wOrg, hOrg, w, h, bpp in SHAPES:
        rx, ry = U.synthetic_remap(w, h, wOrg, hOrg)
        nG = 256 if bpp == 1 else 65536
        G = U.G_from_file(U.response_file_values(nG))[:nG]
        vi = U.vignette_inv(U.vignette8(wOrg, hOrg))
        raws = [U.raw_frame(wOrg, hOrg, bpp, seed=s) for s in range(4)]
        ct = capi.CT(w, h, LEVELS, max_points=4096)
        ct.set_undistort(wOrg, hOrg, rx, ry, G, vi, 2)
        imgs = [U.restate(w, h, r, rx, ry, G, vi, 2, 1.0, 1.0 / 256 if bpp == 2 else 1.0) for r in raws]
        lw = w >> (LEVELS - 1)
        for _ in range(20):  # warm-up: modules, both paths
            ct.upload_raw_image(raws[0], 1.0)
            ct.upload_new_image(imgs[0])
        ct.download_frame(LEVELS - 1, w, h)
        t0 = time.perf_counter()
        for i in range(a.frames):
            ct.upload_raw_image(raws[i & 3], 1.0)
        ct.download_frame(LEVELS - 1, w, h)
        t_raw = (time.perf_counter() - t0) / a.frames
        t0 = time.perf_counter()
        for i in range(a.frames):
            ct.upload_new_image(U.restate(w, h, raws[i & 3], rx, ry, G, vi, 2, 1.0, 1.0 / 256 if bpp == 2 else 1.0))
        ct.download_frame(LEVELS - 1, w, h)
        t_float = (time.perf_counter() - t0) / a.frames
        t0 = time.perf_counter()
        for i in range(a.frames):
            U.restate(w, h, raws[i & 3], rx, ry, G, vi, 2, 1.0, 1.0)
        t_host = (time.perf_counter() - t0) / a.frames
        ok = np.array_equal(ct.download_frame(0, w, h)[..., 0].view(np.uint32), imgs[(a.frames - 1) & 3].view(np.uint32))
        ct.close()
        res["shapes"].append(dict(name=name, raw=[wOrg, hOrg], out=[w, h], bytes_per_px=bpp, raw_path_ms=1e3 * t_raw, float_path_ms=1e3 * t_float,
                                  host_undistort_ms=1e3 * t_host, h2d_bytes_raw=wOrg * hOrg * bpp, h2d_bytes_float=w * h * 4, last_frame_bit_identical=ok,
                                  lw_coarsest=lw))
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        open(a.out, "w").write(line + "\n")


if __name__ == "__main__":
    main()
