"""TEST INFRASTRUCTURE ONLY — bindings and cases of the activation-selection oracles (dmv_ba_select_activation).

  restate(case)   liborc.so: the CPU restatement of makeDistanceMap, growDistBFS, addIntoDistFinal and activatePointsMT's selection loop
                  (orc_activation.cpp)
  reference(case) _ref/libactivation_ref.so: the REFERENCE's own CoarseDistanceMap around a line-for-line mirror of the loop
                  (ref_activation.cpp, built by ref_build.sh); also returns the [KRKi | Kt] tables it computed
  make_case(...)  seeded windows shared by the CPU pin, the golden fixture, the device tests and tools/bench_activation.py"""
import ctypes as C
import functools

import numpy as np

from . import orc, ref
from .orc import f32p, f64p, i32p, u8p

REF_LIB = "libactivation_ref.so"

IMM_KEYS = ("u", "v", "idepth_min", "idepth_max", "status", "interval", "quality", "type")
KEEP, DELETE, OPTIMIZE = 0, 1, 2
MIN_TRACE_QUALITY = 3.0  # setting_minTraceQuality


@functools.cache
def orc_lib():
    L = orc.lib()
    L.orc_act_select.restype = C.c_int
    L.orc_act_select.argtypes = [C.c_int, C.c_int, C.c_int, C.c_int, f32p, u8p, C.c_int, f32p, f32p, f32p, i32p, i32p, f32p, f32p, f32p, f32p, i32p,
                                 f32p, f32p, f32p, C.c_float, C.c_float, i32p, i32p, f32p]
    L.orc_act_grow.argtypes = [C.c_int, C.c_int, f32p, C.c_int, i32p]
    return L


def ref_available():
    return ref.built(REF_LIB)


@functools.cache
def ref_lib():
    L = ref.open_ref(REF_LIB)
    L.ref_act_select.restype = C.c_int
    L.ref_act_select.argtypes = [C.c_int, C.c_int, f64p, C.c_int, C.c_int, f64p, f64p, u8p, C.c_int, f32p, f32p, f32p, i32p, i32p, f32p, f32p, f32p,
                                 f32p, i32p, f32p, f32p, f32p, C.c_float, C.c_float, i32p, i32p, f32p, f32p]
    L.ref_act_grow.argtypes = [C.c_int, C.c_int, f32p, C.c_int, i32p]
    return L


def _n(case):
    return int(case["off"][-1])


def reference(case):
    """(action, toOptimize indexes, map, tables12) from the reference's CoarseDistanceMap and the mirrored loop"""
    n, w1, h1 = _n(case), case["w"] // 2, case["h"] // 2
    act, opt = np.zeros(max(n, 1), np.int32), np.zeros(max(n, 1), np.int32)
    m, tab = np.zeros(w1 * h1, np.float32), np.zeros(12 * case["nf"], np.float32)
    I = case["imm"]
    k = ref_lib().ref_act_select(case["w"], case["h"], case["K"], case["nf"], case["newest"], case["R9"], case["t3"], case["flagged"], len(case["act_u"]),
                                 case["act_u"], case["act_v"], case["act_id"], case["act_host"], case["off"], *[I[key] for key in IMM_KEYS],
                                 case["min_act_dist"], MIN_TRACE_QUALITY, act, opt, m, tab)
    return act[:n], opt[:k], m, tab


def restate(case, tab12):
    """(action, toOptimize indexes, map) from the CPU restatement, for the given [KRKi | Kt] tables"""
    n, w1, h1 = _n(case), case["w"] // 2, case["h"] // 2
    act, opt, m = np.zeros(max(n, 1), np.int32), np.zeros(max(n, 1), np.int32), np.zeros(w1 * h1, np.float32)
    I = case["imm"]
    k = orc_lib().orc_act_select(w1, h1, case["nf"], case["newest"], np.ascontiguousarray(tab12, np.float32), case["flagged"], len(case["act_u"]),
                                 case["act_u"], case["act_v"], case["act_id"], case["act_host"], case["off"], *[I[key] for key in IMM_KEYS],
                                 case["min_act_dist"], MIN_TRACE_QUALITY, act, opt, m)
    return act[:n], opt[:k], m


def flood(lib, w, h, m, cells):
    """addIntoDistFinal for each (x, y) of cells in order, on a copy of the level-1 map m; lib = "orc" or "ref" """
    out = np.ascontiguousarray(m, np.float32).copy()
    xy = np.ascontiguousarray(np.asarray(cells, np.int32).reshape(-1))
    if lib == "orc":
        orc_lib().orc_act_grow(w // 2, h // 2, out, len(xy) // 2, xy)
    else:
        ref_lib().ref_act_grow(w, h, out, len(xy) // 2, xy)
    return out


def tables(case):
    """[KRKi | Kt] per frame in float32 from the case's poses (K[1] * R * Ki[0], K[1] * t of newest * host^-1): the device tests' tables.
    Not bit-equal to the reference's Eigen products, and it need not be: the restatement and the device read the same tables."""
    fx, fy, cx, cy = case["K"]
    K0 = np.array([[fx, 0, cx], [0, fy, cy], [0, 0, 1]], np.float32)
    K1 = np.array([[fx * 0.5, 0, (cx + 0.5) / 2 - 0.5], [0, fy * 0.5, (cy + 0.5) / 2 - 0.5], [0, 0, 1]], np.float32)
    Ki0 = np.linalg.inv(K0.astype(np.float64)).astype(np.float32)
    Rn, tn = case["R9"][9 * case["newest"]:9 * case["newest"] + 9].reshape(3, 3), case["t3"][3 * case["newest"]:3 * case["newest"] + 3]
    out = np.zeros((case["nf"], 12), np.float32)
    for f in range(case["nf"]):
        Rf, tf = case["R9"][9 * f:9 * f + 9].reshape(3, 3), case["t3"][3 * f:3 * f + 3]
        R = Rn @ Rf.T
        t = tn - R @ tf
        out[f, :9] = (K1 @ R.astype(np.float32) @ Ki0).reshape(-1)
        out[f, 9:] = K1 @ t.astype(np.float32)
    return out.reshape(-1)


def _rot(rng, s):
    a = rng.normal(0, s, 3)
    th = np.linalg.norm(a)
    if th == 0:
        return np.eye(3)
    k = a / th
    Kx = np.array([[0, -k[2], k[1]], [k[2], 0, -k[0]], [-k[1], k[0], 0]])
    return np.eye(3) + np.sin(th) * Kx + (1 - np.cos(th)) * Kx @ Kx


def make_case(w=640, h=480, nf=7, n_active=2000, n_imm=1500, seed=0, min_act_dist=2.0, specials=False, cluster=None, border=False, flagged=(0,),
              imm_counts=None, act_outside=False):
    """A window of nf keyframes, the newest last.  Frame 0 has the newest frame's pose exactly (identity relative motion), so a level-0 pixel
    (2x, 2y) of frame 0 lands in level-1 cell (x, y): cluster = (x, y, r) puts every immature point of frame 0 in a (2r+1)^2 block of cells
    there, border = True puts frame 0's active and immature points on the border ring of the map and one cell inside it.  specials adds
    active and immature points whose projections are NaN, huge, or behind the camera (ptp[2] <= 0).  imm_counts overrides the immature
    points per frame (the newest frame's included)."""
    rng = np.random.default_rng(seed)
    K = np.array([0.7 * w, 0.7 * w, w / 2 - 0.5, h / 2 - 0.5], np.float64)
    R9, t3 = np.zeros(9 * nf), np.zeros(3 * nf)
    for f in range(nf):
        if f == 0 or f == nf - 1:
            R, t = np.eye(3), np.zeros(3)
        else:
            R, t = _rot(rng, 0.02), rng.normal(0, 0.03, 3)
            t[2] = 0.05 if f % 2 else -0.05
        R9[9 * f:9 * f + 9], t3[3 * f:3 * f + 3] = R.reshape(-1), t
    fl = np.zeros(nf, np.uint8)
    for f in flagged:
        if 0 <= f < nf - 1:
            fl[f] = 1
    w1, h1 = w // 2, h // 2
    ah = rng.integers(0, nf, n_active).astype(np.int32)
    au = rng.uniform(0, w - 1, n_active).astype(np.float32)
    av = rng.uniform(0, h - 1, n_active).astype(np.float32)
    aid = rng.uniform(0.2, 2.0, n_active).astype(np.float32)
    if border and n_active > 0:
        ring = [(x, 0) for x in range(w1)] + [(x, h1 - 1) for x in range(w1)] + [(0, y) for y in range(h1)] + [(w1 - 1, y) for y in range(h1)]
        ring += [(x, 1) for x in range(1, w1 - 1)] + [(w1 - 2, y) for y in range(1, h1 - 1)]
        sel = rng.choice(len(ring), min(len(ring), max(1, n_active // 4)), replace=False)
        for j, s in enumerate(sel):
            ah[j], au[j], av[j] = 0, 2 * ring[s][0], 2 * ring[s][1]
    if act_outside:
        au[:] = -2000.0
    if specials and n_active >= 8:
        aid[:3] = [np.nan, 3e38, -50.0]
        aid[3:6] = [1e30, np.inf, -1e4]
        ah[:6] = [1, 1, 1, 2, 2, 2]
        ah[6], au[6] = 0, 1e12   # frame 0's projection is the identity: u / 1 beyond int's range
    counts = list(imm_counts) if imm_counts is not None else [n_imm] * nf
    off = np.zeros(nf + 1, np.int32)
    off[1:] = np.cumsum(counts)
    n = int(off[-1])
    I = dict(u=rng.uniform(0, w - 1, n).astype(np.float32), v=rng.uniform(0, h - 1, n).astype(np.float32))
    a = rng.uniform(0.1, 2.0, n).astype(np.float32)
    b = (a * rng.uniform(1.0, 1.5, n)).astype(np.float32)
    I["idepth_min"], I["idepth_max"] = a, b
    I["status"] = rng.choice([0, 1, 2, 3, 4, 5], n, p=[0.6, 0.05, 0.05, 0.15, 0.1, 0.05]).astype(np.int32)
    I["interval"] = rng.uniform(0, 9, n).astype(np.float32)
    I["quality"] = rng.uniform(2.0, 20, n).astype(np.float32)
    I["type"] = rng.choice([1.0, 2.0, 4.0], n, p=[0.6, 0.3, 0.1]).astype(np.float32)
    I["idepth_max"][rng.random(n) < 0.03] = np.nan
    n0 = counts[0]
    if cluster is not None and n0 > 0:
        x, y, r = cluster
        I["u"][:n0] = 2 * rng.integers(max(1, x - r), min(w1 - 1, x + r + 1), n0)
        I["v"][:n0] = 2 * rng.integers(max(1, y - r), min(h1 - 1, y + r + 1), n0)
    if border and n0 > 0:
        ring = [(x, 1) for x in range(1, w1)] + [(w1 - 1, y) for y in range(1, h1)] + [(x, 2) for x in range(2, w1 - 1)] + [(w1 - 2, y) for y in range(2, h1 - 1)]
        sel = rng.integers(0, len(ring), n0)
        I["u"][:n0] = [2 * ring[s][0] for s in sel]
        I["v"][:n0] = [2 * ring[s][1] for s in sel]
    if specials and n > off[2] + 8:
        j = int(off[1])  # frame 1 (t_z = +0.05) and frame 2 (t_z = -0.05)
        for k, (lo, hi) in enumerate([(3e38, 3e38), (1e30, 1e30), (1e3, 1e3), (-1e3, -1e3 + 0.5)]):
            for base in (j, int(off[2])):
                I["idepth_min"][base + k], I["idepth_max"][base + k] = lo, hi
                I["status"][base + k], I["interval"][base + k], I["quality"][base + k] = 0, 1.0, 10.0
        I["u"][0], I["idepth_min"][0], I["idepth_max"][0], I["status"][0], I["interval"][0], I["quality"][0] = 1e12, 1.0, 1.0, 0, 1.0, 10.0
    for key in IMM_KEYS:
        I[key] = np.ascontiguousarray(I[key])
    return dict(w=w, h=h, K=K, nf=nf, newest=nf - 1, R9=R9, t3=t3, flagged=fl, act_u=au, act_v=av, act_id=aid, act_host=ah, off=off, imm=I,
                min_act_dist=float(min_act_dist))


# the seeded windows of the CPU pin and of tests/golden/golden_activation.npz (small maps keep the fixture small; the device tests add the
# camera sizes)
CASES = {
    "c3": dict(w=320, h=240, n_active=1000, n_imm=400, seed=11, min_act_dist=2.0),
    "c3_mad0": dict(w=320, h=240, n_active=1000, n_imm=400, seed=12, min_act_dist=0.0),
    "c3_mad4": dict(w=320, h=240, n_active=1000, n_imm=400, seed=13, min_act_dist=4.0),
    "first_keyframes": dict(w=320, h=240, n_active=30, n_imm=800, seed=14, min_act_dist=0.0, nf=3),
    "specials": dict(w=320, h=240, n_active=600, n_imm=300, seed=15, min_act_dist=4.0, specials=True),
    "specials_mad0": dict(w=320, h=240, n_active=600, n_imm=300, seed=16, min_act_dist=0.0, specials=True),
    "cluster": dict(w=320, h=240, n_active=200, n_imm=300, seed=17, min_act_dist=4.0, cluster=(60, 50, 3)),
    "border": dict(w=320, h=240, n_active=400, n_imm=300, seed=18, min_act_dist=1.0, border=True),
    "empty_active": dict(w=320, h=240, n_active=0, n_imm=300, seed=19, min_act_dist=2.0),
    "active_outside": dict(w=320, h=240, n_active=300, n_imm=300, seed=20, min_act_dist=2.0, act_outside=True),
    "sparse_hosts": dict(w=320, h=240, n_active=300, seed=21, min_act_dist=1.0, imm_counts=(0, 300, 0, 250, 0, 200, 50)),
    "odd_size": dict(w=322, h=242, n_active=500, n_imm=200, seed=22, min_act_dist=3.0, border=True),
}
