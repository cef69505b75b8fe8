"""The exact refusals of the coarse tracker's tracking and tracing calls: the return code and the whole dmv_last_error() text, compared by
equality, so a message that gains or loses a `handles[i]: ` prefix, or a check that moves ahead of another, fails here.

dmv_ct_track and dmv_ct_track_tries name nothing but the fault.  dmv_ct_track_many, dmv_ct_track_tries_many and dmv_ct_trace_many first
check the member list (count, NULL members, duplicates), then refuse a member's own arguments with its position in front; the two tracking
calls then probe every member and ask for one cluster size, which the tracing call does not need."""
import ctypes as C

import pytest

from dmvio_b200.capi import DMV_ERR_INVALID, DMV_ERR_STATE, DMV_OK
from gpu_harness import capi, close, ct_handle, ct_scene, gpu, near_truth_tries, set_cluster, track_kw, tries_kw  # noqa: F401

SINGLE = ["dmv_ct_track", "dmv_ct_track_tries"]
MANY = ["dmv_ct_track_many", "dmv_ct_track_tries_many", "dmv_ct_trace_many"]
TRACKS = {"dmv_ct_track", "dmv_ct_track_many"}
TRIES = {"dmv_ct_track_tries", "dmv_ct_track_tries_many"}
SCENE = "tma0_160x120"
CLUSTER_5 = "DMV_CT_CLUSTER=5: expected 16, 8 or 4"


def blank(capi, fn):
    """an all-zero argument block of fn"""
    return capi.CTTrackArgs() if fn in TRACKS else capi.CTTriesArgs() if fn in TRIES else capi.TraceJob()


def call(capi, fn, hs, args, n=None):
    """fn through its raw symbol; returns (rc, dmv_last_error()).  Single calls: hs is one handle or None, args one block or None.  Calls over
    several handles: hs is a list (None entries are NULL members) or None, args a list of blocks or None, n defaults to len(hs)."""
    L = capi.lib()
    if fn in SINGLE:
        out = capi.CTTrackResult() if fn in TRACKS else capi.CTTriesResult()
        rc = getattr(L, fn)(None if hs is None else hs.h, None if args is None else C.byref(args), C.byref(out))
        return rc, L.dmv_last_error().decode()
    m = max(len(hs or []), len(args or []), 1)
    H = None if hs is None else (C.c_void_p * m)(*[None if g is None else g.h.value for g in hs])
    A = None if args is None else (type(args[0]) * m)(*args)
    n = len(hs or []) if n is None else n
    if fn == "dmv_ct_trace_many":
        rc = L.dmv_ct_trace_many(H, n, A, None)
    else:
        out = ((capi.CTTrackResult if fn in TRACKS else capi.CTTriesResult) * m)()
        rc = getattr(L, fn)(H, n, A, out)
    return rc, L.dmv_last_error().decode()


def refused(capi, fn, hs, args, text, code=DMV_ERR_INVALID, n=None):
    assert call(capi, fn, hs, args, n) == (code, text)


def test_refusals_without_a_handle(capi):
    """the checks that need no handle and no device"""
    for fn in SINGLE:
        refused(capi, fn, None, blank(capi, fn), "null argument")
        refused(capi, fn, None, None, "null argument")
    for fn in MANY:
        a = blank(capi, fn)
        refused(capi, fn, None, [a], "null argument", n=1)
        refused(capi, fn, [None], None, "null argument")
        refused(capi, fn, [None], [a], "n = 0: expected 1 to 16 handles", n=0)
        refused(capi, fn, [None], [a], "n = -1: expected 1 to 16 handles", n=-1)
        refused(capi, fn, [None] * 17, [a] * 17, "n = 17: expected 1 to 16 handles")
        refused(capi, fn, [None], [a], "handles[0] is NULL")
        refused(capi, fn, [None, None], [a, a], "handles[0] is NULL")


class Blocks:
    """argument blocks for handles loaded with the scene (trace: an empty job, which an accepted call answers without a launch)"""

    def __init__(self, capi, sc):
        self.capi, self.sc, self.keep = capi, sc, []
        self.Rs, self.ts = near_truth_tries(sc)

    def __call__(self, fn, **over):
        if fn in TRACKS:
            return self.capi._track_args(self.sc["levels"], **track_kw(self.sc, **over))
        if fn in TRIES:
            A, arrays = self.capi._tries_args(self.sc["levels"], self.Rs, self.ts, **tries_kw(self.sc, **over))
            self.keep.append(arrays)
            return A
        return self.capi.TraceJob()


@pytest.mark.gpu
@pytest.mark.parametrize("fn", SINGLE)
def test_single_handle_refusals(capi, gpu, orc, synth, monkeypatch, fn):
    set_cluster(monkeypatch)
    sc = ct_scene(orc, synth, SCENE)
    L = sc["levels"]
    g, noK = ct_handle(capi, sc), ct_handle(capi, sc, k=False)
    B = Blocks(capi, sc)
    refused(capi, fn, None, B(fn), "null argument")
    refused(capi, fn, g, None, "null argument")
    for c in (-1, L):
        refused(capi, fn, g, B(fn, coarsest=c), "coarsestLvl out of range")
    refused(capi, fn, noK, B(fn), "dmv_ct_set_K(level) first", DMV_ERR_STATE)
    refused(capi, fn, noK, B(fn, coarsest=L), "coarsestLvl out of range")   # the level range before the intrinsics
    if fn in TRIES:
        for n in (0, 33):
            A = B(fn)
            A.n = n
            refused(capi, fn, g, A, f"n = {n}: expected 1 to 32 tries")
            A.R = None
            refused(capi, fn, g, A, f"n = {n}: expected 1 to 32 tries")   # the count before the pointers
        for field in ("R", "t"):
            A = B(fn, coarsest=L)
            setattr(A, field, None)
            refused(capi, fn, g, A, "null R / t")   # the pointers before the level range
    # the probe's refusal, after every argument check
    set_cluster(monkeypatch, "5")
    h = ct_handle(capi, sc)
    refused(capi, fn, h, B(fn), CLUSTER_5)
    refused(capi, fn, h, B(fn), CLUSTER_5)   # a refused probe is repeated by the next call
    refused(capi, fn, h, B(fn, coarsest=L), "coarsestLvl out of range")
    close(g, noK, h)


@pytest.mark.gpu
@pytest.mark.parametrize("fn", MANY)
def test_many_handle_refusals(capi, gpu, orc, synth, monkeypatch, fn):
    set_cluster(monkeypatch)
    sc = ct_scene(orc, synth, SCENE)
    L = sc["levels"]
    gs = [ct_handle(capi, sc) for _ in range(17)]
    B = Blocks(capi, sc)
    a = B(fn)
    # the member list
    refused(capi, fn, gs[:1], [a], "n = 0: expected 1 to 16 handles", n=0)
    refused(capi, fn, gs, [a] * 17, "n = 17: expected 1 to 16 handles")
    refused(capi, fn, None, [a] * 2, "null argument", n=2)
    refused(capi, fn, gs[:2], None, "null argument")
    refused(capi, fn, [gs[0], None, gs[2]], [a] * 3, "handles[1] is NULL")
    refused(capi, fn, [gs[0], gs[1], gs[0]], [a] * 3, "handles[0] and handles[2] are the same handle")
    refused(capi, fn, [gs[0], gs[1], gs[1], gs[0]], [a] * 4, "handles[1] and handles[2] are the same handle")
    refused(capi, fn, [gs[0], gs[1], gs[0], None], [a] * 4, "handles[0] and handles[2] are the same handle")
    # a member's own refusal, with its position in front, after the member list
    if fn in TRACKS:
        bad, text = B(fn, coarsest=L), "coarsestLvl out of range"
    elif fn in TRIES:
        bad, text = B(fn), "n = 0: expected 1 to 32 tries"
        bad.n = 0
    else:
        bad, text = capi.TraceJob(1, None, None), "null argument"
    refused(capi, fn, gs[:3], [a, bad, a], f"handles[1]: {text}")
    refused(capi, fn, gs[:4], [a, a, a, bad], f"handles[3]: {text}")
    refused(capi, fn, [gs[0], gs[1], None], [bad, a, a], "handles[2] is NULL")
    if fn in TRIES:
        noR = B(fn)
        noR.R = None
        refused(capi, fn, gs[:3], [a, a, noR], "handles[2]: null R / t")
    noK = ct_handle(capi, sc, k=False)
    if fn == "dmv_ct_trace_many":
        assert call(capi, fn, [gs[0], noK], [a, a])[0] == DMV_OK   # tracing needs no intrinsics
    else:
        refused(capi, fn, [gs[0], gs[1], noK], [a] * 3, "handles[2]: dmv_ct_set_K(level) first", DMV_ERR_STATE)
        refused(capi, fn, [gs[0], noK, gs[1]], [a, a, bad], "handles[1]: dmv_ct_set_K(level) first", DMV_ERR_STATE)
    # the probes, after every member's own checks
    set_cluster(monkeypatch, "5")
    h5 = [ct_handle(capi, sc) for _ in range(2)]
    if fn == "dmv_ct_trace_many":
        assert call(capi, fn, h5, [a, a])[0] == DMV_OK   # tracing does not probe
    else:
        refused(capi, fn, h5, [a, a], f"handles[0]: {CLUSTER_5}")
        refused(capi, fn, h5, [a, bad], f"handles[1]: {text}")
    # one cluster size: a handle probed under DMV_CT_CLUSTER=16 beside one probed under 8
    probed = {}
    for nc in ("16", "8"):
        set_cluster(monkeypatch, nc)
        probed[nc] = ct_handle(capi, sc)
        probed[nc].track(**track_kw(sc))
    set_cluster(monkeypatch)
    pair = [probed["16"], probed["8"]]
    if fn == "dmv_ct_trace_many":
        assert call(capi, fn, pair, [a, a])[0] == DMV_OK   # tracing launches no cluster
    else:
        refused(capi, fn, pair, [a, a], "handles[0] tracks with clusters of 16 CTAs, handles[1] with 8: one launch needs one cluster size")
        refused(capi, fn, pair[::-1], [a, a], "handles[0] tracks with clusters of 8 CTAs, handles[1] with 16: one launch needs one cluster size")
    close(noK, *h5, *pair, *gs)
