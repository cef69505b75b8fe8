"""The oracle pinned to the reference's compiled code (tests/test_ref_pin.py's BA path and marginalisation pins) on windows with what
synth.make_window never produces and real sequences do on every frame (helpers.hard_window): non-finite and textureless pixels, exposures
!= 1 with large affine parameters, saturation, points at the image margins and FEJ centres behind the camera.  Also checks that each exit
of PointFrameResidual::linearize the window was built for is taken, and pins makeImages on images with NaN and inf."""
import numpy as np
import pytest

from helpers import HARD_DESIGNED, HARD_LABELS, RES_IN, RES_OOB, RES_OUTLIER, hard_window
from test_ref_pin import ba_path_bit_exact, marginalization_bit_exact, ref  # noqa: F401  (the "ref" fixture)

HARD_CONFIGS = [dict(nf=5, npts=1000, seed=21), dict(nf=8, npts=1000, seed=99, hosts="all", w=752, h=480)]
MIN_REACHED = 10


def hard_id(c):
    return f"nf{c['nf']}_{c.get('w', 640)}x{c.get('h', 480)}"


def hard_flagged(W, seed):
    """points to marginalise: every point with a residual of each label, and a random third of the others"""
    rng = np.random.default_rng(seed)
    npts = len(W["host"])
    lab = W["labels"]
    pts = set(np.asarray(W["res_point"])[lab != "none"].tolist())
    pts |= set(rng.choice(npts, npts // 3, replace=False).tolist())
    return np.array(sorted(pts), np.int32)


def check_labels(W, newState, newEnergy, newEnergyWithOutlier, TH=512.0):
    """every label gives its designed state (incoming OOB residuals stay OOB); returns {label: residuals reaching it}"""
    lab, live = W["labels"], np.asarray(W["res_state"]) != RES_OOB
    assert np.all(newState[~live] == RES_OOB)
    reached = {}
    for L in HARD_LABELS:
        m = (lab == L) & live
        if L == "none":
            assert not np.any(newState[m] == RES_OOB), "a residual without a designed exit went OOB"
        else:
            bad = np.nonzero(m & (newState != HARD_DESIGNED[L]))[0]
            assert len(bad) == 0, f"{L}: residuals {bad[:10]} end in {newState[bad[:10]]}, not {HARD_DESIGNED[L]}"
        if L == "flat":
            assert np.all(newEnergy[m] == np.float32(TH))
        if HARD_DESIGNED.get(L) == RES_OOB:
            assert np.all(newEnergyWithOutlier[m] == -1)
        reached[L] = int(m.sum())
    i, _ = W["single_nan"].T
    assert sorted(set(W["single_nan"][:, 1].tolist())) == list(range(8))
    assert np.all(newState[i] == RES_OOB) and np.all(lab[i] == "nan")
    return reached


@pytest.mark.parametrize("cfg", HARD_CONFIGS, ids=hard_id)
def test_ba_path_bit_exact_hard(ref, orc, synth, cfg):
    W = hard_window(synth, orc, cfg)
    E_r, r, a_r, p_r = ba_path_bit_exact(ref, orc, synth, cfg, W=W)
    reached = check_labels(W, r["newState"], r["newEnergy"], r["newEnergyWithOutlier"])
    print(f"{hard_id(cfg)}: residuals per label {reached}, states IN/OOB/OUTLIER {np.bincount(r['newState'], minlength=3).tolist()}")
    for L in ("nan", "flat", "border", "behind"):
        assert reached[L] >= MIN_REACHED, (L, reached)
    assert (r["newState"] == RES_IN).mean() >= 0.3               # the systems still carry weight
    assert np.any(r["newState"] == RES_OUTLIER)
    assert np.all(np.isfinite(a_r["HA"])) and np.all(np.isfinite(a_r["Hsc"]))
    for k in ("Hdd", "bd", "Hcd", "HdiF", "bdSumF"):
        assert np.all(np.isfinite(p_r[k])), k


@pytest.mark.parametrize("cfg", HARD_CONFIGS, ids=hard_id)
def test_marginalization_bit_exact_hard(ref, orc, synth, cfg):
    W = hard_window(synth, orc, cfg)
    r = marginalization_bit_exact(ref, orc, synth, cfg, W=W, pts=hard_flagged(W, cfg["seed"]))
    assert np.all(np.isfinite(r["rtz"])) and np.all(np.isfinite(r["H"]))


def test_make_images_non_finite_bit_exact(ref, orc, synth):
    """FrameHessian::makeImages on intensities with NaN blocks, rows, single texels and an inf column: every level of the pyramid (the 2x2
    means carry the NaN and inf up), the non-finite gradients set to 0; and hard_window's dI is its level 0"""
    from helpers import make_images_level0
    W = hard_window(synth, orc, HARD_CONFIGS[0])
    for k in (1, W["nf"] - 1):
        img = W["images"][k]
        assert np.isnan(img).any() and np.isinf(img).any()
        pr, po = ref.make_images(img, W["K"]), orc.make_images(img, W["K"])
        assert len(pr) == len(po) == 4
        for l in range(len(pr)):
            # the gradients of the first and last row are left uninitialised by the reference (HessianBlocks.cpp:L169-179)
            np.testing.assert_array_equal(po[l][1:-1], pr[l][1:-1], err_msg=f"frame {k} level {l}")
            np.testing.assert_array_equal(po[l][..., 0], pr[l][..., 0], err_msg=f"frame {k} level {l}")
            assert np.all(np.isfinite(pr[l][1:-1, :, 1:])), "a non-finite gradient survived"
            assert np.isnan(pr[l][..., 0]).any()
        np.testing.assert_array_equal(W["dI"][k].reshape(pr[0].shape)[1:-1], pr[0][1:-1])
        np.testing.assert_array_equal(make_images_level0(img)[..., 0], pr[0][..., 0])
