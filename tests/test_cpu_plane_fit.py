"""DetectorPlaneFitSize 1..4 on the CPU: the NumPy restatement of build_mask + join_edges (tests/plane_fit.py) against
vectors generated from the unmodified reference (tests/golden/detect_plane_fit.npz), and against the reference itself,
run in a child process per window size, when oracle/_ref is built.  Keyline fields, id mask and kn bit for bit."""
import os

import numpy as np
import pytest

from flow import DOG_THRESH, POS_NEG, SMALL, small_frames
from parity_util import KL_EXACT_DETECT
from plane_fit import plane_fit_pinv, port_detect, ref_detect_child

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "detect_plane_fit.npz")
QVGA = dict(SMALL, cam=dict(w=320, h=240, zfx=260.0, zfy=258.0, ppx=161.0, ppy=118.5), kl_max=9000, kl_ref=5000,
            track_points=4000, sigma0=3.56359)


def _planes(cfg, frames):
    from oracle import portapi
    cam = cfg["cam"]
    out = []
    for fr in frames:
        m = portapi.PortMap(cam["w"], cam["h"], cam["ppx"], cam["ppy"], cam["zfx"], cam["zfy"], cfg["sigma0"],
                            cfg["ksigma"])
        m.rgb2bw(fr)
        m.build()
        out.append((m.plane("img0"), m.plane("dog")))
    return out


def _port_chain(cfg, planes, R, kl_max=None):
    """detect on each frame with the threshold chained, like the reference child."""
    cam = cfg["cam"]
    t, l, res = cfg["thresh"], 0, []
    for img0, dog in planes:
        kn, t, l, kl, mask = port_detect(img0, dog, R, POS_NEG, DOG_THRESH, kl_max or cfg["kl_max"], t, l,
                                         cfg["kl_ref"], cfg["gain"], cfg["tmax"], cfg["tmin"], cam["ppx"], cam["ppy"])
        res.append((kn, t, l, kl, mask))
    return res


def _same_keylines(a, b, tag):
    assert len(a) == len(b), "%s: kn %d vs %d" % (tag, len(a), len(b))
    for f in KL_EXACT_DETECT:
        x, y = np.asarray(a[f]), np.asarray(b[f])
        if x.dtype.kind == "f":
            u = np.uint32 if x.dtype.itemsize == 4 else np.uint64
            x, y = x.view(u), y.view(u)
        assert np.array_equal(x, y), "%s: field %s differs at %d keylines" % (tag, f, int((x != y).sum()))


def test_pinv_restatement_is_the_pseudo_inverse():
    """The restated plane_fit_pinv is Phi's pseudo inverse at every radius (its bits are pinned by the golden and
    reference comparisons below, which depend on them)."""
    p = plane_fit_pinv(2)
    phi = np.array([(j, i, 1.0) for i in range(-2, 3) for j in range(-2, 3)])
    assert np.allclose(p, np.linalg.pinv(phi), rtol=0, atol=1e-15)
    for R in (1, 3, 4):
        n = 2 * R + 1
        phi = np.array([(j, i, 1.0) for i in range(-R, R + 1) for j in range(-R, R + 1)])
        assert plane_fit_pinv(R).shape == (3, n * n)
        assert np.allclose(plane_fit_pinv(R), np.linalg.pinv(phi), rtol=0, atol=1e-14)


def test_join_probe_below_the_last_row():
    """R = 1: a keyline on row h-2 whose zero crossing lies just under half a pixel below it.  In float32, y + ys rounds to
    h - 1.5, so its c_p rounds to row h-1, and the NextPoint probes of the row below fall past the end of the mask.  They
    count as "no keyline" (the reference reads past its buffer there); the keyline gets n_id = -1."""
    w, h = 752, 480
    xk, yk = 300, h - 2
    a, b, delta = 0.1, 10.0, 6e-6
    yc = (0.5 - delta) * (a * a + b * b) / (b * b)   # zero line of the plane at yk + yc: closest point ys = 0.5 - delta
    yy, xx = np.mgrid[0:h, 0:w].astype(np.float64)
    dog = (a * (xx - xk) + b * (yy - (yk + yc))).astype(np.float32)
    img0 = (100.0 * xx).astype(np.float32)          # a gradient far above the threshold everywhere
    kn, _, _, kl, mask = port_detect(img0, dog, 1, POS_NEG, DOG_THRESH, 40000, 0.01, 0, 15000, 0.0, 1.0, 0.0, 376.0,
                                     240.0)
    cy = kl["c_p"][:, 1]
    last = (kl["p_inx"] // w == yk) & ((cy.astype(np.float64) + 0.5).astype(int) == h - 1)
    assert last.sum() >= 1, "no keyline rounds to row h-1"
    assert (kl["m_m"][last, 0] > 0).all()            # m.x > 0: NextPoint probes row y + 1 = h
    assert (kl["n_id"][last] == -1).all()
    assert (mask[h - 1] == -1).all() and (mask[:, -1] == -1).all()


@pytest.mark.parametrize("R", [1, 3, 4])
def test_port_matches_golden(R):
    z = np.load(GOLD)
    from rebvo_b200.capi import KEYLINE
    f0, f1 = small_frames()
    got = _port_chain(SMALL, _planes(SMALL, (f0, f1)), R)
    for i, (kn, t, l, kl, mask) in enumerate(got):
        want = z["r%d_f%d_kn_tresh" % (R, i)]
        assert [kn, t, l] == want.tolist(), (R, i, [kn, t, l], want)
        _same_keylines(z["r%d_f%d_kl" % (R, i)].view(KEYLINE), kl, "R=%d f%d" % (R, i))
        assert np.array_equal(z["r%d_f%d_mask" % (R, i)], mask)
        assert (mask[:R, :] == -1).all() and (mask[:, :R] == -1).all()
        assert (mask[-R:, :] == -1).all() and (mask[:, -R:] == -1).all()
        assert kn > 1000


@pytest.mark.parametrize("R", [1, 2, 3, 4])
@pytest.mark.parametrize("cut", [False, True], ids=["full", "kl_max_cut"])
def test_port_matches_reference_qvga(R, cut, tmp_path):
    """The unmodified reference in a child process (one window size per process) on the 320x240 seed-23 pair: full
    detection, and a kl_max cut below the candidate count of the first frame."""
    from oracle import refapi
    from rebvo_b200 import synth
    if not refapi.available():
        pytest.skip("oracle/_ref not built")
    c = QVGA
    f0, f1 = synth.frame_pair(seed=23, w=320, h=240, nrect=90, shift=(-1.6, 0.9))
    planes = _planes(c, (f0, f1))
    kl_max = c["kl_max"]
    if cut:   # below the candidate count: the first frame's full detection at this R, less a third
        kl_max = _port_chain(c, planes[:1], R)[0][0] * 2 // 3
    ref = ref_detect_child(tmp_path, np.stack([f0, f1]), R, c["cam"], c["sigma0"], c["ksigma"], c["thresh"], kl_max,
                           c["kl_ref"], c["gain"], c["tmax"], c["tmin"], POS_NEG, DOG_THRESH, c["track_points"])
    got = _port_chain(c, planes, R, kl_max)
    for i, (kn, t, l, kl, mask) in enumerate(got):
        assert [kn, t, l] == ref["f%d_kn_tresh" % i].tolist(), (R, i)
        _same_keylines(ref["f%d_kl" % i], kl, "R=%d f%d" % (R, i))
        assert np.array_equal(ref["f%d_mask" % i], mask)
    if cut:
        assert got[0][0] == kl_max
    else:
        assert got[0][0] > 2000
