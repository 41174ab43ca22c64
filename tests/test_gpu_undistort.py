"""SURVEY.md 8(f) rank 1: image_undistort::undistort<true> on RGB24 -- integer-exact, so the CUDA remap must equal
the reference's bit for bit, including the frame border where taps fall outside the image."""
import numpy as np
import pytest

import ingress_states
from pipeline_util import EUROC_KC

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("kc", [EUROC_KC, [0.12, -0.05, 0.01, -0.002, 0.003], [0, 0, 0, 0, 0]])
def test_undistort_matches_reference(built, kc):
    from oracle import refapi
    from rebvo_b200 import capi, synth
    if not refapi.available():
        pytest.skip("oracle/_ref not built")
    cam = synth.EUROC
    rng = np.random.default_rng(5)
    img = rng.integers(0, 256, (cam["h"], cam["w"], 3), dtype=np.uint8)
    img2 = synth.Sequence(w=cam["w"], h=cam["h"], seed=3).frame(2)[1]
    ctx = capi.Ctx(cam, 3.56359, 1.2599)
    und = capi.Undistort(ctx, kc)
    for im in (img, img2):
        ref = refapi.undistort_rgb(cam, kc, im)
        got = und.apply(im)
        assert np.array_equal(ref, got), "mismatch in %d bytes" % int((ref != got).sum())
    und.close()
    ctx.close()


@pytest.mark.parametrize("name", sorted(ingress_states.MAPS))
def test_undistort_maps_match_reference(built, name):
    """The maps of tests/ingress_states.py: every tap count the map can have (0, 1, 2, 4), principal points on integers and
    on x.5, kc = 0 (exact weights), the KITTI and odd-width geometries, on random, edge and all-255 frames."""
    from oracle import refapi
    from rebvo_b200 import capi
    if not refapi.available():
        pytest.skip("oracle/_ref not built")
    c = ingress_states.MAPS[name]
    ctx = capi.Ctx(c["cam"], 3.56359, 1.2599)
    und = capi.Undistort(ctx, c["kc"])
    try:
        for key in (("rand", 0), ("edge", 1), ("white",)):
            im = ingress_states.frame(c["cam"], key)
            ref = refapi.undistort_rgb(c["cam"], c["kc"], im)
            got = und.apply(im)
            assert np.array_equal(ref, got), "%s %s: mismatch in %d bytes" % (name, key, int((ref != got).sum()))
    finally:
        und.close()
        ctx.close()
