"""Scale space on awkward geometries: widths / heights that are not multiples of the 32-column chunks, 32-row bands and 64x32
tiles of the TMA kernels (partial tiles are clipped by the tensor maps, border tiles take the zero-fill path), down to 32x32,
where the (32 + d)-row windows of the box-average row pass are taller than the image, and both box plans (sigma0 = 1.78:
boxes 3/3/5 + 3/5/5, sigma0 = 3.56: 7/7/7 + 9/9/9).  Every plane must equal the reference's (sspace::build, compiled from
the reference's sources) bit for bit."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

GEOMETRIES = [(36, 33), (64, 48), (100, 76), (200, 150), (328, 244), (752, 97), (32, 32)]


def _planes(w, h, sigma0, rgb):
    from rebvo_b200 import capi
    cam = dict(w=w, h=h, zfx=300.0, zfy=300.0, ppx=w / 2.0, ppy=h / 2.0)
    ctx = capi.Ctx(cam, sigma0, 1.2599, kl_capacity=20000)
    m = ctx.new_map()
    m.upload_rgb(rgb)
    m.dog_build()
    out = {k: m.plane(k).copy() for k in ("gray", "img0", "img1", "dog")}
    m.close()
    ctx.close()
    return out


@pytest.mark.parametrize("sigma0", [1.7818, 3.56359])
def test_odd_geometries_bitwise(built, sigma0):
    from oracle import refapi
    rng = np.random.default_rng(5)
    for (w, h) in GEOMETRIES:
        rgb = rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
        rgb[h // 3:, w // 4:] //= 3   # an edge, so that the planes are not just noise
        r = refapi.RefMap(w, h, w / 2.0, h / 2.0, 300.0, 300.0, sigma0, 1.2599)
        r.rgb2bw(rgb)
        r.build()
        got = _planes(w, h, sigma0, rgb)
        for k in ("gray", "img0", "img1", "dog"):
            ref = r.plane(k)
            assert ref.shape == got[k].shape
            assert np.array_equal(ref.view(np.uint32), got[k].view(np.uint32)), "%dx%d sigma0 %.2f plane %s: %d pixels differ" % (
                w, h, sigma0, k, int((ref.view(np.uint32) != got[k].view(np.uint32)).sum()))

