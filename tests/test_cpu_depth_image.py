"""The dense inverse-depth image of a depth grid (rb_depth_image, rb_pipeline_depth_image) written out in NumPy float32: the
arithmetic of depth_filler::getImgRho (include/visualizer/depth_filler.h:246-280) at integer pixel coordinates, as
include/rebvo_b200.h states it, pinned against the header's own getImgRho on crafted grids written straight into
depth_filler::data (oracle/_ref/libref_depth_image.so, built by oracle/ref_depth_image.py).  Runs without a GPU."""
import numpy as np
import pytest


def img_axis(n_px, block, n_cells):
    """Per pixel coordinate v = 0..n_px-1: (floor cell, ceil cell, weight) of one axis.
    x_histo = x / (float)block - 0.5: a float quotient, the subtraction in double, stored as float; floor / ceil clamped to
    [0, n_cells - 1]; dx = x_histo - xf in float."""
    q = np.arange(n_px, dtype=np.float32) / np.float32(block)
    hist = (q.astype(np.float64) - 0.5).astype(np.float32)
    f = np.clip(np.floor(hist.astype(np.float64)), 0, n_cells - 1).astype(np.int64)
    c = np.clip(np.ceil(hist.astype(np.float64)), 0, n_cells - 1).astype(np.int64)
    d = hist - f.astype(np.float32)
    assert d.dtype == np.float32
    return f, c, d


def depth_image(cell_rho, cell_s_rho, w, h, bw, bh):
    """(rho, s_rho) float32 [h, w]: v00*(1-dx)*(1-dy) + v10*dx*(1-dy) + v01*(1-dx)*dy + v11*dx*dy left to right in float32,
    with the four cells' values cast to float."""
    xf, xc, dx = img_axis(w, bw, cell_rho.shape[1])
    yf, yc, dy = img_axis(h, bh, cell_rho.shape[0])
    dx, dy = dx[None, :], dy[:, None]
    one = np.float32(1)
    out = []
    for cells in (cell_rho, cell_s_rho):
        g = np.asarray(cells, np.float64).astype(np.float32)
        v00, v10 = g[yf[:, None], xf[None, :]], g[yf[:, None], xc[None, :]]
        v01, v11 = g[yc[:, None], xf[None, :]], g[yc[:, None], xc[None, :]]
        a = v00 * (one - dx) * (one - dy)
        b = v10 * dx * (one - dy)
        c = v01 * (one - dx) * dy
        d = v11 * dx * dy
        r = ((a + b) + c) + d
        assert r.dtype == np.float32
        out.append(r)
    return out[0], out[1]


def _ref():
    from oracle import ref_depth, ref_depth_image
    if not ref_depth_image.available():
        if ref_depth.available():   # the reference was compiled here, so this library must have been too
            pytest.fail("oracle/_ref/libref_depth.so was built but oracle/_ref/libref_depth_image.so was not")
        pytest.skip("oracle/_ref/libref_depth_image.so not built")
    return ref_depth_image


def crafted_grid(rng, gw, gh, kind):
    """Cell values of the kinds a fill produces: fused cells (rho up to 65535 / 1e4, small s_rho), the empty grid's prior
    (rho 1, s_rho 40), zeros, and doubles that are not floats (so the cast to float rounds)."""
    if kind == "random":
        return rng.uniform(0, 6.5535, (gh, gw)), rng.uniform(1e-5, 40, (gh, gw))
    if kind == "extremes":
        rho = rng.choice([0.0, 1e-4, 6.5535, 1.0, 1 / 3, 5e-324, 1e-40, 1e20], (gh, gw))
        s_rho = rng.choice([1e-4 / np.sqrt(200), 40.0, 1e-4, 1e10, 0.0, 2.0 / 3], (gh, gw))
        return rho, s_rho
    if kind == "prior":
        return np.ones((gh, gw)), np.full((gh, gw), 40.0)
    raise ValueError(kind)


def float_exact(ref):
    """getImgRho returns a float widened to double: the float32 planes hold it exactly."""
    f = ref.astype(np.float32)
    assert np.array_equal(f.astype(np.float64), ref, equal_nan=True)
    return f


def assert_bits(got, want, what):
    bad = np.argwhere(got.view(np.uint32) != want.view(np.uint32))
    assert len(bad) == 0, "%s: %d pixels differ, first %s: %r vs %r" % (what, len(bad), bad[0], got[tuple(bad[0])],
                                                                      want[tuple(bad[0])])


# frame sizes and blocks: multiples, remainder columns and rows, 1x1 blocks, gw = 1, gh = 1, one block = the whole frame
CASES = [(80, 60, 10, 10), (83, 67, 10, 10), (64, 48, 16, 16), (71, 53, 7, 13), (40, 30, 1, 1), (45, 31, 40, 4),
         (45, 31, 3, 31), (45, 31, 45, 31), (45, 31, 25, 17), (752, 480, 10, 10), (1241, 376, 16, 16), (33, 32, 2, 3)]


@pytest.mark.parametrize("kind", ["random", "extremes", "prior"])
@pytest.mark.parametrize("w,h,bw,bh", CASES, ids=["%dx%d_b%dx%d" % c for c in CASES])
def test_restatement_equals_get_img_rho(built, w, h, bw, bh, kind):
    ref = _ref()
    gw, gh = w // bw, h // bh
    rng = np.random.default_rng(w * 7 + h * 13 + bw * 17 + bh)
    cr, cs = crafted_grid(rng, gw, gh, kind)
    want_r, want_s = ref.depth_image_cells(w, h, bw, bh, cr, cs)
    got_r, got_s = depth_image(cr, cs, w, h, bw, bh)
    assert_bits(got_r, float_exact(want_r), "rho %dx%d block %dx%d %s" % (w, h, bw, bh, kind))
    assert_bits(got_s, float_exact(want_s), "s_rho %dx%d block %dx%d %s" % (w, h, bw, bh, kind))


def test_clamps_documented():
    """The two clamped cases of the definition, without the reference: left of the first cell centre dx is negative and
    xf = xc = 0; past gw * bw (a remainder column) xf = xc = gw - 1 and dx may exceed 1."""
    xf, xc, dx = img_axis(29, 10, 2)       # 2 cells of 10 px, 9 remainder columns
    assert (xf[:5] == 0).all() and (xc[:5] == 0).all() and (dx[:5] < 0).all() and dx[0] == np.float32(-0.5)
    assert xf[5] == 0 and dx[5] == 0 and xf[14] == 0 and xc[14] == 1
    assert (xf[15:] == 1).all() and (xc[15:] == 1).all() and dx[25] == 1 and (dx[26:] > 1).all()
    # on a one-cell axis every pixel reads the one cell; the weights of the four terms still apply
    xf, xc, dx = img_axis(45, 45, 1)
    assert (xf == 0).all() and (xc == 0).all() and dx[0] == np.float32(-0.5) and dx[44] > 0.47
    r, _ = depth_image(np.array([[1 / 3]]), np.array([[1.0]]), 45, 31, 45, 31)
    assert np.all(np.abs(r - np.float32(1 / 3)) <= 4 * np.finfo(np.float32).eps)
