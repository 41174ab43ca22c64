"""Detection masks without a GPU: the masked restatement (tests/detect_mask.py) is the detector itself with an all-ones
mask, and with partial masks it keeps keylines off zero bytes, keeps the unmasked candidates in raster order and cuts at the
kl_max-th unmasked candidate; the Python wrappers refuse masks that cannot be read in place before they call the library."""
import numpy as np
import pytest

import front_states as fs
from detect_mask import candidates, mask_families, port_detect_masked
from plane_fit import port_detect

CAM = fs.CAM
B = fs.BASE


def _box(a, r):
    """Mean over a (2r+1)^2 window, edges clamped."""
    p = np.pad(a, r, mode="edge")
    c = np.cumsum(np.cumsum(np.pad(p, ((1, 0), (1, 0))), 0), 1)
    k = 2 * r + 1
    return (c[k:, k:] - c[:-k, k:] - c[k:, :-k] + c[:-k, :-k]) / (k * k)


def planes(seed):
    """Float32 (img0, dog) of an edge frame: a smoothed plane and a difference of two smoothings (the masked detector's
    logic needs planes with edges, not the reference's scale space)."""
    g = fs.edge_frame(CAM["w"], CAM["h"], seed).astype(np.float64)
    img0 = _box(_box(g, 1), 1)
    dog = (img0 - _box(_box(g, 2), 1)).astype(np.float32)
    return img0.astype(np.float32), dog


def detect(pl, R, keep, kl_max=40000, tresh=B["tresh"], l_kl_num=0, gain=0.0):
    return port_detect_masked(*pl, R, B["per_hist"], B["dog_thresh"], kl_max, tresh, l_kl_num, B["kl_ref"], gain,
                              B["tmax"], B["tmin"], CAM["ppx"], CAM["ppy"], keep)


def same(a, b):
    assert a[:3] == b[:3]
    assert a[3].tobytes() == b[3].tobytes()
    assert np.array_equal(a[4], b[4])


@pytest.mark.parametrize("R", [1, 2, 3, 4])
def test_all_ones_is_the_detector(R):
    for seed in (3, 11):
        pl = planes(seed)
        want = port_detect(*pl, R, B["per_hist"], B["dog_thresh"], 40000, B["tresh"], 0, B["kl_ref"], 0.0, B["tmax"],
                           B["tmin"], CAM["ppx"], CAM["ppy"])
        assert want[0] > 100
        same(detect(pl, R, None), want)
        same(detect(pl, R, np.ones((CAM["h"], CAM["w"]), np.uint8)), want)
        same(detect(pl, R, np.full((CAM["h"], CAM["w"]), 255, np.uint8)), want)


@pytest.mark.parametrize("R", [1, 2, 3, 4])
def test_partial_masks(R):
    pl = planes(5)
    cand = candidates(*pl, R, B["per_hist"], B["dog_thresh"], B["tresh"])
    kl_max = len(cand) // 2
    for name, keep in mask_families(CAM["w"], CAM["h"], R, cand, kl_max).items():
        kn, _, l, kl, idmask = detect(pl, R, keep, kl_max)
        kept = cand[keep.reshape(-1)[cand] != 0]
        assert l == kn == min(len(kept), kl_max), name
        # the keylines are the first kl_max unmasked candidates in raster order, none on a zero byte
        assert np.array_equal(kl["p_inx"], kept[:kn]), name
        assert np.all(keep.reshape(-1)[kl["p_inx"]] != 0), name
        assert np.array_equal(np.nonzero(idmask.reshape(-1) >= 0)[0], kept[:kn]), name


class _NoLibrary:
    def __getattr__(self, name):
        def call(*a):
            raise AssertionError("the wrapper called %s" % name)
        return call


def _pipeline(w=64, h=48):
    from rebvo_b200 import capi
    pl = object.__new__(capi.Pipeline)
    pl.L, pl.w, pl.h, pl.max_batch, pl.device, pl._out_dev, pl.h_ = _NoLibrary(), w, h, 4, 0, False, None
    return pl


@pytest.mark.parametrize("masks", [
    np.ones((2, 48, 64), np.uint8),                       # host masks: per-frame masks are device memory
    [np.ones((48, 64), np.uint8)],
    [],
], ids=["host_batch", "host_list", "empty"])
def test_mask_table_refuses(masks):
    from rebvo_b200 import capi
    with pytest.raises(ValueError):
        capi.mask_table(masks, 64, 48)


@pytest.mark.parametrize("mask", [
    np.ones((48, 65), np.uint8),                          # shape
    np.ones((48, 64), np.float32),                        # dtype
    np.ones((2, 48, 64), np.uint8),                       # more than one mask
], ids=["shape", "dtype", "batch"])
def test_set_detect_mask_refuses(mask):
    pl = _pipeline()
    with pytest.raises(ValueError):
        pl.set_detect_mask(mask)


def test_push_masked_refuses_host_masks():
    pl = _pipeline()
    with pytest.raises(ValueError):
        pl.push_masked(np.zeros((1, 48, 64, 3), np.uint8), np.ones((1, 48, 64), np.uint8), [0.0])
