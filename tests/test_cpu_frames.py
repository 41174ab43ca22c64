"""Pipeline.push_frames' layout rules without a GPU: capi.frame_table turns per-frame arrays or one array of frames into the
rb_frame table of rb_pipeline_push_frames(_dev) -- format, memory, and one {data, step} per frame -- and refuses with
ValueError every layout it cannot pass as it is."""
import numpy as np
import pytest

from rebvo_b200 import capi

W, H = 40, 33


class FakeDev:
    """A device array as __cuda_array_interface__ describes it (the pointer is never dereferenced)."""

    def __init__(self, ptr, shape, strides=None, typestr="|u1"):
        self.__cuda_array_interface__ = dict(shape=shape, strides=strides, typestr=typestr, data=(ptr, False), version=3)


def base(a):
    return a.__array_interface__["data"][0]


def test_packed_batch():
    rgb = np.zeros((5, H, W, 3), np.uint8)
    fmt, dev, tbl = capi.frame_table(rgb, W, H)
    assert (fmt, dev) == (capi.FRAME_RGB24, False)
    assert tbl == [(base(rgb) + i * 3 * W * H, 3 * W) for i in range(5)]
    mono = np.zeros((2, H, W), np.uint8)
    fmt, dev, tbl = capi.frame_table(mono, W, H)
    assert fmt == capi.FRAME_MONO8 and tbl == [(base(mono) + i * W * H, W) for i in range(2)]


def test_views_and_lists():
    big = np.zeros((H + 10, W + 17, 3), np.uint8)
    crop = big[3:3 + H, 5:5 + W]
    fmt, dev, tbl = capi.frame_table([crop, crop], W, H)
    assert fmt == capi.FRAME_RGB24 and tbl == [(base(big) + 3 * (W + 17) * 3 + 5 * 3, 3 * (W + 17))] * 2
    # frames in reverse order in one buffer: a negative frame stride is fine, each frame has its own pointer
    buf = np.zeros((4, H, W + 3), np.uint8)[::-1, :, 1:1 + W]
    fmt, dev, tbl = capi.frame_table(buf, W, H)
    assert fmt == capi.FRAME_MONO8
    assert [p for p, _ in tbl] == [base(buf) - i * H * (W + 3) for i in range(4)] and {s for _, s in tbl} == {W + 3}
    # per-frame steps differ
    a, b = np.zeros((H, W + 1), np.uint8)[:, :W], np.zeros((H, 512), np.uint8)[:, :W]
    assert [s for _, s in capi.frame_table([a, b], W, H)[2]] == [W + 1, 512]


def test_device_frames():
    fmt, dev, tbl = capi.frame_table([FakeDev(1001, (H, W, 3), (512, 3, 1)), FakeDev(77, (H, W, 3))], W, H)
    assert (fmt, dev) == (capi.FRAME_RGB24, True) and tbl == [(1001, 512), (77, 3 * W)]
    fmt, dev, tbl = capi.frame_table(FakeDev(4096, (3, H, W), (-H * 64, 64, 1)), W, H)
    assert (fmt, dev) == (capi.FRAME_MONO8, True) and tbl == [(4096 - i * H * 64, 64) for i in range(3)]


@pytest.mark.parametrize("bad", [
    np.zeros((H, W, 3), np.uint8)[:, ::2][:, :W // 2],                 # wrong shape
    np.zeros((H, 2 * W, 3), np.uint8)[:, ::2],                          # pixel stride 6
    np.zeros((H, W, 4), np.uint8)[..., :3],                             # pixel stride 4 (RGBA buffer)
    np.zeros((H, W, 3), np.uint8)[..., ::-1],                           # channel stride -1 (BGR view)
    np.zeros((H, W), np.uint8).T.copy().T,                              # column-major mono: pixel stride H
    np.zeros((H, W), np.uint8)[::-1],                                   # bottom-up: negative step
    np.zeros((H, W), np.uint16),                                        # dtype
    np.zeros((H, W), np.uint8).tolist(),                                # not an array
])
def test_refused_layouts(bad):
    with pytest.raises(ValueError):
        capi.frame_table([bad], W, H)


def test_refused_mixes():
    host, dev = np.zeros((H, W), np.uint8), FakeDev(64, (H, W))
    with pytest.raises(ValueError):
        capi.frame_table([host, dev], W, H)
    with pytest.raises(ValueError):
        capi.frame_table([np.zeros((H, W, 3), np.uint8), host], W, H)
    with pytest.raises(ValueError):
        capi.frame_table([], W, H)
    with pytest.raises(ValueError):
        capi.frame_table(np.zeros((0, H, W), np.uint8), W, H)
    with pytest.raises(ValueError):
        capi.frame_table(FakeDev(64, (H, W), typestr="<f4"), W, H)


def test_torch_host_tensor_refused():
    """A torch tensor in host memory is neither a NumPy array nor a device frame: no silent conversion."""
    torch = pytest.importorskip("torch")
    with pytest.raises(ValueError):
        capi.frame_table([torch.zeros((H, W), dtype=torch.uint8)], W, H)
