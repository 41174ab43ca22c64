"""Asynchronous pushes without a GPU: the ctypes prototypes of rb_pipeline_set_async / enqueue / enqueue_frames / wait / poll
are the header's, the Python wrappers refuse a bad format or shape before they call the library, and a pipeline still
cannot be created without a device."""
import ctypes as C
import os
import re

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

# the C parameter types of these calls as ctypes sees them
C_TYPES = {"rb_pipeline *": C.c_void_p, "int": C.c_int, "int64_t": C.c_int64, "int64_t *": C.POINTER(C.c_int64),
           "const uint8_t *": C.c_void_p, "const double *": C.c_void_p, "const rb_frame *": C.c_void_p,
           "rb_nav *": C.c_void_p}


def _declarations():
    hdr = open(os.path.join(ROOT, "include", "rebvo_b200.h")).read()
    hdr = re.sub(r"/\*.*?\*/", "", hdr, flags=re.S)
    out = {}
    for ret, name, params in re.findall(r"\b(int)\s+(rb_pipeline_(?:set_async|enqueue\w*|wait|poll))\s*\(([^)]*)\)\s*;", hdr):
        types = []
        for prm in params.split(","):
            prm = " ".join(prm.split())
            m = re.match(r"(.*?)\s*\b\w+$", prm)
            types.append(m.group(1).strip())
        out[name] = (ret, types)
    return out


def test_prototypes_match_the_header():
    from rebvo_b200 import capi
    decl = _declarations()
    assert sorted(decl) == sorted(capi.PROTOTYPES) == ["rb_pipeline_enqueue", "rb_pipeline_enqueue_frames",
                                                       "rb_pipeline_poll", "rb_pipeline_set_async", "rb_pipeline_wait"]
    for name, (ret, types) in decl.items():
        res, args = capi.PROTOTYPES[name]
        assert res is C.c_int and ret == "int", name
        assert [C_TYPES[t] for t in types] == args, (name, types)
        assert name in capi.SYMBOLS


class _NoLibrary:
    """Stands for the library: any call into it fails the test."""

    def __getattr__(self, name):
        def call(*a):
            raise AssertionError("the wrapper called %s" % name)
        return call


def _pipeline(w=64, h=48, max_batch=4):
    from rebvo_b200 import capi
    pl = object.__new__(capi.Pipeline)
    pl.L, pl.w, pl.h, pl.max_batch, pl.device, pl._out_dev, pl.h_ = _NoLibrary(), w, h, max_batch, 0, False, None
    return pl


@pytest.mark.parametrize("frames,ts,fmt", [
    (np.zeros((2, 48, 64, 3), np.uint8), [0.0, 0.1], "bgr"),            # unknown format
    (np.zeros((2, 48, 64, 3), np.uint8), [0.0, 0.1], "mono"),           # RGB frames as mono
    (np.zeros((2, 48, 64), np.uint8), [0.0, 0.1], "rgb"),               # mono frames as RGB
    (np.zeros((2, 48, 64, 3), np.uint16), [0.0, 0.1], "rgb"),           # dtype
    (np.zeros((2, 48, 63, 3), np.uint8), [0.0, 0.1], "rgb"),            # width
    (np.zeros((3, 48, 64, 3), np.uint8), [0.0, 0.1], "rgb"),            # frames != timestamps
    (np.zeros((5, 48, 64), np.uint8), [0.0] * 5, "mono"),               # more than max_batch
    (np.zeros((0, 48, 64), np.uint8), [], "mono"),                      # none
    ([np.zeros((48, 64), np.uint8)] * 2, [0.0, 0.1], "rgb"),            # strided mono frames as RGB
    ([np.zeros((48, 64, 3), np.uint8)] * 2, [0.0], "rgb"),              # strided: frames != timestamps
    ([np.zeros((48, 64, 3), np.uint8)[:, ::2]] * 2, [0.0, 0.1], "rgb"),  # strided: pixel stride
    ("frames", [0.0], "rgb"),                                           # not an array
])
def test_enqueue_refuses_bad_frames_before_the_library(frames, ts, fmt):
    pl = _pipeline()
    with pytest.raises(ValueError):
        pl.enqueue(frames, ts, fmt)


def test_enqueue_arguments_of_good_frames():
    """What the wrapper would pass: packed host frames in place (a copy only for non-contiguous ones), strided frames as a
    table; the objects it keeps alive until the wait."""
    from rebvo_b200 import capi
    pl = _pipeline()
    rgb = np.zeros((3, 48, 64, 3), np.uint8)
    fn, args, keep, on_dev = pl._enqueue_args(rgb, [0, 1, 2], "rgb")
    assert callable(fn)
    assert args[:2] == (capi.FRAME_RGB24, 0) and args[2].value == rgb.__array_interface__["data"][0] and not on_dev
    assert keep[0] is rgb
    mono = np.zeros((2, 48, 128), np.uint8)[:, :, ::2]
    _, args, keep, _ = pl._enqueue_args(mono, [0, 1], "mono")
    assert keep[0].flags.c_contiguous and args[2].value == keep[0].__array_interface__["data"][0]
    frames = [np.zeros((48, 80, 3), np.uint8)[:, :64] for _ in range(2)]
    _, args, keep, _ = pl._enqueue_args(frames, [0, 1], "rgb")
    assert args[:2] == (capi.FRAME_RGB24, 0) and keep[0] is frames and keep[1]["step"].tolist() == [240, 240]


def test_create_without_a_device_still_fails(built):
    import torch
    from rebvo_b200 import capi, synth
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    with pytest.raises(capi.RbError):
        capi.Pipeline(capi.default_params(synth.EUROC), max_batch=2)
