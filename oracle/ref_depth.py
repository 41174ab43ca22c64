"""TEST INFRASTRUCTURE ONLY.  Recipe and ctypes binding of oracle/_ref/libref_depth.so: the unmodified reference depth_filler
(src/visualizer/depth_filler.cpp, compiled where it lies with build_ref's level-B flags) and oracle/ref_depth.cpp, which runs
the viewer's per-packet sequence (visualizer.cpp:436-440) on net_keyline records.  Like build_ref, build() does nothing where
the reference sources are absent (the GPU box uses the prebuilt library).

A library of its own rather than two more translation units in libref_mtrack.so: build_ref.py, ref_shim.cpp and refapi.py
stay as they are, and this one only compiles the unmodified depth_filler.cpp with build_ref's level-B flags (rebvolib's own)
plus the window below; it links with --no-undefined, so nothing else of the reference is pulled in."""
import ctypes as C
import os

import numpy as np

from oracle import build_ref

HERE = os.path.dirname(os.path.abspath(__file__))
LIB = os.path.join(build_ref.OUT, "libref_depth.so")


def build(force=False):
    if not os.path.isdir(build_ref.REF):
        return False
    srcs = [os.path.join(HERE, "ref_depth.cpp"), os.path.join(build_ref.REF, "src", "visualizer", "depth_filler.cpp")]
    # (and the headers whose inline code the fill runs: get3DPos, Img2Hom, Image::GetIndex, struct net_keyline)
    inc = os.path.join(build_ref.REF, "include")
    deps = srcs + [__file__] + [os.path.join(inc, h) for h in ("visualizer/depth_filler.h", "UtilLib/cam_model.h",
                                                               "VideoLib/image.h", "VideoLib/video_io.h",
                                                               "CommLib/net_keypoint.h")]
    if not force and os.path.exists(LIB) and all(os.path.getmtime(LIB) > os.path.getmtime(d) for d in deps):
        return True
    toon = os.path.join(build_ref.OUT, "toon")
    shim = os.path.join(build_ref.OUT, "shim")
    if not os.path.isdir(os.path.join(toon, "TooN")) or not os.path.exists(os.path.join(shim, "fix_gcc13.h")):
        raise RuntimeError("run oracle/build_ref.py first (TooN and the include shims)")
    os.makedirs(os.path.join(build_ref.OUT, "obj"), exist_ok=True)
    # the reference's own flags (rebvolib/Makefile:16-17), as build_ref.build
    cxx = ["g++", "-std=c++11", "-O2", "-m64", "-fPIC", "-w", "-include", os.path.join(shim, "fix_gcc13.h"), "-I" + shim,
           "-I" + os.path.join(build_ref.REF, "include"), "-I" + os.path.join(build_ref.REF, "src"), "-I" + toon]
    objs = []
    for s in srcs:
        o = os.path.join(build_ref.OUT, "obj", "d_" + os.path.basename(s).replace(".cpp", ".o"))
        build_ref.run(cxx + ["-c", s, "-o", o])
        objs.append(o)
    build_ref.run(["g++", "-shared", "-o", LIB] + objs + ["-Wl,--no-undefined", "-lm"])
    return True


_lib = None


def available():
    return os.path.exists(LIB)


def lib():
    global _lib
    if _lib is None:
        _lib = C.CDLL(LIB)
        _lib.ref_depth_fill_net.argtypes = [C.c_int, C.c_int, C.c_float, C.c_float, C.c_float, C.c_float, C.c_int, C.c_int,
                                            C.c_double, C.c_int, C.c_int, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p,
                                            C.c_void_p, C.c_void_p, C.c_void_p]
    return _lib


def depth_fill_net(cam, records, block_w, block_h, thresh_rel_rho, thresh_match_num, iter_num):
    """The reference's depth grid of uint8 [n, 15] net_keyline records: dict of gh x gw arrays rho, s_rho, dist, fixed
    (int32) and the float min_dist (depth_filler::GetMinDist)."""
    rec = np.ascontiguousarray(records, np.uint8).reshape(-1, 15)
    gw, gh = cam["w"] // block_w, cam["h"] // block_h
    out = {k: np.zeros((gh, gw), np.float64) for k in ("rho", "s_rho", "dist")}
    out["fixed"] = np.zeros((gh, gw), np.int32)
    md = C.c_double(0)
    r = lib().ref_depth_fill_net(cam["w"], cam["h"], cam["ppx"], cam["ppy"], cam["zfx"], cam["zfy"], block_w, block_h,
                                 float(thresh_rel_rho), int(thresh_match_num), int(iter_num),
                                 rec.ctypes.data_as(C.c_void_p), len(rec),
                                 *(out[k].ctypes.data_as(C.c_void_p) for k in ("rho", "s_rho", "dist", "fixed")),
                                 C.byref(md))
    if r:
        raise RuntimeError("ref_depth_fill_net failed (%d)" % r)
    out["min_dist"] = md.value
    return out


if __name__ == "__main__":
    print(build(force=True))
