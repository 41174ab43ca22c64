"""TEST INFRASTRUCTURE ONLY.  Recipe and ctypes binding of oracle/_ref/libref_depth_image.so: the unmodified reference
depth_filler (src/visualizer/depth_filler.cpp, compiled where it lies with build_ref's level-B flags) and
oracle/ref_depth_image.cpp, which samples a grid at every pixel with the header's own depth_filler::getImgRho.  Like
build_ref, build() does nothing where the reference sources are absent (the GPU box uses the prebuilt library).

A library of its own next to libref_depth.so, so that ref_depth.cpp and its recipe stay as they are; it links with
--no-undefined, so nothing else of the reference is pulled in."""
import ctypes as C
import os

import numpy as np

from oracle import build_ref

HERE = os.path.dirname(os.path.abspath(__file__))
LIB = os.path.join(build_ref.OUT, "libref_depth_image.so")


def build(force=False):
    if not os.path.isdir(build_ref.REF):
        return False
    srcs = [os.path.join(HERE, "ref_depth_image.cpp"), os.path.join(build_ref.REF, "src", "visualizer", "depth_filler.cpp")]
    # (and the headers whose inline code the fill and the sampling run: getImgRho, get3DPos, Img2Hom, Image, net_keyline)
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
        o = os.path.join(build_ref.OUT, "obj", "di_" + os.path.basename(s).replace(".cpp", ".o"))
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
        _lib.ref_depth_image_net.argtypes = [C.c_int, C.c_int, C.c_float, C.c_float, C.c_float, C.c_float, C.c_int, C.c_int,
                                             C.c_double, C.c_int, C.c_int, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p]
        _lib.ref_depth_image_cells.argtypes = [C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p,
                                               C.c_void_p]
    return _lib


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def depth_image_net(cam, records, block_w, block_h, thresh_rel_rho, thresh_match_num, iter_num):
    """(rho, s_rho): h x w float64 arrays of getImgRho at every pixel of the reference's depth grid of uint8 [n, 15]
    net_keyline records (the viewer's sequence, as ref_depth.depth_fill_net)."""
    rec = np.ascontiguousarray(records, np.uint8).reshape(-1, 15)
    rho, s_rho = np.zeros((cam["h"], cam["w"])), np.zeros((cam["h"], cam["w"]))
    r = lib().ref_depth_image_net(cam["w"], cam["h"], cam["ppx"], cam["ppy"], cam["zfx"], cam["zfy"], block_w, block_h,
                                  float(thresh_rel_rho), int(thresh_match_num), int(iter_num), _p(rec), len(rec),
                                  _p(rho), _p(s_rho))
    if r:
        raise RuntimeError("ref_depth_image_net failed (%d)" % r)
    return rho, s_rho


def depth_image_cells(w, h, block_w, block_h, cell_rho, cell_s_rho):
    """(rho, s_rho): h x w float64 arrays of getImgRho at every pixel of a grid whose gh x gw cells (gw = w // block_w,
    gh = h // block_h) are written straight into depth_filler::data."""
    gw, gh = w // block_w, h // block_h
    cr = np.ascontiguousarray(cell_rho, np.float64).reshape(gh, gw)
    cs = np.ascontiguousarray(cell_s_rho, np.float64).reshape(gh, gw)
    rho, s_rho = np.zeros((h, w)), np.zeros((h, w))
    lib().ref_depth_image_cells(w, h, block_w, block_h, _p(cr), _p(cs), _p(rho), _p(s_rho))
    return rho, s_rho


if __name__ == "__main__":
    print(build(force=True))
