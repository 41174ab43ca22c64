"""TEST INFRASTRUCTURE ONLY.  Recipe and bindings of the reference in live IMU mode (ImuMode=1):

  oracle/_ref/ref_live_imu           oracle/ref_live_imu.cpp on the compiled reference (build_ref's level-B objects)
  oracle/_ref/shim_live_imu          the same driver on the shim (build_shim_rebvo's objects, librebvo_b200.so)
  oracle/_ref/libref_imu_grabber.so  the unmodified ImuGrabber (src/UtilLib/imugrabber.cpp) + oracle/ref_imu_grabber.cpp

Files of their own, like ref_depth.py: build_ref.py and ref_driver.cpp stay as they are.  The drivers link the objects
build_ref.build and build_ref.build_shim_rebvo leave in oracle/_ref/obj, so build() runs after those.  Like build_ref, it does
nothing where the reference sources are absent (the GPU box uses the prebuilt files)."""
import ctypes as C
import os

import numpy as np

from oracle import build_ref

HERE = os.path.dirname(os.path.abspath(__file__))
EXE = os.path.join(build_ref.OUT, "ref_live_imu")
SHIM_EXE = os.path.join(build_ref.OUT, "shim_live_imu")
GRABBER_LIB = os.path.join(build_ref.OUT, "libref_imu_grabber.so")
DRIVER = os.path.join(HERE, "ref_live_imu.cpp")


def _fresh(out, deps):
    return os.path.exists(out) and all(os.path.getmtime(out) > os.path.getmtime(d) for d in deps)


def build(force=False):
    if not os.path.isdir(build_ref.REF):
        return False
    out, ref = build_ref.OUT, build_ref.REF
    toon, shim = os.path.join(out, "toon"), os.path.join(out, "shim")
    if not os.path.isdir(os.path.join(toon, "TooN")) or not os.path.exists(os.path.join(shim, "fix_gcc13.h")):
        raise RuntimeError("run oracle/build_ref.py first (TooN and the include shims)")
    obj = os.path.join(out, "obj")
    os.makedirs(obj, exist_ok=True)
    blas_dir, blas = build_ref.openblas()
    link = [blas, "-Wl,-rpath," + blas_dir, "-Wl,--allow-shlib-undefined", "-lpthread"]
    # the reference's own flags (rebvolib/Makefile:16-17), as build_ref.build
    base = ["g++", "-std=c++11", "-O2", "-m64", "-fPIC", "-w", "-include", os.path.join(shim, "fix_gcc13.h")]
    cxx_ref = base + ["-I" + shim, "-I" + os.path.join(ref, "include"), "-I" + os.path.join(ref, "src"), "-I" + toon]

    # the ImuGrabber binding: imugrabber.cpp and what LoadDataSet calls (Configurator::ShrinkWS)
    srcs = [os.path.join(HERE, "ref_imu_grabber.cpp"), os.path.join(ref, "src", "UtilLib", "imugrabber.cpp"),
            os.path.join(ref, "src", "UtilLib", "configurator.cpp")]
    if force or not _fresh(GRABBER_LIB, srcs + [__file__]):
        objs = []
        for s in srcs:
            o = os.path.join(obj, "g_" + os.path.basename(s).replace(".cpp", ".o"))
            build_ref.run(cxx_ref + ["-c", s, "-o", o])
            objs.append(o)
        build_ref.run(["g++", "-shared", "-o", GRABBER_LIB] + objs + ["-Wl,--no-undefined", "-lpthread"])

    # the driver on the compiled reference: build_ref.build's level-B objects without its ref_driver.cpp
    b_objs = [os.path.join(obj, "b_" + os.path.basename(n) + ".o") for n in build_ref.B_NAMES] + [os.path.join(obj, "b_stubs.o")]
    if force or not _fresh(EXE, [DRIVER, __file__] + b_objs):
        o = os.path.join(obj, "b_ref_live_imu.o")
        build_ref.run(cxx_ref + ["-c", DRIVER, "-o", o])
        build_ref.run(["g++", "-o", EXE] + b_objs + [o] + link)

    # the driver on the shim: build_ref.build_shim_rebvo's objects (the reference's non-hot-path TUs on the include overlay)
    repo = os.path.dirname(HERE)
    lib = os.path.join(repo, "rebvo_b200", "librebvo_b200.so")
    s_objs = [os.path.join(obj, "s_" + os.path.basename(n) + ".o") for n in build_ref.B_NAMES
              if n not in build_ref.HOT_PATH_TUS] + [os.path.join(obj, "s_stubs.o")]
    if force or not _fresh(SHIM_EXE, [DRIVER, __file__, lib, os.path.join(repo, "include", "rebvo_b200_shim.hpp")] + s_objs):
        cxx_shim = base + ["-I" + os.path.join(out, "include_overlay"), "-I" + os.path.join(repo, "include"), "-I" + shim,
                           "-I" + os.path.join(ref, "src"), "-I" + toon]
        o = os.path.join(obj, "s_ref_live_imu.o")
        build_ref.run(cxx_shim + ["-c", DRIVER, "-o", o])
        build_ref.run(["g++", "-o", SHIM_EXE] + s_objs + [o] + build_ref.link_gpu_lib(lib) + link)
    return True


def write_samples(path, samples):
    """The raw sample file of ref_live_imu (ImuSamples=): float64 rows {t, gyro xyz, accel xyz}."""
    np.ascontiguousarray(samples, np.float64).reshape(-1, 7).tofile(path)


def run(frames_file, samples, out_file, params=None, exe=None, sample_time=0.005, buffer_size=1000, timeout=600):
    """(info, records) of the reference in live IMU mode on a raw frame file: ref_live_imu (default) or SHIM_EXE, with the
    samples pushed frame by frame.  params: the key=value arguments of refapi.run_full_rebvo (refapi.ref_params_from)."""
    from oracle import refapi
    imu = out_file + ".imu"
    write_samples(imu, samples)
    kv = dict(params or {})
    kv.update(ImuSamples=imu, SampleTime=float(sample_time), CircBufferSize=int(buffer_size))
    try:
        return refapi.run_full_rebvo(frames_file, out_file, kv, timeout=timeout, exe=exe or EXE)
    finally:
        os.remove(imu)


_lib = None


def available():
    return os.path.exists(GRABBER_LIB)


def lib():
    global _lib
    if _lib is None:
        _lib = C.CDLL(GRABBER_LIB)
        _lib.ref_imu_grabber_new.restype = C.c_void_p
        _lib.ref_imu_grabber_new.argtypes = [C.c_int, C.c_double]
        _lib.ref_imu_grabber_free.argtypes = [C.c_void_p]
        _lib.ref_imu_grabber_push.argtypes = [C.c_void_p, C.c_void_p, C.c_int]
        _lib.ref_imu_grabber_grab.argtypes = [C.c_void_p, C.c_double, C.c_double, C.c_void_p]
    return _lib


class Grabber:
    """The reference's ImuGrabber(list_size, tsamp): push(rows) -> number stored before PushData's overflow_error;
    grab(tstart, tend) -> GrabAndIntegrate as 23 doubles {n, dt, Rot, giro, acel, cacel, dgiro}."""

    def __init__(self, list_size, tsample):
        self.h = lib().ref_imu_grabber_new(int(list_size), float(tsample))

    def push(self, rows):
        rows = np.ascontiguousarray(rows, np.float64).reshape(-1, 7)
        return lib().ref_imu_grabber_push(self.h, rows.ctypes.data_as(C.c_void_p), len(rows))

    def grab(self, tstart, tend):
        out = np.zeros(23)
        lib().ref_imu_grabber_grab(self.h, float(tstart), float(tend), out.ctypes.data_as(C.c_void_p))
        return out

    def close(self):
        if self.h:
            lib().ref_imu_grabber_free(self.h)
            self.h = None


if __name__ == "__main__":
    print(build(force=True))
