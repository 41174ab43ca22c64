"""TEST INFRASTRUCTURE ONLY.  Recipe for oracle/_ref/ref_rebvo_pg: the level-B reference (the unmodified 3-thread REBVO,
oracle/build_ref.py) driven by oracle/ref_driver.cpp through oracle/ref_pose_graph.cpp, which also saves REBVO::poses
(pose_graph::saveToFile, the reference's poses_list.ps) to PoseGraphFile=path.  Links the level-B objects
build_ref.build(level_b=True) compiled; like that recipe it does nothing where the reference sources are absent (the GPU box
uses the prebuilt executable)."""
import os

from oracle import build_ref

HERE = os.path.dirname(os.path.abspath(__file__))
EXE = os.path.join(build_ref.OUT, "ref_rebvo_pg")


def build(force=False):
    if not os.path.isdir(build_ref.REF):
        return False
    src = os.path.join(HERE, "ref_pose_graph.cpp")
    objs = [os.path.join(build_ref.OUT, "obj", "b_%s.o" % os.path.basename(n)) for n in build_ref.B_NAMES]
    objs.append(os.path.join(build_ref.OUT, "obj", "b_stubs.o"))
    deps = [src, os.path.join(HERE, "ref_driver.cpp"), __file__] + objs
    if not force and os.path.exists(EXE) and all(os.path.getmtime(EXE) > os.path.getmtime(d) for d in deps):
        return True
    toon = os.path.join(build_ref.OUT, "toon")
    shim = os.path.join(build_ref.OUT, "shim")
    blas_dir, blas = build_ref.openblas()
    # build_ref.build's level-B compile flags (the reference's own: rebvolib/Makefile:16-17) and link line, in its order (the
    # driver's object last), so that this executable is ref_rebvo plus the save
    drv = os.path.join(build_ref.OUT, "obj", "pg_ref_pose_graph.o")
    build_ref.run(["g++", "-std=c++11", "-O2", "-m64", "-fPIC", "-w", "-include", os.path.join(shim, "fix_gcc13.h"),
                   "-I" + shim, "-I" + os.path.join(build_ref.REF, "include"), "-I" + os.path.join(build_ref.REF, "src"),
                   "-I" + toon, "-c", src, "-o", drv])
    build_ref.run(["g++", "-o", EXE] + objs + [drv, blas, "-Wl,-rpath," + blas_dir, "-Wl,--allow-shlib-undefined",
                                                "-lpthread"])
    return True


if __name__ == "__main__":
    print(build(force=True))
