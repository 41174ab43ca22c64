"""Drop-in boundary test: tests/shim_driver.cpp = the reference's FirstThr/SecondThread call sequence written
against include/rebvo_b200_shim.hpp (same class and method names as the reference's mtracklib) and compiled with
the reference's non-hot-path headers.  Its trajectory must equal rb_pipeline_push's and the reference's."""
import os
import subprocess

import numpy as np
import pytest

from pipeline_util import assert_shim_equals, euroc_stream, frames_file, run_pipeline, run_reference

pytestmark = pytest.mark.gpu
NF = 30


def test_shim_classes_reproduce_reference_flow(built, tmp_path):
    from oracle import refapi
    from rebvo_b200 import capi, synth
    exe = os.path.join(os.path.dirname(refapi.EXE), "shim_driver")
    if not os.path.exists(exe):
        pytest.skip("oracle/_ref/shim_driver not built (needs the reference headers)")
    ts, fr = euroc_stream(NF, seed=9)
    path = frames_file(tmp_path, ts, fr)
    r = subprocess.run([refapi.runnable(exe, str(tmp_path)), path, path + ".shim"], capture_output=True, text=True,
                       timeout=600, env=refapi.lib_env())
    assert r.returncode == 0, r.stderr[-2000:]
    with open(path + ".shim", "rb") as f:
        n, sz = np.frombuffer(f.read(8), np.int32)
        assert sz == refapi.OUTREC.itemsize
        shim = np.frombuffer(f.read(), refapi.OUTREC, count=n)
    nav = run_pipeline(capi.default_params(synth.EUROC), ts, fr, 10).nav
    assert len(shim) == NF
    assert_shim_equals(nav, shim)
    assert np.abs(shim["PoseLie"] - nav["PoseLie"]).max() <= 1e-9
    ref = run_reference(tmp_path, ts, fr, required=False)
    if ref is not None:
        rec = ref[1]
        m = min(len(rec), NF - 1)
        assert np.array_equal(rec["kn"][:m], shim["kn"][:m])
        ate = float(np.sqrt(((rec["Pos"][:m] - shim["Pos"][:m]) ** 2).sum(1).mean()))
        print("shim vs reference ATE %.3e m" % ate)
        assert ate <= 1e-7
