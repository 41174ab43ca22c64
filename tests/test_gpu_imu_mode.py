"""Config 3 (IMU fusion, ImuMode=2: gyro pre-rotation, Minimizer_V, ExtRotVel, BiasCorrect, scale / gravity / bias
filter) end to end.  The reference's own SecondThread IMU branch (rebvo_second_t.cpp:182-336, unmodified, with its
ScaleEstimator and ImuGrabber) runs once on the reference's CPU hot path (oracle/_ref/ref_rebvo) and once on
librebvo_b200 through the shim (oracle/_ref/shim_rebvo): same frames, same synthetic IMU csv."""
import os

import numpy as np
import pytest

from pipeline_util import assert_knife_edge, euroc_sequence, run_pipeline, run_reference, shim_exe

pytestmark = pytest.mark.gpu
NF = 50


def test_imu_mode_trajectory(built, tmp_path):
    from oracle import refapi
    from rebvo_b200 import synth
    if not (os.path.exists(shim_exe()) and os.path.exists(refapi.EXE)):
        pytest.skip("oracle/_ref/shim_rebvo / ref_rebvo not built (need the reference sources)")
    seq = euroc_sequence()
    ts, fr = seq.frames(NF)
    imu = synth.imu_samples(seq, NF)
    _, ref = run_reference(tmp_path, ts, fr, imu=imu)
    _, rec = run_reference(tmp_path, ts, fr, exe=shim_exe(), imu=imu)
    n = min(len(ref), len(rec))
    print("IMU mode: K ref %s gpu %s" % (ref["K"][n - 1], rec["K"][n - 1]))
    assert np.isfinite(ref["Pos"][:n]).all() and np.isfinite(rec["Pos"][:n]).all()
    assert_knife_edge(ref, rec, NF - 2, "IMU mode")
    assert np.allclose(ref["K"][:n], rec["K"][:n], rtol=1e-6, atol=1e-12)


def test_imu_mode_pipeline_vs_reference(built, tmp_path):
    """The product's own IMU-mode flow (rb_pipeline_set_imu: csrc/imu_flow.cuh + imu_filter.h) against the reference's CPU
    build with ImuMode=2 on the same frames and the same synthetic IMU samples."""
    from rebvo_b200 import capi, synth
    seq = euroc_sequence()
    ts, fr = seq.frames(NF)
    imu = synth.imu_samples(seq, NF)
    p = capi.default_params(synth.EUROC)
    _, ref = run_reference(tmp_path, ts, fr, p, imu=imu)
    nav = run_pipeline(p, ts, fr, 10, imu=imu).nav
    n = min(len(ref), len(nav))
    print("IMU pipeline: K ref %.12g gpu %.12g" % (ref["K"][n - 1], nav["K"][n - 1]))
    assert np.isfinite(nav["Pos"][:n]).all()
    assert_knife_edge(ref, nav, NF - 2, "IMU pipeline")
    assert np.allclose(ref["K"][1:n], nav["K"][1:n], rtol=1e-6, atol=1e-12)   # (record 0 is the untracked first frame)
    assert np.abs(ref["PoseLie"][:n] - nav["PoseLie"][:n]).max() <= 1e-3
