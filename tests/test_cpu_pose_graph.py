"""Pose graph file (poses_list.ps, pose_graph::saveToFile, written by rebvorun at exit): rb_odometry_format_pose_graph must
reproduce, byte for byte, the file the unmodified reference writes (oracle/_ref/ref_rebvo_pg with PoseGraphFile=) when it is fed
the reference's own records.  Host code: runs without a GPU."""
import ctypes as C

import numpy as np

from pipeline_util import euroc_stream, run_reference


def test_pose_graph_file_matches_reference(built, tmp_path):
    from oracle import build_pose_graph
    from rebvo_b200 import capi
    ts, fr = euroc_stream(14)
    ps = str(tmp_path / "poses_list.ps")
    run_reference(tmp_path, ts, fr, exe=build_pose_graph.EXE, PoseGraphFile=ps)
    want = open(ps, "rb").read()
    recs = capi.read_pose_graph(ps)
    assert len(recs) >= 10 and len(want) == 4 + 652 * len(recs)
    # vision-only records: K = 1, WK = 0, no IMU measurements, an information matrix that is symmetric
    assert np.all(recs["K"] == 1) and np.all(recs["WK"] == 0) and np.all(recs["KF_ID"] == -1)
    assert not recs["VisualMeas"].any() and not recs["Rs"].any()
    W = recs["WrelPosPose"][1:]
    assert np.allclose(W, W.transpose(0, 2, 1), rtol=1e-9, atol=1e-9 * np.abs(W).max())
    assert capi.format_pose_graph(recs) == want
    # untracked records are not part of the file
    first = np.zeros(1, capi.ODOM)
    assert capi.format_pose_graph(np.concatenate([first, recs])) == want
    assert capi.format_pose_graph(first) == b"\0\0\0\0"
    # capacity handling: too small a buffer reports the size needed and writes nothing beyond it
    need = C.c_size_t(0)
    r = capi.lib().rb_odometry_format_pose_graph(recs.ctypes.data_as(C.c_void_p), len(recs), None, C.c_size_t(0),
                                                  C.byref(need))
    assert r != 0 and need.value == len(want)
    buf = C.create_string_buffer(b"\xab" * len(want))
    r = capi.lib().rb_odometry_format_pose_graph(recs.ctypes.data_as(C.c_void_p), len(recs), buf, C.c_size_t(len(want) - 1),
                                                  C.byref(need))
    assert r != 0 and need.value == len(want) and buf.raw[len(want) - 1:len(want)] == b"\xab"
    assert capi.lib().rb_odometry_format_pose_graph(None, -1, None, C.c_size_t(0), C.byref(need)) != 0
