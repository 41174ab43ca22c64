"""On-disk formats of the third thread (SURVEY.md 8(f) rank 4): rb_nav_format_trajectory / rb_nav_format_log must reproduce,
byte for byte, the TrayFile and the pose / map records of the LogFile the unmodified reference writes (SaveLog=1,
rebvo_third_t.cpp:259-311, 373-397) when they are fed the values of the reference's own output callbacks.  Host code: runs
without a GPU."""
import numpy as np

from pipeline_util import euroc_stream, run_reference


LOG_KEYS = ("Kp_cv", "RKp_cv", "Rot_cv", "Vel_cv", "t_cv", "dt_cv", "i_cv", "Pose_cv", "Pos_cv", "K_cv", "KLN_cv")


def test_trajectory_and_log_files_match_reference(built, tmp_path):
    from rebvo_b200 import capi
    ts, fr = euroc_stream(14)
    tray, log = str(tmp_path / "tray.txt"), str(tmp_path / "log.m")
    info, rec = run_reference(tmp_path, ts, fr, SaveLog=1, TrayFile=tray, LogFile=log)
    assert len(rec) >= 10
    nav = np.zeros(len(rec), capi.NAV)
    for k in ("t", "dt", "Pos", "PoseLie", "Pose", "Rot", "Vel", "K", "Kp", "RKp", "kn"):
        nav[k] = rec[k]
    want = open(tray).read()
    got = capi.format_trajectory(nav, 1.0)
    assert want.count("\n") == len(rec)
    assert got == want
    # a line is "t x y z  qx qy qz qw " with 18 digits: the TUM evaluation tools' format
    tok = want.splitlines()[3].split()
    assert len(tok) == 8 and all("e" in t and len(t.split("e")[0].lstrip("-")) == 20 for t in tok)
    want_log = "".join(l + "\n" for l in open(log).read().splitlines() if l.split("(")[0] in LOG_KEYS)
    got_log = capi.format_log(nav, first_index=1, frame_id0=int(rec["p_id"][0]))
    assert np.array_equal(rec["p_id"], rec["p_id"][0] + np.arange(len(rec)))
    assert got_log == want_log
    # capacity handling: too small a buffer reports the size needed
    import ctypes as C
    need = C.c_size_t(0)
    r = capi.lib().rb_nav_format_trajectory(nav.ctypes.data_as(C.c_void_p), len(nav), C.c_double(1.0), None, C.c_size_t(0), C.byref(need))
    assert r != 0 and need.value == len(want)
