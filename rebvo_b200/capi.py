"""ctypes binding of librebvo_b200.so (include/rebvo_b200.h).  No fallback: if the CUDA library is missing
or no CUDA device is present the calls raise."""
import ctypes as C
import os

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("REBVO_B200_LIB") or os.path.join(HERE, "librebvo_b200.so")   # (override: A/B builds of tools/build_alt.py)


class RbError(RuntimeError):
    pass


class Camera(C.Structure):
    _fields_ = [("w", C.c_int32), ("h", C.c_int32), ("ppx", C.c_float), ("ppy", C.c_float),
                ("zfx", C.c_float), ("zfy", C.c_float)]


class DetectParams(C.Structure):
    _fields_ = [("plane_fit_size", C.c_int32), ("pos_neg_thresh", C.c_double), ("dog_thresh", C.c_double),
                ("kl_max", C.c_int32), ("kl_ref", C.c_int32), ("gain", C.c_double),
                ("thresh_max", C.c_double), ("thresh_min", C.c_double)]


class Params(C.Structure):
    _fields_ = [("cam", Camera), ("Sigma0", C.c_double), ("KSigma", C.c_double), ("det", DetectParams),
                ("DetectorThresh", C.c_double), ("TrackPoints", C.c_int32), ("QCutOffNumBins", C.c_int32),
                ("QCutOffQuantile", C.c_double), ("SearchRange", C.c_int32), ("TrackerIterNum", C.c_int32),
                ("TrackerInitIterNum", C.c_int32), ("TrackerInitType", C.c_int32),
                ("TrackerMatchThresh", C.c_double), ("LocationUncertaintyMatch", C.c_double),
                ("MatchThreshModule", C.c_double), ("MatchThreshAngle", C.c_double),
                ("ReweigthDistance", C.c_double), ("MatchNumThresh", C.c_uint32), ("MatchThreshold", C.c_int32),
                ("RegularizeThresh", C.c_double), ("ReshapeQAbsolute", C.c_double),
                ("ReshapeQRelative", C.c_double), ("LocationUncertainty", C.c_double),
                ("DoReScaling", C.c_double), ("config_fps", C.c_double), ("kl_capacity", C.c_int32)]


class ImuParams(C.Structure):
    """rb_imu_params (include/rebvo_b200.h); defaults = the IMU block of app/rebvorun/GlobalConfig_EuRoC_2.txt"""
    _fields_ = [("TimeDesinc", C.c_double), ("InitBias", C.c_int32), ("InitBiasFrameNum", C.c_int32),
                ("BiasInitGuess", C.c_double * 3), ("GiroMeasStdDev", C.c_double), ("GiroBiasStdDev", C.c_double),
                ("AcelMeasStdDev", C.c_double), ("g_module", C.c_double), ("g_module_uncer", C.c_double),
                ("g_uncert", C.c_double), ("VBiasStdDev", C.c_double), ("ScaleStdDevInit", C.c_double),
                ("use_se3", C.c_int32), ("pad", C.c_int32), ("Rc2i", C.c_double * 9), ("Tc2i", C.c_double * 3)]


def default_imu_params(**over):
    p = ImuParams()
    p.TimeDesinc, p.InitBias, p.InitBiasFrameNum = 0.0, 0, 10
    p.GiroMeasStdDev, p.GiroBiasStdDev, p.AcelMeasStdDev = 1.6968e-4, 1.9393e-5, 2e-3
    p.g_module, p.g_module_uncer, p.g_uncert, p.VBiasStdDev, p.ScaleStdDevInit = 9.8, 100e3, 2e-3, 1e-7, 1.2e-3
    for k, v in over.items():
        setattr(p, k, v)
    return p


NAV = np.dtype([("t", "f8"), ("dt", "f8"), ("Rot", "f8", 9), ("RotLie", "f8", 3), ("Vel", "f8", 3),
                ("Pose", "f8", 9), ("PoseLie", "f8", 3), ("Pos", "f8", 3), ("V", "f8", 3), ("W", "f8", 3),
                ("K", "f8"), ("Kp", "f8"), ("RKp", "f8"), ("s_rho_p", "f8"), ("score", "f8"), ("kn", "i4"),
                ("matches", "i4"), ("fwd_matches", "i4"), ("estimation_ok", "i4"), ("thresh", "f4"),
                ("retuned_thresh", "f4")])

# struct KeyLine of the reference (168 bytes) == rb_keyline
KEYLINE = np.dtype({
    "names": ["p_inx", "m_m", "u_m", "n_m", "score", "c_p", "rho", "s_rho", "rho_nr", "s_rho_nr",
              "rho0", "s_rho0", "p_m", "p_m_0", "m_id", "m_id_f", "m_id_kf", "m_num", "m_m0", "n_m0",
              "p_id", "n_id", "net_id", "stereo_m_id", "stereo_rho", "stereo_s_rho"],
    "formats": ["i4", ("f4", 2), ("f4", 2), "f4", "f4", ("f4", 2), "f8", "f8", "f8", "f8", "f8", "f8",
                ("f4", 2), ("f4", 2), "i4", "i4", "i4", "i4", ("f4", 2), "f8", "i4", "i4", "i4", "i4",
                "f8", "f8"],
    "offsets": [0, 4, 12, 20, 24, 28, 40, 48, 56, 64, 72, 80, 88, 96, 104, 108, 112, 116, 120, 128,
                136, 140, 144, 148, 152, 160],
    "itemsize": 168})

# every symbol include/rebvo_b200.h declares
SYMBOLS = ["rb_ctx_create", "rb_ctx_destroy", "rb_last_error", "rb_ctx_sync", "rb_ctx_box_plan",
           "rb_ctx_launch_count", "rb_map_create", "rb_map_destroy", "rb_map_clone", "rb_map_upload_rgb", "rb_map_upload_mono",
           "rb_map_upload_gray",
           "rb_map_dog_build", "rb_map_get_plane", "rb_map_detect", "rb_map_detect_ss", "rb_map_reestimate_thresh", "rb_map_knum",
           "rb_map_counters",
           "rb_map_sync_host_keylines", "rb_map_load_keylines", "rb_map_get_mask", "rb_map_quantile",
           "rb_map_build_field", "rb_map_get_field", "rb_try_vel_rot", "rb_minimizer_rv", "rb_forward_match",
           "rb_map_rotate_keylines", "rb_directed_matching", "rb_map_regularize", "rb_map_ekf_update",
           "rb_map_rescale_opt", "rb_map_set_frame_count", "rb_pipeline_create", "rb_pipeline_destroy",
           "rb_pipeline_last_error", "rb_pipeline_push", "rb_pipeline_push_dev", "rb_pipeline_push_mono",
           "rb_pipeline_push_mono_dev", "rb_pipeline_reset",
           "rb_pipeline_map", "rb_pipeline_launch_count", "rb_pipeline_stage_ms", "rb_pipeline_stream",
           "rb_pipeline_event_record", "rb_pipeline_event_elapsed", "rb_pipeline_event_elapsed_between", "rb_pipeline_bench_pass",
           "rb_pipeline_set_imu", "rb_pipeline_set_mirror", "rb_pipeline_mirror", "rb_pipeline_set_undistort",
           "rb_pipeline_stage_profile",
           "rb_undistort_create", "rb_undistort_destroy", "rb_undistort_rgb", "rb_undistort_rgb_dev",
           "rb_try_vel", "rb_minimizer_v", "rb_ext_rot_vel", "rb_bias_correct", "rb_map_pack_net_keylines",
           "rb_nav_format_trajectory", "rb_nav_format_log", "rb_map_scale_space_path"]

_lib = None


def _format_nav(fn, nav, *args):
    nav = np.ascontiguousarray(nav, NAV)
    need = C.c_size_t(0)
    getattr(lib(), fn)(_p(nav), len(nav), *args, None, C.c_size_t(0), C.byref(need))
    buf = C.create_string_buffer(max(need.value, 1))
    r = getattr(lib(), fn)(_p(nav), len(nav), *args, buf, C.c_size_t(need.value), C.byref(need))
    if r:
        raise RbError("%s failed (%d)" % (fn, r))
    return buf.raw[:need.value].decode()


def format_trajectory(nav, time_scale=1.0):
    """Text of the reference's trajectory file (TrayFile, rebvo_third_t.cpp:311) for these NAV records."""
    return _format_nav("rb_nav_format_trajectory", nav, C.c_double(time_scale))


def format_log(nav, first_index=1, frame_id0=0):
    """Pose / map records of the reference's m-file log (LogFile, rebvo_third_t.cpp:265-281) for these NAV records."""
    return _format_nav("rb_nav_format_log", nav, C.c_longlong(first_index), C.c_longlong(frame_id0))


def lib():
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise RbError("librebvo_b200.so is not built (run `python -c 'import __graft_entry__ as g; g.build()'`); "
                          "there is no CPU fallback")
        L = C.CDLL(LIB_PATH)
        L.rb_last_error.restype = C.c_char_p
        L.rb_pipeline_last_error.restype = C.c_char_p
        L.rb_ctx_launch_count.restype = C.c_int64
        L.rb_pipeline_launch_count.restype = C.c_int64
        L.rb_pipeline_map.restype = C.c_void_p
        L.rb_pipeline_stream.restype = C.c_void_p
        _lib = L
    return _lib


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def default_params(cam, **over):
    """REBVOParameters subset; defaults = app/rebvorun/GlobalConfig_EuRoC_2.txt with TrackerInitType=2."""
    p = Params()
    p.cam = Camera(cam["w"], cam["h"], cam["ppx"], cam["ppy"], cam["zfx"], cam["zfy"])
    p.Sigma0, p.KSigma = 3.56359, 1.2599
    p.det = DetectParams(2, 0.4, 0.095259868922420, 40000, 15000, 5e-7, 0.5, 0.005)
    p.DetectorThresh = 0.01
    p.TrackPoints = 12000
    p.QCutOffNumBins = 100
    p.QCutOffQuantile = 0.9
    p.SearchRange = 40
    p.TrackerIterNum, p.TrackerInitIterNum, p.TrackerInitType = 5, 2, 2
    p.TrackerMatchThresh = 0.5
    p.LocationUncertaintyMatch, p.MatchThreshModule, p.MatchThreshAngle = 2, 1, 45
    p.ReweigthDistance = 2
    p.MatchNumThresh = 0
    p.MatchThreshold = 500
    p.RegularizeThresh, p.ReshapeQAbsolute, p.ReshapeQRelative, p.LocationUncertainty = 0.5, 1e-4, 1.6968e-4, 1
    p.DoReScaling = 0
    p.config_fps = 20
    p.kl_capacity = 40000
    for k, v in over.items():
        if hasattr(p.det, k):
            setattr(p.det, k, v)
        else:
            setattr(p, k, v)
    return p


class Ctx:
    def __init__(self, cam, sigma0, ksigma, kl_capacity=50000, device=0):
        self.L = lib()
        self.cam = Camera(cam["w"], cam["h"], cam["ppx"], cam["ppy"], cam["zfx"], cam["zfy"])
        self.w, self.h = cam["w"], cam["h"]
        h = C.c_void_p()
        r = self.L.rb_ctx_create(C.byref(h), device, C.byref(self.cam), C.c_double(sigma0), C.c_double(ksigma),
                                 kl_capacity)
        self.h_ = h
        if r:
            msg = self.L.rb_last_error(h).decode() if h else ""
            raise RbError("rb_ctx_create failed (%d) %s" % (r, msg))
        self.kcap = kl_capacity

    def check(self, r):
        if r:
            raise RbError("librebvo_b200 error %d: %s" % (r, self.L.rb_last_error(self.h_).decode()))

    def box_plan(self):
        d = np.zeros(6, np.int32)
        s = np.zeros(2)
        self.check(self.L.rb_ctx_box_plan(self.h_, _p(d), _p(s)))
        return d.reshape(2, 3), s

    def launches(self):
        return self.L.rb_ctx_launch_count(self.h_)

    def new_map(self):
        return Map(self)

    def close(self):
        if self.h_:
            self.L.rb_ctx_destroy(self.h_)
            self.h_ = None


class Undistort:
    """image_undistort of the reference (rad-tan model, 16.16 fixed-point bilinear RGB remap)."""

    def __init__(self, ctx, kc):
        self.ctx = ctx
        kc = np.ascontiguousarray(kc, np.float64)
        h = C.c_void_p()
        ctx.check(ctx.L.rb_undistort_create(ctx.h_, _p(kc), C.byref(h)))
        self.h_ = h

    def apply(self, rgb):
        rgb = np.ascontiguousarray(rgb, np.uint8)
        out = np.empty_like(rgb)
        self.ctx.check(self.ctx.L.rb_undistort_rgb(self.h_, _p(rgb), _p(out)))
        return out

    def close(self):
        if self.h_:
            self.ctx.L.rb_undistort_destroy(self.h_)
            self.h_ = None


class Map:
    def __init__(self, ctx, handle=None):
        self.ctx, self.L = ctx, ctx.L
        self.owned = handle is None
        if handle is None:
            h = C.c_void_p()
            ctx.check(self.L.rb_map_create(ctx.h_, C.byref(h)))
            handle = h
        self.h_ = handle
        self.w, self.h = ctx.w, ctx.h

    def close(self):
        if self.h_ and self.owned:
            self.L.rb_map_destroy(self.h_)
        self.h_ = None

    def clone(self):
        h = C.c_void_p()
        self.ctx.check(self.L.rb_map_clone(self.h_, C.byref(h)))
        m = Map(self.ctx, h)
        m.owned = True
        return m

    def upload_rgb(self, rgb):
        rgb = np.ascontiguousarray(rgb, np.uint8)
        assert rgb.size == self.w * self.h * 3
        self.ctx.check(self.L.rb_map_upload_rgb(self.h_, _p(rgb)))
        self.ctx.check(self.L.rb_ctx_sync(self.ctx.h_))

    def upload_mono(self, img):
        """8-bit grayscale frame (h, w): the RGB24 frame (img, img, img) as far as the gray plane is concerned."""
        img = np.ascontiguousarray(img, np.uint8)
        assert img.size == self.w * self.h
        self.ctx.check(self.L.rb_map_upload_mono(self.h_, _p(img)))
        self.ctx.check(self.L.rb_ctx_sync(self.ctx.h_))

    def upload_gray(self, g):
        g = np.ascontiguousarray(g, np.float32)
        self.ctx.check(self.L.rb_map_upload_gray(self.h_, _p(g)))
        self.ctx.check(self.L.rb_ctx_sync(self.ctx.h_))

    def dog_build(self):
        self.ctx.check(self.L.rb_map_dog_build(self.h_))

    def plane(self, which):
        idx = {"img0": 0, "img1": 1, "dog": 2, "dx": 3, "dy": 4, "gray": 5}[which]
        out = np.empty((self.h, self.w), np.float32)
        self.ctx.check(self.L.rb_map_get_plane(self.h_, idx, _p(out)))
        return out

    def detect(self, det, tresh, l_kl_num):
        t, l, kn = C.c_double(tresh), C.c_int(l_kl_num), C.c_int(0)
        self.ctx.check(self.L.rb_map_detect(self.h_, C.byref(det), C.byref(t), C.byref(l), C.byref(kn)))
        return kn.value, t.value, l.value

    def reestimate(self, knum, nbins):
        o = C.c_float(0)
        self.ctx.check(self.L.rb_map_reestimate_thresh(self.h_, knum, nbins, C.byref(o)))
        return o.value

    def knum(self):
        k = C.c_int(0)
        self.ctx.check(self.L.rb_map_knum(self.h_, C.byref(k)))
        return k.value

    def counters(self):
        """(fwd_match, nmatch, reg_num) of the frame that built this map"""
        out = (C.c_int * 3)()
        self.ctx.check(self.L.rb_map_counters(self.h_, out))
        return tuple(out)

    def keylines(self):
        kn = self.knum()
        out = np.zeros(max(kn, 1), KEYLINE)
        k = C.c_int(0)
        self.ctx.check(self.L.rb_map_sync_host_keylines(self.h_, _p(out), len(out), C.byref(k)))
        return out[:kn]

    def scale_space_path(self):
        """bit 0: row passes on TMA tiles, bit 1: last box + DoG on TMA tiles (after dog_build)."""
        return int(self.L.rb_map_scale_space_path(self.h_))

    def pack_net(self, k_prof=1.0, capacity=None):
        """15-byte net_keyline records (uint8 array [n, 15]) packed on the device."""
        cap = capacity if capacity is not None else max(self.knum(), 1)
        out = np.zeros((cap, 15), np.uint8)
        k = C.c_int(0)
        self.ctx.check(self.L.rb_map_pack_net_keylines(self.h_, C.c_double(k_prof), _p(out), cap, C.byref(k)))
        return out[:k.value]

    def load_keylines(self, kl, mask):
        kl = np.ascontiguousarray(kl, KEYLINE)
        mask = np.ascontiguousarray(mask, np.int32)
        self.ctx.check(self.L.rb_map_load_keylines(self.h_, _p(kl), len(kl), _p(mask)))

    def mask(self):
        out = np.empty((self.h, self.w), np.int32)
        self.ctx.check(self.L.rb_map_get_mask(self.h_, _p(out)))
        return out

    def quantile(self, smin, smax, perc, n):
        o = C.c_double(0)
        self.ctx.check(self.L.rb_map_quantile(self.h_, C.c_double(smin), C.c_double(smax), C.c_double(perc), n,
                                              C.byref(o)))
        return o.value

    def build_field(self, radius, min_mod):
        self.ctx.check(self.L.rb_map_build_field(self.h_, radius, C.c_float(min_mod)))

    def field(self):
        out = np.empty((self.h, self.w, 2), np.int32)
        self.ctx.check(self.L.rb_map_get_field(self.h_, _p(out)))
        return out

    def set_frame_count(self, fc):
        self.ctx.check(self.L.rb_map_set_frame_count(self.h_, C.c_uint32(fc)))

    def try_vel_rot(self, old, X, reweight, procjf, match_thresh, s_rho_min, match_num_thresh, k_huber, res_in):
        X = np.array(X, np.float64)
        kn = old.knum()
        res_in = np.ascontiguousarray(res_in[:kn], np.float64)
        res_out = np.full(kn, np.nan)
        JtJ, JtF, s = np.zeros((6, 6)), np.zeros(6), C.c_double(0)
        self.ctx.check(self.L.rb_try_vel_rot(self.h_, old.h_, _p(X), int(reweight), int(procjf),
                                             C.c_double(match_thresh), C.c_double(s_rho_min),
                                             C.c_uint32(match_num_thresh), C.c_double(k_huber), _p(res_in),
                                             _p(res_out), _p(JtJ), _p(JtF), C.byref(s)))
        return s.value, JtJ, JtF, res_out

    def minimizer_rv(self, old, V, W, match_thresh, iter_max, init_type, reweight, max_s_rho, match_num_thresh,
                     init_iter):
        V, W = np.array(V, np.float64), np.array(W, np.float64)
        RV, RW, WX = np.zeros((3, 3)), np.zeros((3, 3)), np.zeros((6, 6))
        e1, e2, sc = C.c_double(0), C.c_double(0), C.c_double(0)
        self.ctx.check(self.L.rb_minimizer_rv(self.h_, old.h_, _p(V), _p(W), _p(RV), _p(RW),
                                              C.c_double(match_thresh), iter_max, init_type, C.c_double(reweight),
                                              C.byref(e1), C.byref(e2), C.c_double(max_s_rho),
                                              C.c_uint32(match_num_thresh), int(init_iter), _p(WX), C.byref(sc)))
        return dict(F=sc.value, V=V, W=W, RVel=RV, RW0=RW, W_X=WX, rel_err=e1.value, rel_err_score=e2.value)

    def try_vel(self, old, V, match_thresh, s_rho_min, match_num_thresh, residuals, rw_dist, min_mod):
        V = np.array(V, np.float64)
        res = np.ascontiguousarray(residuals[:old.knum()], np.float64).copy()
        JtJ, JtF, s = np.zeros((3, 3)), np.zeros(3), C.c_double(0)
        self.ctx.check(self.L.rb_try_vel(self.h_, old.h_, _p(V), C.c_double(match_thresh), C.c_double(s_rho_min),
                                         C.c_uint32(match_num_thresh), _p(res), C.c_double(rw_dist), C.c_float(min_mod),
                                         _p(JtJ), _p(JtF), C.byref(s)))
        return s.value, JtJ, JtF, res

    def minimizer_v(self, old, V, match_thresh, iter_max, s_rho_min, match_num_thresh, rw_dist, min_mod):
        V = np.array(V, np.float64)
        RV, s = np.zeros((3, 3)), C.c_double(0)
        self.ctx.check(self.L.rb_minimizer_v(self.h_, old.h_, _p(V), _p(RV), C.c_double(match_thresh), iter_max,
                                             C.c_double(s_rho_min), C.c_uint32(match_num_thresh), C.c_double(rw_dist),
                                             C.c_float(min_mod), C.byref(s)))
        return dict(F=s.value, V=V, RVel=RV)

    def ext_rot_vel(self, V, loc_unc, hub):
        V = np.array(V, np.float64)
        Wx, Rx, X, ok = np.zeros((6, 6)), np.zeros((6, 6)), np.zeros(6), C.c_int(0)
        self.ctx.check(self.L.rb_ext_rot_vel(self.h_, _p(V), _p(Wx), _p(Rx), _p(X), C.c_double(loc_unc),
                                             C.c_double(hub), C.byref(ok)))
        return bool(ok.value), Wx, Rx, X

    def forward_match(self, new):
        n = C.c_int(0)
        self.ctx.check(self.L.rb_forward_match(self.h_, new.h_, C.byref(n)))
        return n.value

    def rotate(self, R):
        R = np.ascontiguousarray(R, np.float64)
        self.ctx.check(self.L.rb_map_rotate_keylines(self.h_, _p(R)))

    def directed_matching(self, old, V, RVel, BackRot, thr_mod, thr_ang, max_radius, loc_unc):
        V = np.ascontiguousarray(V, np.float64)
        RVel = np.ascontiguousarray(RVel, np.float64)
        BackRot = np.ascontiguousarray(BackRot, np.float64)
        n = C.c_int(0)
        self.ctx.check(self.L.rb_directed_matching(self.h_, old.h_, _p(V), _p(RVel), _p(BackRot),
                                                   C.c_double(thr_mod), C.c_double(thr_ang),
                                                   C.c_double(max_radius), C.c_double(loc_unc), C.byref(n)))
        return n.value

    def regularize(self, thresh):
        n = C.c_int(0)
        self.ctx.check(self.L.rb_map_regularize(self.h_, C.c_double(thresh), C.byref(n)))
        return n.value

    def ekf(self, V, qabs, loc_unc):
        V = np.ascontiguousarray(V, np.float64)
        self.ctx.check(self.L.rb_map_ekf_update(self.h_, _p(V), C.c_double(qabs), C.c_double(loc_unc)))

    def rescale(self, s_rho_min, match_num_min, re_escale):
        kp, rkp = C.c_double(0), C.c_double(0)
        self.ctx.check(self.L.rb_map_rescale_opt(self.h_, C.c_double(s_rho_min), C.c_uint32(match_num_min),
                                                 int(re_escale), C.byref(kp), C.byref(rkp)))
        return kp.value, rkp.value


class Pipeline:
    """REBVO per-frame flow on one GPU (rb_pipeline_*)."""

    def __init__(self, params, max_batch=32, device=0):
        self.L = lib()
        self.params = params
        self.w, self.h = params.cam.w, params.cam.h
        self.max_batch = max_batch
        h = C.c_void_p()
        r = self.L.rb_pipeline_create(C.byref(h), device, C.byref(params), max_batch)
        self.h_ = h
        if r:
            msg = self.L.rb_pipeline_last_error(h).decode() if h else ""
            raise RbError("rb_pipeline_create failed (%d) %s" % (r, msg))

    def check(self, r):
        if r:
            raise RbError("librebvo_b200 error %d: %s" % (r, self.L.rb_pipeline_last_error(self.h_).decode()))

    def push(self, rgb, ts):
        """rgb: (n,h,w,3) uint8 host array (or a raw host pointer int with n given by len(ts))."""
        ts = np.ascontiguousarray(ts, np.float64)
        n = len(ts)
        nav = np.zeros(n, NAV)
        if isinstance(rgb, np.ndarray):
            rgb = np.ascontiguousarray(rgb, np.uint8)
            ptr = _p(rgb)
        else:
            ptr = C.c_void_p(int(rgb))
        self.check(self.L.rb_pipeline_push(self.h_, ptr, _p(ts), n, _p(nav)))
        return nav

    def push_mono(self, frames, ts):
        """frames: (n,h,w) uint8 host array of 8-bit grayscale frames (or a raw host pointer int with n given by len(ts)).
        Same records as push() of the frames replicated into three channels."""
        ts = np.ascontiguousarray(ts, np.float64)
        n = len(ts)
        nav = np.zeros(n, NAV)
        if isinstance(frames, np.ndarray):
            frames = np.ascontiguousarray(frames, np.uint8)
            ptr = _p(frames)
        else:
            ptr = C.c_void_p(int(frames))
        self.check(self.L.rb_pipeline_push_mono(self.h_, ptr, _p(ts), n, _p(nav)))
        return nav

    def push_mono_dev(self, dev_ptr, ts):
        """Mono frames already in device memory (4-byte aligned pointer), read in place."""
        ts = np.ascontiguousarray(ts, np.float64)
        nav = np.zeros(len(ts), NAV)
        self.check(self.L.rb_pipeline_push_mono_dev(self.h_, C.c_void_p(int(dev_ptr)), _p(ts), len(ts), _p(nav)))
        return nav

    def set_imu(self, samples, imu_params=None):
        """IMU mode (BASELINE configs[2]): samples = float64 [n, 7] rows {t, gyro xyz, accel xyz}."""
        samples = np.ascontiguousarray(samples, np.float64)
        ip = imu_params if imu_params is not None else default_imu_params()
        self.check(self.L.rb_pipeline_set_imu(self.h_, C.byref(ip), _p(samples), len(samples)))

    def push_dev(self, dev_ptr, ts):
        ts = np.ascontiguousarray(ts, np.float64)
        nav = np.zeros(len(ts), NAV)
        self.check(self.L.rb_pipeline_push_dev(self.h_, C.c_void_p(int(dev_ptr)), _p(ts), len(ts), _p(nav)))
        return nav

    def reset(self):
        self.check(self.L.rb_pipeline_reset(self.h_))

    def launches(self):
        return self.L.rb_pipeline_launch_count(self.h_)

    def stage_ms(self):
        out = np.zeros(6, np.float32)
        self.check(self.L.rb_pipeline_stage_ms(self.h_, _p(out)))
        return out

    def stream(self):
        return self.L.rb_pipeline_stream(self.h_)

    def event_record(self, slot):
        self.check(self.L.rb_pipeline_event_record(self.h_, slot))

    def event_elapsed_from(self, other, a, b):
        """ms between event a of pipeline `other` and event b of this pipeline (pipelines sharing a GPU)."""
        ms = C.c_float(0)
        self.check(self.L.rb_pipeline_event_elapsed_between(other.h_, a, self.h_, b, C.byref(ms)))
        return ms.value

    def event_elapsed(self, a, b):
        ms = C.c_float(0)
        self.check(self.L.rb_pipeline_event_elapsed(self.h_, a, b, C.byref(ms)))
        return ms.value

    def stage_profile(self):
        out = np.zeros(16)
        fr = C.c_longlong(0)
        self.check(self.L.rb_pipeline_stage_profile(self.h_, _p(out), C.byref(fr)))
        names = ["copies", "gray", "scale_space", "detect", "reestimate", "quantile+field", "minimizer",
                 "fwdmatch+rotate", "directed_match", "regularize+ekf", "rescale", "pose/nav", "nav_copy"]
        return {n: 1e3 * out[i] / max(fr.value, 1) for i, n in enumerate(names)}, fr.value

    def bench_pass(self, pass_id, nimg, iters):
        ms, by = C.c_float(0), C.c_double(0)
        self.check(self.L.rb_pipeline_bench_pass(self.h_, pass_id, nimg, iters, C.byref(ms), C.byref(by)))
        return ms.value, by.value

    def set_undistort(self, kc):
        """UseUndistort=1 with kc = (KcR2, KcR4, KcR6, KcP1, KcP2); None / zeros = off."""
        if kc is None:
            self.check(self.L.rb_pipeline_set_undistort(self.h_, None))
        else:
            a = np.ascontiguousarray(kc, np.float64)
            assert a.shape == (5,)
            self.check(self.L.rb_pipeline_set_undistort(self.h_, _p(a)))

    def set_mirror(self, mode=1):
        """Per-frame host mirror of the edge map, written while the following frames are tracked: mode 1 = the reference's 168-byte KeyLine
        records, 2 = its 15-byte net_keyline wire records, 0 = off."""
        self.check(self.L.rb_pipeline_set_mirror(self.h_, int(mode)))
        self._mirror_mode = int(mode)

    def mirror(self, i):
        """View (no copy) of the records of frame `i` of the last push: KEYLINE[n] (mode 1) or uint8[n, 15] (mode 2); valid until
        the next push."""
        p, kn = C.c_void_p(0), C.c_int(0)
        self.check(self.L.rb_pipeline_mirror(self.h_, i, C.byref(p), C.byref(kn)))
        net = getattr(self, "_mirror_mode", 1) == 2
        if kn.value == 0:
            return np.zeros((0, 15), np.uint8) if net else np.zeros(0, KEYLINE)
        rec = 15 if net else KEYLINE.itemsize
        buf = (C.c_char * (kn.value * rec)).from_address(p.value)
        if net:
            return np.frombuffer(buf, dtype=np.uint8).reshape(kn.value, 15)
        return np.frombuffer(buf, dtype=KEYLINE, count=kn.value)

    def map(self, age=0):
        """Edge map of the ring: age 0 = newest.  Returns a Map view bound to a throw-away context facade."""
        h = self.L.rb_pipeline_map(self.h_, age)
        if not h:
            return None
        facade = _CtxFacade(self)
        return Map(facade, handle=C.c_void_p(h))

    def close(self):
        if self.h_:
            self.L.rb_pipeline_destroy(self.h_)
            self.h_ = None


class _CtxFacade:
    def __init__(self, pl):
        self.L, self.w, self.h, self.pl = pl.L, pl.w, pl.h, pl
        self.h_ = None

    def check(self, r):
        self.pl.check(r)
