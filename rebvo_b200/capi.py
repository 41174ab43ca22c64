"""ctypes binding of librebvo_b200.so (include/rebvo_b200.h).  No fallback: if the CUDA library is missing
or no CUDA device is present the calls raise."""
import collections
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

# rb_odometry: the reference's OdometryMeas (pose graph record) + whether the frame was tracked
ODOM = np.dtype([("relPosPose", "f8", 6), ("WrelPosPose", "f8", (6, 6)), ("AcelMeas", "f8", 3), ("VisualMeas", "f8", 3),
                 ("GMeas", "f8", 3), ("Rs", "f8", (3, 3)), ("Rv", "f8", (3, 3)), ("Rg", "f8", (3, 3)), ("K", "f8"),
                 ("WK", "f8"), ("QK", "f8"), ("KF_ID", "i4"), ("tracked", "i4")])
# one record of the pose graph file (pose_graph::saveToFile): ODOM without `tracked`, unpadded
PS_REC = np.dtype([(n, ODOM.fields[n][0]) for n in ODOM.names if n != "tracked"])

# rb_match_update_out: what the per-frame map chain leaves besides the two maps (rb_map_match_update)
MATCH_UPDATE_OUT = np.dtype([("nmatch", "i4"), ("fwd_match", "i4"), ("reg_num", "i4"), ("do_map", "i4"), ("est_ok", "i4"),
                             ("klm_num", "i4"), ("V", "f8", 3), ("Kp", "f8"), ("P_Kp", "f8"), ("P_V", "f8", (3, 3)),
                             ("Pose", "f8", (3, 3)), ("Pos", "f8", 3), ("RotLie", "f8", 3), ("PoseLie", "f8", 3)])

# rb_depth_cell: one cell of the viewer's depth grid (depth_filler's df_point rho, s_rho, dist, fixed)
DEPTH_CELL = np.dtype([("rho", "f8"), ("s_rho", "f8"), ("dist", "f8"), ("fixed", "i4"), ("_pad", "i4")])


class DepthParams(C.Structure):
    """rb_depth_params: depth_filler's block size and the viewer's DF_ThreshRelRho, DF_ThreshMatchNum, DF_IterNum."""
    _fields_ = [("block_w", C.c_int32), ("block_h", C.c_int32), ("thresh_rel_rho", C.c_double),
                ("thresh_match_num", C.c_int32), ("iter_num", C.c_int32)]


def depth_params(block_w=10, block_h=10, thresh_rel_rho=1.0, thresh_match_num=5, iter_num=10):
    """DepthParams; the defaults are every shipped viewer configuration's (visualizer.cpp:303, ThreshRelRho=1,
    ThreshMatchNum=5, IterNum=10)."""
    return DepthParams(block_w, block_h, thresh_rel_rho, thresh_match_num, iter_num)


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
           "rb_ctx_launch_count", "rb_ctx_minimizer_clusters", "rb_map_create", "rb_map_destroy", "rb_map_clone", "rb_map_upload_rgb", "rb_map_upload_mono",
           "rb_map_upload_gray",
           "rb_map_dog_build", "rb_map_get_plane", "rb_map_detect", "rb_map_detect_ss", "rb_map_reestimate_thresh", "rb_map_knum",
           "rb_map_counters",
           "rb_map_sync_host_keylines", "rb_map_load_keylines", "rb_map_get_mask", "rb_map_quantile",
           "rb_map_build_field", "rb_map_get_field", "rb_try_vel_rot", "rb_minimizer_rv", "rb_minimizer_rv_forward", "rb_forward_match",
           "rb_map_rotate_keylines", "rb_directed_matching", "rb_map_regularize", "rb_map_ekf_update",
           "rb_map_rescale_opt", "rb_map_set_frame_count", "rb_map_match_update", "rb_pipeline_create", "rb_pipeline_destroy",
           "rb_pipeline_last_error", "rb_pipeline_push", "rb_pipeline_push_dev", "rb_pipeline_push_mono",
           "rb_pipeline_push_mono_dev", "rb_pipeline_reset",
           "rb_pipeline_map", "rb_pipeline_launch_count", "rb_pipeline_stage_ms", "rb_pipeline_stream",
           "rb_pipeline_event_record", "rb_pipeline_event_elapsed", "rb_pipeline_event_elapsed_between", "rb_pipeline_bench_pass",
           "rb_pipeline_set_imu", "rb_pipeline_set_imu_live", "rb_pipeline_push_imu", "rb_pipeline_set_mirror", "rb_pipeline_mirror", "rb_pipeline_set_undistort",
           "rb_pipeline_stage_profile",
           "rb_undistort_create", "rb_undistort_destroy", "rb_undistort_rgb", "rb_undistort_rgb_dev",
           "rb_try_vel", "rb_minimizer_v", "rb_ext_rot_vel", "rb_bias_correct", "rb_map_pack_net_keylines",
           "rb_nav_format_trajectory", "rb_nav_format_log", "rb_odometry_format_pose_graph", "rb_pipeline_set_odometry",
           "rb_pipeline_odometry", "rb_depth_fill_net", "rb_pipeline_set_depth", "rb_pipeline_depth", "rb_depth_image",
           "rb_pipeline_set_depth_image", "rb_pipeline_depth_image", "rb_pipeline_set_output_memory",
           "rb_pipeline_set_consumer_stream", "rb_pipeline_mirror_dev", "rb_pipeline_depth_dev", "rb_pipeline_depth_image_dev",
           "rb_pipeline_push_frames", "rb_pipeline_push_frames_dev", "rb_pipeline_batch_plane", "rb_pipeline_save_state",
           "rb_pipeline_load_state", "rb_state_info", "rb_pipeline_set_async", "rb_pipeline_enqueue",
           "rb_pipeline_enqueue_frames", "rb_pipeline_wait", "rb_pipeline_poll", "rb_map_detect_masked",
           "rb_pipeline_set_detect_mask", "rb_pipeline_push_masked", "rb_pipeline_masked_enqueue"]

# ctypes prototypes of the asynchronous pushes (their tickets are int64_t, which ctypes' default conversion would cut to int)
PROTOTYPES = {
    "rb_pipeline_set_async": (C.c_int, [C.c_void_p, C.c_int]),
    "rb_pipeline_enqueue": (C.c_int, [C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_int, C.POINTER(C.c_int64)]),
    "rb_pipeline_enqueue_frames": (C.c_int, [C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_int,
                                             C.POINTER(C.c_int64)]),
    "rb_pipeline_wait": (C.c_int, [C.c_void_p, C.c_int64, C.c_void_p]),
    "rb_pipeline_poll": (C.c_int, [C.c_void_p, C.POINTER(C.c_int64)]),
}

_lib = None


# rb_frame: the first byte of row 0 and the bytes from one row to the next
FRAME = np.dtype([("data", "<u8"), ("step", "<i8")])


FRAME_RGB24, FRAME_MONO8 = 0, 1


def _array_layout(a):
    """(on_device, shape, byte strides, dtype is uint8, address of element 0) of a NumPy array, a torch CUDA tensor or an
    object with __cuda_array_interface__ (torch tensors are read directly: building the interface dict costs more than
    the rest of a frame's checks)"""
    if isinstance(a, np.ndarray):
        return False, a.shape, a.strides, a.dtype == np.uint8, a.__array_interface__["data"][0]
    if type(a).__module__.startswith("torch") and hasattr(a, "data_ptr"):
        if not a.is_cuda:
            raise ValueError("frames: a torch tensor in host memory (pass tensor.numpy())")
        return True, tuple(a.shape), tuple(a.stride()), str(a.dtype) == "torch.uint8", a.data_ptr()
    if not hasattr(a, "__cuda_array_interface__"):
        raise ValueError("frames: NumPy arrays (host) or CUDA arrays (__cuda_array_interface__), not %s" % type(a).__name__)
    ai = a.__cuda_array_interface__
    shape, strides = tuple(ai["shape"]), ai.get("strides")
    if strides is None:   # C-contiguous
        strides = tuple(int(np.prod(shape[k + 1:], dtype=np.int64)) * np.dtype(ai["typestr"]).itemsize
                        for k in range(len(shape)))
    return True, shape, tuple(strides), np.dtype(ai["typestr"]) == np.uint8, int(ai["data"][0])


def frame_table(frames, w, h):
    """How push_frames passes `frames` to rb_pipeline_push_frames(_dev), without copying anything: (format, on_device,
    [(data pointer, step)] per frame).  `frames` is a sequence of per-frame arrays or one array of frames, with any frame
    stride; a frame is uint8 (h, w, 3) RGB24 or (h, w) mono8.  NumPy arrays are host frames, objects with
    __cuda_array_interface__ (torch CUDA tensors among them) device frames.  Within a frame the channel and pixel strides
    must be 1 and 3 bytes (RGB24) or the pixel stride 1 byte (mono8), and the row stride is the step, at least one row of
    pixels.  Anything else -- another dtype, shape or stride, host and device frames or two formats in one push, an empty
    push -- raises ValueError."""
    batch = not isinstance(frames, (list, tuple))
    items = [frames] if batch else list(frames)
    if not items:
        raise ValueError("frames: no frames")
    fmt = dev = None
    table = []
    for a in items:
        on_dev, shape, strides, u8, base = _array_layout(a)
        if not u8:
            raise ValueError("frames: dtype %s, not uint8" % (a.dtype if hasattr(a, "dtype") else "?"))
        fshape, fstrides = (shape[1:], strides[1:]) if batch else (shape, strides)
        if fshape == (h, w, 3):
            f, ok = FRAME_RGB24, fstrides[1:] == (3, 1)
        elif fshape == (h, w):
            f, ok = FRAME_MONO8, fstrides[1] == 1
        else:
            raise ValueError("frames: frame shape %s, not (%d, %d, 3) (RGB24) or (%d, %d) (mono8)" % (fshape, h, w, h, w))
        if not ok:
            raise ValueError("frames: pixel / channel strides %s bytes; the frames must have 3, 1 (RGB24) or 1 (mono8)"
                             % (fstrides[1:],))
        step = int(fstrides[0])
        if step < w * (3 if f == FRAME_RGB24 else 1):
            raise ValueError("frames: row stride %d bytes is shorter than a row" % step)
        if fmt is not None and (f, on_dev) != (fmt, dev):
            raise ValueError("frames: one format, all in host or all in device memory, in one push")
        fmt, dev = f, on_dev
        if batch:
            table += [(base + i * int(strides[0]), step) for i in range(shape[0])]
        else:
            table.append((base, step))
    if not table:
        raise ValueError("frames: no frames")
    return fmt, dev, table


def _mask_layout(a, h, w, what):
    """(on_device, [(address, row stride)] per mask) of one (h, w) mask or one (n, h, w) array of masks, bool or uint8 with a
    pixel stride of 1 byte and any row stride: the bytes the library reads in place.  ValueError otherwise."""
    on_dev, shape, strides, u8, base = _array_layout(a)
    dt = str(getattr(a, "dtype", ""))
    if not (u8 or dt in ("bool", "torch.bool") or
            (hasattr(a, "__cuda_array_interface__") and a.__cuda_array_interface__["typestr"] == "|b1")):
        raise ValueError("%s: dtype %s, not bool or uint8" % (what, dt or "?"))
    if len(shape) not in (2, 3) or tuple(shape[-2:]) != (h, w):
        raise ValueError("%s: shape %s, not (%d, %d) or (n, %d, %d)" % (what, tuple(shape), h, w, h, w))
    if strides[-1] != 1 or strides[-2] < w:
        raise ValueError("%s: strides %s bytes; masks need a pixel stride of 1 and a row stride of at least %d"
                         % (what, tuple(strides), w))
    if len(shape) == 2:
        return on_dev, [(base, int(strides[0]))]
    return on_dev, [(base + i * int(strides[0]), int(strides[1])) for i in range(shape[0])]


def mask_table(masks, w, h):
    """How push_masked / enqueue pass per-frame detection masks, without copying anything: the FRAME table of a list of
    CUDA (h, w) arrays or one CUDA (n, h, w) array, bool or uint8, any row stride.  ValueError for host arrays or anything
    that cannot be read in place."""
    items = list(masks) if isinstance(masks, (list, tuple)) else [masks]
    table = []
    for a in items:
        on_dev, t = _mask_layout(a, h, w, "masks")
        if not on_dev:
            raise ValueError("masks: per-frame masks are device arrays (CUDA tensors); use set_detect_mask for a host mask")
        table += t
    if not table:
        raise ValueError("masks: no masks")
    return np.array(table, FRAME)


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


def format_pose_graph(recs):
    """Bytes of the reference's pose graph file (poses_list.ps, pose_graph::saveToFile) for these ODOM records; records with
    tracked == 0 are left out."""
    recs = np.ascontiguousarray(recs, ODOM)
    need = C.c_size_t(0)
    lib().rb_odometry_format_pose_graph(_p(recs), len(recs), None, C.c_size_t(0), C.byref(need))
    buf = C.create_string_buffer(max(need.value, 1))
    r = lib().rb_odometry_format_pose_graph(_p(recs), len(recs), buf, C.c_size_t(need.value), C.byref(need))
    if r:
        raise RbError("rb_odometry_format_pose_graph failed (%d)" % r)
    return buf.raw[:need.value]


def read_pose_graph(path):
    """The records of a pose graph file (pose_graph::loadFromFile) as ODOM records with tracked = 1."""
    with open(path, "rb") as f:
        data = f.read()
    n = int(np.frombuffer(data, np.uint32, count=1)[0])
    if len(data) != 4 + n * PS_REC.itemsize:
        raise ValueError("%s: %d bytes, not a pose graph of %d records" % (path, len(data), n))
    ps = np.frombuffer(data, PS_REC, count=n, offset=4)
    out = np.zeros(n, ODOM)
    for k in PS_REC.names:
        out[k] = ps[k]
    out["tracked"] = 1
    return out


# rb_state_info (include/rebvo_b200.h, session checkpoints); mode: STATE_VISION, STATE_IMU_DATASET or STATE_IMU_LIVE
class StateInfo(C.Structure):
    _fields_ = [("version", C.c_uint32), ("mode", C.c_int32), ("bytes", C.c_uint64), ("cam", Camera), ("Sigma0", C.c_double),
                ("KSigma", C.c_double), ("kl_capacity", C.c_int32), ("kn", C.c_int32), ("n_pushed", C.c_int64)]


STATE_VISION, STATE_IMU_DATASET, STATE_IMU_LIVE = 0, 1, 2


def state_info(blob):
    """What a session blob (Pipeline.save_state) holds: version, bytes, camera, Sigma0, KSigma, kl_capacity, mode, frames
    pushed (n_pushed) and the newest map's keyline count (kn).  Host only.  RbError for a blob whose header or checksum is
    wrong."""
    blob = bytes(blob)
    out = StateInfo()
    r = lib().rb_state_info(blob, C.c_size_t(len(blob)), C.byref(out))
    if r:
        raise RbError("rb_state_info: not a valid state blob (%d)" % r)
    d = {k: getattr(out, k) for k, _ in StateInfo._fields_ if k != "cam"}
    d.update({k: getattr(out.cam, k) for k, _ in Camera._fields_})
    return d


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
        for name, (res, args) in PROTOTYPES.items():
            getattr(L, name).restype = res
            getattr(L, name).argtypes = args
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

    def minimizer_clusters(self):
        """thread-block clusters of one Minimizer_RV launch: REBVO_B200_MIN_G (default 4) when all fit, else 1"""
        return self.L.rb_ctx_minimizer_clusters(self.h_)

    def new_map(self):
        return Map(self)

    def depth_fill_net(self, records, params=None):
        """The viewer's depth grid (depth_filler, visualizer.cpp:436-440) of uint8 [n, 15] net_keyline records on this
        context's camera: (DEPTH_CELL [gh, gw], min_dist)."""
        params = params if params is not None else depth_params()
        rec = np.ascontiguousarray(records, np.uint8).reshape(-1, 15)
        gw, gh = self.w // max(params.block_w, 1), self.h // max(params.block_h, 1)
        out = np.zeros(max(gw * gh, 1), DEPTH_CELL)
        cw, ch, md = C.c_int(0), C.c_int(0), C.c_double(0)
        self.check(self.L.rb_depth_fill_net(self.h_, _p(rec), len(rec), C.byref(params), _p(out), C.byref(cw), C.byref(ch),
                                            C.byref(md)))
        return out[:cw.value * ch.value].reshape(ch.value, cw.value), md.value

    def depth_image(self, cells, params=None, s_rho=True):
        """The dense inverse-depth image of a grid (DEPTH_CELL [gh, gw], as depth_fill_net returns it): depth_filler::getImgRho
        at every pixel of this context's frame.  (rho, s_rho or None) as float32 [h, w] arrays."""
        params = params if params is not None else depth_params()
        cells = np.ascontiguousarray(cells, DEPTH_CELL)
        if cells.ndim != 2:
            raise ValueError("cells: a [gh, gw] grid")
        rho = np.zeros((self.h, self.w), np.float32)
        srho = np.zeros((self.h, self.w), np.float32) if s_rho else None
        self.check(self.L.rb_depth_image(self.h_, _p(cells), cells.shape[1], cells.shape[0], C.byref(params), _p(rho),
                                         _p(srho) if s_rho else None))
        return rho, srho

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

    def detect_masked(self, det, mask, tresh, l_kl_num, ss=None):
        """detect() with a host detection mask, (h, w) bool or uint8 with any row stride: no keyline where it is zero
        (rb_map_detect_masked).  ss: the map whose scale space is read (default this one)."""
        mask = np.asarray(mask)
        if mask.dtype == np.bool_:
            mask = mask.view(np.uint8)
        if mask.dtype != np.uint8 or mask.shape != (self.h, self.w) or mask.strides[1] != 1:
            mask = np.ascontiguousarray(mask, np.uint8)
        t, l, kn = C.c_double(tresh), C.c_int(l_kl_num), C.c_int(0)
        self.ctx.check(self.L.rb_map_detect_masked(self.h_, (ss or self).h_, C.byref(det), _p(mask),
                                                   C.c_int64(mask.strides[0]), C.byref(t), C.byref(l), C.byref(kn)))
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

    def minimizer_rv_forward(self, old, V, W, match_thresh, iter_max, init_type, reweight, max_s_rho, match_num_thresh,
                             init_iter):
        """minimizer_rv as the per-frame pipeline runs it, then FordwardMatch of old into this map; the result also
        holds fwd_match, the distinct new keylines matched"""
        V, W = np.array(V, np.float64), np.array(W, np.float64)
        RV, RW, WX = np.zeros((3, 3)), np.zeros((3, 3)), np.zeros((6, 6))
        e1, e2, sc, n = C.c_double(0), C.c_double(0), C.c_double(0), C.c_int(0)
        self.ctx.check(self.L.rb_minimizer_rv_forward(self.h_, old.h_, _p(V), _p(W), _p(RV), _p(RW),
                                                      C.c_double(match_thresh), iter_max, init_type, C.c_double(reweight),
                                                      C.byref(e1), C.byref(e2), C.c_double(max_s_rho),
                                                      C.c_uint32(match_num_thresh), int(init_iter), _p(WX), C.byref(sc),
                                                      C.byref(n)))
        return dict(F=sc.value, V=V, W=W, RVel=RV, RW0=RW, W_X=WX, rel_err=e1.value, rel_err_score=e2.value,
                    fwd_match=n.value)

    def match_update(self, old, V, P_V, BackRot, R0, do_match, thr_mod, thr_ang, max_radius, loc_unc_match,
                     match_threshold, reg_thresh, q_abs, loc_unc, Pose, Pos, K):
        """The pipeline's map chain on this map (new) and old: FordwardMatch along old's m_id_f, directed_matching
        against old rotated by R0, the match-count gate, Regularize_1_iter, the EKF, old rotated in place, and the pose
        integration from (Pose, Pos).  Returns one MATCH_UPDATE_OUT record."""
        a = [np.ascontiguousarray(v, np.float64) for v in (V, P_V, BackRot, R0)]
        Pose = np.array(Pose, np.float64)
        Pos = np.array(Pos, np.float64)
        out = np.zeros(1, MATCH_UPDATE_OUT)
        self.ctx.check(self.L.rb_map_match_update(self.h_, old.h_, *[_p(v) for v in a], int(do_match),
                                                  C.c_double(thr_mod), C.c_double(thr_ang), C.c_double(max_radius),
                                                  C.c_double(loc_unc_match), int(match_threshold), C.c_double(reg_thresh),
                                                  C.c_double(q_abs), C.c_double(loc_unc), _p(Pose), _p(Pos),
                                                  C.c_double(K), _p(out)))
        return out[0]

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


class _CudaArray:
    """A device buffer for torch.as_tensor (__cuda_array_interface__): no copy, no ownership."""

    def __init__(self, ptr, shape, typestr, strides):
        self.__cuda_array_interface__ = dict(shape=tuple(shape), typestr=typestr, data=(int(ptr), False),
                                             strides=tuple(strides) if shape else None, version=3)


def _dev_view(ptr, shape, dtype, strides, device):
    """torch CUDA tensor over device memory the pipeline owns on CUDA device `device`; strides in bytes."""
    import torch
    dev = torch.device("cuda", device)
    if 0 in shape:
        return torch.empty(shape, dtype=dtype, device=dev)
    typestr = {torch.uint8: "|u1", torch.int32: "<i4", torch.float32: "<f4", torch.float64: "<f8"}[dtype]
    return torch.as_tensor(_CudaArray(ptr, shape, typestr, strides), device=dev)


# DEPTH_CELL fields of the grid's device views
DepthDev = collections.namedtuple("DepthDev", "rho s_rho dist fixed min_dist")


class Pipeline:
    """REBVO per-frame flow on one GPU (rb_pipeline_*)."""

    def __init__(self, params, max_batch=32, device=0):
        self.L = lib()
        self.params = params
        self.w, self.h = params.cam.w, params.cam.h
        self.max_batch = max_batch
        self.device = device
        self._out_dev = False
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
        self._consumer_fence()
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
        self._consumer_fence()
        self.check(self.L.rb_pipeline_push_mono(self.h_, ptr, _p(ts), n, _p(nav)))
        return nav

    def push_frames(self, frames, ts):
        """Strided frames, read where they are (no copy): a sequence of per-frame arrays or one array of frames with any
        frame stride, uint8 (h, w, 3) RGB24 or (h, w) mono8 frames whose row stride is the step (see frame_table).  NumPy
        arrays go through rb_pipeline_push_frames, CUDA arrays (torch tensors, __cuda_array_interface__) through
        rb_pipeline_push_frames_dev.  Device frames are ordered after the work torch enqueued so far on its current stream of
        the pipeline's device: the pipeline's stream waits for an event recorded there (no host synchronisation); frames
        written on another stream must be complete before the call.  Same records as push / push_mono of the same pixels."""
        fmt, on_dev, table = frame_table(frames, self.w, self.h)
        ts = np.ascontiguousarray(ts, np.float64)
        n = len(ts)
        if len(table) != n:
            raise ValueError("push_frames: %d frames, %d timestamps" % (len(table), n))
        if on_dev:
            self._after_torch_stream()
        fr = np.array(table, FRAME)
        nav = np.zeros(n, NAV)
        self._consumer_fence()
        fn = self.L.rb_pipeline_push_frames_dev if on_dev else self.L.rb_pipeline_push_frames
        self.check(fn(self.h_, fmt, _p(fr), _p(ts), n, _p(nav)))
        return nav

    def set_detect_mask(self, mask):
        """A fixed detection mask for every later push and enqueue (rb_pipeline_set_detect_mask): (h, w) bool or uint8, a
        NumPy array or a CUDA array, any row stride; no keyline is detected where it is zero.  None clears it.  A CUDA mask is
        copied after the work torch enqueued so far on its current stream."""
        if mask is None:
            self.check(self.L.rb_pipeline_set_detect_mask(self.h_, None, C.c_int64(0), 0))
            return
        if isinstance(mask, np.ndarray):
            if mask.dtype == np.bool_:
                mask = mask.view(np.uint8)
            if mask.ndim == 2 and mask.strides[1] != 1:
                mask = np.ascontiguousarray(mask)
        on_dev, table = _mask_layout(mask, self.h, self.w, "set_detect_mask")
        if len(table) != 1:
            raise ValueError("set_detect_mask: one (%d, %d) mask" % (self.h, self.w))
        if on_dev:
            self._after_torch_stream()
        ptr, step = table[0]
        self.check(self.L.rb_pipeline_set_detect_mask(self.h_, C.c_void_p(ptr), C.c_int64(step), int(on_dev)))

    def push_masked(self, frames, masks, ts):
        """push_frames with per-frame detection masks (rb_pipeline_push_masked): masks is a list of CUDA (h, w) arrays or one
        CUDA (n, h, w) array, bool or uint8, any row stride, read in place (see mask_table); no keyline is detected where a
        frame's mask is zero.  Frames as push_frames takes them, host or device.  Frames and masks are ordered after the work
        torch enqueued so far on its current stream.  A fixed mask (set_detect_mask) applies as well."""
        fmt, on_dev, table = frame_table(frames, self.w, self.h)
        mt = mask_table(masks, self.w, self.h)
        ts = np.ascontiguousarray(ts, np.float64)
        n = len(ts)
        if len(table) != n or len(mt) != n:
            raise ValueError("push_masked: %d frames, %d masks, %d timestamps" % (len(table), len(mt), n))
        self._after_torch_stream()
        fr = np.array(table, FRAME)
        nav = np.zeros(n, NAV)
        self._consumer_fence()
        self.check(self.L.rb_pipeline_push_masked(self.h_, fmt, int(on_dev), _p(fr), _p(mt), _p(ts), n, _p(nav)))
        return nav

    def _after_torch_stream(self):
        """The pipeline's stream waits for the work torch enqueued so far on its current stream of this device: an event
        recorded there (one event, reused: a wait takes the record made just before it)."""
        import torch
        if getattr(self, "_order", None) is None:
            dev = torch.device("cuda", self.device)
            self._order = (dev, torch.cuda.ExternalStream(self.stream(), device=dev), torch.cuda.Event())
        dev, ext, ev = self._order
        ev.record(torch.cuda.current_stream(dev))
        ext.wait_event(ev)

    def push_mono_dev(self, dev_ptr, ts):
        """Mono frames already in device memory (4-byte aligned pointer), read in place."""
        ts = np.ascontiguousarray(ts, np.float64)
        nav = np.zeros(len(ts), NAV)
        self._consumer_fence()
        self.check(self.L.rb_pipeline_push_mono_dev(self.h_, C.c_void_p(int(dev_ptr)), _p(ts), len(ts), _p(nav)))
        return nav

    def set_imu(self, samples, imu_params=None):
        """IMU mode (BASELINE configs[2]): samples = float64 [n, 7] rows {t, gyro xyz, accel xyz}."""
        samples = np.ascontiguousarray(samples, np.float64)
        ip = imu_params if imu_params is not None else default_imu_params()
        self.check(self.L.rb_pipeline_set_imu(self.h_, C.byref(ip), _p(samples), len(samples)))

    def set_imu_live(self, imu_params=None, sample_time=0.005, buffer_size=1000):
        """Live IMU mode (ImuMode=1): an empty ring of `buffer_size` samples (CircBufferSize) integrated with the step
        `sample_time` (SampleTime), fed by push_imu.  The defaults are those of the reference's EuRoC ROS configuration."""
        ip = imu_params if imu_params is not None else default_imu_params()
        self.check(self.L.rb_pipeline_set_imu_live(self.h_, C.byref(ip), C.c_double(sample_time), int(buffer_size)))

    def push_imu(self, samples):
        """Append float64 [n, 7] rows {t, gyro xyz, accel xyz} in time order, all or none.  RbError when the ring cannot hold
        them (push frames first), outside live IMU mode, or when a timestamp goes backwards.  A frame push that the samples do
        not cover raises RbError and changes nothing: push the missing samples and repeat it."""
        samples = np.ascontiguousarray(samples, np.float64).reshape(-1, 7)
        self.check(self.L.rb_pipeline_push_imu(self.h_, _p(samples), len(samples)))

    def push_dev(self, dev_ptr, ts):
        ts = np.ascontiguousarray(ts, np.float64)
        nav = np.zeros(len(ts), NAV)
        self._consumer_fence()
        self.check(self.L.rb_pipeline_push_dev(self.h_, C.c_void_p(int(dev_ptr)), _p(ts), len(ts), _p(nav)))
        return nav

    def set_async(self, depth):
        """Asynchronous pushes (enqueue, wait, poll): up to `depth` (1..8) tickets in flight, 0 = off (the default).  Between
        pushes, with no ticket outstanding; allocates the output ring and a second scale-space workspace."""
        self.check(self.L.rb_pipeline_set_async(self.h_, int(depth)))

    def _enqueue_args(self, frames, ts, fmt):
        """(C function, argument tuple, objects to keep alive) of an enqueue; ValueError for anything the library would
        refuse for its format or shape."""
        if fmt not in ("rgb", "mono"):
            raise ValueError("enqueue: fmt 'rgb' or 'mono', not %r" % (fmt,))
        n = len(ts)
        if not 1 <= n <= self.max_batch:
            raise ValueError("enqueue: %d timestamps, the pipeline takes 1..%d frames" % (n, self.max_batch))
        want = FRAME_MONO8 if fmt == "mono" else FRAME_RGB24
        if isinstance(frames, (list, tuple)):
            f, on_dev, table = frame_table(frames, self.w, self.h)
            if f != want:
                raise ValueError("enqueue: %s frames with fmt=%r" % ("mono8" if f == FRAME_MONO8 else "RGB24", fmt))
            if len(table) != n:
                raise ValueError("enqueue: %d frames, %d timestamps" % (len(table), n))
            fr = np.array(table, FRAME)
            return self.L.rb_pipeline_enqueue_frames, (want, int(on_dev), _p(fr)), (frames, fr), on_dev
        shape = (n, self.h, self.w) + (() if fmt == "mono" else (3,))
        on_dev, got, strides, u8, base = _array_layout(frames)
        if not u8 or tuple(got) != shape:
            raise ValueError("enqueue: packed %s frames are uint8 %s, not %s %s"
                             % (fmt, shape, getattr(frames, "dtype", "?"), tuple(got)))
        packed = tuple(int(np.prod(shape[k + 1:], dtype=np.int64)) for k in range(len(shape)))
        if tuple(strides) != packed:
            if on_dev:
                raise ValueError("enqueue: device frames must be packed (contiguous); pass a list of frames for strided ones")
            frames = np.ascontiguousarray(frames)
            base = frames.__array_interface__["data"][0]
        return self.L.rb_pipeline_enqueue, (want, int(on_dev), C.c_void_p(base)), (frames,), on_dev

    def enqueue(self, frames, ts, fmt="rgb", masks=None):
        """Hand over n frames without waiting for them (rb_pipeline_enqueue / enqueue_frames); returns the ticket to wait.
        frames: a uint8 host array or torch CUDA tensor of packed frames, (n, h, w, 3) for fmt="rgb" or (n, h, w) for
        fmt="mono", or a list of strided frames as push_frames takes them.  The frames are kept alive until the ticket is
        waited.  Device frames: the call first waits (on the host) for the work torch enqueued so far on its current stream,
        so that they are complete.  Device output mode: the enqueue's writes wait for torch's current stream, as a push's.
        masks: per-frame detection masks as push_masked takes them (rb_pipeline_masked_enqueue), kept alive with the frames
        and read after the work torch enqueued so far on its current stream.  RbError when `depth` tickets are outstanding
        (nothing changes) or asynchronous pushes are off."""
        fn, args, keep, on_dev = self._enqueue_args(frames, ts, fmt)
        if masks is not None:
            f, on_dev, table = frame_table(frames, self.w, self.h)
            mt = mask_table(masks, self.w, self.h)
            if len(mt) != len(ts):
                raise ValueError("enqueue: %d masks, %d timestamps" % (len(mt), len(ts)))
            fr = np.array(table, FRAME)
            fn, args, keep = self.L.rb_pipeline_masked_enqueue, (f, int(on_dev), _p(fr), _p(mt)), (frames, fr, masks, mt)
            self._after_torch_stream()
        ts = np.ascontiguousarray(ts, np.float64)
        if on_dev or self._out_dev:
            import torch
            cur = torch.cuda.current_stream(self.device)
            if on_dev:
                cur.synchronize()
            if self._out_dev and getattr(self, "_consumer", None) != cur.cuda_stream:
                self.set_consumer_stream(cur.cuda_stream)
        ticket = C.c_int64(-1)
        self.check(fn(self.h_, *args, _p(ts), len(ts), C.byref(ticket)))
        if not hasattr(self, "_inflight"):
            self._inflight = {}
        self._inflight[ticket.value] = (len(ts), keep)
        return ticket.value

    def wait(self, ticket):
        """Block until `ticket` is complete and retire it with every earlier one; returns its NAV records.  Until the next
        wait or push, odometry(), mirror(), depth(), depth_image() and their _dev forms give the ticket's outputs."""
        inflight = getattr(self, "_inflight", {})
        n = inflight.get(int(ticket), (0, None))[0]
        nav = np.zeros(n, NAV)
        r = self.L.rb_pipeline_wait(self.h_, C.c_int64(int(ticket)), _p(nav) if n else None)
        if n:
            for t in [t for t in inflight if t <= int(ticket)]:
                del inflight[t]
        self.check(r)
        return nav

    def poll(self):
        """The newest ticket whose work is complete (-1 if none), without blocking."""
        t = C.c_int64(-1)
        self.check(self.L.rb_pipeline_poll(self.h_, C.byref(t)))
        return t.value

    def reset(self):
        self.check(self.L.rb_pipeline_reset(self.h_))

    def save_state(self):
        """The tracking session as a blob (bytes): load it into a pipeline of the same geometry, here or in another process
        or on another GPU, and the pushes continue the session exactly (rb_pipeline_save_state)."""
        need = C.c_size_t(0)
        r = self.L.rb_pipeline_save_state(self.h_, None, C.c_size_t(0), C.byref(need))
        if r and need.value == 0:
            self.check(r)
        buf = C.create_string_buffer(need.value)
        self.check(self.L.rb_pipeline_save_state(self.h_, buf, C.c_size_t(need.value), C.byref(need)))
        return buf.raw[:need.value]

    def load_state(self, blob):
        """Replace this pipeline's session with the blob's (rb_pipeline_load_state).  RbError, with the pipeline unchanged,
        for a corrupt blob or one of another version, geometry or mode."""
        blob = bytes(blob)
        self.check(self.L.rb_pipeline_load_state(self.h_, blob, C.c_size_t(len(blob))))

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

    def batch_plane(self, slot, which):
        """Plane `which` ("gray", "img0" or "dog") of slot `slot` of the last scale-space batch, (h, w) float32.  After a host
        push cut into a head and the rest (REBVO_B200_SUB) the slots hold the rest."""
        idx = {"img0": 0, "dog": 2, "gray": 5}[which]
        out = np.empty((self.h, self.w), np.float32)
        self.check(self.L.rb_pipeline_batch_plane(self.h_, int(slot), idx, _p(out)))
        return out

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

    def set_odometry(self, on=True):
        """Per-frame odometry records (the reference's pose graph measurements) with every push: on / off between pushes."""
        self.check(self.L.rb_pipeline_set_odometry(self.h_, int(bool(on))))

    def odometry(self):
        """ODOM[n]: record i for frame i of the last push (a copy)."""
        p, n = C.c_void_p(0), C.c_int(0)
        self.check(self.L.rb_pipeline_odometry(self.h_, C.byref(p), C.byref(n)))
        buf = (C.c_char * (n.value * ODOM.itemsize)).from_address(p.value)
        return np.frombuffer(buf, dtype=ODOM, count=n.value).copy()

    def set_depth(self, params):
        """Per-frame depth grid (the viewer's depth_filler on every frame's net_keyline records) with every push:
        DepthParams to switch it on, None to switch it off."""
        self.check(self.L.rb_pipeline_set_depth(self.h_, C.byref(params) if params is not None else None))

    def depth(self, i):
        """(DEPTH_CELL [gh, gw], min_dist) of frame i of the last push (a copy)."""
        p, gw, gh, md = C.c_void_p(0), C.c_int(0), C.c_int(0), C.c_double(0)
        self.check(self.L.rb_pipeline_depth(self.h_, i, C.byref(p), C.byref(gw), C.byref(gh), C.byref(md)))
        n = gw.value * gh.value
        buf = (C.c_char * (n * DEPTH_CELL.itemsize)).from_address(p.value)
        return np.frombuffer(buf, dtype=DEPTH_CELL, count=n).reshape(gh.value, gw.value).copy(), md.value

    def set_depth_image(self, mode):
        """Per-frame dense inverse-depth image of the depth grid (depth_filler::getImgRho at every pixel) with every push
        while the grid is on: 1 = the rho plane, 2 = the rho and s_rho planes, 0 = off."""
        self.check(self.L.rb_pipeline_set_depth_image(self.h_, int(mode)))

    def depth_image(self, i):
        """Views (no copy) of the image of frame i of the last push: (rho, s_rho or None) as float32 [h, w]; valid until the
        next push."""
        r, s = C.c_void_p(0), C.c_void_p(0)
        self.check(self.L.rb_pipeline_depth_image(self.h_, i, C.byref(r), C.byref(s)))
        n = self.w * self.h

        def view(p):
            return np.frombuffer((C.c_char * (4 * n)).from_address(p), dtype=np.float32).reshape(self.h, self.w)
        return view(r.value), (view(s.value) if s.value else None)

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

    def set_output_memory(self, where):
        """Where the mirror, the depth grid and the depth image go: "host" (the default; mirror(), depth(), depth_image()) or
        "device" (mirror_dev(), depth_dev(), depth_image_dev(), depth_images_dev(): torch CUDA tensors, no copy).  Between
        pushes; the outputs of the last push are dropped when it changes."""
        if where not in ("host", "device"):
            raise ValueError("where: 'host' or 'device'")
        self.check(self.L.rb_pipeline_set_output_memory(self.h_, int(where == "device")))
        self._out_dev = where == "device"

    def set_consumer_stream(self, stream):
        """Device mode: each push first waits for the work enqueued on `stream` (a cudaStream_t handle, as an int; 0 is the
        legacy default stream) when it is called.  The push wrappers set torch.cuda.current_stream() before each push in
        device mode; this call is for pushes made through the C functions.  self.stream() waits for nothing."""
        self.check(self.L.rb_pipeline_set_consumer_stream(self.h_, C.c_void_p(int(stream))))
        self._consumer = int(stream)

    def _consumer_fence(self):
        """Device mode: the push overwrites no output before the work torch enqueued so far on its current stream (which
        may still read the last push's outputs) is done."""
        if self._out_dev:
            import torch
            self.set_consumer_stream(torch.cuda.current_stream(self.device).cuda_stream)

    def mirror_dev(self, i):
        """Device mode: the records of frame i of the last push as a uint8 CUDA tensor [kn, rec] (rec = 168 in mode 1,
        15 in mode 2), no copy; valid until the next push."""
        import torch
        p, kn = C.c_void_p(0), C.c_int(0)
        self.check(self.L.rb_pipeline_mirror_dev(self.h_, i, C.byref(p), C.byref(kn)))
        rec = 15 if getattr(self, "_mirror_mode", 1) == 2 else KEYLINE.itemsize
        return _dev_view(p.value, (kn.value, rec), torch.uint8, (rec, 1), self.device)

    def depth_dev(self, i):
        """Device mode: the grid of frame i of the last push as CUDA tensors over its DEPTH_CELL records, no copy:
        DepthDev(rho, s_rho, dist: float64 [gh, gw]; fixed: int32 [gh, gw]; min_dist: float64 0-d); valid until the next
        push."""
        import torch
        p, gw, gh, md = C.c_void_p(0), C.c_int(0), C.c_int(0), C.c_void_p(0)
        self.check(self.L.rb_pipeline_depth_dev(self.h_, i, C.byref(p), C.byref(gw), C.byref(gh), C.byref(md)))
        shape, strides = (gh.value, gw.value), (gw.value * DEPTH_CELL.itemsize, DEPTH_CELL.itemsize)
        f = {n: (p.value + DEPTH_CELL.fields[n][1]) for n in ("rho", "s_rho", "dist", "fixed")}
        return DepthDev(*(_dev_view(f[n], shape, torch.float64, strides, self.device) for n in ("rho", "s_rho", "dist")),
                        _dev_view(f["fixed"], shape, torch.int32, strides, self.device),
                        _dev_view(md.value, (), torch.float64, (), self.device))

    def depth_image_dev(self, i):
        """Device mode: the image of frame i of the last push as float32 CUDA tensors (rho, s_rho or None) [h, w], no copy;
        valid until the next push."""
        import torch
        r, s = C.c_void_p(0), C.c_void_p(0)
        self.check(self.L.rb_pipeline_depth_image_dev(self.h_, i, C.byref(r), C.byref(s)))

        def view(ptr):
            return _dev_view(ptr, (self.h, self.w), torch.float32, (4 * self.w, 4), self.device)
        return view(r.value), (view(s.value) if s.value else None)

    def depth_images_dev(self):
        """Device mode: the images of every frame of the last push as float32 CUDA tensors (rho, s_rho or None) [n, h, w],
        frame after frame a padded plane stride apart (no copy); valid until the next push."""
        import torch
        r, s = C.c_void_p(0), C.c_void_p(0)
        self.check(self.L.rb_pipeline_depth_image_dev(self.h_, 0, C.byref(r), C.byref(s)))
        n = 1
        while n < self.max_batch and self.L.rb_pipeline_depth_image_dev(self.h_, n, C.byref(C.c_void_p()), None) == 0:
            n += 1
        plane = (self.w * self.h + 63) // 64 * 64
        step = 4 * plane * (2 if s.value else 1)
        strides = (step, 4 * self.w, 4)

        def view(ptr):
            return _dev_view(ptr, (n, self.h, self.w), torch.float32, strides, self.device)
        return view(r.value), (view(s.value) if s.value else None)

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
