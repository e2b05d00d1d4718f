"""ctypes binding of libefusion.so (include/efusion_b200.h).

This is the thinnest possible host layer: it loads the in-tree shared library that holds the sm_90a kernels and
calls its C ABI. There is no CPU fallback: if the library is missing or the call fails, an exception is raised.
"""
from __future__ import annotations

import ctypes as C
import os

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libefusion.so")
_LIB = None


class EfError(RuntimeError):
    pass


class EfConfig(C.Structure):
    _fields_ = [("width", C.c_int32), ("height", C.c_int32), ("fx", C.c_float), ("fy", C.c_float), ("cx", C.c_float),
                ("cy", C.c_float), ("time_delta", C.c_int32), ("count_thresh", C.c_int32), ("err_thresh", C.c_float),
                ("cov_thresh", C.c_float), ("close_loops", C.c_int32), ("iclnuim", C.c_int32), ("reloc", C.c_int32),
                ("photo_thresh", C.c_float), ("confidence", C.c_float), ("depth_cutoff", C.c_float),
                ("icp_weight", C.c_float), ("fast_odom", C.c_int32), ("fern_thresh", C.c_float), ("so3", C.c_int32),
                ("frame_to_frame_rgb", C.c_int32), ("capacity", C.c_int32), ("device", C.c_int32),
                ("skip_mid_predict", C.c_int32)]


class EfLoopResult(C.Structure):
    _fields_ = [("ran", C.c_int32), ("accepted", C.c_int32), ("n_constraints", C.c_int32), ("lastICPError", C.c_float),
                ("lastICPCount", C.c_float), ("cov_diag", C.c_double * 6), ("T_wc_est", C.c_double * 16)]


class EfDeformResult(C.Structure):
    _fields_ = [("n_nodes", C.c_int32), ("n_enabled", C.c_int32), ("n_constraints", C.c_int32), ("iterations", C.c_int32),
                ("stop", C.c_int32), ("bandwidth", C.c_int32), ("error", C.c_float), ("meanConsErr", C.c_float)]


class EfLocalDeform(C.Structure):
    _fields_ = [("solved", C.c_int32), ("applied", C.c_int32), ("result", EfDeformResult), ("deforms", C.c_int32),
                ("last_deform_time", C.c_int32), ("n_nodes", C.c_int32)]


class EfRenderView(C.Structure):
    _fields_ = [("width", C.c_int32), ("height", C.c_int32), ("mvp", C.c_float * 16), ("mv", C.c_float * 16), ("threshold", C.c_float),
                ("color_type", C.c_int32), ("unstable", C.c_int32), ("draw_window", C.c_int32), ("time", C.c_int32),
                ("time_delta", C.c_int32), ("phong", C.c_int32), ("sign_mult", C.c_float)]


def camera_view(T_wc, fx, fy, cx, cy, w, h, near=0.1, far=1000.0, **flags) -> EfRenderView:
    """EfRenderView of a pinhole camera at pose T_wc (4x4 camera-to-world) through ef_render_camera: window pixel (i, j) samples the
    ray through image pixel centre (i + 0.5, j + 0.5), so a render from the tracked pose with the frame's intrinsics lines up with the
    input image, top row first. flags: threshold, color_type, unstable, draw_window, time, time_delta, phong, sign_mult (defaults:
    the confidence threshold 10, colour type 2, sign_mult -1, the rest 0)."""
    v = EfRenderView()
    v.width, v.height = int(w), int(h)
    v.threshold, v.color_type, v.sign_mult = 10.0, 2, -1.0
    _chk(lib().ef_render_camera(_p(_T(T_wc)), _f(fx), _f(fy), _f(cx), _f(cy), int(w), int(h), _f(near), _f(far), v.mvp, v.mv))
    for k, val in flags.items():
        if k in ("width", "height", "mvp", "mv") or not hasattr(v, k):
            raise KeyError(k)
        setattr(v, k, val)
    return v


class EfModelView(C.Structure):
    _fields_ = [("T_wc", C.c_double * 16), ("fx", C.c_float), ("fy", C.c_float), ("cx", C.c_float), ("cy", C.c_float), ("width", C.c_int32),
                ("height", C.c_int32), ("max_depth", C.c_float), ("conf_threshold", C.c_float), ("time", C.c_int32), ("max_time", C.c_int32),
                ("time_delta", C.c_int32)]


def model_view(T_wc, fx, fy, cx, cy, w, h, max_depth, conf_threshold, time, max_time, time_delta) -> EfModelView:
    """EfModelView of combinedPredict at pose T_wc (4x4 camera-to-world) through a w x h pinhole camera. The time window is
    combinedPredict's: ACTIVE = (tick, tick, time_delta), INACTIVE = (0, tick - time_delta, time_delta)."""
    v = EfModelView()
    v.T_wc[:] = [float(x) for x in np.asarray(T_wc, np.float64).reshape(16)]
    v.fx, v.fy, v.cx, v.cy = float(fx), float(fy), float(cx), float(cy)
    v.width, v.height = int(w), int(h)
    v.max_depth, v.conf_threshold = float(max_depth), float(conf_threshold)
    v.time, v.max_time, v.time_delta = int(time), int(max_time), int(time_delta)
    return v


class EfFuseView(C.Structure):
    _fields_ = [("T_wc", C.c_double * 16), ("fx", C.c_float), ("fy", C.c_float), ("cx", C.c_float), ("cy", C.c_float), ("width", C.c_int32),
                ("height", C.c_int32), ("depth_cutoff", C.c_float), ("max_depth", C.c_float), ("weighting", C.c_float),
                ("conf_threshold", C.c_float), ("time", C.c_int32), ("time_delta", C.c_int32)]


def fuse_view(T_wc, fx, fy, cx, cy, w, h, time, weighting=1.0, depth_cutoff=3.0, max_depth=20.0, conf_threshold=10.0,
              time_delta=200) -> EfFuseView:
    """EfFuseView of an RGB-D frame taken at pose T_wc (4x4 camera-to-world) through a w x h pinhole camera, fused at tick `time`.
    For the second camera of a rig, `time` is the tick of the tracked frame it accompanies (get_tick() - 1 after that frame)."""
    v = EfFuseView()
    v.T_wc[:] = [float(x) for x in np.asarray(T_wc, np.float64).reshape(16)]
    v.fx, v.fy, v.cx, v.cy = float(fx), float(fy), float(cx), float(cy)
    v.width, v.height = int(w), int(h)
    v.depth_cutoff, v.max_depth, v.weighting, v.conf_threshold = float(depth_cutoff), float(max_depth), float(weighting), float(conf_threshold)
    v.time, v.time_delta = int(time), int(time_delta)
    return v


class EfOdomStats(C.Structure):
    _fields_ = [("lastICPError", C.c_float), ("lastICPCount", C.c_float), ("lastRGBError", C.c_float), ("lastRGBCount", C.c_float),
                ("lastSO3Error", C.c_float), ("lastSO3Count", C.c_float), ("lastA", C.c_double * 36), ("lastb", C.c_double * 6)]


class EfTrackView(C.Structure):
    _fields_ = [("model", EfModelView), ("depth_cutoff", C.c_float), ("icp_weight", C.c_float), ("rgb_only", C.c_int32),
                ("pyramid", C.c_int32), ("fast_odom", C.c_int32)]


class EfTrackResult(C.Structure):
    _fields_ = [("T_wc", C.c_double * 16), ("stats", EfOdomStats), ("covariance", C.c_double * 36), ("dense_enough", C.c_int32)]


def track_view(T_wc, fx, fy, cx, cy, w, h, time, max_time=None, time_delta=200, depth_cutoff=3.0, max_depth=20.0, conf_threshold=10.0,
               icp_weight=10.0, rgb_only=False, pyramid=True, fast_odom=False) -> EfTrackView:
    """EfTrackView of an RGB-D frame of a w x h pinhole camera, tracked against the map from the guess T_wc (4x4 camera-to-world).
    The model is combinedPredict's window (time, max_time, time_delta); max_time None is `time`, the ACTIVE window the frame tracks
    against at tick `time`. The defaults are the frame's: depth_cutoff 3 m, max_depth 20 m, confidence 10, icp_weight 10."""
    v = EfTrackView()
    v.model = model_view(T_wc, fx, fy, cx, cy, w, h, max_depth, conf_threshold, time, time if max_time is None else max_time, time_delta)
    v.depth_cutoff, v.icp_weight = float(depth_cutoff), float(icp_weight)
    v.rgb_only, v.pyramid, v.fast_odom = int(bool(rgb_only)), int(bool(pyramid)), int(bool(fast_odom))
    return v


def unpack_track_result(res):
    """(T_wc (4, 4), stats (a STATS_DTYPE record, as Context.odom_stats), covariance (6, 6), dense_enough) of an EfTrackResult, or of
    its bytes as ef_track_view_device wrote them."""
    if not isinstance(res, EfTrackResult):
        res = EfTrackResult.from_buffer_copy(bytes(res))
    stats = np.frombuffer(bytes(res.stats), STATS_DTYPE)[0].copy()
    return (np.array(res.T_wc[:]).reshape(4, 4), stats, np.array(res.covariance[:]).reshape(6, 6), bool(res.dense_enough))


class EfCameraConfig(C.Structure):
    _fields_ = [("width", C.c_int32), ("height", C.c_int32), ("fx", C.c_float), ("fy", C.c_float), ("cx", C.c_float), ("cy", C.c_float),
                ("depth_cutoff", C.c_float), ("max_depth", C.c_float), ("conf_threshold", C.c_float), ("time_delta", C.c_int32),
                ("icp_weight", C.c_float), ("rgb_only", C.c_int32), ("pyramid", C.c_int32), ("fast_odom", C.c_int32), ("so3", C.c_int32),
                ("frame_to_frame_rgb", C.c_int32), ("close_loops", C.c_int32)]


class EfCameraFrame(C.Structure):
    _fields_ = [("time", C.c_int32), ("weight_multiplier", C.c_float), ("has_pose", C.c_int32), ("T_wc", C.c_double * 16),
                ("fuse", C.c_int32)]


class EfCameraResult(C.Structure):
    _fields_ = [("T_wc", C.c_double * 16), ("stats", EfOdomStats), ("covariance", C.c_double * 36), ("tracked", C.c_int32),
                ("dense_enough", C.c_int32), ("weighting", C.c_float)]


MAX_CAMERAS = 4  # EF_MAX_CAMERAS


def camera_config(w, h, fx, fy, cx, cy, depth_cutoff=3.0, max_depth=20.0, conf_threshold=10.0, time_delta=200, icp_weight=10.0,
                  rgb_only=False, pyramid=True, fast_odom=False, so3=True, frame_to_frame_rgb=False, close_loops=False) -> EfCameraConfig:
    """EfCameraConfig of a w x h pinhole camera. The defaults are the frame's (ef_default_config and the ElasticFusion constructor):
    depth_cutoff 3 m, maxDepthProcessed 20 m, confidence 10, time_delta 200, icp_weight 10, pyramid and SO(3) on. close_loops: its
    frames close local loops on the context's graph (a context with close_loops = 2)."""
    c = EfCameraConfig()
    c.width, c.height = int(w), int(h)
    c.fx, c.fy, c.cx, c.cy = float(fx), float(fy), float(cx), float(cy)
    c.depth_cutoff, c.max_depth, c.conf_threshold = float(depth_cutoff), float(max_depth), float(conf_threshold)
    c.time_delta, c.icp_weight = int(time_delta), float(icp_weight)
    c.rgb_only, c.pyramid, c.fast_odom = int(bool(rgb_only)), int(bool(pyramid)), int(bool(fast_odom))
    c.so3, c.frame_to_frame_rgb = int(bool(so3)), int(bool(frame_to_frame_rgb))
    c.close_loops = int(bool(close_loops))
    return c


def camera_frame(time, weight_multiplier=1.0, T_wc=None, fuse=True) -> EfCameraFrame:
    """EfCameraFrame: the frame is stamped and predicted at `time`; T_wc (4x4 camera-to-world) sets the pose instead of tracking."""
    f = EfCameraFrame()
    f.time, f.weight_multiplier, f.fuse = int(time), float(weight_multiplier), int(bool(fuse))
    if T_wc is not None:
        f.has_pose = 1
        f.T_wc[:] = np.asarray(T_wc, np.float64).reshape(16).tolist()
    return f


class EfRigConfig(C.Structure):
    _fields_ = [("n", C.c_int32), ("cameras", C.c_void_p * MAX_CAMERAS), ("T_0i", (C.c_double * 16) * MAX_CAMERAS), ("joint_so3", C.c_int32)]


class EfRigFrame(C.Structure):
    _fields_ = [("time", C.c_int32), ("weight_multiplier", C.c_float), ("has_pose", C.c_int32), ("T_wc", C.c_double * 16),
                ("fuse", C.c_int32)]


class EfRigResult(C.Structure):
    _fields_ = [("T_wc", C.c_double * 16), ("lastA", C.c_double * 36), ("lastb", C.c_double * 6), ("covariance", C.c_double * 36),
                ("tracked", C.c_int32)]


class EfRigLoopResult(C.Structure):
    _fields_ = [("ran", C.c_int32), ("accepted", C.c_int32), ("n_constraints", C.c_int32), ("member_constraints", C.c_int32 * MAX_CAMERAS),
                ("lastICPError", C.c_float), ("lastICPCount", C.c_float), ("cov_diag", C.c_double * 6), ("T_wc_curr", C.c_double * 16),
                ("T_wc_est", C.c_double * 16)]


def rig_frame(time, weight_multiplier=1.0, T_wc=None, fuse=True) -> EfRigFrame:
    """EfRigFrame: the rig's frame is stamped and predicted at `time`; T_wc (4x4 camera-to-world of member 0) sets the pose."""
    f = EfRigFrame()
    f.time, f.weight_multiplier, f.fuse = int(time), float(weight_multiplier), int(bool(fuse))
    if T_wc is not None:
        f.has_pose = 1
        f.T_wc[:] = np.asarray(T_wc, np.float64).reshape(16).tolist()
    return f


def unpack_rig_result(res):
    """(T_wc (4, 4), lastA (6, 6), lastb (6,), covariance (6, 6), tracked) of an EfRigResult or its bytes."""
    if not isinstance(res, EfRigResult):
        res = EfRigResult.from_buffer_copy(bytes(res))
    return (np.array(res.T_wc[:]).reshape(4, 4), np.array(res.lastA[:]).reshape(6, 6), np.array(res.lastb[:]),
            np.array(res.covariance[:]).reshape(6, 6), bool(res.tracked))


def _local_deform(call):
    """(info dict, graph (n, 4) float32) of ef_local_deform_result or ef_camera_deform_result, called as call(out, nodes, n_out)"""
    res = EfLocalDeform()
    nodes = np.zeros((1023, 4), np.float32)
    n = C.c_int32()
    _chk(call(C.byref(res), nodes, C.byref(n)))
    info = dict(solved=bool(res.solved), applied=bool(res.applied), result={k: getattr(res.result, k) for k, _ in EfDeformResult._fields_},
                deforms=res.deforms, last_deform_time=res.last_deform_time, n_nodes=res.n_nodes)
    return info, nodes[:n.value].copy()


def unpack_camera_result(res):
    """(T_wc (4, 4), stats (STATS_DTYPE), covariance (6, 6), {tracked, dense_enough, weighting}) of an EfCameraResult or its bytes."""
    if not isinstance(res, EfCameraResult):
        res = EfCameraResult.from_buffer_copy(bytes(res))
    stats = np.frombuffer(bytes(res.stats), STATS_DTYPE)[0].copy()
    info = dict(tracked=bool(res.tracked), dense_enough=bool(res.dense_enough), weighting=float(res.weighting))
    return np.array(res.T_wc[:]).reshape(4, 4), stats, np.array(res.covariance[:]).reshape(6, 6), info


# outputs of a model view: dtype and channels per pixel
VIEW_OUTPUTS = {"image": (np.uint8, 4), "vertex": (np.float32, 4), "normal": (np.float32, 4), "time": (np.uint16, 1)}

TRACE_DTYPE = np.dtype([
    ("kind", "<i4"), ("level", "<i4"), ("iter", "<i4"), ("rgb_count", "<i4"), ("rgb_sigma", "<i4"),
    ("sigma_val", "<f4"),
    ("A_icp", "<f4", (36,)), ("b_icp", "<f4", (6,)), ("icp_residual", "<f4", (2,)),
    ("A_rgb", "<f4", (36,)), ("b_rgb", "<f4", (6,)),
    ("A_so3", "<f4", (9,)), ("b_so3", "<f4", (3,)), ("so3_residual", "<f4", (2,)),
    ("lastA", "<f8", (36,)), ("lastb", "<f8", (6,)), ("result", "<f8", (6,)),
], align=True)

STATS_DTYPE = np.dtype([("lastICPError", "<f4"), ("lastICPCount", "<f4"), ("lastRGBError", "<f4"),
                        ("lastRGBCount", "<f4"), ("lastSO3Error", "<f4"), ("lastSO3Count", "<f4"),
                        ("lastA", "<f8", (36,)), ("lastb", "<f8", (6,))], align=True)

DATATERM_DTYPE = np.dtype([("zero_x", "<i2"), ("zero_y", "<i2"), ("one_x", "<i2"), ("one_y", "<i2"),
                           ("diff", "<f4"), ("valid", "<i4")])

# buffer ids (include/efusion_b200.h)
BUF = dict(RGB=0, DEPTH_RAW=1, DEPTH_FILTERED=2, DEPTH_METRIC=3, DEPTH_METRIC_FILTERED=4, RGBA=5, INDEX=10, VERT_CONF=11,
           COLOR_TIME=12, NORM_RAD=13, IMAGE=14, VERTEX=15, NORMAL=16, TIME=17, OLD_IMAGE=18, OLD_VERTEX=19,
           OLD_NORMAL=20, OLD_TIME=21, SYNTH_DEPTH=22, FILL_IMAGE=30, FILL_VERTEX=31, FILL_NORMAL=32, VMAP_CURR=40,
           NMAP_CURR=41, VMAP_G_PREV=42, NMAP_G_PREV=43, LAST_DEPTH=44, NEXT_DEPTH=45, LAST_IMAGE=46, NEXT_IMAGE=47,
           LAST_NEXT_IMAGE=48, DIDX=49, DIDY=50, DEPTH_TMP=51, CORRES=52, VMAPS_TMP=53)

_BUF_FMT = {  # id -> (dtype, channels/planes kind)
    0: (np.uint8, "c3"), 1: (np.uint16, "c1"), 2: (np.uint16, "c1"), 3: (np.float32, "c1"), 4: (np.float32, "c1"),
    5: (np.uint8, "c4"), 10: (np.uint32, "c1"), 11: (np.float32, "c4"), 12: (np.float32, "c4"), 13: (np.float32, "c4"),
    14: (np.uint8, "c4"), 15: (np.float32, "c4"), 16: (np.float32, "c4"), 17: (np.uint16, "c1"), 18: (np.uint8, "c4"),
    19: (np.float32, "c4"), 20: (np.float32, "c4"), 21: (np.uint16, "c1"), 22: (np.float32, "c1"),
    30: (np.uint8, "c4"), 31: (np.float32, "c4"), 32: (np.float32, "c4"),
    40: (np.float32, "p3"), 41: (np.float32, "p3"), 42: (np.float32, "p3"), 43: (np.float32, "p3"),
    44: (np.float32, "c1"), 45: (np.float32, "c1"), 46: (np.uint8, "c1"), 47: (np.uint8, "c1"), 48: (np.uint8, "c1"),
    49: (np.int16, "c1"), 50: (np.int16, "c1"), 51: (np.uint16, "c1"), 52: (DATATERM_DTYPE, "c1"),
    53: (np.float32, "c4"),
}


def lib():
    """Loads libefusion.so; raises if the CUDA extension has not been built (no fallback path exists)."""
    global _LIB
    if _LIB is None:
        path = os.environ.get("EF_LIB", LIB_PATH)  # EF_LIB: an instrumented build of the same library (scripts/phase_profile.py)
        if not os.path.exists(path):
            raise EfError(f"{path} is missing: run `python -c 'import __graft_entry__ as g; g.build()'` or ./build.sh")
        _LIB = C.CDLL(path)
        _LIB.ef_error_string.restype = C.c_char_p
        _LIB.ef_stream.restype = C.c_void_p
    return _LIB


def _chk(rc):
    if rc != 0:
        raise EfError(f"libefusion call failed ({rc}): {lib().ef_error_string(rc).decode()}")


def _p(a):
    if a is None:
        return None
    assert a.flags["C_CONTIGUOUS"]
    return a.ctypes.data_as(C.c_void_p)


def _f(x):
    return C.c_float(float(x))


def _T(T):
    return None if T is None else np.ascontiguousarray(T, np.float64)


def default_config(width, height, fx, fy, cx, cy, **overrides) -> EfConfig:
    cfg = EfConfig()
    lib().ef_default_config(C.byref(cfg), width, height, _f(fx), _f(fy), _f(cx), _f(cy))
    for k, v in overrides.items():
        if not hasattr(cfg, k):
            raise KeyError(k)
        setattr(cfg, k, v)
    return cfg


class Context:
    """One EfContext: one device, one stream. Mirrors the stage API of include/efusion_b200.h."""

    def __init__(self, cfg: EfConfig, stream: int | None = None):
        self.cfg = cfg
        self.w, self.h = cfg.width, cfg.height
        self.h_ctx = C.c_void_p()
        _chk(lib().ef_create(C.byref(cfg), C.c_void_p(stream) if stream else None, C.byref(self.h_ctx)))

    def close(self):
        if getattr(self, "h_ctx", None):
            lib().ef_destroy(self.h_ctx)
            self.h_ctx = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    # ---- named buffers
    def _shape(self, bid, level):
        dt, kind = _BUF_FMT[bid % 100]
        r, c = (self.h >> level, self.w >> level) if bid % 100 >= 40 and bid % 100 != 53 else (self.h, self.w)
        if kind == "c1":
            return dt, (r, c)
        if kind == "p3":
            return dt, (3 * r, c)
        return dt, (r, c, int(kind[1]))

    def buffer_ptr(self, name, level=0, which=0):
        bid = BUF[name] + (100 * which if BUF[name] >= 40 else 0)
        ptr = C.c_void_p()
        nbytes = C.c_size_t()
        _chk(lib().ef_buffer(self.h_ctx, bid, level, C.byref(ptr), C.byref(nbytes)))
        return ptr.value, nbytes.value

    def download(self, name, level=0, which=0):
        bid = BUF[name] + (100 * which if BUF[name] >= 40 else 0)
        dt, shape = self._shape(bid, level)
        out = np.zeros(shape, dt)
        _chk(lib().ef_download(self.h_ctx, bid, level, _p(out), C.c_size_t(out.nbytes)))
        return out

    def upload(self, name, arr, level=0, which=0):
        bid = BUF[name] + (100 * which if BUF[name] >= 40 else 0)
        dt, shape = self._shape(bid, level)
        a = np.ascontiguousarray(arr, dt)
        assert a.shape == tuple(shape), (a.shape, shape)
        _chk(lib().ef_upload(self.h_ctx, bid, level, _p(a), C.c_size_t(a.nbytes)))

    def sync(self):
        _chk(lib().ef_sync(self.h_ctx))

    @property
    def stream(self):
        return lib().ef_stream(self.h_ctx)

    def launch_count(self):
        n = C.c_int64()
        _chk(lib().ef_launch_count(self.h_ctx, C.byref(n)))
        return n.value

    # ---- whole frame
    def process_frame(self, rgb, depth, timestamp=0, weight_multiplier=1.0, T_wc=None):
        """rgb = depth = None consumes the frame staged by prefetch_frame()."""
        if rgb is None and depth is None:
            _chk(lib().ef_process_frame(self.h_ctx, None, None, C.c_int64(timestamp), _f(weight_multiplier), _p(_T(T_wc))))
            return
        rgb = np.ascontiguousarray(rgb, np.uint8)
        depth = np.ascontiguousarray(depth, np.uint16)
        _chk(lib().ef_process_frame(self.h_ctx, _p(rgb), _p(depth), C.c_int64(timestamp), _f(weight_multiplier), _p(_T(T_wc))))

    def prefetch_frame(self, rgb, depth):
        """Look-ahead: stage + preprocess the NEXT frame (host arrays) on the side stream."""
        rgb = np.ascontiguousarray(rgb, np.uint8)
        depth = np.ascontiguousarray(depth, np.uint16)
        _chk(lib().ef_prefetch_frame(self.h_ctx, _p(rgb), _p(depth)))

    def prefetch_frame_device(self, rgb_ptr, depth_ptr):
        _chk(lib().ef_prefetch_frame_device(self.h_ctx, C.c_void_p(rgb_ptr), C.c_void_p(depth_ptr)))

    def finish_frame(self):
        _chk(lib().ef_finish_frame(self.h_ctx))

    def process_frame_device(self, rgb_ptr, depth_ptr, timestamp=0, weight_multiplier=1.0, T_wc=None):
        _chk(lib().ef_process_frame_device(self.h_ctx, C.c_void_p(rgb_ptr), C.c_void_p(depth_ptr), C.c_int64(timestamp),
                                           _f(weight_multiplier), _p(_T(T_wc))))

    def process_frame_begin(self, rgb, depth, timestamp=0, weight_multiplier=1.0, T_wc=None):
        rgb = np.ascontiguousarray(rgb, np.uint8)
        depth = np.ascontiguousarray(depth, np.uint16)
        _chk(lib().ef_process_frame_begin(self.h_ctx, _p(rgb), _p(depth), C.c_int64(timestamp), _f(weight_multiplier), _p(_T(T_wc))))

    def process_frame_end(self, T_override=None, nodes=None, fern_accepted=False):
        nd = None if nodes is None else np.ascontiguousarray(nodes, np.float32).reshape(-1, 16)
        _chk(lib().ef_process_frame_end(self.h_ctx, _p(_T(T_override)), _p(nd), 0 if nd is None else len(nd), int(fern_accepted)))

    def local_loop_result(self):
        """(info dict, src (n,3), dst (n,3), times (n,)) of the last frame's local loop closure front half."""
        res = EfLoopResult()
        cap = (self.w // 20) * (self.h // 20)
        src = np.zeros((cap, 3), np.float64)
        dst = np.zeros((cap, 3), np.float64)
        tm = np.zeros(cap, np.int32)
        n = C.c_int32()
        _chk(lib().ef_local_loop_result(self.h_ctx, C.byref(res), _p(src), _p(dst), _p(tm), cap, C.byref(n)))
        info = dict(ran=res.ran, accepted=res.accepted, n_constraints=res.n_constraints, lastICPError=res.lastICPError,
                    lastICPCount=res.lastICPCount, cov_diag=np.array(res.cov_diag[:]), T_wc_est=np.array(res.T_wc_est[:]).reshape(4, 4))
        return info, src[:n.value].copy(), dst[:n.value].copy(), tm[:n.value].copy()

    def deform_solve(self, node_pos, node_times, src, dst, src_times, dst_times=None, pin=False, last_deform_time=0):
        """Local-loop-closure deformation solve (ef_deform_solve). Returns (info dict, nodes16 (n,16) float32,
        constraint nodes (m,4) int32, constraint weights (m,4) float64, R (n,3,3) float64, t (n,3) float64); m counts the pin
        constraints when pin is set."""
        pos = np.ascontiguousarray(node_pos, np.float64).reshape(-1, 3)
        nt = np.ascontiguousarray(node_times, np.int32)
        s = np.ascontiguousarray(src, np.float64).reshape(-1, 3)
        d = np.ascontiguousarray(dst, np.float64).reshape(-1, 3)
        st = np.ascontiguousarray(src_times, np.int32)
        dt = None if dst_times is None else np.ascontiguousarray(dst_times, np.int32)
        n, nc = len(pos), len(s)
        m = 2 * nc if pin else nc
        nodes = np.zeros((max(n, 1), 16), np.float32)
        cn = np.zeros((max(m, 1), 4), np.int32)
        cw = np.zeros((max(m, 1), 4), np.float64)
        rt = np.zeros((max(n, 1), 12), np.float64)
        res = EfDeformResult()
        _chk(lib().ef_deform_solve(self.h_ctx, _p(pos), _p(nt), n, _p(s), _p(d), _p(st), _p(dt), nc, int(pin), int(last_deform_time),
                                   _p(nodes), _p(rt), _p(cn), _p(cw), C.byref(res)))
        info = {k: getattr(res, k) for k, _ in EfDeformResult._fields_}
        R = rt[:n, :9].reshape(n, 3, 3).transpose(0, 2, 1).copy()  # column-major -> R[i, row, col]
        return info, nodes[:n], cn[:m], cw[:m], R, rt[:n, 9:].copy()

    def local_deform_result(self):
        """close_loops = 2: (info dict, graph (n, 4) float32: x y z time per node) of the last frame's in-frame loop closure.
        info: solved, applied, result (EfDeformResult fields, all zero unless solved), deforms, last_deform_time, n_nodes."""
        return _local_deform(lambda res, nodes, n: lib().ef_local_deform_result(self.h_ctx, res, _p(nodes), len(nodes), n))

    def predict(self):
        _chk(lib().ef_predict(self.h_ctx))

    def get_pose(self):
        T = np.zeros((4, 4), np.float64)
        _chk(lib().ef_get_pose(self.h_ctx, _p(T)))
        return T

    def set_pose(self, T):
        _chk(lib().ef_set_pose(self.h_ctx, _p(_T(T))))

    def get_tick(self):
        t = C.c_int32()
        _chk(lib().ef_get_tick(self.h_ctx, C.byref(t)))
        return t.value

    def set_tick(self, t):
        _chk(lib().ef_set_tick(self.h_ctx, int(t)))

    def set(self, **kw):
        fns = dict(rgb_only=("ef_set_rgb_only", int), icp_weight=("ef_set_icp_weight", _f), pyramid=("ef_set_pyramid", int),
                   fast_odom=("ef_set_fast_odom", int), so3=("ef_set_so3", int),
                   frame_to_frame_rgb=("ef_set_frame_to_frame_rgb", int),
                   confidence_threshold=("ef_set_confidence_threshold", _f), depth_cutoff=("ef_set_depth_cutoff", _f))
        for k, v in kw.items():
            name, conv = fns[k]
            _chk(getattr(lib(), name)(self.h_ctx, conv(v)))

    # ---- tracker stages
    def odom_init_icp_depth(self, depth_ptr, cutoff, which=0):
        _chk(lib().ef_odom_init_icp_depth(self.h_ctx, which, C.c_void_p(depth_ptr), _f(cutoff)))

    def odom_init_icp_pred(self, vtx_ptr, nrm_ptr, which=0):
        _chk(lib().ef_odom_init_icp_pred(self.h_ctx, which, C.c_void_p(vtx_ptr), C.c_void_p(nrm_ptr)))

    def odom_init_icp_model(self, vtx_ptr, nrm_ptr, T_wc, which=0):
        _chk(lib().ef_odom_init_icp_model(self.h_ctx, which, C.c_void_p(vtx_ptr), C.c_void_p(nrm_ptr), _p(_T(T_wc))))

    def odom_init_rgb(self, rgba_ptr, which=0):
        _chk(lib().ef_odom_init_rgb(self.h_ctx, which, C.c_void_p(rgba_ptr)))

    def odom_init_rgb_model(self, rgba_ptr, which=0):
        _chk(lib().ef_odom_init_rgb_model(self.h_ctx, which, C.c_void_p(rgba_ptr)))

    def odom_init_first_rgb(self, rgba_ptr, which=0):
        _chk(lib().ef_odom_init_first_rgb(self.h_ctx, which, C.c_void_p(rgba_ptr)))

    def odom_track(self, T_wc, rgb_only=False, icp_weight=10.0, pyramid=True, fast_odom=False, so3=True, which=0, max_trace=48):
        T = _T(T_wc).copy()
        trace = np.zeros(max_trace, TRACE_DTYPE)
        n = C.c_int32()
        _chk(lib().ef_odom_track(self.h_ctx, which, _p(T), int(rgb_only), _f(icp_weight), int(pyramid), int(fast_odom), int(so3),
                                 _p(trace), max_trace, C.byref(n)))
        return T, trace[:n.value]

    def odom_stats(self, which=0):
        st = np.zeros(1, STATS_DTYPE)
        _chk(lib().ef_odom_stats(self.h_ctx, which, _p(st)))
        return st[0]

    def odom_covariance(self, which=0):
        cov = np.zeros((6, 6), np.float64)
        _chk(lib().ef_odom_covariance(self.h_ctx, which, _p(cov)))
        return cov

    def icp_step(self, level, Rcurr, tcurr, Rprev_inv, tprev, which=0):
        f32 = lambda a: np.ascontiguousarray(a, np.float32)
        A, b, res = np.zeros((6, 6), np.float32), np.zeros(6, np.float32), np.zeros(2, np.float32)
        Rc, tc, Rp, tp = f32(Rcurr), f32(tcurr), f32(Rprev_inv), f32(tprev)
        _chk(lib().ef_icp_step(self.h_ctx, which, level, _p(Rc), _p(tc), _p(Rp), _p(tp), _p(A), _p(b), _p(res)))
        return A, b, res

    def icp_step_async(self, level, Rcurr=None, tcurr=None, Rprev_inv=None, tprev=None, which=0):
        if Rcurr is None:
            _chk(lib().ef_icp_step_async(self.h_ctx, which, level, None, None, None, None))
            return
        f32 = lambda a: np.ascontiguousarray(a, np.float32)
        Rc, tc, Rp, tp = f32(Rcurr), f32(tcurr), f32(Rprev_inv), f32(tprev)
        _chk(lib().ef_icp_step_async(self.h_ctx, which, level, _p(Rc), _p(tc), _p(Rp), _p(tp)))

    def icp_dense_pass_async(self, level, which=0):
        _chk(lib().ef_icp_dense_pass_async(self.h_ctx, which, level))

    def rgb_residual(self, level, krkinv, kt, which=0):
        kk = np.ascontiguousarray(krkinv, np.float32)
        k3 = np.ascontiguousarray(kt, np.float32)
        sigma, count = C.c_int32(), C.c_int32()
        _chk(lib().ef_rgb_residual(self.h_ctx, which, level, _p(kk), _p(k3), C.byref(sigma), C.byref(count)))
        return sigma.value, count.value

    def rgb_step(self, level, sigma, which=0):
        A, b = np.zeros((6, 6), np.float32), np.zeros(6, np.float32)
        _chk(lib().ef_rgb_step(self.h_ctx, which, level, _f(sigma), _p(A), _p(b)))
        return A, b

    def so3_step(self, image_basis, kinv, krlr, which=0):
        f32 = lambda a: np.ascontiguousarray(a, np.float32)
        A, b, res = np.zeros((3, 3), np.float32), np.zeros(3, np.float32), np.zeros(2, np.float32)
        ib, ki, kr = f32(image_basis), f32(kinv), f32(krlr)
        _chk(lib().ef_so3_step(self.h_ctx, which, _p(ib), _p(ki), _p(kr), _p(A), _p(b), _p(res)))
        return A, b, res

    # ---- preprocess + map stages
    def preprocess_depth(self, raw_ptr, cutoff, filtered_ptr, metric_ptr, metric_filtered_ptr):
        _chk(lib().ef_preprocess_depth(self.h_ctx, C.c_void_p(raw_ptr), _f(cutoff), C.c_void_p(filtered_ptr),
                                       C.c_void_p(metric_ptr), C.c_void_p(metric_filtered_ptr)))

    def map_initialise(self):
        _chk(lib().ef_map_initialise(self.h_ctx))

    def map_predict_indices(self, T_wc, time, max_depth, time_delta):
        _chk(lib().ef_map_predict_indices(self.h_ctx, _p(_T(T_wc)), int(time), _f(max_depth), int(time_delta)))

    def map_fuse(self, T_wc, time, max_depth, weighting):
        _chk(lib().ef_map_fuse(self.h_ctx, _p(_T(T_wc)), int(time), _f(max_depth), _f(weighting)))

    def map_clean(self, T_wc, time, conf_threshold, time_delta, max_depth):
        _chk(lib().ef_map_clean(self.h_ctx, _p(_T(T_wc)), int(time), _f(conf_threshold), int(time_delta), _f(max_depth)))

    def map_clean_deform(self, T_wc, time, conf_threshold, time_delta, max_depth, nodes, is_fern=False):
        nd = np.ascontiguousarray(nodes, np.float32).reshape(-1, 16)
        _chk(lib().ef_map_clean_deform(self.h_ctx, _p(_T(T_wc)), int(time), _f(conf_threshold), int(time_delta), _f(max_depth), _p(nd), len(nd),
                                       int(is_fern)))

    def map_raycast(self, T_wc, max_depth, conf_threshold, time, max_time, time_delta, mode=0):
        _chk(lib().ef_map_raycast(self.h_ctx, _p(_T(T_wc)), _f(max_depth), _f(conf_threshold), int(time), int(max_time),
                                  int(time_delta), int(mode)))

    def map_fill_in(self, passthrough_geometry=False, passthrough_image=False):
        _chk(lib().ef_map_fill_in(self.h_ctx, int(passthrough_geometry), int(passthrough_image)))

    def dense_enough(self):
        out = C.c_int32()
        _chk(lib().ef_dense_enough(self.h_ctx, C.byref(out)))
        return bool(out.value)

    def map_count(self):
        n = C.c_int32()
        _chk(lib().ef_map_count(self.h_ctx, C.byref(n)))
        return n.value

    def map_download(self):
        n = self.map_count()
        out = np.zeros((max(n, 1), 12), np.float32)
        cnt = C.c_int32()
        _chk(lib().ef_map_download(self.h_ctx, _p(out), n, C.byref(cnt)))
        return out[:n]

    def map_download_new(self):
        out = np.zeros((self.w * self.h, 12), np.float32)
        cnt = C.c_int32()
        _chk(lib().ef_map_download_new(self.h_ctx, _p(out), self.w * self.h, C.byref(cnt)))
        return out[:cnt.value].copy()

    def map_upload_range(self, surfels, first):
        s = np.ascontiguousarray(surfels, np.float32)
        _chk(lib().ef_map_upload_range(self.h_ctx, _p(s), int(first), len(s)))

    def join_lookahead(self):
        _chk(lib().ef_join_lookahead(self.h_ctx))

    def stage_ms(self):
        """EF_STAGE_TIMING=1 (set before the context is created): ms per stage of the last frame, index as in the header."""
        out = (C.c_float * 16)()
        n = lib().ef_debug_stage_ms(self.h_ctx, out)
        return [out[i] for i in range(n)]

    def lookahead_ms(self):
        """EF_STAGE_TIMING=1: (start, end) of the last prefetch's side-stream work, ms after the start of the frame in flight
        when it was enqueued; None without a timed prefetch."""
        out = (C.c_float * 2)()
        n = lib().ef_debug_lookahead_ms(self.h_ctx, out)
        return (out[0], out[1]) if n == 2 else None

    def render(self, view: EfRenderView):
        """ef_render_map: the map drawn as the reference viewer draws it, (H, W, 4) uint8, row 0 = window y 0."""
        out = np.zeros((view.height, view.width, 4), np.uint8)
        _chk(lib().ef_render_map(self.h_ctx, C.byref(view), _p(out)))
        return out

    def render_device(self, view: EfRenderView, ptr):
        """ef_render_map_device: the same into device memory at ptr (H*W*4 bytes), asynchronous on the context's stream."""
        _chk(lib().ef_render_map_device(self.h_ctx, C.byref(view), C.c_void_p(ptr)))

    def predict_view(self, view: EfModelView, outputs=("image", "vertex", "normal", "time")):
        """ef_map_predict_view: combinedPredict at the view's pose, camera and size, without touching the frame. Returns a dict of the
        requested outputs: image (H, W, 4) uint8, vertex and normal (H, W, 4) float32, time (H, W) uint16; row 0 is the top image
        row, uncovered pixels are zero, the depth is vertex[..., 2]."""
        out = {}
        for name in outputs:
            dt, ch = VIEW_OUTPUTS[name]
            out[name] = np.zeros((view.height, view.width, ch) if ch > 1 else (view.height, view.width), dt)
        _chk(lib().ef_map_predict_view(self.h_ctx, C.byref(view), *(_p(out.get(n)) for n in VIEW_OUTPUTS)))
        return out

    def predict_view_device(self, view: EfModelView, image=0, vertex=0, normal=0, time=0):
        """ef_map_predict_view_device: the same into device memory (H*W*4, H*W*16, H*W*16, H*W*2 bytes; 0 = not wanted),
        asynchronous on the context's stream."""
        _chk(lib().ef_map_predict_view_device(self.h_ctx, C.byref(view), *(C.c_void_p(p or None) for p in (image, vertex, normal, time))))

    def fuse_view(self, view: EfFuseView, rgb, depth):
        """ef_map_fuse_view: fuses an RGB-D frame of the view's camera into the map -- rgb (H, W, 3) uint8, depth (H, W) uint16
        millimetres -- without touching the frame's pose, tick, textures or tracker state. Synchronises."""
        r = np.ascontiguousarray(rgb, np.uint8)
        d = np.ascontiguousarray(depth, np.uint16)
        assert r.shape == (view.height, view.width, 3) and d.shape == (view.height, view.width), (r.shape, d.shape)
        _chk(lib().ef_map_fuse_view(self.h_ctx, C.byref(view), _p(r), _p(d)))

    def fuse_view_device(self, view: EfFuseView, rgb_ptr, depth_ptr):
        """ef_map_fuse_view_device: the same from device memory (H*W*3 and H*W*2 bytes), asynchronous on the context's stream."""
        _chk(lib().ef_map_fuse_view_device(self.h_ctx, C.byref(view), C.c_void_p(rgb_ptr or None), C.c_void_p(depth_ptr or None)))

    def track_view(self, view: EfTrackView, rgb, depth, max_trace=0):
        """ef_track_view: tracks an RGB-D frame of the view's camera -- rgb (H, W, 3) uint8, depth (H, W) uint16 millimetres -- against
        the map from the view's guess, without touching the frame. Synchronises. Returns (T_wc (4, 4), stats (as odom_stats),
        covariance (6, 6), dense_enough, trace (the first max_trace Gauss-Newton records, TRACE_DTYPE))."""
        h, w = view.model.height, view.model.width
        r = np.ascontiguousarray(rgb, np.uint8)
        d = np.ascontiguousarray(depth, np.uint16)
        assert r.shape == (h, w, 3) and d.shape == (h, w), (r.shape, d.shape)
        res = EfTrackResult()
        trace = np.zeros(max(max_trace, 1), TRACE_DTYPE)
        n = C.c_int32()
        _chk(lib().ef_track_view(self.h_ctx, C.byref(view), _p(r), _p(d), C.byref(res), _p(trace) if max_trace else None, int(max_trace),
                                 C.byref(n)))
        return (*unpack_track_result(res), trace[:n.value].copy())

    def track_view_device(self, view: EfTrackView, rgb_ptr, depth_ptr, result_ptr):
        """ef_track_view_device: the same from device memory (H*W*3 and H*W*2 bytes) into an EfTrackResult in device memory
        (ctypes.sizeof(EfTrackResult) bytes, 8-byte aligned; unpack_track_result reads its bytes), asynchronous on the context's stream."""
        _chk(lib().ef_track_view_device(self.h_ctx, C.byref(view), C.c_void_p(rgb_ptr or None), C.c_void_p(depth_ptr or None),
                                        C.c_void_p(result_ptr or None)))

    def camera(self, cfg: EfCameraConfig) -> "Camera":
        """ef_camera_create: a camera of this context (at most MAX_CAMERAS live ones)."""
        return Camera(self, cfg)

    def rig(self, cameras, extrinsics=None, joint_so3=False) -> "Rig":
        """ef_rig_create: the cameras tracked as one rigid body; extrinsics[i] is T_0i (4x4, camera i -> cameras[0]'s camera; default:
        identities); joint_so3: one SO(3) pre-alignment over every member's images instead of member 0's."""
        return Rig(self, cameras, extrinsics, joint_so3)

    def map_upload(self, surfels):
        s = np.ascontiguousarray(surfels, np.float32)
        _chk(lib().ef_map_upload(self.h_ctx, _p(s), len(s)))


class Camera:
    """One EfCamera of a Context: a second RGB-D sensor run frame after frame against the context's map (include/efusion_b200.h)."""

    def __init__(self, ctx: Context, cfg: EfCameraConfig):
        self.ctx, self.cfg = ctx, cfg
        self.w, self.h = cfg.width, cfg.height
        self.h_cam = C.c_void_p()
        _chk(lib().ef_camera_create(ctx.h_ctx, C.byref(cfg), C.byref(self.h_cam)))

    def close(self):
        """ef_camera_destroy (a no-op once the camera or its context is closed)"""
        if getattr(self, "h_cam", None) and self.ctx.h_ctx:
            _chk(lib().ef_camera_destroy(self.ctx.h_ctx, self.h_cam))
        self.h_cam = None

    def frame(self, rgb, depth, time, weight_multiplier=1.0, T_wc=None, fuse=True, max_trace=0):
        """ef_camera_frame: rgb (H, W, 3) uint8, depth (H, W) uint16 millimetres; T_wc sets the pose instead of tracking. Synchronises.
        Returns (T_wc (4, 4), stats (as Context.odom_stats), covariance (6, 6), {tracked, dense_enough, weighting}, trace (the first
        max_trace Gauss-Newton records of a tracked frame, TRACE_DTYPE))."""
        r = np.ascontiguousarray(rgb, np.uint8)
        d = np.ascontiguousarray(depth, np.uint16)
        assert r.shape == (self.h, self.w, 3) and d.shape == (self.h, self.w), (r.shape, d.shape)
        f = camera_frame(time, weight_multiplier, T_wc, fuse)
        res = EfCameraResult()
        trace = np.zeros(max(max_trace, 1), TRACE_DTYPE)
        n = C.c_int32()
        _chk(lib().ef_camera_frame(self.ctx.h_ctx, self.h_cam, C.byref(f), _p(r), _p(d), C.byref(res), _p(trace) if max_trace else None,
                                   int(max_trace), C.byref(n)))
        return (*unpack_camera_result(res), trace[:n.value].copy())

    def frame_device(self, rgb_ptr, depth_ptr, result_ptr, time, weight_multiplier=1.0, T_wc=None, fuse=True):
        """ef_camera_frame_device: the same from device memory (H*W*3 and H*W*2 bytes) into an EfCameraResult in device memory
        (ctypes.sizeof(EfCameraResult) bytes, 8-byte aligned; unpack_camera_result reads its bytes), asynchronous on the context's stream."""
        f = camera_frame(time, weight_multiplier, T_wc, fuse)
        _chk(lib().ef_camera_frame_device(self.ctx.h_ctx, self.h_cam, C.byref(f), C.c_void_p(rgb_ptr or None), C.c_void_p(depth_ptr or None),
                                          C.c_void_p(result_ptr or None)))

    def deform_result(self):
        """close_loops: (info dict, graph) of the camera's last frame, as Context.local_deform_result returns them (solved, applied and
        result are the camera's; deforms, last_deform_time and the graph the context's)."""
        return _local_deform(lambda res, nodes, n: lib().ef_camera_deform_result(self.ctx.h_ctx, self.h_cam, res, _p(nodes), len(nodes), n))

    def buffer_ptr(self, name, level=0):
        ptr, nbytes = C.c_void_p(), C.c_size_t()
        _chk(lib().ef_camera_buffer(self.ctx.h_ctx, self.h_cam, BUF[name], level, C.byref(ptr), C.byref(nbytes)))
        return ptr.value, nbytes.value

    def download(self, name, level=0):
        """A buffer of the camera (ef_camera_buffer: its inputs, prediction, fill-in and pyramids) as Context.download shapes it."""
        bid = BUF[name]
        dt, kind = _BUF_FMT[bid]
        r, c = (self.h >> level, self.w >> level) if bid >= 40 and bid != 53 else (self.h, self.w)
        shape = (r, c) if kind == "c1" else (3 * r, c) if kind == "p3" else (r, c, int(kind[1]))
        out = np.zeros(shape, dt)
        ptr, nbytes = self.buffer_ptr(name, level)
        assert nbytes == out.nbytes, (name, nbytes, out.nbytes)
        self.ctx.sync()
        # cudaMemcpy of the CUDA runtime the library links (device to host = 2)
        _chk(lib().cudaMemcpy(_p(out), C.c_void_p(ptr), C.c_size_t(nbytes), 2))
        return out


class Rig:
    """One EfRig of a Context: cameras bolted together at known extrinsics, tracked as one rigid body (include/efusion_b200.h)."""

    def __init__(self, ctx: Context, cameras, extrinsics=None, joint_so3=False):
        self.ctx, self.cameras = ctx, list(cameras)
        self.n = len(self.cameras)
        cfg = EfRigConfig()
        cfg.n = self.n
        cfg.joint_so3 = 1 if joint_so3 else 0
        for i, cam in enumerate(self.cameras[:MAX_CAMERAS]):
            cfg.cameras[i] = cam.h_cam.value if cam.h_cam else None
            T = np.eye(4) if extrinsics is None else np.asarray(extrinsics[i], np.float64)
            cfg.T_0i[i][:] = T.reshape(16).tolist()
        self.h_rig = C.c_void_p()
        _chk(lib().ef_rig_create(ctx.h_ctx, C.byref(cfg), C.byref(self.h_rig)))

    def close(self):
        """ef_rig_destroy (a no-op once the rig, one of its cameras or its context is closed)"""
        if getattr(self, "h_rig", None) and self.ctx.h_ctx and all(c.h_cam for c in self.cameras):
            _chk(lib().ef_rig_destroy(self.ctx.h_ctx, self.h_rig))
        self.h_rig = None

    def frame(self, inputs, time, weight_multiplier=1.0, T_wc=None, fuse=True, max_trace=0):
        """ef_rig_frame: inputs[i] = (rgb (H, W, 3) uint8, depth (H, W) uint16 millimetres) of member i; T_wc (member 0's) sets the pose
        instead of tracking. Synchronises. Returns (the members' results as Camera.frame unpacks them, each with its trace,
        unpack_rig_result of the rig's)."""
        arrs = []
        for cam, (rgb, depth) in zip(self.cameras, inputs):
            r, d = np.ascontiguousarray(rgb, np.uint8), np.ascontiguousarray(depth, np.uint16)
            assert r.shape == (cam.h, cam.w, 3) and d.shape == (cam.h, cam.w), (r.shape, d.shape)
            arrs.append((r, d))
        assert len(arrs) == self.n
        rgbs = (C.c_void_p * self.n)(*[r.ctypes.data for r, _ in arrs])
        depths = (C.c_void_p * self.n)(*[d.ctypes.data for _, d in arrs])
        members = (EfCameraResult * self.n)()
        out = EfRigResult()
        trace = np.zeros(max(max_trace, 1) * self.n, TRACE_DTYPE)
        n_trace = (C.c_int32 * self.n)()
        f = rig_frame(time, weight_multiplier, T_wc, fuse)
        _chk(lib().ef_rig_frame(self.ctx.h_ctx, self.h_rig, C.byref(f), rgbs, depths, members, C.byref(out),
                                _p(trace) if max_trace else None, int(max_trace), n_trace))
        res = [(*unpack_camera_result(members[i]), trace[i * max_trace:i * max_trace + n_trace[i]].copy()) for i in range(self.n)]
        return res, unpack_rig_result(out)

    def frame_device(self, rgb_ptrs, depth_ptrs, members_ptr, result_ptr, time, weight_multiplier=1.0, T_wc=None, fuse=True):
        """ef_rig_frame_device: the same from device memory into device results (members_ptr: n EfCameraResult, result_ptr: one
        EfRigResult, 8-byte aligned), asynchronous on the context's stream."""
        rgbs = (C.c_void_p * self.n)(*rgb_ptrs)
        depths = (C.c_void_p * self.n)(*depth_ptrs)
        f = rig_frame(time, weight_multiplier, T_wc, fuse)
        _chk(lib().ef_rig_frame_device(self.ctx.h_ctx, self.h_rig, C.byref(f), rgbs, depths, C.c_void_p(members_ptr or None),
                                       C.c_void_p(result_ptr or None)))

    def loop_result(self):
        """A closing rig: (info dict, src (n,3), dst (n,3), times (n,), member_counts (n_members,)) of its last frame's front half, as
        Context.local_loop_result returns the frame's; the constraints are the members', concatenated in member order."""
        res = EfRigLoopResult()
        cap = sum((c.w // 20) * (c.h // 20) for c in self.cameras)
        src = np.zeros((cap, 3), np.float64)
        dst = np.zeros((cap, 3), np.float64)
        tm = np.zeros(cap, np.int32)
        n = C.c_int32()
        _chk(lib().ef_rig_loop_result(self.ctx.h_ctx, self.h_rig, C.byref(res), _p(src), _p(dst), _p(tm), cap, C.byref(n)))
        info = dict(ran=res.ran, accepted=res.accepted, n_constraints=res.n_constraints, lastICPError=res.lastICPError,
                    lastICPCount=res.lastICPCount, cov_diag=np.array(res.cov_diag[:]), T_wc_curr=np.array(res.T_wc_curr[:]).reshape(4, 4),
                    T_wc_est=np.array(res.T_wc_est[:]).reshape(4, 4))
        counts = np.array(res.member_constraints[:self.n], np.int32)
        return info, src[:n.value].copy(), dst[:n.value].copy(), tm[:n.value].copy(), counts

    def deform_result(self):
        """A closing rig: (info dict, graph) of its last frame, as Camera.deform_result returns them (solved, applied and result are
        the rig's; deforms, last_deform_time and the graph the context's)."""
        return _local_deform(lambda res, nodes, n: lib().ef_rig_deform_result(self.ctx.h_ctx, self.h_rig, res, _p(nodes), len(nodes), n))
