"""TEST INFRASTRUCTURE ONLY — ctypes binding for the CPU oracle (oracle/libef_oracle.so).

Imported only by tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs.
The product package (elasticfusion_b200/) never imports this module.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB = None


def build(force: bool = False) -> str:
    so = os.path.join(_HERE, "libef_oracle.so")
    srcs = [os.path.join(_HERE, f) for f in ("efo_track.cpp", "efo_map.cpp", "efo_pipeline.cpp", "ef_oracle.h",
                                             "efo_common.h", "efo_linalg.h")]
    stale = (not os.path.exists(so)) or any(os.path.getmtime(s) > os.path.getmtime(so) for s in srcs)
    if force or stale:
        subprocess.check_call(["make", "-C", _HERE, "libef_oracle.so"], stdout=subprocess.DEVNULL)
    return so


def lib():
    global _LIB
    if _LIB is None:
        _LIB = C.CDLL(build())
        _LIB.efo_odom_create.restype = C.c_void_p
        _LIB.efo_fusion_create.restype = C.c_void_p
        _LIB.efo_odom_buffer.restype = C.c_void_p
        _LIB.efo_fusion_buffer.restype = C.c_void_p
        _LIB.efo_fusion_map.restype = C.c_void_p
        _LIB.efo_fusion_odometry.restype = C.c_void_p
    return _LIB


def set_threads(n: int) -> None:
    """OpenMP thread count of the oracle (torchrun exports OMP_NUM_THREADS=1, which libgomp may already have read)."""
    lib()
    try:
        C.CDLL("libgomp.so.1").omp_set_num_threads(int(n))
    except OSError:
        pass


def get_threads() -> int:
    """OpenMP team size the oracle will use."""
    lib()
    try:
        return int(C.CDLL("libgomp.so.1").omp_get_max_threads())
    except OSError:
        return 1


class DataTerm(C.Structure):
    _fields_ = [("zero_x", C.c_int16), ("zero_y", C.c_int16), ("one_x", C.c_int16), ("one_y", C.c_int16),
                ("diff", C.c_float), ("valid", C.c_int32)]


DATATERM_DTYPE = np.dtype([("zero_x", "<i2"), ("zero_y", "<i2"), ("one_x", "<i2"), ("one_y", "<i2"),
                           ("diff", "<f4"), ("valid", "<i4")])

TRACE_DTYPE = np.dtype([
    ("kind", "<i4"), ("level", "<i4"), ("iter", "<i4"), ("rgb_count", "<i4"), ("rgb_sigma", "<i4"),
    ("sigma_val", "<f4"),
    ("A_icp", "<f4", (36,)), ("b_icp", "<f4", (6,)), ("icp_residual", "<f4", (2,)),
    ("A_rgb", "<f4", (36,)), ("b_rgb", "<f4", (6,)),
    ("A_so3", "<f4", (9,)), ("b_so3", "<f4", (3,)), ("so3_residual", "<f4", (2,)),
    ("lastA", "<f8", (36,)), ("lastb", "<f8", (6,)), ("result", "<f8", (6,)),
], align=True)


class Config(C.Structure):
    _fields_ = [("width", C.c_int), ("height", C.c_int), ("fx", C.c_float), ("fy", C.c_float), ("cx", C.c_float),
                ("cy", C.c_float), ("time_delta", C.c_int), ("confidence", C.c_float), ("depth_cutoff", C.c_float),
                ("icp_weight", C.c_float), ("fast_odom", C.c_int), ("so3", C.c_int), ("frame_to_frame_rgb", C.c_int),
                ("pyramid", C.c_int), ("rgb_only", C.c_int), ("capacity", C.c_int)]


class LoopResult(C.Structure):
    _fields_ = [("ran", C.c_int32), ("accepted", C.c_int32), ("n_constraints", C.c_int32), ("lastICPError", C.c_float),
                ("lastICPCount", C.c_float), ("cov_diag", C.c_double * 6), ("T_wc_est", C.c_double * 16)]


def _p(a, t=None):
    if a is None:
        return None
    assert a.flags["C_CONTIGUOUS"], "array must be C contiguous"
    return a.ctypes.data_as(C.c_void_p)


def _f(x):
    return C.c_float(float(x))


# ------------------------------------------------------------------ image kernels
def pyr_down_u16(src):
    r, c = src.shape
    dst = np.zeros((r // 2, c // 2), np.uint16)
    lib().efo_pyr_down_u16(_p(src), r, c, _p(dst))
    return dst


def create_vmap(depth, fx, fy, cx, cy, cutoff, out=None):
    r, c = depth.shape
    vmap = np.full((3 * r, c), np.nan, np.float32) if out is None else out
    lib().efo_create_vmap(_p(depth), r, c, _f(fx), _f(fy), _f(cx), _f(cy), _f(cutoff), _p(vmap))
    return vmap


def create_nmap(vmap):
    r, c = vmap.shape[0] // 3, vmap.shape[1]
    nmap = np.full((3 * r, c), np.nan, np.float32)
    lib().efo_create_nmap(_p(vmap), r, c, _p(nmap))
    return nmap


def transform_maps(vmap, nmap, R, t):
    r, c = vmap.shape[0] // 3, vmap.shape[1]
    R = np.ascontiguousarray(R, np.float32)
    t = np.ascontiguousarray(t, np.float32)
    lib().efo_transform_maps(_p(vmap), _p(nmap), r, c, _p(R), _p(t))


def copy_maps(vtx4, nrm4):
    r, c = vtx4.shape[:2]
    tmp = np.zeros((r, c, 4), np.float32)
    vmap = np.zeros((3 * r, c), np.float32)
    nmap = np.zeros((3 * r, c), np.float32)
    lib().efo_copy_maps(_p(vtx4), _p(nrm4), r, c, _p(tmp), _p(vmap), _p(nmap))
    return tmp, vmap, nmap


def resize_map(m, normalize):
    r, c = m.shape[0] // 3, m.shape[1]
    out = np.full((3 * (r // 2), c // 2), np.nan, np.float32)
    lib().efo_resize_map(_p(m), r, c, _p(out), int(normalize))
    return out


def pyr_down_gauss_f(src):
    r, c = src.shape
    dst = np.zeros((r // 2, c // 2), np.float32)
    lib().efo_pyr_down_gauss_f(_p(src), r, c, _p(dst))
    return dst


def pyr_down_u8(src):
    r, c = src.shape
    dst = np.zeros((r // 2, c // 2), np.uint8)
    lib().efo_pyr_down_u8(_p(src), r, c, _p(dst))
    return dst


def vertices_to_depth(vmaps_tmp, cutoff):
    r, c = vmaps_tmp.shape[:2]
    dst = np.zeros((r, c), np.float32)
    lib().efo_vertices_to_depth(_p(vmaps_tmp), r, c, _f(cutoff), _p(dst))
    return dst


def rgba_to_intensity(rgba):
    r, c = rgba.shape[:2]
    dst = np.zeros((r, c), np.uint8)
    lib().efo_rgba_to_intensity(_p(rgba), r, c, _p(dst))
    return dst


def sobel(src):
    r, c = src.shape
    dx = np.zeros((r, c), np.int16)
    dy = np.zeros((r, c), np.int16)
    lib().efo_sobel(_p(src), r, c, _p(dx), _p(dy))
    return dx, dy


def project_points(depth, fx, fy, cx, cy):
    r, c = depth.shape
    cloud = np.zeros((r, c, 3), np.float32)
    lib().efo_project_points(_p(depth), r, c, _f(fx), _f(fy), _f(cx), _f(cy), _p(cloud))
    return cloud


# ------------------------------------------------------------------ reductions
def icp_step(Rcurr, tcurr, vmap_curr, nmap_curr, Rprev_inv, tprev, fx, fy, cx, cy, vmap_g_prev, nmap_g_prev,
             dist_thres, angle_thres):
    r, c = vmap_curr.shape[0] // 3, vmap_curr.shape[1]
    A = np.zeros((6, 6), np.float32)
    b = np.zeros(6, np.float32)
    res = np.zeros(2, np.float32)
    f32 = lambda a: np.ascontiguousarray(a, np.float32)
    Rc, tc, Rp, tp = f32(Rcurr), f32(tcurr), f32(Rprev_inv), f32(tprev)
    lib().efo_icp_step(_p(Rc), _p(tc), _p(vmap_curr), _p(nmap_curr), _p(Rp), _p(tp), _f(fx), _f(fy), _f(cx), _f(cy),
                       _p(vmap_g_prev), _p(nmap_g_prev), _f(dist_thres), _f(angle_thres), r, c, _p(A), _p(b), _p(res))
    return A, b, res


def rgb_residual(min_scale, dIdx, dIdy, last_depth, next_depth, last_image, next_image, max_depth_delta, kt, krkinv):
    r, c = next_image.shape
    corres = np.zeros((r, c), DATATERM_DTYPE)
    sigma = C.c_int(0)
    count = C.c_int(0)
    kt = np.ascontiguousarray(kt, np.float32)
    kk = np.ascontiguousarray(krkinv, np.float32)
    lib().efo_rgb_residual(_f(min_scale), _p(dIdx), _p(dIdy), _p(last_depth), _p(next_depth), _p(last_image),
                           _p(next_image), _p(corres), _f(max_depth_delta), _p(kt), _p(kk), r, c, C.byref(sigma),
                           C.byref(count))
    return corres, sigma.value, count.value


def rgb_step(corres, sigma, cloud, fx, fy, dIdx, dIdy, sobel_scale):
    r, c = corres.shape
    A = np.zeros((6, 6), np.float32)
    b = np.zeros(6, np.float32)
    lib().efo_rgb_step(_p(corres), _f(sigma), _p(cloud), _f(fx), _f(fy), _p(dIdx), _p(dIdy), _f(sobel_scale), r, c,
                       _p(A), _p(b))
    return A, b


def so3_step(last_image, next_image, image_basis, kinv, krlr):
    r, c = next_image.shape
    A = np.zeros((3, 3), np.float32)
    b = np.zeros(3, np.float32)
    res = np.zeros(2, np.float32)
    f32 = lambda a: np.ascontiguousarray(a, np.float32)
    ib, ki, kr = f32(image_basis), f32(kinv), f32(krlr)
    lib().efo_so3_step(_p(last_image), _p(next_image), _p(ib), _p(ki), _p(kr), r, c, _p(A), _p(b), _p(res))
    return A, b, res


# ------------------------------------------------------------------ odometry object
class Odometry:
    BUF = {"vmap_curr": (0, np.float32, 3), "nmap_curr": (1, np.float32, 3), "vmap_g_prev": (2, np.float32, 3),
           "nmap_g_prev": (3, np.float32, 3), "lastDepth": (4, np.float32, 1), "nextDepth": (5, np.float32, 1),
           "lastImage": (6, np.uint8, 1), "nextImage": (7, np.uint8, 1), "lastNextImage": (8, np.uint8, 1),
           "dIdx": (9, np.int16, 1), "dIdy": (10, np.int16, 1), "depth_tmp": (11, np.uint16, 1)}

    def __init__(self, width, height, cx, cy, fx, fy, dist_thresh=0.10,
                 angle_thresh=float(np.sin(np.float32(20.0) * np.float32(3.14159254) / np.float32(180.0))),
                 handle=None):
        self.w, self.h = width, height
        self._own = handle is None
        self.hnd = C.c_void_p(handle) if handle is not None else C.c_void_p(
            lib().efo_odom_create(width, height, _f(cx), _f(cy), _f(fx), _f(fy), _f(dist_thresh), _f(angle_thresh)))

    def __del__(self):
        if getattr(self, "_own", False) and self.hnd:
            lib().efo_odom_destroy(self.hnd)
            self.hnd = None

    def init_icp_depth(self, depth, cutoff):
        lib().efo_odom_init_icp_depth(self.hnd, _p(depth), _f(cutoff))

    def init_icp_pred(self, vtx4, nrm4):
        lib().efo_odom_init_icp_pred(self.hnd, _p(vtx4), _p(nrm4))

    def init_icp_model(self, vtx4, nrm4, T_wc):
        T = np.ascontiguousarray(T_wc, np.float64)
        lib().efo_odom_init_icp_model(self.hnd, _p(vtx4), _p(nrm4), _p(T))

    def init_rgb(self, rgba):
        lib().efo_odom_init_rgb(self.hnd, _p(rgba))

    def init_rgb_model(self, rgba):
        lib().efo_odom_init_rgb_model(self.hnd, _p(rgba))

    def init_first_rgb(self, rgba):
        lib().efo_odom_init_first_rgb(self.hnd, _p(rgba))

    def track(self, T_wc, rgb_only=False, icp_weight=10.0, pyramid=True, fast_odom=False, so3=True, max_trace=64):
        T = np.ascontiguousarray(T_wc, np.float64).copy()
        trace = np.zeros(max_trace, TRACE_DTYPE)
        n = lib().efo_odom_track(self.hnd, _p(T), int(rgb_only), _f(icp_weight), int(pyramid), int(fast_odom), int(so3),
                                 _p(trace), max_trace)
        return T, trace[:n]

    def stats(self):
        out = np.zeros(8, np.float32)
        lib().efo_odom_stats(self.hnd, _p(out))
        return dict(zip(["lastICPError", "lastICPCount", "lastRGBError", "lastRGBCount", "lastSO3Error", "lastSO3Count"],
                        out[:6].tolist()))

    def last_system(self):
        A = np.zeros((6, 6), np.float64)
        b = np.zeros(6, np.float64)
        lib().efo_odom_last_system(self.hnd, _p(A), _p(b))
        return A, b

    def buffer(self, name, level):
        which, dt, planes = self.BUF[name]
        r, c = self.h >> level, self.w >> level
        ptr = lib().efo_odom_buffer(self.hnd, which, level)
        n = planes * r * c
        arr = np.ctypeslib.as_array(C.cast(ptr, C.POINTER(np.ctypeslib.as_ctypes_type(dt))), shape=(n,))
        return arr.reshape(planes * r, c).copy()


# ------------------------------------------------------------------ preprocess + map stages
def bilateral(depth, max_d):
    r, c = depth.shape
    out = np.zeros((r, c), np.uint16)
    lib().efo_bilateral(_p(depth), r, c, _f(max_d), _p(out))
    return out


def metric(depth, max_d):
    r, c = depth.shape
    out = np.zeros((r, c), np.float32)
    lib().efo_metric(_p(depth), r, c, _f(max_d), _p(out))
    return out


def _cam4(K):
    return np.array([K.cx, K.cy, K.fx, K.fy], np.float32)


def feedback_buffer(rgb, depth_metric, K, time, max_depth):
    r, c = depth_metric.shape
    out = np.zeros((r * c, 12), np.float32)
    cam = _cam4(K)
    n = lib().efo_feedback_buffer(_p(rgb), _p(depth_metric), r, c, _p(cam), int(time), _f(max_depth), _p(out))
    return out[:n].copy()


def map_initialise(raw_fb, filt_fb):
    out = np.zeros((len(raw_fb), 12), np.float32)
    n = lib().efo_map_initialise(_p(np.ascontiguousarray(raw_fb)), len(raw_fb), _p(np.ascontiguousarray(filt_fb)),
                                 len(filt_fb), 0, _p(out))
    return out[:n]


def predict_indices(surfels, T_wc, time, max_depth, time_delta, K):
    r, c = K.height, K.width
    index = np.zeros((r, c), np.uint32)
    vc = np.zeros((r, c, 4), np.float32)
    ct = np.zeros((r, c, 4), np.float32)
    nr = np.zeros((r, c, 4), np.float32)
    T = np.ascontiguousarray(T_wc, np.float64)
    cam = _cam4(K)
    lib().efo_predict_indices(_p(surfels), len(surfels), _p(T), int(time), _f(max_depth), int(time_delta), r, c,
                              _p(cam), _p(index), _p(vc), _p(ct), _p(nr))
    return index, vc, ct, nr


def fuse(surfels, T_wc, time, rgb, depth_raw, depth_filt, index, vc, ct, nr, max_depth, weighting, K):
    """Returns (updated surfels, new unstable surfels)."""
    r, c = K.height, K.width
    m = np.ascontiguousarray(surfels, np.float32).copy()
    new = np.zeros((r * c, 12), np.float32)
    T = np.ascontiguousarray(T_wc, np.float64)
    cam = _cam4(K)
    n = lib().efo_fuse(_p(m), len(m), _p(T), int(time), _p(rgb), _p(depth_raw), _p(depth_filt), _p(index), _p(vc),
                       _p(ct), _p(nr), _f(max_depth), _f(weighting), r, c, _p(cam), _p(new))
    return m, new[:n].copy()


def clean(surfels, new_unstable, T_wc, time, index, vc, ct, nr, conf_threshold, time_delta, max_depth, K):
    r, c = K.height, K.width
    out = np.zeros((len(surfels) + len(new_unstable), 12), np.float32)
    T = np.ascontiguousarray(T_wc, np.float64)
    cam = _cam4(K)
    s = np.ascontiguousarray(surfels, np.float32)
    nu = np.ascontiguousarray(new_unstable, np.float32)
    n = lib().efo_clean(_p(s), len(s), _p(nu), len(nu), _p(T), int(time), _p(index), _p(vc), _p(ct), _p(nr),
                        _f(conf_threshold), int(time_delta), _f(max_depth), r, c, _p(cam), _p(out))
    return out[:n].copy()


def clean_deform(surfels, new_unstable, T_wc, time, index, vc, ct, conf_threshold, time_delta, max_depth, K, nodes, depth, is_fern=False):
    """clean with a deformation graph: nodes (n, 16) float32, depth = synthesizeDepth output."""
    r, c = K.height, K.width
    out = np.zeros((len(surfels) + len(new_unstable), 12), np.float32)
    T = np.ascontiguousarray(T_wc, np.float64)
    cam = _cam4(K)
    s = np.ascontiguousarray(surfels, np.float32)
    nu = np.ascontiguousarray(new_unstable, np.float32).reshape(-1, 12)
    nd = np.ascontiguousarray(nodes, np.float32).reshape(-1, 16)
    d = np.ascontiguousarray(depth, np.float32)
    n = lib().efo_clean_deform(_p(s), len(s), _p(nu), len(nu), _p(T), int(time), _p(index), _p(vc), _p(ct), _f(conf_threshold),
                               int(time_delta), _f(max_depth), r, c, _p(cam), _p(nd), len(nd), _p(d), int(is_fern), _p(out))
    return out[:n].copy()


def combined_predict(surfels, T_wc, max_depth, conf_threshold, time, max_time, time_delta, K, depth_only=False):
    r, c = K.height, K.width
    T = np.ascontiguousarray(T_wc, np.float64)
    cam = _cam4(K)
    s = np.ascontiguousarray(surfels, np.float32)
    if depth_only:
        d = np.zeros((r, c), np.float32)
        lib().efo_combined_predict(_p(s), len(s), _p(T), _f(max_depth), _f(conf_threshold), int(time), int(max_time),
                                   int(time_delta), r, c, _p(cam), None, None, None, None, _p(d), 1)
        return d
    image = np.zeros((r, c, 4), np.uint8)
    vertex = np.zeros((r, c, 4), np.float32)
    normal = np.zeros((r, c, 4), np.float32)
    tm = np.zeros((r, c), np.uint16)
    lib().efo_combined_predict(_p(s), len(s), _p(T), _f(max_depth), _f(conf_threshold), int(time), int(max_time),
                               int(time_delta), r, c, _p(cam), _p(image), _p(vertex), _p(normal), _p(tm), None, 0)
    return image, vertex, normal, tm


def fill_vertex(existing4, raw_depth, passthrough, K):
    out = np.zeros_like(existing4)
    cam = _cam4(K)
    lib().efo_fill_vertex(_p(existing4), _p(raw_depth), int(passthrough), K.height, K.width, _p(cam), _p(out))
    return out


def fill_normal(existing4, raw_depth, passthrough, K):
    out = np.zeros_like(existing4)
    cam = _cam4(K)
    lib().efo_fill_normal(_p(existing4), _p(raw_depth), int(passthrough), K.height, K.width, _p(cam), _p(out))
    return out


def fill_image(existing4, rgb, passthrough):
    out = np.zeros_like(existing4)
    r, c = existing4.shape[:2]
    lib().efo_fill_image(_p(existing4), _p(rgb), int(passthrough), r, c, _p(out))
    return out


def dense_enough(image4, factor=20):
    r, c = image4.shape[:2]
    return bool(lib().efo_dense_enough(_p(image4), r, c, factor))


# ------------------------------------------------------------------ pipeline
INT_MAX_HALF = 2147483647 // 2


class Fusion:
    BUFS = {"image": (0, np.uint8, 4), "vertex": (1, np.float32, 4), "normal": (2, np.float32, 4),
            "time": (3, np.uint16, 1), "fill_image": (4, np.uint8, 4), "fill_vertex": (5, np.float32, 4),
            "fill_normal": (6, np.float32, 4), "depth_filtered": (7, np.uint16, 1), "depth_metric": (8, np.float32, 1),
            "depth_metric_filtered": (9, np.float32, 1), "index": (10, np.uint32, 1), "vert_conf": (11, np.float32, 4),
            "color_time": (12, np.float32, 4), "norm_rad": (13, np.float32, 4)}

    def __init__(self, K, time_delta=INT_MAX_HALF, confidence=10.0, depth_cutoff=3.0, icp_weight=10.0, fast_odom=False,
                 so3=True, frame_to_frame_rgb=False, pyramid=True, rgb_only=False, capacity=3072 * 3072 // 4):
        self.K = K
        self.cfg = Config(K.width, K.height, K.fx, K.fy, K.cx, K.cy, time_delta, confidence, depth_cutoff, icp_weight,
                          int(fast_odom), int(so3), int(frame_to_frame_rgb), int(pyramid), int(rgb_only), capacity)
        self.hnd = C.c_void_p(lib().efo_fusion_create(C.byref(self.cfg)))

    def __del__(self):
        if getattr(self, "hnd", None):
            lib().efo_fusion_destroy(self.hnd)
            self.hnd = None

    def process_frame(self, rgb, depth, timestamp=0, weight_multiplier=1.0, T_wc=None):
        rgb = np.ascontiguousarray(rgb, np.uint8)
        depth = np.ascontiguousarray(depth, np.uint16)
        T = None if T_wc is None else np.ascontiguousarray(T_wc, np.float64)
        lib().efo_fusion_process_frame(self.hnd, _p(rgb), _p(depth), C.c_int64(timestamp), _f(weight_multiplier), _p(T))

    def process_frame_deform(self, rgb, depth, timestamp=0, weight_multiplier=1.0, T_wc=None, T_override=None, nodes=None, fern_accepted=False):
        rgb = np.ascontiguousarray(rgb, np.uint8)
        depth = np.ascontiguousarray(depth, np.uint16)
        T = None if T_wc is None else np.ascontiguousarray(T_wc, np.float64)
        To = None if T_override is None else np.ascontiguousarray(T_override, np.float64)
        nd = None if nodes is None else np.ascontiguousarray(nodes, np.float32).reshape(-1, 16)
        lib().efo_fusion_process_frame_deform(self.hnd, _p(rgb), _p(depth), C.c_int64(timestamp), _f(weight_multiplier), _p(T), _p(To),
                                              _p(nd), 0 if nd is None else len(nd), int(fern_accepted))

    def set_map(self, surfels):
        """Replaces the model by `surfels` ((n, 12) float32, cut to the capacity) and re-renders the model view (predict())."""
        s = np.ascontiguousarray(surfels, np.float32).reshape(-1, 12)
        lib().efo_fusion_set_map(self.hnd, _p(s), len(s))

    def set_loop_closure(self, enabled=True, count_thresh=35000, err_thresh=5e-05, cov_thresh=1e-05):
        lib().efo_fusion_set_loop_closure(self.hnd, int(enabled), int(count_thresh), _f(err_thresh), _f(cov_thresh))

    def loop_result(self):
        """(info dict, src (n,3), dst (n,3), times (n,)) of the last frame's local loop closure front half."""
        res = LoopResult()
        cap = (self.K.width // 20) * (self.K.height // 20)
        src = np.zeros((cap, 3), np.float64)
        dst = np.zeros((cap, 3), np.float64)
        tm = np.zeros(cap, np.int32)
        n = lib().efo_fusion_loop_result(self.hnd, C.byref(res), _p(src), _p(dst), _p(tm), cap)
        info = dict(ran=res.ran, accepted=res.accepted, n_constraints=res.n_constraints, lastICPError=res.lastICPError,
                    lastICPCount=res.lastICPCount, cov_diag=np.array(res.cov_diag[:]), T_wc_est=np.array(res.T_wc_est[:]).reshape(4, 4))
        return info, src[:n].copy(), dst[:n].copy(), tm[:n].copy()

    @property
    def pose(self):
        T = np.zeros((4, 4), np.float64)
        lib().efo_fusion_pose(self.hnd, _p(T))
        return T

    @property
    def count(self):
        return lib().efo_fusion_count(self.hnd)

    @property
    def tick(self):
        return lib().efo_fusion_tick(self.hnd)

    def map(self):
        n = self.count
        ptr = lib().efo_fusion_map(self.hnd)
        return np.ctypeslib.as_array(C.cast(ptr, C.POINTER(C.c_float)), shape=(n * 12,)).reshape(n, 12).copy()

    def odometry(self):
        return Odometry(self.K.width, self.K.height, self.K.cx, self.K.cy, self.K.fx, self.K.fy,
                        handle=lib().efo_fusion_odometry(self.hnd))

    def buffer(self, name):
        which, dt, ch = self.BUFS[name]
        ptr = lib().efo_fusion_buffer(self.hnd, which)
        n = self.K.height * self.K.width * ch
        arr = np.ctypeslib.as_array(C.cast(ptr, C.POINTER(np.ctypeslib.as_ctypes_type(dt))), shape=(n,))
        return arr.reshape((self.K.height, self.K.width, ch) if ch > 1 else (self.K.height, self.K.width)).copy()

    def timers(self):
        out = np.zeros(4, np.float64)
        lib().efo_fusion_timers(self.hnd, _p(out))
        return dict(zip(["preprocess", "tracking", "mapping", "predict"], out.tolist()))
