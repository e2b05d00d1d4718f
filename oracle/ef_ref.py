"""TEST INFRASTRUCTURE ONLY — ctypes binding for oracle/_ref/libef_ref.so: the REFERENCE's own CUDA tracking kernels
(Core/Cuda/reduce.cu, cudafuncs.cu compiled unmodified from the reference tree) behind oracle/ref_harness.cu.
Needs a GPU. Used to pin the CPU oracle and as the timed tracking baseline (bench.py --impl reference)."""
from __future__ import annotations

import ctypes as C
import os

import numpy as np

from . import ef_oracle as eo

_HERE = os.path.dirname(os.path.abspath(__file__))
SO = os.path.join(_HERE, "_ref", "libef_ref.so")
_LIB = None


def available() -> bool:
    if not os.path.exists(SO):
        return False
    try:
        import torch

        return torch.cuda.is_available()
    except Exception:
        return False


def lib():
    global _LIB
    if _LIB is None:
        _LIB = C.CDLL(SO)
        _LIB.efr_create.restype = C.c_void_p
        _LIB.efr_time_icp_step.restype = C.c_double
    return _LIB


def _p(a):
    assert a.flags["C_CONTIGUOUS"]
    return a.ctypes.data_as(C.c_void_p)


def _f(x):
    return C.c_float(float(x))


_BUF = {"vmap_curr": (0, np.float32, 3), "nmap_curr": (1, np.float32, 3), "vmap_g_prev": (2, np.float32, 3),
        "nmap_g_prev": (3, np.float32, 3), "lastDepth": (4, np.float32, 1), "nextDepth": (5, np.float32, 1),
        "lastImage": (6, np.uint8, 1), "nextImage": (7, np.uint8, 1), "lastNextImage": (8, np.uint8, 1),
        "dIdx": (9, np.int16, 1), "dIdy": (10, np.int16, 1), "depth_tmp": (11, np.uint16, 1),
        "corres": (12, eo.DATATERM_DTYPE, 1)}


class RefOdometry:
    def __init__(self, K):
        self.K = K
        self.h = C.c_void_p(lib().efr_create(K.width, K.height, _f(K.cx), _f(K.cy), _f(K.fx), _f(K.fy)))

    def __del__(self):
        if getattr(self, "h", None):
            lib().efr_destroy(self.h)
            self.h = None

    def init_icp_depth(self, depth, cutoff):
        lib().efr_init_icp_depth(self.h, _p(depth), _f(cutoff))

    def init_icp_pred(self, v4, n4):
        lib().efr_init_icp_pred(self.h, _p(v4), _p(n4))

    def init_icp_model(self, v4, n4, T):
        T = np.ascontiguousarray(T, np.float64)
        lib().efr_init_icp_model(self.h, _p(v4), _p(n4), _p(T))

    def init_rgb(self, rgba):
        lib().efr_init_rgb(self.h, _p(rgba))

    def init_rgb_model(self, rgba):
        lib().efr_init_rgb_model(self.h, _p(rgba))

    def init_first_rgb(self, rgba):
        lib().efr_init_first_rgb(self.h, _p(rgba))

    def track(self, T_wc, rgb_only=False, icp_weight=10.0, pyramid=True, fast_odom=False, so3=True, max_trace=64):
        T = np.ascontiguousarray(T_wc, np.float64).copy()
        trace = np.zeros(max_trace, eo.TRACE_DTYPE)
        n = lib().efr_track(self.h, _p(T), int(rgb_only), _f(icp_weight), int(pyramid), int(fast_odom), int(so3), _p(trace), max_trace)
        return T, trace[:n]

    def buffer(self, name, level):
        which, dt, planes = _BUF[name]
        r, c = self.K.height >> level, self.K.width >> level
        out = np.zeros((planes * r, c), dt)
        lib().efr_download(self.h, which, level, _p(out))
        return out

    def icp_step(self, level, Rcurr, tcurr, Rprev_inv, tprev):
        f32 = lambda a: np.ascontiguousarray(a, np.float32)
        A, b, res = np.zeros((6, 6), np.float32), np.zeros(6, np.float32), np.zeros(2, np.float32)
        a0, a1, a2, a3 = f32(Rcurr), f32(tcurr), f32(Rprev_inv), f32(tprev)
        lib().efr_icp_step(self.h, level, _p(a0), _p(a1), _p(a2), _p(a3), _p(A), _p(b), _p(res))
        return A, b, res

    def time_icp_step(self, level, Rcurr, tcurr, Rprev_inv, tprev, reps=50):
        f32 = lambda a: np.ascontiguousarray(a, np.float32)
        a0, a1, a2, a3 = f32(Rcurr), f32(tcurr), f32(Rprev_inv), f32(tprev)
        return lib().efr_time_icp_step(self.h, level, _p(a0), _p(a1), _p(a2), _p(a3), reps)

    def rgb_residual(self, level, krkinv, kt):
        kk, k3 = np.ascontiguousarray(krkinv, np.float32), np.ascontiguousarray(kt, np.float32)
        sigma, count = C.c_int(), C.c_int()
        lib().efr_rgb_residual(self.h, level, _p(kk), _p(k3), C.byref(sigma), C.byref(count))
        return sigma.value, count.value

    def rgb_step(self, level, sigma):
        A, b = np.zeros((6, 6), np.float32), np.zeros(6, np.float32)
        lib().efr_rgb_step(self.h, level, _f(sigma), _p(A), _p(b))
        return A, b

    def so3_step(self, image_basis, kinv, krlr):
        f32 = lambda a: np.ascontiguousarray(a, np.float32)
        A, b, res = np.zeros((3, 3), np.float32), np.zeros(3, np.float32), np.zeros(2, np.float32)
        a0, a1, a2 = f32(image_basis), f32(kinv), f32(krlr)
        lib().efr_so3_step(self.h, _p(a0), _p(a1), _p(a2), _p(A), _p(b), _p(res))
        return A, b, res

    def timers(self):
        out = np.zeros(2, np.float64)
        lib().efr_timers(self.h, _p(out))
        return {"ref_init_s": out[0], "ref_track_s": out[1]}


class TrackerBackend(C.Structure):
    _fields_ = [("handle", C.c_void_p), ("init_icp_model", C.c_void_p), ("init_rgb_model", C.c_void_p), ("init_icp_depth", C.c_void_p),
                ("init_rgb", C.c_void_p), ("init_first_rgb", C.c_void_p), ("track", C.c_void_p)]


class HybridFusion(eo.Fusion):
    """The reference arm: the CPU-oracle pipeline with its tracker replaced by the reference's CUDA kernels."""

    def __init__(self, K, **kw):
        super().__init__(K, **kw)
        self.ref = RefOdometry(K)
        fn = lambda name: C.cast(getattr(lib(), name), C.c_void_p)
        self.backend = TrackerBackend(self.ref.h, fn("efr_init_icp_model"), fn("efr_init_rgb_model"), fn("efr_init_icp_depth"),
                                      fn("efr_init_rgb"), fn("efr_init_first_rgb"), fn("efr_track"))
        eo.lib().efo_fusion_set_tracker(self.hnd, C.byref(self.backend))

    def timers(self):
        t = super().timers()
        t.update(self.ref.timers())
        return t
