"""TEST INFRASTRUCTURE ONLY — ctypes binding of the CPU oracle of the global-surface render (oracle/efo_render.cpp ->
oracle/libef_render_oracle.so, compiled on first use with the flags of the other oracle sources; into a temporary directory when
the tree is read-only). The product package never imports this module."""
from __future__ import annotations

import ctypes as C
import os
import subprocess
import tempfile

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
SO = os.path.join(_HERE, "libef_render_oracle.so")
_SRCS = [os.path.join(_HERE, f) for f in ("efo_render.cpp", "efo_common.h")]
CXXFLAGS = ["-O2", "-std=c++17", "-fPIC", "-fopenmp", "-ffp-contract=off", "-fno-fast-math", "-Wall", "-Wno-unknown-pragmas"]
_LIB = None


def build(force: bool = False) -> str:
    so = SO if os.access(_HERE, os.W_OK) else os.path.join(tempfile.gettempdir(), f"libef_render_oracle.{os.getuid()}.so")
    stale = (not os.path.exists(so)) or any(os.path.getmtime(s) > os.path.getmtime(so) for s in _SRCS)
    if force or stale:
        tmp = so + f".{os.getpid()}.tmp"
        subprocess.check_call(["/usr/bin/g++", *CXXFLAGS, "-shared", "-o", tmp, _SRCS[0]])
        os.replace(tmp, so)
    return so


def lib():
    global _LIB
    if _LIB is None:
        _LIB = C.CDLL(build())
    return _LIB


def _p(a):
    assert a.flags["C_CONTIGUOUS"], "array must be C contiguous"
    return a.ctypes.data_as(C.c_void_p)


class RenderView(C.Structure):
    """EfoRenderView: the layout of EfRenderView (include/efusion_b200.h)."""
    _fields_ = [("width", C.c_int32), ("height", C.c_int32), ("mvp", C.c_float * 16), ("mv", C.c_float * 16), ("threshold", C.c_float),
                ("color_type", C.c_int32), ("unstable", C.c_int32), ("draw_window", C.c_int32), ("time", C.c_int32),
                ("time_delta", C.c_int32), ("phong", C.c_int32), ("sign_mult", C.c_float)]


def _view(v):
    out = RenderView()
    for k, t in RenderView._fields_:
        val = getattr(v, k)
        setattr(out, k, t(*val[:]) if k in ("mvp", "mv") else val)
    return out


def render(surfels, view, keys=False):
    """draw_global_surface.{vert,geom,frag} (phong = 0) or _phong.frag (phong = 1) of surfels (n,12) for a view with EfRenderView's
    fields: (H, W, 4) uint8, row 0 = window y 0; with keys=True also the winning (d24 << 32 | id) key per pixel (~0: none)."""
    v = _view(view)
    s = np.ascontiguousarray(surfels, np.float32).reshape(-1, 12)
    rgba = np.zeros((v.height, v.width, 4), np.uint8)
    k = np.zeros((v.height, v.width), np.uint64)
    lib().efo_render(_p(s), len(s), C.byref(v), _p(rgba), _p(k))
    return (rgba, k) if keys else rgba


def render_margins(surfels, view, keys, slack=0.05):
    """Per pixel, over the fragments of every surfel: (rim, edge, runner) -- the least |dot(tc,tc) - 1|, the least distance to the
    strip's diagonal, the quad's border or the near / far plane, and the least key of a surfel other than the winner's."""
    v = _view(view)
    s = np.ascontiguousarray(surfels, np.float32).reshape(-1, 12)
    rim, edge = np.zeros((v.height, v.width), np.float32), np.zeros((v.height, v.width), np.float32)
    runner = np.zeros((v.height, v.width), np.uint64)
    lib().efo_render_margins(_p(s), len(s), C.byref(v), _p(np.ascontiguousarray(keys, np.uint64)), C.c_float(slack), _p(rim), _p(edge),
                             _p(runner))
    return rim, edge, runner
