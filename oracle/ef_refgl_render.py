"""TEST INFRASTRUCTURE ONLY — ctypes binding of oracle/gl/ref_gl_render.cpp: the REFERENCE's global-surface shaders
(draw_global_surface.{vert,geom,frag}, draw_global_surface_phong.frag) executed unmodified on Mesa llvmpipe, in the GL context of
oracle/ef_refgl.RefGL. Compiled on first use into oracle/_ref/gl/libef_refgl_render.so; like ef_refgl, it needs Mesa, the reference
tree and an interpreter started through ef_refgl.env()."""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

from oracle import ef_refgl as rg

_SRC = os.path.join(os.path.dirname(os.path.abspath(__file__)), "gl", "ref_gl_render.cpp")
SO = os.path.join(rg.GL_DIR, "libef_refgl_render.so")
_LIB = None


def build(force: bool = False) -> str:
    deps = [_SRC, os.path.join(os.path.dirname(_SRC), "ref_gl.h")]
    if force or not os.path.exists(SO) or any(os.path.getmtime(d) > os.path.getmtime(SO) for d in deps):
        os.makedirs(rg.GL_DIR, exist_ok=True)
        subprocess.check_call(["/usr/bin/g++", "-O1", "-std=c++17", "-fPIC", "-shared", "-o", SO, _SRC, "-ldl"])
    return SO


def available() -> bool:
    return rg.available() and os.path.exists(_SRC)


def render(gl: rg.RefGL, surfels, view):
    """GlobalModel::renderPointCloud / drawFXAA's colour pass for a view with EfRenderView's fields, in the context of `gl`:
    (H, W, 4) uint8 as glReadPixels returns it (row 0 = window y 0)."""
    global _LIB
    if _LIB is None:
        _LIB = C.CDLL(build())
        _LIB.efgr_log.restype = C.c_char_p
    p = lambda a: a.ctypes.data_as(C.c_void_p)
    f = lambda x: C.c_float(float(x))
    s = np.ascontiguousarray(surfels, np.float32).reshape(-1, 12)
    out = np.zeros((view.height, view.width, 4), np.uint8)
    mvp = np.ascontiguousarray(np.array(view.mvp[:], np.float32))
    mv = np.ascontiguousarray(np.array(view.mv[:], np.float32))
    rc = _LIB.efgr_render((rg.mesa_dir() + "/libGL.so.1").encode(), rg.SHADERS.encode(), p(s), len(s), int(view.width), int(view.height),
                          p(mvp), p(mv), f(view.threshold), int(view.color_type), int(view.unstable), int(view.draw_window), int(view.time),
                          int(view.time_delta), int(view.phong), f(view.sign_mult), p(out))
    if rc:
        raise RuntimeError(f"efgr_render failed ({rc}):\n" + _LIB.efgr_log().decode() + gl.log())
    return out
