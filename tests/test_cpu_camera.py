"""ef_camera_* without a GPU: the layouts of EfCameraConfig / EfCameraFrame / EfCameraResult as a C compiler and the ctypes mirror in
capi.py see them, the argument checks that need no device, and the Python helpers."""
import ctypes
import os
import subprocess

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EF_EINVAL = -1


def test_camera_struct_layout_matches_ctypes(tmp_path):
    from elasticfusion_b200 import capi

    fields = {"EfCameraConfig": [f for f, _ in capi.EfCameraConfig._fields_], "EfCameraFrame": [f for f, _ in capi.EfCameraFrame._fields_],
              "EfCameraResult": [f for f, _ in capi.EfCameraResult._fields_]}
    exprs = []
    for s, names in fields.items():
        exprs.append(f"sizeof({s})")
        exprs += [f"offsetof({s}, {n})" for n in names]
    exprs.append("EF_MAX_CAMERAS")
    src = tmp_path / "layout.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "efusion_b200.h"\nint main(void) {\n' +
                   "".join(f'  printf("%zu\\n", (size_t)({e}));\n' for e in exprs) + "  return 0;\n}\n")
    exe = tmp_path / "layout"
    subprocess.check_call(["/usr/bin/gcc", "-std=c99", "-Wall", "-Werror", f"-I{ROOT}/include", str(src), "-o", str(exe)])
    got = [int(x) for x in subprocess.check_output([str(exe)], text=True).split()]
    want = []
    for s, names in fields.items():
        T = getattr(capi, s)
        want.append(ctypes.sizeof(T))
        want += [getattr(T, n).offset for n in names]
    want.append(capi.MAX_CAMERAS)
    assert got == want


def test_camera_calls_reject_null_arguments():
    from elasticfusion_b200 import capi

    lib, C = capi.lib(), ctypes
    cfg = capi.camera_config(424, 240, 300.0, 300.0, 212.0, 120.0)
    cam = C.c_void_p()
    assert lib.ef_camera_create(None, C.byref(cfg), C.byref(cam)) == EF_EINVAL
    assert lib.ef_camera_destroy(None, None) == EF_EINVAL
    f = capi.camera_frame(3, T_wc=np.eye(4))
    res = capi.EfCameraResult()
    rgb = np.zeros((240, 424, 3), np.uint8)
    depth = np.zeros((240, 424), np.uint16)
    assert lib.ef_camera_frame(None, None, C.byref(f), capi._p(rgb), capi._p(depth), C.byref(res), None, 0, None) == EF_EINVAL
    assert lib.ef_camera_frame_device(None, None, C.byref(f), None, None, None) == EF_EINVAL
    ptr, n = C.c_void_p(), C.c_size_t()
    assert lib.ef_camera_buffer(None, None, capi.BUF["IMAGE"], 0, C.byref(ptr), C.byref(n)) == EF_EINVAL


def test_camera_helpers_and_result_unpacking():
    from elasticfusion_b200 import capi

    c = capi.camera_config(330, 246, 290.0, 280.0, 161.5, 125.0, time_delta=50, icp_weight=100.0, rgb_only=True, so3=False,
                           frame_to_frame_rgb=True)
    assert (c.width, c.height, c.time_delta, c.icp_weight) == (330, 246, 50, 100.0)
    assert (c.depth_cutoff, c.max_depth, c.conf_threshold) == (3.0, 20.0, 10.0)
    assert (c.rgb_only, c.pyramid, c.fast_odom, c.so3, c.frame_to_frame_rgb) == (1, 1, 0, 0, 1)
    T = np.eye(4)
    T[:3, 3] = (0.1, -0.2, 0.3)
    f = capi.camera_frame(7, 0.5, T, fuse=False)
    assert (f.time, f.weight_multiplier, f.has_pose, f.fuse) == (7, 0.5, 1, 0)
    assert np.array_equal(np.array(f.T_wc[:]).reshape(4, 4), T)
    g = capi.camera_frame(8)
    assert (g.has_pose, g.fuse) == (0, 1)
    r = capi.EfCameraResult()
    r.T_wc[:] = T.reshape(16).tolist()
    r.stats.lastRGBCount = 9.0
    r.covariance[7] = 3.0
    r.tracked, r.dense_enough, r.weighting = 1, 0, 0.75
    for src in (r, bytes(r)):
        Tu, st, cov, info = capi.unpack_camera_result(src)
        assert np.array_equal(Tu, T) and st["lastRGBCount"] == 9.0 and cov[1, 1] == 3.0
        assert info == dict(tracked=True, dense_enough=False, weighting=0.75)
