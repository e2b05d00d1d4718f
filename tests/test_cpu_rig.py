"""ef_rig_* without a GPU: the layouts of EfRigConfig / EfRigFrame / EfRigResult as a C compiler and the ctypes mirror in capi.py see
them, the argument checks that need no device, and the Python helpers."""
import ctypes
import os
import subprocess

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EF_EINVAL = -1


def test_rig_struct_layout_matches_ctypes(tmp_path):
    from elasticfusion_b200 import capi

    fields = {s: [f for f, _ in getattr(capi, s)._fields_] for s in ("EfRigConfig", "EfRigFrame", "EfRigResult")}
    exprs = []
    for s, names in fields.items():
        exprs.append(f"sizeof({s})")
        exprs += [f"offsetof({s}, {n})" for n in names]
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
    assert got == want


def test_rig_calls_reject_null_arguments():
    from elasticfusion_b200 import capi

    lib, C = capi.lib(), ctypes
    cfg = capi.EfRigConfig()
    cfg.n = 1
    cfg.T_0i[0][:] = np.eye(4).reshape(16).tolist()
    rig = C.c_void_p()
    assert lib.ef_rig_create(None, C.byref(cfg), C.byref(rig)) == EF_EINVAL
    assert lib.ef_rig_destroy(None, None) == EF_EINVAL
    f = capi.rig_frame(3, T_wc=np.eye(4))
    rgb = np.zeros((240, 424, 3), np.uint8)
    depth = np.zeros((240, 424), np.uint16)
    rgbs, depths = (C.c_void_p * 1)(rgb.ctypes.data), (C.c_void_p * 1)(depth.ctypes.data)
    members, out = (capi.EfCameraResult * 1)(), capi.EfRigResult()
    assert lib.ef_rig_frame(None, None, C.byref(f), rgbs, depths, members, C.byref(out), None, 0, None) == EF_EINVAL
    assert lib.ef_rig_frame_device(None, None, C.byref(f), rgbs, depths, None, None) == EF_EINVAL


def test_rig_helpers_and_result_unpacking():
    from elasticfusion_b200 import capi

    T = np.eye(4)
    T[:3, 3] = (0.1, -0.2, 0.3)
    f = capi.rig_frame(7, 0.5, T, fuse=False)
    assert (f.time, f.weight_multiplier, f.has_pose, f.fuse) == (7, 0.5, 1, 0)
    assert np.array_equal(np.array(f.T_wc[:]).reshape(4, 4), T)
    g = capi.rig_frame(8)
    assert (g.has_pose, g.fuse) == (0, 1)
    r = capi.EfRigResult()
    r.T_wc[:] = T.reshape(16).tolist()
    r.lastA[7] = 2.0
    r.lastb[5] = -1.0
    r.covariance[14] = 3.0
    r.tracked = 1
    for src in (r, bytes(r)):
        Tu, A, b, cov, tracked = capi.unpack_rig_result(src)
        assert np.array_equal(Tu, T) and A[1, 1] == 2.0 and b[5] == -1.0 and cov[2, 2] == 3.0 and tracked
