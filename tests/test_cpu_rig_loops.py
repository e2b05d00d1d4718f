"""ef_rig_loop_result / ef_rig_deform_result without a GPU: the layout of EfRigLoopResult as a C compiler and the ctypes mirror in
capi.py see it, and the argument checks that need no device."""
import ctypes
import os
import subprocess

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EF_EINVAL = -1


def test_rig_loop_result_layout_matches_ctypes(tmp_path):
    from elasticfusion_b200 import capi

    names = [f for f, _ in capi.EfRigLoopResult._fields_]
    exprs = ["sizeof(EfRigLoopResult)"] + [f"offsetof(EfRigLoopResult, {n})" for n in names]
    src = tmp_path / "layout.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "efusion_b200.h"\nint main(void) {\n' +
                   "".join(f'  printf("%zu\\n", (size_t)({e}));\n' for e in exprs) + "  return 0;\n}\n")
    exe = tmp_path / "layout"
    subprocess.check_call(["/usr/bin/gcc", "-std=c99", "-Wall", "-Werror", f"-I{ROOT}/include", str(src), "-o", str(exe)])
    got = [int(x) for x in subprocess.check_output([str(exe)], text=True).split()]
    T = capi.EfRigLoopResult
    assert got == [ctypes.sizeof(T)] + [getattr(T, n).offset for n in names]


def test_rig_loop_calls_reject_null_arguments():
    from elasticfusion_b200 import capi

    lib, C = capi.lib(), ctypes
    lr, ld, n = capi.EfRigLoopResult(), capi.EfLocalDeform(), C.c_int32()
    src = np.zeros((4, 3), np.float64)
    nodes = np.zeros((4, 4), np.float32)
    assert lib.ef_rig_loop_result(None, None, C.byref(lr), capi._p(src), capi._p(src), None, 4, C.byref(n)) == EF_EINVAL
    assert lib.ef_rig_loop_result(None, None, None, None, None, None, 0, None) == EF_EINVAL
    assert lib.ef_rig_deform_result(None, None, C.byref(ld), capi._p(nodes), 4, C.byref(n)) == EF_EINVAL
    assert lib.ef_rig_deform_result(None, None, None, None, 0, None) == EF_EINVAL
