"""close_loops = 2 without a GPU: argument checks of the C ABI, the result struct's layout as C and ctypes see it, and the C++
drop-in's deviceLoopClosure constructor parameter."""
import ctypes
import os
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EF_EINVAL = -1


def test_create_rejects_unknown_close_loops_modes():
    from elasticfusion_b200 import capi

    lib = capi.lib()
    out = ctypes.c_void_p()
    for v in (3, -1, 100):
        cfg = capi.default_config(320, 240, 264.0, 264.0, 160.0, 120.0, close_loops=v)
        assert lib.ef_create(ctypes.byref(cfg), None, ctypes.byref(out)) == EF_EINVAL, v
        assert not out.value


def test_local_deform_result_validates_its_arguments():
    from elasticfusion_b200 import capi

    lib = capi.lib()
    res = capi.EfLocalDeform()
    n = ctypes.c_int32()
    assert lib.ef_local_deform_result(None, ctypes.byref(res), None, 0, ctypes.byref(n)) == EF_EINVAL
    assert "ef_local_deform_result" in open(os.path.join(ROOT, "include", "efusion_b200.h")).read()
    assert hasattr(lib, "ef_local_deform_result")


def test_local_deform_struct_layout_matches_ctypes(tmp_path):
    """EfLocalDeform as a C compiler lays it out equals the ctypes mirror in capi.py; EfLoopResult / EfDeformResult keep theirs."""
    from elasticfusion_b200 import capi

    src = tmp_path / "layout.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "efusion_b200.h"\n'
                   "int main(void) {\n"
                   '  printf("%zu %zu %zu %zu %zu %zu %zu %zu %zu\\n", sizeof(EfLocalDeform), offsetof(EfLocalDeform, applied),\n'
                   "         offsetof(EfLocalDeform, result), offsetof(EfLocalDeform, deforms), offsetof(EfLocalDeform, last_deform_time),\n"
                   "         offsetof(EfLocalDeform, n_nodes), sizeof(EfDeformResult), sizeof(EfLoopResult), offsetof(EfLoopResult, T_wc_est));\n"
                   "  return 0;\n}\n")
    exe = tmp_path / "layout"
    subprocess.check_call(["/usr/bin/gcc", "-std=c99", "-Wall", "-Werror", f"-I{ROOT}/include", str(src), "-o", str(exe)])
    got = [int(x) for x in subprocess.check_output([str(exe)], text=True).split()]
    L, D, R = capi.EfLocalDeform, capi.EfDeformResult, capi.EfLoopResult
    assert got == [ctypes.sizeof(L), L.applied.offset, L.result.offset, L.deforms.offset, L.last_deform_time.offset, L.n_nodes.offset,
                   ctypes.sizeof(D), ctypes.sizeof(R), R.T_wc_est.offset]
    assert got[6] == 32 and got[7] == 200 and got[8] == 72


def test_dropin_device_loop_closure_compiles(tmp_path):
    """ElasticFusion(..., closeLoops, ..., device, deviceLoopClosure) and getDeforms() compile against include/efusion/."""
    src = tmp_path / "dlc.cpp"
    src.write_text("#include <ElasticFusion.h>\n"
                   "int main() {\n"
                   "  Resolution::getInstance(320, 240);\n"
                   "  Intrinsics::getInstance(264, 264, 160, 120);\n"
                   '  ElasticFusion e(12, 3000, 5e-05f, 1e-4f, true, false, false, 115, 10, 3, 10, false, 0.3095f, true, false, "", 400000, 0, true);\n'
                   "  return e.getDeforms();\n}\n")
    so = os.path.join(ROOT, "elasticfusion_b200", "libefusion.so")
    if not os.path.exists(so):
        subprocess.check_call(["bash", os.path.join(ROOT, "build.sh")])
    subprocess.check_call(["/usr/bin/g++", "-std=c++17", "-O1", "-Wall", "-Werror", f"-I{ROOT}/include/efusion", f"-I{ROOT}/include", str(src),
                           "-o", str(tmp_path / "dlc"), f"-L{ROOT}/elasticfusion_b200", "-lefusion", "-L/usr/local/cuda/lib64", "-lcudart"])
