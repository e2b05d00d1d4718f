"""ef_camera_* with close_loops without a GPU: the config field's default and keyword, and the argument checks of
ef_camera_deform_result that need no device (the field's offset is checked by test_cpu_camera's layout test)."""
import ctypes

import numpy as np

EF_EINVAL = -1


def test_camera_config_close_loops_default_and_keyword():
    from elasticfusion_b200 import capi

    assert capi.camera_config(424, 240, 300.0, 300.0, 212.0, 120.0).close_loops == 0
    assert capi.camera_config(424, 240, 300.0, 300.0, 212.0, 120.0, close_loops=True).close_loops == 1
    assert capi.EfCameraConfig().close_loops == 0  # a zero-initialised struct: open loop
    assert [f for f, _ in capi.EfCameraConfig._fields_][-1] == "close_loops"


def test_camera_deform_result_rejects_null_and_foreign_handles():
    from elasticfusion_b200 import capi

    lib, C = capi.lib(), ctypes
    out = capi.EfLocalDeform()
    nodes = np.zeros((4, 4), np.float32)
    n = C.c_int32()
    assert lib.ef_camera_deform_result(None, None, C.byref(out), capi._p(nodes), 4, C.byref(n)) == EF_EINVAL
    assert lib.ef_camera_deform_result(None, None, None, None, 0, None) == EF_EINVAL
    assert lib.ef_camera_deform_result(None, None, C.byref(out), None, 0, None) == EF_EINVAL
