"""ef_track_view without a GPU: the layouts of EfTrackView / EfTrackResult as a C compiler and the ctypes mirror in capi.py see them,
the argument checks that need no device, and the Python view helper."""
import ctypes
import os
import subprocess

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EF_EINVAL = -1


def test_track_view_struct_layout_matches_ctypes(tmp_path):
    from elasticfusion_b200 import capi

    src = tmp_path / "layout.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "efusion_b200.h"\n'
                   "int main(void) {\n"
                   '  printf("%zu %zu %zu %zu %zu %zu %zu %zu %zu %zu %zu %zu\\n", sizeof(EfTrackView), offsetof(EfTrackView, depth_cutoff),\n'
                   "         offsetof(EfTrackView, icp_weight), offsetof(EfTrackView, rgb_only), offsetof(EfTrackView, pyramid),\n"
                   "         offsetof(EfTrackView, fast_odom), sizeof(EfTrackResult), offsetof(EfTrackResult, stats),\n"
                   "         offsetof(EfTrackResult, covariance), offsetof(EfTrackResult, dense_enough), sizeof(EfOdomStats),\n"
                   "         offsetof(EfOdomStats, lastA));\n"
                   "  return 0;\n}\n")
    exe = tmp_path / "layout"
    subprocess.check_call(["/usr/bin/gcc", "-std=c99", "-Wall", "-Werror", f"-I{ROOT}/include", str(src), "-o", str(exe)])
    got = [int(x) for x in subprocess.check_output([str(exe)], text=True).split()]
    V, R, S = capi.EfTrackView, capi.EfTrackResult, capi.EfOdomStats
    assert got == [ctypes.sizeof(V), V.depth_cutoff.offset, V.icp_weight.offset, V.rgb_only.offset, V.pyramid.offset, V.fast_odom.offset,
                   ctypes.sizeof(R), R.stats.offset, R.covariance.offset, R.dense_enough.offset, ctypes.sizeof(S), S.lastA.offset]
    assert ctypes.sizeof(S) == capi.STATS_DTYPE.itemsize and S.lastA.offset == capi.STATS_DTYPE.fields["lastA"][1]


def test_track_view_rejects_null_context():
    from elasticfusion_b200 import capi

    lib = capi.lib()
    v = capi.track_view(np.eye(4), 300.0, 300.0, 212.0, 120.0, 424, 240, 5)
    res = capi.EfTrackResult()
    rgb = np.zeros((240, 424, 3), np.uint8)
    depth = np.zeros((240, 424), np.uint16)
    assert lib.ef_track_view(None, ctypes.byref(v), capi._p(rgb), capi._p(depth), ctypes.byref(res), None, 0, None) == EF_EINVAL
    assert lib.ef_track_view_device(None, ctypes.byref(v), None, None, None) == EF_EINVAL


def test_track_view_helper_and_result_unpacking():
    from elasticfusion_b200 import capi

    T = np.eye(4)
    T[:3, 3] = (0.1, -0.2, 0.3)
    v = capi.track_view(T, 300.0, 310.0, 200.0, 120.5, 424, 240, 7, time_delta=50, icp_weight=100.0, rgb_only=True, fast_odom=True)
    m = v.model
    assert (m.width, m.height, m.time, m.max_time, m.time_delta) == (424, 240, 7, 7, 50)
    assert (m.max_depth, m.conf_threshold, v.depth_cutoff, v.icp_weight) == (20.0, 10.0, 3.0, 100.0)
    assert (v.rgb_only, v.pyramid, v.fast_odom) == (1, 1, 1)
    assert np.array_equal(np.array(m.T_wc[:]).reshape(4, 4), T)
    assert capi.track_view(T, 1, 1, 0, 0, 32, 32, 9, max_time=3).model.max_time == 3
    r = capi.EfTrackResult()
    r.T_wc[:] = T.reshape(16).tolist()
    r.stats.lastICPCount = 12.0
    r.stats.lastA[7] = 2.5
    r.covariance[35] = 4.0
    r.dense_enough = 1
    for src in (r, bytes(r)):
        Tu, st, cov, dense = capi.unpack_track_result(src)
        assert np.array_equal(Tu, T) and st["lastICPCount"] == 12.0 and st["lastA"][7] == 2.5 and cov[5, 5] == 4.0 and dense
