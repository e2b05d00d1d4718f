"""combinedPredict at cameras of the caller's choosing (ef_map_predict_view) against the reference's own splat.vert + combo_splat.frag
executed on Mesa llvmpipe: tests/golden/ref_view_*.npz (written by tests/golden/make_view_golden.py) hold, per camera, the outputs the
shaders wrote for a few poses and time windows over the map of tests/golden/ref_render_320x240.npz. The cameras differ from the one
the map was captured with (80x60, fx = fy): other intrinsics with fx != fy and an off-centre principal point, and a 16:9 size.

Here the CPU oracle (oracle/efo_map.cpp, combined_predict with the view's K) is checked against them; tests/test_gpu_model_view.py
checks the product. Both use the tolerances the splat section of tests/test_gl_golden.py applies: image and time may differ at 5e-4
of the pixels (pow(r, 2) at a disc edge), vertex and normal agree to 5e-5 / 1e-5 where image and time agree."""
import os

import numpy as np
import pytest

from elasticfusion_b200 import synth
from test_gl_golden import frac_differ, mad
from test_render_golden import look_at

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = os.path.join(HERE, "golden")
MAP_FIXTURE = os.path.join(GOLDEN, "ref_render_320x240.npz")
CAMERAS = {"320x240": synth.Intrinsics(320, 240, 300.0, 280.0, 150.5, 125.0), "256x144": synth.Intrinsics(256, 144, 200.0, 200.0, 140.0, 70.0)}
BIG = 2147483647 // 2
TICK = 4  # the map's last frame
STEP = 3  # the fixtures keep every STEP-th pixel (row-major) of each output


def fixture_path(name):
    return os.path.join(GOLDEN, f"ref_view_{name}.npz")


def load_map():
    return np.load(MAP_FIXTURE)["map"]


def views(surfels):
    """name -> dict(T, max_depth, conf_threshold, time, max_time, time_delta) of the views every camera is checked at."""
    mv = np.load(MAP_FIXTURE)["vf"][0][18:34].astype(np.float64).reshape(4, 4).T  # the fixture's capture pose, as its model-view
    T0 = np.linalg.inv(mv)
    pos = surfels[:, :3].astype(np.float64)
    thr = float(np.percentile(surfels[:, 3], 40))  # (after a few frames no surfel has reached the reference's threshold of 10)
    eye = T0[:3, 3] + 0.3 * T0[:3, 0] - 0.2 * T0[:3, 1]
    T1 = look_at(eye, pos.mean(0))
    near = float(np.median((pos - eye) @ T1[:3, 2]))
    return {
        "active": dict(T=T0, max_depth=20.0, conf_threshold=thr, time=TICK, max_time=TICK, time_delta=BIG),
        "inactive": dict(T=T0, max_depth=20.0, conf_threshold=0.5, time=0, max_time=TICK - 2, time_delta=2),
        "oblique_near": dict(T=T1, max_depth=near, conf_threshold=thr, time=TICK, max_time=TICK, time_delta=BIG),
    }


def load_fixture(name):
    z = np.load(fixture_path(name))
    assert int(z["gl_error"]) == 0 and "llvmpipe" in str(z["gl_log"])
    w, h, fx, fy, cx, cy = z["K"]
    K = synth.Intrinsics(int(w), int(h), float(fx), float(fy), float(cx), float(cy))
    out = {}
    for n in (str(x) for x in z["names"]):
        md, ct, t, mt, td = z["args_" + n]
        out[n] = dict(T=z["T_" + n], max_depth=float(md), conf_threshold=float(ct), time=int(t), max_time=int(mt), time_delta=int(td),
                      gl=tuple(z[k + "_" + n] for k in ("image", "vertex", "normal", "time")))
    return K, out


def cut(a):
    """what a fixture keeps of a full-size output: every STEP-th pixel, row-major"""
    a = np.asarray(a)
    return a.reshape(-1, *a.shape[2:])[::STEP]


def check_against(K, vs, predict, label):
    """predict(K, view dict) -> (image, vertex, normal, time) at full size, compared with the shaders' outputs of every view."""
    for n, v in vs.items():
        out = [cut(a) for a in predict(K, v)]
        ref = v["gl"]
        what = f"{label} {n}"
        assert frac_differ(out[0], ref[0]) <= 5e-4 and frac_differ(out[3], ref[3]) <= 5e-4, what
        same = (out[3] == ref[3]) & (out[0] == ref[0]).all(axis=-1)
        assert mad(out[1][same], ref[1][same]) <= 5e-5 and mad(out[2][same], ref[2][same]) <= 1e-5, what
        covered = (ref[1][:, 2] > 0).mean()
        print(f"{what}: {covered:.3f} covered, {1 - same.mean():.2e} differ")
        assert covered > 0.2, what


def oracle_predict(surfels):
    from oracle import ef_oracle as eo

    return lambda K, v: eo.combined_predict(surfels, v["T"], v["max_depth"], v["conf_threshold"], v["time"], v["max_time"], v["time_delta"], K)


@pytest.mark.parametrize("name", sorted(CAMERAS))
def test_oracle_matches_reference_view(name):
    """oracle/efo_map.cpp's combined_predict at a camera of its own == the reference's splat shaders on Mesa at that camera."""
    K, vs = load_fixture(name)
    C = CAMERAS[name]
    assert (K.width, K.height, K.fx, K.fy, K.cx, K.cy) == (C.width, C.height, C.fx, C.fy, C.cx, C.cy)
    check_against(K, vs, oracle_predict(load_map()), "oracle " + name)


def test_fixture_views_are_the_generators():
    """The fixtures hold the views views() defines (a changed generator needs new fixtures)."""
    surfels = load_map()
    for name in CAMERAS:
        _, vs = load_fixture(name)
        want = views(surfels)
        assert sorted(vs) == sorted(want)
        for n, v in want.items():
            assert np.array_equal(vs[n]["T"], v["T"]) and vs[n]["max_depth"] == np.float64(v["max_depth"]), (name, n)
