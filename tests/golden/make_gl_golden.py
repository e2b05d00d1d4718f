"""Generates tests/golden/ref_mapping_160x120.npz: the outputs of every GLSL pass of the reference's mapping half, produced by
the REFERENCE's OWN SHADER FILES (Core/Shaders of the reference tree, unmodified) executed on Mesa llvmpipe through
oracle/gl/ref_gl_harness.cpp (`make -C oracle refgl`, which needs the reference tree):  python tests/golden/make_gl_golden.py

The chain of inputs is the one a frame goes through (the stage outputs of the CPU oracle feed the next stage on both sides, so
every pass is compared on identical inputs; tests/test_gl_golden.py:oracle_inputs recomputes them); `gl_*` arrays are what the
reference's shaders computed, the large ones cut to a regular sample (test_gl_golden.shrink)."""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from oracle import ef_refgl as rg  # noqa: E402

if not rg.in_gl_process():
    if not rg.available():
        raise SystemExit("oracle/_ref/gl is not built (make -C oracle refgl) or Mesa / the reference tree is absent")
    rg.run_script(os.path.abspath(__file__), *sys.argv[1:])
    raise SystemExit(0)

from elasticfusion_b200 import synth  # noqa: E402
from oracle import ef_oracle as eo  # noqa: E402
import test_gl_golden as tg  # noqa: E402

MAXD, BIG = 20.0, 2 ** 30


CONFIGS = {
    "default": dict(K=(160, 120, 132.0, 132.0, 80.0, 60.0), seed=7, speed=1.0),
    # the ICL-NUIM camera (fx != fy, half-pixel principal point; SURVEY 8d S1) at a quarter and at half of its resolution, and an
    # off-centre camera with another aspect ratio
    "icl": dict(K=(160, 120, 481.2 / 4, 480.0 / 4, 319.5 / 4, 239.5 / 4), seed=11, speed=1.0),
    "offcentre": dict(K=(192, 144, 150.0, 155.0, 90.3, 70.7), seed=23, speed=2.0),
    "icl320": dict(K=(320, 240, 481.2 / 2, 480.0 / 2, 319.5 / 2, 239.5 / 2), seed=5, speed=1.5),
}


def build(config="default"):
    """The reference shaders' outputs of every pass for one configuration, and the inputs they were given (a dict of arrays)."""
    cfg = CONFIGS[config]
    K = synth.Intrinsics(int(cfg["K"][0]), int(cfg["K"][1]), *[float(x) for x in cfg["K"][2:]])
    g = tg.oracle_inputs(K, cfg["seed"], cfg["speed"])
    gl = rg.RefGL(K)
    out = {"K": np.array([K.width, K.height, K.fx, K.fy, K.cx, K.cy], np.float64), "seed": np.array(cfg["seed"]), "speed": np.array(cfg["speed"]),
           "gl_log": np.array(gl.log())}
    T, tick, tick_t, td = g["T"], int(g["tick"]), int(g["tick_t"]), int(g["td"])
    # ---- frame 0: preprocess + first-frame map
    out.update(gl_bilateral=gl.bilateral(g["depth0"], 3.0), gl_metric=gl.metric(g["depth0"], 3.0))
    raw = gl.feedback_buffer(g["rgb0"], eo.metric(g["depth0"], 3.0), 1, MAXD)
    fil = gl.feedback_buffer(g["rgb0"], eo.metric(g["filt0"], 3.0), 1, MAXD)
    out.update(gl_initial_map=gl.map_initialise(raw, fil))
    rawb = gl.feedback_buffer(g["rgbb"], eo.metric(g["depthb"], 3.0), 1, MAXD)
    filb = gl.feedback_buffer(g["rgbb"], eo.metric(g["filtb"], 3.0), 1, MAXD)
    out.update(gl_boundary_raw_count=np.array(len(rawb)), gl_boundary_filt_count=np.array(len(filb)), gl_boundary_map=gl.map_initialise(rawb, filb))
    # ---- the map after 4 frames, frame 4 as the measurement
    m = g["map"]
    ig = gl.predict_indices(m, T, tick, MAXD, BIG)
    out.update(gl_index=ig[0], gl_vert_conf=ig[1], gl_color_time=ig[2], gl_norm_rad=ig[3])
    io = (g["index_in"], g["vert_conf_in"], g["color_time_in"], g["norm_rad_in"])
    fused_gl, new_gl = gl.fuse(m, T, tick, g["rgb4"], eo.metric(g["depth4"], 3.0), eo.metric(g["filt4"], 3.0), *io, MAXD, 0.73)
    out.update(gl_fused=fused_gl, gl_fuse_feedback=new_gl)
    io2 = (g["index2_in"], g["vert_conf2_in"], g["color_time2_in"], g["norm_rad2_in"])
    out.update(gl_cleaned=gl.clean(g["fused_in"], new_gl, T, tick, *io2, 10.0, BIG, MAXD))
    mt = g["map_t"]
    it = (g["index_t_in"], g["vert_conf_t_in"], g["color_time_t_in"], g["norm_rad_t_in"])
    out.update(gl_index_t=gl.predict_indices(mt, T, tick_t, MAXD, td)[0])
    none = np.zeros((0, 12), np.float32)
    out.update(gl_cleaned_t=gl.clean(mt, none, T, tick_t, *it, 10.0, td, MAXD))
    out.update(gl_cleaned_deformed=gl.clean(mt, none, T, tick_t, *it, 10.0, td, MAXD, nodes=g["nodes"], depth=g["synth_depth_t_in"]))
    # ---- model raycast (ACTIVE, INACTIVE, depth) and fill-in
    ms = g["map_stable"]
    pg = gl.combined_predict(ms, T, MAXD, 10.0, tick, tick, BIG)
    out.update(gl_image=pg[0], gl_vertex=pg[1], gl_normal=pg[2], gl_time=pg[3],
               gl_synth_depth=gl.combined_predict(ms, T, MAXD, 10.0, tick, tick, BIG, depth_only=True))
    pin = gl.combined_predict(mt, T, MAXD, 10.0, 0, tick_t - td, td)
    out.update(gl_old_image=pin[0], gl_old_vertex=pin[1], gl_old_normal=pin[2], gl_old_time=pin[3])
    vi, ni, ii, filt4, rgb4 = g["vertex_in"], g["normal_in"], g["image_in"], g["filt4"], g["rgb4"]
    out.update(gl_fill_vertex=gl.fill_vertex(vi, filt4, 0), gl_fill_normal=gl.fill_normal(ni, filt4, 0), gl_fill_image=gl.fill_image(ii, rgb4, 0),
               gl_fill_vertex_pass=gl.fill_vertex(vi, filt4, 1), gl_fill_image_pass=gl.fill_image(ii, rgb4, 1))
    out["gl_error"] = np.array(int(gl.lib.efg_gl_error()))
    return out, g, K


def main():
    if len(sys.argv) > 2 and sys.argv[1] == "--check":
        # live pin of the oracle in another configuration: nothing is written; the oracle is compared with what the shaders just
        # produced, with the same pass-by-pass checks the fixture test applies
        out, g, K = build(sys.argv[2])
        assert int(out["gl_error"]) == 0 and "llvmpipe" in str(out["gl_log"])
        tg.run_all(tg.Oracle(K), dict(g, **out), K, False)
        print("LIVE OK", sys.argv[2])
        return
    if len(sys.argv) == 1:  # one process per configuration: the GL harness keeps the frame size of its first context
        import subprocess

        for config in tg.FIXTURES:
            subprocess.check_call([sys.executable, os.path.abspath(__file__), config])
        return
    config = sys.argv[1]
    out, _, _ = build(config)
    path = tg.fixture_path(config)
    np.savez_compressed(path, **tg.shrink(out, tg.FIXTURES[config]))
    print("wrote", path, os.path.getsize(path) // 1024, "KiB; gl error", int(out["gl_error"]))
    print(out["gl_log"])


if __name__ == "__main__":
    main()
