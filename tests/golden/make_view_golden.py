"""Generates tests/golden/ref_view_*.npz: IndexMap::combinedPredict (splat.vert + combo_splat.frag of the reference tree, unmodified)
executed on Mesa llvmpipe through oracle/gl/ref_gl_harness.cpp (`make -C oracle refgl`, which needs the reference tree), at cameras
other than the one the map was captured with:
    python tests/golden/make_view_golden.py

The map is the one of tests/golden/ref_render_320x240.npz (the CPU oracle after a few frames of the noisy synthetic sequence at
80x60). The harness fixes its camera when it starts, so each camera of test_view_golden.CAMERAS runs in a process of its own and
writes one fixture: the camera, and per view its pose, window and every test_view_golden.STEP-th pixel of the four outputs the
shaders wrote."""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from oracle import ef_refgl as rg  # noqa: E402

import test_view_golden as tv  # noqa: E402

if not rg.in_gl_process():
    if not rg.available():
        raise SystemExit("oracle/_ref/gl is not built (make -C oracle refgl) or Mesa / the reference tree is absent")
    for name in sorted(tv.CAMERAS):
        rg.run_script(os.path.abspath(__file__), name)
    raise SystemExit(0)


def main(name):
    K = tv.CAMERAS[name]
    gl = rg.RefGL(K)
    surfels = tv.load_map()
    out = {"map_source": np.array(os.path.basename(tv.MAP_FIXTURE)), "K": np.array([K.width, K.height, K.fx, K.fy, K.cx, K.cy], np.float64),
           "gl_log": np.array(gl.log())}
    vs = tv.views(surfels)
    out["names"] = np.array(sorted(vs))
    for n in sorted(vs):
        v = vs[n]
        out["T_" + n] = v["T"]
        out["args_" + n] = np.array([v["max_depth"], v["conf_threshold"], v["time"], v["max_time"], v["time_delta"]], np.float64)
        img, vtx, nrm, tm = gl.combined_predict(surfels, v["T"], v["max_depth"], v["conf_threshold"], v["time"], v["max_time"], v["time_delta"])
        out.update({k + "_" + n: tv.cut(a) for k, a in zip(("image", "vertex", "normal", "time"), (img, vtx, nrm, tm))})
        print(name, n, f"{(vtx[..., 2] > 0).mean():.3f} covered")
    out["gl_error"] = np.array(int(gl.lib.efg_gl_error()))
    path = tv.fixture_path(name)
    np.savez_compressed(path, **out)
    print("wrote", path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main(sys.argv[1])
