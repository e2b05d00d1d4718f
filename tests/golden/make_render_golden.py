"""Generates tests/golden/ref_render_{160x120,320x240}.npz: the global-surface render of the reference's viewer
(GlobalModel::renderPointCloud and the colour pass of GUI::drawFXAA), produced by the REFERENCE's OWN SHADER FILES
(draw_global_surface.{vert,geom,frag} and draw_global_surface_phong.frag of the reference tree, unmodified) executed on Mesa llvmpipe
through oracle/gl/ref_gl_render.cpp in the context of oracle/gl/ref_gl_harness.cpp (`make -C oracle refgl`, which needs the
reference tree):
    python tests/golden/make_render_golden.py           writes the fixtures
    python tests/golden/make_render_golden.py --check   renders the fixtures' views live and compares them with the CPU oracle

Each fixture holds the map (the CPU oracle's after a few frames of the noisy synthetic sequence, tests/test_render_golden.build_map),
every view's EfRenderView fields and the RGBA image the shaders drew."""
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

import test_render_golden as tr  # noqa: E402
from oracle import ef_refgl_render as rgr  # noqa: E402
from oracle import ef_render_oracle as ero  # noqa: E402


def main(check):
    gl = rg.RefGL(tr.MAP_K)
    if check:
        for size in sorted(tr.FIXTURES):
            surfels, vs, _ = tr.load_fixture(size)
            live = {n: rgr.render(gl, surfels, v) for n, v in vs.items()}
            tr.check_against(surfels, vs, live, lambda v: ero.render(surfels, v), "live " + size)
        assert int(gl.lib.efg_gl_error()) == 0
        return
    surfels, T, tick = tr.build_map()
    print(len(surfels), "surfels")
    for size, path in sorted(tr.FIXTURES.items()):
        vs = tr.views(surfels, T, tick, size)
        names = sorted(vs)
        out = {"map": surfels, "names": np.array(names), "gl_log": np.array(gl.log())}
        arr = [vs[n].as_array() for n in names]
        out["vi"], out["vf"] = np.stack([a[0] for a in arr]), np.stack([a[1] for a in arr])
        for n in names:
            out["img_" + n] = rgr.render(gl, surfels, vs[n])
            print(size, n, int(np.count_nonzero(out["img_" + n][..., 3])), "pixels drawn")
        out["gl_error"] = np.array(int(gl.lib.efg_gl_error()))
        np.savez_compressed(path, **out)
        print("wrote", path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main("--check" in sys.argv[1:])
