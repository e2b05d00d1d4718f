"""Generates tests/golden/ref_fuse_sparse_160x120.npz: the index map and the fuse pass of the REFERENCE's OWN SHADER FILES (Core/Shaders
of the reference tree, unmodified) executed on Mesa llvmpipe through oracle/gl/ref_gl_harness.cpp (`make -C oracle refgl`, which
needs the reference tree), on the sparse and the dense room map of tests/test_sparse_golden.py:  python tests/golden/make_sparse_golden.py

The inputs are the ones the test recomputes (test_sparse_golden.sparse_inputs); only the shaders' outputs are stored."""
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

import test_sparse_golden as ts  # noqa: E402


def main():
    gl = rg.RefGL(ts.small_K())
    out = {}
    for case, n in sorted(ts.CASES.items()):
        g = ts.sparse_inputs(n)
        out[case + "_index"] = gl.predict_indices(g["map"], g["T"], ts.TICK, ts.MAXD, ts.BIG)[0]
        fused, fb = gl.fuse(g["map"], g["T"], ts.TICK, g["rgb"], g["dm"], g["dmf"], *g["idx"], ts.MAXD, ts.WEIGHT)
        ids = ts.changed_ids(g["map"], fused)
        out.update({case + "_ids": ids, case + "_rows": fused[ids], case + "_matched": np.array(int((fb[:, 7] == -1).sum())),
                    case + "_new_n": np.array(int((fb[:, 7] == -2).sum()))})
        print(case, len(g["map"]), "surfels:", len(ids), "changed,", int(out[case + "_matched"]), "matched,",
              int(out[case + "_new_n"]), "new")
    out["gl_log"] = np.array(gl.log())
    out["gl_error"] = np.array(int(gl.lib.efg_gl_error()))
    np.savez_compressed(ts.FIXTURE, **out)
    print("wrote", ts.FIXTURE, os.path.getsize(ts.FIXTURE) // 1024, "KiB; gl error", int(out["gl_error"]))


if __name__ == "__main__":
    main()
