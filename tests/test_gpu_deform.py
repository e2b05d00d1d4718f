"""Device deformation-graph solve of the local loop closure (ef_deform_solve) against the reference's own solver.

tests/golden/ref_deform.npz holds inputs and outputs of the reference's DeformationGraph.cpp + CholeskyDecomp.cpp, compiled
unmodified (tests/golden/make_deform_golden.py): synthetic graphs and accepted closures of the oracle pipeline. The device
assembles the normal equations directly and runs its own block-band Cholesky; the reference factorises the materialised
JᵀJ (here through Eigen's LLᵀ behind a CHOLMOD stand-in), so the two agree in rounding only. Node selection and the number of
Gauss-Newton iterations must agree exactly; the stop reason is compared with the CPU restatement oracle/efo_deform.py, which
reports it.
"""
import ctypes
import os

import numpy as np
import pytest

from oracle import efo_deform as ed

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ref_deform.npz")
# Bars. On an H100 the fp64 R of the device differs from the reference's by at most 1.1e-12 and t by at most 4.2e-11 relative
# to the largest |t| over these cases (the CPU restatement: 5.9e-13 and 2.4e-11); 1e-9 leaves a margin above 20. nodes16 are float32 casts of those values:
# a cast may flip by one ulp (2.4e-7 at magnitude ~2).
RT_REL = 1e-9
NODE_ATOL = 4e-7
ERR_REL = 1e-6


def golden_cases():
    g = np.load(GOLDEN)
    out = []
    for name in g["cases"]:
        args = {k.split("/")[-1]: g[k] for k in g.files if k.startswith(f"{name}/in/")}
        args["pin"] = bool(args["pin"])
        args["last_deform_time"] = int(args["last_deform_time"])
        ref = {k.split("/", 1)[1]: g[k] for k in g.files if k.startswith(f"{name}/") and "/in/" not in k}
        out.append((str(name), args, ref))
    return out


CASES = golden_cases()


@pytest.fixture(scope="module")
def ctx():
    from elasticfusion_b200 import capi

    c = capi.Context(capi.default_config(320, 240, 264.0, 264.0, 160.0, 120.0, capacity=10000))
    yield c
    c.close()


def _case(name):
    return next(a for n, a, _ in CASES if n == name)


@pytest.mark.parametrize("name,args,ref", CASES, ids=[c[0] for c in CASES])
def test_device_solve_matches_the_reference_solver(ctx, name, args, ref):
    info, nodes, cn, cw, R, t = ctx.deform_solve(**args)
    m = len(args["src"]) * (2 if args["pin"] else 1)
    assert info["n_constraints"] == m and info["n_nodes"] == len(args["node_pos"])
    # identical neighbour selection; weights from the same fp64 formula
    assert np.array_equal(cn, ref["cons_nodes"])
    assert np.abs(cw - ref["cons_weights"]).max() <= 1e-15
    # identical Gauss-Newton decisions: iteration count against the reference, stop reason against the CPU restatement
    assert info["iterations"] == int(ref["iterations"]), (info, int(ref["iterations"]))
    cpu = ed.deform_solve(**args)[0]
    assert (info["iterations"], info["stop"]) == (cpu["iterations"], cpu["stop"]), (info, cpu)
    assert info["stop"] not in (5, 6)
    assert abs(info["error"] - float(ref["error"])) <= ERR_REL * max(abs(float(ref["error"])), 1e-30), (info, ref["error"])
    assert abs(info["meanConsErr"] - float(ref["meanConsErr"])) <= ERR_REL * abs(float(ref["meanConsErr"])), (info, ref["meanConsErr"])
    dR = np.abs(R - ref["R"]).max()
    dt = np.abs(t - ref["t"]).max() / max(np.abs(ref["t"]).max(), 1e-3)
    dn = np.abs(nodes.astype(np.float64) - ref["nodes16"]).max()
    print(f"{name}: iterations {info['iterations']} stop {info['stop']} bandwidth {info['bandwidth']} error {info['error']:.6g} "
          f"meanConsErr {info['meanConsErr']:.6g}  |dR| {dR:.3g}  |dt|/|t| {dt:.3g}  |d nodes16| {dn:.3g}")
    assert dR <= RT_REL and dt <= RT_REL
    assert dn <= NODE_ATOL
    if name == "pinned_three_iterations":
        assert info["iterations"] == 3 and info["stop"] == 0
    if info["n_enabled"] == 0:
        assert np.array_equal(nodes, ref["nodes16"])  # nothing may move
    else:
        assert np.abs(t).max() > 1e-3  # the solve did move the graph


def test_device_solve_is_deterministic(ctx):
    args = _case("max_graph")
    a = ctx.deform_solve(**args)
    b = ctx.deform_solve(**args)
    assert a[0] == b[0]
    for x, y in zip(a[1:], b[1:]):
        assert np.array_equal(x, y)


def test_solved_graph_reduces_constraint_error(ctx):
    """A rigid displacement of the constraint targets is followed: the mean constraint error falls well below the shift."""
    args = _case("unpinned_200")
    before = float(np.linalg.norm(args["dst"] - args["src"], axis=1).mean())
    info = ctx.deform_solve(**args)[0]
    assert info["meanConsErr"] < 0.05 * before, (info, before)


def test_deform_solve_rejects_bad_graphs(ctx):
    from elasticfusion_b200 import capi

    pos, times, src, dst, st, dt = ed.synthetic_case(1024, 10, seed=1)
    args = dict(node_pos=pos, node_times=times, src=src, dst=dst, src_times=st, dst_times=dt)
    with pytest.raises(capi.EfError):
        ctx.deform_solve(**args)  # MAX_GRAPH_NODES
    args = dict(args, node_pos=pos[:4], node_times=times[:4])
    with pytest.raises(capi.EfError):
        ctx.deform_solve(**args)  # fewer than k + 1 nodes
    args = dict(args, node_pos=pos[:50], node_times=times[:50][::-1].copy())
    with pytest.raises(capi.EfError):
        ctx.deform_solve(**args)  # the graph must be in time order
    lib = capi.lib()
    res = capi.EfDeformResult()
    assert lib.ef_deform_solve(ctx.h_ctx, None, None, 10, None, None, None, None, 1, 0, 0, None, None, None, None,
                               ctypes.byref(res)) == -1
