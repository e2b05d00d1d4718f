"""CPU checks of the deformation-solve restatement (oracle/efo_deform.py) against the reference's own solver (the stored
fixture tests/golden/ref_deform.npz, and live when oracle/_ref/libef_refdef.so is built), and of ef_deform_solve's argument
validation."""
import ctypes
import os

import numpy as np
import pytest

from oracle import efo_deform as ed

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ref_deform.npz")
# measured spread of the restatement against the reference: R / t within 2.4e-11 relative, error and meanConsErr equal
RT_REL = 1e-9


def _golden():
    g = np.load(GOLDEN)
    out = []
    for name in g["cases"]:
        args = {k.split("/")[-1]: g[k] for k in g.files if k.startswith(f"{name}/in/")}
        args["pin"] = bool(args["pin"])
        args["last_deform_time"] = int(args["last_deform_time"])
        ref = {k.split("/", 1)[1]: g[k] for k in g.files if k.startswith(f"{name}/") and "/in/" not in k}
        out.append((str(name), args, ref))
    return out


CASES = _golden()


def _compare(ours, ref):
    info, nodes, cn, cw, R, t = ours
    assert np.array_equal(cn, ref["cons_nodes"])
    assert np.abs(cw - ref["cons_weights"]).max() <= 1e-15
    assert info["iterations"] == int(ref["iterations"])
    assert abs(info["error"] - float(ref["error"])) <= 1e-6 * max(abs(float(ref["error"])), 1e-30)
    assert abs(info["meanConsErr"] - float(ref["meanConsErr"])) <= 1e-6 * abs(float(ref["meanConsErr"]))
    assert np.abs(R - ref["R"]).max() <= RT_REL
    assert np.abs(t - ref["t"]).max() <= RT_REL * max(np.abs(ref["t"]).max(), 1e-3)
    assert np.abs(nodes.astype(np.float64) - ref["nodes16"]).max() <= 4e-7


def test_fixture_covers_the_required_cases():
    names = [c[0] for c in CASES]
    assert {"pinned_200", "unpinned_200", "prefix_fixed", "all_fixed", "five_nodes", "max_graph"} <= set(names)
    pipeline = [c for c in CASES if c[0].startswith("pipeline_")]
    assert len(pipeline) >= 2 and pipeline[0][1]["pin"] and not pipeline[1][1]["pin"] and pipeline[1][1]["last_deform_time"] > 0
    big = dict((n, a) for n, a, _ in CASES)["max_graph"]
    assert len(big["node_pos"]) == 1023 and len(big["src"]) == 768 and big["pin"]
    assert int(dict((n, r) for n, _, r in CASES)["pinned_three_iterations"]["iterations"]) == 3


@pytest.mark.parametrize("name,args,ref", CASES, ids=[c[0] for c in CASES])
def test_restatement_matches_the_reference_fixture(name, args, ref):
    _compare(ed.deform_solve(**args), ref)


@pytest.mark.skipif(not ed.ref_available(), reason="oracle/_ref/libef_refdef.so not built (needs the reference tree)")
@pytest.mark.parametrize("name,args,ref", CASES[:3] + CASES[-2:], ids=[c[0] for c in CASES[:3] + CASES[-2:]])
def test_restatement_matches_the_reference_solver_live(name, args, ref):
    live = ed.ref_solve(**args)
    assert live[0]["iterations"] == int(ref["iterations"])
    _compare(ed.deform_solve(**args), dict(ref, R=live[4], t=live[5], cons_nodes=live[2], cons_weights=live[3],
                                           nodes16=live[1], error=live[0]["error"], meanConsErr=live[0]["meanConsErr"]))


def test_neighbours_follow_connect_graph_seq():
    nb = ed.neighbours(9)
    assert nb[0] == [1, 2, 3, 4] and nb[1] == [0, 2, 3, 4]
    assert nb[4] == [3, 5, 2, 6]
    assert nb[7] == [4, 5, 6, 8] and nb[8] == [4, 5, 6, 7]
    assert all(len(x) == 4 for x in nb)


def test_weights_pick_the_nearest_nodes_of_the_time_window():
    pos, times, src, dst, st, dt = ed.synthetic_case(100, 40, seed=3)
    S, D, T = ed.expand_constraints(src, dst, st, dt, True)
    for l in range(len(S)):
        ids, w = ed.weight_point(pos, times, S[l], int(T[l]))
        assert ids == sorted(ids) and len(set(ids)) == ed.K
        assert abs(sum(w) - 1) < 1e-12 and min(w) >= 0
        assert ids[-1] - ids[0] < ed.LOOKBACK  # one 20-node window
        # the node nearest in time is in that window, and a closer node never weighs less
        f = int(np.argmin(np.abs(times.astype(np.int64) - int(T[l]))))
        assert ids[-1] - ed.LOOKBACK < f < ids[0] + ed.LOOKBACK
        d = [np.linalg.norm(pos[j] - S[l]) for j in ids]
        for a in range(ed.K):
            for b in range(ed.K):
                if d[a] < d[b]:
                    assert w[a] >= w[b]


def test_gauss_newton_step_is_the_least_squares_step():
    """The band-Cholesky step on JᵀJ equals a dense least-squares solve of J delta = -r."""
    pos, times, src, dst, st, dt = ed.synthetic_case(40, 30, seed=5)
    S, D, T = ed.expand_constraints(src, dst, st, dt, True)
    s = ed.Solver(pos, times, S, D, T, int(times[10]))
    r = s.residual()
    J = s.jacobian()
    assert J.shape == (len(r), 12 * s.N)
    delta = s.solve_normal(J, r)
    ref = np.linalg.lstsq(J.toarray(), -r, rcond=None)[0]
    assert np.abs(delta - ref).max() <= 1e-9 * np.abs(ref).max()


def test_rigid_shift_is_followed():
    """Constraints that all ask for one translation are met by the solved graph, which stays rigid."""
    pos, times, src, _, st, _ = ed.synthetic_case(60, 80, seed=2)
    shift = np.array([0.02, -0.01, 0.015])
    info, nodes, _, _, R, t = ed.deform_solve(pos, times, src, src + shift, st)
    assert info["meanConsErr"] < 1e-4, info
    near = np.unique(ed.Solver(pos, times, src, src + shift, st, 0).cnode)
    assert np.abs(t[near] - shift).max() < 2e-3
    assert np.abs(R[near] - np.eye(3)).max() < 2e-2


def test_fixed_nodes_do_not_move():
    pos, times, src, dst, st, dt = ed.synthetic_case(80, 40, seed=4)
    ldt = int(times[40])
    info, nodes, _, _, R, t = ed.deform_solve(pos, times, src, dst, st, dt, pin=True, last_deform_time=ldt)
    fixed = times <= ldt
    assert info["n_enabled"] == int((~fixed).sum())
    assert np.array_equal(t[fixed], np.zeros_like(t[fixed])) and np.array_equal(R[fixed], np.tile(np.eye(3), (fixed.sum(), 1, 1)))
    assert np.array_equal(nodes[:, 15], times.astype(np.float32))


def test_deform_abi_argument_validation_without_gpu():
    from elasticfusion_b200 import capi

    lib = capi.lib()
    res = capi.EfDeformResult()
    pos = np.zeros((10, 3))
    tm = np.arange(10, dtype=np.int32)
    one = np.zeros((1, 3))
    t1 = np.zeros(1, np.int32)
    p = lambda a: a.ctypes.data_as(ctypes.c_void_p)
    # every call is rejected before the device is touched
    assert lib.ef_deform_solve(None, p(pos), p(tm), 10, p(one), p(one), p(t1), p(t1), 1, 1, 0, None, None, None, None,
                               ctypes.byref(res)) == -1
    assert lib.ef_deform_solve(None, None, None, 0, None, None, None, None, 0, 0, 0, None, None, None, None, None) == -1
    assert ctypes.sizeof(capi.EfDeformResult) == 32
