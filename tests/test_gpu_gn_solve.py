"""The Gauss-Newton solve of the tracker, iteration by iteration, against float64 numpy.

For every traced SE(3) iteration of getIncrementalTransformation (RGBDOdometry.cpp:492-551), on the coarse-level cluster path
(k_gn_cluster, the default) and on the two-kernel path (EF_GN_CLUSTER=0):
- lastA / lastb are the reduced systems combined with the ICP weight;
- `result` is the unpivoted LDL^T solution of lastA x = lastb;
- the pose each iteration hands to the next (resultRt = [rodrigues(x[3:]) | x[:3]] * resultRt) composes to the tracker's output;
- two runs of the same call are bit-identical, trace and pose."""
import numpy as np
import pytest

from elasticfusion_b200 import capi, synth

gpu = pytest.mark.gpu
BIG = 2147483647 // 2
ICP_WEIGHT = 10.0

SIZES = {
    "640x480": synth.K_DEFAULT,
    "424x240": synth.Intrinsics(424, 240, 212.0, 212.0, 212.0, 120.0),  # level-2 width 106: not a multiple of four
}


def ldlt_solve(A, b):
    """Unpivoted LDL^T of a symmetric 6x6 system in float64 (the order of efm::ldlt_solve_unrolled)."""
    n = len(b)
    L, D = np.eye(n), np.zeros(n)
    for j in range(n):
        D[j] = A[j, j] - sum(L[j, k] * L[j, k] * D[k] for k in range(j))
        for i in range(j + 1, n):
            L[i, j] = (A[i, j] - sum(L[i, k] * L[j, k] * D[k] for k in range(j))) / D[j]
    y = np.zeros(n)
    for i in range(n):
        y[i] = b[i] - sum(L[i, k] * y[k] for k in range(i))
    y /= D
    x = np.zeros(n)
    for i in reversed(range(n)):
        x[i] = y[i] - sum(L[k, i] * x[k] for k in range(i + 1, n))
    return x


def rodrigues(r):
    R = np.eye(3)
    theta = float(np.sqrt(r @ r))
    if theta >= np.finfo(np.float64).eps:
        c, s = np.cos(theta), np.sin(theta)
        k = r / theta
        kx = np.array([[0, -k[2], k[1]], [k[2], 0, -k[0]], [-k[1], k[0], 0]])
        R = c * np.eye(3) + (1.0 - c) * np.outer(k, k) + s * kx
    return R


def track_twice(K, monkeypatch, cluster):
    monkeypatch.delenv("EF_GN_CLUSTER_LEVELS", raising=False)
    if cluster:
        monkeypatch.delenv("EF_GN_CLUSTER", raising=False)
    else:
        monkeypatch.setenv("EF_GN_CLUSTER", "0")
    ctx = capi.Context(capi.default_config(K.width, K.height, K.fx, K.fy, K.cx, K.cy, capacity=400000, time_delta=BIG))
    try:
        for i, (rgb, depth, _) in enumerate(synth.sequence(4, K, seed=11, noise=True)):
            ctx.process_frame(rgb, depth, i)
        T_prev = ctx.get_pose()
        runs = [ctx.odom_track(T_prev, icp_weight=ICP_WEIGHT, so3=False) for _ in range(2)]
    finally:
        ctx.close()
    return T_prev, runs


@gpu
@pytest.mark.parametrize("cluster", [True, False], ids=["cluster", "two-kernel"])
@pytest.mark.parametrize("size", list(SIZES))
def test_gn_solve_per_iteration(size, cluster, monkeypatch):
    T_prev, runs = track_twice(SIZES[size], monkeypatch, cluster)
    (T_out, trace), (T_out2, trace2) = runs
    assert trace.tobytes() == trace2.tobytes() and T_out.tobytes() == T_out2.tobytes(), "two runs differ"

    se3 = [t for t in trace if t["kind"] == 0]
    assert [(int(t["level"]), int(t["iter"])) for t in se3] == [(lv, it) for lv, n in ((2, 4), (1, 5), (0, 10)) for it in range(n)]
    w = float(np.float32(ICP_WEIGHT))
    resultRt = np.eye(4)
    for t in se3:
        where = (size, int(t["level"]), int(t["iter"]))
        A_icp, A_rgb = t["A_icp"].astype(np.float64).reshape(6, 6), t["A_rgb"].astype(np.float64).reshape(6, 6)
        b_icp, b_rgb = t["b_icp"].astype(np.float64), t["b_rgb"].astype(np.float64)
        A, b, x = t["lastA"].reshape(6, 6), t["lastb"], t["result"]
        assert (A_icp == A_icp.T).all() and (A_rgb == A_rgb.T).all() and (A == A.T).all(), ("symmetric", where)
        # w^2 a and w b are exact in float64 for float32 a, b and w = 10: a contracted multiply-add rounds the same single sum
        A_ref, b_ref = A_rgb + w * w * A_icp, b_rgb + w * b_icp
        assert (np.abs(A - A_ref) <= 1e-12 * np.abs(A_ref)).all(), ("lastA", where)
        assert (np.abs(b - b_ref) <= 1e-12 * np.abs(b_ref)).all(), ("lastb", where)
        # the same unpivoted LDL^T in float64: equal up to the rounding of the device's reciprocals, a few ulp times cond(A)
        x_ref = ldlt_solve(A, b)
        assert np.abs(x - x_ref).max() <= np.linalg.cond(A) * 1e-14 * np.abs(x_ref).max(), ("ldlt", where, x, x_ref)
        assert np.abs(A @ x - b).max() <= 1e-10 * (np.linalg.norm(A, np.inf) * np.abs(x).max() + np.abs(b).max()), ("residual", where)
        inc = np.eye(4)
        inc[:3, :3] = rodrigues(np.asarray(x[3:], np.float64))
        inc[:3, 3] = x[:3]
        resultRt = inc @ resultRt
    # the pose the last iteration leaves: [Rprev | tprev] * rgbOdom^-1 in float (RGBDOdometry.cpp:543-551), then the jump
    # check and the orthogonalisation of the finish (:555-569)
    f32 = np.float32
    Rprev, tprev = T_prev[:3, :3].astype(f32), T_prev[:3, 3].astype(f32)
    rot, trn = resultRt[:3, :3].astype(f32), resultRt[:3, 3].astype(f32)
    Rinv = rot.T
    Rcurr, tcurr = Rprev @ Rinv, Rprev @ -(Rinv @ trn) + tprev
    if np.linalg.norm(tcurr - tprev) > 0.3:
        Rcurr, tcurr = Rprev, tprev
    U, _, Vt = np.linalg.svd(Rcurr.astype(np.float64))
    assert np.abs(T_out[:3, :3] - U @ Vt).max() < 1e-6, size
    assert np.abs(T_out[:3, 3] - tcurr.astype(np.float64)).max() < 1e-6, size
