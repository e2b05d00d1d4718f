"""Fuse's association-conflict rule against the REFERENCE'S OWN GLSL SHADERS: tests/golden/ref_fuse_sparse_160x120.npz holds what
the reference's index_map and data / update shaders (unmodified, on Mesa llvmpipe; generator tests/golden/make_sparse_golden.py)
computed on room maps of ~20 k surfels (sparser than the quarter pixel grid fuse samples: many pixels pick the same surfel and
only the lowest draw index may update it, SURVEY App. A-17) and ~400 k surfels (denser: almost every matched pixel owns its
surfel), measured by one frame of the 160x120 synthetic sequence at its ground-truth pose.

The inputs are recomputed here from synth.room_surfels and the synthetic frames (the index-map input of fuse is the CPU oracle's,
as in test_gl_golden.py), so the fixture holds only the shaders' outputs: the index map, the rows fuse changed and their ids,
the number of matched measurements and of new surfels."""
import os

import numpy as np
import pytest

from test_gl_golden import COLS, frac_differ

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FIXTURE = os.path.join(ROOT, "tests", "golden", "ref_fuse_sparse_160x120.npz")
MAXD, BIG = 20.0, 2 ** 30
SEED, FRAME, TICK, WEIGHT = 7, 3, 4, 0.73
CASES = {"sparse": 20000, "dense": 400000}


def small_K():
    from elasticfusion_b200 import synth

    return synth.Intrinsics(160, 120, 132.0, 132.0, 80.0, 60.0)


def sparse_inputs(n_surfels, K=None):
    """A room map of ~n_surfels stable surfels in the sequence's world frame, frame FRAME as the measurement at its ground-truth
    pose, and the oracle's index map of the map (the index input of fuse on both sides)."""
    from elasticfusion_b200 import synth
    from oracle import ef_oracle as eo

    K = K or small_K()
    rgb, depth, T = list(synth.sequence(FRAME + 1, K, seed=SEED, noise=True))[FRAME]
    T_w_room = np.linalg.inv(synth.trajectory(1, seed=SEED)[0])
    m = synth.room_surfels(n_surfels, T_w_room, view_depth=1.5, focal=K.fx)
    filt = eo.bilateral(depth, 3.0)
    g = dict(K=K, map=m, T=T, rgb=rgb, depth=depth, filt=filt, dm=eo.metric(depth, 3.0), dmf=eo.metric(filt, 3.0))
    g["idx"] = eo.predict_indices(m, T, TICK, MAXD, BIG, K)
    return g


def changed_ids(before, after):
    """Ids of the surfels whose 12 floats are not bit-identical (NaN == NaN)."""
    same = (before == after) | (np.isnan(before) & np.isnan(after))
    return np.flatnonzero(~same.all(axis=1)).astype(np.uint32)


def active_pixels(dm, tick):
    """Pixels of the quarter grid fuse measures this frame (data.vert: x, y of this tick's parity, all four neighbours with a
    depth, 0 < z <= maxDepth): each one is either matched to a surfel or becomes a new one."""
    rows, cols = dm.shape
    jj, ii = np.mgrid[0:rows, 0:cols]
    p = np.pad(dm, 1, mode="edge")
    ok = (ii % 2 == tick % 2) & (jj % 2 == tick % 2) & (dm > 0) & (dm <= MAXD)
    ok &= (p[1:-1, :-2] != 0) & (p[1:-1, 2:] != 0) & (p[:-2, 1:-1] != 0) & (p[2:, 1:-1] != 0)
    return int(ok.sum())


def oracle_fuse(g):
    from oracle import ef_oracle as eo

    return eo.fuse(g["map"], g["T"], TICK, g["rgb"], g["dm"], g["dmf"], *g["idx"], MAXD, WEIGHT, g["K"])


@pytest.fixture(scope="module")
def Z():
    z = dict(np.load(FIXTURE))
    assert int(z["gl_error"]) == 0 and "llvmpipe" in str(z["gl_log"])
    return z


def check_case(Z, case, g, index, fused, new):
    """index / fused / new: the implementation's index map, fused map and new surfels on the inputs g."""
    assert frac_differ(index, Z[case + "_index"]) <= 5e-4  # a window coordinate within float rounding of a snapping boundary
    ids = changed_ids(g["map"], fused)
    assert np.array_equal(ids, Z[case + "_ids"]), (case, len(ids), len(Z[case + "_ids"]), len(np.setxor1d(ids, Z[case + "_ids"])))
    ref = Z[case + "_rows"]
    got = fused[ids]
    assert frac_differ(got[:, COLS], ref[:, COLS], 1e-5) == 0, case
    assert np.abs(got[:, 3] - ref[:, 3]).max() <= 1e-5 * max(1.0, np.abs(ref[:, 3]).max()), case
    assert len(new) == int(Z[case + "_new_n"]), (case, len(new), int(Z[case + "_new_n"]))
    # every active pixel of the quarter grid is either new or matched: the shaders' count of matched measurements
    matched = int(Z[case + "_matched"])
    assert active_pixels(g["dm"], TICK) == matched + len(new)
    return matched - len(ids)  # measurements that lost their surfel to a lower draw index


@pytest.mark.parametrize("case", sorted(CASES))
def test_oracle_fuse_conflicts_match_reference_shaders(Z, case):
    """oracle/efo_map.cpp == the reference's shaders on a sparse and a dense map: the index map, the exact set of surfels fuse
    changed, their rows and the new-surfel count. On the sparse map over a thousand measurements lose their surfel to a lower
    draw index, so the winner rule is what the changed rows pin."""
    from oracle import ef_oracle as eo

    g = sparse_inputs(CASES[case])
    index = eo.predict_indices(g["map"], g["T"], TICK, MAXD, BIG, g["K"])[0]
    fused, new = oracle_fuse(g)
    lost = check_case(Z, case, g, index, fused, new)
    if case == "sparse":
        assert lost >= 1000, lost
    else:
        assert len(Z[case + "_ids"]) > 1000


@pytest.mark.gpu
@pytest.mark.parametrize("case", sorted(CASES))
def test_product_fuse_conflicts_match_reference_shaders(Z, case):
    """libefusion.so == the reference's shaders, through the C ABI, on the same inputs."""
    from elasticfusion_b200 import capi

    g = sparse_inputs(CASES[case])
    K = g["K"]
    ctx = capi.Context(capi.default_config(K.width, K.height, K.fx, K.fy, K.cx, K.cy, capacity=500000, time_delta=BIG))
    try:
        ctx.upload("RGB", g["rgb"])
        ctx.upload("DEPTH_METRIC", g["dm"])
        ctx.upload("DEPTH_METRIC_FILTERED", g["dmf"])
        ctx.map_upload(g["map"])
        ctx.map_predict_indices(g["T"], TICK, MAXD, BIG)
        index = ctx.download("INDEX")
        for name, a in zip(("INDEX", "VERT_CONF", "COLOR_TIME", "NORM_RAD"), g["idx"]):
            ctx.upload(name, a)  # fuse reads the oracle's index map, as the shaders did
        ctx.map_fuse(g["T"], TICK, MAXD, WEIGHT)
        check_case(Z, case, g, index, ctx.map_download(), ctx.map_download_new())
    finally:
        ctx.close()
