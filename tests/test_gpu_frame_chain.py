"""Steps of the frame chain that run inside the kernel producing their inputs.

- The two order-preserving compactions: fuse's new surfels (k_fuse_update) and the tracker's photometric candidate list
  (k_sobel_cand). Checked against the CPU oracle at the edges of the item count (no new surfel, every active pixel new, no
  candidate at any level), at a size whose tiles take more than one wave of CTAs, and for run-to-run determinism.
- The frame's prediction, whose raycast also runs the fill-in and counts denseEnough's samples: checked against the stage
  API's separate raycast and fill-in calls."""
import numpy as np
import pytest

from util import assert_same, rel_err

pytestmark = pytest.mark.gpu

MAXD = 20.0
BIG = 2147483647 // 2
COLS = [0, 1, 2, 4, 5, 6, 7, 8, 9, 10, 11]  # every column but the confidence (expf: <= 2 ulp apart from the oracle's libm)


def intrinsics(w, h):
    from elasticfusion_b200 import synth

    f = 0.825 * w
    return synth.Intrinsics(w, h, f, f, w / 2.0, h / 2.0)


def make_ctx(K, **kw):
    from elasticfusion_b200 import capi

    kw.setdefault("capacity", 4 * K.width * K.height)
    kw.setdefault("time_delta", BIG)
    return capi.Context(capi.default_config(K.width, K.height, K.fx, K.fy, K.cx, K.cy, **kw))


def fuse_once(K, rgb, depth, surfels, T, tick, w=0.73):
    """One stage-API index map + fuse on a fresh context holding `surfels`; returns (map, new surfels)."""
    from oracle import ef_oracle as eo

    filt = eo.bilateral(depth, 3.0)
    ctx = make_ctx(K)
    try:
        ctx.upload("RGB", rgb)
        ctx.upload("DEPTH_METRIC", eo.metric(depth, 3.0))
        ctx.upload("DEPTH_METRIC_FILTERED", eo.metric(filt, 3.0))
        ctx.map_upload(surfels)
        ctx.map_predict_indices(T, tick, MAXD, BIG)
        ctx.map_fuse(T, tick, MAXD, w)
        return ctx.map_download(), ctx.map_download_new()
    finally:
        ctx.close()


def oracle_fuse(K, rgb, depth, surfels, T, tick, w=0.73):
    from oracle import ef_oracle as eo

    filt = eo.bilateral(depth, 3.0)
    idx = eo.predict_indices(surfels, T, tick, MAXD, BIG, K)
    return eo.fuse(surfels, T, tick, rgb, eo.metric(depth, 3.0), eo.metric(filt, 3.0), *idx, MAXD, w, K)


@pytest.mark.parametrize("size", [(640, 480), (1920, 1080)])
@pytest.mark.parametrize("tick", [2, 3])
def test_fuse_every_active_pixel_new(size, tick):
    """Empty map: every active pixel of the quarter grid (both parities) becomes a new surfel, in draw order. At 1920x1080 the
    quarter grid is 4050 tiles, more than one resident wave of k_fuse_update."""
    from elasticfusion_b200 import synth

    K = intrinsics(*size)
    rgb, depth, T = next(iter(synth.sequence(1, K, seed=11, noise=True)))
    T = np.asarray(T, np.float64)
    empty = np.zeros((0, 12), np.float32)
    _, ref_new = oracle_fuse(K, rgb, depth, empty, T, tick)
    assert len(ref_new) > 0.5 * (size[0] // 2) * (size[1] // 2)
    got_map, got_new = fuse_once(K, rgb, depth, empty, T, tick)
    assert len(got_map) == 0
    assert len(got_new) == len(ref_new)
    assert_same(got_new[:, COLS], ref_new[:, COLS], "new surfels")
    assert rel_err(got_new[:, 3], ref_new[:, 3]) < 1e-6
    _, again = fuse_once(K, rgb, depth, empty, T, tick)
    assert again.tobytes() == got_new.tobytes()


def test_fuse_no_new_surfel(frames, K):
    """No valid depth: no pixel takes part, nothing is added and the map is left as it was."""
    from util import run_oracle

    f = run_oracle(frames, K, 2)
    m = f.map()
    rgb, depth, _ = frames[2]
    got_map, got_new = fuse_once(K, rgb, np.zeros_like(depth), m, f.pose, f.tick)
    assert len(got_new) == 0
    assert_same(got_map, m, "map")


def test_fuse_matches_oracle_and_is_deterministic(frames, K):
    """A map of earlier frames: the new surfels interleave with matched pixels across tiles."""
    from util import run_oracle

    f = run_oracle(frames, K, 4)
    m = f.map()
    rgb, depth, _ = frames[4]
    _, ref_new = oracle_fuse(K, rgb, depth, m, f.pose, f.tick)
    got_map, got_new = fuse_once(K, rgb, depth, m, f.pose, f.tick)
    assert len(got_new) > 100
    # acosf (the normal-angle gate) may associate a handful of pixels differently from the oracle
    assert abs(len(got_new) - len(ref_new)) <= 2
    if len(got_new) == len(ref_new):
        assert_same(got_new[:, COLS], ref_new[:, COLS], "new surfels")
    map2, new2 = fuse_once(K, rgb, depth, m, f.pose, f.tick)
    assert new2.tobytes() == got_new.tobytes() and map2.tobytes() == got_map.tobytes()


def run_frames(K, frames, **kw):
    ctx = make_ctx(K, **kw)
    try:
        for i, (rgb, depth, _) in enumerate(frames):
            ctx.process_frame(rgb, depth, i)
        return ctx.get_pose(), ctx.map_download()
    finally:
        ctx.close()


def test_no_photometric_candidates():
    """A black colour image has no candidate at any level (the 4x4 non-zero test fails everywhere): the frame tracks on
    geometry alone, as the oracle does."""
    from elasticfusion_b200 import synth
    from oracle import ef_oracle as eo

    K = intrinsics(320, 240)
    frames = [(np.zeros_like(rgb), depth, T) for rgb, depth, T in synth.sequence(3, K, seed=3, noise=True)]
    pose, m = run_frames(K, frames)
    ref = eo.Fusion(K, capacity=4 * K.width * K.height)
    for i, (rgb, depth, _) in enumerate(frames):
        ref.process_frame(rgb, depth, i)
    assert np.isfinite(pose).all()
    assert np.abs(pose - ref.pose).max() < 1e-4, (pose, ref.pose)
    assert abs(len(m) - ref.count) <= max(2, ref.count // 1000)


def test_frame_chain_deterministic_multiwave():
    """1920x1080: both compactions run over more tiles than one resident wave. Two contexts give the same pose and map bytes."""
    from elasticfusion_b200 import synth

    K = intrinsics(1920, 1080)
    frames = list(synth.sequence(3, K, seed=5, noise=True))
    p1, m1 = run_frames(K, frames)
    p2, m2 = run_frames(K, frames)
    assert len(m1) > 0
    assert p1.tobytes() == p2.tobytes()
    assert m1.tobytes() == m2.tobytes()


@pytest.mark.parametrize("lookahead", [False, True])
@pytest.mark.parametrize("size", [(640, 480), (424, 240)])
def test_fused_predict_matches_stage_api(size, lookahead):
    """The frame's prediction runs the fill-in and counts denseEnough's samples inside the raycast. After every frame its
    fill-in buffers and dense flag must equal the separate raycast + fill-in calls of the stage API on the same state, and
    the flag must equal denseEnough over the downloaded image."""
    from elasticfusion_b200 import synth
    from oracle import ef_oracle as eo

    K = intrinsics(*size)
    frames = list(synth.sequence(30, K, seed=9, noise=True))
    ctx = make_ctx(K)
    names = ("FILL_VERTEX", "FILL_NORMAL", "FILL_IMAGE")
    try:
        if lookahead:
            ctx.prefetch_frame(frames[0][0], frames[0][1])
        for i, (rgb, depth, _) in enumerate(frames):
            if lookahead:
                ctx.process_frame_device(None, None, i)
                if i + 1 < len(frames):
                    ctx.prefetch_frame(frames[i + 1][0], frames[i + 1][1])
                ctx.finish_frame()
            else:
                ctx.process_frame(rgb, depth, i)
            fused = [ctx.download(n) for n in names]
            dense = ctx.dense_enough()
            assert dense == bool(eo.dense_enough(ctx.download("IMAGE"))), i
            tick = ctx.get_tick() - 1  # the prediction ran before the frame advanced the tick
            ctx.map_raycast(None, MAXD, 10.0, tick, tick, BIG, 0)
            ctx.map_fill_in(False, False)
            for n, a in zip(names, fused):
                assert ctx.download(n).tobytes() == a.tobytes(), (n, i)
            assert ctx.dense_enough() == dense, i
    finally:
        ctx.close()
