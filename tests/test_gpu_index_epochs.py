"""The index map's tagged z-buffer across many passes.

Every index pass tags its keys with its own tag and no pass clears the buffer; the host re-arms it once every 255 passes. A
stale key read as live, or a missed re-arm, shows up as a texel that differs from the same pass run on a fresh buffer.
- 600 stage-API passes on one context, alternating two poses that see different texels (two re-arms): the four textures of
  every pass equal those of the first pass at that pose, bit for bit.
- 300 frames at 320x240 (more than two re-arms) through ef_process_frame, whose index passes write no textures and whose fuse
  and clean read the keys, against the same frames with the mapping half run through the stage API, whose passes write the
  textures and whose fuse and clean read them: poses, maps and textures bit-identical after every frame."""
import numpy as np
import pytest

from util import assert_same

pytestmark = pytest.mark.gpu

MAXD = 20.0
BIG = 2147483647 // 2
TEX = ("INDEX", "VERT_CONF", "COLOR_TIME", "NORM_RAD")


def textures(ctx):
    return [ctx.download(n).copy() for n in TEX]


def test_stage_passes_across_tag_wraps():
    from elasticfusion_b200 import capi, synth

    K = synth.K_DEFAULT
    frames = list(synth.sequence(12, K, seed=42, noise=True))
    ctx = capi.Context(capi.default_config(K.width, K.height, K.fx, K.fy, K.cx, K.cy, capacity=1000000, time_delta=BIG))
    try:
        for i, (rgb, depth, _) in enumerate(frames):
            ctx.process_frame(rgb, depth, i)
        tick = ctx.get_tick()
        T0 = ctx.get_pose()
        T1 = T0.copy()
        T1[:3, 3] += np.array([0.35, -0.1, 0.2])  # a shifted view: a different set of occupied texels
        ref = {}
        for k in range(600):
            which = k % 2
            ctx.map_predict_indices(T1 if which else T0, tick, MAXD, BIG)
            got = textures(ctx)
            if which not in ref:
                ref[which] = got
                continue
            for name, g, r in zip(TEX, got, ref[which]):
                assert_same(g, r, f"{name} of pass {k}")
        occ0, occ1 = ref[0][0] > 0, ref[1][0] > 0
        assert occ0.mean() > 0.3 and occ1.mean() > 0.3
        assert (occ0 != occ1).mean() > 0.01  # the two views do not light the same texels
    finally:
        ctx.close()


def test_frame_path_matches_stage_api_across_tag_wraps():
    from elasticfusion_b200 import capi, synth

    K = synth.Intrinsics(320, 240, 264.0, 264.0, 160.0, 120.0)
    frames = list(synth.sequence(300, K, seed=5, noise=True))
    cfg = capi.default_config(K.width, K.height, K.fx, K.fy, K.cx, K.cy, capacity=2000000, time_delta=200)
    a = capi.Context(cfg)
    b = capi.Context(cfg)
    try:
        for i, (rgb, depth, _) in enumerate(frames):
            a.process_frame(rgb, depth, i)
            # b: the same frame with its mapping half (ElasticFusion.cpp:536-593) run through the stage API, at the frame's
            # tick, pose and fusion weighting (None / -1: the tracker's device-resident values)
            b.process_frame_begin(rgb, depth, i)
            tick = b.get_tick()
            if tick > 1:
                b.map_predict_indices(None, tick, MAXD, cfg.time_delta)
                b.map_fuse(None, tick, MAXD, -1.0)
                b.map_predict_indices(None, tick, MAXD, cfg.time_delta)
                b.map_clean(None, tick, cfg.confidence, cfg.time_delta, MAXD)
            b.set(rgb_only=True)  # the frame's end then runs only the prediction and advances the tick
            b.process_frame_end()
            b.set(rgb_only=False)
            assert_same(a.get_pose(), b.get_pose(), f"pose of frame {i}")
            assert a.map_count() == b.map_count(), i
            assert_same(a.map_download(), b.map_download(), f"map of frame {i}")
            for name, x, y in zip(TEX, textures(a), textures(b)):
                assert_same(x, y, f"{name} of frame {i}")
        assert (a.download("INDEX") > 0).mean() > 0.3
    finally:
        a.close()
        b.close()
