"""Scheduling of the frame look-ahead against the frame in flight (EF_LA_AFTER_TRACK): the switch changes when the side
stream's work starts, never what it computes."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

BIG = 2147483647 // 2
N_FRAMES = 12
SWITCHES = [dict(EF_LA_AFTER_TRACK="0"), dict(EF_LA_AFTER_TRACK="1")]
SIZES = {"640x480": None, "424x240": (424, 240, 308.0, 212.0, 120.0)}


@pytest.fixture(scope="module", params=sorted(SIZES))
def seq(request):
    from elasticfusion_b200 import synth

    s = SIZES[request.param]
    K = synth.K_DEFAULT if s is None else synth.Intrinsics(s[0], s[1], s[2], s[2], s[3], s[4])
    return K, list(synth.sequence(N_FRAMES, K, seed=42, noise=True))


def make_ctx(K, monkeypatch, env, stream=None):
    from elasticfusion_b200 import capi

    for k, v in env.items():
        monkeypatch.setenv(k, v)
    try:
        return capi.Context(capi.default_config(K.width, K.height, K.fx, K.fy, K.cx, K.cy, capacity=500000, time_delta=BIG),
                            stream=stream)
    finally:
        for k in env:
            monkeypatch.delenv(k)


def device_frames(frames):
    import torch

    dev = [(torch.from_numpy(np.ascontiguousarray(r)).cuda(), torch.from_numpy(np.ascontiguousarray(d).view(np.int16)).cuda())
           for r, d, _ in frames]
    torch.cuda.synchronize()
    return dev


def run_plain(ctx, frames):
    poses = []
    for i, (rgb, depth, _) in enumerate(frames):
        ctx.process_frame(rgb, depth, i)
        poses.append(ctx.get_pose())
    return np.array(poses), ctx.map_count(), ctx.map_download()


def run_lookahead(ctx, dev, per_frame=None):
    poses = []
    ctx.prefetch_frame_device(dev[0][0].data_ptr(), dev[0][1].data_ptr())
    for i in range(len(dev)):
        ctx.process_frame_device(None, None, i)
        if i + 1 < len(dev):
            ctx.prefetch_frame_device(dev[i + 1][0].data_ptr(), dev[i + 1][1].data_ptr())
        ctx.join_lookahead()
        if per_frame:
            per_frame(i)
        ctx.finish_frame()
        poses.append(ctx.get_pose())
    return np.array(poses), ctx.map_count(), ctx.map_download()


def assert_identical(a, b, what):
    assert np.array_equal(a[0], b[0]), (what, np.abs(a[0] - b[0]).max())
    assert a[1] == b[1], (what, a[1], b[1])
    assert np.array_equal(a[2], b[2], equal_nan=True), what


def test_lookahead_matches_plain_under_every_switch(seq, monkeypatch):
    """Plain calls and the device look-ahead, with the side stream started at frame start or after the cluster, give
    bit-identical poses, counts and maps."""
    K, frames = seq
    dev = device_frames(frames)
    ref = None
    for env in SWITCHES:
        for mode in ("plain", "lookahead"):
            ctx = make_ctx(K, monkeypatch, env)
            try:
                out = run_plain(ctx, frames) if mode == "plain" else run_lookahead(ctx, dev)
            finally:
                ctx.close()
            if ref is None:
                ref = out
                assert np.isfinite(out[0]).all() and out[1] > 0
            else:
                assert_identical(out, ref, (env, mode))


def test_caller_stream_and_library_stream(seq, monkeypatch):
    """A caller-supplied stream and a library-owned one give the same results; ef_stream() stays the caller's stream, and
    syncing it alone is enough for the frame's stage events to be complete."""
    import torch

    K, frames = seq
    dev = device_frames(frames)
    stream = torch.cuda.Stream()
    out = {}
    for name, s in (("library", None), ("caller", stream.cuda_stream)):
        ctx = make_ctx(K, monkeypatch, {"EF_STAGE_TIMING": "1"}, stream=s)
        try:
            if s is not None:
                assert ctx.stream == s

            def check(i):
                if i > 0:
                    ms = ctx.stage_ms()  # synchronises ef_stream() only; an incomplete event reads as 0
                    assert all(ms[k] > 0 for k in (5, 8, 11)), (name, i, ms)

            out[name] = run_lookahead(ctx, dev, check)
        finally:
            ctx.close()
    assert_identical(out["caller"], out["library"], "caller vs library stream")


@pytest.mark.parametrize("env", SWITCHES, ids=lambda e: "after_track=" + e["EF_LA_AFTER_TRACK"])
def test_stage_timing_monotonic(seq, monkeypatch, env):
    """Stage events of a frame are in order, the side stream's work starts after the frame does and ends after it starts, and
    with EF_LA_AFTER_TRACK=1 it starts no earlier than the Gauss-Newton loop's first launch (stage event 4)."""
    K, frames = seq
    dev = device_frames(frames)
    ctx = make_ctx(K, monkeypatch, dict(env, EF_STAGE_TIMING="1"))
    seen = []

    def check(i):
        ms = ctx.stage_ms()
        assert len(ms) == 12 and min(ms) >= 0.0, (i, ms)
        side = ctx.lookahead_ms()
        if i + 1 < len(dev):
            assert side is not None and 0.0 <= side[0] <= side[1], (i, side)
            if i > 0:
                t4 = sum(ms[1:5])
                if env["EF_LA_AFTER_TRACK"] == "1":
                    assert side[0] >= t4 - 1e-3, (i, side, t4)
                seen.append(i)

    try:
        run_lookahead(ctx, dev, check)
    finally:
        ctx.close()
    assert len(seen) == len(dev) - 2


def test_failed_prefetch_then_plain_calls(seq, monkeypatch):
    """A prefetch rejected for its arguments leaves nothing pending: plain calls then run the sequence bit-identically to
    a context that never saw the failed call."""
    from elasticfusion_b200 import capi

    K, frames = seq
    ref_ctx = make_ctx(K, monkeypatch, {})
    try:
        ref = run_plain(ref_ctx, frames)
    finally:
        ref_ctx.close()
    ctx = make_ctx(K, monkeypatch, {})
    try:
        ctx.process_frame(frames[0][0], frames[0][1], 0)
        with pytest.raises(capi.EfError):
            capi._chk(capi.lib().ef_prefetch_frame_device(ctx.h_ctx, None, None))
        with pytest.raises(capi.EfError):
            ctx.process_frame(None, None, 1)  # nothing was staged
        poses = [ctx.get_pose()]
        for i in range(1, len(frames)):
            ctx.process_frame(frames[i][0], frames[i][1], i)
            poses.append(ctx.get_pose())
        assert_identical((np.array(poses), ctx.map_count(), ctx.map_download()), ref, "after a failed prefetch")
    finally:
        ctx.close()
