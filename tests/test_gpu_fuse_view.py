"""ef_map_fuse_view / ef_map_fuse_view_device on the GPU: an RGB-D frame of a second camera fused into the map. The map equals, byte for
byte and in order, what a context built for that camera makes of the same map with the stage calls (preprocess, predictIndices, fuse,
predictIndices, clean); it equals the CPU oracle's stages with the bars of test_gpu_sensor_sizes.py; the frame's own state is left
untouched; and interleaved with frames (also with close_loops = 2 and the look-ahead) it gives the poses and maps of the host-composed
recipe."""
import numpy as np
import pytest

from util import assert_same, rel_err

from elasticfusion_b200 import capi, synth
from oracle import ef_oracle as eo

pytestmark = pytest.mark.gpu
MAXD, BIG, CUTOFF = 20.0, 2147483647 // 2, 3.0


def _k(w, h, f, cx=None, cy=None, fy=None):
    return synth.Intrinsics(w, h, f, f if fy is None else fy, w / 2 if cx is None else cx, h / 2 if cy is None else cy)


# camera B of each case; "own" is the context's camera (K_DEFAULT)
CAMERAS = {
    "own": synth.K_DEFAULT,
    "320x240_offcentre": _k(320, 240, 280.0, 130.0, 140.0, fy=250.0),
    "424x240": _k(424, 240, 305.0),
    "1280x720": _k(1280, 720, 915.0),
    "1920x1080": _k(1920, 1080, 1188.0),
}
TINY = {"33x17": _k(33, 17, 20.0, 15.5, 9.0), "1x1": synth.Intrinsics(1, 1, 1.0, 1.0, 0.5, 0.5)}
# (time offset from the frame's tick, weighting, time_delta, conf_threshold); the last culls the unstable surfels not seen for > 20 ticks
PARAMS = {"tick": (-1, 1.0, BIG, 10.0), "later_odd": (2, 0.4, 200, 10.0), "window": (5, 2.5, 3, 1.0), "cull": (26, 1.0, BIG, 10.0)}


def cam_offset(deg=8.0, t=(0.05, -0.03, 0.02)):
    """T_AB: camera B relative to camera A (a small rotation about y and a translation, as a rig's second sensor)"""
    a = np.radians(deg)
    T = np.eye(4)
    T[:3, :3] = [[np.cos(a), 0, np.sin(a)], [0, 1, 0], [-np.sin(a), 0, np.cos(a)]]
    T[:3, 3] = t
    return T


def b_frame(T_room_a, Kb, T_AB, seed):
    """rgb, depth of camera B at the room pose of camera A composed with T_AB"""
    rgb, depth, _, _ = synth.render(T_room_a @ T_AB, Kb, noise_seed=seed)
    return rgb, depth


def make_ctx(K, capacity, **kw):
    kw.setdefault("time_delta", BIG)
    return capi.Context(capi.default_config(K.width, K.height, K.fx, K.fy, K.cx, K.cy, capacity=capacity, **kw))


def recipe(surfels, capacity, Kb, T, rgb, depth, time, weighting, td, conf, cutoff=CUTOFF, maxd=MAXD):
    """the stage calls in a context built for camera B, on an uploaded copy of the map; returns the map after clean"""
    c = make_ctx(Kb, capacity)
    try:
        c.map_upload(surfels)
        c.upload("RGB", rgb)
        c.upload("DEPTH_RAW", depth)
        ptr = lambda n: c.buffer_ptr(n)[0]
        c.preprocess_depth(ptr("DEPTH_RAW"), cutoff, ptr("DEPTH_FILTERED"), ptr("DEPTH_METRIC"), ptr("DEPTH_METRIC_FILTERED"))
        c.map_predict_indices(T, time, maxd, td)
        c.map_fuse(T, time, maxd, weighting)
        c.map_predict_indices(T, time, maxd, td)
        c.map_clean(T, time, conf, td, maxd)
        return c.map_download()
    finally:
        c.close()


def view_of(Kb, T, time, weighting=1.0, td=BIG, conf=10.0, cutoff=CUTOFF, maxd=MAXD):
    return capi.fuse_view(T, Kb.fx, Kb.fy, Kb.cx, Kb.cy, Kb.width, Kb.height, time, weighting=weighting, depth_cutoff=cutoff, max_depth=maxd,
                          conf_threshold=conf, time_delta=td)


CAP = 1_000_000


@pytest.fixture(scope="module")
def base(frames, K):
    """A 640x480 context after the 8 `frames`, its map and tick, and the room pose of frame 7 (camera A of the views)."""
    ctx = make_ctx(K, CAP)
    for i, (rgb, depth, _) in enumerate(frames):
        ctx.process_frame(rgb, depth, i)
    traj = synth.trajectory(len(frames), seed=42)
    yield dict(ctx=ctx, surfels=ctx.map_download(), tick=ctx.get_tick(), T_room=traj[-1], T0inv=np.linalg.inv(traj[0]))
    ctx.close()


def b_case(base, Kb, seed=5):
    T_AB = np.eye(4) if Kb is synth.K_DEFAULT else cam_offset()
    rgb, depth = b_frame(base["T_room"], Kb, T_AB, seed)
    return base["T0inv"] @ base["T_room"] @ T_AB, rgb, depth


def fused(base, Kb, T, rgb, depth, time, w, td, conf):
    ctx = base["ctx"]
    ctx.map_upload(base["surfels"])
    ctx.fuse_view(view_of(Kb, T, time, w, td, conf), rgb, depth)
    return ctx.map_download()


@pytest.mark.parametrize("param", sorted(PARAMS))
@pytest.mark.parametrize("cam", sorted(CAMERAS))
def test_recipe_bit_for_bit(base, cam, param):
    Kb = CAMERAS[cam]
    dt, w, td, conf = PARAMS[param]
    time = base["tick"] + dt
    T, rgb, depth = b_case(base, Kb)
    got = fused(base, Kb, T, rgb, depth, time, w, td, conf)
    ref = recipe(base["surfels"], CAP, Kb, T, rgb, depth, time, w, td, conf)
    assert_same(got, ref, f"{cam} {param}")
    n0 = len(base["surfels"])
    if param == "cull":  # clean culled the unstable surfels no frame has seen for > 20 ticks (the view's own are kept)
        assert (got[:, 6] < time).sum() < 0.9 * n0, ((got[:, 6] < time).sum(), n0)
    elif param == "tick":
        assert len(got) > n0 + 100 * min(1.0, Kb.width * Kb.height / 307200.0)  # the view added surfels
        assert (got[:n0] != base["surfels"]).any()  # and updated some


def oracle_chain(surfels, Kb, T, rgb, depth, time, w, td, conf, filt=None):
    if filt is None:
        filt = eo.bilateral(depth, CUTOFF)
    dm, dmf = eo.metric(depth, CUTOFF), eo.metric(filt, CUTOFF)
    idx = eo.predict_indices(surfels, T, time, MAXD, td, Kb)
    f, new = eo.fuse(surfels, T, time, rgb, dm, dmf, *idx, MAXD, w, Kb)
    idx2 = eo.predict_indices(f, T, time, MAXD, td, Kb)
    return f, new, eo.clean(f, new, T, time, *idx2, conf, td, MAXD, Kb)


@pytest.mark.parametrize("cam", ["320x240_offcentre", "424x240", "33x17", "1x1"])
def test_oracle_stages(base, cam):
    """bilateral, metric, predict_indices, fuse, predict_indices and clean of the CPU oracle at B's K on the same map, with the bars of
    test_gpu_sensor_sizes.py::test_fuse_then_clean: acosf (the normal-angle gate) and expf (the confidence) are the only non-IEEE-exact
    operations, so the new unstable surfels may differ by 2 in number, and at most 2 of the map's own surfels may differ beyond 2e-6
    relative; when the counts agree the new surfels are bit-exact but for their confidence (1e-6 relative). The view's surfels are told
    apart by their init time (`time`, later than any in the map). The bilateral filter flips 1 mm on <= 1e-4 of the pixels against
    libm's expf (test_gpu_sensor_sizes.py::test_preprocess_depth), so where a context can be built for B (32x32 and up) the oracle's
    fuse reads the product's filtered depth, checked against the oracle's with that bar; below, the oracle's own."""
    Kb = {**CAMERAS, **TINY}[cam]
    time = base["tick"]
    T, rgb, depth = b_case(base, Kb)
    got = fused(base, Kb, T, rgb, depth, time, 0.73, BIG, 10.0)
    filt = None
    if Kb.width >= 32 and Kb.height >= 32:
        c = make_ctx(Kb, 1000)
        try:
            c.upload("DEPTH_RAW", depth)
            ptr = lambda n: c.buffer_ptr(n)[0]
            c.preprocess_depth(ptr("DEPTH_RAW"), CUTOFF, ptr("DEPTH_FILTERED"), ptr("DEPTH_METRIC"), ptr("DEPTH_METRIC_FILTERED"))
            filt = c.download("DEPTH_FILTERED")
        finally:
            c.close()
        diff = np.abs(filt.astype(np.int32) - eo.bilateral(depth, CUTOFF).astype(np.int32))
        assert diff.max() <= 1 and (diff > 0).sum() <= max(8, 1e-4 * diff.size), (diff.max(), (diff > 0).sum())
    _, new, ref = oracle_chain(base["surfels"], Kb, T, rgb, depth, time, 0.73, BIG, 10.0, filt)
    old_g, old_r = got[got[:, 6] < time], ref[ref[:, 6] < time]
    new_g, new_r = got[got[:, 6] == time], ref[ref[:, 6] == time]
    assert len(old_g) + len(new_g) == len(got) and len(old_r) + len(new_r) == len(ref)
    assert abs(len(old_g) - len(old_r)) <= 2 and abs(len(new_g) - len(new_r)) <= 2, (len(old_g), len(old_r), len(new_g), len(new_r))
    if len(old_g) == len(old_r):
        close_rows = np.isclose(old_g, old_r, rtol=2e-6, atol=1e-7, equal_nan=True).all(axis=1)
        assert (~close_rows).sum() <= 2, f"{(~close_rows).sum()} of the map's surfels differ"
        assert ((old_g == old_r) | (np.isnan(old_g) & np.isnan(old_r))).all(axis=1).mean() > 0.9
    if len(new_g) == len(new_r):
        cols = [0, 1, 2, 4, 5, 6, 7, 8, 9, 10, 11]
        assert_same(new_g[:, cols], new_r[:, cols], cam)
        assert len(new_g) == 0 or rel_err(new_g[:, 3], new_r[:, 3]) < 1e-6
    if Kb.width >= 320:
        assert len(new) > 50 and len(new_g) > 50


FRAME_TEX = ("RGB", "DEPTH_RAW", "DEPTH_FILTERED", "DEPTH_METRIC", "DEPTH_METRIC_FILTERED", "RGBA", "INDEX", "VERT_CONF", "COLOR_TIME",
             "NORM_RAD", "IMAGE", "VERTEX", "NORMAL", "TIME", "OLD_IMAGE", "OLD_VERTEX", "OLD_NORMAL", "OLD_TIME", "SYNTH_DEPTH",
             "FILL_IMAGE", "FILL_VERTEX", "FILL_NORMAL")


def frame_state(ctx):
    return ([ctx.get_pose().tobytes(), ctx.get_tick(), ctx.dense_enough(), ctx.odom_stats().tobytes(), ctx.map_download_new().tobytes()]
            + [ctx.download(b).tobytes() for b in FRAME_TEX])


def test_frame_untouched(base, K):
    """A view changes the map and nothing else of the frame. A stage-API fuse at the frame's camera first leaves a non-empty unstable
    list for ef_map_download_new to report."""
    ctx = base["ctx"]
    ctx.map_upload(base["surfels"])
    T_A = base["T0inv"] @ base["T_room"]
    ctx.map_predict_indices(T_A, base["tick"], MAXD, BIG)
    ctx.map_fuse(T_A, base["tick"], MAXD, 1.0)
    before = frame_state(ctx)
    assert len(ctx.map_download_new()) > 100
    n0 = ctx.map_count()
    for cam in ("424x240", "1920x1080"):
        T, rgb, depth = b_case(base, CAMERAS[cam])
        ctx.fuse_view(view_of(CAMERAS[cam], T, base["tick"] - 1), rgb, depth)
    assert ctx.map_count() != n0
    after = frame_state(ctx)
    for k, (a, b) in enumerate(zip(before, after)):
        assert a == b, (["pose", "tick", "dense", "odom_stats", "new"] + list(FRAME_TEX))[k]


def test_resident_5M_1080p_matches_recipe():
    K = synth.K_DEFAULT
    traj = synth.trajectory(2, seed=42)
    room = synth.room_surfels(5_000_000, np.linalg.inv(traj[0]), view_depth=1.5, focal=K.fx)
    cap = 5_600_000
    Kb = CAMERAS["1920x1080"]
    T = np.linalg.inv(traj[0]) @ traj[1]
    rgb, depth, _, _ = synth.render(traj[1], Kb, noise_seed=11)
    ctx = make_ctx(K, cap)
    try:
        ctx.set_tick(2)  # as after a first frame
        ctx.map_upload(room)
        ctx.fuse_view(view_of(Kb, T, 1), rgb, depth)
        got = ctx.map_download()
    finally:
        ctx.close()
    ref = recipe(room, cap, Kb, T, rgb, depth, 1, 1.0, BIG, 10.0)
    assert len(got) > len(room)
    assert_same(got, ref, "5M 1080p")


@pytest.mark.parametrize("close_loops", [0, 2])
def test_continuation_matches_host_recipe(close_loops):
    """30 frames at 320x240 with a 424x240 frame of camera B (at the ground-truth pose of A composed with T_AB) fused after every 5th
    frame: poses and maps after every frame equal the run that composes the same thing on the host (download the map, the stage
    recipe in a camera-B context, upload it back). With close_loops = 2 the views go between ef_process_frame_device and
    ef_finish_frame while the look-ahead holds the next frame."""
    import torch

    KA, Kb, T_AB = _k(320, 240, 264.0), CAMERAS["424x240"], cam_offset()
    n, cap = 30, 400_000
    frames = list(synth.sequence(n, KA, seed=9, noise=True))
    traj = synth.trajectory(n, seed=9)
    T0inv = np.linalg.inv(traj[0])
    views = {i: (T0inv @ traj[i] @ T_AB, *b_frame(traj[i], Kb, T_AB, 100 + i)) for i in range(4, n, 5)}
    dev = [(torch.from_numpy(np.ascontiguousarray(r)).cuda(), torch.from_numpy(np.ascontiguousarray(d).view(np.int16)).cuda())
           for r, d, _ in frames]
    torch.cuda.synchronize()

    def run(composed):
        ctx = make_ctx(KA, cap, time_delta=200, close_loops=close_loops)
        out = []
        try:
            if close_loops == 2:
                ctx.prefetch_frame_device(dev[0][0].data_ptr(), dev[0][1].data_ptr())
            for i in range(n):
                if close_loops == 2:
                    ctx.process_frame_device(None, None, i)
                    if i + 1 < n:
                        ctx.prefetch_frame_device(dev[i + 1][0].data_ptr(), dev[i + 1][1].data_ptr())
                else:
                    ctx.process_frame(frames[i][0], frames[i][1], i)
                tick = i + 1  # the tick of this frame (ef_get_tick() - 1 after it)
                if i in views and not composed:
                    T, rgb, depth = views[i]
                    ctx.fuse_view(view_of(Kb, T, tick, td=200), rgb, depth)
                if close_loops == 2:
                    ctx.finish_frame()
                if i in views and composed:
                    T, rgb, depth = views[i]
                    ctx.map_upload(recipe(ctx.map_download(), cap, Kb, T, rgb, depth, tick, 1.0, 200, 10.0))
                out.append((ctx.get_pose(), ctx.map_download()))
        finally:
            ctx.close()
        return out

    a, b = run(False), run(True)
    for i, ((Ta, ma), (Tb, mb)) in enumerate(zip(a, b)):
        assert_same(Ta, Tb, f"pose {i}")
        assert_same(ma, mb, f"map {i}")
    assert len(a[-1][1]) > len(a[3][1])


def test_api_behaviour(base, K):
    import torch

    ctx = base["ctx"]
    Kb = CAMERAS["424x240"]
    T, rgb, depth = b_case(base, Kb)
    v = view_of(Kb, T, base["tick"] - 1)
    host = fused(base, Kb, T, rgb, depth, base["tick"] - 1, 1.0, BIG, 10.0)
    # deterministic
    assert_same(fused(base, Kb, T, rgb, depth, base["tick"] - 1, 1.0, BIG, 10.0), host, "repeat")
    # the device call gives the same map, and ef_map_count is right straight after it
    r = torch.from_numpy(np.ascontiguousarray(rgb)).cuda()
    d = torch.from_numpy(np.ascontiguousarray(depth).view(np.int16)).cuda()
    torch.cuda.synchronize()
    ctx.map_upload(base["surfels"])
    ctx.fuse_view_device(v, r.data_ptr(), d.data_ptr())
    assert ctx.map_count() == len(host)
    assert_same(ctx.map_download(), host, "device")
    # EF_EINVAL for each bad field and NULL inputs; the map is left as it is
    fields = [("width", 0), ("width", 16385), ("height", 0), ("height", 16385), ("fx", 0.0), ("fy", 0.0), ("fx", float("nan")),
              ("fy", float("inf")), ("cx", float("nan")), ("cy", float("-inf")), ("depth_cutoff", 0.0), ("depth_cutoff", -1.0),
              ("depth_cutoff", float("nan")), ("max_depth", 0.0), ("max_depth", float("inf")), ("weighting", -0.5),
              ("weighting", float("nan")), ("weighting", float("inf")), ("conf_threshold", float("nan")), ("time", -1), ("time_delta", -1)]
    bads = []
    for f, val in fields:
        b = view_of(Kb, T, base["tick"] - 1)
        setattr(b, f, val)
        bads.append(b)
    for i in (0, 5, 11, 15):
        b = view_of(Kb, T, base["tick"] - 1)
        b.T_wc[i] = float("nan") if i % 2 else float("inf")
        bads.append(b)
    L, C = capi.lib(), capi.C
    hr, hd = capi._p(np.ascontiguousarray(rgb)), capi._p(np.ascontiguousarray(depth))
    dr, dd = C.c_void_p(r.data_ptr()), C.c_void_p(d.data_ptr())
    for b in bads:
        assert L.ef_map_fuse_view(ctx.h_ctx, C.byref(b), hr, hd) == -1, [(f, getattr(b, f)) for f, _ in b._fields_ if f != "T_wc"]
        assert L.ef_map_fuse_view_device(ctx.h_ctx, C.byref(b), dr, dd) == -1
    assert L.ef_map_fuse_view(ctx.h_ctx, C.byref(v), None, hd) == -1
    assert L.ef_map_fuse_view(ctx.h_ctx, C.byref(v), hr, None) == -1
    assert L.ef_map_fuse_view_device(ctx.h_ctx, C.byref(v), None, dd) == -1
    assert L.ef_map_fuse_view_device(ctx.h_ctx, C.byref(v), dr, C.c_void_p(d.data_ptr() + 1)) == -1
    assert L.ef_map_fuse_view(ctx.h_ctx, None, hr, hd) == -1
    assert_same(ctx.map_download(), host, "after rejected calls")


def test_state_rules(K, frames):
    """EF_ESTATE before the first frame and between ef_process_frame_begin and _end; allowed after ef_process_frame_device with the
    next frame staged, where ef_map_count after ef_finish_frame includes the view's surfels."""
    import torch

    Kb = CAMERAS["424x240"]
    rgb_b, depth_b = b_frame(synth.trajectory(3, seed=42)[1], Kb, cam_offset(), 3)
    ctx = make_ctx(K, CAP)
    L, C = capi.lib(), capi.C
    try:
        v = view_of(Kb, np.eye(4), 1)
        hr, hd = capi._p(np.ascontiguousarray(rgb_b)), capi._p(np.ascontiguousarray(depth_b))
        assert L.ef_map_fuse_view(ctx.h_ctx, C.byref(v), hr, hd) == -3
        ctx.process_frame(frames[0][0], frames[0][1], 0)
        ctx.process_frame_begin(frames[1][0], frames[1][1], 1)
        assert L.ef_map_fuse_view(ctx.h_ctx, C.byref(v), hr, hd) == -3
        ctx.process_frame_end()
        # after ef_process_frame_device, with frame 3 staged: the view fuses into the map frame 2 leaves
        dev = [torch.from_numpy(np.ascontiguousarray(a)).cuda() for a in (frames[2][0], frames[2][1].view(np.int16), frames[3][0],
                                                                         frames[3][1].view(np.int16), rgb_b, depth_b.view(np.int16))]
        torch.cuda.synchronize()
        ctx.process_frame_device(dev[0].data_ptr(), dev[1].data_ptr(), 2)
        ctx.prefetch_frame_device(dev[2].data_ptr(), dev[3].data_ptr())
        ctx.fuse_view_device(view_of(Kb, frames[2][2] @ cam_offset(), 3), dev[4].data_ptr(), dev[5].data_ptr())
        ctx.finish_frame()
        n = ctx.map_count()
        assert n == len(ctx.map_download())
        ctx.process_frame(None, None, 3)  # the staged frame is intact
    finally:
        ctx.close()


def test_interleaved_with_model_views_and_renders(base):
    """Fuse views of different sizes, model views and renders interleaved on one context give the same maps as each fuse view alone
    on a fresh context holding the same map."""
    ctx, tick = base["ctx"], base["tick"]
    seq = ["1920x1080", "424x240", "1280x720", "320x240_offcentre"]
    T_A = base["T0inv"] @ base["T_room"]
    ctx.map_upload(base["surfels"])
    maps = []
    for k, cam in enumerate(seq):
        Kb = CAMERAS[cam]
        T, rgb, depth = b_case(base, Kb, seed=20 + k)
        before = ctx.map_download()
        ctx.fuse_view(view_of(Kb, T, tick - 1 + k), rgb, depth)
        maps.append((before, Kb, T, rgb, depth, tick - 1 + k, ctx.map_download()))
        Kv = CAMERAS[seq[-1 - k]]
        ctx.predict_view(capi.model_view(T_A, Kv.fx, Kv.fy, Kv.cx, Kv.cy, Kv.width, Kv.height, MAXD, 1.0, tick, tick, BIG))
        ctx.render(capi.camera_view(T_A, Kv.fx, Kv.fy, Kv.cx, Kv.cy, Kv.width, Kv.height, threshold=1.0))
    K = synth.K_DEFAULT
    for before, Kb, T, rgb, depth, time, got in maps:
        fresh = make_ctx(K, CAP)
        try:
            fresh.set_tick(2)
            fresh.map_upload(before)
            fresh.fuse_view(view_of(Kb, T, time), rgb, depth)
            assert_same(got, fresh.map_download(), f"{Kb.width}x{Kb.height}")
        finally:
            fresh.close()
