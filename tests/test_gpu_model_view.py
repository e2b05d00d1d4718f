"""ef_map_predict_view / ef_map_predict_view_device on the GPU: combinedPredict at the frame's own camera equals the frame's raycast,
at any camera it equals the CPU oracle bit for bit and the reference's shaders within the splat tolerances (tests/golden/ref_view_*.npz),
it leaves every piece of frame state untouched, shares the render's z-buffer, and validates its input."""
import itertools

import numpy as np
import pytest

import test_view_golden as tv
from test_gpu_configs import loop_state  # noqa: F401  (fixture)
from util import assert_same

from elasticfusion_b200 import capi, synth
from oracle import ef_oracle as eo

pytestmark = pytest.mark.gpu
MAXD, BIG = 20.0, 2147483647 // 2
NAMES = ("image", "vertex", "normal", "time")
FRAME_BUFS = {0: ("IMAGE", "VERTEX", "NORMAL", "TIME"), 1: ("OLD_IMAGE", "OLD_VERTEX", "OLD_NORMAL", "OLD_TIME")}


def make_ctx(K, capacity=500_000, **kw):
    kw.setdefault("time_delta", BIG)
    return capi.Context(capi.default_config(K.width, K.height, K.fx, K.fy, K.cx, K.cy, capacity=capacity, **kw))


def view_of(T, K, max_depth=MAXD, conf=10.0, time=1, max_time=1, td=BIG):
    return capi.model_view(T, K.fx, K.fy, K.cx, K.cy, K.width, K.height, max_depth, conf, time, max_time, td)


def oracle(surfels, T, K, max_depth=MAXD, conf=10.0, time=1, max_time=1, td=BIG):
    return eo.combined_predict(surfels, T, max_depth, conf, time, max_time, td, K)


def check_oracle(ctx, surfels, T, K, label, **kw):
    got = ctx.predict_view(view_of(T, K, **kw))
    ref = oracle(surfels, T, K, **kw)
    for n, r in zip(NAMES, ref):
        assert_same(got[n], r, f"{label} {n}")
    return got


@pytest.fixture(scope="module")
def frames_ctx(frames, K):
    """A context after the 8 `frames` at 640x480, its map, pose and tick, and a confidence threshold that keeps the upper 60 % of the
    surfels (after a few frames no surfel has reached the reference's default of 10)."""
    ctx = make_ctx(K, capacity=1_000_000)
    for i, (rgb, depth, _) in enumerate(frames):
        ctx.process_frame(rgb, depth, i)
    surfels = ctx.map_download()
    yield ctx, surfels, ctx.get_pose(), ctx.get_tick(), float(np.percentile(surfels[:, 3], 40))
    ctx.close()


def test_frame_camera_equals_raycast(frames_ctx, K, loop_state):  # noqa: F811
    """At the context's own camera the view equals what ef_map_raycast mode 0 / 1 writes into IMAGE..TIME / OLD_*, byte for byte:
    on the map `frames` leave (ACTIVE) and on the loop-closure state of test_gpu_configs (ACTIVE and INACTIVE)."""
    ctx, _, T, tick, thr = frames_ctx
    cases = [(ctx, T, (MAXD, thr, tick, tick, BIG), 0, "frames active")]
    s = loop_state
    lctx = make_ctx(s["K"], time_delta=s["td"])
    lctx.map_upload(s["m"])
    cases += [(lctx, s["T"], (MAXD, 10.0, s["tick"], s["tick"], s["td"]), 0, "loop active"),
              (lctx, s["T"], (MAXD, 10.0, 0, s["tick"] - s["td"], s["td"]), 1, "loop inactive")]
    try:
        for c, T_, args, mode, label in cases:
            got = c.predict_view(capi.model_view(T_, K.fx, K.fy, K.cx, K.cy, K.width, K.height, *args))
            c.map_raycast(T_, *args, mode)
            assert (got["vertex"][..., 2] > 0).mean() > 0.3, label
            for n, b in zip(NAMES, FRAME_BUFS[mode]):
                assert_same(got[n], c.download(b), f"{label} {n}")
    finally:
        lctx.close()


def away(T):
    """the same camera turned around its y axis"""
    R = np.diag([-1.0, 1.0, -1.0, 1.0])
    return T @ R


CASES = {
    "1x1": dict(K=synth.Intrinsics(1, 1, 1.0, 1.0, 0.5, 0.5)),
    "17x13": dict(K=synth.Intrinsics(17, 13, 14.0, 14.0, 8.5, 6.5)),
    "160x120": dict(K=synth.Intrinsics(160, 120, 132.0, 132.0, 80.0, 60.0)),
    "1920x1080": dict(K=synth.Intrinsics(1920, 1080, 1188.0, 1188.0, 960.0, 540.0)),
    "fx_ne_fy": dict(K=synth.Intrinsics(400, 300, 420.0, 300.0, 200.0, 150.0)),
    "pp_off_centre": dict(K=synth.Intrinsics(320, 240, 264.0, 264.0, 60.0, 200.0)),
    "pp_outside": dict(K=synth.Intrinsics(320, 240, 264.0, 264.0, -80.0, 300.0)),
    "small_max_depth": dict(K=synth.Intrinsics(320, 240, 264.0, 264.0, 160.0, 120.0), max_depth="median"),
    "finite_window": dict(K=synth.Intrinsics(320, 240, 264.0, 264.0, 160.0, 120.0), window=True),
}


@pytest.mark.parametrize("case", sorted(CASES))
def test_any_camera_matches_oracle(frames_ctx, case):
    ctx, surfels, T, tick, thr = frames_ctx
    c = CASES[case]
    kw = dict(time=tick, max_time=tick, td=BIG, conf=thr)
    if c.get("window"):
        kw = dict(time=tick, max_time=tick - 2, td=3, conf=thr)  # last seen in [tick - 3, tick - 2]
    if "max_depth" in c:  # the median depth of the map in front of the camera: about half of what is in view is cut
        z = (surfels[:, :3].astype(np.float64) - T[:3, 3]) @ T[:3, 2]
        kw["max_depth"] = float(np.median(z[z > 0]))
    got = check_oracle(ctx, surfels, T, c["K"], case, **kw)
    if c["K"].width >= 17:
        assert (got["vertex"][..., 2] > 0).mean() > 0.01, case


def test_views_from_outside_and_facing_away_are_empty(frames_ctx, K):
    ctx, surfels, T, tick, thr = frames_ctx
    outside = T.copy()
    outside[:3, 3] -= 50.0 * T[:3, 2]  # 50 m behind the camera, the room beyond max_depth
    for label, T_ in (("outside", outside), ("away", away(T))):
        got = check_oracle(ctx, surfels, T_, K, label, conf=thr, time=tick, max_time=tick)
        for n in NAMES:
            assert not got[n].any(), (label, n)


@pytest.mark.parametrize("name", sorted(tv.CAMERAS))
def test_product_matches_reference_view(name):
    K, vs = tv.load_fixture(name)
    surfels = tv.load_map()
    ctx = make_ctx(tv.CAMERAS["320x240"], capacity=100_000)
    ctx.map_upload(surfels)

    def predict(K, v):
        out = ctx.predict_view(capi.model_view(v["T"], K.fx, K.fy, K.cx, K.cy, K.width, K.height, v["max_depth"], v["conf_threshold"], v["time"],
                                               v["max_time"], v["time_delta"]))
        return tuple(out[n] for n in NAMES)

    try:
        tv.check_against(K, vs, predict, "product " + name)
    finally:
        ctx.close()


def test_resident_5M_1080p_matches_oracle():
    K = synth.K_DEFAULT
    room = synth.room_surfels(5_000_000, np.linalg.inv(synth.trajectory(1, seed=42)[0]), view_depth=1.5, focal=K.fx)
    ctx = make_ctx(K, capacity=5_600_000)
    ctx.map_upload(room)
    traj = synth.trajectory(2, seed=42)
    T = np.linalg.inv(traj[0]) @ traj[1]
    try:
        got = check_oracle(ctx, room, T, synth.Intrinsics(1920, 1080, 1188.0, 1188.0, 960.0, 540.0), "5M 1080p", time=1, max_time=1)
        assert (got["vertex"][..., 2] > 0).mean() > 0.9
    finally:
        ctx.close()


def frame_state(ctx):
    return ([ctx.get_pose().tobytes(), ctx.map_download().tobytes(), ctx.map_count(), ctx.dense_enough()]
            + [ctx.download(b).tobytes() for b in ("INDEX", "VERT_CONF", "COLOR_TIME", "NORM_RAD", "IMAGE", "VERTEX", "NORMAL", "TIME",
                                                   "FILL_IMAGE", "FILL_VERTEX", "FILL_NORMAL")])


@pytest.mark.parametrize("close_loops", [2, 0])
def test_view_between_frames_changes_nothing(close_loops):
    """30 frames with a view at another camera after every frame (with close_loops = 2: between ef_process_frame_device and
    ef_finish_frame, the next frame staged by the look-ahead) leave poses, map, index textures, the predicted model, the fill-in and
    denseEnough byte-identical to the same run without views."""
    import torch

    K = synth.Intrinsics(320, 240, 264.0, 264.0, 160.0, 120.0)
    frames = list(synth.sequence(30, K, seed=9, noise=True))
    dev = [(torch.from_numpy(np.ascontiguousarray(r)).cuda(), torch.from_numpy(np.ascontiguousarray(d).view(np.int16)).cuda()) for r, d, _ in frames]
    bufs = [torch.zeros(640 * 480 * b, dtype=torch.uint8, device="cuda") for b in (4, 16, 16, 2)]
    torch.cuda.synchronize()

    def run(view):
        ctx = capi.Context(capi.default_config(K.width, K.height, K.fx, K.fy, K.cx, K.cy, capacity=400_000, close_loops=close_loops))
        states = []
        if close_loops == 2:
            ctx.prefetch_frame_device(dev[0][0].data_ptr(), dev[0][1].data_ptr())
        for i in range(len(frames)):
            if close_loops == 2:
                ctx.process_frame_device(None, None, i)
                if i + 1 < len(frames):
                    ctx.prefetch_frame_device(dev[i + 1][0].data_ptr(), dev[i + 1][1].data_ptr())
            else:
                ctx.process_frame(frames[i][0], frames[i][1], i)
            if view:
                T = frames[i][2]
                if i % 2:
                    ctx.predict_view(capi.model_view(T, 300.0, 250.0, 100.0, 90.0, 200, 150, 3.0, 1.0, i + 1, i + 1, 200))
                else:
                    v = capi.model_view(T, 2 * K.fx, 2 * K.fy, 2 * K.cx, 2 * K.cy, 640, 480, MAXD, 10.0, 0, i - 5, 5)
                    ctx.predict_view_device(v, *(b.data_ptr() for b in bufs))
            if close_loops == 2:
                ctx.finish_frame()
            states.append(frame_state(ctx))
        ctx.close()
        return states

    plain, viewed = run(False), run(True)
    for i, (a, b) in enumerate(zip(plain, viewed)):
        for k, (x, y) in enumerate(zip(a, b)):
            assert x == y, (i, k)


def test_shared_zbuffer_interleaved_with_render(frames_ctx):
    """Renders and views at different sizes (large, small, then large again) share the off-frame z-buffer: each output equals the
    same call made alone on a fresh context."""
    ctx, surfels, T, tick, thr = frames_ctx
    big, small = synth.Intrinsics(1280, 960, 1056.0, 1056.0, 640.0, 480.0), synth.Intrinsics(200, 150, 165.0, 165.0, 100.0, 75.0)
    calls = [("view", big), ("render", small), ("view", small), ("render", big), ("view", big), ("view", small), ("render", small)]

    def call(c, kind, Kc):
        if kind == "render":
            return [c.render(capi.camera_view(T, Kc.fx, Kc.fy, Kc.cx, Kc.cy, Kc.width, Kc.height, threshold=thr))]
        out = c.predict_view(view_of(T, Kc, conf=thr, time=tick, max_time=tick))
        return [out[n] for n in NAMES]

    mixed = [call(ctx, kind, Kc) for kind, Kc in calls]
    for (kind, Kc), got in zip(calls, mixed):
        fresh = make_ctx(synth.K_DEFAULT, capacity=len(surfels) + 1000)
        fresh.map_upload(surfels)
        alone = call(fresh, kind, Kc)
        fresh.close()
        for a, b in zip(got, alone):
            assert_same(a, b, f"{kind} {Kc.width}x{Kc.height}")


def test_api_behaviour(frames_ctx, K):
    import torch

    ctx, _, T, tick, thr = frames_ctx
    Kv = synth.Intrinsics(300, 200, 280.0, 250.0, 140.0, 110.0)
    v = view_of(T, Kv, conf=thr, time=tick, max_time=tick)
    full = ctx.predict_view(v)
    # documented shapes and dtypes
    assert full["image"].shape == (200, 300, 4) and full["image"].dtype == np.uint8
    assert full["vertex"].shape == (200, 300, 4) and full["vertex"].dtype == np.float32
    assert full["normal"].shape == (200, 300, 4) and full["normal"].dtype == np.float32
    assert full["time"].shape == (200, 300) and full["time"].dtype == np.uint16
    assert (full["vertex"][..., 2] > 0).mean() > 0.3
    # deterministic
    again = ctx.predict_view(v)
    for n in NAMES:
        assert_same(again[n], full[n], n)
    # every subset of outputs gives the same images, on the host and on the device
    for k in range(1, 5):
        for subset in itertools.combinations(NAMES, k):
            part = ctx.predict_view(v, subset)
            assert sorted(part) == sorted(subset)
            for n in subset:
                assert_same(part[n], full[n], f"host {subset} {n}")
            bufs = {n: torch.zeros(full[n].nbytes, dtype=torch.uint8, device="cuda") for n in subset}
            ctx.predict_view_device(v, **{n: b.data_ptr() for n, b in bufs.items()})
            ctx.sync()
            for n, b in bufs.items():
                assert_same(b.cpu().numpy().view(full[n].dtype).reshape(full[n].shape), full[n], f"device {subset} {n}")
    # EF_EINVAL for each bad field and for all-NULL outputs
    host = {n: np.zeros_like(a) for n, a in full.items()}
    dbuf = {n: torch.zeros(a.nbytes, dtype=torch.uint8, device="cuda") for n, a in full.items()}
    fields = [("width", 0), ("width", 16385), ("height", 0), ("height", 16385), ("fx", 0.0), ("fy", 0.0), ("fx", float("nan")),
              ("fy", float("inf")), ("cx", float("nan")), ("cy", float("-inf")), ("max_depth", 0.0), ("max_depth", -1.0),
              ("max_depth", float("inf")), ("max_depth", float("nan")), ("conf_threshold", float("nan"))]
    bads = []
    for f, val in fields:
        b = view_of(T, Kv, conf=thr, time=tick, max_time=tick)
        setattr(b, f, val)
        bads.append(b)
    for i in (0, 5, 11, 15):
        b = view_of(T, Kv, conf=thr, time=tick, max_time=tick)
        b.T_wc[i] = float("nan") if i % 2 else float("inf")
        bads.append(b)
    L = capi.lib()
    hp = [capi._p(host[n]) for n in NAMES]
    dp = [capi.C.c_void_p(dbuf[n].data_ptr()) for n in NAMES]
    for b in bads:
        assert L.ef_map_predict_view(ctx.h_ctx, capi.C.byref(b), *hp) == -1, [(f, getattr(b, f)) for f, _ in b._fields_ if f != "T_wc"]
        assert L.ef_map_predict_view_device(ctx.h_ctx, capi.C.byref(b), *dp) == -1
    assert L.ef_map_predict_view(ctx.h_ctx, capi.C.byref(v), None, None, None, None) == -1
    assert L.ef_map_predict_view_device(ctx.h_ctx, capi.C.byref(v), None, None, None, None) == -1
    assert L.ef_map_predict_view(ctx.h_ctx, None, *hp) == -1
    # and the context is still usable
    after = ctx.predict_view(v)
    for n in NAMES:
        assert_same(after[n], full[n], n)
