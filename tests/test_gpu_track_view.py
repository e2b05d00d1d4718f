"""ef_track_view / ef_track_view_device on the GPU: an RGB-D frame of another camera tracked against the map from a pose guess. The result
equals, byte for byte, what a context built for that camera gives with the stage calls (predict the view, initICPModel, initRGBModel,
preprocess, initICP, initRGB, track without SO(3)); it agrees with the CPU oracle's tracker with the bars of test_gpu_sensor_sizes.py;
it recovers ground-truth poses as well as the oracle does; and it leaves every frame output untouched."""
import numpy as np
import pytest

from util import assert_same, rel_err, rgba_of

from elasticfusion_b200 import capi, synth
from oracle import ef_oracle as eo

pytestmark = pytest.mark.gpu
MAXD, BIG, CUTOFF = 20.0, 2147483647 // 2, 3.0
CAP = 1_000_000
EF_EINVAL, EF_ESTATE = -1, -3
# the maps below come from at most a dozen frames, where few surfels reach the frame's confidence of 10 (the frame tracks them through
# the fill-in); the views predict the surfels seen at least twice or so
CONF = 2.0


def _k(w, h, f, cx=None, cy=None, fy=None):
    return synth.Intrinsics(w, h, f, f if fy is None else fy, w / 2 if cx is None else cx, h / 2 if cy is None else cy)


# camera B of each case; "own" is the context's camera (K_DEFAULT)
CAMERAS = {
    "own": synth.K_DEFAULT,
    "320x240_offcentre": _k(320, 240, 280.0, 130.0, 140.0, fy=250.0),
    "424x240": _k(424, 240, 305.0),
    "1280x720": _k(1280, 720, 915.0),
    "1920x1080": _k(1920, 1080, 1188.0),
    "330x246": _k(330, 246, 290.0, 161.5, 125.0),  # not a multiple of 4 on either side
}
# tracker settings of each case: (rgb_only, icp_weight, pyramid, fast_odom)
MODES = {"default": (False, 10.0, True, False), "rgb_only": (True, 10.0, True, False), "icp_only": (False, 100.0, True, False),
         "fast_odom": (False, 10.0, True, True), "no_pyramid": (False, 10.0, False, False)}
CASES = {f"{m}-1": (m, 1.0) for m in MODES} | {"default-0": ("default", 0.0), "default-3": ("default", 3.0)}


def cam_offset(deg=8.0, t=(0.05, -0.03, 0.02)):
    """T_AB: camera B relative to camera A (a small rotation about y and a translation, as a rig's second sensor)"""
    a = np.radians(deg)
    T = np.eye(4)
    T[:3, :3] = [[np.cos(a), 0, np.sin(a)], [0, 1, 0], [-np.sin(a), 0, np.cos(a)]]
    T[:3, 3] = t
    return T


def perturb(T, d):
    """T moved by d cm along (1, -1, 1)/sqrt(3) and turned by d degrees about (1, 2, -1)/sqrt(6)"""
    ax = np.array([1.0, 2.0, -1.0]) / np.sqrt(6.0)
    a = np.radians(d)
    Kx = np.array([[0, -ax[2], ax[1]], [ax[2], 0, -ax[0]], [-ax[1], ax[0], 0]])
    D = np.eye(4)
    D[:3, :3] = np.eye(3) + np.sin(a) * Kx + (1 - np.cos(a)) * Kx @ Kx
    D[:3, 3] = 0.01 * d * np.array([1.0, -1.0, 1.0]) / np.sqrt(3.0)
    return T @ D


def b_frame(T_room_a, Kb, T_AB, seed):
    """rgb, depth of camera B at the room pose of camera A composed with T_AB"""
    rgb, depth, _, _ = synth.render(T_room_a @ T_AB, Kb, noise_seed=seed)
    return rgb, depth


def make_ctx(K, capacity=CAP, **kw):
    kw.setdefault("time_delta", BIG)
    return capi.Context(capi.default_config(K.width, K.height, K.fx, K.fy, K.cx, K.cy, capacity=capacity, **kw))


def view_of(Kb, guess, time, mode="default", td=BIG, conf=CONF):
    rgb_only, icp_weight, pyramid, fast_odom = MODES[mode]
    return capi.track_view(guess, Kb.fx, Kb.fy, Kb.cx, Kb.cy, Kb.width, Kb.height, time, time_delta=td, conf_threshold=conf,
                           icp_weight=icp_weight, rgb_only=rgb_only, pyramid=pyramid, fast_odom=fast_odom)


def recipe(surfels, Kb, view, rgb, depth):
    """the stage calls in a fresh context built for camera B, on an uploaded copy of the map: (T, stats, covariance, trace, image)"""
    import torch

    m = view.model
    guess = np.array(m.T_wc[:]).reshape(4, 4)
    c = make_ctx(Kb)
    try:
        c.map_upload(surfels)
        n = Kb.width * Kb.height
        img = torch.zeros(n * 4, dtype=torch.uint8, device="cuda")
        vtx = torch.zeros(n * 4, dtype=torch.float32, device="cuda")
        nrm = torch.zeros(n * 4, dtype=torch.float32, device="cuda")
        torch.cuda.synchronize()
        c.predict_view_device(m, image=img.data_ptr(), vertex=vtx.data_ptr(), normal=nrm.data_ptr())
        c.sync()
        c.odom_init_icp_model(vtx.data_ptr(), nrm.data_ptr(), guess)
        c.odom_init_rgb_model(img.data_ptr())
        c.upload("DEPTH_RAW", depth)
        c.upload("RGBA", rgba_of(rgb))
        ptr = lambda name: c.buffer_ptr(name)[0]
        c.preprocess_depth(ptr("DEPTH_RAW"), view.depth_cutoff, ptr("DEPTH_FILTERED"), 0, 0)
        c.odom_init_icp_depth(ptr("DEPTH_FILTERED"), m.max_depth)
        c.odom_init_rgb(ptr("RGBA"))
        T, trace = c.odom_track(guess, rgb_only=bool(view.rgb_only), icp_weight=view.icp_weight, pyramid=bool(view.pyramid),
                                fast_odom=bool(view.fast_odom), so3=False)
        image = img.cpu().numpy().reshape(Kb.height, Kb.width, 4)
        return T, c.odom_stats(), c.odom_covariance(), trace, image
    finally:
        c.close()


def assert_bytes(a, b, what):
    """byte-identical records (stats, trace; neither has padding), naming the first field that differs"""
    a, b = np.asarray(a), np.asarray(b)
    assert a.shape == b.shape, (what, a.shape, b.shape)
    if a.tobytes() != b.tobytes():
        bad = [n for n in a.dtype.names if a[n].tobytes() != b[n].tobytes()]
        raise AssertionError(f"{what}: fields {bad} differ")


def assert_result_same(got, ref, what):
    (Tg, sg, cg, dg, trg), (Tr, sr, cr, trr, image) = got, ref
    assert_same(Tg, Tr, f"{what} pose")
    assert_bytes(sg, sr, f"{what} stats")
    assert_same(cg, cr, f"{what} covariance")
    assert_bytes(trg, trr, f"{what} trace")
    assert dg == bool(eo.dense_enough(image)), what


@pytest.fixture(scope="module")
def base(frames, K):
    """A 640x480 context after the 8 `frames`, its map and tick, and the room pose of frame 7 (camera A of the views)."""
    ctx = make_ctx(K)
    for i, (rgb, depth, _) in enumerate(frames):
        ctx.process_frame(rgb, depth, i)
    traj = synth.trajectory(len(frames), seed=42)
    yield dict(ctx=ctx, surfels=ctx.map_download(), tick=ctx.get_tick(), T_room=traj[-1], T0inv=np.linalg.inv(traj[0]))
    ctx.close()


def b_case(base, Kb, seed=5):
    """(true pose of camera B in the map, rgb, depth)"""
    T_AB = np.eye(4) if Kb is synth.K_DEFAULT else cam_offset()
    rgb, depth = b_frame(base["T_room"], Kb, T_AB, seed)
    return base["T0inv"] @ base["T_room"] @ T_AB, rgb, depth


@pytest.mark.parametrize("case", sorted(CASES))
@pytest.mark.parametrize("cam", sorted(CAMERAS))
def test_recipe_bit_for_bit(base, cam, case):
    Kb = CAMERAS[cam]
    mode, d = CASES[case]
    T, rgb, depth = b_case(base, Kb)
    v = view_of(Kb, perturb(T, d), base["tick"], mode)
    ctx = base["ctx"]
    ctx.map_upload(base["surfels"])
    got = ctx.track_view(v, rgb, depth, max_trace=48)
    assert_result_same(got, recipe(base["surfels"], Kb, v, rgb, depth), f"{cam} {case}")
    assert len(got[4]) == {"fast_odom": 12, "no_pyramid": 10}.get(mode, 19) or mode == "rgb_only"
    assert got[1]["lastICPCount"] > 0 or mode == "rgb_only"


@pytest.mark.parametrize("where", ["empty_map", "facing_away"])
def test_nothing_seen(base, where):
    """An empty map, and a view that sees no surfel: the call succeeds with the recipe's result. No term is valid, every system is
    zero, the pose is the guess as k_gn_finish rebuilds it from its float rotation (within 1e-6), lastICPError is 0/0 and the
    covariance, the inverse of a zero lastA, is not finite."""
    Kb = CAMERAS["424x240"]
    T, rgb, depth = b_case(base, Kb)
    surfels = base["surfels"][:0] if where == "empty_map" else base["surfels"]
    guess = T.copy()
    if where == "facing_away":  # turned 180 degrees about the camera's y axis: every surfel of the map is behind it
        guess = T @ np.diag([-1.0, 1.0, -1.0, 1.0])
    v = view_of(Kb, guess, base["tick"])
    ctx = base["ctx"]
    ctx.map_upload(surfels)
    got = ctx.track_view(v, rgb, depth, max_trace=48)
    assert_result_same(got, recipe(surfels, Kb, v, rgb, depth), where)
    Tg, st, cov, dense, trace = got
    print(where, "pose - guess", np.abs(Tg - guess).max(), "stats", {k: st[k] for k in ("lastICPCount", "lastRGBCount", "lastICPError",
          "lastRGBError")}, "lastA", np.abs(st["lastA"]).max(), "cov finite", np.isfinite(cov).all(), "dense", dense)
    assert not dense
    assert np.abs(Tg - guess).max() < 1e-6
    assert st["lastICPCount"] == 0 and st["lastRGBCount"] == 0 and np.isnan(st["lastICPError"])
    assert not np.abs(st["lastA"]).any() and not np.isfinite(cov).all()


@pytest.fixture(scope="module")
def oracle_sizes():
    from test_gpu_sensor_sizes import compare_trace_with_oracle, perturbed_pixels, small_frame_factor

    return compare_trace_with_oracle, perturbed_pixels, small_frame_factor


def oracle_track(Kb, guess, image, vertex, normal, filt, rgb, **cfg):
    od = eo.Odometry(Kb.width, Kb.height, Kb.cx, Kb.cy, Kb.fx, Kb.fy)
    od.init_icp_model(vertex, normal, guess)
    od.init_rgb_model(image)
    od.init_icp_depth(filt, MAXD)
    od.init_rgb(rgba_of(rgb))
    return od.track(guess, so3=False, **cfg)


def product_filtered(Kb, depth):
    c = make_ctx(Kb, 1000)
    try:
        c.upload("DEPTH_RAW", depth)
        p = lambda n: c.buffer_ptr(n)[0]
        c.preprocess_depth(p("DEPTH_RAW"), CUTOFF, p("DEPTH_FILTERED"), 0, 0)
        return c.download("DEPTH_FILTERED")
    finally:
        c.close()


@pytest.mark.parametrize("cam", ["320x240_offcentre", "424x240"])
def test_oracle_tracker(base, cam, oracle_sizes):
    """The CPU oracle's tracker on the view's own prediction and the live frame (its filtered depth taken from the product, as in
    test_gpu_fuse_view.py: the bilateral filter flips 1 mm on <= 1e-4 of the pixels against libm's expf), with the bars of
    test_gpu_sensor_sizes.py::test_full_track_matches_oracle: below 640x480 level 0 is held to twice the oracle's own sensitivity to a
    1 mm change of one raw depth pixel (filtered by the oracle), never looser than 50x the 640x480 bar. The final pose is held there
    to that ceiling (5e-4): eight perturbed pixels of one view are too few to estimate the pose's sensitivity (they move it by < 5e-6
    here, against 2.4e-4 measured at 424x240 in test_gpu_sensor_sizes.py), while the product's pose, the sum of level-0 increments
    that each pass their bars, differs from the oracle's by 2.5e-5 at 424x240 (measured on an H100)."""
    compare, perturbed_pixels, small_frame_factor = oracle_sizes
    Kb = CAMERAS[cam]
    T, rgb, depth = b_case(base, Kb)
    guess = perturb(T, 1.0)
    v = view_of(Kb, guess, base["tick"])
    ctx = base["ctx"]
    ctx.map_upload(base["surfels"])
    Tp, _, _, _, trp = ctx.track_view(v, rgb, depth, max_trace=48)
    out = ctx.predict_view(v.model, outputs=("image", "vertex", "normal"))
    filt = product_filtered(Kb, depth)
    inputs = (Kb, guess, out["image"], out["vertex"], out["normal"])
    To, tro = oracle_track(*inputs, filt, rgb)
    bars = dict(result=2e-5, lastA=1e-3, icp=0, rgb=0, pose=1e-5)
    if small_frame_factor(Kb) > 1.0:
        s = dict(result=0.0, lastA=0.0, icp=0.0, rgb=0.0, pose=0.0)
        T0, tr0 = oracle_track(*inputs, eo.bilateral(depth, CUTOFF), rgb)
        ref = {int(t["iter"]): t for t in tr0 if t["level"] == 0}
        for y, x in perturbed_pixels(depth):
            d1 = depth.copy()
            d1[y, x] += 1
            T1, tr1 = oracle_track(*inputs, eo.bilateral(d1, CUTOFF), rgb)
            for t in tr1:
                if t["level"] != 0:
                    continue
                b = ref[int(t["iter"])]
                s["result"] = max(s["result"], float(np.abs(t["result"] - b["result"]).max()))
                s["lastA"] = max(s["lastA"], rel_err(t["lastA"], b["lastA"]))
                s["icp"] = max(s["icp"], float(abs(t["icp_residual"][1] - b["icp_residual"][1])))
                s["rgb"] = max(s["rgb"], float(abs(int(t["rgb_count"]) - int(b["rgb_count"]))))
            s["pose"] = max(s["pose"], float(np.abs(T1 - T0).max()))
        bars = dict(result=min(1e-3, max(2e-5, 2 * s["result"])), lastA=min(5e-2, max(1e-3, 2 * s["lastA"])), icp=2 * s["icp"],
                    rgb=2 * s["rgb"], pose=5e-4)
    compare(trp, tro, Tp, To, bars, cam)


def test_accuracy_against_ground_truth():
    """A map fused at ground-truth poses from 12 frames of the noisy sequence; camera-B frames at three other cameras tracked from
    guesses 2 and 4 cm / degrees off. The recovered pose is as close to the truth as the oracle tracker gets on the same inputs (its
    error plus the 1e-5 pose bar of the oracle comparison, plus 1e-4 where the two solves may part at level 0 below 640x480), and its
    rotation is closer than the guess's; both errors are printed. How close either gets is the map's and the frame's doing: a few
    walls seen from a short, slow trajectory leave translation weakly constrained, and from 4 cm off at 320x240 neither tracker gets
    nearer than the guess in translation (measured: 53.5 mm for both)."""
    K = synth.K_DEFAULT
    n = 12
    frames = list(synth.sequence(n, K, seed=17, noise=True))
    traj = synth.trajectory(n, seed=17)
    T0inv = np.linalg.inv(traj[0])
    ctx = make_ctx(K)
    try:
        for i, (rgb, depth, T) in enumerate(frames):
            ctx.process_frame(rgb, depth, i, T_wc=T)
        tick = ctx.get_tick()
        rows = []
        for cam, k, d in (("424x240", 9, 2.0), ("320x240_offcentre", 5, 4.0), ("1280x720", 11, 2.0)):
            Kb = CAMERAS[cam]
            rgb, depth = b_frame(traj[k], Kb, cam_offset(), 300 + k)
            T = T0inv @ traj[k] @ cam_offset()
            guess = perturb(T, d)
            v = view_of(Kb, guess, tick)
            Tp = ctx.track_view(v, rgb, depth)[0]
            out = ctx.predict_view(v.model, outputs=("image", "vertex", "normal"))
            To, _ = oracle_track(Kb, guess, out["image"], out["vertex"], out["normal"], product_filtered(Kb, depth), rgb)
            err = lambda A: (float(np.linalg.norm(A[:3, 3] - T[:3, 3])),
                             float(np.degrees(np.arccos(np.clip((np.trace(A[:3, :3].T @ T[:3, :3]) - 1) / 2, -1, 1)))))
            (tp, rp), (to, ro), (tg, rg) = err(Tp), err(To), err(guess)
            rows.append((cam, d, tg, rg, tp, rp, to, ro))
            print(f"{cam}: guess {tg * 100:.2f} cm {rg:.2f} deg -> product {tp * 1000:.3f} mm {rp:.4f} deg, oracle {to * 1000:.3f} mm "
                  f"{ro:.4f} deg")
            slack = 1e-5 + (1e-4 if Kb.width * Kb.height < 640 * 480 else 0.0)
            assert tp <= to + slack and rp <= ro + np.degrees(slack), rows[-1]
            assert rp < rg, rows[-1]
    finally:
        ctx.close()


FRAME_TEX = ("RGB", "DEPTH_RAW", "DEPTH_FILTERED", "DEPTH_METRIC", "DEPTH_METRIC_FILTERED", "RGBA", "INDEX", "VERT_CONF", "COLOR_TIME",
             "NORM_RAD", "IMAGE", "VERTEX", "NORMAL", "TIME", "OLD_IMAGE", "OLD_VERTEX", "OLD_NORMAL", "OLD_TIME", "SYNTH_DEPTH",
             "FILL_IMAGE", "FILL_VERTEX", "FILL_NORMAL")
ODOM_BUF = ("VMAP_CURR", "NMAP_CURR", "VMAP_G_PREV", "NMAP_G_PREV", "LAST_DEPTH", "NEXT_DEPTH", "LAST_IMAGE", "NEXT_IMAGE", "LAST_NEXT_IMAGE",
            "DIDX", "DIDY", "DEPTH_TMP", "CORRES")


def frame_state(ctx, close_loops):
    s = [ctx.get_pose().tobytes(), ctx.get_tick(), ctx.dense_enough(), ctx.map_download().tobytes()]
    s += [ctx.odom_stats(w).tobytes() for w in (0, 1)]
    s += [ctx.download(b).tobytes() for b in FRAME_TEX]
    s += [ctx.download(b, level=lv, which=w).tobytes() for w in (0, 1) for b in ODOM_BUF for lv in range(3)]
    s += [ctx.download("VMAPS_TMP", which=w).tobytes() for w in (0, 1)]
    if close_loops:
        info, src, dst, times = ctx.local_loop_result()
        s += [repr({k: np.asarray(v).tobytes() for k, v in info.items()}), src.tobytes(), dst.tobytes(), times.tobytes()]
    if close_loops == 2:
        info, graph = ctx.local_deform_result()
        s += [repr(info), graph.tobytes()]
    return s


@pytest.mark.parametrize("close_loops", [0, 2])
def test_frame_untouched(close_loops):
    """30 frames at 320x240 with a 424x240 track view after every frame: the frame's poses, map, every EF_BUF_* buffer (the pyramids of
    both trackers included), ef_odom_stats(0 / 1), ef_dense_enough and the loop-closure results equal the same run without views. With
    close_loops = 0 the views use the host call; with close_loops = 2 and the look-ahead they use the device call between
    ef_process_frame_device and ef_finish_frame, with the next frame staged."""
    import torch

    KA, Kb, T_AB = _k(320, 240, 264.0), CAMERAS["424x240"], cam_offset()
    n = 30
    frames = list(synth.sequence(n, KA, seed=9, noise=True))
    traj = synth.trajectory(n, seed=9)
    T0inv = np.linalg.inv(traj[0])
    views = {i: (T0inv @ traj[i] @ T_AB, *b_frame(traj[i], Kb, T_AB, 100 + i)) for i in range(0, n, 6)}
    dev = [(torch.from_numpy(np.ascontiguousarray(r)).cuda(), torch.from_numpy(np.ascontiguousarray(d).view(np.int16)).cuda())
           for r, d, _ in frames]
    vdev = {i: (torch.from_numpy(np.ascontiguousarray(r)).cuda(), torch.from_numpy(np.ascontiguousarray(d).view(np.int16)).cuda())
            for i, (_, r, d) in views.items()}
    out_dev = torch.zeros(capi.C.sizeof(capi.EfTrackResult), dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()

    def run(with_views):
        ctx = make_ctx(KA, 400_000, time_delta=200, close_loops=close_loops)
        states, results = [], []
        try:
            if close_loops == 2:
                ctx.prefetch_frame_device(dev[0][0].data_ptr(), dev[0][1].data_ptr())
            for i in range(n):
                j = max(k for k in views if k <= i)  # the camera-B frame nearest before this one
                T, rgb, depth = views[j]
                v = view_of(Kb, perturb(T, 1.0), i + 1, td=200)
                if close_loops == 2:
                    ctx.process_frame_device(None, None, i)
                    if i + 1 < n:
                        ctx.prefetch_frame_device(dev[i + 1][0].data_ptr(), dev[i + 1][1].data_ptr())
                    if with_views:
                        ctx.track_view_device(v, vdev[j][0].data_ptr(), vdev[j][1].data_ptr(), out_dev.data_ptr())
                    ctx.finish_frame()
                    if with_views:
                        ctx.sync()
                        results.append(capi.unpack_track_result(out_dev.cpu().numpy().tobytes()))
                else:
                    ctx.process_frame(frames[i][0], frames[i][1], i)
                    if with_views:
                        results.append(ctx.track_view(v, rgb, depth))
                states.append(frame_state(ctx, close_loops))
        finally:
            ctx.close()
        return states, results

    (a, res), (b, _) = run(True), run(False)
    names = ["pose", "tick", "dense", "map", "odom_stats 0", "odom_stats 1"] + list(FRAME_TEX)
    for i, (sa, sb) in enumerate(zip(a, b)):
        for k, (x, y) in enumerate(zip(sa, sb)):
            assert x == y, (i, names[k] if k < len(names) else k)
    assert len(res) == n and all(np.isfinite(r[0]).all() for r in res)


def test_determinism_host_device(base):
    import torch

    ctx = base["ctx"]
    Kb = CAMERAS["1280x720"]
    T, rgb, depth = b_case(base, Kb)
    v = view_of(Kb, perturb(T, 2.0), base["tick"])
    ctx.map_upload(base["surfels"])
    first = ctx.track_view(v, rgb, depth, max_trace=48)
    again = ctx.track_view(v, rgb, depth, max_trace=48)
    for k in (0, 2, 3):
        assert_same(np.asarray(first[k]), np.asarray(again[k]), f"repeat {k}")
    assert_bytes(first[1], again[1], "repeat stats")
    assert_bytes(first[4], again[4], "repeat trace")
    r = torch.from_numpy(np.ascontiguousarray(rgb)).cuda()
    d = torch.from_numpy(np.ascontiguousarray(depth).view(np.int16)).cuda()
    out = torch.zeros(capi.C.sizeof(capi.EfTrackResult), dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()
    ctx.track_view_device(v, r.data_ptr(), d.data_ptr(), out.data_ptr())
    ctx.sync()
    Td, sd, cd, dd = capi.unpack_track_result(out.cpu().numpy().tobytes())
    assert_same(Td, first[0], "device pose")
    assert_bytes(sd, first[1], "device stats")
    assert dd == first[3]
    # the device inverse is compiled without FMA contraction, like the host's x86-64 code, so the covariance agrees bit for bit; the
    # fall-back bar (1e-12 of its largest entry) would hold if a build contracted it
    dc = np.abs(cd - first[2]).max()
    print("covariance |device - host| max", dc, "bit-identical", (cd == first[2]).all())
    assert dc <= 1e-12 * np.abs(first[2]).max()


def test_interleaving(base):
    """Track views of other sizes, model views, fuse views and renders interleaved on one context: each track view gives what it gives
    on a fresh context holding the map it saw."""
    ctx, tick = base["ctx"], base["tick"]
    T_A = base["T0inv"] @ base["T_room"]
    ctx.map_upload(base["surfels"])
    seq = ["1920x1080", "424x240", "330x246", "1280x720", "320x240_offcentre"]
    done = []
    for k, cam in enumerate(seq):
        Kb = CAMERAS[cam]
        T, rgb, depth = b_case(base, Kb, seed=20 + k)
        v = view_of(Kb, perturb(T, 1.0 + k), tick)
        done.append((ctx.map_download(), Kb, v, rgb, depth, ctx.track_view(v, rgb, depth, max_trace=48)))
        Kv = CAMERAS[seq[-1 - k]]
        ctx.predict_view(capi.model_view(T_A, Kv.fx, Kv.fy, Kv.cx, Kv.cy, Kv.width, Kv.height, MAXD, CONF, tick, tick, BIG))
        ctx.render(capi.camera_view(T_A, Kv.fx, Kv.fy, Kv.cx, Kv.cy, Kv.width, Kv.height, threshold=1.0))
        if k % 2 == 0:
            Tf, rf, df = b_case(base, Kv, seed=40 + k)
            ctx.fuse_view(capi.fuse_view(Tf, Kv.fx, Kv.fy, Kv.cx, Kv.cy, Kv.width, Kv.height, tick - 1, time_delta=BIG), rf, df)
    for surfels, Kb, v, rgb, depth, got in done:
        fresh = make_ctx(synth.K_DEFAULT)
        try:
            fresh.map_upload(surfels)
            ref = fresh.track_view(v, rgb, depth, max_trace=48)
        finally:
            fresh.close()
        for k in (0, 2, 3):
            assert_same(np.asarray(got[k]), np.asarray(ref[k]), f"{Kb.width}x{Kb.height} {k}")
        assert_bytes(got[1], ref[1], f"{Kb.width}x{Kb.height} stats")
        assert_bytes(got[4], ref[4], f"{Kb.width}x{Kb.height} trace")


def test_api_behaviour(base):
    import torch

    ctx = base["ctx"]
    Kb = CAMERAS["424x240"]
    T, rgb, depth = b_case(base, Kb)
    v = view_of(Kb, T, base["tick"])
    ctx.map_upload(base["surfels"])
    fields = [("width", 31), ("width", 4097), ("height", 31), ("height", 4097), ("fx", 0.0), ("fy", 0.0), ("fx", float("nan")),
              ("fy", float("inf")), ("cx", float("nan")), ("cy", float("-inf")), ("max_depth", 0.0), ("max_depth", float("inf")),
              ("conf_threshold", float("nan"))]
    bads = []
    for f, val in fields:
        b = view_of(Kb, T, base["tick"])
        setattr(b.model, f, val)
        bads.append(b)
    for i in (0, 5, 11, 15):
        b = view_of(Kb, T, base["tick"])
        b.model.T_wc[i] = float("nan") if i % 2 else float("inf")
        bads.append(b)
    for f, val in (("depth_cutoff", 0.0), ("depth_cutoff", -1.0), ("depth_cutoff", float("nan")), ("depth_cutoff", float("inf")),
                   ("icp_weight", -0.5), ("icp_weight", float("nan")), ("icp_weight", float("inf"))):
        b = view_of(Kb, T, base["tick"])
        setattr(b, f, val)
        bads.append(b)
    L, C = capi.lib(), capi.C
    hr, hd = capi._p(np.ascontiguousarray(rgb)), capi._p(np.ascontiguousarray(depth))
    r = torch.from_numpy(np.ascontiguousarray(rgb)).cuda()
    d = torch.from_numpy(np.ascontiguousarray(depth).view(np.int16)).cuda()
    out = torch.zeros(1024, dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()
    dr, dd, do = C.c_void_p(r.data_ptr()), C.c_void_p(d.data_ptr()), C.c_void_p(out.data_ptr())
    res, n = capi.EfTrackResult(), C.c_int32()
    trace = np.zeros(4, capi.TRACE_DTYPE)
    for b in bads:
        what = [(f, getattr(b.model, f)) for f, _ in b.model._fields_ if f != "T_wc"] + [(f, getattr(b, f)) for f in ("depth_cutoff", "icp_weight")]
        assert L.ef_track_view(ctx.h_ctx, C.byref(b), hr, hd, C.byref(res), None, 0, C.byref(n)) == EF_EINVAL, what
        assert L.ef_track_view_device(ctx.h_ctx, C.byref(b), dr, dd, do) == EF_EINVAL, what
    assert L.ef_track_view(None, C.byref(v), hr, hd, C.byref(res), None, 0, None) == EF_EINVAL
    assert L.ef_track_view(ctx.h_ctx, None, hr, hd, C.byref(res), None, 0, None) == EF_EINVAL
    assert L.ef_track_view(ctx.h_ctx, C.byref(v), None, hd, C.byref(res), None, 0, None) == EF_EINVAL
    assert L.ef_track_view(ctx.h_ctx, C.byref(v), hr, None, C.byref(res), None, 0, None) == EF_EINVAL
    assert L.ef_track_view(ctx.h_ctx, C.byref(v), hr, hd, None, None, 0, None) == EF_EINVAL
    assert L.ef_track_view(ctx.h_ctx, C.byref(v), hr, hd, C.byref(res), capi._p(trace), -1, None) == EF_EINVAL
    assert L.ef_track_view(ctx.h_ctx, C.byref(v), hr, hd, C.byref(res), None, 4, None) == EF_EINVAL
    assert L.ef_track_view_device(None, C.byref(v), dr, dd, do) == EF_EINVAL
    assert L.ef_track_view_device(ctx.h_ctx, None, dr, dd, do) == EF_EINVAL
    assert L.ef_track_view_device(ctx.h_ctx, C.byref(v), None, dd, do) == EF_EINVAL
    assert L.ef_track_view_device(ctx.h_ctx, C.byref(v), dr, None, do) == EF_EINVAL
    assert L.ef_track_view_device(ctx.h_ctx, C.byref(v), dr, dd, None) == EF_EINVAL
    assert L.ef_track_view_device(ctx.h_ctx, C.byref(v), dr, C.c_void_p(d.data_ptr() + 1), do) == EF_EINVAL
    assert L.ef_track_view_device(ctx.h_ctx, C.byref(v), dr, dd, C.c_void_p(out.data_ptr() + 4)) == EF_EINVAL
    # the smallest and a valid call with a trace shorter than the schedule
    assert L.ef_track_view(ctx.h_ctx, C.byref(v), hr, hd, C.byref(res), capi._p(trace), 4, C.byref(n)) == 0 and n.value == 4
    K32 = _k(32, 32, 30.0)
    r32, d32 = b_frame(base["T_room"], K32, np.eye(4), 1)
    assert ctx.track_view(view_of(K32, T, base["tick"]), r32, d32)[0].shape == (4, 4)


def test_state_rules(K, frames):
    """No EF_ESTATE: before the first frame on an uploaded map, between ef_process_frame_begin and _end, with a prefetched frame staged,
    and between ef_process_frame_device and ef_finish_frame; the frames that follow are those of a run without views."""
    import torch

    Kb = CAMERAS["424x240"]
    traj = synth.trajectory(len(frames), seed=42)
    T0inv = np.linalg.inv(traj[0])
    rgb_b, depth_b = b_frame(traj[1], Kb, cam_offset(), 3)
    T_b = T0inv @ traj[1] @ cam_offset()
    src = make_ctx(K)
    try:
        for i in range(4):
            src.process_frame(frames[i][0], frames[i][1], i)
        surfels = src.map_download()
    finally:
        src.close()
    dev = [torch.from_numpy(np.ascontiguousarray(a)).cuda() for a in (frames[2][0], frames[2][1].view(np.int16), frames[3][0],
                                                                     frames[3][1].view(np.int16), rgb_b, depth_b.view(np.int16))]
    out = torch.zeros(1024, dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()

    first = make_ctx(K)
    try:  # before the first frame, on an uploaded map
        first.map_upload(surfels)
        _, st, _, dense, _ = first.track_view(view_of(Kb, perturb(T_b, 1.0), 5), rgb_b, depth_b)
        assert st["lastICPCount"] > 0
    finally:
        first.close()

    def run(with_views):
        ctx = make_ctx(K)
        poses = []
        try:
            ctx.process_frame(frames[0][0], frames[0][1], 0)
            ctx.process_frame_begin(frames[1][0], frames[1][1], 1)
            if with_views:
                ctx.track_view(view_of(Kb, perturb(T_b, 1.0), 2), rgb_b, depth_b)
            ctx.process_frame_end()
            poses.append(ctx.get_pose())
            ctx.process_frame_device(dev[0].data_ptr(), dev[1].data_ptr(), 2)
            ctx.prefetch_frame_device(dev[2].data_ptr(), dev[3].data_ptr())
            if with_views:
                ctx.track_view_device(view_of(Kb, perturb(T_b, 1.0), 3), dev[4].data_ptr(), dev[5].data_ptr(), out.data_ptr())
            ctx.finish_frame()
            poses.append(ctx.get_pose())
            if with_views:
                ctx.track_view(view_of(Kb, perturb(T_b, 1.0), 3), rgb_b, depth_b)  # with the prefetched frame staged
            ctx.process_frame(None, None, 3)
            poses.append(ctx.get_pose())
            return poses, ctx.map_download()
        finally:
            ctx.close()

    (pa, ma), (pb, mb) = run(True), run(False)
    for k, (x, y) in enumerate(zip(pa, pb)):
        assert_same(x, y, f"pose {k}")
    assert_same(ma, mb, "map")
