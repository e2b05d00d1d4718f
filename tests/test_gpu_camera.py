"""ef_camera_* on the GPU: a second RGB-D sensor run frame after frame against the context's map. A camera equals, byte for byte,
ElasticFusion::processFrame run by a context built for its camera (close_loops = 0); it and the frame leave each other's results as
they are; on a rig it tracks about as well as a context of its own; and its calls follow the state rules of the header."""
import numpy as np
import pytest

from util import assert_same

from elasticfusion_b200 import capi, synth
from test_gpu_track_view import CAMERAS, FRAME_TEX, _k, assert_bytes, b_frame, cam_offset, frame_state

pytestmark = pytest.mark.gpu
EF_EINVAL, EF_ESTATE = -1, -3
N_FRAMES = 10
# tracker settings of each case, as EfCameraConfig / the frame's setters take them
SETTINGS = {"default": {}, "no_so3": dict(so3=False), "frame_to_frame_rgb": dict(frame_to_frame_rgb=True), "rgb_only": dict(rgb_only=True),
            "fast_odom": dict(fast_odom=True), "no_pyramid": dict(pyramid=False), "icp_only": dict(icp_weight=100.0),
            "low_confidence": dict(conf_threshold=2.0)}
# at the frame's confidence of 10, ten frames leave the prediction too sparse for denseEnough and the tracker always takes the fill-in;
# at 2 the 330x246 camera tracks against the prediction itself at calls 9 and 10 (measured on an H100), which this case asserts
DENSE_CASE = ("330x246", "low_confidence")
PRED = ("IMAGE", "VERTEX", "NORMAL", "TIME", "FILL_IMAGE", "FILL_VERTEX", "FILL_NORMAL")


def ctx_for(K, capacity=1_000_000, **kw):
    return capi.Context(capi.default_config(K.width, K.height, K.fx, K.fy, K.cx, K.cy, capacity=capacity, **kw))


def cam_cfg(K, settings=None):
    return capi.camera_config(K.width, K.height, K.fx, K.fy, K.cx, K.cy, **(settings or {}))


def set_frame(ctx, s):
    """the frame's settings of a case (EfConfig's so3 / frame_to_frame_rgb / fast_odom / icp_weight / confidence have setters too)"""
    ctx.set(**{("confidence_threshold" if k == "conf_threshold" else k): v for k, v in s.items()})


def reference_run(Kb, frames, settings, capacity, resident=None):
    """Context B for camera B (close_loops = 0) through ef_process_frame. Per frame: (dense_enough before it, pose, stats, covariance,
    map, prediction + fill-in). resident: surfels uploaded after frame 1 (and frame 1's prediction redone on them at tick 1)."""
    B = ctx_for(Kb, capacity)
    out = []
    try:
        set_frame(B, settings)
        for k, (rgb, depth, _) in enumerate(frames):
            dense = B.dense_enough()
            B.process_frame(rgb, depth, k)
            if k == 0 and resident is not None:
                B.map_upload(np.concatenate([resident, B.map_download()]))
                B.set_tick(1)
                B.predict()
                B.set_tick(2)
            out.append(dict(dense=dense, T=B.get_pose(), stats=B.odom_stats(0), cov=B.odom_covariance(0), map=B.map_download(),
                            pred={b: B.download(b) for b in PRED}))
    finally:
        B.close()
    return out


def camera_run(Kb, frames, settings, capacity, first_map):
    """Context A (its own 640x480 camera) after one frame of its own, B's map after frame 1 uploaded, then the camera: the first call
    at B's pose with fuse = 0 and time 1, calls k = 2..10 tracked and fused at time k."""
    KA = synth.K_DEFAULT
    own = next(synth.sequence(1, KA, seed=7, noise=True))
    A = ctx_for(KA, capacity)
    out = []
    try:
        A.process_frame(own[0], own[1], 0)
        A.map_upload(first_map["map"])
        cam = A.camera(cam_cfg(Kb, settings))
        for k, (rgb, depth, _) in enumerate(frames):
            if k == 0:
                T, st, cov, info, tr = cam.frame(rgb, depth, 1, T_wc=first_map["T"], fuse=False)
            else:
                T, st, cov, info, tr = cam.frame(rgb, depth, k + 1, max_trace=48)
            out.append(dict(dense=info["dense_enough"], tracked=info["tracked"], T=T, stats=st, cov=cov, map=A.map_download(),
                            pred={b: cam.download(b) for b in PRED}, trace=tr))
        cam.close()
    finally:
        A.close()
    return out


def compare_runs(got, ref, what):
    for k, (g, r) in enumerate(zip(got, ref)):
        w = f"{what} call {k + 1}"
        assert_same(g["T"], r["T"], f"{w} pose")
        assert_bytes(g["stats"], r["stats"], f"{w} stats")
        assert_same(g["cov"], r["cov"], f"{w} covariance")
        assert g["dense"] == r["dense"], w
        assert g["map"].shape == r["map"].shape, (w, g["map"].shape, r["map"].shape)
        assert g["map"].tobytes() == r["map"].tobytes(), f"{w} map"
        for b in PRED:
            assert_same(g["pred"][b], r["pred"][b], f"{w} {b}")
        assert g["tracked"] == (k > 0), w


CASES = [(cam, "default") for cam in sorted(CAMERAS)] + [(cam, s) for cam in ("424x240", "330x246") for s in sorted(SETTINGS) if s != "default"]


@pytest.mark.parametrize("cam,setting", CASES)
def test_camera_equals_process_frame(cam, setting):
    Kb, s = CAMERAS[cam], SETTINGS[setting]
    frames = list(synth.sequence(N_FRAMES, Kb, seed=11, noise=True))
    ref = reference_run(Kb, frames, s, 4_000_000)
    got = camera_run(Kb, frames, s, 4_000_000, ref[0])
    compare_runs(got, ref, f"{cam} {setting}")
    assert got[-1]["map"].shape[0] > got[0]["map"].shape[0] or s.get("rgb_only")
    dense = [k + 1 for k, g in enumerate(got) if g["dense"]]
    print(cam, setting, "dense enough at calls", dense)
    assert dense or (cam, setting) != DENSE_CASE


def test_camera_equals_process_frame_resident_5m():
    """The same at 1920x1080 on a resident map of 5 M surfels (the room's walls, uploaded after frame 1 in both runs)."""
    Kb = CAMERAS["1920x1080"]
    frames = list(synth.sequence(4, Kb, seed=11, noise=True))
    room = synth.room_surfels(5_000_000, np.linalg.inv(synth.trajectory(1, seed=11)[0]), view_depth=1.5, focal=Kb.fx)
    ref = reference_run(Kb, frames, {}, 8_000_000, resident=room)
    got = camera_run(Kb, frames, {}, 8_000_000, ref[0])
    assert ref[0]["map"].shape[0] > 5_000_000
    compare_runs(got, ref, "resident 5M")


def rig_inputs(n, seed=9):
    KA, Kb, T_AB = _k(320, 240, 264.0), CAMERAS["424x240"], cam_offset()
    frames = list(synth.sequence(n, KA, seed=seed, noise=True))
    traj = synth.trajectory(n, seed=seed)
    T0inv = np.linalg.inv(traj[0])
    bframes = [b_frame(traj[i], Kb, T_AB, 500 + i) for i in range(n)]
    truth = [T0inv @ traj[i] @ T_AB for i in range(n)]
    return KA, Kb, frames, bframes, truth


def rig_run(close_loops, n=30, camera_maps=None, frame_maps=None):
    """Frame A then camera B (time = tick - 1) for n frames. close_loops = 2 runs the look-ahead and the camera's device call between
    ef_process_frame_device and ef_finish_frame; 0 the host calls. camera_maps: instead of each camera call, upload that map.
    frame_maps: camera B alone on a context that uploads, before each call, the map the frame left. Returns the frame's states, the
    map after each frame, the map after each camera call, and the camera's results and buffers."""
    import torch

    KA, Kb, frames, bframes, truth = rig_inputs(n)
    ctx = ctx_for(KA, 400_000, time_delta=200, close_loops=close_loops)
    states, after_frame, after_cam, cam_out = [], [], [], []
    dev = [(torch.from_numpy(np.ascontiguousarray(r)).cuda(), torch.from_numpy(np.ascontiguousarray(d).view(np.int16)).cuda())
           for r, d, _ in frames]
    bdev = [(torch.from_numpy(np.ascontiguousarray(r)).cuda(), torch.from_numpy(np.ascontiguousarray(d).view(np.int16)).cuda())
            for r, d in bframes]
    out_dev = torch.zeros(capi.C.sizeof(capi.EfCameraResult), dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()
    cam = ctx.camera(capi.camera_config(Kb.width, Kb.height, Kb.fx, Kb.fy, Kb.cx, Kb.cy, time_delta=200))
    try:
        if frame_maps is not None:
            ctx.process_frame(frames[0][0], frames[0][1], 0)  # (a fused camera frame needs a context past its first frame)
            for i in range(n):
                ctx.map_upload(frame_maps[i])
                pose = truth[0] if i == 0 else None
                cam_out.append((cam.frame(*bframes[i], i + 1, T_wc=pose, max_trace=48), {b: cam.download(b) for b in PRED}))
            return states, after_frame, after_cam, cam_out
        if close_loops == 2:
            ctx.prefetch_frame_device(dev[0][0].data_ptr(), dev[0][1].data_ptr())
        for i in range(n):
            pose = truth[0] if i == 0 else None
            if close_loops == 2:
                ctx.process_frame_device(None, None, i)
                if i + 1 < n:
                    ctx.prefetch_frame_device(dev[i + 1][0].data_ptr(), dev[i + 1][1].data_ptr())
                if camera_maps is None:
                    cam.frame_device(bdev[i][0].data_ptr(), bdev[i][1].data_ptr(), out_dev.data_ptr(), i + 1, T_wc=pose)
                else:
                    ctx.map_upload(camera_maps[i])
                ctx.finish_frame()
                if camera_maps is None:
                    ctx.sync()
                    res = capi.unpack_camera_result(out_dev.cpu().numpy().tobytes())
            else:
                ctx.process_frame(frames[i][0], frames[i][1], i)
                if camera_maps is None:
                    after_frame.append(ctx.map_download())
                    res = cam.frame(*bframes[i], ctx.get_tick() - 1, T_wc=pose, max_trace=48)
                else:
                    ctx.map_upload(camera_maps[i])
            if camera_maps is None:
                after_cam.append(ctx.map_download())
                cam_out.append((res, {b: cam.download(b) for b in PRED}))
            states.append(frame_state(ctx, close_loops))
    finally:
        ctx.close()
    return states, after_frame, after_cam, cam_out


@pytest.fixture(scope="module")
def rig0():
    return rig_run(0)


@pytest.mark.parametrize("close_loops", [0, 2])
def test_frame_untouched_by_camera(close_loops, rig0):
    """(a) the rig's frame outputs equal a replay where each camera call is replaced by the upload of the map it left"""
    states, _, after_cam, _ = rig0 if close_loops == 0 else rig_run(2)
    replay, _, _, _ = rig_run(close_loops, camera_maps=after_cam)
    names = ["pose", "tick", "dense", "map", "odom_stats 0", "odom_stats 1"] + list(FRAME_TEX)
    for i, (sa, sb) in enumerate(zip(states, replay)):
        for k, (x, y) in enumerate(zip(sa, sb)):
            assert x == y, (close_loops, i, names[k] if k < len(names) else k)


def test_camera_untouched_by_frame(rig0):
    """(b) camera B's calls alone, each on the map the rig's frame left, give the rig's results and buffers byte for byte"""
    _, after_frame, _, cam_out = rig0
    _, _, _, alone = rig_run(0, frame_maps=after_frame)
    for i, ((ra, ba), (rb, bb)) in enumerate(zip(cam_out, alone)):
        assert_same(ra[0], rb[0], f"call {i} pose")
        assert_bytes(ra[1], rb[1], f"call {i} stats")
        assert_same(ra[2], rb[2], f"call {i} covariance")
        assert ra[3] == rb[3], i
        assert_bytes(ra[4], rb[4], f"call {i} trace")
        for b in PRED:
            assert_same(ba[b], bb[b], f"call {i} {b}")


def test_rig_accuracy(rig0):
    """Camera B's translation error against ground truth (T_A T_AB) over the rig, and that of a camera-B context on B's sequence alone.
    The bar (rig <= 2x solo) was set before either number had been measured; the first run on an H100 gave 18.0 mm on the rig and
    22.9 mm alone (camera B tracks against a map that camera A's frames fill in as well)."""
    _, _, _, cam_out = rig0
    n = len(cam_out)
    KA, Kb, frames, bframes, truth = rig_inputs(n)
    est = np.array([r[0][0] for r in cam_out])
    rig = synth.ate_rmse(est, np.array(truth))
    solo_ctx = ctx_for(Kb, 400_000, time_delta=200)
    try:
        poses = []
        for i, (rgb, depth) in enumerate(bframes):
            solo_ctx.process_frame(rgb, depth, i)
            poses.append(solo_ctx.get_pose())
    finally:
        solo_ctx.close()
    gt_solo = np.array([np.linalg.inv(truth[0]) @ T for T in truth])
    solo = synth.ate_rmse(np.array(poses), gt_solo)
    print(f"camera B translation RMSE: rig {rig * 1000:.3f} mm, solo context {solo * 1000:.3f} mm over {n} frames")
    assert np.isfinite(rig) and rig <= 2.0 * solo + 1e-4, (rig, solo)


@pytest.fixture(scope="module")
def small_map():
    """a 640x480 context after 6 frames, its map, and camera B's inputs (424x240, at cam_offset of frame 5)"""
    K = synth.K_DEFAULT
    frames = list(synth.sequence(6, K, seed=42, noise=True))
    traj = synth.trajectory(6, seed=42)
    ctx = ctx_for(K, time_delta=200)
    for i, (rgb, depth, _) in enumerate(frames):
        ctx.process_frame(rgb, depth, i)
    Kb = CAMERAS["424x240"]
    bf = [b_frame(traj[i], Kb, cam_offset(), 40 + i) for i in (4, 5)]
    truth = [np.linalg.inv(traj[0]) @ traj[i] @ cam_offset() for i in (4, 5)]
    yield dict(ctx=ctx, map=ctx.map_download(), tick=ctx.get_tick(), Kb=Kb, bf=bf, truth=truth)
    ctx.close()


def two_calls(ctx, m, cam, device=False):
    import torch

    if not device:
        a = cam.frame(*m["bf"][0], m["tick"] - 1, T_wc=m["truth"][0], max_trace=48)
        b = cam.frame(*m["bf"][1], m["tick"] - 1, max_trace=48)
        return a[:4], b[:4]
    out = torch.zeros(capi.C.sizeof(capi.EfCameraResult), dtype=torch.uint8, device="cuda")
    ins = [(torch.from_numpy(np.ascontiguousarray(r)).cuda(), torch.from_numpy(np.ascontiguousarray(d).view(np.int16)).cuda()) for r, d in m["bf"]]
    torch.cuda.synchronize()
    res = []
    for k, (r, d) in enumerate(ins):
        cam.frame_device(r.data_ptr(), d.data_ptr(), out.data_ptr(), m["tick"] - 1, T_wc=m["truth"][0] if k == 0 else None)
        ctx.sync()
        res.append(capi.unpack_camera_result(out.cpu().numpy().tobytes()))
    return res


def same_result(a, b, what):
    assert_same(a[0], b[0], f"{what} pose")
    assert_bytes(a[1], b[1], f"{what} stats")
    assert_same(a[2], b[2], f"{what} covariance")
    assert a[3] == b[3], what


def test_host_device_and_repeat(small_map):
    m, ctx = small_map, small_map["ctx"]
    runs = []
    for device in (False, True, False):
        ctx.map_upload(m["map"])
        cam = ctx.camera(cam_cfg(m["Kb"]))
        runs.append((two_calls(ctx, m, cam, device), ctx.map_download(), cam.download("IMAGE")))
        cam.close()
    for r in runs[1:]:
        for k in range(2):
            same_result(r[0][k], runs[0][0][k], f"call {k}")
        assert r[1].tobytes() == runs[0][1].tobytes()
        assert_same(r[2], runs[0][2], "prediction")
    assert runs[0][0][1][3]["tracked"] and not runs[0][0][0][3]["tracked"]
    assert runs[0][0][0][3]["weighting"] == 1.0


def test_fuse_0_leaves_the_map(small_map):
    m, ctx = small_map, small_map["ctx"]
    ctx.map_upload(m["map"])
    cam = ctx.camera(cam_cfg(m["Kb"]))
    try:
        cam.frame(*m["bf"][0], m["tick"] - 1, T_wc=m["truth"][0], fuse=False)
        T, st, cov, info, _ = cam.frame(*m["bf"][1], m["tick"] - 1, fuse=False)
        assert info["tracked"] and st["lastICPCount"] > 0
        assert ctx.map_download().tobytes() == m["map"].tobytes()
        err = np.linalg.norm(T[:3, 3] - m["truth"][1][:3, 3])
        print("fuse = 0: translation error", err)
        assert err < 0.02
    finally:
        cam.close()


def test_bad_arguments_and_state_rules(small_map):
    import torch

    m, ctx, Kb = small_map, small_map["ctx"], small_map["Kb"]
    L, C = capi.lib(), capi.C
    h = C.c_void_p()
    bad_cfgs = [("width", 31), ("width", 4097), ("height", 31), ("height", 4097), ("fx", 0.0), ("fy", float("nan")), ("cx", float("inf")),
                ("cy", float("nan")), ("depth_cutoff", 0.0), ("depth_cutoff", float("nan")), ("max_depth", -1.0), ("max_depth", float("inf")),
                ("conf_threshold", float("nan")), ("time_delta", -1), ("icp_weight", -0.5), ("icp_weight", float("nan"))]
    for f, v in bad_cfgs:
        c = cam_cfg(Kb)
        setattr(c, f, v)
        assert L.ef_camera_create(ctx.h_ctx, C.byref(c), C.byref(h)) == EF_EINVAL, f
    assert L.ef_camera_create(ctx.h_ctx, None, C.byref(h)) == EF_EINVAL
    assert L.ef_camera_create(ctx.h_ctx, C.byref(cam_cfg(Kb)), None) == EF_EINVAL
    cam = ctx.camera(cam_cfg(Kb))
    other = ctx_for(synth.K_DEFAULT)
    rgb, depth = (np.ascontiguousarray(a) for a in m["bf"][0])
    hr, hd = capi._p(rgb), capi._p(depth)
    r = torch.from_numpy(rgb).cuda()
    d = torch.from_numpy(depth.view(np.int16)).cuda()
    out = torch.zeros(1024, dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()
    dr, dd, do = C.c_void_p(r.data_ptr()), C.c_void_p(d.data_ptr()), C.c_void_p(out.data_ptr())
    res, n = capi.EfCameraResult(), C.c_int32()
    try:
        good = capi.camera_frame(m["tick"] - 1, T_wc=m["truth"][0])
        bads = []
        for f, v in (("time", -1), ("weight_multiplier", -1.0), ("weight_multiplier", float("nan"))):
            b = capi.camera_frame(m["tick"] - 1, T_wc=m["truth"][0])
            setattr(b, f, v)
            bads.append(b)
        b = capi.camera_frame(m["tick"] - 1, T_wc=m["truth"][0])
        b.T_wc[5] = float("nan")
        bads.append(b)
        for b in bads:
            assert L.ef_camera_frame(ctx.h_ctx, cam.h_cam, C.byref(b), hr, hd, C.byref(res), None, 0, None) == EF_EINVAL
            assert L.ef_camera_frame_device(ctx.h_ctx, cam.h_cam, C.byref(b), dr, dd, do) == EF_EINVAL
        g = C.byref(good)
        assert L.ef_camera_frame(other.h_ctx, cam.h_cam, g, hr, hd, C.byref(res), None, 0, None) == EF_EINVAL
        assert L.ef_camera_frame(ctx.h_ctx, None, g, hr, hd, C.byref(res), None, 0, None) == EF_EINVAL
        assert L.ef_camera_frame(ctx.h_ctx, cam.h_cam, None, hr, hd, C.byref(res), None, 0, None) == EF_EINVAL
        assert L.ef_camera_frame(ctx.h_ctx, cam.h_cam, g, None, hd, C.byref(res), None, 0, None) == EF_EINVAL
        assert L.ef_camera_frame(ctx.h_ctx, cam.h_cam, g, hr, None, C.byref(res), None, 0, None) == EF_EINVAL
        assert L.ef_camera_frame(ctx.h_ctx, cam.h_cam, g, hr, hd, None, None, 0, None) == EF_EINVAL
        assert L.ef_camera_frame(ctx.h_ctx, cam.h_cam, g, hr, hd, C.byref(res), None, 4, None) == EF_EINVAL
        assert L.ef_camera_frame(ctx.h_ctx, cam.h_cam, g, hr, hd, C.byref(res), None, -1, None) == EF_EINVAL
        assert L.ef_camera_frame_device(ctx.h_ctx, cam.h_cam, g, dr, C.c_void_p(d.data_ptr() + 1), do) == EF_EINVAL
        assert L.ef_camera_frame_device(ctx.h_ctx, cam.h_cam, g, dr, dd, C.c_void_p(out.data_ptr() + 4)) == EF_EINVAL
        assert L.ef_camera_frame_device(ctx.h_ctx, cam.h_cam, g, None, dd, do) == EF_EINVAL
        assert L.ef_camera_destroy(other.h_ctx, cam.h_cam) == EF_EINVAL
        p, nb = C.c_void_p(), C.c_size_t()
        for bid in (capi.BUF["INDEX"], capi.BUF["OLD_IMAGE"], capi.BUF["SYNTH_DEPTH"], 140, 99, -1):
            assert L.ef_camera_buffer(ctx.h_ctx, cam.h_cam, bid, 0, C.byref(p), C.byref(nb)) == EF_EINVAL, bid
        assert L.ef_camera_buffer(ctx.h_ctx, cam.h_cam, capi.BUF["VMAP_CURR"], 3, C.byref(p), C.byref(nb)) == EF_EINVAL
        assert L.ef_camera_buffer(ctx.h_ctx, cam.h_cam, capi.BUF["VMAP_CURR"], 2, C.byref(p), C.byref(nb)) == 0
        assert nb.value == (Kb.width >> 2) * (Kb.height >> 2) * 12
        # first call without a pose
        nopose = capi.camera_frame(m["tick"] - 1)
        assert L.ef_camera_frame(ctx.h_ctx, cam.h_cam, C.byref(nopose), hr, hd, C.byref(res), None, 0, None) == EF_ESTATE
        assert L.ef_camera_frame_device(ctx.h_ctx, cam.h_cam, C.byref(nopose), dr, dd, do) == EF_ESTATE
        # fuse = 1 before the context's first frame; fuse = 0 runs there
        fresh = other.camera(cam_cfg(Kb))
        other.map_upload(m["map"])
        assert L.ef_camera_frame(other.h_ctx, fresh.h_cam, g, hr, hd, C.byref(res), None, 0, None) == EF_ESTATE
        fresh.frame(rgb, depth, 3, T_wc=m["truth"][0], fuse=False)
        assert fresh.frame(*m["bf"][1], 3, fuse=False)[3]["tracked"]
        # fuse = 1 between ef_process_frame_begin and _end; fuse = 0 runs there
        K = synth.K_DEFAULT
        f6 = synth.render(synth.trajectory(7, seed=42)[6], K, noise_seed=1)
        ctx.process_frame_begin(f6[0], f6[1], 6)
        assert L.ef_camera_frame(ctx.h_ctx, cam.h_cam, g, hr, hd, C.byref(res), None, 0, None) == EF_ESTATE
        cam.frame(rgb, depth, m["tick"] - 1, T_wc=m["truth"][0], fuse=False)
        ctx.process_frame_end()
        # a fifth live camera; destroying one frees its slot
        more = [ctx.camera(cam_cfg(Kb)) for _ in range(capi.MAX_CAMERAS - 1)]
        assert L.ef_camera_create(ctx.h_ctx, C.byref(cam_cfg(Kb)), C.byref(h)) == EF_ESTATE
        more[1].close()
        again = ctx.camera(cam_cfg(CAMERAS["330x246"]))
        rgb2, depth2, _, _ = synth.render(synth.trajectory(1, seed=42)[0], CAMERAS["330x246"], noise_seed=2)
        assert again.frame(rgb2, depth2, 7, weight_multiplier=0.5, T_wc=np.eye(4))[3]["weighting"] == 0.5
        for c in more:
            c.close()
        again.close()
    finally:
        cam.close()
        other.close()  # (with `fresh` still live: ef_destroy frees it)


def test_destroy_frees_live_cameras():
    import torch

    K = synth.K_DEFAULT
    free0 = torch.cuda.mem_get_info()[0]
    for _ in range(3):
        ctx = ctx_for(K, 100_000)
        for cam in ("1920x1080", "1280x720"):
            Kb = CAMERAS[cam]
            ctx.camera(cam_cfg(Kb))
        ctx.close()
    torch.cuda.synchronize()
    lost = free0 - torch.cuda.mem_get_info()[0]
    print("device memory not returned after 3 contexts with live cameras:", lost)
    assert lost < 64 << 20
