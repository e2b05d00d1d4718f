"""ef_camera_* with close_loops = 1 on the GPU: a camera's frames close local loops on the context's map and deformation graph. A closing
camera equals, byte for byte, ElasticFusion::processFrame with close_loops = 2 in a context built for its camera; on a rig the frame sees
exactly the map, graph and Deformation bookkeeping the camera leaves; nothing changes before the first closure; and the new calls follow
the header's rules."""
import hashlib

import numpy as np
import pytest

from test_gpu_camera import PRED
from test_gpu_loop_closure import ACCEPT_ALL, LOOP_CFG, N_FRAMES, sample_graph
from test_gpu_track_view import _k, assert_bytes, b_frame, cam_offset
from util import assert_same

from elasticfusion_b200 import capi, synth

pytestmark = pytest.mark.gpu
EF_EINVAL, EF_ESTATE = -1, -3
K_LOOP = synth.Intrinsics(320, 240, 264.0, 264.0, 160.0, 120.0)  # the loop sequence's camera
# cameras rendered along the loop sequence's trajectory (seed 21, speed 2.5)
LOOP_CAMERAS = {"320x240": K_LOOP, "424x240": _k(424, 240, 305.0), "330x246_offcentre": _k(330, 246, 290.0, 150.0, 131.0, fy=272.0)}
# forced closures: every registration accepted, a short time window and a low confidence
FORCED = dict(LOOP_CFG, time_delta=4, confidence=2.0, **ACCEPT_ALL)
FORCED_CAMERAS = {"1280x720": (_k(1280, 720, 915.0), 4_000_000), "1920x1080": (_k(1920, 1080, 1188.0), 8_000_000)}


def digest(a):
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


def make_ctx(K, **kw):
    return capi.Context(capi.default_config(K.width, K.height, K.fx, K.fy, K.cx, K.cy, **kw))


def cam_cfg(K, cfg, close_loops=True):
    return capi.camera_config(K.width, K.height, K.fx, K.fy, K.cx, K.cy, time_delta=cfg["time_delta"],
                              conf_threshold=cfg.get("confidence", 10.0), close_loops=close_loops)


def record(dense, T, stats, cov, m, pred, deform):
    info, graph = deform
    return dict(dense=dense, T=T, stats=stats, cov=cov, count=len(m), map=digest(m), pred={b: digest(p) for b, p in pred.items()},
                info=info, graph=graph)


def inactive_copy(m):
    """m displaced by a few millimetres, confident, first seen at tick 1 and last seen at -time_delta: surfels that no index map or
    ACTIVE prediction draws from tick 1 on (time - lastTime > time_delta), so no frame fuses into them, and that only the INACTIVE
    prediction (0, time - time_delta, time_delta) may draw"""
    c = m.copy()
    c[:, 0:3] += np.array([0.004, -0.003, 0.002], np.float32)
    c[:, 3] += 10.0
    c[:, 6], c[:, 7] = 1.0, -float(FORCED["time_delta"])
    return c


def reference_run(Kb, frames, cfg, extra=None):
    """A context built for camera B with close_loops = 2 over B's frames; per frame its outputs and the map it leaves. extra: surfels
    appended to the map after frame 1 (its prediction and graph stay those of frame 1's own map)"""
    B = make_ctx(Kb, close_loops=2, **cfg)
    out, first = [], None
    try:
        for k, (rgb, depth, _) in enumerate(frames):
            dense = B.dense_enough()
            B.process_frame(rgb, depth, k)
            m = B.map_download()
            if k == 0:
                first = dict(map=m, T=B.get_pose(), after=None)
                if extra is not None:
                    m = np.concatenate([m, extra(m)])
                    B.map_upload(m)
                    first["after"] = m
            out.append(record(dense, B.get_pose(), B.odom_stats(0), B.odom_covariance(0), m, {b: B.download(b) for b in PRED},
                              B.local_deform_result()))
    finally:
        B.close()
    return out, first


def camera_run(Kb, frames, cfg, first):
    """Context A (its own 640x480 camera, close_loops = 2) after one frame of its own, B's first map uploaded, then the closing camera:
    the first call at B's pose with fuse = 0 and time 1, call k at time k + 1 (with reference_run's extra surfels uploaded after the
    first call)"""
    KA = synth.K_DEFAULT
    own = next(synth.sequence(1, KA, seed=7, noise=True))
    A = make_ctx(KA, close_loops=2, **cfg)
    out = []
    try:
        A.process_frame(own[0], own[1], 0)
        A.map_upload(first["map"])
        cam = A.camera(cam_cfg(Kb, cfg))
        for k, (rgb, depth, _) in enumerate(frames):
            if k == 0:
                T, st, cov, info, _ = cam.frame(rgb, depth, 1, T_wc=first["T"], fuse=False)
                if first["after"] is not None:
                    A.map_upload(first["after"])
            else:
                T, st, cov, info, _ = cam.frame(rgb, depth, k + 1)
            out.append(record(info["dense_enough"], T, st, cov, A.map_download(), {b: cam.download(b) for b in PRED}, cam.deform_result()))
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
        assert (g["count"], g["map"]) == (r["count"], r["map"]), f"{w} map"
        assert g["pred"] == r["pred"], f"{w} prediction"
        assert g["info"] == r["info"], (w, g["info"], r["info"])
        assert np.array_equal(g["graph"], r["graph"]), f"{w} graph"


def applied_closures(run):
    """(call index, pinned, last_deform_time before it) of every applied closure of a run"""
    out, deforms, last = [], 0, 0
    for k, r in enumerate(run):
        if r["info"]["applied"]:
            out.append(dict(call=k, pinned=deforms == 0, last_deform_time=last))
        deforms, last = r["info"]["deforms"], r["info"]["last_deform_time"]
    return out


@pytest.mark.parametrize("cam", sorted(LOOP_CAMERAS))
def test_closing_camera_equals_process_frame(cam):
    """130 frames of the loop sequence: the camera equals a camera-B context with close_loops = 2 after every call"""
    Kb = LOOP_CAMERAS[cam]
    frames = list(synth.sequence(N_FRAMES, Kb, seed=21, noise=True, speed=2.5))
    ref, first = reference_run(Kb, frames, LOOP_CFG)
    got = camera_run(Kb, frames, LOOP_CFG, first)
    compare_runs(got, ref, cam)
    applied = applied_closures(got)
    print(cam, "applied closures:", applied)
    assert len(applied) >= 1, cam
    if cam == "320x240":  # as test_gpu_loop_closure asserts for this sequence
        assert len(applied) >= 2 and applied[0]["pinned"] and applied[0]["last_deform_time"] == 0, applied
        assert any(not a["pinned"] and a["last_deform_time"] > 0 for a in applied[1:]), applied


@pytest.mark.parametrize("cam", sorted(FORCED_CAMERAS))
def test_forced_closures_at_large_sizes(cam):
    """Every registration accepted at 1280x720 and 1920x1080, with a displaced INACTIVE copy of the first map: still the camera-B context
    after every call. Measured on an H100: every call from the fifth on solves (the graph exists from the first), and every fourth
    call (time_delta) takes 80-85 % of the (W/20)(H/20) grid; at most 2 (W/20)(H/20) constraints including pins."""
    Kb, capacity = FORCED_CAMERAS[cam]
    cfg = dict(FORCED, capacity=capacity)
    frames = list(synth.sequence(20, Kb, seed=21, noise=True, speed=2.5))
    ref, first = reference_run(Kb, frames, cfg, extra=inactive_copy)
    got = camera_run(Kb, frames, cfg, first)
    compare_runs(got, ref, cam)
    solved = [(k, g["info"]["result"]["n_constraints"], g["info"]["result"]["stop"]) for k, g in enumerate(got) if g["info"]["solved"]]
    print(cam, "solves (call, constraints incl. pins, stop):", solved)
    grid = (Kb.width // 20) * (Kb.height // 20)
    assert [k for k, _, _ in solved] == list(range(4, len(frames))), cam
    assert all(g["info"]["applied"] for g in got[4:]) and all(n <= 2 * grid for _, n, _ in solved)
    assert max(n for _, n, _ in solved) > grid // 2


# ---- the rig: frame A (320x240, close_loops = 2, look-ahead) and closing camera B (424x240) ------------------------------------------
RIG_B = LOOP_CAMERAS["424x240"]


def rig_inputs(n):
    frames = list(synth.sequence(n, K_LOOP, seed=21, noise=True, speed=2.5))
    traj = synth.trajectory(n, seed=21, speed=2.5)
    T0inv = np.linalg.inv(traj[0])
    bframes = [b_frame(traj[i], RIG_B, cam_offset(), 500 + i) for i in range(n)]
    truth = [T0inv @ traj[i] @ cam_offset() for i in range(n)]
    return frames, bframes, truth


def rig_run(close_loops, n=N_FRAMES, keep_maps=False):
    """The look-ahead frame, then the camera's device call between ef_process_frame_device and ef_finish_frame, time = tick - 1. Per
    frame: the frame's pose, the map after the frame and after the camera, the frame's and the camera's closure, the camera's result."""
    import torch

    frames, bframes, truth = rig_inputs(n)
    ctx = make_ctx(K_LOOP, close_loops=2, **LOOP_CFG)
    dev = [tuple(torch.from_numpy(np.ascontiguousarray(a).view(np.int16) if a.dtype == np.uint16 else np.ascontiguousarray(a)).cuda()
                 for a in f[:2]) for f in frames]
    bdev = [tuple(torch.from_numpy(np.ascontiguousarray(a).view(np.int16) if a.dtype == np.uint16 else np.ascontiguousarray(a)).cuda()
                  for a in f) for f in bframes]
    out_dev = torch.zeros(capi.C.sizeof(capi.EfCameraResult), dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()
    rec = []
    cam = ctx.camera(cam_cfg(RIG_B, LOOP_CFG, close_loops))
    try:
        ctx.prefetch_frame_device(dev[0][0].data_ptr(), dev[0][1].data_ptr())
        for i in range(n):
            ctx.process_frame_device(None, None, i)
            m_frame = ctx.map_download()
            frame_deform = ctx.local_deform_result()[0]
            if i + 1 < n:
                ctx.prefetch_frame_device(dev[i + 1][0].data_ptr(), dev[i + 1][1].data_ptr())
            cam.frame_device(bdev[i][0].data_ptr(), bdev[i][1].data_ptr(), out_dev.data_ptr(), i + 1, T_wc=truth[0] if i == 0 else None)
            ctx.finish_frame()
            ctx.sync()
            res = capi.unpack_camera_result(out_dev.cpu().numpy().tobytes())
            m = ctx.map_download()
            info, graph = ctx.local_deform_result()
            rec.append(dict(pose=ctx.get_pose(), after_frame=digest(m_frame), after_cam=digest(m), map=m if keep_maps else None,
                            frame=frame_deform, cam=cam.deform_result()[0] if close_loops else None, final=info, graph=graph, res=res))
    finally:
        cam.close()
        ctx.close()
    return rec


@pytest.fixture(scope="module")
def rig_closing():
    return rig_run(True, keep_maps=True)


def test_rig_frame_sees_the_map_the_camera_leaves(rig_closing):
    """(a) the rig's frame equals a close_loops = 1 context running the host recipe (begin, local_loop_result, deform_solve, end), in
    which each camera call is replaced by the upload of the map it left, its deforms / last_deform_time and the graph re-sampled"""
    rig = rig_closing
    frames, _, _ = rig_inputs(len(rig))
    ctx = make_ctx(K_LOOP, close_loops=1, **LOOP_CFG)
    deforms, last, graph = 0, 0, None
    try:
        for i, (rgb, depth, _) in enumerate(frames):
            r = rig[i]
            ctx.process_frame_begin(rgb, depth, i)
            info, src, dst, tms = ctx.local_loop_result()
            T_over = nodes = solved = None
            if info["ran"] and info["accepted"] and graph is not None and len(src) > 0:
                tick = ctx.get_tick()
                solved, nodes16, *_ = ctx.deform_solve(graph[:, :3], graph[:, 3].astype(np.int32), src, dst, np.full(len(src), tick, np.int32),
                                                       tms, pin=deforms == 0, last_deform_time=last)
                if solved["stop"] != 6:
                    T_over, nodes = info["T_wc_est"], nodes16
                    deforms, last = deforms + 1, tick
            ctx.process_frame_end(T_over, nodes)
            assert np.array_equal(ctx.get_pose(), r["pose"]), i
            assert digest(ctx.map_download()) == r["after_frame"], i
            f = r["frame"]
            assert (f["solved"], f["applied"]) == (solved is not None, T_over is not None), i
            if solved is not None:
                assert f["result"] == solved, i
            assert (f["deforms"], f["last_deform_time"]) == (deforms, last), i
            # the camera call, replayed
            ctx.map_upload(r["map"])
            deforms, last = r["cam"]["deforms"], r["cam"]["last_deform_time"]
            g = sample_graph(r["map"])
            if g is not None:
                graph = g
            assert np.array_equal(r["graph"], graph if graph is not None else np.zeros((0, 4), np.float32)), i
    finally:
        ctx.close()


def test_rig_bookkeeping_and_accuracy(rig_closing):
    """(b) up to the first applied closure of either side the rig equals the same rig with an open-loop camera; (c) deforms counts the
    applied closures of both sides, last_deform_time is the latest one's time, the first is pinned; (d) camera B's translation RMSE with
    and without its closures, reported (a synthetic run may get worse: no bar)"""
    rig = rig_closing
    open_rig = rig_run(False)
    events = []  # (frame index, side) of every applied closure, in order
    deforms, last = 0, 0
    for i, r in enumerate(rig):
        for side in ("frame", "cam"):
            d = r[side]
            if d["applied"]:
                events.append((i, side, d["result"]["n_constraints"]))
                deforms, last = deforms + 1, i + 1  # both sides run at time = tick = i + 1
            assert (d["deforms"], d["last_deform_time"]) == (deforms, last), (i, side)
            assert not d["solved"] or d["result"]["n_constraints"] > 0
        assert (r["final"]["deforms"], r["final"]["last_deform_time"]) == (deforms, last), i
    print("applied closures (frame index, side, constraints incl. pins):", events)
    assert any(s == "cam" for _, s, _ in events), events
    first = min([e[0] for e in events] + [i for i, r in enumerate(open_rig) if r["frame"]["applied"]])
    assert first > 0
    for i in range(first):
        a, b = rig[i], open_rig[i]
        assert np.array_equal(a["pose"], b["pose"]), i
        assert (a["after_frame"], a["after_cam"]) == (b["after_frame"], b["after_cam"]), i
        assert_same(a["res"][0], b["res"][0], f"frame {i} camera pose")
        assert_bytes(a["res"][1], b["res"][1], f"frame {i} camera stats")
    truth = np.array(rig_inputs(len(rig))[2])
    rmse = {name: synth.ate_rmse(np.array([r["res"][0] for r in run]), truth) for name, run in (("closing", rig), ("open", open_rig))}
    print(f"camera B translation RMSE over {len(rig)} frames: with its closures {rmse['closing'] * 1000:.3f} mm, "
          f"open loop {rmse['open'] * 1000:.3f} mm")
    assert all(np.isfinite(v) for v in rmse.values())


# ---- calls and errors -------------------------------------------------------------------------------------------------------------------
FORCED_SMALL = dict(FORCED, capacity=800_000)


def forced_context(frames):
    """a 320x240 context (close_loops = 2, every registration accepted) after 12 loop-sequence frames"""
    ctx = make_ctx(K_LOOP, close_loops=2, **FORCED_SMALL)
    for i, (rgb, depth, _) in enumerate(frames[:12]):
        ctx.process_frame(rgb, depth, i)
    return ctx


@pytest.fixture(scope="module")
def forced_small():
    """forced_context, its map and pose, and the next frames"""
    frames = list(synth.sequence(16, K_LOOP, seed=21, noise=True, speed=2.5))
    ctx = forced_context(frames)
    yield dict(ctx=ctx, all=frames, map=ctx.map_download(), T=ctx.get_pose(), frames=[f[:2] for f in frames[11:16]])
    ctx.close()


def closing_calls(m, device):
    """a closing camera on a fresh forced_context (Deformation's bookkeeping starts at zero): a has_pose call, then four tracked and
    fused calls; results, maps and closures"""
    import torch

    ctx = forced_context(m["all"])
    cam = ctx.camera(cam_cfg(K_LOOP, FORCED_SMALL))
    out = []
    try:
        out_dev = torch.zeros(capi.C.sizeof(capi.EfCameraResult), dtype=torch.uint8, device="cuda")
        for k, (rgb, depth) in enumerate(m["frames"]):
            T = m["T"] if k == 0 else None
            if device:
                r = torch.from_numpy(np.ascontiguousarray(rgb)).cuda()
                d = torch.from_numpy(np.ascontiguousarray(depth).view(np.int16)).cuda()
                torch.cuda.synchronize()
                cam.frame_device(r.data_ptr(), d.data_ptr(), out_dev.data_ptr(), 12 + k, T_wc=T)
                ctx.sync()
                res = capi.unpack_camera_result(out_dev.cpu().numpy().tobytes())
            else:
                res = cam.frame(rgb, depth, 12 + k, T_wc=T)[:4]
            out.append((res, digest(ctx.map_download()), cam.deform_result()))
        cam.close()
    finally:
        ctx.close()
    return out


def test_host_and_device_calls_are_identical(forced_small):
    runs = [closing_calls(forced_small, device) for device in (False, True)]
    for k, (a, b) in enumerate(zip(*runs)):
        assert_same(a[0][0], b[0][0], f"call {k} pose")
        assert_bytes(a[0][1], b[0][1], f"call {k} stats")
        assert_same(a[0][2], b[0][2], f"call {k} covariance")
        assert a[0][3] == b[0][3] and a[1] == b[1], k
        assert a[2][0]["solved"] == b[2][0]["solved"] and a[2][0]["applied"] == b[2][0]["applied"], k
        assert a[2][0]["result"] == b[2][0]["result"] and np.array_equal(a[2][1], b[2][1]), k
    print("solved at calls", [k for k, a in enumerate(runs[0]) if a[2][0]["solved"]])


@pytest.mark.parametrize("kind", ["fuse_0", "rgb_only"])
def test_calls_without_front_half_sample_the_graph(forced_small, kind):
    """fuse = 0 and rgb_only calls run no front half (nothing solved) but leave the graph sampled from the map they leave"""
    m, ctx = forced_small, forced_small["ctx"]
    big = np.concatenate([m["map"]] * 3)  # more surfels: a graph of other nodes than the one the fixture's frames sampled
    ctx.map_upload(big)
    cfg = cam_cfg(K_LOOP, FORCED_SMALL)
    cfg.rgb_only = int(kind == "rgb_only")
    cam = ctx.camera(cfg)
    try:
        for k, (rgb, depth) in enumerate(m["frames"][:3]):
            cam.frame(rgb, depth, 12 + k, T_wc=m["T"] if k == 0 else None, fuse=(kind != "fuse_0"))
            info, graph = cam.deform_result()
            after = ctx.map_download()
            assert not info["solved"] and not info["applied"], k
            assert np.array_equal(graph, sample_graph(after)), k
        assert after.tobytes() == big.tobytes()  # neither writes a surfel
    finally:
        cam.close()


def test_config_and_state_errors(forced_small):
    m, ctx = forced_small, forced_small["ctx"]
    L, C = capi.lib(), capi.C
    h = C.c_void_p()
    for mode in (0, 1):
        other = make_ctx(K_LOOP, close_loops=mode, capacity=100_000)
        try:
            assert L.ef_camera_create(other.h_ctx, C.byref(cam_cfg(K_LOOP, LOOP_CFG)), C.byref(h)) == EF_EINVAL, mode
            other.camera(cam_cfg(K_LOOP, LOOP_CFG, close_loops=False)).close()
        finally:
            other.close()
    for v in (2, -1):
        c = cam_cfg(K_LOOP, LOOP_CFG)
        c.close_loops = v
        assert L.ef_camera_create(ctx.h_ctx, C.byref(c), C.byref(h)) == EF_EINVAL, v
    open_cam = ctx.camera(cam_cfg(K_LOOP, LOOP_CFG, close_loops=False))
    closing = ctx.camera(cam_cfg(K_LOOP, LOOP_CFG))
    other = make_ctx(K_LOOP, close_loops=2, capacity=100_000)
    out, n = capi.EfLocalDeform(), C.c_int32()
    nodes = np.zeros((8, 4), np.float32)
    try:
        assert L.ef_camera_deform_result(ctx.h_ctx, open_cam.h_cam, C.byref(out), capi._p(nodes), 8, C.byref(n)) == EF_ESTATE
        assert L.ef_camera_deform_result(other.h_ctx, closing.h_cam, C.byref(out), capi._p(nodes), 8, C.byref(n)) == EF_EINVAL
        assert L.ef_camera_deform_result(ctx.h_ctx, closing.h_cam, None, capi._p(nodes), 8, C.byref(n)) == EF_EINVAL
        assert L.ef_camera_deform_result(ctx.h_ctx, closing.h_cam, C.byref(out), None, 8, C.byref(n)) == EF_EINVAL
        assert L.ef_camera_deform_result(ctx.h_ctx, closing.h_cam, C.byref(out), capi._p(nodes), -1, C.byref(n)) == EF_EINVAL
        assert L.ef_camera_deform_result(ctx.h_ctx, closing.h_cam, C.byref(out), None, 0, None) == 0
        assert not out.solved and not out.applied
    finally:
        open_cam.close()
        closing.close()
        other.close()


def test_destroy_frees_closing_cameras():
    import torch

    K = synth.K_DEFAULT
    free0 = torch.cuda.mem_get_info()[0]
    for _ in range(3):
        ctx = make_ctx(K, close_loops=2, capacity=100_000)
        for name in ("1920x1080", "1280x720"):
            Kb = FORCED_CAMERAS[name][0]
            ctx.camera(cam_cfg(Kb, LOOP_CFG))  # freed by ef_destroy
        cam = ctx.camera(cam_cfg(Kb, LOOP_CFG))
        cam.close()  # freed by ef_camera_destroy
        ctx.close()
    torch.cuda.synchronize()
    lost = free0 - torch.cuda.mem_get_info()[0]
    print("device memory not returned after 3 contexts with live closing cameras:", lost)
    assert lost < 64 << 20
