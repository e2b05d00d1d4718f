"""ef_rig_* on the GPU: cameras tracked as one rigid body. A one-member rig equals its camera byte for byte; two identical members
solve exactly twice one system; the joint update solves the members' systems mapped through the adjoint and keeps the rig rigid; the
rig tracks about as well as its cameras alone; the frame is untouched; and the calls follow the header's rules."""
import ctypes

import numpy as np
import pytest

from util import assert_same

from elasticfusion_b200 import capi, synth
from test_gpu_camera import PRED, cam_cfg, ctx_for, set_frame
from test_gpu_track_view import CAMERAS, FRAME_TEX, assert_bytes, b_frame, cam_offset, frame_state

pytestmark = pytest.mark.gpu
EF_EINVAL, EF_ESTATE = -1, -3
N_FRAMES = 10
SETTINGS = {"default": {}, "no_so3": dict(so3=False), "fast_odom": dict(fast_odom=True), "no_pyramid": dict(pyramid=False),
            "icp_only": dict(icp_weight=100.0), "frame_to_frame_rgb": dict(frame_to_frame_rgb=True)}


@pytest.fixture
def no_cluster(monkeypatch):
    """contexts whose frames and cameras run every Gauss-Newton iteration as launches, as a rig does"""
    monkeypatch.setenv("EF_GN_CLUSTER", "0")


def first_map(Kb, frames, settings):
    B = ctx_for(Kb, 4_000_000)
    try:
        set_frame(B, settings)
        B.process_frame(frames[0][0], frames[0][1], 0)
        return dict(map=B.map_download(), T=B.get_pose())
    finally:
        B.close()


def member_run(Kb, frames, settings, first, as_rig):
    """camera_run of test_gpu_camera with the camera alone or as a one-member rig"""
    KA = synth.K_DEFAULT
    own = next(synth.sequence(1, KA, seed=7, noise=True))
    A = ctx_for(KA, 4_000_000)
    out = []
    try:
        A.process_frame(own[0], own[1], 0)
        A.map_upload(first["map"])
        cam = A.camera(cam_cfg(Kb, settings))
        rig = A.rig([cam]) if as_rig else None
        for k, (rgb, depth, _) in enumerate(frames):
            kw = dict(T_wc=first["T"], fuse=False) if k == 0 else dict(max_trace=48)
            if as_rig:
                (res,), _ = rig.frame([(rgb, depth)], 1 if k == 0 else k + 1, **kw)
            else:
                res = cam.frame(rgb, depth, 1 if k == 0 else k + 1, **kw)
            T, st, cov, info, tr = res
            out.append(dict(T=T, stats=st, cov=cov, info=info, trace=tr, map=A.map_download(), pred={b: cam.download(b) for b in PRED}))
        if rig:
            rig.close()
        cam.close()
    finally:
        A.close()
    return out


@pytest.mark.parametrize("cam", ["424x240", "330x246"])
@pytest.mark.parametrize("setting", sorted(SETTINGS))
def test_one_member_rig_equals_camera(cam, setting, no_cluster):
    Kb, s = CAMERAS[cam], SETTINGS[setting]
    frames = list(synth.sequence(N_FRAMES, Kb, seed=11, noise=True))
    first = first_map(Kb, frames, s)
    ref = member_run(Kb, frames, s, first, False)
    got = member_run(Kb, frames, s, first, True)
    for k, (g, r) in enumerate(zip(got, ref)):
        w = f"{cam} {setting} call {k + 1}"
        assert_same(g["T"], r["T"], f"{w} pose")
        assert_bytes(g["stats"], r["stats"], f"{w} stats")
        assert_same(g["cov"], r["cov"], f"{w} covariance")
        assert g["info"] == r["info"], w
        assert_bytes(g["trace"], r["trace"], f"{w} trace")
        assert g["map"].tobytes() == r["map"].tobytes(), f"{w} map"
        for b in PRED:
            assert_same(g["pred"][b], r["pred"][b], f"{w} {b}")
    assert len(got[-1]["trace"]) > 0


def test_two_identical_members_are_one(no_cluster):
    """members 0 and 1 with the same camera, T_01 = I and the same inputs, fuse = 0 on an uploaded map: the joint system is exactly
    twice one member's, its LDL^T solve is exact under that power-of-two scale, so the poses equal the one-member rig's"""
    Kb = CAMERAS["424x240"]
    frames = list(synth.sequence(6, Kb, seed=11, noise=True))
    first = first_map(Kb, frames, {})
    runs = []
    for n in (1, 2):
        KA = synth.K_DEFAULT
        own = next(synth.sequence(1, KA, seed=7, noise=True))
        A = ctx_for(KA, 4_000_000)
        try:
            A.process_frame(own[0], own[1], 0)
            A.map_upload(first["map"])
            cams = [A.camera(cam_cfg(Kb)) for _ in range(n)]
            rig = A.rig(cams)
            out = []
            for k, (rgb, depth, _) in enumerate(frames):
                kw = dict(T_wc=first["T"]) if k == 0 else dict(max_trace=48)
                out.append(rig.frame([(rgb, depth)] * n, k + 1, fuse=False, **kw))
            runs.append(out)
            assert A.map_download().tobytes() == first["map"].tobytes()
        finally:
            A.close()
    for k, ((one, r1), (two, r2)) in enumerate(zip(*runs)):
        assert_same(r2[0], r1[0], f"frame {k} rig pose")
        for m in range(2):
            assert_same(two[m][0], one[0][0], f"frame {k} member {m} pose")
        if k == 0:
            continue
        assert_same(r2[1], 2.0 * two[1][1]["lastA"].reshape(6, 6), f"frame {k} joint lastA")
        assert_same(r2[2], 2.0 * two[1][1]["lastb"], f"frame {k} joint lastb")
        assert_same(r1[1], one[0][1]["lastA"].reshape(6, 6), f"frame {k} one-member lastA")
        t0, t1 = two[0][4], two[1][4]
        t0 = t0[t0["kind"] == 0]
        assert len(t0) == len(t1) > 0
        assert_same(t0["result"], t1["result"], f"frame {k} joint result")
        assert_same(t0["lastA"], t1["lastA"], f"frame {k} own systems")


def rig_scene(n, seed=9):
    """the rig_inputs scene of test_gpu_camera: member 0 a 320x240 camera A on the room trajectory, member 1 the 424x240 camera B at
    T_AB = cam_offset(); ground truth of both"""
    KA, Kb, T_AB = synth.Intrinsics(320, 240, 264.0, 264.0, 160.0, 120.0), CAMERAS["424x240"], cam_offset()
    frames = list(synth.sequence(n, KA, seed=seed, noise=True))
    traj = synth.trajectory(n, seed=seed)
    T0inv = np.linalg.inv(traj[0])
    bframes = [b_frame(traj[i], Kb, T_AB, 500 + i) for i in range(n)]
    truth = [[T0inv @ traj[i], T0inv @ traj[i] @ T_AB] for i in range(n)]
    return KA, Kb, T_AB, frames, bframes, truth


def rig_scene_run(n, joint):
    """Context A initialised by A's frame 0, then each frame through a rig of cameras A and B (joint) or through both cameras alone,
    all at time i + 1 (the first at the true pose). Returns per frame the members' results and the rig result (joint only)."""
    KA, Kb, T_AB, frames, bframes, truth = rig_scene(n)
    ctx = ctx_for(KA, 400_000, time_delta=200)
    out = []
    try:
        ctx.process_frame(frames[0][0], frames[0][1], 0)
        ca = ctx.camera(capi.camera_config(KA.width, KA.height, KA.fx, KA.fy, KA.cx, KA.cy, time_delta=200))
        cb = ctx.camera(capi.camera_config(Kb.width, Kb.height, Kb.fx, Kb.fy, Kb.cx, Kb.cy, time_delta=200))
        rig = ctx.rig([ca, cb], [np.eye(4), T_AB]) if joint else None
        for i in range(n):
            inputs = [(frames[i][0], frames[i][1]), bframes[i]]
            if joint:
                out.append(rig.frame(inputs, i + 1, T_wc=truth[0][0] if i == 0 else None, max_trace=48))
            else:
                out.append(([c.frame(*x, i + 1, T_wc=truth[0][m] if i == 0 else None) for m, (c, x) in enumerate(zip((ca, cb), inputs))], None))
    finally:
        ctx.close()
    return out, truth, T_AB


@pytest.fixture(scope="module")
def rig30():
    return rig_scene_run(30, True)


def adjoint(T):
    R, p = T[:3, :3], T[:3, 3]
    px = np.array([[0, -p[2], p[1]], [p[2], 0, -p[0]], [-p[1], p[0], 0]])
    Ad = np.zeros((6, 6))
    Ad[:3, :3], Ad[:3, 3:], Ad[3:, 3:] = R, px @ R, R
    return Ad


def test_joint_solve_matches_float64_restatement(rig30):
    out, _, T_AB = rig30
    Ad1 = adjoint(np.linalg.inv(T_AB))
    w = 10.0
    worst, checked = 0.0, 0
    for i, (members, rig) in enumerate(out):
        T0, T1 = members[0][0], members[1][0]
        assert np.abs(T1 - T0 @ T_AB).max() <= 1e-12, (i, np.abs(T1 - T0 @ T_AB).max())
        assert_same(rig[0], T0, f"frame {i} rig pose")
        if i == 0:
            assert not rig[4]
            continue
        tr0, tr1 = members[0][4], members[1][4]
        tr0 = tr0[tr0["kind"] == 0]
        assert len(tr0) == len(tr1) == 19, (i, len(tr0), len(tr1))
        for r0, r1 in zip(tr0, tr1):
            A, b = np.zeros((6, 6)), np.zeros(6)
            for r, Ad in ((r0, np.eye(6)), (r1, Ad1)):
                Am = r["A_rgb"].astype(np.float64).reshape(6, 6) + w * w * r["A_icp"].astype(np.float64).reshape(6, 6)
                bm = r["b_rgb"].astype(np.float64) + w * r["b_icp"].astype(np.float64)
                assert np.allclose(Am, r["lastA"].reshape(6, 6), rtol=1e-12, atol=0) and np.allclose(bm, r["lastb"], rtol=1e-12, atol=0)
                A += Ad.T @ Am @ Ad
                b += Ad.T @ bm
            x = r0["result"]
            assert_same(r1["result"], x, f"frame {i} result")
            res = float(np.abs(A @ x - b).max() / np.abs(b).max())
            worst = max(worst, res)
            checked += 1
    print(f"joint solve: {checked} iterations, worst relative residual {worst:.2e}")
    assert worst <= 1e-9


def test_rig_accuracy(rig30):
    """Translation RMSE of both members against ground truth, jointly and as two independent cameras on the same map. The bar (rig <=
    independent + 2 mm per member) is a guess made before any measurement."""
    out, truth, _ = rig30
    solo, _, _ = rig_scene_run(30, False)
    rmse = {}
    for mode, run in (("rig", out), ("independent", solo)):
        for m in range(2):
            est = np.array([r[0][m][0] for r in run])
            rmse[mode, m] = synth.ate_rmse(est, np.array([t[m] for t in truth])) * 1000
    print("translation RMSE (mm): " + ", ".join(f"{mode} member {m}: {v:.2f}" for (mode, m), v in rmse.items()))
    for m in range(2):
        assert rmse["rig", m] <= rmse["independent", m] + 2.0, rmse


def frame_rig_run(close_loops, n=12, rig_maps=None):
    """Frame A (320x240) with a rig of cameras B (424x240) and C (330x246) after each frame (time = tick - 1). close_loops = 2 runs the
    look-ahead and the rig's device call between ef_process_frame_device and ef_finish_frame. rig_maps: instead of each rig call, upload
    that map. Returns the frame's states and the map after each rig call."""
    import torch

    KA, Kb, T_AB, frames, bframes, truth = rig_scene(n)
    Kc, T_AC = CAMERAS["330x246"], cam_offset(-6.0, (-0.04, 0.02, 0.01))
    traj = synth.trajectory(n, seed=9)
    cframes = [b_frame(traj[i], Kc, T_AC, 900 + i) for i in range(n)]
    T_BC = np.linalg.inv(T_AB) @ T_AC
    ctx = ctx_for(KA, 400_000, time_delta=200, close_loops=close_loops)
    states, after = [], []
    dev = lambda a: torch.from_numpy(np.ascontiguousarray(a) if a.dtype != np.uint16 else np.ascontiguousarray(a).view(np.int16)).cuda()
    fdev = [(dev(r), dev(d)) for r, d, _ in frames]
    rdev = [[(dev(r), dev(d)) for r, d in (bframes[i], cframes[i])] for i in range(n)]
    members = torch.zeros(2 * ctypes.sizeof(capi.EfCameraResult), dtype=torch.uint8, device="cuda")
    result = torch.zeros(ctypes.sizeof(capi.EfRigResult), dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()
    try:
        cams = [ctx.camera(capi.camera_config(K.width, K.height, K.fx, K.fy, K.cx, K.cy, time_delta=200)) for K in (Kb, Kc)]
        rig = ctx.rig(cams, [np.eye(4), T_BC])
        if close_loops == 2:
            ctx.prefetch_frame_device(fdev[0][0].data_ptr(), fdev[0][1].data_ptr())
        for i in range(n):
            pose = truth[0][1] if i == 0 else None
            if close_loops == 2:
                ctx.process_frame_device(None, None, i)
                if i + 1 < n:
                    ctx.prefetch_frame_device(fdev[i + 1][0].data_ptr(), fdev[i + 1][1].data_ptr())
                if rig_maps is None:
                    rig.frame_device([r.data_ptr() for r, _ in rdev[i]], [d.data_ptr() for _, d in rdev[i]], members.data_ptr(),
                                     result.data_ptr(), i + 1, T_wc=pose)
                else:
                    ctx.map_upload(rig_maps[i])
                ctx.finish_frame()
            else:
                ctx.process_frame(frames[i][0], frames[i][1], i)
                if rig_maps is None:
                    rig.frame([bframes[i], cframes[i]], ctx.get_tick() - 1, T_wc=pose)
                else:
                    ctx.map_upload(rig_maps[i])
            after.append(ctx.map_download())
            states.append(frame_state(ctx, close_loops))
    finally:
        ctx.close()
    return states, after


@pytest.mark.parametrize("close_loops", [0, 2])
def test_frame_untouched_by_rig(close_loops):
    states, after = frame_rig_run(close_loops)
    assert after[-1].shape[0] > 0
    replay, _ = frame_rig_run(close_loops, rig_maps=after)
    names = ["pose", "tick", "dense", "map", "odom_stats 0", "odom_stats 1"] + list(FRAME_TEX)
    for i, (sa, sb) in enumerate(zip(states, replay)):
        for k, (x, y) in enumerate(zip(sa, sb)):
            assert x == y, (close_loops, i, names[k] if k < len(names) else k)


def test_host_and_device_calls_agree():
    """ef_rig_frame and ef_rig_frame_device give the same members' results, rig result and map, bit for bit, fused and not"""
    import torch

    n = 5
    KA, Kb, T_AB, frames, bframes, truth = rig_scene(n)
    dev = lambda a: torch.from_numpy(np.ascontiguousarray(a) if a.dtype != np.uint16 else np.ascontiguousarray(a).view(np.int16)).cuda()
    outs = []
    for device in (False, True):
        ctx = ctx_for(KA, 400_000, time_delta=200)
        got = []
        try:
            ctx.process_frame(frames[0][0], frames[0][1], 0)
            ca = ctx.camera(capi.camera_config(KA.width, KA.height, KA.fx, KA.fy, KA.cx, KA.cy, time_delta=200))
            cb = ctx.camera(capi.camera_config(Kb.width, Kb.height, Kb.fx, Kb.fy, Kb.cx, Kb.cy, time_delta=200))
            rig = ctx.rig([ca, cb], [np.eye(4), T_AB])
            members = torch.zeros(2 * ctypes.sizeof(capi.EfCameraResult), dtype=torch.uint8, device="cuda")
            result = torch.zeros(ctypes.sizeof(capi.EfRigResult), dtype=torch.uint8, device="cuda")
            for i in range(n):
                inputs = [(frames[i][0], frames[i][1]), bframes[i]]
                pose, fuse = (truth[0][0] if i == 0 else None), i != 2
                if device:
                    t = [(dev(r), dev(d)) for r, d in inputs]
                    torch.cuda.synchronize()
                    rig.frame_device([r.data_ptr() for r, _ in t], [d.data_ptr() for _, d in t], members.data_ptr(), result.data_ptr(), i + 1,
                                     T_wc=pose, fuse=fuse)
                    ctx.sync()
                    mb = members.cpu().numpy().tobytes()
                    sz = ctypes.sizeof(capi.EfCameraResult)
                    got.append(([capi.unpack_camera_result(mb[m * sz:(m + 1) * sz]) for m in range(2)],
                                capi.unpack_rig_result(result.cpu().numpy().tobytes()), ctx.map_download()))
                else:
                    res, r = rig.frame(inputs, i + 1, T_wc=pose, fuse=fuse)
                    got.append(([x[:4] for x in res], r, ctx.map_download()))
        finally:
            ctx.close()
        outs.append(got)
    for i, (h, d) in enumerate(zip(*outs)):
        for m in range(2):
            assert_same(h[0][m][0], d[0][m][0], f"{i} pose {m}")
            assert_bytes(h[0][m][1], d[0][m][1], f"{i} stats {m}")
            assert_same(h[0][m][2], d[0][m][2], f"{i} covariance {m}")
            assert h[0][m][3] == d[0][m][3], i
        for a, b in zip(h[1], d[1]):
            assert_same(a, b, f"{i} rig result")
        assert h[2].tobytes() == d[2].tobytes(), i


def test_rules_and_release():
    """every EF_EINVAL / EF_ESTATE rule of ef_rig_*, and the rig freed by ef_rig_destroy, ef_camera_destroy of a member and ef_destroy"""
    lib, C = capi.lib(), ctypes
    KA, Kb, T_AB, frames, bframes, truth = rig_scene(2)
    ctx = ctx_for(KA, 400_000, time_delta=200)
    other = ctx_for(KA, 100_000)
    try:
        cfg = lambda K, **kw: capi.camera_config(K.width, K.height, K.fx, K.fy, K.cx, K.cy, **kw)
        ca, cb = ctx.camera(cfg(KA)), ctx.camera(cfg(Kb))
        foreign = other.camera(cfg(Kb))

        def create(cams, ext=None):
            c = capi.EfRigConfig()
            c.n = len(cams)
            for i, cam in enumerate(cams):
                c.cameras[i] = cam.h_cam.value
                c.T_0i[i][:] = (np.eye(4) if ext is None else ext[i]).reshape(16).tolist()
            h = C.c_void_p()
            return lib.ef_rig_create(ctx.h_ctx, C.byref(c), C.byref(h)), h

        assert create([])[0] == EF_EINVAL
        assert create([ca, ca])[0] == EF_EINVAL
        assert create([ca, foreign])[0] == EF_EINVAL
        shear = np.eye(4)
        shear[0, 1] = 1e-3
        assert create([ca, cb], [np.eye(4), shear])[0] == EF_EINVAL
        bad_row = np.eye(4)
        bad_row[3, 0] = 1.0
        assert create([ca, cb], [np.eye(4), bad_row])[0] == EF_EINVAL
        nan = np.eye(4)
        nan[0, 3] = np.nan
        assert create([ca, cb], [np.eye(4), nan])[0] == EF_EINVAL
        assert create([ca, cb], [T_AB, np.eye(4)])[0] == EF_EINVAL  # T_0i[0] is not the identity
        for kw in (dict(icp_weight=5.0), dict(pyramid=False), dict(fast_odom=True), dict(so3=False), dict(rgb_only=True)):
            odd = ctx.camera(cfg(Kb, **kw))
            assert create([ca, odd])[0] == EF_EINVAL, kw
            odd.close()
        # a close_loops member needs a close_loops = 2 context
        loops_ctx = ctx_for(KA, 100_000, close_loops=2)
        try:
            lc, lo = loops_ctx.camera(cfg(Kb, close_loops=True)), loops_ctx.camera(cfg(Kb))
            c = capi.EfRigConfig()
            c.n = 2
            c.cameras[0], c.cameras[1] = lo.h_cam.value, lc.h_cam.value
            c.T_0i[0][:] = c.T_0i[1][:] = np.eye(4).reshape(16).tolist()
            assert lib.ef_rig_create(loops_ctx.h_ctx, C.byref(c), C.byref(C.c_void_p())) == EF_EINVAL
        finally:
            loops_ctx.close()

        rig = ctx.rig([ca, cb], [np.eye(4), T_AB])
        assert create([cb])[0] == EF_EINVAL  # a camera belongs to at most one rig
        inputs = [(frames[0][0], frames[0][1]), bframes[0]]
        with pytest.raises(capi.EfError, match=r"\(-3\)"):
            rig.frame(inputs, 1, fuse=False)  # the first frame must set the pose
        with pytest.raises(capi.EfError, match=r"\(-3\)"):
            rig.frame(inputs, 1, T_wc=np.eye(4))  # fuse before the context's first frame
        rig.frame(inputs, 1, T_wc=np.eye(4), fuse=False)
        with pytest.raises(capi.EfError, match=r"\(-3\)"):
            cb.frame(*bframes[0], 1, fuse=False)  # a member's own frames wait for ef_rig_destroy
        for bad in (dict(time=-1), dict(weight_multiplier=-1.0), dict(weight_multiplier=float("nan")), dict(T_wc=np.full((4, 4), np.inf))):
            args = dict(time=2, weight_multiplier=1.0, T_wc=None) | bad
            with pytest.raises(capi.EfError, match=r"\(-1\)"):
                rig.frame(inputs, args["time"], args["weight_multiplier"], args["T_wc"], fuse=False)
        f = capi.rig_frame(2, fuse=False)
        members, out = (capi.EfCameraResult * 2)(), capi.EfRigResult()
        r, d = np.ascontiguousarray(inputs[0][0]), np.ascontiguousarray(inputs[0][1])
        ptrs = lambda *a: (C.c_void_p * 2)(*a)
        assert lib.ef_rig_frame(ctx.h_ctx, rig.h_rig, C.byref(f), ptrs(r.ctypes.data, None), ptrs(d.ctypes.data, d.ctypes.data), members,
                                C.byref(out), None, 0, None) == EF_EINVAL
        assert lib.ef_rig_frame(ctx.h_ctx, rig.h_rig, C.byref(f), ptrs(r.ctypes.data, r.ctypes.data), ptrs(d.ctypes.data, d.ctypes.data),
                                members, C.byref(out), None, -1, None) == EF_EINVAL
        assert lib.ef_rig_frame(other.h_ctx, rig.h_rig, C.byref(f), ptrs(r.ctypes.data, r.ctypes.data), ptrs(d.ctypes.data, d.ctypes.data),
                                members, C.byref(out), None, 0, None) == EF_EINVAL
        assert lib.ef_rig_frame_device(ctx.h_ctx, rig.h_rig, C.byref(f), ptrs(1, 1), ptrs(3, 3), 8, 8) == EF_EINVAL  # unaligned depth
        assert lib.ef_rig_destroy(other.h_ctx, rig.h_rig) == EF_EINVAL
        assert cb.download("IMAGE").shape == (Kb.height, Kb.width, 4)  # ef_camera_buffer still works on members
        # released by ef_rig_destroy: the members run alone again
        rig.close()
        cb.frame(*bframes[0], 1, T_wc=truth[0][1], fuse=False)
        # ... by ef_camera_destroy of a member
        rig2 = ctx.rig([ca, cb], [np.eye(4), T_AB])
        h = rig2.h_rig
        ca.close()
        assert lib.ef_rig_destroy(ctx.h_ctx, h) == EF_EINVAL
        cb.frame(*bframes[0], 1, T_wc=truth[0][1], fuse=False)
        # ... and by ef_destroy (a rig still live when its context goes)
        ctx.rig([cb], [np.eye(4)])
    finally:
        ctx.close()
        other.close()
