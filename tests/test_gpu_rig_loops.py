"""ef_rig_* with closing members on the GPU: a rig whose members all have close_loops = 1 closes local loops as one body. A one-member
closing rig equals its closing camera byte for byte; on a two-member rig the joint acceptance test, the concatenated constraints and the
one deformation solve agree with what the rig reports and the rig stays rigid through its closures; forced closures on a four-member rig
solve every call; the frame sees exactly the map and bookkeeping the rig leaves; and the new calls follow the header's rules."""
import numpy as np
import pytest

from test_gpu_camera import PRED
from test_gpu_camera_loops import (FORCED, K_LOOP, LOOP_CAMERAS, RIG_B, applied_closures, cam_cfg, compare_runs, digest, inactive_copy,
                                   make_ctx, record, rig_inputs)
from test_gpu_loop_closure import LOOP_CFG, N_FRAMES, sample_graph
from test_gpu_track_view import _k, assert_bytes, b_frame, cam_offset
from util import assert_same

from elasticfusion_b200 import capi, synth

pytestmark = pytest.mark.gpu
EF_EINVAL, EF_ESTATE = -1, -3


@pytest.fixture
def no_cluster(monkeypatch):
    """contexts whose frames and cameras run every Gauss-Newton iteration as launches, as a rig does"""
    monkeypatch.setenv("EF_GN_CLUSTER", "0")


def grid(K):
    return (K.width // 20) * (K.height // 20)


# ---- 1. a one-member closing rig is its closing camera ---------------------------------------------------------------------------------
def first_loop_map(Kb, frames, cfg):
    B = make_ctx(Kb, close_loops=2, **cfg)
    try:
        B.process_frame(frames[0][0], frames[0][1], 0)
        return dict(map=B.map_download(), T=B.get_pose())
    finally:
        B.close()


def member_run(Kb, frames, cfg, first, as_rig):
    """camera_run of test_gpu_camera_loops with the closing camera alone or as a one-member rig"""
    KA = synth.K_DEFAULT
    own = next(synth.sequence(1, KA, seed=7, noise=True))
    A = make_ctx(KA, close_loops=2, **cfg)
    out = []
    try:
        A.process_frame(own[0], own[1], 0)
        A.map_upload(first["map"])
        cam = A.camera(cam_cfg(Kb, cfg))
        rig = A.rig([cam]) if as_rig else None
        for k, (rgb, depth, _) in enumerate(frames):
            kw = dict(T_wc=first["T"], fuse=False) if k == 0 else {}
            if as_rig:
                (res,), _ = rig.frame([(rgb, depth)], 1 if k == 0 else k + 1, **kw)
                deform = rig.deform_result()
            else:
                res = cam.frame(rgb, depth, 1 if k == 0 else k + 1, **kw)
                deform = cam.deform_result()
            T, st, cov, info, _ = res
            out.append(record(info["dense_enough"], T, st, cov, A.map_download(), {b: cam.download(b) for b in PRED}, deform))
        if rig:
            rig.close()
        cam.close()
    finally:
        A.close()
    return out


@pytest.mark.parametrize("cam", sorted(LOOP_CAMERAS))
def test_one_member_rig_equals_closing_camera(cam, no_cluster):
    """130 frames of the loop sequence: after every call, pose, stats, covariance, dense_enough, map, prediction, deform result and graph"""
    Kb = LOOP_CAMERAS[cam]
    frames = list(synth.sequence(N_FRAMES, Kb, seed=21, noise=True, speed=2.5))
    first = first_loop_map(Kb, frames, LOOP_CFG)
    ref = member_run(Kb, frames, LOOP_CFG, first, as_rig=False)
    got = member_run(Kb, frames, LOOP_CFG, first, as_rig=True)
    compare_runs(got, ref, cam)
    applied = applied_closures(got)
    print(cam, "applied closures:", applied)
    assert len(applied) >= 1, cam


# ---- 2. a two-member closing rig over the loop sequence --------------------------------------------------------------------------------
def rig_loop_inputs(n):
    """member 0 on the loop sequence (320x240), member 1 (424x240) at cam_offset(); the members' true poses"""
    frames, bframes, _ = rig_inputs(n)
    traj = synth.trajectory(n, seed=21, speed=2.5)
    T0inv = np.linalg.inv(traj[0])
    truth0 = [T0inv @ traj[i] for i in range(n)]
    return [[f[:2], b] for f, b in zip(frames, bframes)], truth0


def record_rig_call(ctx, rig, res, closing):
    rec = dict(T=[r[0] for r in res], stats=[r[1] for r in res], map=digest(ctx.map_download()))
    if closing:
        rec["loop"] = rig.loop_result()
        rec["deform"] = rig.deform_result()
    return rec


def two_member_run(closing, n=N_FRAMES, cfg=LOOP_CFG):
    """a 320x240 context (close_loops = 2) after its first loop frame; then the rig at that pose (fuse = 0, time 1) and at times 2, 3, ..."""
    inputs, _ = rig_loop_inputs(n)
    ctx = make_ctx(K_LOOP, close_loops=2, **cfg)
    out = []
    try:
        ctx.process_frame(inputs[0][0][0], inputs[0][0][1], 0)
        cams = [ctx.camera(cam_cfg(K, cfg, closing)) for K in (K_LOOP, RIG_B)]
        rig = ctx.rig(cams, [np.eye(4), cam_offset()])
        T0 = ctx.get_pose()
        for k in range(n):
            kw = dict(T_wc=T0, fuse=False) if k == 0 else {}
            res, _ = rig.frame(inputs[k], k + 1, **kw)
            out.append(record_rig_call(ctx, rig, res, closing))
        # the solves, restated from what the rig reported: the graph the previous call left, its bookkeeping, the reported constraints
        for k in range(1, n if closing else 0):
            info, _ = out[k]["deform"]
            if info["solved"]:
                prev, graph = out[k - 1]["deform"]
                _, src, dst, tms, _ = out[k]["loop"]
                res, *_ = ctx.deform_solve(graph[:, :3], graph[:, 3].astype(np.int32), src, dst, np.full(len(src), k + 1, np.int32), tms,
                                           pin=prev["deforms"] == 0, last_deform_time=prev["last_deform_time"])
                out[k]["restated"] = res
        rig.close()
        for c in cams:
            c.close()
    finally:
        ctx.close()
    return out


def check_rig_closures(run, members, cfg, T_0i):
    """the checks every closing-rig run passes: rigid after every call, the reported acceptance, the constraints and the solve"""
    for k, r in enumerate(run):
        for i in range(1, len(members)):
            assert np.abs(r["T"][i] - r["T"][0] @ T_0i[i]).max() <= 1e-12, (k, i)
        info, src, dst, tms, counts = r["loop"]
        dinfo, _ = r["deform"]
        if not info["ran"]:
            assert not dinfo["solved"] and info["n_constraints"] == 0, k
            continue
        ok = (np.all(info["cov_diag"] <= float(np.float32(cfg["cov_thresh"]))) and info["lastICPCount"] > cfg["count_thresh"]
              and np.float32(info["lastICPError"]) < np.float32(cfg["err_thresh"]))
        assert bool(info["accepted"]) == bool(ok), (k, info)
        assert counts.sum() == info["n_constraints"] == len(src), (k, counts, info["n_constraints"])
        assert all(c <= grid(K) for c, K in zip(counts, members)), (k, counts)
        if len(src):
            M = info["T_wc_est"] @ np.linalg.inv(info["T_wc_curr"])  # T_est_i T_curr_i^-1 is the same for every member
            want = src @ M[:3, :3].T + M[:3, 3]
            assert np.abs(dst - want).max() <= 1e-9 * max(1.0, np.abs(dst).max()), k
        assert dinfo["applied"] == (dinfo["solved"] and dinfo["result"]["stop"] != 6), k
        if dinfo["solved"]:
            assert dinfo["result"] == r["restated"], (k, dinfo["result"], r["restated"])


@pytest.fixture(scope="module")
def two_member():
    return two_member_run(True), two_member_run(False)


def test_two_member_rig_closes_loops(two_member):
    closing, open_rig = two_member
    T_0i = [np.eye(4), cam_offset()]
    check_rig_closures(closing, [K_LOOP, RIG_B], LOOP_CFG, T_0i)
    applied = [k for k, r in enumerate(closing) if r["deform"][0]["applied"]]
    accepted = [k for k, r in enumerate(closing) if r["loop"][0]["accepted"]]
    print("two-member rig: accepted at calls", accepted, "applied at calls", applied,
          "member constraints", [tuple(closing[k]["loop"][4]) for k in applied])
    assert applied, "the joint test accepted no closure on the loop sequence"
    for k in range(applied[0]):  # before the first closure: the open-loop rig, byte for byte
        a, b = closing[k], open_rig[k]
        assert a["map"] == b["map"], k
        for i in range(2):
            assert_same(a["T"][i], b["T"][i], f"call {k} member {i} pose")
            assert_bytes(a["stats"][i], b["stats"][i], f"call {k} member {i} stats")
    _, truth0 = rig_loop_inputs(len(closing))
    truth = [np.array(truth0), np.array([T @ T_0i[1] for T in truth0])]
    for name, run in (("closing", closing), ("open-loop", open_rig)):
        rmse = [synth.ate_rmse(np.array([r["T"][i] for r in run]), truth[i]) * 1000 for i in range(2)]
        print(f"{name} rig translation RMSE over {len(run)} calls: member 0 {rmse[0]:.3f} mm, member 1 {rmse[1]:.3f} mm")


# ---- 3. forced closures on a four-member rig --------------------------------------------------------------------------------------------
FOUR = [synth.K_DEFAULT, _k(424, 240, 305.0), _k(330, 246, 290.0, 150.0, 131.0, fy=272.0), _k(1280, 720, 915.0)]
FOUR_T = [np.eye(4), cam_offset(), cam_offset(-10.0, (-0.06, 0.02, 0.01)), cam_offset(4.0, (0.0, 0.05, -0.03))]


def test_forced_closures_on_four_members():
    n = 12
    cfg = dict(FORCED, capacity=4_000_000)
    traj = synth.trajectory(n, seed=21, speed=2.5)
    T0inv = np.linalg.inv(traj[0])
    inputs = [[b_frame(traj[i], K, T, 700 + 10 * i + m) for m, (K, T) in enumerate(zip(FOUR, FOUR_T))] for i in range(n)]
    ctx = make_ctx(synth.K_DEFAULT, close_loops=2, **cfg)
    run = []
    try:
        ctx.process_frame(inputs[0][0][0], inputs[0][0][1], 0)
        m = ctx.map_download()
        ctx.map_upload(np.concatenate([m, inactive_copy(m)]))
        cams = [ctx.camera(cam_cfg(K, cfg)) for K in FOUR]
        rig = ctx.rig(cams, FOUR_T)
        for k in range(n):
            kw = dict(T_wc=T0inv @ traj[0], fuse=False) if k == 0 else {}
            res, _ = rig.frame(inputs[k], k + 1, **kw)
            run.append(record_rig_call(ctx, rig, res, True))
        for k in range(1, n):
            if run[k]["deform"][0]["solved"]:
                prev, graph = run[k - 1]["deform"]
                _, src, dst, tms, _ = run[k]["loop"]
                run[k]["restated"] = ctx.deform_solve(graph[:, :3], graph[:, 3].astype(np.int32), src, dst, np.full(len(src), k + 1, np.int32),
                                                      tms, pin=prev["deforms"] == 0, last_deform_time=prev["last_deform_time"])[0]
        rig.close()
        for c in cams:
            c.close()
    finally:
        ctx.close()
    check_rig_closures(run, FOUR, cfg, FOUR_T)
    solved = [(k, r["deform"][0]["result"]["n_constraints"], tuple(r["loop"][4])) for k, r in enumerate(run) if r["deform"][0]["solved"]]
    print("four-member rig solves (call, constraints incl. pins, member constraints):", solved)
    assert set(range(4, n)) <= {k for k, _, _ in solved}  # (measured on an H100: from the third call on)
    assert all(r["deform"][0]["applied"] for r in run[4:])
    assert all(c <= 2 * sum(grid(K) for K in FOUR) for _, c, _ in solved)
    assert any(sum(1 for c in counts if c > 0) >= 2 for _, _, counts in solved)


# ---- 4. the frame and a closing rig on one map --------------------------------------------------------------------------------------------
RIG_C = LOOP_CAMERAS["330x246_offcentre"]
T_BC = cam_offset(-6.0, (-0.04, 0.01, 0.02))


def frame_rig_run(n=N_FRAMES):
    """the look-ahead frame (320x240), then the closing rig's device call (424x240 at cam_offset(), 330x246 beside it) between
    ef_process_frame_device and ef_finish_frame, time = tick - 1"""
    import torch

    frames, bframes, truth = rig_inputs(n)
    traj = synth.trajectory(n, seed=21, speed=2.5)
    cframes = [b_frame(traj[i], RIG_C, cam_offset() @ T_BC, 900 + i) for i in range(n)]

    def dev(a):
        return torch.from_numpy(np.ascontiguousarray(a).view(np.int16) if a.dtype == np.uint16 else np.ascontiguousarray(a)).cuda()

    ctx = make_ctx(K_LOOP, close_loops=2, **LOOP_CFG)
    fdev = [(dev(f[0]), dev(f[1])) for f in frames]
    mdev = [[(dev(b[0]), dev(b[1])), (dev(c[0]), dev(c[1]))] for b, c in zip(bframes, cframes)]
    members = torch.zeros(2 * capi.C.sizeof(capi.EfCameraResult), dtype=torch.uint8, device="cuda")
    out = torch.zeros(capi.C.sizeof(capi.EfRigResult), dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()
    cams = [ctx.camera(cam_cfg(K, LOOP_CFG)) for K in (RIG_B, RIG_C)]
    rig = ctx.rig(cams, [np.eye(4), T_BC])
    rec = []
    try:
        ctx.prefetch_frame_device(fdev[0][0].data_ptr(), fdev[0][1].data_ptr())
        for i in range(n):
            ctx.process_frame_device(None, None, i)
            m_frame = ctx.map_download()
            frame_deform = ctx.local_deform_result()[0]
            if i + 1 < n:
                ctx.prefetch_frame_device(fdev[i + 1][0].data_ptr(), fdev[i + 1][1].data_ptr())
            rig.frame_device([p[0].data_ptr() for p in mdev[i]], [p[1].data_ptr() for p in mdev[i]], members.data_ptr(), out.data_ptr(), i + 1,
                             T_wc=truth[0] if i == 0 else None)
            ctx.finish_frame()
            ctx.sync()
            rec.append(dict(pose=ctx.get_pose(), after_frame=digest(m_frame), map=ctx.map_download(), frame=frame_deform,
                            rig=rig.deform_result()[0], final=ctx.local_deform_result()))
    finally:
        rig.close()
        for c in cams:
            c.close()
        ctx.close()
    return rec


def test_frame_sees_the_map_the_rig_leaves():
    """the frame equals a close_loops = 1 context running the host recipe, in which each rig call is replaced by the upload of the map it
    left and its deforms / last_deform_time; deforms counts the applied closures of both sides"""
    rig = frame_rig_run()
    frames, _, _ = rig_inputs(len(rig))
    ctx = make_ctx(K_LOOP, close_loops=1, **LOOP_CFG)
    deforms, last, graph, events = 0, 0, None, []
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
                    events.append((i, "frame"))
            ctx.process_frame_end(T_over, nodes)
            assert np.array_equal(ctx.get_pose(), r["pose"]), i
            assert digest(ctx.map_download()) == r["after_frame"], i
            f = r["frame"]
            assert (f["solved"], f["applied"]) == (solved is not None, T_over is not None), i
            assert (f["deforms"], f["last_deform_time"]) == (deforms, last), i
            # the rig call, replayed
            if r["rig"]["applied"]:
                events.append((i, "rig"))
                deforms, last = deforms + 1, i + 1
            assert (r["rig"]["deforms"], r["rig"]["last_deform_time"]) == (deforms, last), i
            ctx.map_upload(r["map"])
            g = sample_graph(r["map"])
            if g is not None:
                graph = g
            assert np.array_equal(r["final"][1], graph if graph is not None else np.zeros((0, 4), np.float32)), i
    finally:
        ctx.close()
    print("applied closures (frame index, side):", events)


# ---- 5. calls and rules -------------------------------------------------------------------------------------------------------------------
FORCED_SMALL = dict(FORCED, capacity=800_000)


def forced_rig_calls(device, fuse=True):
    """a 320x240 context (close_loops = 2, every registration accepted) after 12 loop frames, then a closing rig (320x240 + 424x240):
    a has_pose call, then four more; per call the members' results, the map, the loop and deform results"""
    import torch

    frames = list(synth.sequence(16, K_LOOP, seed=21, noise=True, speed=2.5))
    traj = synth.trajectory(16, seed=21, speed=2.5)
    ctx = make_ctx(K_LOOP, close_loops=2, **FORCED_SMALL)
    out = []
    try:
        for i, (rgb, depth, _) in enumerate(frames[:12]):
            ctx.process_frame(rgb, depth, i)
        T = ctx.get_pose()
        if not fuse:  # more surfels: a graph of other nodes than the one the context's frames sampled
            ctx.map_upload(np.concatenate([ctx.map_download()] * 3))
        cams = [ctx.camera(cam_cfg(K, FORCED_SMALL)) for K in (K_LOOP, RIG_B)]
        rig = ctx.rig(cams, [np.eye(4), cam_offset()])
        members = torch.zeros(2 * capi.C.sizeof(capi.EfCameraResult), dtype=torch.uint8, device="cuda")
        res_dev = torch.zeros(capi.C.sizeof(capi.EfRigResult), dtype=torch.uint8, device="cuda")
        for k in range(5):
            inp = [frames[11 + k][:2], b_frame(traj[11 + k], RIG_B, cam_offset(), 600 + k)]
            kw = dict(T_wc=T if k == 0 else None, fuse=fuse)
            if device:
                t = [(torch.from_numpy(np.ascontiguousarray(r)).cuda(), torch.from_numpy(np.ascontiguousarray(d).view(np.int16)).cuda())
                     for r, d in inp]
                torch.cuda.synchronize()
                rig.frame_device([a.data_ptr() for a, _ in t], [b.data_ptr() for _, b in t], members.data_ptr(), res_dev.data_ptr(), 12 + k, **kw)
                ctx.sync()
                raw = members.cpu().numpy().tobytes()
                n = capi.C.sizeof(capi.EfCameraResult)
                res = [capi.unpack_camera_result(raw[i * n:(i + 1) * n])[:3] for i in range(2)]
                T_rig = capi.unpack_rig_result(res_dev.cpu().numpy().tobytes())[0]
            else:
                r, rr = rig.frame(inp, 12 + k, **kw)
                res, T_rig = [x[:3] for x in r], rr[0]
            out.append(dict(res=res, T_rig=T_rig, map=ctx.map_download(), loop=rig.loop_result(), deform=rig.deform_result()))
        rig.close()
        for c in cams:
            c.close()
    finally:
        ctx.close()
    return out


def test_host_and_device_calls_are_identical():
    runs = [forced_rig_calls(device) for device in (False, True)]
    for k, (a, b) in enumerate(zip(*runs)):
        for i in range(2):
            assert_same(a["res"][i][0], b["res"][i][0], f"call {k} member {i} pose")
            assert_bytes(a["res"][i][1], b["res"][i][1], f"call {k} member {i} stats")
            assert_same(a["res"][i][2], b["res"][i][2], f"call {k} member {i} covariance")
        assert_same(a["T_rig"], b["T_rig"], f"call {k} rig pose")
        assert np.array_equal(a["T_rig"], a["res"][0][0]), k  # the rig's pose is member 0's, closed or not
        assert a["map"].tobytes() == b["map"].tobytes(), k
        la, lb = a["loop"], b["loop"]
        assert all(np.array_equal(x, y) for x, y in zip(la[1:], lb[1:])), k
        assert {x: str(v) for x, v in la[0].items()} == {x: str(v) for x, v in lb[0].items()}, k
        assert a["deform"][0] == b["deform"][0] and np.array_equal(a["deform"][1], b["deform"][1]), k
    print("solved at calls", [k for k, a in enumerate(runs[0]) if a["deform"][0]["solved"]])
    assert any(a["deform"][0]["applied"] for a in runs[0])


def test_fuse_0_and_first_calls_sample_the_graph():
    run = forced_rig_calls(False, fuse=False)
    for k, r in enumerate(run):
        info, graph = r["deform"]
        assert not r["loop"][0]["ran"] and not info["solved"] and not info["applied"], k
        assert np.array_equal(graph, sample_graph(r["map"])), k


def test_rules_and_release():
    import torch

    L, C = capi.lib(), capi.C
    ctx = make_ctx(K_LOOP, close_loops=2, capacity=100_000)
    other = make_ctx(K_LOOP, close_loops=2, capacity=100_000)
    frames = list(synth.sequence(3, K_LOOP, seed=21, noise=True, speed=2.5))
    try:
        ctx.process_frame(frames[0][0], frames[0][1], 0)
        a, b = ctx.camera(cam_cfg(K_LOOP, LOOP_CFG)), ctx.camera(cam_cfg(RIG_B, LOOP_CFG))
        o1, o2 = ctx.camera(cam_cfg(K_LOOP, LOOP_CFG, False)), ctx.camera(cam_cfg(RIG_B, LOOP_CFG, False))
        open_rig = ctx.rig([o1, o2], [np.eye(4), cam_offset()])
        rig = ctx.rig([a, b], [np.eye(4), cam_offset()])
        lr, ld, n = capi.EfRigLoopResult(), capi.EfLocalDeform(), C.c_int32()
        nodes = np.zeros((8, 4), np.float32)
        buf = np.zeros((64, 3), np.float64)
        assert L.ef_rig_loop_result(ctx.h_ctx, open_rig.h_rig, C.byref(lr), None, None, None, 0, None) == EF_ESTATE
        assert L.ef_rig_deform_result(ctx.h_ctx, open_rig.h_rig, C.byref(ld), None, 0, None) == EF_ESTATE
        assert L.ef_rig_loop_result(other.h_ctx, rig.h_rig, C.byref(lr), None, None, None, 0, None) == EF_EINVAL
        assert L.ef_rig_deform_result(other.h_ctx, rig.h_rig, C.byref(ld), None, 0, None) == EF_EINVAL
        assert L.ef_rig_loop_result(ctx.h_ctx, None, C.byref(lr), None, None, None, 0, None) == EF_EINVAL
        assert L.ef_rig_loop_result(ctx.h_ctx, rig.h_rig, None, None, None, None, 0, None) == EF_EINVAL
        assert L.ef_rig_loop_result(ctx.h_ctx, rig.h_rig, C.byref(lr), capi._p(buf), None, None, -1, None) == EF_EINVAL
        assert L.ef_rig_deform_result(ctx.h_ctx, rig.h_rig, None, None, 0, None) == EF_EINVAL
        assert L.ef_rig_deform_result(ctx.h_ctx, rig.h_rig, C.byref(ld), None, 8, C.byref(n)) == EF_EINVAL
        assert L.ef_rig_deform_result(ctx.h_ctx, rig.h_rig, C.byref(ld), capi._p(nodes), -1, C.byref(n)) == EF_EINVAL
        assert L.ef_rig_loop_result(ctx.h_ctx, rig.h_rig, C.byref(lr), None, None, None, 0, None) == 0 and not lr.ran
        assert L.ef_rig_deform_result(ctx.h_ctx, rig.h_rig, C.byref(ld), None, 0, None) == 0 and not ld.solved
        assert L.ef_camera_deform_result(ctx.h_ctx, a.h_cam, C.byref(ld), None, 0, None) == EF_ESTATE
        # after ef_rig_destroy, a mixed rig is refused and the members close loops alone again
        open_rig.close()
        rig.close()
        cfg = capi.EfRigConfig()
        cfg.n = 2
        cfg.cameras[0], cfg.cameras[1] = o1.h_cam.value, b.h_cam.value
        cfg.T_0i[0][:] = np.eye(4).reshape(16).tolist()
        cfg.T_0i[1][:] = cam_offset().reshape(16).tolist()
        h = C.c_void_p()
        assert L.ef_rig_create(ctx.h_ctx, C.byref(cfg), C.byref(h)) == EF_EINVAL
        assert L.ef_camera_deform_result(ctx.h_ctx, a.h_cam, C.byref(ld), None, 0, None) == 0
        a.frame(frames[1][0], frames[1][1], 2, T_wc=ctx.get_pose())
        a.frame(frames[2][0], frames[2][1], 3)
        info, graph = a.deform_result()
        assert np.array_equal(graph, sample_graph(ctx.map_download()))
        # ef_camera_destroy of a member and ef_destroy free a closing rig
        rig2 = ctx.rig([a, b], [np.eye(4), cam_offset()])
        b.close()
        assert L.ef_rig_loop_result(ctx.h_ctx, rig2.h_rig, C.byref(lr), None, None, None, 0, None) == EF_EINVAL
        ctx.rig([a], [np.eye(4)])  # freed by ef_destroy
    finally:
        ctx.close()
        other.close()
    free0 = torch.cuda.mem_get_info()[0]
    for _ in range(3):
        c = make_ctx(synth.K_DEFAULT, close_loops=2, capacity=100_000)
        cams = [c.camera(cam_cfg(K, LOOP_CFG)) for K in FOUR]
        c.rig(cams, FOUR_T)
        c.close()
    torch.cuda.synchronize()
    lost = free0 - torch.cuda.mem_get_info()[0]
    print("device memory not returned after 3 contexts with live closing rigs:", lost)
    assert lost < 64 << 20
