"""close_loops = 2: local loop closures closed inside ef_process_frame (Core/ElasticFusion.cpp:447-534 and 593, Core/Deformation.cpp).

End-to-end comparisons against the CPU oracle are chaotic on the loop sequence (product and oracle drift millimetres apart and
disagree on some acceptances, see test_local_loop_front_half_over_a_sequence). So the mode is pinned bit for bit to the recipe a
closed-loop host runs with close_loops = 1 (INTEGRATION.md §3c), which is built from stages that are pinned one by one:
ef_process_frame_begin, ef_local_loop_result, the graph sampled from ef_map_download, ef_deform_solve and ef_process_frame_end."""
import hashlib
import os
import subprocess

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BIG = 2147483647 // 2
N_FRAMES = 130
# the loop sequence of test_local_loop_front_half_over_a_sequence
LOOP_CFG = dict(time_delta=12, count_thresh=3000, err_thresh=5e-5, cov_thresh=1e-4, capacity=400000)
# accept every registration: the edge cases below need an accepted front half, not a good one
ACCEPT_ALL = dict(count_thresh=0, err_thresh=1e30, cov_thresh=1e30)


def make_ctx(K, **kw):
    from elasticfusion_b200 import capi

    return capi.Context(capi.default_config(K.width, K.height, K.fx, K.fy, K.cx, K.cy, **kw))


def digest(m):
    return hashlib.sha256(np.ascontiguousarray(m).tobytes()).hexdigest()


def sample_graph(m):
    """Deformation::sampleGraphModel as a host restates it: x y z and colorTime.z of surfels 0, 5000, ..., at most 1023 nodes;
    None when 4 or fewer come out (the previous graph stays)."""
    s = m[::5000][:1023]
    return np.ascontiguousarray(s[:, [0, 1, 2, 6]]) if len(s) > 4 else None


@pytest.fixture(scope="module")
def loop_seq():
    from elasticfusion_b200 import synth

    K2 = synth.Intrinsics(320, 240, 264.0, 264.0, 160.0, 120.0)
    return K2, list(synth.sequence(N_FRAMES, K2, seed=21, noise=True, speed=2.5))


@pytest.fixture(scope="module")
def mode2_run(loop_seq):
    """Context A: close_loops = 2 through ef_process_frame. Per frame: pose, surfel count, map digest, graph, query result."""
    K2, frames = loop_seq
    ctx = make_ctx(K2, close_loops=2, **LOOP_CFG)
    rec = []
    try:
        for i, (rgb, depth, _) in enumerate(frames):
            ctx.process_frame(rgb, depth, i)
            m = ctx.map_download()
            info, graph = ctx.local_deform_result()
            rec.append(dict(pose=ctx.get_pose(), count=len(m), map=digest(m), graph=graph, info=info))
    finally:
        ctx.close()
    return rec


def test_mode2_equals_the_host_recipe_in_lockstep(loop_seq, mode2_run):
    """Context B runs close_loops = 1 with INTEGRATION.md §3c written out: begin, local_loop_result, the graph sampled from the
    previous frame's map, deform_solve(pin = deforms == 0, last_deform_time), end(T_wc_est, nodes), Deformation's bookkeeping.
    After every frame both contexts hold the same pose, surfels (bytes) and graph."""
    K2, frames = loop_seq
    ctx = make_ctx(K2, close_loops=1, **LOOP_CFG)
    deforms, last, graph = 0, 0, None
    applied = []
    try:
        for i, (rgb, depth, _) in enumerate(frames):
            ctx.process_frame_begin(rgb, depth, i)
            info, src, dst, tms = ctx.local_loop_result()
            T_over = nodes = None
            solved = None
            if info["ran"] and info["accepted"] and graph is not None and len(src) > 0:
                tick = ctx.get_tick()
                solved, nodes16, *_ = ctx.deform_solve(graph[:, :3], graph[:, 3].astype(np.int32), src, dst, np.full(len(src), tick, np.int32),
                                                       tms, pin=deforms == 0, last_deform_time=last)
                if solved["stop"] != 6:
                    T_over, nodes = info["T_wc_est"], nodes16
                    applied.append(dict(frame=i, pinned=deforms == 0, last_deform_time=last, stop=solved["stop"]))
                    deforms += 1
                    last = tick
            ctx.process_frame_end(T_over, nodes)
            m = ctx.map_download()
            g = sample_graph(m)
            if g is not None:
                graph = g
            a = mode2_run[i]
            assert np.array_equal(a["pose"], ctx.get_pose()), i
            assert a["count"] == len(m) and a["map"] == digest(m), i
            assert np.array_equal(a["graph"], graph if graph is not None else np.zeros((0, 4), np.float32)), i
            ia = a["info"]
            assert (ia["solved"], ia["applied"]) == (solved is not None, T_over is not None), i
            if solved is not None:
                assert ia["result"] == solved, i
            assert (ia["deforms"], ia["last_deform_time"], ia["n_nodes"]) == (deforms, last, 0 if graph is None else len(graph)), i
    finally:
        ctx.close()
    # the sequence closes loops more than once: the first closure pinned, a later one unpinned with an earlier closure's time fixed
    assert len(applied) >= 2, applied
    assert applied[0]["pinned"] and applied[0]["last_deform_time"] == 0, applied
    assert any(not a["pinned"] and a["last_deform_time"] > 0 for a in applied[1:]), applied


def test_mode2_with_lookahead_is_identical(loop_seq, mode2_run):
    """The same run driven by prefetch_frame / process_frame_device / finish_frame (the mid-frame read-back sits between the
    look-ahead's side stream and the main stream)."""
    K2, frames = loop_seq
    ctx = make_ctx(K2, close_loops=2, **LOOP_CFG)
    try:
        ctx.prefetch_frame(frames[0][0], frames[0][1])
        for i in range(len(frames)):
            ctx.process_frame_device(None, None, i)
            if i + 1 < len(frames):
                ctx.prefetch_frame(frames[i + 1][0], frames[i + 1][1])
            ctx.finish_frame()
            m = ctx.map_download()
            info, graph = ctx.local_deform_result()
            a = mode2_run[i]
            assert np.array_equal(a["pose"], ctx.get_pose()), i
            assert a["count"] == len(m) and a["map"] == digest(m), i
            assert np.array_equal(a["graph"], graph) and info == a["info"], i
    finally:
        ctx.close()


def test_mode2_changes_nothing_until_it_applies_a_graph(loop_seq, mode2_run):
    """Up to the first applied closure a mode-2 run is a mode-1 run (sampling and the read-back leave the frame alone); on that
    frame the pose and the map move."""
    K2, frames = loop_seq
    first = next(i for i, a in enumerate(mode2_run) if a["info"]["applied"])
    ctx = make_ctx(K2, close_loops=1, **LOOP_CFG)
    try:
        for i, (rgb, depth, _) in enumerate(frames[:first + 1]):
            ctx.process_frame(rgb, depth, i)
            m = ctx.map_download()
            a = mode2_run[i]
            if i < first:
                assert np.array_equal(a["pose"], ctx.get_pose()), i
                assert a["count"] == len(m) and a["map"] == digest(m), i
            else:
                assert not np.array_equal(a["pose"], ctx.get_pose())
                assert a["map"] != digest(m)
    finally:
        ctx.close()


def test_accepted_front_half_without_a_graph_applies_nothing(small_K, small_frames):
    """A 160x120 frame leaves at most 19 200 surfels, 4 sampled nodes: no graph. A given map of < 20 001 surfels, made of an ACTIVE
    half and a displaced INACTIVE half, gets an accepted front half; mode 2 then solves and applies nothing and equals mode 1."""
    K = small_K
    base = make_ctx(K, capacity=200000, time_delta=BIG)
    try:
        for i in range(4):
            base.process_frame(small_frames[i][0], small_frames[i][1], i)
        m, T = base.map_download()[:20000].copy(), base.get_pose()
    finally:
        base.close()
    assert len(m) > 5000
    m[:, 3] += 10.0
    inactive = (np.arange(len(m)) % 2) == 0
    m[:, 7] = np.where(inactive, 40.0, 295.0)
    m[:, 6] = np.where(inactive, 10.0, 250.0)
    m[inactive, 0:3] += np.array([0.004, -0.003, 0.002], np.float32)
    out = {}
    for mode in (1, 2):
        ctx = make_ctx(K, capacity=200000, time_delta=200, close_loops=mode, **ACCEPT_ALL)
        try:
            ctx.process_frame(small_frames[0][0], small_frames[0][1], 0)
            if mode == 2:
                info, graph = ctx.local_deform_result()
                assert info["n_nodes"] == 0 and len(graph) == 0
            ctx.map_upload(m)
            ctx.set_tick(300)
            ctx.process_frame(small_frames[4][0], small_frames[4][1], 4, T_wc=T)
            res = ctx.local_loop_result()[0]
            assert res["ran"] == 1 and res["accepted"] == 1 and res["n_constraints"] > 0
            mm = ctx.map_download()
            out[mode] = (ctx.get_pose(), mm)
            if mode == 2:
                info, _ = ctx.local_deform_result()
                assert not info["solved"] and not info["applied"] and info["deforms"] == 0 and info["last_deform_time"] == 0
                assert len(mm) <= 20000 and info["n_nodes"] == 0  # still 4 nodes or fewer at the end of this frame
        finally:
            ctx.close()
    assert np.array_equal(out[1][0], out[2][0])
    assert out[1][1].tobytes() == out[2][1].tobytes()


def test_resident_5m_map_samples_1023_nodes():
    """A resident 5.2 M-surfel map samples 1023 nodes (the cap), surfels 0, 5000, ..., 5 110 000 of the map after the frame."""
    from elasticfusion_b200 import synth

    K = synth.K_DEFAULT
    frames = list(synth.sequence(2, K, seed=42, noise=True))
    room = synth.room_surfels(5_200_000, np.linalg.inv(synth.trajectory(1, seed=42)[0]), view_depth=1.5, focal=K.fx)
    assert len(room) > 5_115_000
    ctx = make_ctx(K, capacity=5_600_000, time_delta=BIG, close_loops=2)
    try:
        ctx.process_frame(frames[0][0], frames[0][1], 0)
        ctx.map_upload(np.zeros((len(room), 12), np.float32))
        step = 1 << 21
        for c0 in range(0, len(room), step):
            ctx.map_upload_range(room[c0:c0 + step], c0)
        ctx.predict()
        ctx.process_frame(frames[1][0], frames[1][1], 1, T_wc=frames[1][2])
        info, graph = ctx.local_deform_result()
        m = ctx.map_download()
    finally:
        ctx.close()
    assert info["n_nodes"] == 1023 and len(graph) == 1023
    assert np.array_equal(graph, m[0:5_110_001:5000][:, [0, 1, 2, 6]])


def test_stage_split_is_refused_in_mode2(small_K, small_frames):
    """close_loops = 2 closes its loops inside ef_process_frame: the begin / end split of closed-loop hosts is EF_ESTATE."""
    from elasticfusion_b200 import capi

    ctx = make_ctx(small_K, capacity=200000, close_loops=2)
    try:
        with pytest.raises(capi.EfError, match=r"\(-3\)"):
            ctx.process_frame_begin(small_frames[0][0], small_frames[0][1], 0)
        with pytest.raises(capi.EfError, match=r"\(-3\)"):
            ctx.process_frame_end()
        ctx.process_frame(small_frames[0][0], small_frames[0][1], 0)  # the context is untouched
        assert ctx.get_tick() == 2
    finally:
        ctx.close()
    ctx = make_ctx(small_K, capacity=200000, close_loops=1)
    try:
        with pytest.raises(capi.EfError, match=r"\(-3\)"):
            ctx.local_deform_result()
    finally:
        ctx.close()


def test_headless_cli_closes_loops_like_the_c_abi(tmp_path, loop_seq, mode2_run):
    """tools/ElasticFusionHeadless -dlc (no -o) on a .klg of the loop sequence: the .freiburg's last pose is mode 2's, and
    getDeforms() reports the query's count. The log reader drops the last frame, so N-1 frames are processed."""
    from elasticfusion_b200 import synth

    K2, frames = loop_seq
    exe = os.path.join(ROOT, "tools", "ElasticFusionHeadless")
    if not os.path.exists(exe):
        subprocess.check_call(["bash", os.path.join(ROOT, "build.sh")])
    klg = str(tmp_path / "loop.klg")
    synth.write_klg(klg, [(f[0], f[1]) for f in frames])
    cal = str(tmp_path / "cal.txt")
    open(cal, "w").write(f"{K2.fx} {K2.fy} {K2.cx} {K2.cy}\n")
    out = subprocess.check_output([exe, "-l", klg, "-cal", cal, "-w", str(K2.width), "-h", str(K2.height), "-t", "12", "-ic", "3000",
                                   "-ie", "5e-05", "-cv", "1e-4", "-cap", "400000", "-dlc"], text=True, stderr=subprocess.STDOUT)
    assert "open-loop" not in out
    assert f"{N_FRAMES - 1} frames" in out
    last = mode2_run[N_FRAMES - 2]
    assert int(out.split("deforms")[1].split()[0]) == last["info"]["deforms"] > 0
    lines = open(klg + ".freiburg").read().strip().split("\n")
    assert len(lines) == N_FRAMES - 1
    t = np.array([float(x) for x in lines[-1].split()[1:4]])
    assert np.abs(t - last["pose"][:3, 3]).max() < 1e-6  # printed with 6 decimals
