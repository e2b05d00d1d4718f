"""GPU tests of the surfel map on the map states the published large-map numbers are measured on, and on a map sparser than the
quarter pixel grid fuse samples.

The other map tests grow their maps from a few frames (~300 k surfels at 640x480, ~2 M at 1920x1080). Here:

  * bench-5M / bench-20M: the resident maps of bench.py's 640x480-5M and 1280x960-20M workloads, built the same way (frame 0
    through the public call, the map replaced by synth.room_surfels, predict()). k_index_scatter makes many grid-stride rounds,
    the visible list holds millions of entries, and the clean pass walks tens of thousands of tiles with its look-back and the
    in-place compaction that writes into the input ranges of earlier tiles. Each config asserts the property it exists for.
  * sparse: 640x480 with ~300 k room surfels, where many matched pixels pick the same surfel and only the lowest draw index
    may update it (SURVEY App. A-17). The config asserts that at least a quarter of the matched pixels lose that conflict.

The stage tests give the surfels a seeded spread of lastTime and confidence (spread_map), so that the time-window tests, the
INACTIVE raycast and the stale-surfel cull of clean see both sides of their conditions. The pipeline tests use the plain bench
recipe. A 20 M map is 960 MB per host copy: copies are freed once compared and large arrays are compared in chunks.
"""
import os

import numpy as np
import pytest

from util import assert_same, rel_err

pytestmark = pytest.mark.gpu

MAXD = 20.0
BIG = 2147483647 // 2
SEED = 42  # bench.py's sequence seed
N_FRAMES = 5  # frame 0 + the 4 frames run after the map is populated
CHUNK = 1 << 21
# name: (frame scale of the 640x480 camera, resident surfels, capacity)
CONFIGS = {
    "sparse": (1, 300_000, 600_000),
    "bench-5M": (1, 5_000_000, 5_600_000),
    "bench-20M": (2, 20_000_000, 21_500_000),
}
# stage tests: the measurement is frame STAGE_FRAME at its ground-truth pose, at tick STAGE_TICK with lastTime in [1, STAGE_TICK]
STAGE_FRAME, STAGE_TICK, STAGE_TD, WEIGHT = 1, 60, 30, 0.73
COLS = [0, 1, 2, 4, 5, 6, 7, 8, 9, 10, 11]  # all but the confidence (expf)


# ------------------------------------------------------------------------------------------------------------------ helpers
def diff_rows(a, b):
    """Indices of the rows of a and b (same shape) that are not identical (NaN == NaN), compared chunk by chunk."""
    assert a.shape == b.shape, (a.shape, b.shape)
    out = []
    for c0 in range(0, len(a), CHUNK):
        x, y = a[c0:c0 + CHUNK], b[c0:c0 + CHUNK]
        same = ((x == y) | (np.isnan(x) & np.isnan(y))).all(axis=1)
        out.append(np.flatnonzero(~same) + c0)
    return np.concatenate(out) if out else np.zeros(0, np.int64)


def assert_rows_same(a, b, what):
    bad = diff_rows(a, b)
    assert len(bad) == 0, f"{what}: {len(bad)} of {len(a)} surfels differ, first {bad[:5]}"


def assert_surfels_same(got, ref, what):
    """Bit-exact but for the confidence (expf), which may differ by ulps."""
    assert got.shape == ref.shape, (what, got.shape, ref.shape)
    for c0 in range(0, len(ref), CHUNK):
        assert_same(got[c0:c0 + CHUNK, COLS], ref[c0:c0 + CHUNK, COLS], what)
        assert rel_err(got[c0:c0 + CHUNK, 3], ref[c0:c0 + CHUNK, 3]) < 1e-6, what


def assert_kept(got, M, culled, what):
    """got == M without the rows `culled` (sorted), in order, compared chunk by chunk without materialising M[keep]."""
    keep = np.ones(len(M), bool)
    keep[culled] = False
    assert len(got) == int(keep.sum()), (what, len(got), int(keep.sum()))
    pos = 0
    for c0 in range(0, len(M), CHUNK):
        sel = M[c0:c0 + CHUNK][keep[c0:c0 + CHUNK]]
        assert_rows_same(got[pos:pos + len(sel)], sel, f"{what} (rows {pos}..)")
        pos += len(sel)


def active_pixels(dm, tick):
    """Pixels of the quarter grid fuse measures at `tick` (data.vert: this tick's parity in x and y, all four neighbours with a
    depth, 0 < z <= maxDepth): each one either matches a surfel or becomes a new one."""
    rows, cols = dm.shape
    jj, ii = np.mgrid[0:rows, 0:cols]
    p = np.pad(dm, 1, mode="edge")
    ok = (ii % 2 == tick % 2) & (jj % 2 == tick % 2) & (dm > 0) & (dm <= MAXD)
    ok &= (p[1:-1, :-2] != 0) & (p[1:-1, 2:] != 0) & (p[:-2, 1:-1] != 0) & (p[2:, 1:-1] != 0)
    return int(ok.sum())


def spread_map(room, seed=5):
    """The room map with lastTime spread over [1, STAGE_TICK] and a quarter of the surfels unstable (confidence 5 < 10): the
    finite time window drops about half of the map, and clean culls the unstable ones older than 20 frames."""
    rng = np.random.RandomState(seed)
    m = room.copy()
    n = len(m)
    m[:, 7] = rng.randint(1, STAGE_TICK + 1, n).astype(np.float32)
    m[:, 3] = np.where(rng.uniform(size=n) < 0.25, 5.0, 20.0).astype(np.float32)
    return m


def make_ctx(R, **kw):
    from elasticfusion_b200 import capi

    K = R["K"]
    return capi.Context(capi.default_config(K.width, K.height, K.fx, K.fy, K.cx, K.cy, capacity=R["capacity"], time_delta=BIG, **kw))


def populate(ctx, R):
    """bench.populate_map: frame 0 through the public call, the map replaced by the room surfels, the model view re-rendered."""
    rgb0, depth0, _ = R["frames"][0]
    ctx.process_frame(rgb0, depth0, 0)
    ctx.map_upload(R["room"])
    ctx.predict()
    ctx.sync()


def stage_inputs(ctx, R):
    """Frame STAGE_FRAME's preprocessed inputs, uploaded; returns them with the frame's pose."""
    from oracle import ef_oracle as eo

    rgb, depth, T = R["frames"][STAGE_FRAME]
    filt = eo.bilateral(depth, 3.0)
    g = dict(rgb=rgb, depth=depth, filt=filt, dm=eo.metric(depth, 3.0), dmf=eo.metric(filt, 3.0), T=T)
    for name, key in (("RGB", "rgb"), ("DEPTH_RAW", "depth"), ("DEPTH_FILTERED", "filt"), ("DEPTH_METRIC", "dm"),
                      ("DEPTH_METRIC_FILTERED", "dmf")):
        ctx.upload(name, g[key])
    return g


# ------------------------------------------------------------------------------------------------------------------ fixtures
@pytest.fixture(scope="module", params=list(CONFIGS))
def R(request):
    """One resident-map configuration: camera, frames 0..4 of bench.py's sequence, the room map. Built once per module and config
    (pytest runs every test of a config before it builds the next)."""
    import torch
    from elasticfusion_b200 import synth

    scale, n, cap = CONFIGS[request.param]
    K = synth.K_DEFAULT if scale == 1 else synth.K_DEFAULT.scaled(scale)
    room = synth.room_surfels(n, np.linalg.inv(synth.trajectory(1, seed=SEED)[0]), view_depth=1.5, focal=K.fx)
    st = dict(name=request.param, K=K, capacity=cap, room=room, frames=list(synth.sequence(N_FRAMES, K, seed=SEED, noise=True)),
              num_sms=torch.cuda.get_device_properties(0).multi_processor_count)
    assert len(room) <= cap and abs(len(room) - n) < 0.01 * n
    yield st
    st.clear()


@pytest.fixture
def spread(R):
    if "spread" not in R:
        R["spread"] = spread_map(R["room"])
    return R["spread"]


# ------------------------------------------------------------------------------------------------------------------ the regime
def test_config_reaches_its_regime(R, spread):
    """Each config keeps the property it exists for. Bench maps: the index map at least 90 % covered, more surfels than 20 x the
    lanes of k_index_scatter's grid (num_sms * 5 CTAs of 256), more clean tiles (512 surfels) than 10 x the CTAs k_clean_move
    runs (num_sms * 4). Sparse: at least a quarter of the matched pixels of the fuse stage test lose their surfel to a lower draw index (oracle)."""
    from oracle import ef_oracle as eo

    K = R["K"]
    if R["name"] == "sparse":
        rgb, depth, T = R["frames"][STAGE_FRAME]
        filt = eo.bilateral(depth, 3.0)
        dm, dmf = eo.metric(depth, 3.0), eo.metric(filt, 3.0)
        idx = eo.predict_indices(spread, T, STAGE_TICK, MAXD, BIG, K)
        fused, new = eo.fuse(spread, T, STAGE_TICK, rgb, dm, dmf, *idx, MAXD, WEIGHT, K)
        matched = active_pixels(dm, STAGE_TICK) - len(new)
        lost = matched - len(diff_rows(fused, spread))
        assert matched > 10000 and lost >= 0.25 * matched, (matched, lost)
        return
    n = len(R["room"])
    assert n > 20 * R["num_sms"] * 5 * 256
    assert (n + 511) // 512 > 10 * R["num_sms"] * 4
    ctx = make_ctx(R)
    try:
        populate(ctx, R)
        ctx.map_predict_indices(ctx.get_pose(), ctx.get_tick(), MAXD, BIG)
        assert (ctx.download("INDEX") > 0).mean() >= 0.9
    finally:
        ctx.close()


# ------------------------------------------------------------------------------------------------------------------ stages
@pytest.mark.parametrize("td", [BIG, STAGE_TD])
def test_predict_indices(R, spread, td):
    """index_map.vert/.frag over the whole resident map, all four attachments bit-exact; with the finite window about half of
    the map is out of it."""
    from oracle import ef_oracle as eo

    ctx = make_ctx(R)
    try:
        T = R["frames"][STAGE_FRAME][2]
        ctx.map_upload(spread)
        ctx.map_predict_indices(T, STAGE_TICK, MAXD, td)
        ref = eo.predict_indices(spread, T, STAGE_TICK, MAXD, td, R["K"])
        for name, r in zip(("INDEX", "VERT_CONF", "COLOR_TIME", "NORM_RAD"), ref):
            assert_same(ctx.download(name), r, name)
        # (points, not discs: the sparse map covers ~9 % of the pixels, a bench map ~94 %; the window keeps ~60 % of a view)
        assert (ref[0] > 0).mean() > (0.04 if R["name"] == "sparse" else 0.5) * (1.0 if td == BIG else 0.5)
    finally:
        ctx.close()


def test_fuse_then_clean(R, spread):
    """fuse on the resident map: the fused map, the new surfels and the exact set of surfels each side changed, identical up to
    the <= 2 surfels an acosf / expf rounding difference may associate differently. Then clean on the oracle's fused state with
    the new surfels appended: the stale unstable surfels are culled and everything behind them moves."""
    from oracle import ef_oracle as eo

    K = R["K"]
    ctx = make_ctx(R)
    try:
        g = stage_inputs(ctx, R)
        T, tick = g["T"], STAGE_TICK
        idx = eo.predict_indices(spread, T, tick, MAXD, BIG, K)
        fused, new = eo.fuse(spread, T, tick, g["rgb"], g["dm"], g["dmf"], *idx, MAXD, WEIGHT, K)
        del idx
        ctx.map_upload(spread)
        ctx.map_predict_indices(T, tick, MAXD, BIG)
        ctx.map_fuse(T, tick, MAXD, WEIGHT)
        got, got_new = ctx.map_download(), ctx.map_download_new()
        ref_ids, got_ids = diff_rows(fused, spread), diff_rows(got, spread)
        flips = np.setxor1d(ref_ids, got_ids)
        assert len(flips) <= 2, f"{len(flips)} surfels changed on one side only: {flips[:8]}"
        assert len(ref_ids) > 5000 and len(new) > 100
        differ = diff_rows(got, fused)
        if len(differ):  # (acosf / expf: the rows that differ must at least be close, and few)
            close = np.isclose(got[differ], fused[differ], rtol=2e-6, atol=1e-7, equal_nan=True).all(axis=1)
            assert (~close).sum() <= 2 and len(differ) <= 0.1 * len(ref_ids), (len(differ), (~close).sum())
        del got
        assert abs(len(got_new) - len(new)) <= 2
        if len(got_new) != len(new):
            return  # a flip between matched and new: the clean comparison below needs the same new surfels on both sides
        assert_surfels_same(got_new, new, "new unstable surfels")

        ctx.map_upload(fused)
        idx2 = eo.predict_indices(fused, T, tick, MAXD, BIG, K)
        ctx.map_predict_indices(T, tick, MAXD, BIG)
        assert_same(ctx.download("INDEX"), idx2[0], "index map of the fused state")
        ref = eo.clean(fused, new, T, tick, *idx2, 10.0, BIG, MAXD, K)
        n_stale = int(((tick - fused[:, 7] > 20) & (fused[:, 3] < 10.0)).sum())
        del idx2
        ctx.map_clean(T, tick, 10.0, BIG, MAXD)
        assert ctx.map_count() == len(ref)
        assert len(fused) + len(new) - len(ref) >= n_stale > 0.05 * len(fused)
        del fused
        assert_surfels_same(ctx.map_download(), ref, "map after clean")
    finally:
        ctx.close()


def test_raycast_and_fill_in(R, spread):
    """combinedPredict over the resident map: ACTIVE (mode 0, all four attachments), INACTIVE (mode 1, the surfels last seen
    before tick - td) and depth only (mode 2), bit-exact; then the fill-in passes and the density test on the ACTIVE view."""
    from oracle import ef_oracle as eo

    K = R["K"]
    ctx = make_ctx(R)
    try:
        g = stage_inputs(ctx, R)
        T, tick, td = g["T"], STAGE_TICK, STAGE_TD
        ctx.map_upload(spread)
        ref = eo.combined_predict(spread, T, MAXD, 10.0, tick, tick, BIG, K)
        ctx.map_raycast(T, MAXD, 10.0, tick, tick, BIG, 0)
        for name, r in zip(("IMAGE", "VERTEX", "NORMAL", "TIME"), ref):
            assert_same(ctx.download(name), r, name)
        assert (ref[1][..., 2] > 0).mean() > 0.5
        old = eo.combined_predict(spread, T, MAXD, 10.0, 0, tick - td, td, K)
        ctx.map_raycast(T, MAXD, 10.0, 0, tick - td, td, 1)
        for name, r in zip(("OLD_IMAGE", "OLD_VERTEX", "OLD_NORMAL", "OLD_TIME"), old):
            assert_same(ctx.download(name), r, name)
        covered = (old[1][..., 2] > 0).mean()
        assert covered > 0.05 and not np.array_equal(old[3], ref[3]), covered  # the INACTIVE view holds another part of the map
        d_ref = eo.combined_predict(spread, T, MAXD, 10.0, tick, tick, BIG, K, depth_only=True)
        ctx.map_raycast(T, MAXD, 10.0, tick, tick, BIG, 2)
        assert_same(ctx.download("SYNTH_DEPTH"), d_ref, "synthesizeDepth")
        ctx.map_raycast(T, MAXD, 10.0, tick, tick, BIG, 0)  # the fill-in reads the ACTIVE view
        ctx.map_fill_in(False, False)
        assert_same(ctx.download("FILL_VERTEX"), eo.fill_vertex(ref[1], g["filt"], 0, K), "fill vertex")
        assert_same(ctx.download("FILL_NORMAL"), eo.fill_normal(ref[2], g["filt"], 0, K), "fill normal")
        assert_same(ctx.download("FILL_IMAGE"), eo.fill_image(ref[0], g["rgb"], 0), "fill image")
        assert ctx.dense_enough() == eo.dense_enough(ref[0])
    finally:
        ctx.close()


# ------------------------------------------------------------------------------------------------------------------ compaction
def cull_patterns(n):
    rng = np.random.RandomState(11)
    mid = (n // 512 // 2) * 512
    tail = n - n // 100
    return {
        "surfel-1": np.array([1]),  # every later surfel moves down by one
        "last": np.array([n - 1]),
        "511-513": np.array([511, 512, 513]),  # both sides of the first tile boundary
        "one-tile": np.arange(mid, mid + 512),  # a whole tile keeps nothing
        "random-10pct": np.sort(rng.choice(n, n // 10, replace=False)),
        "last-1pct": tail + np.sort(rng.choice(n - tail, (n - tail) // 10, replace=False)),  # a long untouched prefix
        "none": np.zeros(0, np.int64),  # the count must stand
    }


def test_clean_compaction_identities(R):
    """The order-preserving in-place compaction, without the oracle: on a settled map M (one predict_indices + one clean, which
    keeps everything), surfels marked culled (lastTime = -1, copy_unstable.vert's w == -1 rule, written with map_upload_range)
    are removed and the result is exactly M without them, with the same textures. Each pattern runs twice on one context (the
    tile dispenser, exit tickets and look-back epoch re-arm between launches); one pattern is cross-checked against the oracle."""
    from oracle import ef_oracle as eo

    ctx = make_ctx(R)
    try:
        populate(ctx, R)
        T, tick = ctx.get_pose(), ctx.get_tick()
        ctx.map_predict_indices(T, tick, MAXD, BIG)
        ctx.map_clean(T, tick, 10.0, BIG, MAXD)
        M = ctx.map_download()
        assert len(M) == len(R["room"])
        assert_rows_same(M, R["room"], "settled map")
        n = len(M)
        for name, culled in cull_patterns(n).items():
            for rep in range(2):
                ctx.map_upload(M)
                if len(culled):
                    lo, hi = int(culled[0]), int(culled[-1]) + 1
                    block = M[lo:hi].copy()
                    block[culled - lo, 7] = -1.0
                    ctx.map_upload_range(block, lo)
                    del block
                ctx.map_clean(T, tick, 10.0, BIG, MAXD)
                assert ctx.map_count() == n - len(culled), (name, rep, ctx.map_count(), n - len(culled))
                got = ctx.map_download()
                assert_kept(got, M, culled, f"{name} #{rep}")
                if name == "random-10pct" and rep == 1:
                    idx = tuple(ctx.download(k) for k in ("INDEX", "VERT_CONF", "COLOR_TIME", "NORM_RAD"))
                    Mc = M.copy()
                    Mc[culled, 7] = -1.0
                    ref = eo.clean(Mc, np.zeros((0, 12), np.float32), T, tick, *idx, 10.0, BIG, MAXD, R["K"])
                    del Mc
                    assert_rows_same(got, ref, "compaction against the oracle")
                    del ref
                del got
    finally:
        ctx.close()


def test_upload_download(R):
    """The map built with chunked map_upload_range downloads identical to one map_upload; a range past the count and an upload
    above the capacity are rejected with EF_EINVAL."""
    import ctypes as C

    from elasticfusion_b200 import capi

    EF_EINVAL = -1  # include/efusion_b200.h
    room = R["room"]
    n = len(room)
    ctx = make_ctx(R)
    try:
        ctx.map_upload(room)
        assert ctx.map_count() == n
        assert_rows_same(ctx.map_download(), room, "map_upload")
        ctx.map_upload(np.zeros((n, 12), np.float32))
        step = max(1, n // 7 + 12345)  # uneven chunks, the last one short
        for c0 in range(0, n, step):
            ctx.map_upload_range(room[c0:c0 + step], c0)
        assert ctx.map_count() == n
        assert_rows_same(ctx.map_download(), room, "chunked map_upload_range")
        one = np.ascontiguousarray(room[:2])
        h = ctx.h_ctx
        assert capi.lib().ef_map_upload_range(h, one.ctypes.data_as(C.c_void_p), n - 1, 2) == EF_EINVAL
        assert capi.lib().ef_map_upload_range(h, one.ctypes.data_as(C.c_void_p), n, 1) == EF_EINVAL
        over = np.empty((R["capacity"] + 1, 12), np.float32)  # (never touched: the size is rejected before any copy)
        assert capi.lib().ef_map_upload(h, over.ctypes.data_as(C.c_void_p), len(over)) == EF_EINVAL
        del over
        assert ctx.map_count() == n  # the rejected calls left the map alone
        assert_rows_same(ctx.map_download()[-3:], room[-3:], "map after the rejected calls")
    finally:
        ctx.close()


# ------------------------------------------------------------------------------------------------------------------ pipeline
def run_device(R, mode="plain", env=None):
    """bench recipe + frames 1..4 (skip_mid_predict = 0). Returns (poses, counts, final map). mode 'lookahead': the frames are
    staged from device memory with prefetch_frame_device while the previous one is in flight."""
    import torch

    old = {k: os.environ.get(k) for k in (env or {})}
    os.environ.update(env or {})
    try:
        ctx = make_ctx(R, skip_mid_predict=0)  # (the switches are read when the context is created)
    finally:
        for k, v in old.items():
            if v is None:
                os.environ.pop(k)
            else:
                os.environ[k] = v
    frames = R["frames"]
    poses, counts = [], []
    try:
        populate(ctx, R)
        if mode == "plain":
            for i in range(1, N_FRAMES):
                ctx.process_frame(frames[i][0], frames[i][1], i)
                poses.append(ctx.get_pose())
                counts.append(ctx.map_count())
        else:
            dev = [(torch.from_numpy(np.ascontiguousarray(r)).cuda(), torch.from_numpy(np.ascontiguousarray(d).view(np.int16)).cuda())
                   for r, d, _ in frames]
            torch.cuda.synchronize()
            ctx.prefetch_frame_device(dev[1][0].data_ptr(), dev[1][1].data_ptr())
            for i in range(1, N_FRAMES):
                ctx.process_frame_device(None, None, i)
                if i + 1 < N_FRAMES:
                    ctx.prefetch_frame_device(dev[i + 1][0].data_ptr(), dev[i + 1][1].data_ptr())
            ctx.finish_frame()
            poses.append(ctx.get_pose())
            counts.append(ctx.map_count())
        return np.array(poses), counts, ctx.map_download()
    finally:
        ctx.close()


N_PERTURB = 8  # depth pixels of frame 1 perturbed, one at a time, to measure the oracle's own sensitivity


def oracle_poses(R, frames):
    """The oracle over the bench recipe (frame 0, Fusion.set_map, frames 1..4): poses after each of frames 1..4, counts."""
    from oracle import ef_oracle as eo

    f = eo.Fusion(R["K"], capacity=R["capacity"])
    f.process_frame(frames[0][0], frames[0][1], 0)
    f.set_map(R["room"])
    assert f.count == len(R["room"]) and f.tick == 2
    poses, counts = [], []
    for i in range(1, N_FRAMES):
        f.process_frame(frames[i][0], frames[i][1], i)
        poses.append(f.pose)
        counts.append(f.count)
    del f
    return np.array(poses), counts


def pipeline_sensitivity(R, base):
    """How far the oracle's poses move from themselves when one depth pixel of frame 1 is 1 mm deeper: the largest |dT| element
    over the N_PERTURB pixels nearest the image centre with a depth in 0.3 - 3 m (test_gpu_sensor_sizes.pipeline_sensitivity)."""
    frames = R["frames"]
    d1 = frames[1][1]
    ys, xs = np.nonzero((d1 > 300) & (d1 < 3000))
    order = np.argsort((ys - d1.shape[0] / 2.0) ** 2 + (xs - d1.shape[1] / 2.0) ** 2, kind="stable")[:N_PERTURB]
    worst = 0.0
    for y, x in zip(ys[order], xs[order]):
        d = d1.copy()
        d[y, x] += 1
        p, _ = oracle_poses(R, frames[:1] + [(frames[1][0], d, frames[1][2])] + frames[2:])
        worst = max(worst, float(np.abs(p - base).max()))
    return worst


def test_pipeline_matches_oracle(R):
    """processFrame over 4 frames after the map is populated, against the oracle started from the same map (Fusion.set_map):
    surfel counts within 0.1 % and poses within 2e-5, the bars of test_gpu_mapping. Where the poses differ by more, the oracle
    itself is not stable at that scale on these maps (tracking against a resident map of flat walls: ICP slides along them and
    the photometric term holds the pose): they are then held to twice the oracle's own 1 mm sensitivity (pipeline_sensitivity),
    never looser than 5e-4, as test_gpu_sensor_sizes holds its small frames."""
    frames = R["frames"]
    ref, ref_counts = oracle_poses(R, frames)
    ctx = make_ctx(R, skip_mid_predict=0)
    got, counts = [], []
    try:
        populate(ctx, R)
        assert ctx.get_tick() == 2
        for i in range(1, N_FRAMES):
            ctx.process_frame(frames[i][0], frames[i][1], i)
            got.append(ctx.get_pose())
            counts.append(ctx.map_count())
        assert ctx.get_tick() == N_FRAMES + 1
    finally:
        ctx.close()
    for i, (c, co) in enumerate(zip(counts, ref_counts)):
        assert abs(c - co) <= max(2, 1e-3 * co), (i + 1, c, co)
    err = float(np.abs(np.array(got)[:, :3, :] - ref[:, :3, :]).max())
    if err >= 2e-5:
        sens = pipeline_sensitivity(R, ref)
        assert err < min(5e-4, max(2e-5, 2.0 * sens)), (err, sens)


def test_pipeline_switches_bit_identical(R):
    """The visible-list second index pass (EF_VISIBLE_LIST=0 renders the whole map twice) and the frame look-ahead change nothing:
    poses, counts and the final map are bit-identical to plain calls with the defaults."""
    p0, c0, m0 = run_device(R)
    p1, c1, m1 = run_device(R, env={"EF_VISIBLE_LIST": "0"})
    assert np.array_equal(p0, p1) and c0 == c1
    assert_rows_same(m1, m0, "EF_VISIBLE_LIST=0")
    del m1
    p2, c2, m2 = run_device(R, mode="lookahead")
    assert np.array_equal(p0[-1], p2[-1]) and c0[-1] == c2[-1]
    assert_rows_same(m2, m0, "look-ahead")
