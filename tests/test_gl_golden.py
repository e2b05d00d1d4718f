"""The mapping half against the REFERENCE'S OWN GLSL SHADERS: tests/golden/ref_mapping_160x120.npz holds the outputs of
the reference's Core/Shaders/*.{vert,geom,frag} (unmodified) executed on Mesa llvmpipe by oracle/gl/ref_gl_harness.cpp
(generator: tests/golden/make_gl_golden.py). Every pass of the GL half is compared on the inputs it was given:

  * CPU (`not gpu`): oracle/efo_map.cpp, the restatement that all other mapping tests use as their checker -- this is what pins it;
  * `-m gpu`: libefusion.so through the C ABI.

The inputs of every pass are the CPU oracle's stage outputs along one frame's chain (oracle_inputs below); they are recomputed
here rather than stored, so the fixture holds only the shaders' outputs. Of the large ones it keeps every STEP-th surfel of a
list and every STEP-th pixel of an image (row-major), and the full length of each list; the implementations' outputs are cut
the same way before they are compared.

Tolerances: integer / index / byte outputs must be identical except for a stated fraction of pixels where a value sits on a
rounding boundary (sub-pixel snapping of a window coordinate at x.5/256, exp() in the bilateral weight, pow(r, 2) at a disc edge:
Mesa evaluates transcendental functions with its own polynomials); float outputs 1e-5 absolute (depths are metres)."""
import os

import numpy as np
import pytest

from util import assert_same, run_oracle

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
MAXD, BIG = 20.0, 2 ** 30
COLS = [0, 1, 2, 4, 5, 6, 7, 8, 9, 10, 11]  # everything but the confidence (exp())
# fixture per camera configuration (tests/golden/make_gl_golden.py:CONFIGS) -> STEP of its sample
FIXTURES = {"default": 8, "icl": 24, "offcentre": 32, "icl320": 128}
SAMPLED = ("gl_initial_map", "gl_fused", "gl_cleaned", "gl_cleaned_t", "gl_cleaned_deformed", "gl_vert_conf", "gl_color_time", "gl_norm_rad",
           "gl_image", "gl_vertex", "gl_normal", "gl_time", "gl_synth_depth", "gl_old_image", "gl_old_vertex", "gl_old_normal", "gl_old_time",
           "gl_fill_vertex", "gl_fill_normal", "gl_fill_image", "gl_fill_vertex_pass", "gl_fill_image_pass")


def graph_for(m, n_nodes=40, seed=4):
    rng = np.random.RandomState(seed)
    idx = np.sort(rng.choice(len(m), n_nodes, replace=False))
    nodes = np.zeros((n_nodes, 16), np.float32)
    for k, i in enumerate(idx):
        w = rng.standard_normal(3) * 0.01
        th = np.linalg.norm(w)
        kx = np.array([[0, -w[2], w[1]], [w[2], 0, -w[0]], [-w[1], w[0], 0]]) / max(th, 1e-12)
        R = np.eye(3) + np.sin(th) * kx + (1 - np.cos(th)) * (kx @ kx)
        nodes[k, 0:3] = m[i, 0:3]
        nodes[k, 3:12] = R.T.reshape(-1)
        nodes[k, 12:15] = rng.standard_normal(3) * 0.01
        nodes[k, 15] = m[i, 6]
    return np.ascontiguousarray(nodes[np.argsort(nodes[:, 15], kind="stable")])


def oracle_inputs(K, seed, speed):
    """The inputs of every pass: frames of the synthetic sequence and the CPU oracle's stage outputs along one frame's chain
    (both sides of every comparison start from these)."""
    from elasticfusion_b200 import synth
    from oracle import ef_oracle as eo

    frames = list(synth.sequence(8, K, seed=seed, noise=True, speed=speed))
    rgb0, depth0, _ = frames[0]
    g = dict(rgb0=rgb0, depth0=depth0, filt0=eo.bilateral(depth0, 3.0))
    # a scene crossing depthCutoff: the two feedback buffers differ in length (SURVEY App. A-29)
    Tb = synth.pose(synth.rot_xyz(0, np.deg2rad(55.0), 0), [-1.6, 0.2, -1.2])
    rgbb, depthb, _, _ = synth.render(Tb, K, noise_seed=77)
    g.update(rgbb=rgbb, depthb=depthb, filtb=eo.bilateral(depthb, 3.0))
    # a map after 4 frames, frame 4 as the measurement
    f = run_oracle(frames, K, 4)
    m, T, tick = f.map(), f.pose, f.tick
    rgb4, depth4, _ = frames[4]
    filt4 = eo.bilateral(depth4, 3.0)
    g.update(map=m, T=T, tick=np.array(tick), rgb4=rgb4, depth4=depth4, filt4=filt4)
    io = eo.predict_indices(m, T, tick, MAXD, BIG, K)
    g.update(index_in=io[0], vert_conf_in=io[1], color_time_in=io[2], norm_rad_in=io[3])
    fused, new = eo.fuse(m, T, tick, rgb4, eo.metric(depth4, 3.0), eo.metric(filt4, 3.0), *io, MAXD, 0.73, K)
    io2 = eo.predict_indices(fused, T, tick, MAXD, BIG, K)
    g.update(fused_in=fused, new_in=new, index2_in=io2[0], vert_conf2_in=io2[1], color_time2_in=io2[2], norm_rad2_in=io2[3])
    # finite time window + un-cull branch: a map with old time stamps
    mt = fused.copy()
    n = len(mt)
    mt[:, 6] = 1 + np.floor(np.arange(n) * 50.0 / n)
    mt[:, 7] = np.maximum(np.where(np.arange(n) % 2 == 0, 20.0, 58.0), mt[:, 6])
    mt[:, 3] += np.where(np.arange(n) % 3 == 0, 10.0, 0.0).astype(np.float32)
    tick_t, td = 60, 8
    it = eo.predict_indices(mt, T, tick_t, MAXD, td, K)
    g.update(map_t=mt, tick_t=np.array(tick_t), td=np.array(td), index_t_in=it[0], vert_conf_t_in=it[1], color_time_t_in=it[2], norm_rad_t_in=it[3])
    # deformation graph inside clean (copy_unstable.vert:132-322)
    g.update(nodes=graph_for(mt), synth_depth_t_in=eo.combined_predict(mt, T, MAXD, 10.0, tick_t, tick_t - td, 65535, K, depth_only=True))
    # model raycast (ACTIVE, INACTIVE, depth) and fill-in
    ms = fused.copy()
    ms[:, 3] += 10.0
    po = eo.combined_predict(ms, T, MAXD, 10.0, tick, tick, BIG, K)
    g.update(map_stable=ms, image_in=po[0], vertex_in=po[1], normal_in=po[2])
    return g


def fixture_path(config):
    return os.path.join(ROOT, "tests", "golden", "ref_mapping_160x120.npz" if config == "default" else f"ref_mapping_{config}.npz")


def cut(G, name, a):
    """`a` reduced to what G holds of output `name`: every step-th surfel of a list or pixel of an image (row-major), or all of it."""
    a = np.asarray(a)
    if name + "_n" not in G:
        return a
    step = int(G["step"])
    if a.ndim == 2 and a.shape[1] == 12:
        return a[::step]
    return a.reshape(-1, *a.shape[2:])[::step]


def full_len(G, name):
    return int(G[name + "_n"]) if name + "_n" in G else len(G[name])


def fuse_feedback(G):
    """What the data pass fed back: the new surfels (w = -2) and the number of matched measurements (w = -1)."""
    if "gl_fuse_feedback" not in G:
        return G["gl_fuse_new"], int(G["gl_fuse_matched"])
    fb = G["gl_fuse_feedback"]
    return fb[fb[:, 7] == -2], int((fb[:, 7] == -1).sum())


def shrink(out, step):
    """The fixture's form of the shaders' outputs: the SAMPLED ones cut to every step-th surfel / pixel, with their full lengths,
    and of the data pass's feedback only the new surfels and the count of matched measurements."""
    res = dict(out, step=np.array(step))
    new, n_matched = fuse_feedback(res)
    del res["gl_fuse_feedback"]
    res.update(gl_fuse_new=new, gl_fuse_matched=np.array(n_matched))
    for name in SAMPLED:
        res[name + "_n"] = np.array(len(out[name]))
        res[name] = cut(res, name, out[name])
    return res


def load(config):
    from elasticfusion_b200 import synth

    z = dict(np.load(fixture_path(config)))
    assert int(z["gl_error"]) == 0 and "llvmpipe" in str(z["gl_log"])
    w, h, fx, fy, cx, cy = z["K"]
    K = synth.Intrinsics(int(w), int(h), float(fx), float(fy), float(cx), float(cy))
    z.update(oracle_inputs(K, int(z["seed"]), float(z["speed"])))
    return z, K


@pytest.fixture(scope="module")
def G():
    return load("default")[0]


@pytest.fixture(scope="module")
def K(G):
    from elasticfusion_b200 import synth

    w, h, fx, fy, cx, cy = G["K"]
    return synth.Intrinsics(int(w), int(h), float(fx), float(fy), float(cx), float(cy))


def frac_differ(a, b, tol=0.0):
    a, b = np.asarray(a), np.asarray(b)
    assert a.shape == b.shape, (a.shape, b.shape)
    if a.dtype.kind == "f":
        both_nan = np.isnan(a) & np.isnan(b)
        d = np.where(both_nan, 0.0, np.abs(a.astype(np.float64) - b.astype(np.float64)))
        bad = ~(d <= tol)
    else:
        bad = a != b
    if bad.ndim > 2:
        bad = bad.reshape(bad.shape[0], bad.shape[1], -1).any(axis=2)
    elif bad.ndim == 2 and a.shape[1] in (4, 12):  # surfel rows, or the RGBA / xyzw pixels of a cut image
        bad = bad.any(axis=1)
    return float(bad.mean())


def mad(a, b):
    """max |a - b| with NaN == NaN (the reference's maps carry NaN normals at depth edges); a one-sided NaN counts as inf."""
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    d = np.abs(a - b)
    d[np.isnan(a) & np.isnan(b)] = 0.0
    d[np.isnan(d)] = np.inf
    return float(d.max()) if d.size else 0.0


def check_surfels(G, name, got, what, tol=1e-5, frac=0.0):
    assert len(got) == full_len(G, name), (what, len(got), full_len(G, name))
    got, ref = cut(G, name, got), G[name]
    assert frac_differ(got[:, COLS], ref[:, COLS], tol) <= frac, (what, frac_differ(got[:, COLS], ref[:, COLS], tol))
    ok = ~np.isnan(ref[:, 3])
    assert np.abs(got[ok, 3] - ref[ok, 3]).max() <= 1e-5 * max(1.0, np.abs(ref[ok, 3]).max()), what


class Oracle:
    """oracle/efo_map.cpp behind the same call names the product side offers below."""

    def __init__(self, K):
        from oracle import ef_oracle as eo

        self.eo, self.K = eo, K

    def bilateral(self, depth):
        return self.eo.bilateral(depth, 3.0)

    def metric(self, depth):
        return self.eo.metric(depth, 3.0)

    def first_frame(self, rgb, depth, filt):
        eo = self.eo
        raw = eo.feedback_buffer(rgb, eo.metric(depth, 3.0), self.K, 1, MAXD)
        fil = eo.feedback_buffer(rgb, eo.metric(filt, 3.0), self.K, 1, MAXD)
        return eo.map_initialise(raw, fil), len(raw), len(fil)

    def predict_indices(self, m, T, tick, td):
        return self.eo.predict_indices(m, T, tick, MAXD, td, self.K)

    def fuse(self, m, T, tick, rgb, depth, filt, idx, w):
        eo = self.eo
        return eo.fuse(m, T, tick, rgb, eo.metric(depth, 3.0), eo.metric(filt, 3.0), *idx, MAXD, w, self.K)

    def clean(self, m, new, T, tick, idx, td, nodes=None, depth=None):
        if nodes is None:
            return self.eo.clean(m, new, T, tick, *idx, 10.0, td, MAXD, self.K)
        return self.eo.clean_deform(m, new, T, tick, idx[0], idx[1], idx[2], 10.0, td, MAXD, self.K, nodes, depth)

    def raycast(self, m, T, time, max_time, td, depth_only=False):
        return self.eo.combined_predict(m, T, MAXD, 10.0, time, max_time, td, self.K, depth_only=depth_only)

    def fill(self, vertex, normal, image, filt, rgb, passthrough):
        eo = self.eo
        return eo.fill_vertex(vertex, filt, passthrough, self.K), eo.fill_normal(normal, filt, passthrough, self.K), eo.fill_image(image, rgb, passthrough)

    def close(self):
        pass


class Product:
    """libefusion.so through the C ABI (stage entry points)."""

    def __init__(self, K):
        from elasticfusion_b200 import capi

        self.K = K
        self.ctx = capi.Context(capi.default_config(K.width, K.height, K.fx, K.fy, K.cx, K.cy, capacity=200000, time_delta=BIG))

    def close(self):
        self.ctx.close()

    def _pre(self, depth):
        c = self.ctx
        c.upload("DEPTH_RAW", depth)
        c.preprocess_depth(c.buffer_ptr("DEPTH_RAW")[0], 3.0, c.buffer_ptr("DEPTH_FILTERED")[0], c.buffer_ptr("DEPTH_METRIC")[0],
                           c.buffer_ptr("DEPTH_METRIC_FILTERED")[0])

    def bilateral(self, depth):
        self._pre(depth)
        return self.ctx.download("DEPTH_FILTERED")

    def metric(self, depth):
        self._pre(depth)
        return self.ctx.download("DEPTH_METRIC")

    def _inputs(self, rgb, depth, filt):
        from oracle import ef_oracle as eo  # (the checker's metric conversion is bit-exact with the product's, asserted above)

        c = self.ctx
        c.upload("RGB", rgb)
        c.upload("DEPTH_RAW", depth)
        c.upload("DEPTH_FILTERED", filt)
        c.upload("DEPTH_METRIC", eo.metric(depth, 3.0))
        c.upload("DEPTH_METRIC_FILTERED", eo.metric(filt, 3.0))

    def first_frame(self, rgb, depth, filt):
        self._inputs(rgb, depth, filt)
        self.ctx.map_initialise()
        return self.ctx.map_download(), None, None

    def _upload_index(self, idx):
        for name, a in zip(("INDEX", "VERT_CONF", "COLOR_TIME", "NORM_RAD"), idx):
            self.ctx.upload(name, a)

    def predict_indices(self, m, T, tick, td):
        c = self.ctx
        c.map_upload(m)
        c.map_predict_indices(T, tick, MAXD, td)
        return tuple(c.download(n) for n in ("INDEX", "VERT_CONF", "COLOR_TIME", "NORM_RAD"))

    def fuse(self, m, T, tick, rgb, depth, filt, idx, w):
        c = self.ctx
        self._inputs(rgb, depth, filt)
        c.map_upload(m)
        self._upload_index(idx)
        c.map_fuse(T, tick, MAXD, w)
        return c.map_download(), c.map_download_new()

    def clean(self, m, new, T, tick, idx, td, nodes=None, depth=None):
        c = self.ctx
        c.map_upload(m)
        assert len(new) == 0 or self._new_ready, "new surfels come from the preceding fuse on this context"
        self._upload_index(idx)
        if nodes is None:
            c.map_clean(T, tick, 10.0, td, MAXD)
        else:
            c.upload("SYNTH_DEPTH", depth)
            c.map_clean_deform(T, tick, 10.0, td, MAXD, nodes)
        return c.map_download()

    _new_ready = False

    def raycast(self, m, T, time, max_time, td, depth_only=False, mode=0):
        c = self.ctx
        c.map_upload(m)
        if depth_only:
            c.map_raycast(T, MAXD, 10.0, time, max_time, td, 2)
            return c.download("SYNTH_DEPTH")
        c.map_raycast(T, MAXD, 10.0, time, max_time, td, mode)
        names = ("IMAGE", "VERTEX", "NORMAL", "TIME") if mode == 0 else ("OLD_IMAGE", "OLD_VERTEX", "OLD_NORMAL", "OLD_TIME")
        return tuple(c.download(n) for n in names)

    def fill(self, vertex, normal, image, filt, rgb, passthrough):
        c = self.ctx
        c.upload("VERTEX", vertex)
        c.upload("NORMAL", normal)
        c.upload("IMAGE", image)
        c.upload("DEPTH_FILTERED", filt)
        c.upload("RGB", rgb)
        c.map_fill_in(bool(passthrough), bool(passthrough))
        return c.download("FILL_VERTEX"), c.download("FILL_NORMAL"), c.download("FILL_IMAGE")


def run_all(S, G, K, is_product):
    T, tick = G["T"], int(G["tick"])
    # ---- depth_bilateral.frag / depth_metric.frag
    d = np.abs(S.bilateral(G["depth0"]).astype(np.int32) - G["gl_bilateral"].astype(np.int32))
    assert d.max() <= 1 and (d > 0).mean() <= 2e-3, (d.max(), (d > 0).mean())  # exp() of the range weight
    assert np.array_equal(S.metric(G["depth0"]) == 0, G["gl_metric"] == 0)
    assert np.abs(S.metric(G["depth0"]) - G["gl_metric"]).max() <= 2.4e-7  # one ulp: value / 1000.0f
    # ---- vertex_feedback.vert/.geom + init_unstable.vert
    m0, n_raw, n_fil = S.first_frame(G["rgb0"], G["depth0"], G["filt0"])
    check_surfels(G, "gl_initial_map", m0, "first-frame map", tol=1e-6)
    m0 = cut(G, "gl_initial_map", m0)
    assert np.array_equal(m0[:, :3], G["gl_initial_map"][:, :3]) and np.array_equal(m0[:, 4:8], G["gl_initial_map"][:, 4:8])
    mb, nb_raw, nb_fil = S.first_frame(G["rgbb"], G["depthb"], G["filtb"])
    assert int(G["gl_boundary_raw_count"]) != int(G["gl_boundary_filt_count"])  # the App. A-29 case is exercised
    if n_raw is not None:
        assert (nb_raw, nb_fil) == (int(G["gl_boundary_raw_count"]), int(G["gl_boundary_filt_count"]))
    check_surfels(G, "gl_boundary_map", mb, "first-frame map across depthCutoff", tol=1e-6)
    # ---- index_map.vert/.frag (incl. the time-window cull)
    idx = S.predict_indices(G["map"], T, tick, BIG)
    assert frac_differ(idx[0], G["gl_index"]) <= 5e-4  # a window coordinate within float rounding of a snapping boundary
    same = idx[0] == G["gl_index"]
    for a, name in zip(idx[1:], ("gl_vert_conf", "gl_color_time", "gl_norm_rad")):
        s = cut(G, name, same)
        assert mad(cut(G, name, a)[s], G[name][s]) <= 1e-6, name
    assert (G["gl_index"] > 0).mean() > 0.5
    idx_t = S.predict_indices(G["map_t"], T, int(G["tick_t"]), int(G["td"]))
    assert frac_differ(idx_t[0], G["gl_index_t"]) <= 5e-4 and 0.1 < (G["gl_index_t"] > 0).mean() < 0.9
    # ---- data.vert/.geom/.frag + update.vert
    idx_in = (G["index_in"], G["vert_conf_in"], G["color_time_in"], G["norm_rad_in"])
    fused, new = S.fuse(G["map"], T, tick, G["rgb4"], G["depth4"], G["filt4"], idx_in, 0.73)
    check_surfels(G, "gl_fused", fused, "fused map", tol=1e-5)
    moved = np.abs(G["gl_fused"][:, :3] - cut(G, "gl_fused", G["map"])[:, :3]).max(axis=1) > 0
    assert moved.mean() * full_len(G, "gl_fused") > 1000
    gl_new, n_matched = fuse_feedback(G)
    assert len(gl_new) > 0 and n_matched > 1000
    check_surfels({"gl_new": gl_new}, "gl_new", new, "new unstable surfels", tol=1e-5)
    # ---- copy_unstable.vert/.geom
    idx2 = (G["index2_in"], G["vert_conf2_in"], G["color_time2_in"], G["norm_rad2_in"])
    if is_product:
        S._new_ready = True  # the product's new-surfel buffer holds what its fuse just emitted
        S.ctx.map_upload(G["fused_in"])
    cleaned = S.clean(G["fused_in"], G["new_in"], T, tick, idx2, BIG)
    check_surfels(G, "gl_cleaned", cleaned, "map after clean", tol=1e-6)
    idx_tin = (G["index_t_in"], G["vert_conf_t_in"], G["color_time_t_in"], G["norm_rad_t_in"])
    none = np.zeros((0, 12), np.float32)
    if is_product:
        S._new_ready = False
        S.ctx.map_upload(G["map_t"][:1])
        S.ctx.map_clean(T, int(G["tick_t"]), 10.0, int(G["td"]), MAXD)  # (drains the new-surfel buffer of the fuse above)
    cleaned_t = S.clean(G["map_t"], none, T, int(G["tick_t"]), idx_tin, int(G["td"]))
    mt = G["map_t"]
    stale = (int(G["tick_t"]) - mt[:, 7] > 20) & (mt[:, 3] < 10.0)
    assert stale.sum() > 1000 and full_len(G, "gl_cleaned_t") == len(mt)  # copy_unstable.vert:126-128 un-culls what left the time window
    check_surfels(G, "gl_cleaned_t", cleaned_t, "map after clean, finite time window", tol=1e-6)
    # ---- copy_unstable.vert with a deformation graph (lines 132-322)
    deformed = S.clean(G["map_t"], none, T, int(G["tick_t"]), idx_tin, int(G["td"]), nodes=G["nodes"], depth=G["synth_depth_t_in"])
    ref = G["gl_cleaned_deformed"]
    assert len(deformed) == full_len(G, "gl_cleaned_deformed") and np.nanmax(np.abs(ref[:, :3] - G["gl_cleaned_t"][:, :3])) > 1e-3
    deformed = cut(G, "gl_cleaned_deformed", deformed)
    assert np.array_equal(np.isnan(deformed), np.isnan(ref))
    ok = ~np.isnan(ref).any(axis=1)
    assert np.abs(deformed[ok][:, [0, 1, 2, 8, 9, 10]] - ref[ok][:, [0, 1, 2, 8, 9, 10]]).max() <= 2e-5
    assert (deformed[ok, 7] != ref[ok, 7]).mean() <= 1e-3  # lastTime refresh: a depth comparison at a 10 cm margin
    # ---- splat.vert + combo_splat.frag / depth_splat.frag: ACTIVE, INACTIVE, depth only
    for m, time, max_time, td, names, mode in ((G["map_stable"], tick, tick, BIG, ("gl_image", "gl_vertex", "gl_normal", "gl_time"), 0),
                                               (G["map_t"], 0, int(G["tick_t"]) - int(G["td"]), int(G["td"]),
                                                ("gl_old_image", "gl_old_vertex", "gl_old_normal", "gl_old_time"), 1)):
        out = S.raycast(m, T, time, max_time, td, mode=mode) if is_product else S.raycast(m, T, time, max_time, td)
        out = [cut(G, n, a) for n, a in zip(names, out)]
        assert frac_differ(out[0], G[names[0]]) <= 5e-4 and frac_differ(out[3], G[names[3]]) <= 5e-4, names  # pow(r, 2) at a disc edge
        same = (out[3] == G[names[3]]) & (out[0] == G[names[0]]).all(axis=-1)
        # (1e-5 m but for a handful of fragments where the ray grazes its disc and the intersection's division amplifies the last
        # bits: 3 of 307 k values reach 1.9e-5 at 320x240)
        assert mad(out[1][same], G[names[1]][same]) <= 5e-5 and mad(out[2][same], G[names[2]][same]) <= 1e-5
        assert frac_differ(out[1][same], G[names[1]][same], 1e-5) <= 1e-4
        assert (G[names[1]][..., 2] > 0).mean() > 0.2
    sd = S.raycast(G["map_stable"], T, tick, tick, BIG, depth_only=True)
    assert frac_differ(cut(G, "gl_synth_depth", sd), G["gl_synth_depth"], 1e-5) <= 5e-4
    # ---- fill_vertex / fill_normal / fill_rgb
    for p, (kv, kn, ki) in ((0, ("gl_fill_vertex", "gl_fill_normal", "gl_fill_image")), (1, ("gl_fill_vertex_pass", None, "gl_fill_image_pass"))):
        fv, fn, fi = S.fill(G["vertex_in"], G["normal_in"], G["image_in"], G["filt4"], G["rgb4"], p)
        fv, fn, fi = cut(G, kv, fv), cut(G, kn, fn) if kn else None, cut(G, ki, fi)
        assert frac_differ(fv, G[kv], 1e-6) == 0
        if kn:
            assert frac_differ(fn, G[kn], 1e-4) <= 1e-3  # normalize(): rsqrt polynomial
        assert_same(fi, G[ki], ki)


def test_oracle_matches_reference_shaders(G, K):
    """oracle/efo_map.cpp == the reference's GLSL on Mesa, pass by pass: the pin of the GL half of the oracle."""
    run_all(Oracle(K), G, K, False)


@pytest.mark.parametrize("config", ["icl", "offcentre", "icl320"])
def test_oracle_matches_reference_shaders_live(config):
    """The same pin in configurations the default fixture does not hold -- the ICL-NUIM camera (fx != fy, half-pixel principal
    point) at a quarter and at half of its resolution, and an off-centre camera with another aspect ratio and faster motion.
    The shaders' outputs were produced by executing them live (tests/golden/make_gl_golden.py) and are stored per configuration."""
    G, K = load(config)
    run_all(Oracle(K), G, K, False)


@pytest.mark.gpu
def test_product_matches_reference_shaders(G, K):
    """libefusion.so == the reference's GLSL on Mesa, pass by pass, through the C ABI."""
    S = Product(K)
    try:
        run_all(S, G, K, True)
    finally:
        S.close()
