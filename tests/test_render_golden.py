"""The global-surface render (draw_global_surface.{vert,geom,frag} / _phong.frag, GlobalModel::renderPointCloud and the colour pass of
GUI::drawFXAA) of the CPU oracle against the reference's own shader files executed on Mesa llvmpipe: tests/golden/ref_render_*.npz
(written by tests/golden/make_render_golden.py) and, where the harness is built, live. Also ef_render_camera against numpy.

Mismatch classes. The oracle rasterises the disc on the quad's plane in float (ef_render.cu uses the same formulation); GL snaps the
strip's vertices to fixed point, sets up two triangles, clips them and interpolates with its own arithmetic. So a pixel may differ
where one of three decisions is within rounding of its threshold, and every differing pixel must be one of:
  * rim: some surfel's |dot(tc, tc) - 1| at the pixel centre is below RIM_EPS;
  * edge: some surfel's pixel centre lies within EDGE_EPS (texcoord units, or NDC depth for the near / far plane) of the strip's
    diagonal, of the quad's border, or of a clip plane;
  * tie: the winner and the best other surfel at the pixel are within TIE_D24 units of 24-bit depth;
  * shade (Phong views only): no channel differs by more than 1. The Phong fragment shader normalises three vectors and raises a
    cosine to the 32nd power; llvmpipe evaluates those with its own approximations, the oracle and the kernels in IEEE float.
The bounds below were set from the first comparison of the fixtures (the shares are printed with -s) and hold with margin.
"""
import os

import numpy as np
import pytest

from elasticfusion_b200 import synth
from oracle import ef_oracle as eo
from oracle import ef_render_oracle as ero

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = os.path.join(HERE, "golden")
FIXTURES = {"160x120": os.path.join(GOLDEN, "ref_render_160x120.npz"), "320x240": os.path.join(GOLDEN, "ref_render_320x240.npz")}

# the map: the CPU oracle after FRAMES frames of the noisy synthetic sequence at 80x60 (its surfels are large enough on screen at
# 160x120 and 320x240 to overlap, and the map stays small enough to keep in the fixture)
MAP_K = synth.Intrinsics(80, 60, 66.0, 66.0, 40.0, 30.0)
FRAMES, SEED = 4, 17

RIM_EPS = 2e-3      # |dot(tc, tc) - 1|
EDGE_EPS = 2e-3     # texcoord units / NDC depth
TIE_D24 = 64        # 24-bit depth units
# share of a view's drawn pixels that may differ at all: the first comparison's largest was 0.08 % (one pixel of the 1208 of the view
# from outside the room), the others 0.02 - 0.04 %
MAX_MISMATCH = 0.005


class View:
    """EfRenderView's fields, as plain attributes."""

    def __init__(self, w, h, mvp, mv, **flags):
        self.width, self.height = int(w), int(h)
        self.mvp, self.mv = [float(x) for x in np.asarray(mvp, np.float32).ravel()], [float(x) for x in np.asarray(mv, np.float32).ravel()]
        self.threshold, self.color_type, self.unstable, self.draw_window = 10.0, 2, 0, 0
        self.time, self.time_delta, self.phong, self.sign_mult = 0, 0, 0, -1.0
        for k, v in flags.items():
            assert hasattr(self, k), k
            setattr(self, k, v)

    def as_array(self):
        """(ints, floats) that describe the view in a fixture."""
        i = np.array([self.width, self.height, self.color_type, self.unstable, self.draw_window, self.time, self.time_delta, self.phong], np.int64)
        f = np.array([self.threshold, self.sign_mult] + list(self.mvp) + list(self.mv), np.float32)
        return i, f

    @staticmethod
    def from_arrays(i, f):
        v = View(i[0], i[1], f[2:18], f[18:34])
        v.color_type, v.unstable, v.draw_window, v.time, v.time_delta, v.phong = (int(x) for x in i[2:8])
        v.threshold, v.sign_mult = float(f[0]), float(f[1])
        return v


def camera_matrices(T_wc, fx, fy, cx, cy, w, h, near, far):
    """numpy statement of ef_render_camera: (mvp, mv), column-major float32 [16]."""
    T = np.asarray(T_wc, np.float64)
    mv = np.eye(4)
    mv[:3, :3] = T[:3, :3].T
    mv[:3, 3] = -T[:3, :3].T @ T[:3, 3]
    P = np.array([[2 * fx / w, 0, 2 * cx / w - 1, 0], [0, 2 * fy / h, 2 * cy / h - 1, 0],
                  [0, 0, (far + near) / (far - near), -2 * far * near / (far - near)], [0, 0, 1, 0]])
    return (P @ mv).astype(np.float32).T.ravel(), mv.astype(np.float32).T.ravel()


def look_at(eye, target, up=(0.0, -1.0, 0.0)):
    """camera-to-world pose at eye looking at target (+z forward, +y down in the image)."""
    eye, target = np.asarray(eye, np.float64), np.asarray(target, np.float64)
    z = target - eye
    z /= np.linalg.norm(z)
    x = np.cross(-np.asarray(up, np.float64), z)
    x /= np.linalg.norm(x)
    y = np.cross(z, x)
    T = np.eye(4)
    T[:3, 0], T[:3, 1], T[:3, 2], T[:3, 3] = x, y, z, eye
    return T


def build_map():
    """(surfels (n,12) float32, last pose, tick) of the oracle after FRAMES frames."""
    ref = eo.Fusion(MAP_K, capacity=200000)
    for i, (rgb, depth, _) in enumerate(synth.sequence(FRAMES, MAP_K, seed=SEED, noise=True)):
        ref.process_frame(rgb, depth, i)
    return ref.map(), ref.pose.copy(), FRAMES


def views(surfels, T, tick, size):
    """name -> View of the fixture at `size` ("160x120" or "320x240")."""
    w, h = (160, 120) if size == "160x120" else (320, 240)
    s = w / MAP_K.width
    fx, fy, cx, cy = MAP_K.fx * s, MAP_K.fy * s, MAP_K.cx * s, MAP_K.cy * s
    # after a few frames no surfel has reached the reference's default threshold of 10: the stable ones here are the upper 60 %
    thr = float(np.percentile(surfels[:, 3], 40))

    def cam(T_, near=0.1, far=1000.0, **kw):
        kw.setdefault("threshold", thr)
        return View(w, h, *camera_matrices(T_, fx, fy, cx, cy, w, h, near, far), **kw)

    pos = surfels[:, :3].astype(np.float64)
    depth = (pos - T[:3, 3]) @ T[:3, 2]
    centre = pos.mean(0)
    out = {}
    if size == "160x120":
        for ct in range(4):
            out[f"type{ct}"] = cam(T, color_type=ct, time=tick)
        out["unstable"] = cam(T, unstable=1)
        out["window"] = cam(T, draw_window=1, time=tick + 3, time_delta=3, color_type=0)
        # an oblique view from outside the room, and one whose near plane cuts the walls in front of the camera
        lo, hi = pos.min(0), pos.max(0)
        eye = centre + np.array([1.2, -0.9, -1.0]) * (hi - lo).max() * 1.5
        out["outside"] = cam(look_at(eye, centre), color_type=1)
        out["near_cut"] = cam(T, near=float(np.percentile(depth, 30)), color_type=0)
        # close to one surfel: single discs cover most of the image
        i = int(np.argmin(np.abs(depth - np.median(depth)) + np.linalg.norm(pos - (T[:3, 3] + T[:3, 2] * np.median(depth)), axis=1)))
        n = surfels[i, 8:11].astype(np.float64)
        n = n if np.dot(n, T[:3, 3] - pos[i]) > 0 else -n
        out["close"] = cam(look_at(pos[i] + n * 1.5 * surfels[i, 11], pos[i]), near=0.005, color_type=1)
        # unstable surfels (confidence below a raised threshold) near the far plane: the depth push drops the ones within a radius
        out["far_unstable"] = cam(T, far=float(depth.max()) * 1.01, unstable=1, color_type=0)
    else:
        out["type2"] = cam(T)
        out["phong_neg"] = cam(T, phong=1, sign_mult=-1.0)
        out["phong_pos"] = cam(T, phong=1, sign_mult=1.0, color_type=0)
        out["unstable"] = cam(T, unstable=1, phong=1)
    return out


def load_fixture(size):
    z = np.load(FIXTURES[size])
    names = [str(x) for x in z["names"]]
    vs = {n: View.from_arrays(z["vi"][k], z["vf"][k]) for k, n in enumerate(names)}
    return z["map"], vs, {n: z["img_" + n] for n in names}


def classify(surfels, view, mine, theirs, keys):
    """(mismatching pixels, counts per class, unexplained pixel list) of two RGBA renders; keys: the oracle's winning keys."""
    diff = np.any(mine != theirs, axis=2)
    nd = int(diff.sum())
    counts = dict(rim=0, edge=0, tie=0, shade=0)
    if nd == 0:
        return 0, counts, []
    rim, edge, runner = ero.render_margins(surfels, view, keys)
    empty = np.uint64(0xFFFFFFFFFFFFFFFF)
    d_win = (keys >> np.uint64(32)).astype(np.int64)
    d_run = (runner >> np.uint64(32)).astype(np.int64)
    tie = (keys != empty) & (runner != empty) & (np.abs(d_win - d_run) <= TIE_D24)
    unexplained = []
    for y, x in zip(*np.nonzero(diff)):
        if rim[y, x] < RIM_EPS:
            counts["rim"] += 1
        elif edge[y, x] < EDGE_EPS:
            counts["edge"] += 1
        elif tie[y, x]:
            counts["tie"] += 1
        elif view.phong and np.abs(mine[y, x].astype(int) - theirs[y, x].astype(int)).max() <= 1:
            counts["shade"] += 1
        else:
            unexplained.append((int(y), int(x), mine[y, x].tolist(), theirs[y, x].tolist(), float(rim[y, x]), float(edge[y, x])))
    return nd, counts, unexplained


def check_against(surfels, views_, images, render, label):
    for name, view in views_.items():
        ref = images[name]
        mine = render(view)
        _, keys = ero.render(surfels, view, keys=True)
        nd, counts, unexplained = classify(surfels, view, mine, ref, keys)
        drawn = max(int(np.count_nonzero(ref[..., 3])), 1)
        print(f"{label} {name}: {drawn} drawn, {nd} differ ({nd / drawn:.4%}): {counts}")
        assert not unexplained, (name, unexplained[:10])
        assert nd <= MAX_MISMATCH * drawn, (name, nd, drawn)


@pytest.mark.parametrize("size", sorted(FIXTURES))
def test_oracle_matches_reference_render(size):
    surfels, vs, images = load_fixture(size)
    assert len(vs) >= 4
    for name, img in images.items():
        assert np.count_nonzero(img[..., 3]) > 0, name  # every view draws something
    check_against(surfels, vs, images, lambda v: ero.render(surfels, v), "oracle")


def test_fixture_views_cover_the_listed_cases():
    _, v1, i1 = load_fixture("160x120")
    _, v2, _ = load_fixture("320x240")
    assert {v.color_type for v in v1.values()} == {0, 1, 2, 3}
    assert {v.unstable for v in v1.values()} == {0, 1} and {v.draw_window for v in v1.values()} == {0, 1}
    assert {v.sign_mult for v in v2.values() if v.phong} == {-1.0, 1.0}
    # the depth push: with the far plane just behind the map, unstable surfels whose depth plus radius reaches 1 are not drawn
    assert np.count_nonzero(i1["far_unstable"][..., 3]) < np.count_nonzero(i1["unstable"][..., 3])


def test_oracle_matches_reference_render_live():
    """The same comparison against the shaders run now (needs oracle/_ref/gl and the reference tree; skipped otherwise)."""
    from oracle import ef_refgl as rg
    from oracle import ef_refgl_render as rgr

    if not rgr.available():
        pytest.skip("Mesa llvmpipe harness (make -C oracle refgl) or the reference shaders are absent")
    import subprocess
    import sys

    script = os.path.join(GOLDEN, "make_render_golden.py")
    r = subprocess.run([sys.executable, script, "--check"], env=rg.env(), capture_output=True, text=True, timeout=1800)
    print(r.stdout[-4000:])
    assert r.returncode == 0, r.stdout[-4000:] + r.stderr[-4000:]


def test_render_camera_matches_numpy():
    """ef_render_camera: a world point projects to the window pixel of its image coordinates, rows as the image has them."""
    from elasticfusion_b200 import capi

    T = look_at([0.3, -0.2, -1.0], [0.1, 0.05, 2.0])
    w, h, fx, fy, cx, cy = 320, 240, 250.0, 260.0, 161.3, 118.7
    v = capi.camera_view(T, fx, fy, cx, cy, w, h, near=0.2, far=50.0)
    mvp, mv = camera_matrices(T, fx, fy, cx, cy, w, h, 0.2, 50.0)
    np.testing.assert_allclose(np.array(v.mvp[:]), mvp, rtol=1e-6, atol=1e-6)
    np.testing.assert_allclose(np.array(v.mv[:]), mv, rtol=1e-6, atol=1e-6)
    rng = np.random.default_rng(0)
    M = np.array(v.mvp[:], np.float64).reshape(4, 4).T
    for _ in range(50):
        u, r, z = rng.uniform(0, w), rng.uniform(0, h), rng.uniform(0.3, 40.0)
        pc = np.array([(u - cx) / fx * z, (r - cy) / fy * z, z, 1.0])
        clip = M @ (T @ pc)
        xw, yw = (clip[0] / clip[3] * 0.5 + 0.5) * w, (clip[1] / clip[3] * 0.5 + 0.5) * h
        assert abs(xw - u) < 1e-3 and abs(yw - r) < 1e-3, (u, r, xw, yw)
        zw = clip[2] / clip[3] * 0.5 + 0.5
        assert abs(zw - (50.0 + 0.2) / (2 * 49.8) + 50.0 * 0.2 / (49.8 * z) - 0.5) < 1e-5
    # invalid input
    for bad in (dict(w=0), dict(w=16385), dict(near=0.0), dict(far=0.1)):
        args = dict(w=w, h=h, near=0.2, far=50.0)
        args.update(bad)
        with pytest.raises(capi.EfError):
            capi.camera_view(T, fx, fy, cx, cy, args["w"], args["h"], near=args["near"], far=args["far"])
    Tn = T.copy()
    Tn[0, 3] = np.nan
    with pytest.raises(capi.EfError):
        capi.camera_view(Tn, fx, fy, cx, cy, w, h)
