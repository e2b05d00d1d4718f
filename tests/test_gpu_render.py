"""ef_render_map / ef_render_map_device on the GPU: the reference's global-surface shaders (tests/golden/ref_render_*.npz, with the
mismatch classes of tests/test_render_golden.py), the CPU oracle on full-size maps, determinism, input validation, and that a render
between frames changes nothing the frame computes."""
import numpy as np
import pytest

import test_render_golden as tr
from elasticfusion_b200 import capi, synth
from oracle import ef_render_oracle as ero

pytestmark = pytest.mark.gpu
BIG = 2147483647 // 2


def ctx_with_map(surfels, K=synth.Intrinsics(160, 120, 132.0, 132.0, 80.0, 60.0), capacity=None, **kw):
    ctx = capi.Context(capi.default_config(K.width, K.height, K.fx, K.fy, K.cx, K.cy, capacity=capacity or max(len(surfels), 1000),
                                           time_delta=BIG, **kw))
    ctx.map_upload(surfels)
    ctx.sync()
    return ctx


def as_capi(v):
    out = capi.EfRenderView()
    for k, t in capi.EfRenderView._fields_:
        val = getattr(v, k)
        setattr(out, k, t(*val[:]) if k in ("mvp", "mv") else val)
    return out


@pytest.mark.parametrize("size", sorted(tr.FIXTURES))
def test_product_matches_reference_render(size):
    surfels, vs, images = tr.load_fixture(size)
    ctx = ctx_with_map(surfels)
    tr.check_against(surfels, vs, images, lambda v: ctx.render(as_capi(v)), "product " + size)
    ctx.close()


# the kernels and the oracle evaluate the same float formulation with no contraction: they are expected to agree bit for bit;
# the bound leaves room for one pixel in 10^5, still classified
ORACLE_SHARE = 1e-5


def check_oracle(surfels, ctx, view, label):
    mine = ctx.render(view)
    ref, keys = ero.render(surfels, view, keys=True)
    nd, counts, unexplained = tr.classify(surfels, view, mine, ref, keys) if np.any(mine != ref) else (0, {}, [])
    drawn = max(int(np.count_nonzero(ref[..., 3])), 1)
    print(f"{label}: {drawn} drawn, {nd} differ from the oracle {counts}")
    assert drawn > 0.2 * view.width * view.height, label
    assert not unexplained and nd <= ORACLE_SHARE * drawn, (label, nd, unexplained[:5])


def test_product_matches_oracle_after_frames(K, frames):
    ctx = capi.Context(capi.default_config(K.width, K.height, K.fx, K.fy, K.cx, K.cy, capacity=1_000_000, time_delta=BIG))
    for i, (rgb, depth, _) in enumerate(frames):
        ctx.process_frame(rgb, depth, i)
    surfels, T, tick = ctx.map_download(), ctx.get_pose(), ctx.get_tick()
    thr = float(np.percentile(surfels[:, 3], 40))
    for name, kw in dict(flat=dict(color_type=2), phong=dict(phong=1, color_type=0), unstable=dict(unstable=1, color_type=3, time=tick),
                         window=dict(draw_window=1, time=tick + 4, time_delta=4, color_type=1)).items():
        v = capi.camera_view(T, K.fx, K.fy, K.cx, K.cy, K.width, K.height, threshold=thr, **kw)
        check_oracle(surfels, ctx, v, "frames " + name)
    ctx.close()


def test_product_matches_oracle_resident_5M():
    K = synth.K_DEFAULT
    room = synth.room_surfels(5_000_000, np.linalg.inv(synth.trajectory(1, seed=42)[0]), view_depth=1.5, focal=K.fx)
    ctx = ctx_with_map(room, K, capacity=5_600_000)
    traj = synth.trajectory(2, seed=42)
    T = np.linalg.inv(traj[0]) @ traj[1]  # frame 1's camera in the world of frame 0
    for name, kw in dict(flat=dict(), phong=dict(phong=1)).items():
        v = capi.camera_view(T, 3 * K.fx, 3 * K.fy, 960.0, 540.0, 1920, 1080, **kw)
        check_oracle(room, ctx, v, "5M " + name)
    ctx.close()


def test_deterministic_and_device_equals_host():
    import torch

    surfels, vs, _ = tr.load_fixture("320x240")
    ctx = ctx_with_map(surfels)
    for name, v in vs.items():
        cv = as_capi(v)
        a, b = ctx.render(cv), ctx.render(cv)
        buf = torch.zeros(v.height * v.width * 4, dtype=torch.uint8, device="cuda")
        ctx.render_device(cv, buf.data_ptr())
        ctx.sync()
        assert np.array_equal(a, b), name
        assert np.array_equal(a, buf.cpu().numpy().reshape(a.shape)), name
    # a larger view grows the render's buffers; a smaller one after it still renders the same image as before
    small = as_capi(tr.load_fixture("160x120")[1]["type2"])
    before = ctx.render(small)
    big = capi.camera_view(np.eye(4), 400.0, 400.0, 640.0, 360.0, 1280, 720)
    ctx.render(big)
    assert np.array_equal(ctx.render(small), before)
    ctx.close()


def test_invalid_views_are_rejected():
    import torch

    ctx = ctx_with_map(tr.load_fixture("160x120")[0])
    good = capi.camera_view(np.eye(4), 132.0, 132.0, 80.0, 60.0, 160, 120)
    buf = torch.zeros(160 * 120 * 4, dtype=torch.uint8, device="cuda")
    out = np.zeros((120, 160, 4), np.uint8)
    bads = []
    for field, val in (("width", 0), ("width", 16385), ("height", 0), ("height", 16385), ("color_type", -1), ("color_type", 4)):
        v = as_capi(good)
        setattr(v, field, val)
        bads.append(v)
    for m, i in (("mvp", 3), ("mvp", 15)):
        v = as_capi(good)
        getattr(v, m)[i] = float("nan")
        bads.append(v)
    v = as_capi(good)
    v.phong, v.mv[12] = 1, float("inf")
    bads.append(v)
    for v in bads:
        assert capi.lib().ef_render_map(ctx.h_ctx, capi.C.byref(v), capi._p(out)) == -1
        assert capi.lib().ef_render_map_device(ctx.h_ctx, capi.C.byref(v), capi.C.c_void_p(buf.data_ptr())) == -1
    # mv is not read without Phong
    v = as_capi(good)
    v.mv[12] = float("nan")
    ctx.render(v)
    ctx.close()


def frame_state(ctx):
    return (ctx.get_pose().copy(), ctx.map_download().tobytes(), ctx.map_count(),
            [ctx.download(b).tobytes() for b in ("INDEX", "VERT_CONF", "COLOR_TIME", "NORM_RAD")])


@pytest.mark.parametrize("close_loops", [2, 0])
def test_render_between_frames_changes_nothing(close_loops):
    """30 frames with a render after every frame (with close_loops = 2: between ef_process_frame_device and ef_finish_frame, the
    next frame staged by the look-ahead) leave poses, map and index textures byte-identical to the same run without renders."""
    import torch

    K = synth.Intrinsics(320, 240, 264.0, 264.0, 160.0, 120.0)
    frames = list(synth.sequence(30, K, seed=9, noise=True))
    dev = [(torch.from_numpy(np.ascontiguousarray(r)).cuda(), torch.from_numpy(np.ascontiguousarray(d).view(np.int16)).cuda()) for r, d, _ in frames]
    buf = torch.zeros(640 * 480 * 4, dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()

    def run(render):
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
            if render:
                T = frames[i][2]
                if i % 2:
                    ctx.render(capi.camera_view(T, K.fx, K.fy, K.cx, K.cy, K.width, K.height, threshold=1.0, unstable=1, color_type=i % 4, time=i + 2))
                else:
                    v = capi.camera_view(T, 2 * K.fx, 2 * K.fy, 2 * K.cx, 2 * K.cy, 640, 480, phong=1, threshold=1.0)
                    ctx.render_device(v, buf.data_ptr())
            if close_loops == 2:
                ctx.finish_frame()
            states.append(frame_state(ctx))
        ctx.close()
        return states

    plain, rendered = run(False), run(True)
    for i, (a, b) in enumerate(zip(plain, rendered)):
        assert np.array_equal(a[0], b[0]), ("pose", i)
        assert a[2] == b[2] and a[1] == b[1], ("map", i)
        assert a[3] == b[3], ("index textures", i)


def read_ppm(path):
    with open(path, "rb") as f:
        data = f.read()
    magic, w, h, mx, rest = data.split(maxsplit=4)
    assert magic == b"P6" and mx == b"255"
    return np.frombuffer(rest, np.uint8).reshape(int(h), int(w), 3)


def test_headless_cli_render_matches_context(tmp_path, small_K, small_frames):
    """tools/ElasticFusionHeadless -render 2: a PPM every 2 frames and after the last one, each equal to Context.render from the pose
    the same frames leave through the C ABI (the map's stable surfels at the input intrinsics, colour type 2). The confidence threshold
    is lowered to 0.5 so that surfels seen once already count as stable."""
    import glob
    import os
    import subprocess

    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    exe = os.path.join(root, "tools", "ElasticFusionHeadless")
    K = small_K
    klg = str(tmp_path / "render.klg")
    synth.write_klg(klg, [(f[0], f[1]) for f in small_frames])
    cal = str(tmp_path / "cal.txt")
    open(cal, "w").write(f"{K.fx} {K.fy} {K.cx} {K.cy}\n")
    subprocess.check_output([exe, "-l", klg, "-cal", cal, "-w", str(K.width), "-h", str(K.height), "-o", "-c", "0.5", "-cap", "500000",
                             "-render", "2"], text=True)
    ppms = sorted(glob.glob(klg + ".render.*.ppm"), key=lambda p: int(p.rsplit(".", 2)[1]))
    n = len(small_frames) - 1  # hasMore() drops the last frame of a log
    assert len(ppms) == 3, ppms
    ctx = capi.Context(capi.default_config(K.width, K.height, K.fx, K.fy, K.cx, K.cy, capacity=500000, time_delta=BIG, confidence=0.5))
    ctx.set_tick(1)  # the CLI's default -s 1
    want = []
    for i, (rgb, d, _) in enumerate(small_frames[:n]):
        ctx.process_frame(rgb, d, i)
        if (i + 1) % 2 == 0 or i + 1 == n:
            img = ctx.render(capi.camera_view(ctx.get_pose(), K.fx, K.fy, K.cx, K.cy, K.width, K.height, threshold=0.5, color_type=2))
            assert np.count_nonzero(img[..., 3]) > 0
            want.append(img[..., :3])
    ctx.close()
    for path, img in zip(ppms, want):
        assert np.array_equal(read_ppm(path), img), path
