"""Cost of a camera that closes local loops (EfCameraConfig.close_loops = 1), on an H100.

1. The rig of tests/test_gpu_camera_loops.py: frame A on the 130-frame 320x240 loop sequence (seed 21, speed 2.5; time_delta 12,
   count_thresh 3000, cov_thresh 1e-4) with close_loops = 2 and the look-ahead, camera B at 424x240 with its device call between
   ef_process_frame_device and ef_finish_frame. Device time of each ef_camera_frame_device call (CUDA events recorded on the context's
   stream right before and after the call; with close_loops = 1 this includes the stream's idle time while the host reads the front
   half's record and the solve's result), for close_loops = 0, and for close_loops = 1 split into calls without a closure and calls
   that applied one. The first call (has_pose, no front half) is left out.
2. The extra device memory of a closing camera over an open-loop one, from cudaMemGetInfo around ef_camera_create, at 424x240,
   640x480 and 1920x1080.

Prints the card's name and power limit first. Usage: python scripts/camera_loop_cost.py [--frames N]
"""
import argparse
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from elasticfusion_b200 import capi, synth  # noqa: E402

LOOP_CFG = dict(time_delta=12, count_thresh=3000, err_thresh=5e-5, cov_thresh=1e-4, capacity=400000)
K_A = synth.Intrinsics(320, 240, 264.0, 264.0, 160.0, 120.0)
K_B = synth.Intrinsics(424, 240, 305.0, 305.0, 212.0, 120.0)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, check=True)
    return q.stdout.strip().split("\n")[0]


def make_ctx(K, **kw):
    return capi.Context(capi.default_config(K.width, K.height, K.fx, K.fy, K.cx, K.cy, **kw))


def cam_cfg(K, close_loops):
    return capi.camera_config(K.width, K.height, K.fx, K.fy, K.cx, K.cy, time_delta=LOOP_CFG["time_delta"], close_loops=close_loops)


def cam_offset(deg=8.0, t=(0.05, -0.03, 0.02)):
    a = np.radians(deg)
    T = np.eye(4)
    T[:3, :3] = [[np.cos(a), 0, np.sin(a)], [0, 1, 0], [-np.sin(a), 0, np.cos(a)]]
    T[:3, 3] = t
    return T


def stats(ms):
    if not ms:
        return "n   0"
    a = np.array(ms)
    return f"n {len(a):3d}  median {np.median(a):7.3f} ms  max {a.max():7.3f} ms"


def rig(n, close_loops):
    """per camera call after the first: (device ms, applied a closure)"""
    import torch

    frames = list(synth.sequence(n, K_A, seed=21, noise=True, speed=2.5))
    traj = synth.trajectory(n, seed=21, speed=2.5)
    T_AB = cam_offset()
    bframes = [synth.render(traj[i] @ T_AB, K_B, noise_seed=500 + i)[:2] for i in range(n)]
    first = np.linalg.inv(traj[0]) @ traj[0] @ T_AB

    def dev(a):
        a = np.ascontiguousarray(a)
        return torch.from_numpy(a.view(np.int16) if a.dtype == np.uint16 else a).cuda()

    fa = [(dev(r), dev(d)) for r, d, _ in frames]
    fb = [(dev(r), dev(d)) for r, d in bframes]
    out = torch.zeros(capi.C.sizeof(capi.EfCameraResult), dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()
    ctx = make_ctx(K_A, close_loops=2, **LOOP_CFG)
    cam = ctx.camera(cam_cfg(K_B, close_loops))
    stream = torch.cuda.ExternalStream(ctx.stream)
    res = []
    try:
        ctx.prefetch_frame_device(fa[0][0].data_ptr(), fa[0][1].data_ptr())
        for i in range(n):
            ctx.process_frame_device(None, None, i)
            if i + 1 < n:
                ctx.prefetch_frame_device(fa[i + 1][0].data_ptr(), fa[i + 1][1].data_ptr())
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(stream)
            cam.frame_device(fb[i][0].data_ptr(), fb[i][1].data_ptr(), out.data_ptr(), i + 1, T_wc=first if i == 0 else None)
            e1.record(stream)
            ctx.finish_frame()
            ctx.sync()
            if i > 0:
                res.append((e0.elapsed_time(e1), bool(close_loops and cam.deform_result()[0]["applied"])))
    finally:
        cam.close()
        ctx.close()
    return res


def extra_memory(K):
    """bytes a closing camera takes beyond an open-loop one of the same size"""
    import torch

    ctx = make_ctx(K_A, close_loops=2, capacity=100_000)
    try:
        free = []
        for close_loops in (0, 1):
            torch.cuda.synchronize()
            f0 = torch.cuda.mem_get_info()[0]
            cam = ctx.camera(cam_cfg(K, close_loops))
            torch.cuda.synchronize()
            free.append(f0 - torch.cuda.mem_get_info()[0])
            cam.close()
        return free[1] - free[0], free[0]
    finally:
        ctx.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=130)
    a = ap.parse_args()
    print("card:", card())
    rig(12, 1)  # module load, first launches
    print(f"rig: frame A {K_A.width}x{K_A.height} (close_loops = 2, look-ahead), camera B {K_B.width}x{K_B.height}, {a.frames} frames; "
          "device time per ef_camera_frame_device (first call excluded)")
    r0 = rig(a.frames, 0)
    print("  close_loops = 0                    ", stats([t for t, _ in r0]))
    r1 = rig(a.frames, 1)
    print("  close_loops = 1, no closure applied", stats([t for t, ap_ in r1 if not ap_]))
    print("  close_loops = 1, closure applied   ", stats([t for t, ap_ in r1 if ap_]))
    print("extra device memory of a closing camera (cudaMemGetInfo, 2 MiB granularity):")
    for w, h, f in ((424, 240, 305.0), (640, 480, 528.0), (1920, 1080, 1188.0)):
        K = synth.Intrinsics(w, h, f, f, w / 2, h / 2)
        extra, base = extra_memory(K)
        print(f"  {w}x{h}: {extra / 2**20:8.1f} MiB = {extra / (w * h):6.1f} B per pixel (an open-loop camera: {base / 2**20:8.1f} MiB)")


if __name__ == "__main__":
    main()
