"""Device time of one rig frame (ef_rig_frame_device) against the same cameras called one by one (ef_camera_frame_device each), for a
two- and a four-member rig of 640x480 cameras on the map a 640x480 context builds from 8 frames of the synthetic sequence. Member i
sits at frame 1's room pose composed with a fixed offset (a few degrees about y and a few centimetres), sees its rendered RGB-D frame
and tracks it from the pose the previous call left, with fuse = 0 and fuse = 1 (time = tick - 1). Each case is timed by CUDA event
pairs on ef_stream() around each of `--reps` back-to-back calls after `--warmup` calls; the median is reported, with the launches per
call. Prints the card's name and power limit, read in the same run, then one JSON line per case.

    python scripts/rig_bench.py [--reps 100] [--warmup 10]
"""
import argparse
import ctypes
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

from track_view_bench import gpu_info, median_ms  # noqa: E402


def offset(i):
    a = np.radians(6.0 * i)
    T = np.eye(4)
    T[:3, :3] = [[np.cos(a), 0, np.sin(a)], [0, 1, 0], [-np.sin(a), 0, np.cos(a)]]
    T[:3, 3] = (0.04 * i, -0.02 * i, 0.01 * i)
    return T


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=100)
    ap.add_argument("--warmup", type=int, default=10)
    a = ap.parse_args()

    import torch

    import bench
    from elasticfusion_b200 import capi, synth

    if not torch.cuda.is_available():
        raise SystemExit("rig_bench needs a CUDA device")
    print(json.dumps({"gpu": gpu_info()}), flush=True)
    K, seed = synth.K_DEFAULT, 42
    rgb, depth = bench.make_frames(K, 8, seed)
    traj = synth.trajectory(2, seed=seed)
    T = np.linalg.inv(traj[0]) @ traj[1]
    for n in (2, 4):
        ctx = capi.Context(capi.default_config(K.width, K.height, K.fx, K.fy, K.cx, K.cy, capacity=2_000_000))
        for i in range(8):
            ctx.process_frame(rgb[i], depth[i], i)
        tick = ctx.get_tick()
        stream = torch.cuda.ExternalStream(ctx.stream)
        cams = [ctx.camera(capi.camera_config(K.width, K.height, K.fx, K.fy, K.cx, K.cy, time_delta=ctx.cfg.time_delta)) for _ in range(n)]
        inputs = []
        for i in range(n):
            vrgb, vdepth, _, _ = synth.render(traj[1] @ offset(i), K, noise_seed=seed + i)
            inputs.append((torch.from_numpy(np.ascontiguousarray(vrgb)).cuda(), torch.from_numpy(np.ascontiguousarray(vdepth).view(np.int16)).cuda()))
        rp, dp = [r.data_ptr() for r, _ in inputs], [d.data_ptr() for _, d in inputs]
        members = torch.zeros(n * ctypes.sizeof(capi.EfCameraResult), dtype=torch.uint8, device="cuda")
        result = torch.zeros(ctypes.sizeof(capi.EfRigResult), dtype=torch.uint8, device="cuda")
        one = torch.zeros(ctypes.sizeof(capi.EfCameraResult), dtype=torch.uint8, device="cuda")
        torch.cuda.synchronize()
        for fuse in (0, 1):
            for mode in ("cameras", "rig"):
                if mode == "rig":
                    rig = ctx.rig(cams, [offset(i) for i in range(n)])
                    rig.frame_device(rp, dp, members.data_ptr(), result.data_ptr(), tick - 1, T_wc=T, fuse=False)
                    call = lambda: rig.frame_device(rp, dp, members.data_ptr(), result.data_ptr(), tick - 1, fuse=bool(fuse))
                else:
                    for i, c in enumerate(cams):
                        c.frame_device(rp[i], dp[i], one.data_ptr(), tick - 1, T_wc=T @ offset(i), fuse=False)

                    def call():
                        for i, c in enumerate(cams):
                            c.frame_device(rp[i], dp[i], one.data_ptr(), tick - 1, fuse=bool(fuse))
                for _ in range(a.warmup):
                    call()
                ctx.sync()
                l0 = ctx.launch_count()
                call()
                launches = ctx.launch_count() - l0
                t = median_ms(stream, a.reps, call)
                print(json.dumps({"members": n, "mode": mode, "camera": f"{K.width}x{K.height}", "fuse": fuse, "median_ms": round(t, 4),
                                  "reps": a.reps, "launches_per_call": launches}), flush=True)
                if mode == "rig":
                    rig.close()
        ctx.close()


if __name__ == "__main__":
    main()
