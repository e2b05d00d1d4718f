"""Device time of one camera frame (ef_camera_frame_device) at 424x240, 640x480, 1280x720 and 1920x1080, on two maps: the one a
640x480 context builds from 8 frames of the synthetic sequence, and the resident room map of 5 M surfels that bench.py times
(bench.populate_map). The camera sits at frame 1's room pose of the sequence, seen by a camera of that size (the same field of view as
the context's); its first call sets that pose, then every call tracks its rendered RGB-D frame from the pose the previous call left,
with fuse = 0 (track and predict) and fuse = 1 (also fuse and clean, at time = tick - 1). Each case is timed by CUDA event pairs around
each of `--reps` back-to-back calls after `--warmup` calls; the median is reported, with the device memory the camera's creation took
(cudaMemGetInfo before and after, so rounded to the allocator's pages; it includes any growth of the z-buffer the camera shares with the
context's other off-frame passes). Prints the card's name and power limit, read in the same run, then one JSON line per case.

    python scripts/camera_bench.py [--reps 200] [--warmup 20] [--maps sequence,5M]
"""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

from track_view_bench import gpu_info, median_ms  # noqa: E402

SIZES = ((424, 240), (640, 480), (1280, 720), (1920, 1080))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--maps", default="sequence,5M")
    a = ap.parse_args()

    import torch

    import bench
    from elasticfusion_b200 import capi, synth

    if not torch.cuda.is_available():
        raise SystemExit("camera_bench needs a CUDA device")
    print(json.dumps({"gpu": gpu_info()}), flush=True)
    K, seed = synth.K_DEFAULT, 42
    rgb, depth = bench.make_frames(K, 8, seed)
    traj = synth.trajectory(2, seed=seed)
    T = np.linalg.inv(traj[0]) @ traj[1]  # frame 1's camera in the world of frame 0
    for name in a.maps.split(","):
        if name == "sequence":
            ctx = capi.Context(capi.default_config(K.width, K.height, K.fx, K.fy, K.cx, K.cy, capacity=2_000_000))
            for i in range(8):
                ctx.process_frame(rgb[i], depth[i], i)
            n = ctx.map_count()
        else:
            n_target = {"5M": 5_000_000}[name]
            ctx = capi.Context(capi.default_config(K.width, K.height, K.fx, K.fy, K.cx, K.cy, capacity=int(n_target * 1.1) + 2_000_000))
            n = bench.populate_map(ctx, K, n_target, seed, rgb[0], depth[0])
        tick = ctx.get_tick()
        stream = torch.cuda.ExternalStream(ctx.stream)
        for (w, h) in SIZES:
            sc = h / K.height
            Kv = synth.Intrinsics(w, h, K.fx * sc, K.fy * sc, w / 2, h / 2)
            vrgb, vdepth, _, _ = synth.render(traj[1], Kv, noise_seed=seed)
            r = torch.from_numpy(np.ascontiguousarray(vrgb)).cuda()
            d = torch.from_numpy(np.ascontiguousarray(vdepth).view(np.int16)).cuda()
            out = torch.zeros(capi.C.sizeof(capi.EfCameraResult), dtype=torch.uint8, device="cuda")
            torch.cuda.synchronize()
            free0 = torch.cuda.mem_get_info()[0]
            cam = ctx.camera(capi.camera_config(w, h, Kv.fx, Kv.fy, Kv.cx, Kv.cy, time_delta=ctx.cfg.time_delta))
            created = free0 - torch.cuda.mem_get_info()[0]
            for fuse in (0, 1):
                cam.frame_device(r.data_ptr(), d.data_ptr(), out.data_ptr(), tick - 1, T_wc=T, fuse=False)
                call = lambda: cam.frame_device(r.data_ptr(), d.data_ptr(), out.data_ptr(), tick - 1, fuse=bool(fuse))
                for _ in range(a.warmup):
                    call()
                ctx.sync()
                t = median_ms(stream, a.reps, call)
                Tt, st, _, info = capi.unpack_camera_result(out.cpu().numpy().tobytes())
                print(json.dumps({"map": name, "surfels_before": n, "surfels_after": ctx.map_count(), "camera": f"{w}x{h}", "fuse": fuse,
                                  "median_ms": round(t, 4), "reps": a.reps, "create_bytes": int(created),
                                  "create_bytes_per_px": round(created / (w * h), 1), "pose_err_mm": round(1000 * float(np.abs(Tt - T)[:3, 3].max()), 3),
                                  "icp_count": float(st["lastICPCount"]), "dense_enough": info["dense_enough"]}), flush=True)
            cam.close()
        ctx.close()


if __name__ == "__main__":
    main()
