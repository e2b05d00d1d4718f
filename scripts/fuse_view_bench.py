"""Device time of one fuse view (ef_map_fuse_view_device: pose staging, preprocess, two index-map passes, fuse and clean) on the resident
room maps bench.py times (5 M and 20 M surfels, built by bench.populate_map through the C ABI: frame 0 of bench.py's sequence, then the
room surfels uploaded), at 640x480 and 1920x1080 views from frame 1's camera, with that camera's rendered RGB-D frame as input. Each case
is timed by a CUDA event pair around each of `--reps` back-to-back calls after `--warmup` calls; the median is reported. Every call
fuses into the map the previous one left (the first calls add the view's new surfels, later ones mostly update them); the map is
uploaded fresh before each case and its count after the timed calls is printed. Prints the card's name and power limit, read in the
same run, then one JSON line per case.

    python scripts/fuse_view_bench.py [--reps 200] [--warmup 20] [--sizes 5M,20M]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def gpu_info():
    r = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                       text=True, timeout=30)
    name, power, clock = [c.strip() for c in r.stdout.strip().split(",")]
    return {"name": name, "power_limit": power, "max_sm_clock": clock}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--sizes", default="5M,20M")
    a = ap.parse_args()

    import torch

    import bench
    from elasticfusion_b200 import capi, synth

    if not torch.cuda.is_available():
        raise SystemExit("fuse_view_bench needs a CUDA device")
    print(json.dumps({"gpu": gpu_info()}), flush=True)
    K, seed = synth.K_DEFAULT, 42
    rgb, depth = bench.make_frames(K, 1, seed)
    traj = synth.trajectory(2, seed=seed)
    T = np.linalg.inv(traj[0]) @ traj[1]  # frame 1's camera in the world of frame 0
    for size in a.sizes.split(","):
        n_target = {"5M": 5_000_000, "20M": 20_000_000}[size]
        ctx = capi.Context(capi.default_config(K.width, K.height, K.fx, K.fy, K.cx, K.cy, capacity=int(n_target * 1.1) + 2_000_000))
        n = bench.populate_map(ctx, K, n_target, seed, rgb[0], depth[0])
        room = ctx.map_download()
        tick, td = ctx.get_tick(), ctx.cfg.time_delta
        stream = torch.cuda.ExternalStream(ctx.stream)
        for (w, h) in ((640, 480), (1920, 1080)):
            s = h / K.height
            Kv = synth.Intrinsics(w, h, K.fx * s, K.fy * s, w / 2, h / 2)
            vrgb, vdepth, _, _ = synth.render(traj[1], Kv, noise_seed=seed)
            r = torch.from_numpy(np.ascontiguousarray(vrgb)).cuda()
            d = torch.from_numpy(np.ascontiguousarray(vdepth).view(np.int16)).cuda()
            v = capi.fuse_view(T, Kv.fx, Kv.fy, Kv.cx, Kv.cy, w, h, tick - 1, weighting=1.0, time_delta=td)
            ctx.map_upload(room)
            for _ in range(a.warmup):
                ctx.fuse_view_device(v, r.data_ptr(), d.data_ptr())
            ctx.sync()
            ev = [torch.cuda.Event(enable_timing=True) for _ in range(a.reps + 1)]
            ev[0].record(stream)
            for i in range(a.reps):
                ctx.fuse_view_device(v, r.data_ptr(), d.data_ptr())
                ev[i + 1].record(stream)
            ev[-1].synchronize()
            ms = float(np.median([ev[i].elapsed_time(ev[i + 1]) for i in range(a.reps)]))
            print(json.dumps({"surfels": n, "view": f"{w}x{h}", "median_ms": round(ms, 4), "reps": a.reps, "count_after": ctx.map_count()}),
                  flush=True)
        ctx.close()
        del room


if __name__ == "__main__":
    main()
