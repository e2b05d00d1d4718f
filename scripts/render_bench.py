"""Device time of one map render (ef_render_map_device: k_render_scatter + k_render_resolve) on resident room maps of 5 M and
20 M surfels (synth.room_surfels, as bench.py builds them), at 640x480 and 1920x1080, flat (colour type 2) and Phong, from frame 1 of
bench.py's sequence. Times come from CUDA events around `--reps` back-to-back renders after `--warmup` renders of the same case.
Prints one JSON line per case and the card's name and power limit, read in the same run.

achieved_GBps counts the algorithmic minimum of bytes a render must move: 16 B per resident surfel for the cull read (position and
confidence) plus 48 B per surfel that survives the vertex shader's test (its whole record). It leaves out the image and the z-buffer
traffic, which depend on the view and on overdraw.

    python scripts/render_bench.py [--reps 50] [--warmup 10] [--sizes 5M,20M]
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
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--sizes", default="5M,20M")
    a = ap.parse_args()

    import torch

    from elasticfusion_b200 import capi, synth

    if not torch.cuda.is_available():
        raise SystemExit("render_bench needs a CUDA device")
    print(json.dumps({"gpu": gpu_info()}), flush=True)
    K = synth.K_DEFAULT
    traj = synth.trajectory(2, seed=42)
    T = np.linalg.inv(traj[0]) @ traj[1]
    for size in a.sizes.split(","):
        n = {"5M": 5_000_000, "20M": 20_000_000}[size]
        room = synth.room_surfels(n, np.linalg.inv(traj[0]), view_depth=1.5, focal=K.fx)
        ctx = capi.Context(capi.default_config(K.width, K.height, K.fx, K.fy, K.cx, K.cy, capacity=len(room) + 1000))
        ctx.map_upload(room)
        ctx.sync()
        stream = torch.cuda.ExternalStream(ctx.stream)
        for (w, h) in ((640, 480), (1920, 1080)):
            s = w / K.width if w == 640 else 1080 / K.height
            buf = torch.empty(w * h * 4, dtype=torch.uint8, device="cuda")
            for mode, kw in (("flat", dict(color_type=2)), ("phong", dict(phong=1, color_type=2))):
                v = capi.camera_view(T, K.fx * s, K.fy * s, w / 2, h / 2, w, h, **kw)
                for _ in range(a.warmup):
                    ctx.render_device(v, buf.data_ptr())
                ctx.sync()
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record(stream)
                for _ in range(a.reps):
                    ctx.render_device(v, buf.data_ptr())
                e1.record(stream)
                e1.synchronize()
                ms = e0.elapsed_time(e1) / a.reps
                img = ctx.render(v)
                stable = int((room[:, 3] > v.threshold).sum())
                min_bytes = 16 * len(room) + 48 * stable
                print(json.dumps({"surfels": len(room), "view": f"{w}x{h}", "mode": mode, "ms": round(ms, 4),
                                  "pixels_drawn": int(np.count_nonzero(img[..., 3])), "surviving_surfels": stable,
                                  "min_bytes": min_bytes, "achieved_GBps": round(min_bytes / (ms * 1e-3) / 1e9, 1)}), flush=True)
        ctx.close()
        del room


if __name__ == "__main__":
    main()
