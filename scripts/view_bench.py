"""Device time of one model view (ef_map_predict_view_device: k_update_pose + k_splat_scatter + k_splat_resolve, all four outputs) on
the resident room maps bench.py times (5 M and 20 M surfels, built by bench.populate_map through the C ABI: frame 0 of bench.py's
sequence, then the room surfels uploaded), at 640x480 and 1920x1080, ACTIVE window, from frame 1's camera. Each case is timed by a
CUDA event pair around each of `--reps` back-to-back calls after `--warmup` calls; the median is reported. Prints the card's name and
power limit, read in the same run, then one JSON line per case.

sweep_bytes is what the scatter must read of the map: pos_conf + color_time (32 B) of every surfel, and norm_rad (16 B) of every
surfel that survives the vertex stage. Survivors are counted on the host as the stable surfels inside the time window whose centre
lies in front of the camera, within max_depth and projects inside the view (the kernel's frustum test also keeps sprites that
overlap the border, so the count is a lower bound by a thin rim). sweep_share is sweep_bytes over the median time, as a share of the
H100 SXM data-sheet bandwidth of 3.35 TB/s; it leaves out the z-buffer and output traffic, which depend on the view.

    python scripts/view_bench.py [--reps 200] [--warmup 20] [--sizes 5M,20M]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

HBM_BYTES_PER_S = 3.35e12  # H100 SXM data sheet


def gpu_info():
    r = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                       text=True, timeout=30)
    name, power, clock = [c.strip() for c in r.stdout.strip().split(",")]
    return {"name": name, "power_limit": power, "max_sm_clock": clock}


def survivors(room, T_wc, K, w, h, max_depth, conf_threshold):
    """surfels whose norm_rad the scatter reads (room surfels share one time stamp inside the window)"""
    T_cw = np.linalg.inv(T_wc)
    n = 0
    for c0 in range(0, len(room), 1 << 22):
        p = room[c0:c0 + (1 << 22), :3].astype(np.float64) @ T_cw[:3, :3].T + T_cw[:3, 3]
        z = p[:, 2]
        ok = (room[c0:c0 + (1 << 22), 3] >= conf_threshold) & (z > 0) & (z <= max_depth)
        with np.errstate(divide="ignore", invalid="ignore"):
            u, v = K.fx * p[:, 0] / z + K.cx, K.fy * p[:, 1] / z + K.cy
        n += int((ok & (u >= 0) & (u < w) & (v >= 0) & (v < h)).sum())
    return n


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
        raise SystemExit("view_bench needs a CUDA device")
    print(json.dumps({"gpu": gpu_info()}), flush=True)
    K, seed = synth.K_DEFAULT, 42
    rgb, depth = bench.make_frames(K, 1, seed)
    traj = synth.trajectory(2, seed=seed)
    T = np.linalg.inv(traj[0]) @ traj[1]  # frame 1's camera in the world of frame 0
    for size in a.sizes.split(","):
        n_target = {"5M": 5_000_000, "20M": 20_000_000}[size]
        ctx = capi.Context(capi.default_config(K.width, K.height, K.fx, K.fy, K.cx, K.cy, capacity=int(n_target * 1.1) + 400_000))
        n = bench.populate_map(ctx, K, n_target, seed, rgb[0], depth[0])
        room = ctx.map_download()
        tick, td = ctx.get_tick(), ctx.cfg.time_delta
        stream = torch.cuda.ExternalStream(ctx.stream)
        for (w, h) in ((640, 480), (1920, 1080)):
            s = h / K.height
            Kv = synth.Intrinsics(w, h, K.fx * s, K.fy * s, w / 2, h / 2)
            v = capi.model_view(T, Kv.fx, Kv.fy, Kv.cx, Kv.cy, w, h, 20.0, 10.0, tick, tick, td)
            bufs = [torch.empty(w * h * b, dtype=torch.uint8, device="cuda") for b in (4, 16, 16, 2)]
            ptrs = [b.data_ptr() for b in bufs]
            for _ in range(a.warmup):
                ctx.predict_view_device(v, *ptrs)
            ctx.sync()
            ev = [torch.cuda.Event(enable_timing=True) for _ in range(a.reps + 1)]
            ev[0].record(stream)
            for i in range(a.reps):
                ctx.predict_view_device(v, *ptrs)
                ev[i + 1].record(stream)
            ev[-1].synchronize()
            ms = float(np.median([ev[i].elapsed_time(ev[i + 1]) for i in range(a.reps)]))
            covered = float((ctx.predict_view(v, ("vertex",))["vertex"][..., 2] > 0).mean())
            surv = survivors(room, T, Kv, w, h, 20.0, 10.0)
            sweep = 32 * n + 16 * surv
            print(json.dumps({"surfels": n, "view": f"{w}x{h}", "window": "active", "median_ms": round(ms, 4), "reps": a.reps,
                              "covered": round(covered, 3), "survivors": surv, "sweep_bytes": sweep,
                              "sweep_GBps": round(sweep / (ms * 1e-3) / 1e9, 1),
                              "sweep_share": round(sweep / (ms * 1e-3) / HBM_BYTES_PER_S, 3)}), flush=True)
        ctx.close()
        del room


if __name__ == "__main__":
    main()
