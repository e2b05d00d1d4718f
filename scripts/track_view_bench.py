"""Device time of one track view (ef_track_view_device) on the resident room maps bench.py times (5 M and 20 M surfels, built by
bench.populate_map through the C ABI: frame 0 of bench.py's sequence, then the room surfels uploaded), at 640x480 and 1920x1080 views of
frame 1's camera, with that camera's rendered RGB-D frame as input and a guess 1 cm / 1 degree off its pose. Each case is timed by CUDA
event pairs around each of `--reps` back-to-back calls after `--warmup` calls; the median is reported. The two parts are timed the same
way on their own: the prediction (ef_map_predict_view_device of the view's model into device buffers) and the rest (the call's median
minus the prediction's). Prints the card's name and power limit, read in the same run, then one JSON line per case.

    python scripts/track_view_bench.py [--reps 200] [--warmup 20] [--sizes 5M,20M]
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


def median_ms(stream, reps, call):
    import torch

    ev = [torch.cuda.Event(enable_timing=True) for _ in range(reps + 1)]
    ev[0].record(stream)
    for i in range(reps):
        call()
        ev[i + 1].record(stream)
    ev[-1].synchronize()
    return float(np.median([ev[i].elapsed_time(ev[i + 1]) for i in range(reps)]))


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
        raise SystemExit("track_view_bench needs a CUDA device")
    print(json.dumps({"gpu": gpu_info()}), flush=True)
    K, seed = synth.K_DEFAULT, 42
    rgb, depth = bench.make_frames(K, 1, seed)
    traj = synth.trajectory(2, seed=seed)
    T = np.linalg.inv(traj[0]) @ traj[1]  # frame 1's camera in the world of frame 0
    c, s = np.cos(np.radians(1.0)), np.sin(np.radians(1.0))
    D = np.array([[c, 0, s, 0.01], [0, 1, 0, 0], [-s, 0, c, 0], [0, 0, 0, 1.0]])
    guess = T @ D
    for size in a.sizes.split(","):
        n_target = {"5M": 5_000_000, "20M": 20_000_000}[size]
        ctx = capi.Context(capi.default_config(K.width, K.height, K.fx, K.fy, K.cx, K.cy, capacity=int(n_target * 1.1) + 2_000_000))
        n = bench.populate_map(ctx, K, n_target, seed, rgb[0], depth[0])
        tick, td = ctx.get_tick(), ctx.cfg.time_delta
        stream = torch.cuda.ExternalStream(ctx.stream)
        for (w, h) in ((640, 480), (1920, 1080)):
            sc = h / K.height
            Kv = synth.Intrinsics(w, h, K.fx * sc, K.fy * sc, w / 2, h / 2)
            vrgb, vdepth, _, _ = synth.render(traj[1], Kv, noise_seed=seed)
            r = torch.from_numpy(np.ascontiguousarray(vrgb)).cuda()
            d = torch.from_numpy(np.ascontiguousarray(vdepth).view(np.int16)).cuda()
            out = torch.zeros(capi.C.sizeof(capi.EfTrackResult), dtype=torch.uint8, device="cuda")
            img = torch.zeros(w * h * 4, dtype=torch.uint8, device="cuda")
            vtx = torch.zeros(w * h * 4, dtype=torch.float32, device="cuda")
            nrm = torch.zeros(w * h * 4, dtype=torch.float32, device="cuda")
            torch.cuda.synchronize()
            v = capi.track_view(guess, Kv.fx, Kv.fy, Kv.cx, Kv.cy, w, h, tick, time_delta=td)
            track = lambda: ctx.track_view_device(v, r.data_ptr(), d.data_ptr(), out.data_ptr())
            predict = lambda: ctx.predict_view_device(v.model, image=img.data_ptr(), vertex=vtx.data_ptr(), normal=nrm.data_ptr())
            for _ in range(a.warmup):
                track()
                predict()
            ctx.sync()
            t_all = median_ms(stream, a.reps, track)
            t_pred = median_ms(stream, a.reps, predict)
            Tt, st, _, dense = capi.unpack_track_result(out.cpu().numpy().tobytes())
            print(json.dumps({"surfels": n, "view": f"{w}x{h}", "median_ms": round(t_all, 4), "predict_ms": round(t_pred, 4),
                              "track_ms": round(t_all - t_pred, 4), "reps": a.reps, "pose_err_mm": round(1000 * float(np.abs(Tt - T)[:3, 3].max()), 3),
                              "icp_count": float(st["lastICPCount"]), "dense_enough": dense}), flush=True)
        ctx.close()


if __name__ == "__main__":
    main()
