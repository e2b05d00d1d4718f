"""Cost of closing local loops inside the frame (close_loops = 2) against the open-loop modes, on an H100.

1. The 130-frame 320x240 loop sequence (seed 21, speed 2.5; time_delta 12, count_thresh 3000, cov_thresh 1e-4) under close_loops =
   0, 1 and 2: milliseconds per ef_process_frame (host clock around the call, which returns after a stream synchronise), split
   into frames whose loop-closure front half accepted and frames where it did not; for mode 2 also the frames that applied a
   graph.
2. One accepted closure on a resident ~5.2 M-surfel 640x480 map, which samples the full 1023-node graph: the frame under mode 2
   against the same frame under mode 1 (front half only). Every registration is accepted there (thresholds opened), so the
   closure's size, not its quality, is what is measured.

Prints the card's name and power limit first. Usage: python scripts/loop_closure_cost.py [--frames N]
"""
import argparse
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from elasticfusion_b200 import capi, synth  # noqa: E402

LOOP_CFG = dict(time_delta=12, count_thresh=3000, err_thresh=5e-5, cov_thresh=1e-4, capacity=400000)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, check=True)
    return q.stdout.strip().split("\n")[0]


def make_ctx(K, **kw):
    return capi.Context(capi.default_config(K.width, K.height, K.fx, K.fy, K.cx, K.cy, **kw))


def timed_frame(ctx, rgb, depth, i, T=None):
    t0 = time.perf_counter()
    ctx.process_frame(rgb, depth, i, T_wc=T)
    return (time.perf_counter() - t0) * 1e3


def stats(ms):
    if not ms:
        return "n 0"
    a = np.array(ms)
    return f"n {len(a):3d}  median {np.median(a):7.2f} ms  mean {a.mean():7.2f} ms  max {a.max():7.2f} ms"


def loop_sequence(n_frames):
    K = synth.Intrinsics(320, 240, 264.0, 264.0, 160.0, 120.0)
    frames = list(synth.sequence(n_frames, K, seed=21, noise=True, speed=2.5))
    warm = make_ctx(K, close_loops=2, **LOOP_CFG)  # module load, first launches
    for i, (rgb, depth, _) in enumerate(frames[:10]):
        warm.process_frame(rgb, depth, i)
    warm.close()
    print(f"loop sequence: {n_frames} frames at {K.width}x{K.height}, per ef_process_frame (frame 0 excluded)")
    for mode in (0, 1, 2):
        ctx = make_ctx(K, close_loops=mode, **LOOP_CFG)
        acc, rej, applied = [], [], []
        for i, (rgb, depth, _) in enumerate(frames):
            ms = timed_frame(ctx, rgb, depth, i)
            if i == 0:
                continue
            accepted = mode > 0 and ctx.local_loop_result()[0]["accepted"]
            (acc if accepted else rej).append(ms)
            if mode == 2:
                info, _ = ctx.local_deform_result()
                if info["applied"]:
                    applied.append((ms, info["result"]["n_nodes"], info["result"]["n_constraints"], info["result"]["iterations"]))
        if mode == 0:
            print(f"  mode 0            all       {stats(rej)}")
        else:
            print(f"  mode {mode}  front half accepted   {stats(acc)}")
            print(f"  mode {mode}  front half rejected   {stats(rej)}")
        if mode == 2:
            print(f"  mode 2  graph applied         {stats([a[0] for a in applied])}")
            if applied:
                print(f"          nodes {min(a[1] for a in applied)}..{max(a[1] for a in applied)}, constraints incl. pins "
                      f"{min(a[2] for a in applied)}..{max(a[2] for a in applied)}, iterations {sorted(set(a[3] for a in applied))}, "
                      f"deforms {ctx.local_deform_result()[0]['deforms']}")
        ctx.close()


def resident_closure():
    K = synth.K_DEFAULT
    frames = list(synth.sequence(3, K, seed=42, noise=True))
    room = synth.room_surfels(5_200_000, np.linalg.inv(synth.trajectory(1, seed=42)[0]), view_depth=1.5, focal=K.fx)
    n = len(room)
    m = room.copy()
    idx = np.arange(n)
    inactive = idx % 2 == 0
    m[:, 6] = (1 + np.floor(idx * 250.0 / n)).astype(np.float32)  # init times ascending with the index, as a map built over time
    m[:, 7] = np.where(inactive, 40.0, 295.0).astype(np.float32)  # at tick 300, time_delta 200: half INACTIVE
    m[inactive, 0:3] += np.array([0.004, -0.003, 0.002], np.float32)
    print(f"resident map: {n} surfels at {K.width}x{K.height}; every registration accepted")
    for mode in (1, 2, 1, 2):
        ctx = make_ctx(K, close_loops=mode, capacity=5_600_000, time_delta=200, count_thresh=0, err_thresh=1e30, cov_thresh=1e30)
        ctx.process_frame(frames[0][0], frames[0][1], 0)
        ctx.map_upload(m)
        ctx.set_tick(300)
        ctx.predict()
        ctx.process_frame(frames[1][0], frames[1][1], 1, T_wc=frames[1][2])  # mode 2: samples the 1023-node graph at its end
        ms = timed_frame(ctx, frames[2][0], frames[2][1], 2, T=frames[2][2])
        lr = ctx.local_loop_result()[0]
        line = f"  mode {mode}  frame {ms:8.2f} ms  front half accepted {lr['accepted']}, {lr['n_constraints']} constraints"
        if mode == 2:
            info, _ = ctx.local_deform_result()
            r = info["result"]
            line += (f"; applied {info['applied']}: {r['n_nodes']} nodes, {r['n_constraints']} constraints, {r['iterations']} iterations, "
                     f"stop {r['stop']}")
        print(line + f", {ctx.map_count()} surfels")
        ctx.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=130)
    args = ap.parse_args()
    print("card:", card())
    loop_sequence(args.frames)
    resident_closure()
    print("card:", card())


if __name__ == "__main__":
    main()
