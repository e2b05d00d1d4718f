"""Cost of a rig that closes local loops (every member with EfCameraConfig.close_loops = 1), on an H100.

Rigs of 2 and 4 cameras at 640x480 on the map a 640x480 context (close_loops = 2) builds from 8 frames of the synthetic sequence. Member i
sits at frame 1's room pose composed with a fixed offset and sees its rendered RGB-D frame; after a has_pose call with fuse = 0, each
timed call tracks and fuses at time = tick - 1. Three cases, each against the same members called one by one (ef_camera_frame_device
each) as closing cameras:

- an open-loop rig (every member close_loops = 0), against open-loop cameras;
- a closing rig on calls without a closure: the context's thresholds (count_thresh 35000 is not reached, so nothing is accepted);
- a closing rig on calls with an applied closure: every registration accepted and a displaced INACTIVE copy of the map (time_delta 4,
  confidence 2), so that calls from the fifth on solve and apply.

Each call is timed by a CUDA event pair on ef_stream() around it; with closing members this includes the stream's idle time while the
host reads the front half's record and the solve's result. Calls are sorted by whether the rig (or any camera) applied a closure, and
the median of each class is reported. Prints the card's name and power limit, read in the same run, then one JSON line per case.

    python scripts/rig_loop_cost.py [--calls 40]
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

from rig_bench import offset  # noqa: E402
from track_view_bench import gpu_info  # noqa: E402

FORCED = dict(time_delta=4, confidence=2.0, count_thresh=0, err_thresh=1e30, cov_thresh=1e30)


def inactive_copy(m, time_delta):
    """m displaced by a few millimetres, confident and last seen at -time_delta: only the INACTIVE prediction draws it"""
    c = m.copy()
    c[:, 0:3] += np.array([0.004, -0.003, 0.002], np.float32)
    c[:, 3] += 10.0
    c[:, 6], c[:, 7] = 1.0, -float(time_delta)
    return c


def run_case(n, forced, mode, calls):
    """median ms per call with and without an applied closure, and the count of each; mode: open_rig, open_cameras, rig, cameras"""
    import torch

    import bench
    from elasticfusion_b200 import capi, synth

    K, seed = synth.K_DEFAULT, 42
    rgb, depth = bench.make_frames(K, 8, seed)
    traj = synth.trajectory(2, seed=seed)
    T = np.linalg.inv(traj[0]) @ traj[1]
    cfg = dict(FORCED) if forced else {}
    ctx = capi.Context(capi.default_config(K.width, K.height, K.fx, K.fy, K.cx, K.cy, capacity=2_000_000, close_loops=2, **cfg))
    try:
        for i in range(8):
            ctx.process_frame(rgb[i], depth[i], i)
        if forced:
            m = ctx.map_download()
            ctx.map_upload(np.concatenate([m, inactive_copy(m, ctx.cfg.time_delta)]))
        tick = ctx.get_tick()
        stream = torch.cuda.ExternalStream(ctx.stream)
        closing = mode in ("rig", "cameras")
        cams = [ctx.camera(capi.camera_config(K.width, K.height, K.fx, K.fy, K.cx, K.cy, time_delta=ctx.cfg.time_delta,
                                              conf_threshold=ctx.cfg.confidence, close_loops=closing)) for _ in range(n)]
        inputs = []
        for i in range(n):
            vrgb, vdepth, _, _ = synth.render(traj[1] @ offset(i), K, noise_seed=seed + i)
            inputs.append((torch.from_numpy(np.ascontiguousarray(vrgb)).cuda(), torch.from_numpy(np.ascontiguousarray(vdepth).view(np.int16)).cuda()))
        rp, dp = [r.data_ptr() for r, _ in inputs], [d.data_ptr() for _, d in inputs]
        members = torch.zeros(n * ctypes.sizeof(capi.EfCameraResult), dtype=torch.uint8, device="cuda")
        result = torch.zeros(ctypes.sizeof(capi.EfRigResult), dtype=torch.uint8, device="cuda")
        one = torch.zeros(ctypes.sizeof(capi.EfCameraResult), dtype=torch.uint8, device="cuda")
        torch.cuda.synchronize()
        if mode in ("rig", "open_rig"):
            rig = ctx.rig(cams, [offset(i) for i in range(n)])
            rig.frame_device(rp, dp, members.data_ptr(), result.data_ptr(), tick - 1, T_wc=T, fuse=False)

            def call():
                rig.frame_device(rp, dp, members.data_ptr(), result.data_ptr(), tick - 1)
                return closing and rig.deform_result()[0]["applied"]
        else:
            for i, c in enumerate(cams):
                c.frame_device(rp[i], dp[i], one.data_ptr(), tick - 1, T_wc=T @ offset(i), fuse=False)

            def call():
                applied = False
                for i, c in enumerate(cams):
                    c.frame_device(rp[i], dp[i], one.data_ptr(), tick - 1)
                    applied = applied or (closing and c.deform_result()[0]["applied"])
                return applied
        times = {False: [], True: []}
        for k in range(calls):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(stream)
            applied = call()
            e1.record(stream)
            e1.synchronize()
            if k >= 4:  # (the first calls: warm-up, and no graph old enough to close against yet)
                times[bool(applied)].append(e0.elapsed_time(e1))
        return {("with_closure" if a else "without_closure"): dict(median_ms=round(float(np.median(t)), 4), calls=len(t))
                for a, t in times.items() if t}
    finally:
        ctx.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=40)
    a = ap.parse_args()

    import torch

    if not torch.cuda.is_available():
        raise SystemExit("rig_loop_cost needs a CUDA device")
    print(json.dumps({"gpu": gpu_info()}), flush=True)
    for n in (2, 4):
        for case, forced, modes in (("open_loop", False, ("open_rig", "open_cameras")), ("closing_no_closure", False, ("rig", "cameras")),
                                    ("closing_forced", True, ("rig", "cameras"))):
            for mode in modes:
                print(json.dumps({"members": n, "camera": "640x480", "case": case, "mode": mode, **run_case(n, forced, mode, a.calls)}),
                      flush=True)


if __name__ == "__main__":
    main()
