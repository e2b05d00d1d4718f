"""Cost of a rig's joint SO(3) pre-alignment (EfRigConfig.joint_so3 = 1) against member 0's (joint_so3 = 0), on an H100.

Rigs of 2 and 4 cameras at 640x480 on the map a 640x480 context builds from 8 frames of the synthetic sequence, with the context's
default gn_cluster (member 0's pre-alignment is then one cluster launch; the joint one is always 1 + SO3_MAX_ITER plain launches).
Member i sits at frame 1's room pose composed with a fixed offset and sees its rendered RGB-D frame. Each round creates a rig of the
same cameras with one of the two settings, makes a has_pose call with fuse = 0 and two warm-up calls, then times `calls` tracked calls
(time = tick - 1) with fuse 0 or 1; the rounds alternate the two settings, so both see the same machine state. Each call is timed by a
CUDA event pair on ef_stream() around ef_rig_frame_device. Prints the card's name and power limit, read in the same run, then one JSON
line per (members, fuse) with the median ms per call of each setting.

    python scripts/rig_so3_cost.py [--rounds 6] [--calls 10]
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


def run_case(n, fuse, rounds, calls):
    """median ms per tracked call of a rig seeded by member 0 and of a joint rig, the rounds alternating the two"""
    import torch

    import bench
    from elasticfusion_b200 import capi, synth

    K, seed = synth.K_DEFAULT, 42
    rgb, depth = bench.make_frames(K, 8, seed)
    traj = synth.trajectory(2, seed=seed)
    T = np.linalg.inv(traj[0]) @ traj[1]
    ctx = capi.Context(capi.default_config(K.width, K.height, K.fx, K.fy, K.cx, K.cy, capacity=4_000_000))
    try:
        for i in range(8):
            ctx.process_frame(rgb[i], depth[i], i)
        tick = ctx.get_tick()
        stream = torch.cuda.ExternalStream(ctx.stream)
        cams = [ctx.camera(capi.camera_config(K.width, K.height, K.fx, K.fy, K.cx, K.cy, time_delta=ctx.cfg.time_delta,
                                              conf_threshold=ctx.cfg.confidence)) for _ in range(n)]
        inputs = []
        for i in range(n):
            vrgb, vdepth, _, _ = synth.render(traj[1] @ offset(i), K, noise_seed=seed + i)
            inputs.append((torch.from_numpy(np.ascontiguousarray(vrgb)).cuda(), torch.from_numpy(np.ascontiguousarray(vdepth).view(np.int16)).cuda()))
        rp, dp = [r.data_ptr() for r, _ in inputs], [d.data_ptr() for _, d in inputs]
        members = torch.zeros(n * ctypes.sizeof(capi.EfCameraResult), dtype=torch.uint8, device="cuda")
        result = torch.zeros(ctypes.sizeof(capi.EfRigResult), dtype=torch.uint8, device="cuda")
        torch.cuda.synchronize()
        times = {False: [], True: []}
        for r in range(2 * rounds):
            joint = r % 2 == 1
            rig = ctx.rig(cams, [offset(i) for i in range(n)], joint_so3=joint)
            rig.frame_device(rp, dp, members.data_ptr(), result.data_ptr(), tick - 1, T_wc=T, fuse=False)
            for k in range(2 + calls):
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record(stream)
                rig.frame_device(rp, dp, members.data_ptr(), result.data_ptr(), tick - 1, fuse=fuse)
                e1.record(stream)
                e1.synchronize()
                if k >= 2:
                    times[joint].append(e0.elapsed_time(e1))
            rig.close()
        return {("joint" if j else "member0"): dict(median_ms=round(float(np.median(t)), 4), calls=len(t)) for j, t in times.items()}
    finally:
        ctx.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=6)
    ap.add_argument("--calls", type=int, default=10)
    a = ap.parse_args()

    import torch

    if not torch.cuda.is_available():
        raise SystemExit("rig_so3_cost needs a CUDA device")
    print(json.dumps({"gpu": gpu_info()}), flush=True)
    for n in (2, 4):
        for fuse in (False, True):
            print(json.dumps({"members": n, "camera": "640x480", "fuse": int(fuse), **run_case(n, fuse, a.rounds, a.calls)}), flush=True)


if __name__ == "__main__":
    main()
