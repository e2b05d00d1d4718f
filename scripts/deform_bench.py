"""Device time of one local-loop-closure deformation solve (ef_deform_solve) at 200, 500 and 1023 graph nodes with 768
constraints plus their pins, on synthetic loop-closure inputs (oracle/efo_deform.synthetic_case). "kernel_ms" is the duration
of the solve kernel alone, as torch.profiler's CUDA activity trace records it; "call_ms" is the whole API call (host-side
constraint expansion, pageable uploads, the kernel, downloads) between CUDA events. Prints one JSON line, with the name and
power limit of the GPU read in the same run. The solve does not run inside ef_process_frame, so there is no per-frame cost
of a deformation-on mode to measure.

    python scripts/deform_bench.py [--reps 20]
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
    try:
        r = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30)
        name, power = [c.strip() for c in r.stdout.strip().split(",")]
        return {"name": name, "power_limit": power}
    except Exception:
        import torch

        return {"name": torch.cuda.get_device_name(0), "power_limit": None}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--constraints", type=int, default=768)
    a = ap.parse_args()

    import torch

    from elasticfusion_b200 import capi
    from oracle import efo_deform as ed

    ctx = capi.Context(capi.default_config(640, 480, 528.0, 528.0, 320.0, 240.0, capacity=10000))
    stream = torch.cuda.ExternalStream(ctx.stream)
    out = {"gpu": gpu_info(), "constraints": a.constraints, "pin": True, "solve_ms": {}}
    for n in (200, 500, 1023):
        pos, times, src, dst, st, dt = ed.synthetic_case(n, a.constraints, seed=n)
        kw = dict(node_pos=pos, node_times=times, src=src, dst=dst, src_times=st, dst_times=dt, pin=True)
        info = ctx.deform_solve(**kw)[0]  # warm-up (allocates the workspace)
        ms = []
        for _ in range(a.reps):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(stream)
            ctx.deform_solve(**kw)
            e1.record(stream)
            e1.synchronize()
            ms.append(e0.elapsed_time(e1))
        from torch.profiler import ProfilerActivity, profile

        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(a.reps):
                ctx.deform_solve(**kw)
        kern = [e.device_time for e in prof.events() if "k_deform_solve" in e.name]
        out["solve_ms"][str(n)] = {"kernel_ms": float(np.median(kern)) / 1e3 if kern else None, "kernel_launches": len(kern),
                                   "call_ms": float(np.median(ms)), "iterations": info["iterations"], "bandwidth": info["bandwidth"]}
    ctx.close()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
