"""How the frame look-ahead overlaps the frame in flight, per scheduling switch, on bench.py's 640x480 sequence.

    python scripts/lookahead_overlap.py [--steps 200] [--warmup 20] [--repeats 1] [--trace DIR] [--out FILE]

Per configuration (environment switches read at ef_create), the way bench.py times `value`: seed 42, frames resident on the
device, 256 MiB L2 flush between frames, one event pair per frame on the context's stream. Per frame:
  frame      start event -> after ef_join_lookahead (bench.py's `value` is steps / sum of these)
  main       start event -> an event on the same stream before the join: the frame in flight alone
  join_wait  frame - main: time the frame waits for the next frame's input side
  nola       the same frames through plain calls without look-ahead
  side       (a second run with EF_STAGE_TIMING=1) start and end of the side stream's work, ms after frame start; each frame is
             preceded by a 1 ms device sleep so that the whole frame is enqueued before it starts, as in the untimed loop
--trace DIR also takes a torch.profiler trace with the side stream started after the cluster (default) and at frame start,
and reports, for k_gn_cluster, k_so3_cluster, k_gn_begin and k_iter1, the gap between the end of the previous kernel on the
same stream and their start.
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bench  # noqa: E402  (make_frames, workload, gpu_info; nothing runs at import)

CONFIGS = {
    "default": {},
    "at_frame_start": {"EF_LA_AFTER_TRACK": "0"},
    "at_frame_start+gn_cluster=8": {"EF_LA_AFTER_TRACK": "0", "EF_GN_CLUSTER": "8"},
    "at_frame_start+gn_cluster=0": {"EF_LA_AFTER_TRACK": "0", "EF_GN_CLUSTER": "0"},
    "gn_cluster=0": {"EF_GN_CLUSTER": "0"},
}
SWITCHES = ("EF_LA_AFTER_TRACK", "EF_GN_CLUSTER", "EF_STAGE_TIMING")


def make_ctx(capi, cfg, stream, env):
    for k in SWITCHES:
        os.environ.pop(k, None)
    os.environ.update(env)
    try:
        return capi.Context(cfg, stream=stream.cuda_stream)
    finally:
        for k in SWITCHES:
            os.environ.pop(k, None)


def run(torch, capi, cfg, stream, flush, rgb_d, depth_d, env, warmup, steps, la, instrument=False):
    """Per-frame dicts (ms) over frames warmup .. warmup+steps-1 of the sequence."""
    ctx = make_ctx(capi, cfg, stream, dict(env, EF_STAGE_TIMING="1") if instrument else env)
    ptr = lambda a, i: a[i].data_ptr()  # noqa: E731
    Ev = lambda: torch.cuda.Event(enable_timing=True)  # noqa: E731
    rows = []
    with torch.cuda.stream(stream):
        if la:
            ctx.prefetch_frame_device(ptr(rgb_d, 0), ptr(depth_d, 0))
        evs = []
        for i in range(warmup + steps):
            timed = i >= warmup
            flush.fill_(i & 0xFF)
            if instrument:
                torch.cuda._sleep(2_000_000)
            s, m, e = Ev(), Ev(), Ev()
            s.record(stream)
            if la:
                ctx.process_frame_device(None, None, i)
                ctx.prefetch_frame_device(ptr(rgb_d, i + 1), ptr(depth_d, i + 1))
                m.record(stream)
                ctx.join_lookahead()
            else:
                ctx.process_frame_device(ptr(rgb_d, i), ptr(depth_d, i), i)
                m.record(stream)
            e.record(stream)
            if instrument:
                ctx.sync()
                side = ctx.lookahead_ms() if la else None
                if timed:
                    rows.append({"frame": s.elapsed_time(e), "main": s.elapsed_time(m), "side": side})
            elif timed:
                evs.append((s, m, e))
    ctx.sync()
    for s, m, e in evs:
        rows.append({"frame": s.elapsed_time(e), "main": s.elapsed_time(m)})
    ctx.close()
    return rows


def summary(rows, nola):
    med = lambda xs: float(statistics.median(xs)) * 1000.0  # noqa: E731  (us)
    f = [r["frame"] for r in rows]
    out = {"value_fps": len(f) / (sum(f) / 1000.0), "frame_us": med(f), "main_us": med([r["main"] for r in rows]),
           "join_wait_us": med([r["frame"] - r["main"] for r in rows]),
           "frame_us_p10_p90": [float(np.percentile(f, 10)) * 1000.0, float(np.percentile(f, 90)) * 1000.0]}
    if nola:
        g = [r["frame"] for r in nola]
        out["nola_fps"] = len(g) / (sum(g) / 1000.0)
        out["nola_frame_us"] = med(g)
        out["lookahead_slows_main_us"] = out["main_us"] - out["nola_frame_us"]
    return out


def trace_gaps(torch, capi, cfg, stream, flush, rgb_d, depth_d, env, path, frames=40):
    """Median gap (us) between the end of the previous kernel on the same stream and the start of each cluster kernel."""
    from torch.profiler import ProfilerActivity, profile

    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        run(torch, capi, cfg, stream, flush, rgb_d, depth_d, env, 10, frames, True)
    prof.export_chrome_trace(path)
    ev = [e for e in json.load(open(path))["traceEvents"] if e.get("cat") == "kernel"]
    by_stream = {}
    for e in sorted(ev, key=lambda e: e["ts"]):
        by_stream.setdefault(e["args"].get("stream"), []).append(e)
    gaps = {}
    for ks in by_stream.values():
        for a, b in zip(ks, ks[1:]):
            for name in ("k_gn_cluster", "k_so3_cluster", "k_iter1", "k_gn_begin"):
                if b["name"].startswith(name) or f" {name}(" in b["name"] or b["name"].split("(")[0].endswith(name):
                    gaps.setdefault(name, []).append(max(0.0, b["ts"] - (a["ts"] + a["dur"])))
    durs = {}
    for e in ev:
        n = e["name"].split("(")[0].split(" ")[-1]
        durs.setdefault(n, []).append(e["dur"])
    return {"wait_after_predecessor_us": {k: {"median": float(np.median(v)), "p90": float(np.percentile(v, 90)), "n": len(v)}
                                          for k, v in gaps.items()},
            "kernel_us_median": {k: float(np.median(v)) for k, v in sorted(durs.items())}}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--repeats", type=int, default=1, help="rounds over all configurations, alternating them")
    ap.add_argument("--configs", default=",".join(CONFIGS))
    ap.add_argument("--trace", metavar="DIR")
    ap.add_argument("--out", metavar="FILE")
    args = ap.parse_args()
    import torch

    from elasticfusion_b200 import capi

    dev = torch.device("cuda", 0)
    K, cap, _, _ = bench.workload("640x480")
    rgb, depth = bench.make_frames(K, args.warmup + args.steps + 2, 42)
    rgb_d = torch.from_numpy(rgb).to(dev)
    depth_d = torch.from_numpy(depth.view(np.int16)).to(dev)
    flush = torch.empty(256 * 1024 * 1024, dtype=torch.uint8, device=dev)
    stream = torch.cuda.Stream(device=dev)
    cfg = capi.default_config(K.width, K.height, K.fx, K.fy, K.cx, K.cy, capacity=cap, time_delta=bench.BIG, device=0)
    res = {"gpu": bench.gpu_info(0), "steps": args.steps, "warmup": args.warmup, "configs": {}}
    names = args.configs.split(",")
    for rep in range(args.repeats):
        for name in names:
            env = CONFIGS[name]
            rows = run(torch, capi, cfg, stream, flush, rgb_d, depth_d, env, args.warmup, args.steps, True)
            nola = run(torch, capi, cfg, stream, flush, rgb_d, depth_d, env, args.warmup, args.steps, False)
            r = summary(rows, nola)
            if rep == 0:
                inst = run(torch, capi, cfg, stream, flush, rgb_d, depth_d, env, args.warmup, args.steps, True, instrument=True)
                side = [x["side"] for x in inst if x["side"]]
                r["instrumented"] = summary(inst, None)
                if side:
                    r["instrumented"]["side_start_us"] = float(np.median([s[0] for s in side])) * 1000.0
                    r["instrumented"]["side_end_us"] = float(np.median([s[1] for s in side])) * 1000.0
            res["configs"].setdefault(name, {"env": env, "runs": []})["runs"].append(r)
            print(name, json.dumps({k: v for k, v in r.items() if k != "instrumented"}), json.dumps(r.get("instrumented")), flush=True)
    if args.trace:
        os.makedirs(args.trace, exist_ok=True)
        res["trace"] = {}
        for name in ("default", "at_frame_start"):
            res["trace"][name] = trace_gaps(torch, capi, cfg, stream, flush, rgb_d, depth_d, CONFIGS[name],
                                            os.path.join(args.trace, f"trace_{name}.json"))
            print(name, json.dumps(res["trace"][name]["wait_after_predecessor_us"]), flush=True)
    print(json.dumps(res["gpu"]))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
