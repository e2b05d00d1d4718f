"""Writes tests/golden/ref_deform.npz: inputs and outputs of the reference's own deformation solver (Core/Utils/
DeformationGraph.cpp + CholeskyDecomp.cpp, compiled unmodified into oracle/_ref/libef_refdef.so by oracle/refdef/Makefile,
driven through Deformation::constrain's local-closure logic).

Cases:
- the synthetic graphs of tests/test_gpu_deform.py (pinned / unpinned, three iterations, a lastDeformTime that holds a prefix
  fixed and one that holds every node fixed, the 5-node minimum, 1023 nodes with 768 constraints plus pins);
- accepted local loop closures of the CPU oracle pipeline on the 320x240, timeDelta 12 loop sequence of
  test_local_loop_front_half_over_a_sequence: the graph is every 5000th surfel of the map after the previous frame (position,
  colorTime.z; sampleGraphModel, Core/Deformation.cpp:232-306), the constraints are the front half's. The first closure is
  pinned with lastDeformTime 0; a later one is unpinned with lastDeformTime = the first one's tick (what the reference does
  after deforming once). The oracle run itself stays open-loop, so later maps are not the deformed ones.

    python tests/golden/make_deform_golden.py      (needs oracle/_ref/libef_refdef.so and libef_oracle.so)
"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

from oracle import efo_deform as ed  # noqa: E402

SYNTHETIC = [  # (name, n_nodes, n_constraints, pin, last_deform_time, shift, seed)
    ("pinned_200", 200, 150, True, 0, 0.03, 211),
    ("unpinned_200", 200, 150, False, 0, 0.03, 211),
    ("pinned_three_iterations", 150, 120, True, 0, 1.0, 161),
    ("prefix_fixed", 300, 200, False, "half", 0.03, 311),
    ("all_fixed", 120, 80, True, "all", 0.03, 131),
    ("five_nodes", 5, 4, True, 0, 0.03, 16),
    ("max_graph", 1023, 768, True, 0, 0.03, 1034),
]


def synthetic_cases():
    for name, n, m, pin, ldt, shift, seed in SYNTHETIC:
        pos, times, src, dst, st, dt = ed.synthetic_case(n, m, seed=seed, shift=shift)
        if ldt == "half":
            ldt = int(times[n // 2])
        elif ldt == "all":
            ldt = int(times[-1])
        yield name, dict(node_pos=pos, node_times=times, src=src, dst=dst, src_times=st, dst_times=dt, pin=pin, last_deform_time=ldt)


def pipeline_cases(max_cases=2):
    from elasticfusion_b200 import synth
    from oracle import ef_oracle as eo

    K2 = synth.Intrinsics(320, 240, 264.0, 264.0, 160.0, 120.0)
    frames = list(synth.sequence(130, K2, seed=21, noise=True, speed=2.5))
    f = eo.Fusion(K2, time_delta=12, capacity=400000)
    f.set_loop_closure(True, count_thresh=3000, err_thresh=5e-5, cov_thresh=1e-4)
    first_tick = None
    out = []
    prev_map = None
    for i, (rgb, depth, _) in enumerate(frames):
        f.process_frame(rgb, depth, i)
        info, src, dst, tm = f.loop_result()
        if info["accepted"] and prev_map is not None and len(src) > 0:
            sample = prev_map[::5000]
            times = sample[:, 6].astype(np.int64)
            if len(sample) > 4 and np.all(np.diff(times) >= 0):
                pin = first_tick is None
                ldt = 0 if pin else first_tick
                if pin or i >= first_tick + 20:
                    out.append((f"pipeline_frame{i}", dict(node_pos=sample[:, :3].astype(np.float64), node_times=times.astype(np.int32),
                                                           src=src, dst=dst, src_times=np.full(len(src), i, np.int32),
                                                           dst_times=tm.astype(np.int32), pin=pin, last_deform_time=ldt)))
                    if pin:
                        first_tick = i
                    if len(out) == max_cases:
                        break
        prev_map = f.map()
    return out


def main():
    assert ed.ref_available(), "build oracle/_ref/libef_refdef.so first (make -C oracle/refdef)"
    arrays = {}
    names = []
    for name, args in list(synthetic_cases()) + pipeline_cases():
        info, nodes, cn, cw, R, t = ed.ref_solve(**args)
        names.append(name)
        for k, v in args.items():
            arrays[f"{name}/in/{k}"] = np.asarray(v)
        arrays[f"{name}/nodes16"] = nodes
        arrays[f"{name}/R"] = R
        arrays[f"{name}/t"] = t
        arrays[f"{name}/cons_nodes"] = cn
        arrays[f"{name}/cons_weights"] = cw
        arrays[f"{name}/error"] = np.float32(info["error"])
        arrays[f"{name}/meanConsErr"] = np.float32(info["meanConsErr"])
        arrays[f"{name}/iterations"] = np.int32(info["iterations"])
        print(f"{name}: nodes {len(nodes)} constraints {len(cn)} iterations {info['iterations']} error {info['error']:.6g} "
              f"meanConsErr {info['meanConsErr']:.6g}")
    arrays["cases"] = np.array(names)
    path = os.path.join(os.path.dirname(os.path.abspath(__file__)), "ref_deform.npz")
    np.savez_compressed(path, **arrays)
    print(f"wrote {path} ({os.path.getsize(path)} bytes)")


if __name__ == "__main__":
    main()
