"""Generates tests/golden/ref_tracking_160x120.npz ON A GPU from the REFERENCE's own CUDA kernels
(oracle/_ref/libef_ref.so = Core/Cuda/reduce.cu + cudafuncs.cu compiled unmodified from the reference tree).

    python tests/golden/make_golden.py OUT.npz

The inputs (depth, colour, predicted model maps, pose) are stored next to the reference outputs so that
tests/test_oracle_golden.py can replay them through the CPU oracle without a GPU or the reference tree.
"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from elasticfusion_b200 import synth  # noqa: E402
from oracle import ef_oracle as eo  # noqa: E402
from oracle import ef_ref  # noqa: E402
from util import rgba_of, run_oracle  # noqa: E402


def main(out):
    K = synth.Intrinsics(160, 120, 132.0, 132.0, 80.0, 60.0)
    frames = list(synth.sequence(5, K, seed=7, noise=True, speed=2.0))
    f = run_oracle(frames, K, 3)  # produces a pose + fill-in model maps to track against
    rgb, depth, _ = frames[3]
    filt = eo.bilateral(depth, 3.0)
    T = f.pose
    vtx, nrm, img = f.buffer("fill_vertex"), f.buffer("fill_normal"), f.buffer("fill_image")
    prev_rgba, rgba = rgba_of(frames[2][0]), rgba_of(rgb)
    ref = ef_ref.RefOdometry(K)
    ref.init_first_rgb(prev_rgba)
    ref.init_icp_model(vtx, nrm, T)
    ref.init_rgb_model(img)
    ref.init_icp_depth(filt, 20.0)
    ref.init_rgb(rgba)
    g = dict(K=np.array([K.width, K.height, K.fx, K.fy, K.cx, K.cy], np.float64), T=T, filt=filt, rgba=rgba, prev_rgba=prev_rgba,
             vtx=vtx.astype(np.float16).astype(np.float32), nrm=nrm.astype(np.float16).astype(np.float32), img=img)
    # model maps are stored at half precision to keep the fixture small; regenerate the reference state from the stored values
    ref = ef_ref.RefOdometry(K)
    ref.init_first_rgb(prev_rgba)
    ref.init_icp_model(g["vtx"], g["nrm"], T)
    ref.init_rgb_model(img)
    ref.init_icp_depth(filt, 20.0)
    ref.init_rgb(rgba)
    for lv in range(3):
        for name in ("depth_tmp", "lastImage", "nextImage", "lastNextImage"):
            g[f"{name}{lv}"] = ref.buffer(name, lv)
        for name in ("vmap_curr", "nmap_curr", "vmap_g_prev", "nmap_g_prev", "lastDepth", "nextDepth"):
            a = ref.buffer(name, lv)
            g[f"{name}{lv}_nan"] = np.packbits(np.isnan(a))
            g[f"{name}{lv}_sum"] = np.array([np.nansum(a.astype(np.float64)), np.nansum(np.abs(a.astype(np.float64)))])
    R = T[:3, :3].astype(np.float32)
    t = T[:3, 3].astype(np.float32)
    dR = np.array([[1, -0.002, 0.001], [0.002, 1, -0.003], [-0.001, 0.003, 1]], np.float32)
    Rc, tc, Rpi = (R @ dR).astype(np.float32), t + np.array([0.004, -0.003, 0.005], np.float32), np.linalg.inv(R).astype(np.float32)
    g.update(Rc=Rc, tc=tc, Rpi=Rpi, tp=t)
    for lv in range(3):
        A, b, r = ref.icp_step(lv, Rc, tc, Rpi, t)
        g[f"icp_A{lv}"], g[f"icp_b{lv}"], g[f"icp_r{lv}"] = A, b, r
        d = np.float32(1 << lv)
        fx, fy, cx, cy = np.float32(K.fx) / d, np.float32(K.fy) / d, np.float32(K.cx) / d, np.float32(K.cy) / d
        Km = np.array([[fx, 0, cx], [0, fy, cy], [0, 0, 1]], np.float64)
        ang = 0.003
        Rz = np.array([[np.cos(ang), -np.sin(ang), 0], [np.sin(ang), np.cos(ang), 0], [0, 0, 1]])
        krk = (Km @ Rz @ np.linalg.inv(Km)).astype(np.float32)
        kt = (Km @ np.array([0.004, -0.002, 0.003])).astype(np.float32)
        sig, cnt = ref.rgb_residual(lv, krk, kt)
        Ar, br = ref.rgb_step(lv, float(np.sqrt(np.float32(cnt))))
        g[f"krk{lv}"], g[f"kt{lv}"], g[f"res{lv}"] = krk, kt, np.array([sig, cnt])
        g[f"rgb_A{lv}"], g[f"rgb_b{lv}"] = Ar, br
        g[f"dIdx{lv}"], g[f"dIdy{lv}"] = ref.buffer("dIdx", lv), ref.buffer("dIdy", lv)
    d = np.float32(4)
    Km = np.array([[np.float32(K.fx) / d, 0, np.float32(K.cx) / d], [0, np.float32(K.fy) / d, np.float32(K.cy) / d], [0, 0, 1]], np.float64)
    a = 0.004
    Rx = np.array([[1, 0, 0], [0, np.cos(a), -np.sin(a)], [0, np.sin(a), np.cos(a)]])
    H, kinv, krlr = (Km @ Rx @ np.linalg.inv(Km)).astype(np.float32), np.linalg.inv(Km).astype(np.float32), (Km @ Rx).astype(np.float32)
    As, bs, rs = ref.so3_step(H, kinv, krlr)
    g.update(so3_H=H, so3_kinv=kinv, so3_krlr=krlr, so3_A=As, so3_b=bs, so3_r=rs)
    Tr, tr = ref.track(T)
    g["track_T"] = Tr
    g["track_trace"] = tr.view(np.uint8)
    np.savez_compressed(out, **g)
    print("wrote", out, os.path.getsize(out), "bytes;", len(tr), "trace records")


if __name__ == "__main__":
    main(sys.argv[1] if len(sys.argv) > 1 else os.path.join(ROOT, "tests", "golden", "ref_tracking_160x120.npz"))
