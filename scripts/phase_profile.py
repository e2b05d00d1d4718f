"""Phase timestamps (%globaltimer) of the last k_iter1 / k_iter2 iteration of pyramid levels 0 and 1, median over frames.
Needs an instrumented build of the library:
   EF_OUT=build/libefusion_prof.so ./build.sh -DEF_PROFILE_PHASES ; EF_LIB=build/libefusion_prof.so python scripts/phase_profile.py [frames]"""
import sys, os, ctypes as C, numpy as np
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from elasticfusion_b200 import synth, capi

n = int(sys.argv[1]) if len(sys.argv) > 1 else 40
SKIP = 5  # first frames: module loading, map still growing from empty
K = synth.K_DEFAULT
frames = list(synth.sequence(n, K, seed=42, noise=True))
BIG = 2147483647 // 2
ctx = capi.Context(capi.default_config(K.width, K.height, K.fx, K.fy, K.cx, K.cy, capacity=1000000, time_delta=BIG))
lib = capi.lib()
cudart = C.CDLL("libcudart.so")
lib.ef_debug_gn.restype = C.c_void_p
gnp = lib.ef_debug_gn(ctx.h_ctx, 0)
sz = lib.ef_debug_gn_size()
off = lib.ef_debug_dbg_offset()
buf = (C.c_char * sz)()
stamps = []
for i, (rgb, d, _) in enumerate(frames):
    ctx.process_frame(rgb, d, i)
    if cudart.cudaDeviceSynchronize() != 0 or cudart.cudaMemcpy(buf, C.c_void_p(gnp), C.c_size_t(sz), 2) != 0:
        raise RuntimeError("reading the GN state failed")
    if i >= SKIP:
        stamps.append(np.frombuffer(buf, dtype=np.int64, count=40, offset=off).copy())
S = np.array(stamps)

# (name, first slot, last slot) of each phase; slots of level L are 20 * L + s
PHASES = [
    ("k_iter1: photometric correspondences", 0, 1),
    ("k_iter1: dense geometric rows", 1, 2),
    ("k_iter1: block reduce + partial", 2, 3),
    ("k_iter1 end -> k_iter2 start (block 0)", 3, 8),
    ("k_iter2: statistics", 8, 9),
    ("k_iter2: photometric rows + presum", 9, 10),
    ("k_iter2: block 0 done -> last ticket", 10, 11),
    ("tail: final sums", 11, 12),
    ("tail: unpack + lastA/lastb", 12, 13),
    ("tail: LDL^T solve", 13, 14),
    ("tail: Rodrigues", 14, 15),
    ("tail: pose, warp and stores", 15, 16),
]
print(f"globaltimer ns, median over {len(S)} frames (the last iteration of each level in each frame)")
print(f"{'phase':42s} {'level 0':>8s} {'level 1':>8s}")
for name, a, b in PHASES:
    print(f"{name:42s} " + " ".join(f"{np.median(S[:, 20 * L + b] - S[:, 20 * L + a]):8.0f}" for L in (0, 1)))
for name, a, b in [("k_iter2 statistics (block 0)", 8, 9), ("post-ticket tail", 11, 16), ("k_iter1 start -> tail end", 0, 16)]:
    print(f"{name:42s} " + " ".join(f"{np.median(S[:, 20 * L + b] - S[:, 20 * L + a]):8.0f}" for L in (0, 1)))
ctx.close()
