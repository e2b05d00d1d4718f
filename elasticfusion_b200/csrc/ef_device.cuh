// Device-side helpers shared by the tracking / mapping kernels.
//
// All translation units are compiled with --fmad=false: every +,-,*,/ and sqrtf below is a single IEEE-754
// operation in the written order, so per-pixel results are bit-reproducible against a plain C restatement of the
// same formulas (the parity tests rely on this; the kernels are HBM/latency bound, not FMA bound).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace ef {

struct f3 {
  float x, y, z;
};
struct m33 {
  f3 r[3];
};

__host__ __device__ __forceinline__ f3 mk3(float x, float y, float z) {
  f3 v;
  v.x = x;
  v.y = y;
  v.z = z;
  return v;
}
__host__ __device__ __forceinline__ f3 operator-(const f3& a, const f3& b) { return mk3(a.x - b.x, a.y - b.y, a.z - b.z); }
__host__ __device__ __forceinline__ f3 operator+(const f3& a, const f3& b) { return mk3(a.x + b.x, a.y + b.y, a.z + b.z); }
__host__ __device__ __forceinline__ f3 operator*(const f3& a, float s) { return mk3(a.x * s, a.y * s, a.z * s); }
__host__ __device__ __forceinline__ f3 cross(const f3& a, const f3& b) {
  return mk3(a.y * b.z - a.z * b.y, a.z * b.x - a.x * b.z, a.x * b.y - a.y * b.x);
}
__host__ __device__ __forceinline__ float dot(const f3& a, const f3& b) { return a.x * b.x + a.y * b.y + a.z * b.z; }
__device__ __forceinline__ float norm(const f3& a) { return sqrtf(dot(a, a)); }
// IEEE 1/sqrt (the reference's rsqrtf is the 2-ulp MUFU approximation)
__device__ __forceinline__ f3 normalized(const f3& a) {
  const float rn = 1.0f / sqrtf(dot(a, a));
  return mk3(a.x * rn, a.y * rn, a.z * rn);
}
__host__ __device__ __forceinline__ f3 mul(const m33& m, const f3& a) { return mk3(dot(m.r[0], a), dot(m.r[1], a), dot(m.r[2], a)); }
__host__ __device__ __forceinline__ m33 load_m33(const float* R) {
  m33 m;
  m.r[0] = mk3(R[0], R[1], R[2]);
  m.r[1] = mk3(R[3], R[4], R[5]);
  m.r[2] = mk3(R[6], R[7], R[8]);
  return m;
}

__device__ __forceinline__ float qnan() { return __int_as_float(0x7fffffff); }
__device__ __forceinline__ float gmin(float x, float y) { return (y < x) ? y : x; }  // GLSL min
__device__ __forceinline__ float gmax(float x, float y) { return (x < y) ? y : x; }  // GLSL max

// 4x4 row-major float pose applied to a point / a direction, accumulation order ((m0*x + m1*y) + m2*z) + m3
// (M: any pointer to float, e.g. a volatile one into shared memory that the compiler must not hold in registers)
template <typename M>
__device__ __forceinline__ f3 xform(M m, const f3& v) {
  return mk3(((m[0] * v.x + m[1] * v.y) + m[2] * v.z) + m[3], ((m[4] * v.x + m[5] * v.y) + m[6] * v.z) + m[7],
             ((m[8] * v.x + m[9] * v.y) + m[10] * v.z) + m[11]);
}
template <typename M>
__device__ __forceinline__ f3 rot(M m, const f3& v) {
  return mk3((m[0] * v.x + m[1] * v.y) + m[2] * v.z, (m[4] * v.x + m[5] * v.y) + m[6] * v.z,
             (m[8] * v.x + m[9] * v.y) + m[10] * v.z);
}

// Warp sum of up to 32 per-lane values by recursive halving ("transpose-reduce"): at each of the 5 stages a lane keeps
// half of its values and trades the other half with its partner, so 32 values cost 31 shuffles + 31 adds instead of
// 32 x 5 for independent shuffle trees. On return lane l holds the warp total of value l in v[0].
template <int N>
__device__ __forceinline__ float warp_reduce_transpose(const float (&in)[N]) {
  static_assert(N <= 32, "at most 32 values");
  const int lane = threadIdx.x & 31;
  float v[32];
#pragma unroll
  for (int k = 0; k < 32; ++k) v[k] = (k < N) ? in[k] : 0.f;
#pragma unroll
  for (int half = 16; half >= 1; half >>= 1) {
    const bool upper = (lane & half) != 0;
#pragma unroll
    for (int k = 0; k < half; ++k) {
      const float send = upper ? v[k] : v[k + half];
      const float keep = upper ? v[k + half] : v[k];
      v[k] = keep + __shfl_xor_sync(0xffffffffu, send, half);
    }
  }
  return v[0];
}

// block sum of N (<= 32) floats held per thread; on return threads 0..N-1 hold the CTA total of value threadIdx.x in v[0]
// (fixed summation order: butterfly inside a warp, then warps in index order).
template <int N, int THREADS>
__device__ __forceinline__ void block_reduce_sum(float (&v)[N], float* smem /* 32 * (THREADS/32) floats */) {
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  const float mine = warp_reduce_transpose<N>(v);
  smem[wid * 32 + lane] = mine;
  __syncthreads();
  if (wid == 0) {
    float t = 0.f;
#pragma unroll
    for (int w = 0; w < THREADS / 32; ++w) t += smem[w * 32 + lane];
    v[0] = t;
  }
}

// Programmatic dependent launch: every kernel of the library starts with this. launch_dependents lets the NEXT kernel
// in the stream be scheduled (its CTAs become resident and park at their own wait) while this grid is still running;
// wait blocks until the PREVIOUS grid has completed and its memory is visible. Because every kernel waits before it
// touches memory, stream order is preserved transitively -- only the launch latency of dependent kernels is hidden.
__device__ __forceinline__ void pdl_enter() {
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
  asm volatile("griddepcontrol.wait;" ::: "memory");
}

// The two halves separately, for the few kernels that do pose-independent work (loads of data no kernel in flight can be
// writing) between them: pdl_launch() first, that work, then pdl_wait() before anything the predecessor may have written.
__device__ __forceinline__ void pdl_launch() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }

// "last block done" ticket: returns true in every thread of the block that arrives last.
__device__ __forceinline__ bool last_block_done(unsigned int* counter) {
  __shared__ bool is_last;
  __syncthreads();
  if (threadIdx.x == 0) {
    // one gpu-scope fence by the thread that takes the ticket: it is cumulative over the CTA's writes ordered before it by
    // the barrier above (release), and again before the CTA reads the other CTAs' results (acquire)
    __threadfence();
    unsigned int t = atomicAdd(counter, 1u);
    is_last = (t == gridDim.x - 1);
    if (is_last) __threadfence();
  }
  __syncthreads();
  return is_last;
}

// Order-preserving compaction in one pass (k_scan_flags, k_clean_move, k_fuse_update, k_sobel_cand): a persistent grid draws tiles
// in order from a dispenser, scans each tile inside the CTA (block_exclusive_scan) and takes the tile's prefix from its predecessors.
//
// Decoupled look-back of one tile, run by one whole warp. Tile states carry the launch's epoch
// in their upper bits ([63:34] epoch, [33:32] status, [31:0] value), so states left by earlier scans read as "not published"
// and nothing has to be cleared between scans. The scan starts at tile `first` with prefix `base`; tiles below `first` are
// never read. Publishes the aggregate, then looks back for the exclusive prefix 32 predecessors at a time (status 1 =
// aggregate only, 2 = inclusive prefix; status and value share one 64-bit word, so no fence is needed), publishes the
// inclusive prefix and returns the exclusive one.
__device__ __forceinline__ int lookback_prefix(unsigned long long* state, int tile, int first, int base, int aggregate, unsigned int epoch) {
  const int lane = threadIdx.x & 31;
  const unsigned long long tag = (unsigned long long)epoch << 34;
  volatile unsigned long long* vstate = state;
  if (tile == first) {
    if (lane == 0) vstate[tile] = tag | (2ull << 32) | (unsigned int)(base + aggregate);
    return base;
  }
  int prefix = 0;
  if (lane == 0) vstate[tile] = tag | (1ull << 32) | (unsigned int)aggregate;
  int look = tile - 1;
  while (true) {
    const int idx = look - lane;
    const unsigned long long w = (idx >= first) ? vstate[idx] : (tag | (2ull << 32));
    const unsigned int st = ((w >> 34) == (unsigned long long)epoch) ? ((unsigned int)(w >> 32) & 3u) : 0u;
    if (__any_sync(0xffffffffu, st == 0)) continue;  // a predecessor has not published yet: re-read
    const unsigned int m2 = __ballot_sync(0xffffffffu, st == 2);
    const int first2 = m2 ? (__ffs(m2) - 1) : 32;
    int val = (lane <= first2) ? (int)(unsigned int)(w & 0xffffffffull) : 0;
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) val += __shfl_xor_sync(0xffffffffu, val, off);
    prefix += val;
    if (m2) break;
    look -= 32;
  }
  if (lane == 0) vstate[tile] = tag | (2ull << 32) | (unsigned int)(prefix + aggregate);
  return prefix;
}

// Exit of a persistent grid that draws tiles from the dispenser counter[0], called by one thread per CTA once the CTA is
// done: it takes an exit ticket from counter[1], and the last CTA to do so re-arms both counters for the next launch and
// gets true. FENCED: gpu-scope fences order the CTA's writes before its ticket (release) and the other CTAs' writes before
// what the last CTA does next (acquire), for a last CTA that reads what the others wrote (k_clean_move's count).
template <bool FENCED>
__device__ __forceinline__ bool dispenser_exit(unsigned int* counter) {
  if (FENCED) __threadfence();
  if (atomicAdd(counter + 1, 1u) != gridDim.x - 1) return false;
  if (FENCED) __threadfence();
  counter[0] = 0u;
  counter[1] = 0u;
  return true;
}

// Exclusive scan of one int per thread over a CTA of THREADS threads (a multiple of 32, at most 1024); also returns the CTA
// total in `aggregate`. Every thread of the CTA must call it; s_warp holds THREADS / 32 ints and may be reused after the next barrier.
template <int THREADS>
__device__ __forceinline__ int block_exclusive_scan(int v, int* s_warp, int& aggregate) {
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  int incl = v;
#pragma unroll
  for (int off = 1; off < 32; off <<= 1) {
    const int t = __shfl_up_sync(0xffffffffu, incl, off);
    if (lane >= off) incl += t;
  }
  if (lane == 31) s_warp[wid] = incl;
  __syncthreads();
  if (wid == 0) {
    int w = (lane < THREADS / 32) ? s_warp[lane] : 0;
#pragma unroll
    for (int off = 1; off < 32; off <<= 1) {
      const int t = __shfl_up_sync(0xffffffffu, w, off);
      if (lane >= off) w += t;
    }
    if (lane < THREADS / 32) s_warp[lane] = w;  // inclusive over warps
  }
  __syncthreads();
  aggregate = s_warp[THREADS / 32 - 1];
  return (wid ? s_warp[wid - 1] : 0) + incl - v;
}

}  // namespace ef
