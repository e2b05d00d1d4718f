// Latency floor of a k_iter1-shaped launch on this GPU: a chain of programmatic-dependent launches of a 600 x 128 grid whose
// threads perform D dependent rounds of memory reads (D = 0: launch / drain only; 1: one round trip; 2, 3: the state -> live maps
// -> gather chain), warm (L2 resident) and cold (a 512 MB working set rotated so every round misses L2), followed by the block
// reduction + partial store k_iter1 ends with. Prints microseconds per launch (CUDA events around 200 chained launches).
//   nvcc -O3 -gencode arch=compute_90a,code=sm_90a -o build/latency_floor scripts/latency_floor.cu
#include <cuda_runtime.h>
#include <stdio.h>
#include <stdlib.h>

__global__ void __launch_bounds__(128, 5) k_chain(const float4* __restrict__ buf, size_t n4, int depth, unsigned salt, float* out) {
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
  asm volatile("griddepcontrol.wait;" ::: "memory");
  size_t i = ((size_t)blockIdx.x * blockDim.x + threadIdx.x + (size_t)salt * 76800u) % n4;
  float acc = 0.f;
  for (int d = 0; d < depth; ++d) {
    const float4 v = buf[i];
    acc += v.x + v.y + v.z + v.w;
    i = (i * 2654435761u + (size_t)__float_as_uint(v.x) % 7u + 12345u) % n4;  // the next address depends on the loaded value
  }
  __shared__ float s[128];
  s[threadIdx.x] = acc;
  __syncthreads();
  if (threadIdx.x < 32) {
    float t = s[threadIdx.x] + s[threadIdx.x + 32] + s[threadIdx.x + 64] + s[threadIdx.x + 96];
    for (int o = 16; o > 0; o >>= 1) t += __shfl_xor_sync(0xffffffffu, t, o);
    if (threadIdx.x == 0) out[blockIdx.x] = t;
  }
}

static float run(cudaStream_t st, const float4* buf, size_t n4, int depth, bool pdl, bool rotate, float* out, int reps) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3(600);
  cfg.blockDim = dim3(128);
  cfg.stream = st;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = pdl ? 1 : 0;
  cudaEvent_t a, b;
  cudaEventCreate(&a);
  cudaEventCreate(&b);
  for (int w = 0; w < 20; ++w) cudaLaunchKernelEx(&cfg, k_chain, buf, n4, depth, (unsigned)(rotate ? w : 0), out);
  cudaEventRecord(a, st);
  for (int r = 0; r < reps; ++r) cudaLaunchKernelEx(&cfg, k_chain, buf, n4, depth, (unsigned)(rotate ? r + 20 : 0), out);
  cudaEventRecord(b, st);
  cudaEventSynchronize(b);
  float ms = 0;
  cudaEventElapsedTime(&ms, a, b);
  return ms * 1000.f / reps;
}

int main() {
  cudaStream_t st;
  cudaStreamCreateWithFlags(&st, cudaStreamNonBlocking);
  const size_t big = (size_t)512 << 20, small = (size_t)8 << 20;
  float4* buf;
  float* out;
  cudaMalloc(&buf, big);
  cudaMalloc(&out, 4096 * 4);
  cudaMemset(buf, 0, big);
  printf("us per launch of a 600 x 128 grid (chained on one stream)\n");
  printf("%-34s %8s %8s\n", "", "PDL", "plain");
  for (int depth = 0; depth <= 3; ++depth) {
    printf("depth %d, L2-warm (8 MB set)       %8.2f %8.2f\n", depth, run(st, buf, small / 16, depth, true, false, out, 200), run(st, buf, small / 16, depth, false, false, out, 200));
    printf("depth %d, L2-cold (512 MB rotated) %8.2f %8.2f\n", depth, run(st, buf, big / 16, depth, true, true, out, 200), run(st, buf, big / 16, depth, false, true, out, 200));
  }
  return 0;
}
