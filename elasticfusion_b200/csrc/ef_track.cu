// Tracking half of the hot path: pyramid construction and the coarse-to-fine geometric + photometric
// Gauss-Newton loop, as hand-written sm_90a kernels.
//
// Behavioural specification = the reference's Core/Cuda/{cudafuncs,reduce}.cu and Core/Utils/RGBDOdometry.cpp
// (cited per kernel). Structure is GPU-first rather than a translation:
//   * every reduction is ONE launch: per-CTA warp-shuffle tree -> per-CTA partial in HBM/L2 -> the CTA that takes
//     the last ticket sums the partials in double and finishes the job (the reference uses 64 CTAs + a second
//     1-CTA kernel + cudaDeviceSynchronize + a blocking D2H per step, reduce.cu:378-386);
//   * the 6x6 / 3x3 solves, the SE(3) update and the next iteration's warp matrices are computed by that last
//     CTA, so the whole SO(3) + 19-iteration SE(3) schedule is a stream of launches with no host round trip;
//   * geometric and photometric systems of one iteration are reduced by the same launch;
//   * grids are sized from the SM count (132 on H100), not the reference's fixed 64 CTAs (types.cuh:64-65);
//   * the back-projected point cloud is recomputed in the photometric step instead of being stored.
#include <float.h>
#include <stddef.h>
#include <stdio.h>
#include <string.h>

#include <new>
#include <utility>

#include "ef_device.cuh"
#include "ef_dmath.cuh"
#include "ef_internal.h"

using namespace ef;

// =============================================================================================
// pyramid / image kernels
// =============================================================================================

// reference pyrDownGaussKernel, cudafuncs.cu:75-121 (sigma_color 30, centre-relative gate, truncating store).
// `fetch(y, x)` abstracts the source so that level 2 can be produced in the same launch as level 1 by recomputing the
// level-1 values it needs from level 0 (identical arithmetic -> identical values, one launch instead of two).
template <typename Fetch>
__device__ __forceinline__ uint16_t pyr_down_u16_at(Fetch fetch, int srows, int scols, int x, int y) {
  const int D = 5;
  const float sigma_color = 30.f;
  const float weights[3] = {0.375f, 0.25f, 0.0625f};
  const int center = fetch(2 * y, 2 * x);
  const int x_mi = max(0, 2 * x - D / 2) - 2 * x;
  const int y_mi = max(0, 2 * y - D / 2) - 2 * y;
  const int x_ma = min(scols, 2 * x - D / 2 + D) - 2 * x;
  const int y_ma = min(srows, 2 * y - D / 2 + D) - 2 * y;
  float sum = 0, wall = 0;
  // fixed 5x5 trip count with predication (same accumulation order): all taps are requested at once
#pragma unroll
  for (int yi = -2; yi <= 2; ++yi)
#pragma unroll
    for (int xi = -2; xi <= 2; ++xi) {
      const bool in = (yi >= y_mi) && (yi < y_ma) && (xi >= x_mi) && (xi < x_ma);
      const int val = in ? fetch(2 * y + yi, 2 * x + xi) : 0;
      if (in && (float)abs(val - center) < 3 * sigma_color) {
        sum += val * weights[abs(xi)] * weights[abs(yi)];
        wall += weights[abs(xi)] * weights[abs(yi)];
      }
    }
  return (uint16_t)__float2int_rz(sum / wall);
}

__global__ void k_pyr_down_u16(const uint16_t* __restrict__ src, int srows, int scols, uint16_t* __restrict__ dst) {
  pdl_enter();
  const int r1 = srows / 2, c1 = scols / 2;
  auto f0 = [&](int yy, int xx) { return (int)src[(size_t)yy * scols + xx]; };
  for (int t = blockIdx.x * blockDim.x + threadIdx.x; t < r1 * c1; t += gridDim.x * blockDim.x) {
    const int y = t / c1, x = t - y * c1;
    dst[t] = pyr_down_u16_at(f0, srows, scols, x, y);
  }
}

// createVMap + createNMap fused (cudafuncs.cu:123-219): the normal is built from the three depths it needs with the
// same arithmetic createVMap would have used, so vmap never has to be re-read. Invalid -> NaN (x flags validity).
__device__ __forceinline__ bool vertex_from_depth(const uint16_t* depth, int cols, int u, int v, float fx_inv, float fy_inv,
                                                  float cx, float cy, float cutoff, f3& out) {
  const float z = depth[v * cols + u] / 1000.f;
  if (z != 0 && z < cutoff) {
    out = mk3(z * (u - cx) * fx_inv, z * (v - cy) * fy_inv, z);
    return true;
  }
  return false;
}

struct VmapArgs {
  const uint16_t* depth[NUM_PYRS];
  float* vmap[NUM_PYRS];
  float* nmap[NUM_PYRS];
  int rows[NUM_PYRS], cols[NUM_PYRS], start[NUM_PYRS + 1];
  float fx_inv[NUM_PYRS], fy_inv[NUM_PYRS], cx[NUM_PYRS], cy[NUM_PYRS];
};
__device__ __forceinline__ void vmap_nmap_at(const uint16_t* __restrict__ depth, int rows, int cols, float fx_inv, float fy_inv, float cx,
                                             float cy, float cutoff, float* __restrict__ vmap, float* __restrict__ nmap, int u, int v) {
  const size_t plane = (size_t)rows * cols;
  const size_t p = (size_t)v * cols + u;
  f3 v00;
  const bool ok00 = vertex_from_depth(depth, cols, u, v, fx_inv, fy_inv, cx, cy, cutoff, v00);
  if (ok00) {
    vmap[p] = v00.x;
    vmap[p + plane] = v00.y;
    vmap[p + 2 * plane] = v00.z;
  } else {
    vmap[p] = qnan();
    vmap[p + plane] = qnan();
    vmap[p + 2 * plane] = qnan();
  }
  f3 n = mk3(qnan(), qnan(), qnan());
  if (ok00 && u != cols - 1 && v != rows - 1) {
    f3 v01, v10;
    if (vertex_from_depth(depth, cols, u + 1, v, fx_inv, fy_inv, cx, cy, cutoff, v01) &&
        vertex_from_depth(depth, cols, u, v + 1, fx_inv, fy_inv, cx, cy, cutoff, v10))
      n = normalized(cross(v01 - v00, v10 - v00));
  }
  nmap[p] = n.x;
  nmap[p + plane] = n.y;
  nmap[p + 2 * plane] = n.z;
}
__global__ void k_vmap_nmap(VmapArgs a, float cutoff) {
  pdl_enter();
  const int total = a.start[NUM_PYRS];
  for (int f = blockIdx.x * blockDim.x + threadIdx.x; f < total; f += gridDim.x * blockDim.x) {
    const int lv = (f >= a.start[2]) ? 2 : (f >= a.start[1] ? 1 : 0);
    const int p = f - a.start[lv];
    const int v = p / a.cols[lv], u = p - v * a.cols[lv];
    vmap_nmap_at(a.depth[lv], a.rows[lv], a.cols[lv], a.fx_inv[lv], a.fy_inv[lv], a.cx[lv], a.cy[lv], cutoff, a.vmap[lv], a.nmap[lv], u, v);
  }
}

// copyMaps (cudafuncs.cu:295-381): predicted float4 vertex/normal maps -> vmaps_tmp (AoS copy) + SoA planes; z==0 -> NaN
__global__ void k_copy_maps(const float4* __restrict__ vtx, const float4* __restrict__ nrm, int rows, int cols, float4* __restrict__ vmaps_tmp,
                            float* __restrict__ vmap, float* __restrict__ nmap) {
  pdl_enter();
  const size_t n = (size_t)rows * cols;
  for (size_t p = (size_t)blockIdx.x * blockDim.x + threadIdx.x; p < n; p += (size_t)gridDim.x * blockDim.x) {
    const float4 vs = vtx[p];
    const float4 ns = nrm[p];
    if (vmaps_tmp) vmaps_tmp[p] = vs;
    f3 vd = mk3(qnan(), qnan(), qnan()), nd = vd;
    if (!(vs.z == 0)) {
      vd = mk3(vs.x, vs.y, vs.z);
      nd = mk3(ns.x, ns.y, ns.z);
    }
    vmap[p] = vd.x;
    vmap[p + n] = vd.y;
    vmap[p + 2 * n] = vd.z;
    nmap[p] = nd.x;
    nmap[p + n] = nd.y;
    nmap[p + 2 * n] = nd.z;
  }
}

// resizeVMap + resizeNMap (cudafuncs.cu:413-490) in one launch: 2x2 box average, any NaN -> NaN, normals renormalised
__global__ void k_resize_maps(const float* __restrict__ vin, const float* __restrict__ nin, int srows, int scols,
                              float* __restrict__ vout, float* __restrict__ nout) {
  pdl_enter();
  const int drows = srows / 2, dcols = scols / 2;
  const int x = blockIdx.x * blockDim.x + threadIdx.x;
  const int y = blockIdx.y * blockDim.y + threadIdx.y;
  if (x >= dcols || y >= drows) return;
  const size_t splane = (size_t)srows * scols, dplane = (size_t)drows * dcols;
  const size_t q = (size_t)y * dcols + x;
  const int xs = x * 2, ys = y * 2;
#pragma unroll
  for (int which = 0; which < 2; ++which) {
    const float* in = which ? nin : vin;
    float* out = which ? nout : vout;
    const float x00 = in[(size_t)(ys + 0) * scols + xs + 0], x01 = in[(size_t)(ys + 0) * scols + xs + 1];
    const float x10 = in[(size_t)(ys + 1) * scols + xs + 0], x11 = in[(size_t)(ys + 1) * scols + xs + 1];
    if (isnan(x00) || isnan(x01) || isnan(x10) || isnan(x11)) {
      out[q] = qnan();
      out[q + dplane] = qnan();
      out[q + 2 * dplane] = qnan();
      continue;
    }
    f3 n;
    n.x = (x00 + x01 + x10 + x11) / 4;
    const float* iy = in + splane;
    n.y = (iy[(size_t)(ys + 0) * scols + xs + 0] + iy[(size_t)(ys + 0) * scols + xs + 1] + iy[(size_t)(ys + 1) * scols + xs + 0] +
           iy[(size_t)(ys + 1) * scols + xs + 1]) / 4;
    const float* iz = in + 2 * splane;
    n.z = (iz[(size_t)(ys + 0) * scols + xs + 0] + iz[(size_t)(ys + 0) * scols + xs + 1] + iz[(size_t)(ys + 1) * scols + xs + 0] +
           iz[(size_t)(ys + 1) * scols + xs + 1]) / 4;
    if (which) n = normalized(n);
    out[q] = n.x;
    out[q + dplane] = n.y;
    out[q + 2 * dplane] = n.z;
  }
}

// tranformMaps (cudafuncs.cu:221-293), all three levels in one launch (blockIdx.y = level), pose from gn->T_wc. The
// reference transforms in place; here the camera-frame maps are kept (the ICP kernel reads those) and the world-frame
// copy is only produced for the stage API / inspection.
struct XformArgs {
  const float* sv[NUM_PYRS];
  const float* sn[NUM_PYRS];
  float* v[NUM_PYRS];
  float* n[NUM_PYRS];
  int rows[NUM_PYRS], cols[NUM_PYRS];
};
__global__ void k_transform_maps(XformArgs a, const GNState* __restrict__ gn) {
  pdl_enter();
  const int lv = blockIdx.y;
  const size_t np = (size_t)a.rows[lv] * a.cols[lv];
  float R[9], t[3];
#pragma unroll
  for (int r = 0; r < 3; ++r) {
#pragma unroll
    for (int c = 0; c < 3; ++c) R[r * 3 + c] = (float)gn->T_wc[r * 4 + c];
    t[r] = (float)gn->T_wc[r * 4 + 3];
  }
  const m33 Rm = load_m33(R);
  const f3 tv = mk3(t[0], t[1], t[2]);
  const float* __restrict__ sv = a.sv[lv];
  const float* __restrict__ sn = a.sn[lv];
  float* __restrict__ vm = a.v[lv];
  float* __restrict__ nm = a.n[lv];
  for (size_t p = (size_t)blockIdx.x * blockDim.x + threadIdx.x; p < np; p += (size_t)gridDim.x * blockDim.x) {
    f3 v = mk3(sv[p], sv[p + np], sv[p + 2 * np]);
    if (!isnan(v.x)) v = mul(Rm, v) + tv;
    vm[p] = v.x;
    vm[p + np] = v.y;
    vm[p + 2 * np] = v.z;
    f3 n = mk3(sn[p], sn[p + np], sn[p + 2 * np]);
    if (!isnan(n.x)) n = mul(Rm, n);
    nm[p] = n.x;
    nm[p + np] = n.y;
    nm[p + 2 * np] = n.z;
  }
}

// verticesToDepth + imageBGRToIntensity fused (cudafuncs.cu:564-610): level-0 depth from vmaps_tmp.z (cutoff 6 m),
// level-0 intensity int(0.114 x + 0.299 y + 0.587 z) from the RGBA8 texel. Either output may be NULL.
__global__ void k_depth_intensity_l0(const float4* __restrict__ vmaps_tmp, const uchar4* __restrict__ rgba, size_t n, float cutoff,
                                     float* __restrict__ depth, uint8_t* __restrict__ image) {
  pdl_enter();
  for (size_t p = (size_t)blockIdx.x * blockDim.x + threadIdx.x; p < n; p += (size_t)gridDim.x * blockDim.x) {
    if (depth) {
      const float z = vmaps_tmp[p].z;
      depth[p] = (z > cutoff || z <= 0) ? qnan() : z;
    }
    if (image) {
      const uchar4 s = rgba[p];
      const int value = __float2int_rz((float)s.x * 0.114f + (float)s.y * 0.299f + (float)s.z * 0.587f);
      image[p] = (uint8_t)value;
    }
  }
}

__device__ __constant__ float c_gauss25[25] = {1, 4, 6, 4, 1, 4, 16, 24, 16, 4, 6, 24, 36, 24, 6, 4, 16, 24, 16, 4, 1, 4, 6, 4, 1};

// pyrDownKernelGaussF + pyrDownKernelIntensityGauss (cudafuncs.cu:383-411,512-562): window [2x-2, min(2x+3, n-1)),
// flipped/shifted tap index, int normaliser, NaN / zero skipping, truncating u8 store. As above, level 2 is produced in the
// same launch by recomputing the level-1 taps it needs.
template <typename Fetch>
__device__ __forceinline__ float pyr_down_f_at(Fetch fetch, int srows, int scols, int x, int y) {
  const int D = 5;
  const int tx = min(2 * x - D / 2 + D, scols - 1);
  const int ty = min(2 * y - D / 2 + D, srows - 1);
  float sum = 0;
  int count = 0;
  const int cy0 = max(0, 2 * y - D / 2), cx0 = max(0, 2 * x - D / 2);
#pragma unroll
  for (int dy = 0; dy < 5; ++dy)
#pragma unroll
    for (int dx = 0; dx < 5; ++dx) {
      const int cy = cy0 + dy, cx = cx0 + dx;
      const bool in = (cy < ty) && (cx < tx);
      const float s = in ? fetch(cy, cx) : 0.f;
      if (in && !isnan(s)) {
        const float w = c_gauss25[(ty - cy - 1) * 5 + (tx - cx - 1)];
        sum += s * w;
        count = __float2int_rz((float)count + w);
      }
    }
  return (float)(sum / (float)count);
}
template <typename Fetch>
__device__ __forceinline__ uint8_t pyr_down_u8_at(Fetch fetch, int srows, int scols, int x, int y) {
  const int D = 5;
  const int tx = min(2 * x - D / 2 + D, scols - 1);
  const int ty = min(2 * y - D / 2 + D, srows - 1);
  float sum = 0;
  int count = 0;
  const int cy0 = max(0, 2 * y - D / 2), cx0 = max(0, 2 * x - D / 2);
#pragma unroll
  for (int dy = 0; dy < 5; ++dy)
#pragma unroll
    for (int dx = 0; dx < 5; ++dx) {
      const int cy = cy0 + dy, cx = cx0 + dx;
      const bool in = (cy < ty) && (cx < tx);
      const int s = in ? fetch(cy, cx) : 0;
      if (in && s > 0) {
        const float w = c_gauss25[(ty - cy - 1) * 5 + (tx - cx - 1)];
        sum += s * w;
        count = __float2int_rz((float)count + w);
      }
    }
  const int v = __float2int_rz(sum / (float)count);  // NaN -> 0
  return (uint8_t)min(max(v, 0), 255);
}

// depth (fp32) and intensity (u8) pyramid level in one launch. Either pair may be NULL.
__global__ void k_pyr_down_depth_image(const float* __restrict__ d0, float* __restrict__ d1, const uint8_t* __restrict__ i0,
                                       uint8_t* __restrict__ i1, int srows, int scols) {
  pdl_enter();
  const int r1 = srows / 2, c1 = scols / 2;
  for (int t = blockIdx.x * blockDim.x + threadIdx.x; t < r1 * c1; t += gridDim.x * blockDim.x) {
    const int y = t / c1, x = t - y * c1;
    if (d0) {
      auto f0 = [&](int yy, int xx) { return d0[(size_t)yy * scols + xx]; };
      d1[t] = pyr_down_f_at(f0, srows, scols, x, y);
    }
    if (i0) {
      auto g0 = [&](int yy, int xx) { return (int)i0[(size_t)yy * scols + xx]; };
      i1[t] = pyr_down_u8_at(g0, srows, scols, x, y);
    }
  }
}

// The model side of a frame (frameToModel.initICPModel + initRGBModel, ElasticFusion.cpp:302-322) in three launches instead of six:
// level 0 = k_copy_maps + k_depth_intensity_l0 in one pass over the predicted textures (the depth IS the vertex z just loaded);
// each coarser level = k_resize_maps + k_pyr_down_depth_image for the same output pixel. Same arithmetic, same outputs; the
// separate kernels remain for the stage API and the trackers that initialise only one half.
__global__ void k_model_level0(const float4* __restrict__ vtxA, const float4* __restrict__ nrmA, const float4* __restrict__ vtxB,
                               const float4* __restrict__ nrmB, const uchar4* __restrict__ rgbaA, const uchar4* __restrict__ rgbaB,
                               const int* __restrict__ dense_count, int forceB_rgb, int rows, int cols, float cutoff, float4* __restrict__ vmaps_tmp,
                               float* __restrict__ vmap, float* __restrict__ nmap, float* __restrict__ depth, uint8_t* __restrict__ image) {
  pdl_enter();
  const size_t n = (size_t)rows * cols;
  const bool useB = dense_count && !dense_enough_of(*dense_count, rows, cols);
  const float4* __restrict__ vtx = useB ? vtxB : vtxA;
  const float4* __restrict__ nrm = useB ? nrmB : nrmA;
  const uchar4* __restrict__ rgba = (forceB_rgb || useB) ? rgbaB : rgbaA;
  for (size_t p = (size_t)blockIdx.x * blockDim.x + threadIdx.x; p < n; p += (size_t)gridDim.x * blockDim.x) {
    const float4 vs = vtx[p];
    const float4 ns = nrm[p];
    const uchar4 s = rgba[p];
    vmaps_tmp[p] = vs;
    f3 vd = mk3(qnan(), qnan(), qnan()), nd = vd;
    if (!(vs.z == 0)) {
      vd = mk3(vs.x, vs.y, vs.z);
      nd = mk3(ns.x, ns.y, ns.z);
    }
    vmap[p] = vd.x;
    vmap[p + n] = vd.y;
    vmap[p + 2 * n] = vd.z;
    nmap[p] = nd.x;
    nmap[p + n] = nd.y;
    nmap[p + 2 * n] = nd.z;
    depth[p] = (vs.z > cutoff || vs.z <= 0) ? qnan() : vs.z;
    image[p] = (uint8_t)__float2int_rz((float)s.x * 0.114f + (float)s.y * 0.299f + (float)s.z * 0.587f);
  }
}

__global__ void k_model_level_down(const float* __restrict__ vin, const float* __restrict__ nin, const float* __restrict__ d0,
                                   const uint8_t* __restrict__ i0, int srows, int scols, float* __restrict__ vout, float* __restrict__ nout,
                                   float* __restrict__ d1, uint8_t* __restrict__ i1) {
  pdl_enter();
  const int drows = srows / 2, dcols = scols / 2;
  const size_t splane = (size_t)srows * scols, dplane = (size_t)drows * dcols;
  for (int t = blockIdx.x * blockDim.x + threadIdx.x; t < drows * dcols; t += gridDim.x * blockDim.x) {
    const int y = t / dcols, x = t - y * dcols;
    const int xs = x * 2, ys = y * 2;
    const size_t q = (size_t)t;
    // resizeVMap + resizeNMap (cudafuncs.cu:413-490): 2x2 box average, any NaN -> NaN, normals renormalised
#pragma unroll
    for (int which = 0; which < 2; ++which) {
      const float* in = which ? nin : vin;
      float* out = which ? nout : vout;
      const float x00 = in[(size_t)(ys + 0) * scols + xs + 0], x01 = in[(size_t)(ys + 0) * scols + xs + 1];
      const float x10 = in[(size_t)(ys + 1) * scols + xs + 0], x11 = in[(size_t)(ys + 1) * scols + xs + 1];
      if (isnan(x00) || isnan(x01) || isnan(x10) || isnan(x11)) {
        out[q] = qnan();
        out[q + dplane] = qnan();
        out[q + 2 * dplane] = qnan();
        continue;
      }
      f3 n;
      n.x = (x00 + x01 + x10 + x11) / 4;
      const float* iy = in + splane;
      n.y = (iy[(size_t)(ys + 0) * scols + xs + 0] + iy[(size_t)(ys + 0) * scols + xs + 1] + iy[(size_t)(ys + 1) * scols + xs + 0] +
             iy[(size_t)(ys + 1) * scols + xs + 1]) / 4;
      const float* iz = in + 2 * splane;
      n.z = (iz[(size_t)(ys + 0) * scols + xs + 0] + iz[(size_t)(ys + 0) * scols + xs + 1] + iz[(size_t)(ys + 1) * scols + xs + 0] +
             iz[(size_t)(ys + 1) * scols + xs + 1]) / 4;
      if (which) n = normalized(n);
      out[q] = n.x;
      out[q + dplane] = n.y;
      out[q + 2 * dplane] = n.z;
    }
    // pyrDownGaussF + pyrDownUcharGauss for the same output pixel
    auto f0 = [&](int yy, int xx) { return d0[(size_t)yy * scols + xx]; };
    d1[t] = pyr_down_f_at(f0, srows, scols, x, y);
    auto g0 = [&](int yy, int xx) { return (int)i0[(size_t)yy * scols + xx]; };
    i1[t] = pyr_down_u8_at(g0, srows, scols, x, y);
  }
}

// computeDerivativeImages / applyKernel (cudafuncs.cu:612-668) for all three levels in one launch, fused with the
// pose-independent gates of computeRgbResidual (reduce.cu:641-660): a pixel is a photometric *candidate* when
// j < cols-5, i < rows-1, its 4x4 neighbourhood of the live image is non-zero, its gradient magnitude passes minScale and
// its depth is finite. None of this changes across the 19 Gauss-Newton iterations, so it is evaluated once per frame and
// the iterations only visit the compacted candidate list (typically ~10 % of the pixels at level 0).
struct SobelArgs {
  const uint8_t* src[NUM_PYRS];
  const float* depth[NUM_PYRS];
  int16_t* dx[NUM_PYRS];
  int16_t* dy[NUM_PYRS];
  int rows[NUM_PYRS], cols[NUM_PYRS];
  int start[NUM_PYRS + 1];
  float minScale[NUM_PYRS];
};
// A persistent grid over tiles of SC_THREADS pixels, drawn in order from the dispenser counter[0]: a candidate takes its slot in
// the list from its tile's exclusive prefix (lookback_prefix), so the list keeps the flat pixel order (level 0, 1, 2) without a
// separate scan. The first pixel of each level publishes the level's start, the last tile the total.
constexpr int SC_THREADS = 256;
__global__ void __launch_bounds__(SC_THREADS) k_sobel_cand(SobelArgs a, int4* __restrict__ cand, GNState* gn, unsigned long long* state,
                                                          unsigned int* counter, unsigned int epoch) {
  pdl_enter();
  const float gsx[9] = {(float)0.52201, (float)0.00000, (float)-0.52201, (float)0.79451, (float)-0.00000,
                        (float)-0.79451, (float)0.52201, (float)0.00000, (float)-0.52201};
  const float gsy[9] = {(float)0.52201, (float)0.79451, (float)0.52201, (float)0.00000, (float)0.00000,
                        (float)0.00000, (float)-0.52201, (float)-0.79451, (float)-0.52201};
  const int total = a.start[NUM_PYRS];
  const int num_tiles = (total + SC_THREADS - 1) / SC_THREADS;
  __shared__ int s_warp[SC_THREADS / 32];
  __shared__ int s_tile, s_prefix;
  while (true) {
    if (threadIdx.x == 0) s_tile = (int)atomicAdd(counter, 1u);
    __syncthreads();
    const int tile = s_tile;
    if (tile >= num_tiles) {
      if (threadIdx.x == 0) dispenser_exit<false>(counter);
      return;
    }
    const int f = tile * SC_THREADS + threadIdx.x;
    const int lv = (f >= a.start[2]) ? 2 : (f >= a.start[1] ? 1 : 0);
    const int rows = a.rows[lv], cols = a.cols[lv];
    const int p = f - a.start[lv];
    const uint8_t* __restrict__ src = a.src[lv];
    const int y = p / cols, x = p - y * cols;
    int valx = 0, valy = 0;
    bool ok = false;
    if (f < total) {
      float dxVal = 0, dyVal = 0;
      int kernelIndex = 8;
      for (int j = max(y - 1, 0); j <= min(y + 1, rows - 1); j++)
        for (int i = max(x - 1, 0); i <= min(x + 1, cols - 1); i++) {
          const float s = (float)src[(size_t)j * cols + i];
          dxVal += s * gsx[kernelIndex];
          dyVal += s * gsy[kernelIndex];
          --kernelIndex;
        }
      valx = (int16_t)__float2int_rz(dxVal);
      valy = (int16_t)__float2int_rz(dyVal);
      a.dx[lv][p] = (int16_t)valx;
      a.dy[lv][p] = (int16_t)valy;
      ok = (x < cols - 5 && y < rows - 1);
      if (ok) {
        const float mTwo = (float)((valx * valx) + (valy * valy));
        ok = (mTwo >= a.minScale[lv]) && !isnan(a.depth[lv][p]);
      }
      if (ok) {
        for (int u = max(y - 2, 0); u < min(y + 2, rows); u++)
          for (int v = max(x - 2, 0); v < min(x + 2, cols); v++) ok = ok && (src[(size_t)u * cols + v] > 0);
      }
    }
    int aggregate;
    const int excl = block_exclusive_scan<SC_THREADS>(ok ? 1 : 0, s_warp, aggregate);
    if (threadIdx.x < 32) {
      const int prefix = lookback_prefix(state, tile, 0, 0, aggregate, epoch);
      if (threadIdx.x == 0) {
        s_prefix = prefix;
        if (tile == num_tiles - 1) gn->cand_base[NUM_PYRS] = prefix + aggregate;
      }
    }
    __syncthreads();
    const int o = s_prefix + excl;
    if (f < total && f == a.start[lv]) gn->cand_base[lv] = o;  // exclusive prefix at the first pixel of the level
    if (ok) {
      const int g = ((int)(uint16_t)valx) | (((int)(uint16_t)valy) << 16);
      cand[o] = make_int4(p, __float_as_int(a.depth[lv][p]), g, (int)src[p]);
    }
    __syncthreads();  // s_tile and s_prefix are rewritten by the next draw
  }
}

// Track view: puts the view tracker's GNState back to what alloc_odom leaves for the view's camera, at the guess (the view's pose,
// staged by its model prediction)
__global__ void k_track_view_reset(GNState* gn, const double* __restrict__ T_wc, int width, int height, float fx, float fy, float cx, float cy) {
  pdl_enter();
  if (threadIdx.x != 0 || blockIdx.x != 0) return;
  gn_initial_state(gn, width, height, fx, fy, cx, cy);
  for (int k = 0; k < 16; ++k) gn->T_wc[k] = T_wc[k];
}

// pose, RGBDOdometry's public results and getCovariance of a tracker
__device__ __forceinline__ void odom_result(const GNState* __restrict__ gn, double* T_wc, EfOdomStats& s, double* covariance) {
  for (int k = 0; k < 16; ++k) T_wc[k] = gn->T_wc[k];
  s.lastICPError = gn->lastICPError;
  s.lastICPCount = gn->lastICPCount;
  s.lastRGBError = gn->lastRGBError;
  s.lastRGBCount = gn->lastRGBCount;
  s.lastSO3Error = gn->lastSO3Error;
  s.lastSO3Count = gn->lastSO3Count;
  for (int k = 0; k < 36; ++k) s.lastA[k] = gn->lastA[k];
  for (int k = 0; k < 6; ++k) s.lastb[k] = gn->lastb[k];
  efm::inv_n<6>(gn->lastA, covariance);  // lastA.lu().inverse(), as ef_odom_covariance
}

// EfTrackResult of a track view (ef_track_view_device): pose, RGBDOdometry's public results, getCovariance and denseEnough
__global__ void k_track_view_result(const GNState* __restrict__ gn, const int* __restrict__ dense_count, int rows, int cols,
                                    EfTrackResult* __restrict__ out) {
  pdl_enter();
  if (threadIdx.x != 0 || blockIdx.x != 0) return;
  odom_result(gn, out->T_wc, out->stats, out->covariance);
  out->dense_enough = dense_enough_of(*dense_count, rows, cols) ? 1 : 0;
}

// EfCameraResult of a camera frame: the above, whether it tracked, denseEnough of the prediction it tracked against and the weighting
__global__ void k_camera_result(const GNState* __restrict__ gn, const int* __restrict__ dense_count, int rows, int cols, int tracked,
                                EfCameraResult* __restrict__ out) {
  pdl_enter();
  if (threadIdx.x != 0 || blockIdx.x != 0) return;
  odom_result(gn, out->T_wc, out->stats, out->covariance);
  out->tracked = tracked;
  out->dense_enough = dense_enough_of(*dense_count, rows, cols) ? 1 : 0;
  out->weighting = gn->weighting;
}

// EfRigResult of a rig frame: member 0's pose, the joint system its tracker state holds and its inverse
__global__ void k_rig_result(const GNState* __restrict__ gn, int tracked, EfRigResult* __restrict__ out) {
  pdl_enter();
  if (threadIdx.x != 0 || blockIdx.x != 0) return;
  for (int k = 0; k < 16; ++k) out->T_wc[k] = gn->T_wc[k];
  for (int k = 0; k < 36; ++k) out->lastA[k] = gn->lastA[k];
  for (int k = 0; k < 6; ++k) out->lastb[k] = gn->lastb[k];
  efm::inv_n<6>(gn->lastA, out->covariance);
  out->tracked = tracked;
}

// =============================================================================================
// host side: RGBDOdometry mirror
// =============================================================================================

namespace {

inline dim3 grid2d(int cols, int rows) { return dim3((cols + 31) / 32, (rows + 7) / 8); }
}  // namespace

namespace ef {

int odom_init_icp_depth(EfContext* ctx, int which, const uint16_t* depth_dev, float cutoff) {
  OdomDev& od = ctx->odom[which];
  ctx->maps_dirty[which] = true;
  CU(cudaMemcpyAsync(od.depth_tmp[0], depth_dev, sizeof(uint16_t) * od.width * od.height, cudaMemcpyDeviceToDevice, ctx->stream));
  for (int i = 1; i < NUM_PYRS; ++i)
    EF_LAUNCH(ctx, k_pyr_down_u16, wave_blocks(ctx, (size_t)od.rows[i] * od.cols[i] * 2), 128, 0, od.depth_tmp[i - 1], od.rows[i - 1], od.cols[i - 1],
              od.depth_tmp[i]);
  VmapArgs va;
  const float* cam = ctx->odom_cam[which];
  for (int i = 0; i < NUM_PYRS; ++i) {
    const int div = 1 << i;
    const float fx = cam[0] / div, fy = cam[1] / div, cx = cam[2] / div, cy = cam[3] / div;
    va.depth[i] = od.depth_tmp[i];
    va.vmap[i] = od.vmap_curr[i];
    va.nmap[i] = od.nmap_curr[i];
    va.rows[i] = od.rows[i];
    va.cols[i] = od.cols[i];
    va.start[i] = od.level_start[i];
    va.fx_inv[i] = 1.f / fx;
    va.fy_inv[i] = 1.f / fy;
    va.cx[i] = cx;
    va.cy[i] = cy;
  }
  va.start[NUM_PYRS] = od.level_start[NUM_PYRS];
  EF_LAUNCH(ctx, k_vmap_nmap, wave_blocks(ctx, (size_t)od.level_start[NUM_PYRS]), 256, 0, va, cutoff);
  CHECK_LAST();
  return 0;
}

static int copy_and_resize(EfContext* ctx, OdomDev& od, const float* vtx4, const float* nrm4, float** vm, float** nm) {
  const size_t n = (size_t)od.width * od.height;
  EF_LAUNCH(ctx, k_copy_maps, wave_blocks(ctx, n), 256, 0, (const float4*)vtx4, (const float4*)nrm4, od.height, od.width, (float4*)od.vmaps_tmp,
            vm[0], nm[0]);
  const dim3 block(32, 8);
  for (int i = 1; i < NUM_PYRS; ++i)
    EF_LAUNCH(ctx, k_resize_maps, grid2d(od.cols[i], od.rows[i]), block, 0, vm[i - 1], nm[i - 1], od.rows[i - 1], od.cols[i - 1], vm[i], nm[i]);
  CHECK_LAST();
  return 0;
}

int odom_init_icp_pred(EfContext* ctx, int which, const float* vtx4, const float* nrm4) {
  OdomDev& od = ctx->odom[which];
  ctx->maps_dirty[which] = true;
  return copy_and_resize(ctx, od, vtx4, nrm4, od.vmap_curr, od.nmap_curr);
}

// pose is taken from gn->T_wc (device) — callers that pass an explicit pose upload it first
int odom_init_icp_model(EfContext* ctx, int which, const float* vtx4, const float* nrm4, bool with_global) {
  OdomDev& od = ctx->odom[which];
  RC(copy_and_resize(ctx, od, vtx4, nrm4, od.vmap_c_prev, od.nmap_c_prev));
  if (!with_global) return 0;  // the frame loop never reads the world-frame copy
  XformArgs a;
  for (int i = 0; i < NUM_PYRS; ++i) {
    a.sv[i] = od.vmap_c_prev[i];
    a.sn[i] = od.nmap_c_prev[i];
    a.v[i] = od.vmap_g_prev[i];
    a.n[i] = od.nmap_g_prev[i];
    a.rows[i] = od.rows[i];
    a.cols[i] = od.cols[i];
  }
  EF_LAUNCH(ctx, k_transform_maps, dim3(wave_blocks(ctx, (size_t)od.width * od.height), NUM_PYRS), 256, 0, a, (const GNState*)od.gn);
  CHECK_LAST();
  return 0;
}

// populateRGBDData (RGBDOdometry.cpp:212-234); with_depth=0 is initFirstRGB (:246-257)
int odom_populate(EfContext* ctx, int which, const uint8_t* rgba, float** destDepths, uint8_t** destImages, bool with_depth,
                  bool with_image) {
  OdomDev& od = ctx->odom[which];
  const size_t n = (size_t)od.width * od.height;
  EF_LAUNCH(ctx, k_depth_intensity_l0, wave_blocks(ctx, n), 256, 0, (const float4*)od.vmaps_tmp, (const uchar4*)rgba, n, od.maxDepthRGB,
            with_depth ? destDepths[0] : (float*)nullptr, with_image ? destImages[0] : (uint8_t*)nullptr);
  for (int i = 0; i + 1 < NUM_PYRS; ++i)
    EF_LAUNCH(ctx, k_pyr_down_depth_image, wave_blocks(ctx, (size_t)od.rows[i + 1] * od.cols[i + 1] * 2), 128, 0,
              with_depth ? destDepths[i] : (const float*)nullptr, with_depth ? destDepths[i + 1] : (float*)nullptr,
              with_image ? (const uint8_t*)destImages[i] : (const uint8_t*)nullptr, with_image ? destImages[i + 1] : (uint8_t*)nullptr, od.rows[i],
              od.cols[i]);
  CHECK_LAST();
  return 0;
}

// initICPModel + initRGBModel of tracker `which` in k_model_level0 / k_model_level_down: the A inputs, or the B ones when dense_count
// is given and not dense enough (the image also when forceB_rgb)
static int odom_model_inputs(EfContext* ctx, int which, const float4* vtxA, const float4* nrmA, const float4* vtxB, const float4* nrmB,
                             const uchar4* imgA, const uchar4* imgB, const int* dense_count, int forceB_rgb) {
  OdomDev& od = ctx->odom[which];
  ctx->maps_dirty[which] = true;
  const size_t n = (size_t)od.width * od.height;
  EF_LAUNCH(ctx, k_model_level0, wave_blocks(ctx, n), 256, 0, vtxA, nrmA, vtxB, nrmB, imgA, imgB, dense_count, forceB_rgb, od.height, od.width,
            od.maxDepthRGB, (float4*)od.vmaps_tmp, od.vmap_c_prev[0], od.nmap_c_prev[0], od.lastDepth[0], od.lastImage[0]);
  for (int i = 0; i + 1 < NUM_PYRS; ++i)
    EF_LAUNCH(ctx, k_model_level_down, wave_blocks(ctx, (size_t)od.rows[i + 1] * od.cols[i + 1] * 2), 128, 0, (const float*)od.vmap_c_prev[i],
              (const float*)od.nmap_c_prev[i], (const float*)od.lastDepth[i], (const uint8_t*)od.lastImage[i], od.rows[i], od.cols[i],
              od.vmap_c_prev[i + 1], od.nmap_c_prev[i + 1], od.lastDepth[i + 1], od.lastImage[i + 1]);
  CHECK_LAST();
  return 0;
}

// frameToModel.initICPModel + initRGBModel with the reference's fill-in choice (ElasticFusion.cpp:302-315) resolved on
// the device: predicted maps when the model view is dense enough, FillIn maps otherwise.
int map_select_model_inputs(EfContext* ctx) {
  Textures& t = ctx->tex;
  return odom_model_inputs(ctx, 0, (const float4*)t.vertex, (const float4*)t.normal, (const float4*)t.fill_vertex, (const float4*)t.fill_normal,
                           (const uchar4*)t.image, (const uchar4*)t.fill_image, (const int*)ctx->map.dense_count, ctx->frame_to_frame_rgb ? 1 : 0);
}

int launch_sobel(EfContext* ctx, int which) {
  OdomDev& od = ctx->odom[which];
  SobelArgs a;
  for (int i = 0; i < NUM_PYRS; ++i) {
    a.src[i] = od.nextImage[i];
    a.depth[i] = od.nextDepth[i];
    a.dx[i] = od.dIdx[i];
    a.dy[i] = od.dIdy[i];
    a.rows[i] = od.rows[i];
    a.cols[i] = od.cols[i];
    a.start[i] = od.level_start[i];
    a.minScale[i] = od.minScale[i];
  }
  a.start[NUM_PYRS] = od.level_start[NUM_PYRS];
  ScanSlot sc;
  ScanTiles* tiles = ctx->odom_tiles[which];
  RC(tiles ? scan_slot(ctx, *tiles, &sc) : scan_slot(ctx, &sc));
  EF_LAUNCH(ctx, k_sobel_cand, wave_blocks(ctx, (size_t)od.level_start[NUM_PYRS], 8, SC_THREADS), SC_THREADS, 0, a, od.cand, od.gn, sc.state,
            sc.counter, sc.epoch);
  ctx->maps_dirty[which] = true;  // k_iter1 / k_iter2 read the list ahead of their dependency wait: fence before the next one
  CHECK_LAST();
  return 0;
}

// ---- one launch sequence for the trackers outside the frame: the track view's and the cameras' -------------------------------
// A tracker's input buffers at its camera's size
struct LiveBuffers {
  uint8_t *rgb, *rgba;  // W*H*3, W*H*4
  uint16_t *depth_raw, *depth_filtered;
  float *depth_metric, *depth_metric_filtered;  // null: not computed
};

// The live side of a frame at tracker `which`'s camera (ElasticFusion.cpp:278-285, initICP and initRGB's intensity half): the inputs
// copied into b.rgb / b.depth_raw when copy is set (rgb and depth then point there), RGBA, the bilateral filter and metric depths,
// the depth pyramid with its vertex / normal maps at max_depth, and the intensity pyramid (nextImage)
static int track_live_side(EfContext* ctx, int which, const LiveBuffers& b, const uint8_t*& rgb, const uint16_t*& depth, bool copy,
                           cudaMemcpyKind kind, float depth_cutoff, float max_depth) {
  OdomDev& od = ctx->odom[which];
  const int w = od.width, h = od.height;
  const size_t n = (size_t)w * h;
  if (copy) {
    CU(cudaMemcpyAsync(b.rgb, rgb, n * 3, kind, ctx->stream));
    CU(cudaMemcpyAsync(b.depth_raw, depth, n * 2, kind, ctx->stream));
    rgb = b.rgb;
    depth = b.depth_raw;
  }
  RC(rgb_to_rgba(ctx, h, w, rgb, b.rgba));
  RC(preprocess_depth(ctx, h, w, depth, depth_cutoff, b.depth_filtered, b.depth_metric, b.depth_metric_filtered));
  RC(odom_init_icp_depth(ctx, which, b.depth_filtered, max_depth));
  return odom_populate(ctx, which, b.rgba, nullptr, od.nextImage, false);
}

// The model side: the predicted maps (A) or, when dense_count is given and not dense enough, the fill-in (B); the image B also when
// frame_to_frame_rgb. initRGB's depth half is the model's (quirk A.2: it reads the vmaps_tmp initICPModel just filled), aliased to it
// unless frame_to_frame_rgb builds it from rgba as the frame does.
struct ModelInputs {
  const float4 *vtxA, *nrmA, *vtxB, *nrmB;
  const uchar4 *imgA, *imgB;
  const int* dense_count;
  bool frame_to_frame_rgb;
  const uint8_t* rgba;
};

// initICPModel + initRGBModel and initRGB's depth half in tracker `which`; unless frame_to_frame_rgb, nextDepth aliases lastDepth until
// track_model_restore puts `saved` back
static int track_model_side(EfContext* ctx, int which, const ModelInputs& m, float* (&saved)[NUM_PYRS]) {
  OdomDev& od = ctx->odom[which];
  RC(odom_model_inputs(ctx, which, m.vtxA, m.nrmA, m.vtxB, m.nrmB, m.imgA, m.imgB, m.dense_count, m.frame_to_frame_rgb ? 1 : 0));
  if (m.frame_to_frame_rgb) return odom_populate(ctx, which, m.rgba, od.nextDepth, od.nextImage, true, false);
  for (int i = 0; i < NUM_PYRS; ++i) {
    saved[i] = od.nextDepth[i];
    od.nextDepth[i] = od.lastDepth[i];
  }
  return 0;
}
static void track_model_restore(EfContext* ctx, int which, const ModelInputs& m, float* const (&saved)[NUM_PYRS]) {
  if (m.frame_to_frame_rgb) return;
  for (int i = 0; i < NUM_PYRS; ++i) ctx->odom[which].nextDepth[i] = saved[i];
}

// initICPModel + initRGBModel, initRGB's depth half, getIncrementalTransformation and its finish with the velocity weighting
// (ElasticFusion.cpp:302-383) in tracker `which`, whose pose is the starting point; the finished pose also into pose_record
static int track_solve(EfContext* ctx, int which, const ModelInputs& m, bool rgb_only, float icp_weight, bool pyramid, bool fast_odom, bool so3,
                       float weight_multiplier, MapPose* pose_record) {
  float* saved[NUM_PYRS];
  RC(track_model_side(ctx, which, m, saved));
  const int rc = odom_track_async(ctx, which, rgb_only, icp_weight, pyramid, fast_odom, so3);
  track_model_restore(ctx, which, m, saved);
  RC(rc);
  return odom_finish_async(ctx, which, weight_multiplier, true, pose_record);
}

// ---- track view (ef_track_view*): the frame's tracking recipe at any camera, in tracker slot VIEW_TRACKER --------------------
// Its inputs, prediction and pyramids live in one arena, allocated by the first call and reallocated for the bounding box of every
// view so far when a view does not fit: each pyramid level of a w x h view then fits the level allocated for W x H >= w x h.
struct TrackViewBuffers {
  Arena arena;             // everything below and every buffer of ctx->odom[VIEW_TRACKER]
  int width, height;       // the size the buffers were allocated for
  uint8_t *rgb, *rgba;     // W*H*3, W*H*4
  uint16_t *depth_raw, *depth_filtered;
  uchar4* image;           // the model prediction at the guess (no fill-in)
  float4 *vertex, *normal;
  int* dense_count;        // lit samples of the predicted image's decimation (k_splat_scatter zeroes it, k_splat_resolve counts)
  ScanTiles scan;          // look-back tile states of the candidate compaction (k_sobel_cand), sized for this tracker's pyramid
};

static TrackViewBuffers& tvb(EfContext* ctx) { return *static_cast<TrackViewBuffers*>(ctx->track_view); }

// look-back tile states of k_sobel_cand for tracker `which`'s pyramid, from `arena`, and routed to its launches
static int alloc_cand_tiles(EfContext* ctx, Arena& arena, int which, ScanTiles& scan) {
  const size_t tiles = (size_t)(ctx->odom[which].level_start[NUM_PYRS] + SC_THREADS - 1) / SC_THREADS + 2;
  CU(arena_alloc(ctx, arena, &scan.state, tiles, 0));
  CU(arena_alloc(ctx, arena, &scan.counter, 4, 0));
  scan.bytes = tiles * 8;
  scan.epoch = 0;
  ctx->odom_tiles[which] = &scan;
  return 0;
}

static int track_view_alloc(EfContext* ctx, TrackViewBuffers& V, int W, int H) {
  const size_t px = (size_t)W * H;
  RC(alloc_odom(ctx, V.arena, VIEW_TRACKER, W, H, 1.f, 1.f, 0.f, 0.f));  // (camera and state: written per call)
  CU(arena_alloc(ctx, V.arena, &V.rgb, px * 3));
  CU(arena_alloc(ctx, V.arena, &V.rgba, px * 4));
  CU(arena_alloc(ctx, V.arena, &V.depth_raw, px));
  CU(arena_alloc(ctx, V.arena, &V.depth_filtered, px));
  CU(arena_alloc(ctx, V.arena, &V.image, px));
  CU(arena_alloc(ctx, V.arena, &V.vertex, px));
  CU(arena_alloc(ctx, V.arena, &V.normal, px));
  CU(arena_alloc(ctx, V.arena, &V.dense_count, 1, 0));
  RC(alloc_cand_tiles(ctx, V.arena, VIEW_TRACKER, V.scan));
  CU(cudaStreamSynchronize(ctx->stream));
  V.width = W;
  V.height = H;
  return 0;
}

// the view's buffers, grown when it does not fit (EF_ENOMEM if they cannot be: the context stays usable)
static int track_view_buffers(EfContext* ctx, int w, int h) {
  if (!ctx->track_view) {
    TrackViewBuffers* nv = new (std::nothrow) TrackViewBuffers();
    if (!nv) return EF_ENOMEM;
    ctx->track_view = nv;
  }
  TrackViewBuffers& V = tvb(ctx);
  if (w <= V.width && h <= V.height) return 0;
  const int W = w > V.width ? w : V.width, H = h > V.height ? h : V.height;
  CU(cudaStreamSynchronize(ctx->stream));  // the previous view may still read the old buffers
  V.arena.release();
  V.width = V.height = 0;
  if (int rc = track_view_alloc(ctx, V, W, H)) {
    V.arena.release();
    V.width = V.height = 0;
    if (rc != (int)cudaErrorMemoryAllocation) return rc;
    cudaGetLastError();  // (an allocation failure is not sticky)
    return EF_ENOMEM;
  }
  return 0;
}

// upload (host inputs), RGBA, bilateral filter, the live pyramids, combinedPredict at the guess, the model pyramids, Sobel + candidates
// and getIncrementalTransformation without SO(3): ElasticFusion.cpp:278-323 for a camera of the caller's
int track_view_async(EfContext* ctx, const EfTrackView* v, const uint8_t* rgb, const uint16_t* depth, bool from_host, EfTrackResult* out_dev) {
  const EfModelView& mv = v->model;
  const int w = mv.width, h = mv.height;
  RC(track_view_buffers(ctx, w, h));
  TrackViewBuffers& V = tvb(ctx);
  OdomDev& od = ctx->odom[VIEW_TRACKER];
  // the view's size inside buffers allocated for V.width x V.height
  od.width = w;
  od.height = h;
  for (int i = 0, flat = 0; i <= NUM_PYRS; ++i) {
    od.level_start[i] = flat;
    if (i == NUM_PYRS) break;
    od.rows[i] = h >> i;
    od.cols[i] = w >> i;
    flat += od.rows[i] * od.cols[i];
  }
  const float cam[4] = {mv.fx, mv.fy, mv.cx, mv.cy};
  memcpy(ctx->odom_cam[VIEW_TRACKER], cam, sizeof(cam));
  const LiveBuffers live = {V.rgb, V.rgba, V.depth_raw, V.depth_filtered, nullptr, nullptr};
  RC(track_live_side(ctx, VIEW_TRACKER, live, rgb, depth, from_host, cudaMemcpyHostToDevice, v->depth_cutoff, mv.max_depth));
  // model side: combinedPredict at the guess (which stages the guess as the view pose), the tracker reset to it, then the solve
  RC(map_predict_view_async(ctx, &mv, reinterpret_cast<uint8_t*>(V.image), reinterpret_cast<float*>(V.vertex),
                            reinterpret_cast<float*>(V.normal), nullptr, V.dense_count));
  EF_LAUNCH(ctx, k_track_view_reset, 1, 32, 0, od.gn, (const double*)ctx->dev_small->view_pose, w, h, mv.fx, mv.fy, mv.cx, mv.cy);
  const ModelInputs m = {V.vertex, V.normal, V.vertex, V.normal, V.image, V.image, nullptr, false, V.rgba};
  RC(track_solve(ctx, VIEW_TRACKER, m, v->rgb_only != 0, v->icp_weight, v->pyramid != 0, v->fast_odom != 0, false, 1.0f, nullptr));
  if (out_dev) EF_LAUNCH(ctx, k_track_view_result, 1, 32, 0, (const GNState*)od.gn, (const int*)V.dense_count, h, w, out_dev);
  CHECK_LAST();
  return 0;
}

int track_view_read(EfContext* ctx, GNState* g, int* lit) {
  CU(cudaMemcpyAsync(g, ctx->odom[VIEW_TRACKER].gn, sizeof(GNState), cudaMemcpyDeviceToHost, ctx->stream));
  CU(cudaMemcpyAsync(lit, tvb(ctx).dense_count, sizeof(int), cudaMemcpyDeviceToHost, ctx->stream));
  CU(cudaStreamSynchronize(ctx->stream));
  return 0;
}

void track_view_free(EfContext* ctx) {
  TrackViewBuffers* V = static_cast<TrackViewBuffers*>(ctx->track_view);
  if (!V) return;
  V->arena.release();
  delete V;
  ctx->track_view = nullptr;
  ctx->odom_tiles[VIEW_TRACKER] = nullptr;
}

// ---- cameras (ef_camera_*): processFrame for a sensor of its own, in tracker slot cam->slot ----------------------------------
static int camera_alloc(EfContext* ctx, EfCamera& c) {
  const EfCameraConfig& k = c.cfg;
  const size_t px = (size_t)k.width * k.height;
  RC(alloc_odom(ctx, c.arena, c.slot, k.width, k.height, k.fx, k.fy, k.cx, k.cy));
  RC(alloc_cand_tiles(ctx, c.arena, c.slot, c.scan));
  CU(arena_alloc(ctx, c.arena, &c.rgba, px * 4, 0));
  CU(arena_alloc(ctx, c.arena, &c.depth_filtered, px, 0));
  CU(arena_alloc(ctx, c.arena, &c.image, px, 0));
  CU(arena_alloc(ctx, c.arena, &c.vertex, px, 0));
  CU(arena_alloc(ctx, c.arena, &c.normal, px, 0));
  CU(arena_alloc(ctx, c.arena, &c.time, px, 0));
  CU(arena_alloc(ctx, c.arena, &c.fill_image, px, 0));
  CU(arena_alloc(ctx, c.arena, &c.fill_vertex, px, 0));
  CU(arena_alloc(ctx, c.arena, &c.fill_normal, px, 0));
  CU(arena_alloc(ctx, c.arena, &c.dense_count, 1, 0));
  CU(arena_alloc(ctx, c.arena, &c.pose, 1, 0));
  CU(arena_alloc(ctx, c.arena, &c.result, 1, 0));
  CU(arena_alloc(ctx, c.arena, &c.dev_T, 16, 0));
  RC(map_camera_target(ctx, c.arena, k.height, k.width, k.fx, k.fy, k.cx, k.cy, &c.target_state, &c.target, &c.rgb, &c.depth_raw));
  c.target.pose = c.pose;
  c.target.weighting = &ctx->odom[c.slot].gn->weighting;
  if (k.close_loops) {  // its local loop closure: a modelToModel tracker, the INACTIVE prediction, the synthesised depth, the constraints
    LoopBuffers& L = c.loop;
    RC(alloc_odom(ctx, c.arena, c.loop_slot, k.width, k.height, k.fx, k.fy, k.cx, k.cy));
    RC(alloc_cand_tiles(ctx, c.arena, c.loop_slot, L.scan));
    CU(arena_alloc(ctx, c.arena, &L.old_image, px, 0));
    CU(arena_alloc(ctx, c.arena, &L.old_vertex, px, 0));
    CU(arena_alloc(ctx, c.arena, &L.old_normal, px, 0));
    CU(arena_alloc(ctx, c.arena, &L.old_time, px, 0));
    CU(arena_alloc(ctx, c.arena, &L.synth_depth, px, 0));
    CU(arena_alloc(ctx, c.arena, &L.loop, 1, 0));
    L.capacity = loop_constraint_capacity(k.width, k.height);
    CU(arena_alloc(ctx, c.arena, &L.src, 3 * (size_t)L.capacity, 0));
    CU(arena_alloc(ctx, c.arena, &L.dst, 3 * (size_t)L.capacity, 0));
    CU(arena_alloc(ctx, c.arena, &L.times, (size_t)L.capacity, 0));
    c.target.synth_depth = L.synth_depth;
  }
  unsigned long long* zbuf = nullptr;
  RC(offframe_zbuf(ctx, px, &zbuf));  // grown here, so that a frame never allocates
  CU(cudaMallocHost((void**)&c.pin_T, sizeof(double) * 16));
  CU(cudaEventCreateWithFlags(&c.pose_sent, cudaEventDisableTiming));
  CU(cudaEventRecord(c.pose_sent, ctx->stream));
  CU(cudaStreamSynchronize(ctx->stream));
  return 0;
}

// everything of a camera, allocated or not
static void camera_release(EfContext* ctx, EfCamera* c) {
  cudaStreamSynchronize(ctx->stream);
  c->arena.release();
  if (c->target_state) map_camera_target_free(c->target_state);
  if (c->pin_T) cudaFreeHost(c->pin_T);
  if (c->pose_sent) cudaEventDestroy(c->pose_sent);
  for (int w : {c->slot, c->loop_slot}) {
    memset(&ctx->odom[w], 0, sizeof(OdomDev));
    ctx->odom_tiles[w] = nullptr;
  }
  delete c;
}

int camera_create(EfContext* ctx, const EfCameraConfig* cfg, EfCamera** out) {
  int i = 0;
  while (i < EF_MAX_CAMERAS && ctx->cameras[i]) ++i;
  if (i == EF_MAX_CAMERAS) return EF_ESTATE;
  EfCamera* c = new (std::nothrow) EfCamera();
  if (!c) return EF_ENOMEM;
  c->slot = CAMERA_TRACKER0 + i;
  c->loop_slot = CAMERA_LOOP_TRACKER0 + i;
  c->cfg = *cfg;
  if (int rc = camera_alloc(ctx, *c)) {
    camera_release(ctx, c);
    if (rc != (int)cudaErrorMemoryAllocation && rc != EF_ENOMEM) return rc;
    cudaGetLastError();  // (an allocation failure is not sticky: the context stays usable)
    return EF_ENOMEM;
  }
  ctx->cameras[i] = c;
  *out = c;
  return 0;
}

void camera_destroy(EfContext* ctx, EfCamera* c) {
  if (c->rig) rig_destroy(ctx, c->rig);
  ctx->cameras[c->slot - CAMERA_TRACKER0] = nullptr;
  camera_release(ctx, c);
}

// combinedPredict at the camera's pose record, size and intrinsics, into nothing yet
static PredictTarget camera_predict_target(const EfCamera* c) {
  const EfCameraConfig& k = c->cfg;
  PredictTarget p = {};
  p.rows = k.height;
  p.cols = k.width;
  p.cx = k.cx;
  p.cy = k.cy;
  p.fx = k.fx;
  p.fy = k.fy;
  p.pose = c->pose;
  return p;
}

// a closing camera's side of the local loop closure: its tracker, its loop tracker, its prediction and LoopBuffers
static LoopSide camera_loop_side(const EfCamera* c) {
  const EfCameraConfig& k = c->cfg;
  const LoopBuffers& L = c->loop;
  LoopSide s = {};
  s.curr = c->slot;
  s.est = c->loop_slot;
  s.rows = k.height;
  s.cols = k.width;
  s.max_depth = k.max_depth;
  s.pyramid = k.pyramid != 0;
  s.fast_odom = k.fast_odom != 0;
  s.vertex = c->vertex;
  s.normal = c->normal;
  s.image = c->image;
  s.old_vertex = L.old_vertex;
  s.old_normal = L.old_normal;
  s.old_image = L.old_image;
  s.old_time = L.old_time;
  s.loop = L.loop;
  s.src = L.src;
  s.dst = L.dst;
  s.times = L.times;
  s.capacity = L.capacity;
  return s;
}

// The predictions of a closing camera's front half (the camera's own and a closing rig's members'): the mid-frame predict() ACTIVE at
// (time, time, time_delta) (ElasticFusion.cpp:387; its fill-in and dense count are left out: only the front half reads this prediction,
// and the end-of-frame predict() rewrites all of it) and the INACTIVE prediction at (0, time - time_delta, time_delta)
static int camera_loop_predict(EfContext* ctx, EfCamera* c, int time) {
  const EfCameraConfig& k = c->cfg;
  PredictTarget p = camera_predict_target(c);
  p.image = c->image;
  p.vertex = c->vertex;
  p.normal = c->normal;
  p.time = c->time;
  RC(map_predict_target_async(ctx, p, k.max_depth, k.conf_threshold, time, time, k.time_delta));
  p.image = c->loop.old_image;
  p.vertex = c->loop.old_vertex;
  p.normal = c->loop.old_normal;
  p.time = c->loop.old_time;
  return map_predict_target_async(ctx, p, k.max_depth, k.conf_threshold, 0, time - k.time_delta, k.time_delta);
}

// close_loops = 1, on a fused frame after the first: the predictions, the front half and the closure at `time`. The result's pose
// becomes the closed one. *n_nodes: the graph the camera's clean applies.
static int camera_close_loop(EfContext* ctx, EfCamera* c, int time, EfCameraResult* result, int* n_nodes) {
  RC(camera_loop_predict(ctx, c, time));
  const LoopSide s = camera_loop_side(c);
  RC(loop_front_half(ctx, s));
  RC(loop_solve_apply(ctx, s, time, c->pose, &c->deform_out, n_nodes));
  if (c->deform_out.applied)
    CU(cudaMemcpyAsync(result->T_wc, ctx->odom[c->slot].gn->T_wc, sizeof(double) * 16, cudaMemcpyDeviceToDevice, ctx->stream));
  return 0;
}

// The steps of a camera frame, which the camera's own frames and a rig's frames share.
// a has_pose T_wc into the camera's dev_T, staged once the previous frame's copy has read the pinned slot (not the whole stream)
static int camera_stage_pose(EfContext* ctx, EfCamera* c, const double* T_wc) {
  CU(cudaEventSynchronize(c->pose_sent));
  memcpy(c->pin_T, T_wc, sizeof(double) * 16);
  CU(cudaMemcpyAsync(c->dev_T, c->pin_T, sizeof(double) * 16, cudaMemcpyHostToDevice, ctx->stream));
  CU(cudaEventRecord(c->pose_sent, ctx->stream));
  return 0;
}

// the live side at the camera (ElasticFusion.cpp:278-285)
static int camera_live(EfContext* ctx, EfCamera* c, const uint8_t* rgb, const uint16_t* depth, bool from_host) {
  const EfCameraConfig& k = c->cfg;
  const LiveBuffers live = {c->rgb, c->rgba, c->depth_raw, c->depth_filtered, c->target.depth_metric, c->target.depth_metric_filtered};
  return track_live_side(ctx, c->slot, live, rgb, depth, true, from_host ? cudaMemcpyHostToDevice : cudaMemcpyDeviceToDevice, k.depth_cutoff,
                         k.max_depth);
}

// the pose of an untracked frame: dev_T, with the weighting
static int camera_set_pose(EfContext* ctx, EfCamera* c, float weight_multiplier) {
  const int which = c->slot;
  if (!c->has_frame) {
    // initFirstRGB: this intensity pyramid is the next frame's previous one. The pose is set with itself as the previous pose (the
    // second k_set_pose), so that the weighting is weight_multiplier.
    OdomDev& od = ctx->odom[which];
    for (int i = 0; i < NUM_PYRS; ++i) std::swap(od.nextImage[i], od.lastNextImage[i]);
    RC(odom_set_pose_async(ctx, which, c->dev_T));
  }
  RC(odom_set_pose_async(ctx, which, c->dev_T));
  return odom_finish_async(ctx, which, weight_multiplier, false, c->pose);
}

// what the camera tracks against: its own prediction of its previous frame, or its fill-in
static ModelInputs camera_model_inputs(const EfCamera* c) {
  return {c->vertex, c->normal, c->fill_vertex, c->fill_normal, c->image, c->fill_image, c->dense_count, c->cfg.frame_to_frame_rgb != 0, c->rgba};
}

// the camera's result (before predict() recounts the dense samples) into out_dev, or its own; returns where it went
static EfCameraResult* camera_result(EfContext* ctx, EfCamera* c, bool tracked, EfCameraResult* out_dev) {
  const EfCameraConfig& k = c->cfg;
  EfCameraResult* result = out_dev ? out_dev : c->result;
  EF_LAUNCH(ctx, k_camera_result, 1, 32, 0, (const GNState*)ctx->odom[c->slot].gn, (const int*)c->dense_count, k.height, k.width, tracked ? 1 : 0,
            result);
  return result;
}

// the map half at `time` (ElasticFusion.cpp:536-585), with the graph of n_nodes nodes the camera's closure left
static int camera_map_half(EfContext* ctx, EfCamera* c, int time, int n_nodes) {
  const EfCameraConfig& k = c->cfg;
  const MapTarget& t = c->target;
  RC(map_predict_indices_async(ctx, t, time, k.max_depth, k.time_delta));
  RC(map_fuse_async(ctx, t, time, k.max_depth, -1.0f));
  RC(map_predict_indices_async(ctx, t, time, k.max_depth, k.time_delta));
  if (n_nodes > 0) {  // ElasticFusion.cpp:559-569: the time-stamp refresh of deformed surfels reads this depth
    PredictTarget d = camera_predict_target(c);
    d.depth = c->loop.synth_depth;
    RC(map_predict_target_async(ctx, d, k.max_depth, k.conf_threshold, time, time - k.time_delta, 65535));
  }
  return map_clean_async(ctx, t, time, k.conf_threshold, k.time_delta, k.max_depth, n_nodes);
}

// predict() with fill-in at `time` (ElasticFusion.cpp:621-653): the model the camera's next frame tracks against
static int camera_predict(EfContext* ctx, EfCamera* c, int time) {
  const EfCameraConfig& k = c->cfg;
  PredictTarget p = camera_predict_target(c);
  p.image = c->image;
  p.vertex = c->vertex;
  p.normal = c->normal;
  p.time = c->time;
  p.dense_count = c->dense_count;
  p.fill_depth = c->depth_filtered;
  p.fill_rgb = c->rgb;
  p.fill_pass_img = k.frame_to_frame_rgb ? 1 : 0;
  p.fill_image = c->fill_image;
  p.fill_vertex = c->fill_vertex;
  p.fill_normal = c->fill_normal;
  return map_predict_target_async(ctx, p, k.max_depth, k.conf_threshold, time, time, k.time_delta);
}

// ElasticFusion::processFrame (reloc = false) at the camera: live side, pose (set, or tracked against the camera's own prediction with
// its fill-in choice, SO(3) and frameToFrameRGB), weighting, with close_loops the local loop closure (camera_close_loop), map half at
// f->time, predict() and, with close_loops, the graph sampled from the map the call leaves (:593)
int camera_frame_async(EfContext* ctx, EfCamera* c, const EfCameraFrame* f, const uint8_t* rgb, const uint16_t* depth, bool from_host,
                       EfCameraResult* out_dev) {
  const EfCameraConfig& k = c->cfg;
  if (f->has_pose) RC(camera_stage_pose(ctx, c, f->T_wc));
  RC(camera_live(ctx, c, rgb, depth, from_host));
  const bool tracked = c->has_frame && !f->has_pose;
  const bool map_half = f->fuse && !k.rgb_only;
  const bool front_half = k.close_loops && map_half && c->has_frame;
  if (!tracked)
    RC(camera_set_pose(ctx, c, f->weight_multiplier));
  else
    RC(track_solve(ctx, c->slot, camera_model_inputs(c), k.rgb_only != 0, k.icp_weight, k.pyramid != 0, k.fast_odom != 0, k.so3 != 0,
                   f->weight_multiplier, c->pose));
  EfCameraResult* result = camera_result(ctx, c, tracked, out_dev);
  memset(&c->deform_out, 0, sizeof(c->deform_out));
  int n_nodes = 0;
  if (front_half) RC(camera_close_loop(ctx, c, f->time, result, &n_nodes));
  if (map_half) RC(camera_map_half(ctx, c, f->time, n_nodes));
  RC(camera_predict(ctx, c, f->time));
  if (k.close_loops) RC(map_sample_graph_async(ctx));
  c->has_frame = true;
  CHECK_LAST();
  return 0;
}

int camera_read(EfContext* ctx, EfCamera* c, EfCameraResult* out, EfSolveTrace* trace, int max_trace, int* n_trace) {
  int trace_n = 0;
  CU(cudaMemcpyAsync(out, c->result, sizeof(EfCameraResult), cudaMemcpyDeviceToHost, ctx->stream));
  CU(cudaMemcpyAsync(&trace_n, (const char*)ctx->odom[c->slot].gn + offsetof(GNState, trace_n), sizeof(int), cudaMemcpyDeviceToHost,
                     ctx->stream));
  CU(cudaStreamSynchronize(ctx->stream));
  const int n = out->tracked ? (trace_n < max_trace ? trace_n : max_trace) : 0;
  if (n_trace) *n_trace = n;
  if (n > 0) {
    CU(cudaMemcpyAsync(trace, ctx->odom[c->slot].trace, sizeof(EfSolveTrace) * n, cudaMemcpyDeviceToHost, ctx->stream));
    CU(cudaStreamSynchronize(ctx->stream));
  }
  return 0;
}

// ---- rigs (ef_rig_*): cameras tracked as one rigid body ----------------------------------------------------------------------
// Ad(T) of a rigid T = [R | p] in the (t, w) order of computeUpdateSE3: [[R, [p]x R], [0, R]], row-major 6x6
static void rig_adjoint(const double* T, double* Ad) {
  const double R[9] = {T[0], T[1], T[2], T[4], T[5], T[6], T[8], T[9], T[10]}, p[3] = {T[3], T[7], T[11]};
  const double px[9] = {0, -p[2], p[1], p[2], 0, -p[0], -p[1], p[0], 0};
  for (int k = 0; k < 36; ++k) Ad[k] = 0;
  for (int r = 0; r < 3; ++r)
    for (int c = 0; c < 3; ++c) {
      double pr = 0;
      for (int k = 0; k < 3; ++k) pr += px[r * 3 + k] * R[k * 3 + c];
      Ad[r * 6 + c] = R[r * 3 + c];
      Ad[r * 6 + 3 + c] = pr;
      Ad[(3 + r) * 6 + 3 + c] = R[r * 3 + c];
    }
}

// the rig's device block (host's extrinsics), its result, the ticket of a joint SO(3) pre-alignment and, for a closing rig, its loop
// record and concatenated constraint buffers
static int rig_alloc(EfContext* ctx, EfRig* r, const RigDev& host) {
  CU(arena_alloc(ctx, r->arena, &r->dev, 1));
  CU(arena_alloc(ctx, r->arena, &r->result, 1, 0));
  CU(cudaMemcpyAsync(r->dev, &host, sizeof(host), cudaMemcpyHostToDevice, ctx->stream));
  if (r->joint_so3) CU(arena_alloc(ctx, r->arena, &r->so3_ticket, 1, 0));
  if (r->closing) {
    CU(arena_alloc(ctx, r->arena, &r->loop, 1, 0));
    CU(arena_alloc(ctx, r->arena, &r->loop_rec, 1, 0));
    CU(arena_alloc(ctx, r->arena, &r->src, 3 * (size_t)r->capacity, 0));
    CU(arena_alloc(ctx, r->arena, &r->dst, 3 * (size_t)r->capacity, 0));
    CU(arena_alloc(ctx, r->arena, &r->times, (size_t)r->capacity, 0));
  }
  CU(cudaStreamSynchronize(ctx->stream));
  return 0;
}

int rig_create(EfContext* ctx, const EfRigConfig* cfg, EfRig** out) {
  int slot = 0;
  while (slot < EF_MAX_CAMERAS && ctx->rigs[slot]) ++slot;
  if (slot == EF_MAX_CAMERAS) return EF_ESTATE;  // (cannot happen: every rig holds a camera of its own)
  EfRig* r = new (std::nothrow) EfRig();
  if (!r) return EF_ENOMEM;
  r->n = cfg->n;
  RigDev host = {};
  for (int m = 0; m < r->n; ++m) {
    r->cams[m] = cfg->cameras[m];
    memcpy(r->T_0i[m], cfg->T_0i[m], sizeof(double) * 16);
    memcpy(host.T_0i[m], cfg->T_0i[m], sizeof(double) * 16);
    efm::se3_inverse(host.T_0i[m], host.T_i0[m]);
    rig_adjoint(host.T_i0[m], host.Ad[m]);
  }
  r->closing = r->cams[0]->cfg.close_loops != 0;  // (ef_rig_create checks that every member agrees)
  r->joint_so3 = cfg->joint_so3 != 0;
  for (int m = 0; m < r->n && r->closing; ++m) r->capacity += r->cams[m]->loop.capacity;
  int rc = rig_alloc(ctx, r, host);
  if (rc) {
    r->arena.release();
    delete r;
    if (rc != (int)cudaErrorMemoryAllocation) return rc;
    cudaGetLastError();  // (an allocation failure is not sticky: the context stays usable)
    return EF_ENOMEM;
  }
  for (int m = 0; m < r->n; ++m) r->cams[m]->rig = r;
  ctx->rigs[slot] = r;
  *out = r;
  return 0;
}

void rig_destroy(EfContext* ctx, EfRig* r) {
  cudaStreamSynchronize(ctx->stream);
  for (int m = 0; m < r->n; ++m) r->cams[m]->rig = nullptr;
  for (EfRig*& q : ctx->rigs)
    if (q == r) q = nullptr;
  r->arena.release();
  delete r;
}

static RigArgs rig_args(const EfContext* ctx, const EfRig* r) {
  RigArgs R = {};
  R.n = r->n;
  for (int m = 0; m < r->n; ++m) {
    const OdomDev& od = ctx->odom[r->cams[m]->slot];
    R.gn[m] = od.gn;
    R.trace[m] = od.trace;
    R.K_levels[m] = od.K_levels;
    R.pose[m] = r->cams[m]->pose;
  }
  R.dev = r->dev;
  return R;
}

// A closing rig's local loop closure on a fused frame after its first: every member's predictions as a closing camera makes them; each
// member's loop tracker set up as loop_front_half sets it up; one joint model-to-model registration over the loop trackers (no pose
// records) and its finish, so T_est_i = T_est_0 * T_0i; the joint acceptance test and the members' constraints; the closure at `time`
// with member 0 as the side whose pose it sets, then member i's pose T_w0 * T_0i. The results' poses become the closed ones.
// *n_nodes: the graph member 0's clean applies.
static int rig_close_loop(EfContext* ctx, EfRig* r, int time, EfCameraResult* const* results, EfRigResult* rig_result, int* n_nodes) {
  const int n = r->n;
  int slots[EF_MAX_CAMERAS];
  RigArgs L = {};
  L.n = n;
  L.dev = r->dev;
  RigLoopArgs a = {};
  a.n = n;
  a.dev = r->dev;
  a.loop = r->loop;
  a.rec = r->loop_rec;
  a.src = r->src;
  a.dst = r->dst;
  a.times = r->times;
  a.capacity = r->capacity;
  for (int m = 0; m < n; ++m) RC(camera_loop_predict(ctx, r->cams[m], time));
  for (int m = 0; m < n; ++m) {
    const LoopSide s = camera_loop_side(r->cams[m]);
    RC(loop_tracker_inputs(ctx, s));
    const OdomDev& od = ctx->odom[s.est];
    slots[m] = s.est;
    L.gn[m] = od.gn;
    L.trace[m] = od.trace;
    L.K_levels[m] = od.K_levels;
    a.curr[m] = ctx->odom[s.curr].gn;
    a.est[m] = od.gn;
    a.vertex[m] = s.vertex;
    a.old_time[m] = s.old_time;
    a.rows[m] = s.rows;
    a.cols[m] = s.cols;
    a.max_depth[m] = s.max_depth;
  }
  const EfCameraConfig& k = r->cams[0]->cfg;
  RC(rig_track_async(ctx, slots, L, 10.0f, k.pyramid != 0, k.fast_odom != 0, false, nullptr));
  RC(rig_finish_async(ctx, L, 1.0f));
  RC(map_rig_loop_constraints_async(ctx, a));
  LoopSide s = {};  // what loop_solve_apply reads: the record, the constraints and member 0's tracker
  s.curr = r->cams[0]->slot;
  s.loop = r->loop;
  s.src = r->src;
  s.dst = r->dst;
  s.times = r->times;
  s.capacity = r->capacity;
  RC(loop_solve_apply(ctx, s, time, r->cams[0]->pose, &r->deform_out, n_nodes));
  if (!r->deform_out.applied) return 0;
  RC(rig_apply_pose_async(ctx, rig_args(ctx, r)));
  for (int m = 0; m < n; ++m)
    CU(cudaMemcpyAsync(results[m]->T_wc, ctx->odom[r->cams[m]->slot].gn->T_wc, sizeof(double) * 16, cudaMemcpyDeviceToDevice, ctx->stream));
  CU(cudaMemcpyAsync(rig_result->T_wc, ctx->odom[r->cams[0]->slot].gn->T_wc, sizeof(double) * 16, cudaMemcpyDeviceToDevice, ctx->stream));
  return 0;
}

// one rig frame: every member's live side; the pose set (member i at T_wc * T_0i) or tracked jointly from every member's model inputs;
// the results; a closing rig's loop closure (rig_close_loop); every member's map half in member order; every member's predict() and,
// for a closing rig, the graph sampled from the map the call leaves
int rig_frame_async(EfContext* ctx, EfRig* r, const EfRigFrame* f, const uint8_t* const* rgb, const uint16_t* const* depth, bool from_host,
                    EfCameraResult* members_dev, EfRigResult* out_dev) {
  const int n = r->n;
  const bool front_half = r->closing && f->fuse && r->has_frame;
  if (r->closing) {  // the record ef_rig_loop_result reads describes this call
    RC(map_loop_reset_async(ctx, r->loop));
    CU(cudaMemsetAsync(r->loop_rec, 0, sizeof(RigLoopDev), ctx->stream));
  }
  if (f->has_pose)
    for (int m = 0; m < n; ++m) {
      double T[16];
      efm::mul4(f->T_wc, r->T_0i[m], T);
      RC(camera_stage_pose(ctx, r->cams[m], T));
    }
  for (int m = 0; m < n; ++m) RC(camera_live(ctx, r->cams[m], rgb[m], depth[m], from_host));
  const bool tracked = r->has_frame && !f->has_pose;
  const RigArgs R = rig_args(ctx, r);
  if (!tracked) {
    for (int m = 0; m < n; ++m) RC(camera_set_pose(ctx, r->cams[m], f->weight_multiplier));
  } else {
    // (the members share icp_weight, pyramid, fast_odom and so3: ef_rig_create checks it)
    const EfCameraConfig& k = r->cams[0]->cfg;
    int slots[EF_MAX_CAMERAS];
    ModelInputs mi[EF_MAX_CAMERAS];
    float* saved[EF_MAX_CAMERAS][NUM_PYRS];
    int rc = 0, ready = 0;
    for (; ready < n && !rc; ++ready) {
      slots[ready] = r->cams[ready]->slot;
      mi[ready] = camera_model_inputs(r->cams[ready]);
      rc = track_model_side(ctx, slots[ready], mi[ready], saved[ready]);
    }
    if (!rc) rc = rig_track_async(ctx, slots, R, k.icp_weight, k.pyramid != 0, k.fast_odom != 0, k.so3 != 0, r->joint_so3 ? r->so3_ticket : nullptr);
    for (int m = 0; m < ready; ++m) track_model_restore(ctx, slots[m], mi[m], saved[m]);
    RC(rc);
    RC(rig_finish_async(ctx, R, f->weight_multiplier));
  }
  EfCameraResult* results[EF_MAX_CAMERAS];
  for (int m = 0; m < n; ++m) results[m] = camera_result(ctx, r->cams[m], tracked, members_dev ? members_dev + m : nullptr);
  EfRigResult* rig_result = out_dev ? out_dev : r->result;
  EF_LAUNCH(ctx, k_rig_result, 1, 32, 0, (const GNState*)R.gn[0], tracked ? 1 : 0, rig_result);
  memset(&r->deform_out, 0, sizeof(r->deform_out));
  int n_nodes = 0;
  if (front_half) RC(rig_close_loop(ctx, r, f->time, results, rig_result, &n_nodes));
  if (f->fuse)  // (only member 0's clean applies the graph: the map is deformed once)
    for (int m = 0; m < n; ++m) RC(camera_map_half(ctx, r->cams[m], f->time, m == 0 ? n_nodes : 0));
  for (int m = 0; m < n; ++m) {
    RC(camera_predict(ctx, r->cams[m], f->time));
    r->cams[m]->has_frame = true;
  }
  if (r->closing) RC(map_sample_graph_async(ctx));
  r->has_frame = true;
  CHECK_LAST();
  return 0;
}

int rig_read(EfContext* ctx, EfRig* r, EfCameraResult* members, EfRigResult* out, EfSolveTrace* trace, int max_trace, int* n_trace) {
  int tn[EF_MAX_CAMERAS] = {};
  for (int m = 0; m < r->n; ++m) {
    CU(cudaMemcpyAsync(&members[m], r->cams[m]->result, sizeof(EfCameraResult), cudaMemcpyDeviceToHost, ctx->stream));
    CU(cudaMemcpyAsync(&tn[m], (const char*)ctx->odom[r->cams[m]->slot].gn + offsetof(GNState, trace_n), sizeof(int), cudaMemcpyDeviceToHost,
                       ctx->stream));
  }
  CU(cudaMemcpyAsync(out, r->result, sizeof(EfRigResult), cudaMemcpyDeviceToHost, ctx->stream));
  CU(cudaStreamSynchronize(ctx->stream));
  for (int m = 0; m < r->n; ++m) {
    const int k = out->tracked ? (tn[m] < max_trace ? tn[m] : max_trace) : 0;
    if (n_trace) n_trace[m] = k;
    if (k > 0)
      CU(cudaMemcpyAsync(trace + (size_t)m * max_trace, ctx->odom[r->cams[m]->slot].trace, sizeof(EfSolveTrace) * k, cudaMemcpyDeviceToHost,
                         ctx->stream));
  }
  CU(cudaStreamSynchronize(ctx->stream));
  return 0;
}

}  // namespace ef
