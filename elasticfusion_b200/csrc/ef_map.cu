// Mapping half of the hot path: the reference's OpenGL/GLSL surfel pipeline (Core/GlobalModel.cpp, Core/IndexMap.cpp,
// Core/Shaders/*.{vert,geom,frag}) rewritten as CUDA kernels over a device-resident surfel structure-of-arrays.
// No OpenGL, no interop: rasterisation is an atomicMin z-buffer on packed (depth24 << 32 | primitive id) keys, which
// reproduces GL_LESS with "earlier primitive wins on ties"; transform feedback is an order-preserving compaction
// driven by a single-pass decoupled look-back scan; the per-surfel "update map" render target (3 x 3072^2 RGBA32F,
// cleared every frame, GlobalModel.cpp:375-378) becomes a 4-byte-per-surfel winner slot touched only by matches.
//
// GL semantics encoded (SURVEY.md App. B), pinned by executing the reference's shader files on Mesa llvmpipe (oracle/gl):
// nearest sampling texel = clamp(floor(coord*size)); window coordinates snapped to 1/256 px; 1-px points cover the pixel whose
// centre lies in the half-open unit square around the snapped position, clipped by centre; point sprites cover the pixel centres
// in the half-open square of their size, size clamped to [1, 2047]; window depth round(z * (2^24-1)); fragments at depth 1.0
// fail GL_LESS against the clear value.
#include <float.h>
#include <stddef.h>

#include <new>
#include <type_traits>

#include "ef_device.cuh"
#include "ef_dmath.cuh"
#include "ef_internal.h"

using namespace ef;

namespace {

constexpr unsigned long long kEmptyKey = ~0ull;
constexpr int SCAN_THREADS = 256, SCAN_ITEMS = 8, SCAN_TILE = SCAN_THREADS * SCAN_ITEMS;

struct Cam {
  float cx, cy, fx, fy;
};

// inputs and outputs of the fill-in (k_fill_in, or mode 0 of k_splat_resolve) and the lit-sample count of denseEnough
struct FillOut {
  const uint16_t* raw_depth;
  const uint8_t* rgb;
  int pass_geom, pass_img;
  float4* vertex;
  float4* normal;
  uchar4* image;
  int* dense_count;
};

__device__ __forceinline__ int texel(float coord, int n) {
  int i = (int)floorf(coord * (float)n);
  return i < 0 ? 0 : (i >= n ? n - 1 : i);
}
// host-side uv buffer value of the reference (GlobalModel.cpp:109-117): (float)i/(float)n + 1.0/(2*(float)n), stored as float
__device__ __forceinline__ float uv_coord(int i, int n) { return (float)((double)((float)i / (float)n) + 1.0 / (double)(2 * (float)n)); }

// color.glsl:19-34
__device__ __forceinline__ float encode_color_bytes(unsigned r, unsigned g, unsigned b) {
  int rgb = (int)r;
  rgb = (rgb << 8) + (int)g;
  rgb = (rgb << 8) + (int)b;
  return (float)rgb;
}
__device__ __forceinline__ float encode_color(const f3& c) {
  int rgb = (int)roundf(c.x * 255.0f);
  rgb = (rgb << 8) + (int)roundf(c.y * 255.0f);
  rgb = (rgb << 8) + (int)roundf(c.z * 255.0f);
  return (float)rgb;
}
__device__ __forceinline__ f3 decode_color(float c) {
  const int ci = (int)c;
  return mk3((float)(ci >> 16 & 0xFF) / 255.0f, (float)(ci >> 8 & 0xFF) / 255.0f, (float)(ci & 0xFF) / 255.0f);
}
// surfels.glsl:19-46
__device__ __forceinline__ float get_radius(float depth, float norm_z, float inv_fx, float inv_fy) {
  const float meanFocal = ((1.0f / fabsf(inv_fx)) + (1.0f / fabsf(inv_fy))) / 2.0f;
  const float sqrt2 = 1.41421356237f;
  const float radius = (depth / meanFocal) * sqrt2;
  float radius_n = radius / fabsf(norm_z);
  radius_n = gmin(2.0f * radius, radius_n);
  return radius_n;
}
__device__ __forceinline__ float confidence(float x, float y, float weighting, float cx, float cy) {
  const float maxRadDist = 400;
  const float twoSigmaSquared = 0.72f;
  const float px = x - cx, py = y - cy;
  const float radialDist = sqrtf(px * px + py * py) / maxRadDist;
  return expf((-(radialDist * radialDist) / twoSigmaSquared)) * weighting;
}
// geometry.glsl:21-40 (float depth sampler, clamp-to-edge)
__device__ __forceinline__ f3 vertex_f(const float* depth, int rows, int cols, int ix, int iy, float x, float y, const Cam& c, float ifx,
                                       float ify) {
  ix = ix < 0 ? 0 : (ix >= cols ? cols - 1 : ix);
  iy = iy < 0 ? 0 : (iy >= rows ? rows - 1 : iy);
  const float z = depth[(size_t)iy * cols + ix];
  return mk3((x - c.cx) * z * ifx, (y - c.cy) * z * ify, z);
}
__device__ __forceinline__ f3 normal_central(const float* depth, int rows, int cols, int ix, int iy, float x, float y, const f3& vPos,
                                             const Cam& c, float ifx, float ify) {
  const f3 xf = vertex_f(depth, rows, cols, ix + 1, iy, x + 1, y, c, ifx, ify);
  const f3 xb = vertex_f(depth, rows, cols, ix - 1, iy, x - 1, y, c, ifx, ify);
  const f3 yf = vertex_f(depth, rows, cols, ix, iy + 1, x, y + 1, c, ifx, ify);
  const f3 yb = vertex_f(depth, rows, cols, ix, iy - 1, x, y - 1, c, ifx, ify);
  const f3 del_x = mk3((xb.x + vPos.x) / 2 - (xf.x + vPos.x) / 2, (xb.y + vPos.y) / 2 - (xf.y + vPos.y) / 2,
                       (xb.z + vPos.z) / 2 - (xf.z + vPos.z) / 2);
  const f3 del_y = mk3((yb.x + vPos.x) / 2 - (yf.x + vPos.x) / 2, (yb.y + vPos.y) / 2 - (yf.y + vPos.y) / 2,
                       (yb.z + vPos.z) / 2 - (yf.z + vPos.z) / 2);
  return normalized(cross(del_x, del_y));
}
// measurement geometry of pixel (i, j) of the reference's uv buffer (vertex_feedback.vert, data.vert): texel centre (tcx, tcy),
// pixel position (x, y) and the vertex of the raw depth; add_filtered() adds the vertex of the filtered depth and its
// normal_central at the same position
struct PixelGeom {
  int i, j;
  float tcx, tcy, x, y;
  f3 v_raw, v_filt, n_filt;
};
__device__ __forceinline__ PixelGeom pixel_geom(const float* depth_raw, int rows, int cols, const Cam& c, float ifx, float ify, int i, int j) {
  PixelGeom g;
  g.i = i;
  g.j = j;
  g.tcx = uv_coord(i, cols);
  g.tcy = uv_coord(j, rows);
  g.x = g.tcx * (float)cols;
  g.y = g.tcy * (float)rows;
  g.v_raw = vertex_f(depth_raw, rows, cols, i, j, g.x, g.y, c, ifx, ify);
  return g;
}
__device__ __forceinline__ void add_filtered(PixelGeom& g, const float* depth_filt, int rows, int cols, const Cam& c, float ifx, float ify) {
  g.v_filt = vertex_f(depth_filt, rows, cols, g.i, g.j, g.x, g.y, c, ifx, ify);
  g.n_filt = normal_central(depth_filt, rows, cols, g.i, g.j, g.x, g.y, g.v_filt, c, ifx, ify);
}
// geometry.glsl:42-60 (ushort mm sampler, integer pixel coords)
__device__ __forceinline__ f3 vertex_u(const uint16_t* depth, int rows, int cols, int ix, int iy, int x, int y, const Cam& c, float ifx,
                                       float ify) {
  ix = ix < 0 ? 0 : (ix >= cols ? cols - 1 : ix);
  iy = iy < 0 ? 0 : (iy >= rows ? rows - 1 : iy);
  const float z = (float)depth[(size_t)iy * cols + ix] / 1000.0f;
  return mk3(((float)x - c.cx) * z * ifx, ((float)y - c.cy) * z * ify, z);
}
// GL rasterises in fixed point: window coordinates are snapped to 1/256 pixel (GL_SUBPIXEL_BITS = 8 on Mesa llvmpipe and on NVIDIA
// GPUs), the pixel-centre offset removed first. A size-1 point then covers the pixel whose centre lies in the half-open unit
// square around the snapped coordinate, a sprite the pixels whose centres lie in the half-open square of its (snapped) size.
// Pinned by running the reference's index_map / splat shaders on Mesa (oracle/gl, tests/golden/ref_mapping_*.npz).
__device__ __forceinline__ int snap256(float w) { return __float2int_rn((w - 0.5f) * 256.0f); }
__device__ __forceinline__ int point_pixel(float w) { return (snap256(w) + 127) >> 8; }
__device__ __forceinline__ void sprite_range(float w, float size, int& p0, int& p1) {
  int fw = __float2int_rn(size * 256.0f);
  if (fw < 256) fw = 256;
  const int x0 = snap256(w) - fw / 2;
  p0 = (x0 + 255) >> 8;
  p1 = ((x0 + fw + 255) >> 8) - 1;
}
__device__ __forceinline__ unsigned int depth24(float zw) {
  if (!(zw > 0.f)) zw = 0.f;
  if (zw > 1.f) zw = 1.f;
  return (unsigned int)rintf(zw * 16777215.0f);
}
// vertex stage of index_map.vert / splat.vert for a camera-space point h: projection to normalised device coordinates,
// the frustum test (false: clipped) and the window coordinates xw, yw with the NDC depth zn
__device__ __forceinline__ bool gl_vertex(const Cam& c, int rows, int cols, float max_depth, const f3& h, float& xw, float& yw, float& zn) {
  const float fcols = (float)cols, frows = (float)rows;
  const float xn = ((((c.fx * h.x) / h.z) + c.cx) - (fcols * 0.5f)) / (fcols * 0.5f);
  const float yn = ((((c.fy * h.y) / h.z) + c.cy) - (frows * 0.5f)) / (frows * 0.5f);
  zn = h.z / max_depth;
  if (!(xn >= -1.f && xn <= 1.f && yn >= -1.f && yn <= 1.f && zn >= -1.f && zn <= 1.f)) return false;
  xw = (xn + 1.0f) * (fcols * 0.5f);
  yw = (yn + 1.0f) * (frows * 0.5f);
  return true;
}


// The reference walks a 4x4 sample window with float loop counters (data.vert:132-160, copy_unstable.vert:75-111):
//   for (float i = c - 2*step; i < c + 2*step; i += step)   with step = half a texel, nearest sampling.
// The samples are monotone and half a texel apart, so they land on at most three consecutive texels t0, t0+1, t0+2, some of
// them twice. This evaluates the float loop literally once per axis (it runs 4 times, 5 when rounding leaves the accumulated
// counter just short of the bound) and returns the first texel with how many samples hit each of the three. No array is
// indexed dynamically (registers only).
struct WinAxis {
  int t0;
  int m[3];
};
__device__ __forceinline__ WinAxis window_axis(float centre, float step, int n) {
  WinAxis A;
  const float lo = centre - (1.0f * step * 2.0f), hi = centre + (1.0f * step * 2.0f);
  A.t0 = texel(lo, n);
  A.m[0] = A.m[1] = A.m[2] = 0;
  float i = lo;
#pragma unroll
  for (int k = 0; k < 6; ++k) {
    if (i < hi) {
      const int d = texel(i, n) - A.t0;
      A.m[0] += (d == 0);
      A.m[1] += (d == 1);
      A.m[2] += (d >= 2);
    }
    i += step;
  }
  return A;
}
// The index map (index_map.vert/.frag). A pass of k_index_scatter leaves one key per texel in `keys`: [63:56] the pass's tag,
// [55:32] window depth d24, [31:0] surfel id. Tags count down from 0xfe, one per pass, and the host re-arms the buffer (all
// 0xff) before they run out, so a key of the current pass is smaller than every key an earlier pass left: atomicMin still picks
// the nearest surfel, the lower id on ties, and no pass has to clear the buffer. A texel is occupied iff its key carries the
// current tag. The textures (EF_BUF_INDEX, VERT_CONF, COLOR_TIME, NORM_RAD) are written from the keys by write_index_texels:
// by the stage API's pass itself, and by the frame's clean for the frame's passes. Inside a frame the map does not change
// between an index pass and its reader (fuse writes only after k_fuse_associate, clean moves surfels only after
// k_clean_flags), so there fuse and clean read the keys and the surfels they name; otherwise (TEX) they read the textures,
// which a stage-API caller may have uploaded or may have changed the map under.
struct IndexMap {
  const unsigned long long* keys;
  unsigned int tag;
  uint32_t* index;
  float4 *vert_conf, *col_time, *norm_rad;
};
__device__ __forceinline__ bool key_live(unsigned long long key, unsigned int tag) { return (unsigned int)(key >> 56) == tag; }
// texel attributes of a surfel: camera-space vertex + confidence, camera-space unit normal + radius (colour + time is copied)
template <typename M>
__device__ __forceinline__ float4 index_vert_conf(M t_inv, const float4& pc) {
  const f3 h = xform(t_inv, mk3(pc.x, pc.y, pc.z));
  return make_float4(h.x, h.y, h.z, pc.w);
}
__device__ __forceinline__ float4 index_norm_rad(const float* t_inv, const float4& nr) {
  const f3 nn = normalized(rot(t_inv, mk3(nr.x, nr.y, nr.z)));
  return make_float4(nn.x, nn.y, nn.z, nr.w);
}
// the textures of texels first, first + stride, ... < n_px; an empty texel is all zeros
__device__ __forceinline__ void write_index_texels(const IndexMap& ix, const MapPose* __restrict__ mp, const float4* __restrict__ pos_conf,
                                                   const float4* __restrict__ color_time, const float4* __restrict__ norm_rad, int n_px,
                                                   int first, int stride) {
  for (int p = first; p < n_px; p += stride) {
    const unsigned long long key = ix.keys[p];
    if (!key_live(key, ix.tag)) {
      ix.index[p] = 0;
      ix.vert_conf[p] = ix.col_time[p] = ix.norm_rad[p] = make_float4(0.f, 0.f, 0.f, 0.f);
      continue;
    }
    const uint32_t id = (uint32_t)key;
    const float4 pc = pos_conf[id], nr = norm_rad[id];
    ix.index[p] = id;
    ix.vert_conf[p] = index_vert_conf(mp->t_inv, pc);
    ix.col_time[p] = color_time[id];
    ix.norm_rad[p] = index_norm_rad(mp->t_inv, nr);
  }
}
// the surfel ids of the window spanned by two axes, cur[3 * x + y] (x outer, y inner, ascending); texels no sample lands on,
// and empty texels, read as 0 (as in the reference, surfel 0 is never a match)
template <bool TEX>
__device__ __forceinline__ void window_index(const IndexMap& ix, int cols, const WinAxis& ax, const WinAxis& ay, uint32_t (&cur)[9]) {
#pragma unroll
  for (int ia = 0; ia < 3; ++ia)
#pragma unroll
    for (int jb = 0; jb < 3; ++jb) {
      cur[ia * 3 + jb] = 0u;
      if (ax.m[ia] > 0 && ay.m[jb] > 0) {
        const int p = (ay.t0 + jb) * cols + (ax.t0 + ia);
        if (TEX) {
          cur[ia * 3 + jb] = ix.index[p];
        } else {
          const unsigned long long key = ix.keys[p];
          cur[ia * 3 + jb] = key_live(key, ix.tag) ? (uint32_t)key : 0u;
        }
      }
    }
}

// ---------------------------------------------------------------------------------------------------------------
// pose upload: T_wc (double) -> float pose and float inverse, as the shader uniforms (GlobalModel.cpp:405,562)
// ---------------------------------------------------------------------------------------------------------------
__global__ void k_update_pose(MapPose* mp, const double* T) {
  pdl_enter();
  if (threadIdx.x != 0 || blockIdx.x != 0) return;
  double inv[16];
  efm::se3_inverse(T, inv);
  for (int k = 0; k < 16; ++k) {
    mp->pose[k] = (float)T[k];
    mp->t_inv[k] = (float)inv[k];
  }
}

// ---------------------------------------------------------------------------------------------------------------
// single-pass exclusive scan of byte flags (decoupled look-back), persistent CTAs, device-resident length
// ---------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(SCAN_THREADS) k_scan_flags(const uint8_t* __restrict__ flags, const int* __restrict__ n_a,
                                                              const int* __restrict__ n_b, int* __restrict__ offsets,
                                                              unsigned long long* state, unsigned int* counter, int* total_out,
                                                              unsigned int epoch) {
  // tile states: see lookback_prefix; the tile dispenser (counter[0]) is reset by the last CTA to leave (dispenser_exit)
  pdl_enter();
  const int n = (n_a ? *n_a : 0) + (n_b ? *n_b : 0);
  const int num_tiles = (n + SCAN_TILE - 1) / SCAN_TILE;
  __shared__ int s_warp[SCAN_THREADS / 32];
  __shared__ int s_tile, s_prefix;
  if (num_tiles == 0) {
    if (blockIdx.x == 0 && threadIdx.x == 0 && total_out) *total_out = 0;
    return;
  }
  while (true) {
    if (threadIdx.x == 0) s_tile = (int)atomicAdd(counter, 1u);
    __syncthreads();
    const int tile = s_tile;
    if (tile >= num_tiles) {
      if (threadIdx.x == 0) dispenser_exit<false>(counter);  // every CTA has drawn its terminating ticket: re-arm for the next scan
      return;
    }
    const int base = tile * SCAN_TILE + threadIdx.x * SCAN_ITEMS;
    int v[SCAN_ITEMS], sum = 0;
#pragma unroll
    for (int k = 0; k < SCAN_ITEMS; ++k) {
      const int i = base + k;
      v[k] = (i < n) ? (flags[i] ? 1 : 0) : 0;
      sum += v[k];
    }
    int aggregate;
    const int thread_excl = block_exclusive_scan<SCAN_THREADS>(sum, s_warp, aggregate);
    if (threadIdx.x < 32) {
      const int prefix = lookback_prefix(state, tile, 0, 0, aggregate, epoch);
      if (threadIdx.x == 0) {
        s_prefix = prefix;
        if (tile == num_tiles - 1 && total_out) *total_out = prefix + aggregate;
      }
    }
    __syncthreads();
    int run = s_prefix + thread_excl;
#pragma unroll
    for (int k = 0; k < SCAN_ITEMS; ++k) {
      const int i = base + k;
      if (i < n) offsets[i] = run;
      run += v[k];
    }
    __syncthreads();
  }
}

// ---------------------------------------------------------------------------------------------------------------
// first frame: vertex_feedback.vert/.geom + init_unstable.vert (FeedbackBuffer.cpp:81-138, GlobalModel.cpp:229-284)
// ---------------------------------------------------------------------------------------------------------------
__global__ void k_feedback_flags(const float* __restrict__ depth_raw, const float* __restrict__ depth_filt, int rows, int cols,
                                 float max_depth, uint8_t* __restrict__ f_raw, uint8_t* __restrict__ f_filt) {
  pdl_enter();
  const int n = rows * cols;
  for (int d = blockIdx.x * blockDim.x + threadIdx.x; d < n; d += gridDim.x * blockDim.x) {
    const int i = d / rows, j = d - i * rows;  // draw order: x-major
    const float zr = depth_raw[(size_t)j * cols + i], zf = depth_filt[(size_t)j * cols + i];
    f_raw[d] = !(zr <= 0 || zr > max_depth);
    f_filt[d] = !(zf <= 0 || zf > max_depth);
  }
}

__global__ void k_init_scatter(const uint8_t* __restrict__ rgb, const float* __restrict__ depth_raw, const float* __restrict__ depth_filt,
                               int rows, int cols, Cam c, int time, const uint8_t* __restrict__ f_raw, const uint8_t* __restrict__ f_filt,
                               const int* __restrict__ off_raw, const int* __restrict__ off_filt, const int* __restrict__ raw_total,
                               int capacity, float4* __restrict__ pos_conf, float4* __restrict__ color_time, float4* __restrict__ norm_rad,
                               int* __restrict__ count) {
  pdl_enter();
  const float ifx = 1.0f / c.fx, ify = 1.0f / c.fy;
  const int n = rows * cols;
  if (blockIdx.x == 0 && threadIdx.x == 0) *count = min(*raw_total, capacity);
  for (int d = blockIdx.x * blockDim.x + threadIdx.x; d < n; d += gridDim.x * blockDim.x) {
    const int i = d / rows, j = d - i * rows;
    if (f_raw[d]) {
      const int k = off_raw[d];
      if (k < capacity) {
        const PixelGeom g = pixel_geom(depth_raw, rows, cols, c, ifx, ify, i, j);
        const uint8_t* px = rgb + ((size_t)j * cols + i) * 3;
        pos_conf[k] = make_float4(g.v_raw.x, g.v_raw.y, g.v_raw.z, confidence(g.x, g.y, 1.0f, c.cx, c.cy));
        // init_unstable.vert: colour.y = 0 (unused), colour.z = 1 (init time); colour.w = time from vertex_feedback.vert
        color_time[k] = make_float4(encode_color_bytes(px[0], px[1], px[2]), 0.f, 1.f, (float)time);
      }
    }
    if (f_filt[d]) {
      const int k = off_filt[d];
      if (k < capacity) {
        PixelGeom g = pixel_geom(depth_raw, rows, cols, c, ifx, ify, i, j);  // (the raw vertex goes unused here)
        add_filtered(g, depth_filt, rows, cols, c, ifx, ify);
        norm_rad[k] = make_float4(g.n_filt.x, g.n_filt.y, g.n_filt.z, get_radius(g.v_filt.z, g.n_filt.z, ifx, ify));
      }
    }
  }
}

// ---------------------------------------------------------------------------------------------------------------
// index map: index_map.vert/.frag (IndexMap.cpp:190-258)
// ---------------------------------------------------------------------------------------------------------------
// MODE 0: every surfel of the map. MODE 1: the same, and every surfel that reaches the z-buffer stage is appended to `vis`
// (unordered; warp-aggregated). MODE 2: only the surfels listed in `vis` are visited.
// The frame loop renders the index map twice with identical arguments, before and after fuse (IndexMap::predictIndices,
// ElasticFusion.cpp:536-556). Fuse only writes surfels it found THROUGH the first index map, i.e. surfels in `vis`; every other
// surfel is bit-for-bit what it was and fails (or cannot win differently in) the second pass exactly as it did in the first, and
// new surfels join the map only in clean. So the second pass over `vis` -- each entry re-tested with its updated state --
// produces the identical index map while reading the in-view part of the map instead of all of it.
template <int MODE>
__global__ void __launch_bounds__(256, 5) k_index_scatter(const float4* __restrict__ pos_conf, const float4* __restrict__ color_time,
                                                          const int* __restrict__ count, const MapPose* __restrict__ mp, int time, float max_depth,
                                                          int time_delta, int rows, int cols, Cam c, unsigned long long* __restrict__ keys,
                                                          unsigned int tag, uint32_t* __restrict__ vis, int* __restrict__ vis_count,
                                                          int vis_capacity) {
  pdl_enter();
  const int n_map = *count;
  const int n = (MODE == 2) ? min(*vis_count, vis_capacity) : n_map;
  // Two surfels per thread and round, in three phases -- 4 loads, 2 projections + 2 z-buffer reads, <= 2 atomics -- so that a
  // thread has independent requests in flight instead of a chain of three (one surfel at a time: 40 us for 5 M surfels,
  // long-scoreboard 20 per issue at 39 % of the DRAM roof). One resident wave of 5 CTAs per SM (<= 51 registers); a small map
  // still gives every thread at most one round.
  constexpr int U = 2;
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  const int stride = gridDim.x * blockDim.x;
  __shared__ int s_vis[256 / 32 + 1];
  for (int bbase = blockIdx.x * blockDim.x; bbase < n; bbase += U * stride) {  // (CTA-uniform bound: the append below synchronises)
    float4 pc[U];
    float last_time[U];
    int ids[U];
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const int i = bbase + threadIdx.x + u * stride;
      ids[u] = -1;
      if (i < n) {
        const int id = (MODE == 2) ? (int)vis[i] : i;
        if (id < n_map) {
          ids[u] = id;
          pc[u] = pos_conf[id];
          last_time[u] = color_time[id].w;
        }
      }
    }
    unsigned long long key[U], cur[U];
    unsigned long long* slot[U];
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const int id = ids[u];
      slot[u] = nullptr;
      if (id < 0) continue;
      const f3 h = xform(mp->t_inv, mk3(pc[u].x, pc[u].y, pc[u].z));
      if (h.z > max_depth || h.z < 0) continue;
      if ((float)time - last_time[u] > (float)time_delta) continue;
      float xw, yw, zn;
      if (!gl_vertex(c, rows, cols, max_depth, h, xw, yw, zn)) continue;
      const int px = point_pixel(xw), py = point_pixel(yw);
      if (px < 0 || py < 0 || px >= cols || py >= rows) continue;
      const unsigned int d24 = depth24(0.5f * zn + 0.5f);
      if (d24 >= 16777215u) continue;
      key[u] = ((unsigned long long)tag << 56) | ((unsigned long long)d24 << 32) | (unsigned int)id;
      slot[u] = &keys[(size_t)py * cols + px];
      cur[u] = __ldcg(slot[u]);
    }
#pragma unroll
    for (int u = 0; u < U; ++u) {
      if (MODE == 1) {
        // one atomic per CTA and round (one per warp put 8 k of them on a single address for a small map: +6 us)
        const unsigned int m = __ballot_sync(0xffffffffu, slot[u] != nullptr);
        if (lane == 0) s_vis[wid] = __popc(m);
        __syncthreads();
        if (threadIdx.x == 0) {
          int tot = 0;
          for (int w = 0; w < 256 / 32; ++w) {
            const int cw = s_vis[w];
            s_vis[w] = tot;
            tot += cw;
          }
          s_vis[256 / 32] = tot ? atomicAdd(vis_count, tot) : 0;
        }
        __syncthreads();
        const int at = s_vis[256 / 32] + s_vis[wid] + __popc(m & ((1u << lane) - 1u));
        if (slot[u] && at < vis_capacity) vis[at] = (uint32_t)ids[u];
        __syncthreads();
      }
      if (slot[u] && cur[u] > key[u]) atomicMin(slot[u], key[u]);  // (a slot only ever decreases: one that cannot win sends no atomic)
    }
  }
}

// the textures of the last index pass, for a caller of the stage API (the frame's second pass has k_clean_flags write them)
__global__ void k_index_textures(IndexMap ix, const float4* __restrict__ pos_conf, const float4* __restrict__ color_time,
                                 const float4* __restrict__ norm_rad, const MapPose* __restrict__ mp, int n_px) {
  pdl_enter();
  write_index_texels(ix, mp, pos_conf, color_time, norm_rad, n_px, blockIdx.x * blockDim.x + threadIdx.x, gridDim.x * blockDim.x);
}

// ---------------------------------------------------------------------------------------------------------------
// fuse: data.vert/.geom/.frag + update.vert (GlobalModel.cpp:356-525)
// ---------------------------------------------------------------------------------------------------------------
struct FuseArgs {
  const uint8_t* rgb;
  const float* depth_raw;
  const float* depth_filt;
  IndexMap ix;  // (read only)
  int rows, cols;
  Cam c;
  int time;
  float max_depth;
};

// Only pixels with x % 2 == y % 2 == time % 2 take part in a frame (data.vert:112, SURVEY App. A-16): the fuse kernels run
// over that quarter grid. q -> (i, j) keeps the reference's draw order (x-major), so compaction order is unchanged.
struct Quarter {
  int p, ni, nj;
};
__device__ __host__ __forceinline__ Quarter quarter_of(int time, int rows, int cols) {
  Quarter q;
  q.p = ((time % 2) + 2) % 2;
  q.ni = (cols - q.p + 1) / 2;
  q.nj = (rows - q.p + 1) / 2;
  return q;
}

// measurement geometry of pixel (i,j) as data.vert builds it; returns false if the pixel takes no part this frame
__device__ __forceinline__ bool fuse_active(const FuseArgs& a, int i, int j, PixelGeom& g) {
  const float ifx = (float)(1.0 / (double)a.c.fx), ify = (float)(1.0 / (double)a.c.fy);
  g = pixel_geom(a.depth_raw, a.rows, a.cols, a.c, ifx, ify, i, j);
  const float ftime = (float)a.time;
  if (!((int)g.x % 2 == (int)ftime % 2 && (int)g.y % 2 == (int)ftime % 2)) return false;
  const int il = max(i - 1, 0), ir = min(i + 1, a.cols - 1), ju = max(j - 1, 0), jd = min(j + 1, a.rows - 1);
  if (a.depth_raw[(size_t)j * a.cols + il] == 0 || a.depth_raw[(size_t)ju * a.cols + i] == 0 ||
      a.depth_raw[(size_t)j * a.cols + ir] == 0 || a.depth_raw[(size_t)jd * a.cols + i] == 0)
    return false;
  return (g.v_raw.z > 0 && g.v_raw.z <= a.max_depth);
}

constexpr uint32_t ASSOC_NONE = 0xffffffffu, ASSOC_NEW = 0xfffffffeu;

template <bool TEX>
__global__ void k_fuse_associate(FuseArgs a, const MapPose* __restrict__ mp, const float4* __restrict__ pos_conf,
                                 const float4* __restrict__ norm_rad, const int* __restrict__ count, uint32_t* __restrict__ assoc,
                                 uint32_t* __restrict__ pending) {
  pdl_enter();
  const Quarter Q = quarter_of(a.time, a.rows, a.cols);
  const int nq = Q.ni * Q.nj;
  const int cnt = *count;
  for (int q = blockIdx.x * blockDim.x + threadIdx.x; q < nq; q += gridDim.x * blockDim.x) {
    const int i = 2 * (q / Q.nj) + Q.p, j = 2 * (q % Q.nj) + Q.p;
    const uint32_t d = (uint32_t)i * a.rows + j;  // draw index in the reference's uv buffer
    PixelGeom g;
    uint32_t res = ASSOC_NONE;
    if (fuse_active(a, i, j, g)) {
      const float ifx = (float)(1.0 / (double)a.c.fx), ify = (float)(1.0 / (double)a.c.fy);
      add_filtered(g, a.depth_filt, a.rows, a.cols, a.c, ifx, ify);
      const f3 vNormLocal = g.n_filt;
      const float fcols = (float)a.cols, frows = (float)a.rows;
      int counter = 0;
      uint32_t best = 0;
      const float scale = 1.0f;  // IndexMap::FACTOR
      const float indexXStep = (1.0f / (fcols * scale)) * 0.5f;
      const float indexYStep = (1.0f / (frows * scale)) * 0.5f;
      float bestDist = 1000;
      const float xl = (g.x - a.c.cx) * ifx;
      const float yl = (g.y - a.c.cy) * ify;
      const float lambda = sqrtf(xl * xl + yl * yl + 1);
      const f3 ray = mk3(xl, yl, 1);
      // duplicates of a texel cannot change the outcome (strict `dist < bestDist`), so each distinct texel is visited once,
      // in the reference's order (x outer, y inner, ascending). All nine index texels are fetched first, then the attributes
      // of the occupied ones column by column: four dependent memory round trips instead of one or two per texel.
      const WinAxis ax = window_axis(g.tcx, indexXStep, a.cols), ay = window_axis(g.tcy, indexYStep, a.rows);
      uint32_t cur[9];
      window_index<TEX>(a.ix, a.cols, ax, ay, cur);
#pragma unroll
      for (int ia = 0; ia < 3; ++ia) {
        float4 vc[3], nr[3];
#pragma unroll
        for (int jb = 0; jb < 3; ++jb) {
          const uint32_t id = cur[ia * 3 + jb];
          if (id > 0U) {
            const int p = (ay.t0 + jb) * a.cols + (ax.t0 + ia);
            vc[jb] = TEX ? a.ix.vert_conf[p] : pos_conf[id];
            nr[jb] = TEX ? a.ix.norm_rad[p] : norm_rad[id];
          }
        }
#pragma unroll
        for (int jb = 0; jb < 3; ++jb)
          if (!TEX && cur[ia * 3 + jb] > 0U) {
            vc[jb] = index_vert_conf(mp->t_inv, vc[jb]);
            nr[jb] = index_norm_rad(mp->t_inv, nr[jb]);
          }
#pragma unroll
        for (int jb = 0; jb < 3; ++jb) {
          const uint32_t current = cur[ia * 3 + jb];
          if (current > 0U) {
            if (fabsf((vc[jb].z * lambda) - (g.v_raw.z * lambda)) < 0.05f) {
              const float dist = norm(cross(ray, mk3(vc[jb].x, vc[jb].y, vc[jb].z))) / norm(ray);
              const f3 nrm = mk3(nr[jb].x, nr[jb].y, nr[jb].z);
              const float ang = acosf(dot(nrm, vNormLocal) / (norm(nrm) * norm(vNormLocal)));
              if (dist < bestDist && (fabsf(nr[jb].z) < 0.75f || fabsf(ang) < 0.5f)) {
                counter++;
                bestDist = dist;
                best = current;
              }
            }
          }
        }
      }
      if (counter > 0) {
        res = best;
        if ((int)best < cnt) atomicMin(&pending[best], d);  // lowest draw index wins the update-map texel
      } else {
        res = ASSOC_NEW;
      }
    }
    assoc[q] = res;
  }
}

__device__ __forceinline__ void fuse_measurement(const FuseArgs& a, const MapPose* mp, float weighting, int i, int j, float4& pos, float4& col,
                                                 float4& nr) {
  const float ifx = (float)(1.0 / (double)a.c.fx), ify = (float)(1.0 / (double)a.c.fy);
  PixelGeom g = pixel_geom(a.depth_raw, a.rows, a.cols, a.c, ifx, ify, i, j);
  const f3 vg = xform(mp->pose, g.v_raw);
  add_filtered(g, a.depth_filt, a.rows, a.cols, a.c, ifx, ify);
  const f3 ng = rot(mp->pose, g.n_filt);
  const uint8_t* px = a.rgb + ((size_t)j * a.cols + i) * 3;
  pos = make_float4(vg.x, vg.y, vg.z, confidence(g.x, g.y, weighting, a.c.cx, a.c.cy));
  col = make_float4(encode_color_bytes(px[0], px[1], px[2]), 0.f, (float)a.time, 0.f);
  nr = make_float4(ng.x, ng.y, ng.z, get_radius(g.v_filt.z, g.n_filt.z, ifx, ify));
}

// one associated pixel q of the quarter grid: a new surfel goes to new_*[k_new]; the pixel that owns a matched surfel's winner slot
// fuses its measurement into it (update.vert:49-84)
__device__ __forceinline__ void fuse_update_item(const FuseArgs& a, const MapPose* __restrict__ mp, float weighting, int cnt, const Quarter& Q, int q,
                                                 uint32_t as, int k_new, uint32_t* __restrict__ pending, float4* __restrict__ pos_conf,
                                                 float4* __restrict__ color_time, float4* __restrict__ norm_rad, float4* __restrict__ new_pos,
                                                 float4* __restrict__ new_col, float4* __restrict__ new_nr) {
  const int i = 2 * (q / Q.nj) + Q.p, j = 2 * (q % Q.nj) + Q.p;
  const uint32_t d = (uint32_t)i * a.rows + j;
  float4 mpos, mcol, mnr;
  if (as == ASSOC_NEW) {
    fuse_measurement(a, mp, weighting, i, j, mpos, mcol, mnr);
    mcol.w = -2.f;
    new_pos[k_new] = mpos;
    new_col[k_new] = mcol;
    new_nr[k_new] = mnr;
    return;
  }
  if ((int)as >= cnt || pending[as] != d) return;
  pending[as] = 0xffffffffu;  // re-arm the slot: exactly one pixel owns it
  fuse_measurement(a, mp, weighting, i, j, mpos, mcol, mnr);
  const float4 s_pos = pos_conf[as], s_col = color_time[as], s_nr = norm_rad[as];
  const float c_k = s_pos.w, aw = mpos.w;
  if (mnr.w < (1.0f + 0.5f) * s_nr.w) {
    const float ck_a = c_k + aw;
    pos_conf[as] = make_float4(((c_k * s_pos.x) + (aw * mpos.x)) / ck_a, ((c_k * s_pos.y) + (aw * mpos.y)) / ck_a,
                               ((c_k * s_pos.z) + (aw * mpos.z)) / ck_a, ck_a);
    const f3 oldCol = decode_color(s_col.x), newCol = decode_color(mcol.x);
    const f3 avg = mk3(((c_k * oldCol.x) + (aw * newCol.x)) / ck_a, ((c_k * oldCol.y) + (aw * newCol.y)) / ck_a,
                       ((c_k * oldCol.z) + (aw * newCol.z)) / ck_a);
    color_time[as] = make_float4(encode_color(avg), s_col.y, s_col.z, (float)a.time);
    f3 nn = mk3(((c_k * s_nr.x) + (aw * mnr.x)) / ck_a, ((c_k * s_nr.y) + (aw * mnr.y)) / ck_a, ((c_k * s_nr.z) + (aw * mnr.z)) / ck_a);
    const float rr = ((c_k * s_nr.w) + (aw * mnr.w)) / ck_a;
    nn = normalized(nn);
    norm_rad[as] = make_float4(nn.x, nn.y, nn.z, rr);
  } else {
    pos_conf[as] = make_float4(s_pos.x, s_pos.y, s_pos.z, c_k + aw);
    color_time[as] = make_float4(s_col.x, s_col.y, s_col.z, (float)a.time);
  }
}

// A persistent grid over tiles of FU_THREADS quarter-grid pixels, drawn in order from the dispenser counter[0]: the new surfels
// of a tile take their slots in new_* from the tile's exclusive prefix (lookback_prefix), so they keep the draw order without a
// separate scan; the last tile publishes the number of new surfels.
constexpr int FU_THREADS = 128;
__global__ void __launch_bounds__(FU_THREADS) k_fuse_update(FuseArgs a, const MapPose* __restrict__ mp, const float* __restrict__ weighting_p,
                                                            const int* __restrict__ count, const uint32_t* __restrict__ assoc,
                                                            uint32_t* __restrict__ pending, float4* __restrict__ pos_conf,
                                                            float4* __restrict__ color_time, float4* __restrict__ norm_rad,
                                                            float4* __restrict__ new_pos, float4* __restrict__ new_col, float4* __restrict__ new_nr,
                                                            int* __restrict__ new_count, unsigned long long* state, unsigned int* counter,
                                                            unsigned int epoch) {
  pdl_enter();
  const Quarter Q = quarter_of(a.time, a.rows, a.cols);
  const int nq = Q.ni * Q.nj;
  const int num_tiles = (nq + FU_THREADS - 1) / FU_THREADS;
  const int cnt = *count;
  const float weighting = *weighting_p;
  __shared__ int s_warp[FU_THREADS / 32];
  __shared__ int s_tile, s_prefix;
  while (true) {
    if (threadIdx.x == 0) s_tile = (int)atomicAdd(counter, 1u);
    __syncthreads();
    const int tile = s_tile;
    if (tile >= num_tiles) {
      if (threadIdx.x == 0) dispenser_exit<false>(counter);
      return;
    }
    const int q = tile * FU_THREADS + threadIdx.x;
    const uint32_t as = (q < nq) ? assoc[q] : ASSOC_NONE;
    int aggregate;
    const int excl = block_exclusive_scan<FU_THREADS>(as == ASSOC_NEW ? 1 : 0, s_warp, aggregate);
    if (threadIdx.x < 32) {
      const int prefix = lookback_prefix(state, tile, 0, 0, aggregate, epoch);
      if (threadIdx.x == 0) {
        s_prefix = prefix;
        if (tile == num_tiles - 1) *new_count = prefix + aggregate;
      }
    }
    __syncthreads();
    if (as != ASSOC_NONE)
      fuse_update_item(a, mp, weighting, cnt, Q, q, as, s_prefix + excl, pending, pos_conf, color_time, norm_rad, new_pos, new_col, new_nr);
    __syncthreads();  // s_tile and s_prefix are rewritten by the next draw
  }
}

// ---------------------------------------------------------------------------------------------------------------
// clean: copy_unstable.vert/.geom without deformation graph (GlobalModel.cpp:527-671)
// ---------------------------------------------------------------------------------------------------------------
struct CleanArgs {
  IndexMap ix;
  int rows, cols;
  Cam c;
  int time;
  float conf_threshold;
  int time_delta;
  // deformation graph (copy_unstable.vert:132-322); n_nodes == 0: none
  const float* nodes;   // 16 floats per node: position 3, rotation 9 (column-major), translation 3, time
  int n_nodes;
  const float* depth;   // IndexMap::depthTex() (synthesizeDepth), read by the time-stamp refresh
  float max_depth;
  int is_fern;
};

// copy_unstable.vert:132-322. The surfel is moved by the weighted rigid motions of the k = 4 nearest of the <= 20 graph nodes
// around its init time (binary search on the node time stamps: 10 back, then forward up to 20 in total), its normal by the
// inverse-transpose rotations; a stable surfel that lands in front of (or < 10 cm behind) the synthesised model depth gets
// lastTime = time. GLSL pow(x, 2) is x * x here (x >= 0 for the k nearest); texel fetches of the node texture (nearest, clamp to
// edge) are array reads with the index clamped at 0.
__device__ __noinline__ void deform_surfel(const CleanArgs& a, const MapPose* mp, float4& pos, float4& col, float4& nr) {
  constexpr int k = 4, lookBack = 20;
  int nearNodes[lookBack];
  float nearDists[lookBack];
#pragma unroll
  for (int i = 0; i < lookBack; i++) {
    nearNodes[i] = -1;
    nearDists[i] = 16777216.0f;
  }
  const float* __restrict__ nodes = a.nodes;
  const int n_nodes = a.n_nodes;
  const int poseTime = (int)col.z;
  int foundIndex = 0;
  int imin = 0, imax = n_nodes - 1, imid = (imin + imax) / 2;
  while (imax >= imin) {
    imid = (imin + imax) / 2;
    const int nodeTime = (int)nodes[(size_t)imid * 16 + 15];
    if (nodeTime < poseTime)
      imin = imid + 1;
    else if (nodeTime > poseTime)
      imax = imid - 1;
    else
      break;
  }
  imin = min(imin, n_nodes - 1);
  const int nodeMin = (int)nodes[(size_t)imin * 16 + 15], nodeMid = (int)nodes[(size_t)imid * 16 + 15],
            nodeMax = (int)nodes[(size_t)max(imax, 0) * 16 + 15];
  if (abs(nodeMin - poseTime) <= abs(nodeMid - poseTime) && abs(nodeMin - poseTime) <= abs(nodeMax - poseTime))
    foundIndex = imin;
  else if (abs(nodeMid - poseTime) <= abs(nodeMin - poseTime) && abs(nodeMid - poseTime) <= abs(nodeMax - poseTime))
    foundIndex = imid;
  else
    foundIndex = imax;
  if (foundIndex == n_nodes) foundIndex = n_nodes - 1;
  const f3 v = mk3(pos.x, pos.y, pos.z);
  int nearNodeIndex = 0, distanceBack = 0;
  for (int j = foundIndex; j >= 0; j--) {
    const f3 d = v - mk3(nodes[(size_t)j * 16], nodes[(size_t)j * 16 + 1], nodes[(size_t)j * 16 + 2]);
    nearNodes[nearNodeIndex] = j;
    nearDists[nearNodeIndex] = sqrtf(dot(d, d));
    nearNodeIndex++;
    if (++distanceBack == lookBack / 2) break;
  }
  for (int j = foundIndex + 1; j < n_nodes; j++) {
    const f3 d = v - mk3(nodes[(size_t)j * 16], nodes[(size_t)j * 16 + 1], nodes[(size_t)j * 16 + 2]);
    nearNodes[nearNodeIndex] = j;
    nearDists[nearNodeIndex] = sqrtf(dot(d, d));
    nearNodeIndex++;
    if (++distanceBack == lookBack) break;
  }
  for (int i = 0; i < lookBack - 1; ++i)
    for (int j = i + 1; j < lookBack; ++j)
      if (nearDists[j] < nearDists[i]) {
        const float t = nearDists[i];
        nearDists[i] = nearDists[j];
        nearDists[j] = t;
        const int t2 = nearNodes[i];
        nearNodes[i] = nearNodes[j];
        nearNodes[j] = t2;
      }
  const float dMax = nearDists[k];
  float w[k], wsum = 0;
  for (int j = 0; j < k; j++) {
    const float* nd = nodes + (size_t)max(nearNodes[j], 0) * 16;
    const f3 d = v - mk3(nd[0], nd[1], nd[2]);
    const float b = 1.0f - (sqrtf(dot(d, d)) / dMax);
    w[j] = b * b;
    wsum += w[j];
  }
  for (int j = 0; j < k; j++) w[j] /= wsum;
  f3 newPos = mk3(0, 0, 0), newNorm = mk3(0, 0, 0);
  const f3 nrm = mk3(nr.x, nr.y, nr.z);
  for (int i = 0; i < k; i++) {
    const float* nd = nodes + (size_t)max(nearNodes[i], 0) * 16;
    const f3 position = mk3(nd[0], nd[1], nd[2]);
    const f3 c0 = mk3(nd[3], nd[4], nd[5]), c1 = mk3(nd[6], nd[7], nd[8]), c2 = mk3(nd[9], nd[10], nd[11]);
    const f3 translation = mk3(nd[12], nd[13], nd[14]);
    const f3 d = v - position;
    const f3 rd = mk3(c0.x * d.x + c1.x * d.y + c2.x * d.z, c0.y * d.x + c1.y * d.y + c2.y * d.z, c0.z * d.x + c1.z * d.y + c2.z * d.z);
    newPos = newPos + ((rd + position) + translation) * w[i];
    const f3 k0 = cross(c1, c2), k1 = cross(c2, c0), k2 = cross(c0, c1);  // cofactors: transpose(inverse(R)) = cof(R) / det(R)
    const float det = dot(c0, k0);
    const f3 tn = mk3((k0.x * nrm.x + k1.x * nrm.y + k2.x * nrm.z) / det, (k0.y * nrm.x + k1.y * nrm.y + k2.y * nrm.z) / det,
                      (k0.z * nrm.x + k1.z * nrm.y + k2.z * nrm.z) / det);
    newNorm = newNorm + tn * w[i];
  }
  pos.x = newPos.x;
  pos.y = newPos.y;
  pos.z = newPos.z;
  const f3 nn = normalized(newNorm);
  nr.x = nn.x;
  nr.y = nn.y;
  nr.z = nn.z;
  if (pos.w > a.conf_threshold && a.is_fern == 0) {
    const f3 lp = xform(mp->t_inv, newPos);
    const float x = ((a.c.fx * lp.x) / lp.z) + a.c.cx, y = ((a.c.fy * lp.y) / lp.z) + a.c.cy;
    if (lp.z > 0 && lp.z < a.max_depth && x > 0 && y > 0 && x < (float)a.cols && y < (float)a.rows) {
      const float currentDepth = a.depth[(size_t)texel(y / (float)a.rows, a.rows) * a.cols + texel(x / (float)a.cols, a.cols)];
      if (currentDepth > 0.0f && lp.z < currentDepth + 0.1f) col.w = (float)a.time;
    }
  }
}

// t_inv_s: the map pose's inverse, in shared memory. The window's surfels are transformed through a volatile view of it: the
// pose is read from shared memory per texel instead of being held in 12 registers across the window.
template <bool TEX>
__device__ __forceinline__ bool clean_test(const CleanArgs& a, const float* t_inv_s, const float4* __restrict__ pos_conf,
                                           const float4* __restrict__ color_time, const float4& pos, float4& col,
                                           const float4* __restrict__ nr_ptr) {
  const float fcols = (float)a.cols, frows = (float)a.rows;
  int test = 1;
  const volatile float* t_inv_v = t_inv_s;
  const f3 localPos = TEX ? xform(t_inv_s, mk3(pos.x, pos.y, pos.z)) : xform(t_inv_v, mk3(pos.x, pos.y, pos.z));
  const float x = ((a.c.fx * localPos.x) / localPos.z) + a.c.cx;
  const float y = ((a.c.fy * localPos.y) / localPos.z) + a.c.cy;
  const float scale = 1.0f;
  const float indexXStep = (1.0f / (fcols * scale)) * 0.5f;
  const float indexYStep = (1.0f / (frows * scale)) * 0.5f;
  int count = 0, zCount = 0;
  if ((float)a.time - col.w < (float)a.time_delta && localPos.z > 0 && x > 0 && y > 0 && x < fcols && y < frows) {
    const float4 nr = *nr_ptr;  // normal + radius: only the surfels in view need them (32 B instead of 48 for the rest)
    const f3 localNorm = normalized(TEX ? rot(t_inv_s, mk3(nr.x, nr.y, nr.z)) : rot(t_inv_v, mk3(nr.x, nr.y, nr.z)));
    // duplicate samples COUNT here (copy_unstable.vert:94,106; SURVEY App. A-19): each distinct texel is read once and
    // weighted by the number of float-loop samples that land on it. Index texels first, attributes of the occupied ones after.
    const WinAxis ax = window_axis(x / fcols, indexXStep, a.cols), ay = window_axis(y / frows, indexYStep, a.rows);
    uint32_t cur[9];
    window_index<TEX>(a.ix, a.cols, ax, ay, cur);
#pragma unroll
    for (int ia = 0; ia < 3; ++ia) {
      float4 vcs[3];
      float2 its[3];  // (init time, last time): the colour half is not read
#pragma unroll
      for (int jb = 0; jb < 3; ++jb) {
        const uint32_t id = cur[ia * 3 + jb];
        if (id > 0U) {
          const int p = (ay.t0 + jb) * a.cols + (ax.t0 + ia);
          vcs[jb] = TEX ? a.ix.vert_conf[p] : pos_conf[id];
          its[jb] = reinterpret_cast<const float2*>(TEX ? a.ix.col_time + p : color_time + id)[1];
        }
      }
#pragma unroll
      for (int jb = 0; jb < 3; ++jb)
        if (!TEX && cur[ia * 3 + jb] > 0U) vcs[jb] = index_vert_conf(t_inv_v, vcs[jb]);
#pragma unroll
      for (int jb = 0; jb < 3; ++jb)
        if (cur[ia * 3 + jb] > 0U) {
          const int m = ax.m[ia] * ay.m[jb];
          const float4 vc = vcs[jb];
          const float2 it = its[jb];
          const float dx = vc.x - localPos.x, dy = vc.y - localPos.y;
          if (it.x < col.z && vc.w > a.conf_threshold && vc.z > localPos.z && vc.z - localPos.z < 0.01f &&
              sqrtf(dx * dx + dy * dy) < nr.w * 1.4f)
            count += m;
          if (it.y == (float)a.time && vc.w > a.conf_threshold && vc.z > localPos.z && vc.z - localPos.z > 0.01f &&
              fabsf(localNorm.z) > 0.85f)
            zCount += m;
        }
    }
  }
  if (count > 8 || zCount > 4) test = 0;
  if (col.w == -2) col.w = (float)a.time;
  if (col.w == -1 || (((float)a.time - col.w) > 20 && pos.w < a.conf_threshold)) test = 0;
  if (col.w > 0 && (float)a.time - col.w > (float)a.time_delta) test = 1;
  return test > 0;
}

// ---- TMA-style 1-D bulk copies (cp.async.bulk, SASS UBLKCP) + mbarrier, used to stage surfel tiles in shared memory ----
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
// global -> shared copy of 8 or 16 bytes that holds no register while in flight (cp.async, completed by cp_async_wait)
template <int BYTES>
__device__ __forceinline__ void cp_async(void* dst_smem, const void* src_gmem) {
  asm volatile("cp.async.ca.shared.global [%0], [%1], %2;" ::"r"(smem_u32(dst_smem)), "l"(src_gmem), "n"(BYTES) : "memory");
}
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_all;" ::: "memory"); }
__device__ __forceinline__ void mbar_init(unsigned long long* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_fence_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void mbar_expect_tx(unsigned long long* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(unsigned long long* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok != 0;
}
// global -> shared, `bytes` a multiple of 16, both addresses 16-byte aligned; completion is signalled on `bar` (complete_tx)
__device__ __forceinline__ void bulk_g2s(void* dst_smem, const void* src_gmem, uint32_t bytes, unsigned long long* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(dst_smem)),
               "l"(src_gmem), "r"(bytes), "r"(smem_u32(bar))
               : "memory");
}

// clean in TWO launches (copy_unstable.vert + transform feedback, GlobalModel.cpp:527-671):
//  k_clean_flags  the keep / cull test of every surfel (old map + this frame's new ones), embarrassingly parallel at full
//                 occupancy: 32 B read per surfel (48 for those in view) and ONE BIT written (a warp ballot per 32 surfels). It
//                 also finds the first tile that has to move: the first one that lost a surfel or holds a new one.
//  k_clean_move   the order-preserving compaction + append, IN PLACE, over the tiles from that first mover on only -- the old,
//                 stable bulk of a map sorted by init time is neither read nor written again. Single-pass decoupled look-back
//                 over tiles of CC_TILE surfels:
//  * persistent CTAs draw tiles from a dispenser; each tile (3 x 8 KB of float4, or its old-map / new-surfel parts) is
//    staged in shared memory by 1-D bulk copies (cp.async.bulk + mbarrier complete_tx), double buffered;
//  * tile t publishes its aggregate only after its input is resident in shared memory, and a tile learns its output offset
//    only from the published states of all its predecessors -- so when it writes [prefix, prefix + kept), which lies inside
//    the input ranges of tiles <= t, every one of those has already been read. Surfels that do not move are not written;
//  * the last CTA to leave publishes the new count and clears the new-surfel count (GlobalModel.cpp:667-670).
// (One fused launch was measured first: in-view tiles take ~10x longer than the rest and the look-back makes every tile wait
// for the slowest tile in flight, 267 us at 5 M surfels; split, the test runs unordered and the ordered part touches little.)
constexpr int CC_THREADS = 256, CC_ITEMS = 2, CC_TILE = CC_THREADS * CC_ITEMS;
struct CcStage {
  float4 pos[CC_TILE], col[CC_TILE], nr[CC_TILE];
};
struct CcShared {
  CcStage st[2];
  unsigned long long bar[2];
  int warp_cnt[CC_ITEMS * (CC_THREADS / 32)];
  int warp_excl[CC_ITEMS * (CC_THREADS / 32)];
  int next_tile, prefix, aggregate;
};

constexpr int CC_WORDS = CC_ITEMS * (CC_THREADS / 32);  // keep-mask words per tile, in (item slab k, warp) order

// ctl[0] tile dispenser, ctl[1] exit tickets, ctl[2] first tile that moves (0xffffffff: none)
constexpr int CF_THREADS = CC_TILE;  // one surfel per thread: the window test is a chain of ~5 dependent gathers, so two surfels per
                                     // thread would double the latency of a small map's pass (27 -> 14 us at 270 k surfels)
// write_tex: the index textures are still to be written from the keys (the frame's passes leave that to this kernel, which
// runs before k_clean_move moves a surfel); reset_count: the visible list the frame's index passes used, re-armed here
template <bool TEX>
__global__ void __launch_bounds__(CF_THREADS, 2) k_clean_flags(CleanArgs a, const MapPose* __restrict__ mp, const float4* __restrict__ pos_conf,
                                                               const float4* __restrict__ color_time, const float4* __restrict__ norm_rad,
                                                               const int* __restrict__ count, const float4* __restrict__ new_pos,
                                                               const float4* __restrict__ new_col, const float4* __restrict__ new_nr,
                                                               const int* __restrict__ new_count, uint32_t* __restrict__ keep_mask,
                                                               unsigned int* ctl, int write_tex, int* __restrict__ reset_count) {
  pdl_enter();
  const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  if (reset_count && blockIdx.x == 0 && tid == 0) *reset_count = 0;
  __shared__ float s_tinv[16];
  if (!TEX && tid < 16) s_tinv[tid] = mp->t_inv[tid];
  __syncthreads();
  const int n_old = *count, total = n_old + *new_count;
  const int num_tiles = (total + CC_TILE - 1) / CC_TILE;
  // The next tile's position and (init time, last time) are requested before this tile is tested: two rounds in flight. They
  // are staged in this thread's own shared-memory slot by cp.async, so they hold no registers across the test.
  __shared__ float4 s_pos[CF_THREADS];
  __shared__ float2 s_time[CF_THREADS];
  auto fetch = [&](int t) {
    const int g = t * CC_TILE + tid;
    if (t < num_tiles && g < total) {
      const bool is_old = g < n_old;
      cp_async<16>(&s_pos[tid], is_old ? pos_conf + g : new_pos + (g - n_old));
      cp_async<8>(&s_time[tid], reinterpret_cast<const float2*>(is_old ? color_time + g : new_col + (g - n_old)) + 1);
    }
  };
  fetch(blockIdx.x);
  for (int t = blockIdx.x; t < num_tiles; t += gridDim.x) {
    const int g0 = t * CC_TILE;
    const int n_in = min(CC_TILE, total - g0);
    // a tile moves when it holds new surfels (they have to be appended), lost one of its own, or a graph deforms the map
    bool moves = (g0 + n_in > n_old) || a.n_nodes > 0;
    // thread = item of the tile: warp w holds items 32 w .. 32 w + 31, i.e. keep-mask word w in k_clean_move's (slab, warp) order
    const int g = g0 + tid;
    cp_async_wait();
    const float4 pos = s_pos[tid];
    const float2 it = s_time[tid];
    float4 col = make_float4(0.f, 0.f, it.x, it.y);  // (clean_test reads only the times)
    fetch(t + gridDim.x);
    bool keep = false;
    if (tid < n_in) {
      const bool is_old = g < n_old;
      keep = clean_test<TEX>(a, TEX ? mp->t_inv : s_tinv, pos_conf, color_time, pos, col, is_old ? norm_rad + g : new_nr + (g - n_old));
    }
    const unsigned int ballot = __ballot_sync(0xffffffffu, keep);
    const unsigned int valid = __ballot_sync(0xffffffffu, tid < n_in);
    if (lane == 0) keep_mask[(size_t)t * CC_WORDS + wid] = ballot;
    moves = moves || ballot != valid;
    if (moves && lane == 0) atomicMin(ctl + 2, (unsigned int)t);
  }
  if (!TEX && write_tex)  // (textures that clean reads are already written)
    write_index_texels(a.ix, mp, pos_conf, color_time, norm_rad, a.rows * a.cols, blockIdx.x * CF_THREADS + tid, gridDim.x * CF_THREADS);
}

template <bool DEFORM>
__global__ void __launch_bounds__(CC_THREADS) k_clean_move(CleanArgs a, const MapPose* __restrict__ mp, float4* pos_conf, float4* color_time,
                                                           float4* norm_rad, int* count, const float4* __restrict__ new_pos,
                                                           const float4* __restrict__ new_col, const float4* __restrict__ new_nr,
                                                           int* new_count, int capacity, const uint32_t* __restrict__ keep_mask,
                                                           unsigned long long* state, unsigned int* ctl, int* total_out, unsigned int epoch) {
  pdl_enter();
  extern __shared__ __align__(128) unsigned char cc_smem_raw[];
  CcShared& S = *reinterpret_cast<CcShared*>(cc_smem_raw);
  const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  const int n_old = *count, total = n_old + *new_count;
  const int num_tiles = (total + CC_TILE - 1) / CC_TILE;
  unsigned int* counter = ctl;
  // tiles below `first` are full and stay where they are: the compaction starts there with prefix first * CC_TILE
  const unsigned int first_u = *(volatile unsigned int*)(ctl + 2);
  const int first = first_u > (unsigned int)num_tiles ? num_tiles : (int)first_u;
  if (tid == 0) {
    mbar_init(&S.bar[0], 1);
    mbar_init(&S.bar[1], 1);
    mbar_fence_init();
  }
  __syncthreads();

  // stage tile `t` into buffer `s` (one thread): the part below n_old comes from the map, the rest from the new-surfel arrays
  auto issue = [&](int t, int s) {
    const int g0 = t * CC_TILE;
    const int n_in = min(CC_TILE, total - g0);
    int n_a = n_old - g0;
    n_a = n_a < 0 ? 0 : (n_a > n_in ? n_in : n_a);
    const int n_b = n_in - n_a;
    mbar_expect_tx(&S.bar[s], (uint32_t)n_in * 48u);
    CcStage& st = S.st[s];
    if (n_a > 0) {
      bulk_g2s(st.pos, pos_conf + g0, (uint32_t)n_a * 16u, &S.bar[s]);
      bulk_g2s(st.col, color_time + g0, (uint32_t)n_a * 16u, &S.bar[s]);
      bulk_g2s(st.nr, norm_rad + g0, (uint32_t)n_a * 16u, &S.bar[s]);
    }
    if (n_b > 0) {
      const int b0 = g0 + n_a - n_old;
      bulk_g2s(st.pos + n_a, new_pos + b0, (uint32_t)n_b * 16u, &S.bar[s]);
      bulk_g2s(st.col + n_a, new_col + b0, (uint32_t)n_b * 16u, &S.bar[s]);
      bulk_g2s(st.nr + n_a, new_nr + b0, (uint32_t)n_b * 16u, &S.bar[s]);
    }
  };

  int cur = 0;
  if (tid == 0) {
    cur = first + (int)atomicAdd(counter, 1u);
    S.next_tile = cur;
    if (cur < num_tiles) issue(cur, 0);
  }
  __syncthreads();
  cur = S.next_tile;
  int stage = 0;
  uint32_t parity[2] = {0u, 0u};
  while (cur < num_tiles) {
    __syncthreads();  // S.next_tile has been read by everyone; the other stage's readers (previous iteration) are done
    if (tid == 0) {
      const int nx = first + (int)atomicAdd(counter, 1u);
      S.next_tile = nx;
      if (nx < num_tiles) issue(nx, stage ^ 1);
    }
    while (!mbar_try_wait(&S.bar[stage], parity[stage])) {
    }
    parity[stage] ^= 1u;
    CcStage& st = S.st[stage];
    const int g0 = cur * CC_TILE;
    const int n_in = min(CC_TILE, total - g0);

    // the keep masks k_clean_flags left for this tile; item index k * CC_THREADS + tid keeps the shared-memory reads
    // conflict-free and the order (k, warp, lane) = map order
    unsigned int ballots[CC_ITEMS];
    bool keep[CC_ITEMS];
    unsigned int deformed = 0;  // bit k: item k was moved by the deformation graph (always rewritten)
#pragma unroll
    for (int k = 0; k < CC_ITEMS; ++k) {
      const int idx = k * CC_THREADS + tid;
      ballots[k] = keep_mask[(size_t)cur * CC_WORDS + k * (CC_THREADS / 32) + wid];
      keep[k] = (ballots[k] >> lane) & 1u;
      if (DEFORM && keep[k] && a.n_nodes > 0) {
        float4 col = st.col[idx];
        if (col.w == -2) col.w = (float)a.time;  // copy_unstable.vert:114-117 -- the shader deforms with the refreshed vColor
        if (col.z != (float)a.time) {
          float4 pos = st.pos[idx], nr = st.nr[idx];
          deform_surfel(a, mp, pos, col, nr);
          st.pos[idx] = pos;
          st.col[idx] = col;
          st.nr[idx] = nr;
          deformed |= 1u << k;
        }
      }
      if (lane == 0) S.warp_cnt[k * (CC_THREADS / 32) + wid] = __popc(ballots[k]);
    }
    __syncthreads();
    if (wid == 0) {
      // exclusive scan of the CC_ITEMS x 8 warp counts (one per lane), then the decoupled look-back
      static_assert(CC_ITEMS * (CC_THREADS / 32) <= 32, "one warp scans the slab x warp counts");
      const int c = (lane < CC_ITEMS * (CC_THREADS / 32)) ? S.warp_cnt[lane] : 0;
      int incl = c;
#pragma unroll
      for (int off = 1; off < 32; off <<= 1) {
        const int t = __shfl_up_sync(0xffffffffu, incl, off);
        if (lane >= off) incl += t;
      }
      if (lane < CC_ITEMS * (CC_THREADS / 32)) S.warp_excl[lane] = incl - c;
      const int aggregate = __shfl_sync(0xffffffffu, incl, 31);
      const int prefix = lookback_prefix(state, cur, first, first * CC_TILE, aggregate, epoch);
      if (lane == 0) {
        S.prefix = prefix;
        S.aggregate = aggregate;
        if (cur == num_tiles - 1) *total_out = prefix + aggregate;
      }
    }
    __syncthreads();
    const int prefix = S.prefix;
    // scatter: kept surfels go to prefix + rank. Old surfels that stay where they are are not written.
    if (!(prefix == g0 && S.aggregate == n_in && g0 + n_in <= n_old) || (DEFORM && a.n_nodes > 0)) {
#pragma unroll
      for (int k = 0; k < CC_ITEMS; ++k) {
        if (!keep[k]) continue;
        const int idx = k * CC_THREADS + tid;
        const int g = g0 + idx;
        const int o = prefix + S.warp_excl[k * (CC_THREADS / 32) + wid] + __popc(ballots[k] & ((1u << lane) - 1u));
        if (o >= capacity || (o == g && g < n_old && !(deformed >> k & 1u))) continue;
        float4 col = st.col[idx];
        if (col.w == -2) col.w = (float)a.time;  // copy_unstable.vert:114-117 (only new surfels carry -2)
        pos_conf[o] = st.pos[idx];
        color_time[o] = col;
        norm_rad[o] = st.nr[idx];
      }
    }
    cur = S.next_tile;
    stage ^= 1;
  }
  // leave: the last CTA to draw its terminating ticket re-arms the dispenser and publishes the counts
  if (tid == 0 && dispenser_exit<true>(counter)) {
    counter[2] = 0xffffffffu;
    if (first < num_tiles) {  // (otherwise nothing was culled and nothing is new: the count stands)
      const int kept = *(volatile int*)total_out;
      *count = kept < capacity ? kept : capacity;
    }
    *new_count = 0;
  }
}

// ---------------------------------------------------------------------------------------------------------------
// model raycast: splat.vert + combo_splat.frag / depth_splat.frag (IndexMap.cpp:293-476)
// ---------------------------------------------------------------------------------------------------------------
struct Splat {
  f3 pos;
  float conf;
  f3 nrm;
  float rad;
  float xw, yw, size;
};
struct RayArgs {
  int rows, cols;
  Cam c;
  float max_depth, conf_threshold;
  int time, max_time, time_delta;
};

__device__ __forceinline__ f3 project_image(const Cam& c, const f3& p) { return mk3(((c.fx * p.x) / p.z) + c.cx, ((c.fy * p.y) / p.z) + c.cy, p.z); }

__device__ __forceinline__ bool splat_vertex(const RayArgs& a, const MapPose* mp, const float4& pc, const float4& ct, const float4* norm_rad,
                                             int id, Splat& sp) {
  const f3 h = xform(mp->t_inv, mk3(pc.x, pc.y, pc.z));
  if (h.z > a.max_depth || h.z < 0 || pc.w < a.conf_threshold || (float)a.time - ct.w > (float)a.time_delta || ct.w > (float)a.max_time)
    return false;
  float zn;
  if (!gl_vertex(a.c, a.rows, a.cols, a.max_depth, h, sp.xw, sp.yw, zn)) return false;
  const float4 nr = norm_rad[id];
  sp.pos = h;
  sp.conf = pc.w;
  sp.nrm = normalized(rot(mp->t_inv, mk3(nr.x, nr.y, nr.z)));
  sp.rad = nr.w;
  const f3 x1 = normalized(mk3((sp.nrm.y - sp.nrm.z), -sp.nrm.x, sp.nrm.x)) * sp.rad * 1.41421356f;
  const f3 y1 = cross(sp.nrm, x1);
  const f3 p1 = project_image(a.c, h + x1), p2 = project_image(a.c, h + y1), p3 = project_image(a.c, h - y1), p4 = project_image(a.c, h - x1);
  const float xs0 = gmin(p1.x, gmin(p2.x, gmin(p3.x, p4.x))), xs1 = gmax(p1.x, gmax(p2.x, gmax(p3.x, p4.x)));
  const float ys0 = gmin(p1.y, gmin(p2.y, gmin(p3.y, p4.y))), ys1 = gmax(p1.y, gmax(p2.y, gmax(p3.y, p4.y)));
  const float xDiff = fabsf(xs1 - xs0), yDiff = fabsf(ys1 - ys0);
  float size = gmax(0.f, gmax(xDiff, yDiff));
  if (!(size >= 1.0f)) size = 1.0f;
  if (size > 2047.0f) size = 2047.0f;
  sp.size = size;
  return true;
}

__device__ __forceinline__ bool splat_fragment(const Splat& sp, const Cam& c, int px, int py, f3& corrected) {
  const float fxc = (float)px + 0.5f, fyc = (float)py + 0.5f;
  const f3 l = normalized(mk3((fxc - c.cx) / c.fx, (fyc - c.cy) / c.fy, 1.0f));
  corrected = l * (dot(sp.pos, sp.nrm) / dot(l, sp.nrm));
  const float sqrRad = sp.rad * sp.rad;
  const f3 diff = corrected - sp.pos;
  return !(dot(diff, diff) > sqrRad);
}

// Point-sprite rasterisation, warp-cooperative and load-balanced. The vertex stage runs one surfel per lane (most of a large
// map is culled there: out of the frustum, unstable, outside the time window). The fragments of the warp's surviving sprites
// (side 1 .. 2047 px, so 1 .. 4 M fragments each) are then enumerated as ONE list that all 32 lanes walk together -- fragment
// f belongs to the sprite whose exclusive fragment-count prefix brackets f -- so a single large sprite is rasterised by the
// whole warp and small ones do not leave lanes idle. A fragment that cannot win (the z-buffer already holds a smaller key;
// keys only ever decrease) skips its atomic. The z-buffer result is order independent (atomicMin on depth24 << 32 | id), so
// the image is identical to the serial rasteriser's.
constexpr int SPLAT_THREADS = 256;
struct SplatWarp {
  float4 pr[32];   // pos.xyz, radius
  float4 nz[32];   // normal.xyz, (unused)
  int4 box[32];    // x0, y0, width, surfel id
  int start[33];   // exclusive prefix of the fragment counts
};

__global__ void __launch_bounds__(SPLAT_THREADS, 4) k_splat_scatter(RayArgs a, const MapPose* __restrict__ mp, const float4* __restrict__ pos_conf,
                                                                 const float4* __restrict__ color_time, const float4* __restrict__ norm_rad,
                                                                 const int* __restrict__ count, unsigned long long* __restrict__ zbuf,
                                                                 int* __restrict__ dense_count) {
  pdl_enter();
  if (dense_count && blockIdx.x == 0 && threadIdx.x == 0) *dense_count = 0;  // counted again by this raycast's k_splat_resolve
  __shared__ SplatWarp sw_all[SPLAT_THREADS / 32];
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  SplatWarp& W = sw_all[wid];
  const int n = *count;
  const int gw = blockIdx.x * (SPLAT_THREADS / 32) + wid, nw = gridDim.x * (SPLAT_THREADS / 32);
  // (the next round's position / colour-time records are requested before this round is rasterised: most surfels of a large
  // map are rejected right after the load, so the loop is a chain of round trips unless two rounds are in flight)
  float4 pc_next = make_float4(0.f, 0.f, 0.f, 0.f), ct_next = pc_next;
  if (gw * 32 + lane < n) {
    pc_next = pos_conf[gw * 32 + lane];
    ct_next = color_time[gw * 32 + lane];
  }
  for (int base = gw * 32; base < n; base += nw * 32) {
    const int id = base + lane;
    const float4 pc_cur = pc_next, ct_cur = ct_next;
    {
      const long long nid = (long long)base + (long long)nw * 32 + lane;
      if (nid < n) {
        pc_next = pos_conf[nid];
        ct_next = color_time[nid];
      }
    }
    Splat sp;
    int x0 = 0, y0 = 0, bw = 0, nfrag = 0;
    if (id < n && splat_vertex(a, mp, pc_cur, ct_cur, norm_rad, id, sp)) {
      int x1, y1;
      sprite_range(sp.xw, sp.size, x0, x1);
      sprite_range(sp.yw, sp.size, y0, y1);
      x0 = max(x0, 0);
      y0 = max(y0, 0);
      x1 = min(x1, a.cols - 1);
      y1 = min(y1, a.rows - 1);
      if (x1 >= x0 && y1 >= y0) {
        bw = x1 - x0 + 1;
        nfrag = bw * (y1 - y0 + 1);
      }
    }
    if (!__any_sync(0xffffffffu, nfrag > 0)) continue;
    int incl = nfrag;
#pragma unroll
    for (int off = 1; off < 32; off <<= 1) {
      const int t = __shfl_up_sync(0xffffffffu, incl, off);
      if (lane >= off) incl += t;
    }
    const int total = __shfl_sync(0xffffffffu, incl, 31);
    W.start[lane] = incl - nfrag;
    if (lane == 31) W.start[32] = total;
    if (nfrag > 0) {
      W.pr[lane] = make_float4(sp.pos.x, sp.pos.y, sp.pos.z, sp.rad);
      W.nz[lane] = make_float4(sp.nrm.x, sp.nrm.y, sp.nrm.z, 0.f);
      W.box[lane] = make_int4(x0, y0, bw, id);
    }
    __syncwarp();
    for (int f = lane; f < total; f += 32) {
      // sprite of fragment f: the last s with start[s] <= f (sprites without fragments share their successor's start)
      int s = 0;
#pragma unroll
      for (int step = 16; step > 0; step >>= 1)
        if (W.start[s + step] <= f) s += step;
      const int4 bx = W.box[s];
      const int local = f - W.start[s];
      const int ry = local / bx.z;
      const int px = bx.x + (local - ry * bx.z), py = bx.y + ry;
      const float4 pr = W.pr[s], nz = W.nz[s];
      Splat q;
      q.pos = mk3(pr.x, pr.y, pr.z);
      q.nrm = mk3(nz.x, nz.y, nz.z);
      q.rad = pr.w;
      f3 cp;
      if (!splat_fragment(q, a.c, px, py, cp)) continue;
      const unsigned int d24 = depth24((cp.z / (2 * a.max_depth)) + 0.5f);
      if (d24 >= 16777215u) continue;
      const unsigned long long key = ((unsigned long long)d24 << 32) | (unsigned int)bx.w;
      unsigned long long* slot = &zbuf[(size_t)py * a.cols + px];
      if (__ldcg(slot) <= key) continue;  // cannot win: the slot only ever decreases
      atomicMin(slot, key);
    }
    __syncwarp();
  }
}

// fill_vertex/normal/rgb.frag (FillIn.cpp:62-191) for pixel (x, y) = p, given the predicted vertex, normal and colour there
__device__ __forceinline__ void fill_in_pixel(const FillOut& f, int rows, int cols, const Cam& c, int x, int y, int p, const float4& sv,
                                              const float4& sn, const uchar4& si) {
  const float ifx = 1.0f / c.fx, ify = 1.0f / c.fy;
  if (sv.z == 0 || f.pass_geom == 1) {
    const f3 v = vertex_u(f.raw_depth, rows, cols, x, y, x, y, c, ifx, ify);
    f.vertex[p] = make_float4(v.x, v.y, v.z, 1.f);
  } else {
    f.vertex[p] = sv;
  }
  if (sn.z == 0 || f.pass_geom == 1) {
    const f3 v = vertex_u(f.raw_depth, rows, cols, x, y, x, y, c, ifx, ify);
    const f3 vx = vertex_u(f.raw_depth, rows, cols, x + 1, y, x + 1, y, c, ifx, ify);
    const f3 vy = vertex_u(f.raw_depth, rows, cols, x, y + 1, x, y + 1, c, ifx, ify);
    const f3 nn = normalized(cross(vx - v, vy - v));
    f.normal[p] = make_float4(nn.x, nn.y, nn.z, 1.f);
  } else {
    f.normal[p] = sn;
  }
  if (((int)si.x + (int)si.y + (int)si.z == 0) || f.pass_img == 1)
    f.image[p] = make_uchar4(f.rgb[(size_t)p * 3 + 0], f.rgb[(size_t)p * 3 + 1], f.rgb[(size_t)p * 3 + 2], 255);
  else
    f.image[p] = si;
}

// Resize::image's nearest decimation by DENSE_FACTOR (Resize.cpp:50-79): sample i of n reads texel texel((i + 0.5) / n, size).
// Whether texel x of `size` is one of those samples (consecutive samples are >= DENSE_FACTOR texels apart).
__device__ __forceinline__ bool is_dense_sample(int x, int size) {
  const int n = size / DENSE_FACTOR;
  const int i0 = (int)(((long long)x * n) / size);
  for (int i = max(i0 - 1, 0); i <= min(i0 + 1, n - 1); ++i)
    if (texel(((float)i + 0.5f) / (float)n, size) == x) return true;
  return false;
}

// Mode 0 (f.vertex != nullptr) also runs the fill-in of each pixel and counts the lit samples of denseEnough's decimation
// into f.dense_count (zeroed by k_splat_scatter of the same raycast): the fill-in reads only pixel p of the outputs written here.
// Without depth_out, each of image / vertex / normal / time_out is written only if given (the frame gives all four; a model
// view may ask for any of them, and only when there is no fill-in).
__global__ void k_splat_resolve(RayArgs a, const MapPose* __restrict__ mp, const float4* __restrict__ pos_conf,
                                const float4* __restrict__ color_time, const float4* __restrict__ norm_rad,
                                unsigned long long* __restrict__ zbuf, uchar4* __restrict__ image, float4* __restrict__ vertex,
                                float4* __restrict__ normal, uint16_t* __restrict__ time_out, float* __restrict__ depth_out, FillOut f) {
  pdl_enter();
  const int n_px = a.rows * a.cols;
  for (int p = blockIdx.x * blockDim.x + threadIdx.x; p < n_px; p += gridDim.x * blockDim.x) {
    const unsigned long long key = zbuf[p];
    zbuf[p] = kEmptyKey;
    const int py = p / a.cols, px = p - py * a.cols;
    if (key == kEmptyKey) {
      if (depth_out) {
        depth_out[p] = 0.f;
      } else {
        const float4 z4 = make_float4(0.f, 0.f, 0.f, 0.f);
        const uchar4 z1 = make_uchar4(0, 0, 0, 0);
        if (image) image[p] = z1;
        if (vertex) vertex[p] = z4;
        if (normal) normal[p] = z4;
        if (time_out) time_out[p] = 0;
        if (f.vertex) fill_in_pixel(f, a.rows, a.cols, a.c, px, py, p, z4, z4, z1);
      }
      continue;
    }
    const uint32_t id = (uint32_t)(key & 0xffffffffull);
    const float4 ct = color_time[id];
    Splat sp;
    splat_vertex(a, mp, pos_conf[id], ct, norm_rad, id, sp);
    f3 cp;
    splat_fragment(sp, a.c, px, py, cp);
    if (depth_out) {
      depth_out[p] = cp.z;
      continue;
    }
    const f3 col = decode_color(ct.x);
    const uchar4 im = make_uchar4((unsigned char)(int)rintf(col.x * 255.0f), (unsigned char)(int)rintf(col.y * 255.0f),
                                  (unsigned char)(int)rintf(col.z * 255.0f), 255);
    const float z = cp.z;
    const float fxc = (float)px + 0.5f, fyc = (float)py + 0.5f;
    const float4 vt = make_float4((fxc - a.c.cx) * z * (1.f / a.c.fx), (fyc - a.c.cy) * z * (1.f / a.c.fy), z, sp.conf);
    const float4 nm = make_float4(sp.nrm.x, sp.nrm.y, sp.nrm.z, sp.rad);
    if (image) image[p] = im;
    if (vertex) vertex[p] = vt;
    if (normal) normal[p] = nm;
    if (time_out) time_out[p] = (uint16_t)(unsigned int)ct.z;
    if (f.dense_count && im.x > 0 && im.y > 0 && im.z > 0 && is_dense_sample(px, a.cols) && is_dense_sample(py, a.rows))
      atomicAdd(f.dense_count, 1);
    if (f.vertex) fill_in_pixel(f, a.rows, a.cols, a.c, px, py, p, vt, nm, im);
  }
}

// ---------------------------------------------------------------------------------------------------------------
// fill-in (fill_vertex/normal/rgb.frag, FillIn.cpp:62-191) in one launch, and the density test
// ---------------------------------------------------------------------------------------------------------------
__global__ void k_fill_in(const float4* __restrict__ vertex, const float4* __restrict__ normal, const uchar4* __restrict__ image, int rows, int cols, Cam c,
                          FillOut f) {
  pdl_enter();
  const int n = rows * cols;
  for (int p = blockIdx.x * blockDim.x + threadIdx.x; p < n; p += gridDim.x * blockDim.x) {
    const int y = p / cols, x = p - y * cols;
    fill_in_pixel(f, rows, cols, c, x, y, p, vertex[p], normal[p], image[p]);
  }
}

// Resize::image (nearest decimation by 20) + the lit-sample count of ElasticFusion::denseEnough (Resize.cpp:50-79,
// ElasticFusion.cpp:256-268) for an image no mode-0 raycast wrote
__global__ void k_dense_enough(const uchar4* __restrict__ image, int rows, int cols, int* __restrict__ count) {
  pdl_enter();
  const int drows = rows / DENSE_FACTOR, dcols = cols / DENSE_FACTOR;
  __shared__ int s_sum;
  if (threadIdx.x == 0) s_sum = 0;
  __syncthreads();
  int local = 0;
  for (int q = threadIdx.x; q < drows * dcols; q += blockDim.x) {
    const int j = q / dcols, i = q - j * dcols;
    const int sx = texel(((float)i + 0.5f) / (float)dcols, cols);
    const int sy = texel(((float)j + 0.5f) / (float)drows, rows);
    const uchar4 s = image[(size_t)sy * cols + sx];
    local += (s.x > 0 && s.y > 0 && s.z > 0) ? 1 : 0;
  }
  atomicAdd(&s_sum, local);
  __syncthreads();
  if (threadIdx.x == 0) *count = s_sum;
}

__global__ void k_set_int(int* p, int v) {
  pdl_enter();
  if (threadIdx.x == 0 && blockIdx.x == 0) *p = v;
}

// AoS (reference Vertex layout) <-> SoA repack for downloadMap / upload
__global__ void k_pack_aos(const float4* __restrict__ a, const float4* __restrict__ b, const float4* __restrict__ c, int n, float4* __restrict__ out) {
  pdl_enter();
  for (int k = blockIdx.x * blockDim.x + threadIdx.x; k < n; k += gridDim.x * blockDim.x) {
    out[(size_t)k * 3 + 0] = a[k];
    out[(size_t)k * 3 + 1] = b[k];
    out[(size_t)k * 3 + 2] = c[k];
  }
}
__global__ void k_unpack_aos(const float4* __restrict__ in, int n, float4* __restrict__ a, float4* __restrict__ b, float4* __restrict__ c) {
  pdl_enter();
  for (int k = blockIdx.x * blockDim.x + threadIdx.x; k < n; k += gridDim.x * blockDim.x) {
    a[k] = in[(size_t)k * 3 + 0];
    b[k] = in[(size_t)k * 3 + 1];
    c[k] = in[(size_t)k * 3 + 2];
  }
}

inline Cam cam_of(const EfContext* ctx) { return Cam{ctx->cfg.cx, ctx->cfg.cy, ctx->cfg.fx, ctx->cfg.fy}; }
inline Cam cam_of(const MapTarget& t) { return Cam{t.cx, t.cy, t.fx, t.fy}; }

}  // namespace

struct MapBuffers {
  int *totals;  // [4] scan totals
  int *fb_off_raw, *fb_off_filt;
  uint8_t *fb_flag_raw, *fb_flag_filt;
  float4* aos;  // staging for download/upload
  size_t aos_bytes;
  ScanTiles scan;  // the frame's compactions (first-frame feedback, fuse, clean, the tracker's candidate list)
};

namespace ef {

static MapBuffers& mb(EfContext* ctx) { return *reinterpret_cast<MapBuffers*>(ctx->map_host); }

// grows the AoS staging buffer to at least `bytes` (never shrinks)
static int aos_reserve(MapBuffers& B, size_t bytes) {
  if (bytes <= B.aos_bytes) return 0;
  if (B.aos) cudaFree(B.aos);
  B.aos = nullptr;
  B.aos_bytes = 0;
  CU(cudaMalloc((void**)&B.aos, bytes));
  B.aos_bytes = bytes;
  return 0;
}

// next tag of the look-back tile states (every look-back compaction)
static int next_scan_epoch(EfContext* ctx, ScanTiles& S) {
  if (++S.epoch >= (1u << 30)) {  // epoch field exhausted (never in practice): start over with clean states
    CU(cudaMemsetAsync(S.state, 0, S.bytes, ctx->stream));
    S.epoch = 1;
  }
  return 0;
}

int alloc_map(EfContext* ctx) {
  MapDev& m = ctx->map;
  memset(&m, 0, sizeof(m));
  const EfConfig& c = ctx->cfg;
  m.rows = c.height;
  m.cols = c.width;
  m.cx = c.cx;
  m.cy = c.cy;
  m.fx = c.fx;
  m.fy = c.fy;
  m.capacity = c.capacity;
  const size_t n = (size_t)c.width * c.height, cap = (size_t)c.capacity;
  MapBuffers* B = new MapBuffers();
  memset(B, 0, sizeof(*B));
  ctx->map_host = B;
  // ONE buffer set: fuse updates matched surfels in place and clean compacts in place (the reference ping-pongs two VBOs,
  // GlobalModel.cpp:71-87, and rewrites the whole map twice per frame)
  CU(ctx_alloc(ctx, &m.pos_conf, cap));
  CU(ctx_alloc(ctx, &m.color_time, cap));
  CU(ctx_alloc(ctx, &m.norm_rad, cap));
  CU(cudaFuncSetAttribute(k_clean_move<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(CcShared)));
  CU(cudaFuncSetAttribute(k_clean_move<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(CcShared)));
  CU(ctx_alloc(ctx, &m.count, 4, 0));
  CU(ctx_alloc(ctx, &m.new_pos, n));
  CU(ctx_alloc(ctx, &m.new_col, n));
  CU(ctx_alloc(ctx, &m.new_nr, n));
  CU(ctx_alloc(ctx, &m.new_count, 4, 0));
  CU(ctx_alloc(ctx, &m.assoc_id, n));
  CU(ctx_alloc(ctx, &m.pending, cap, 0xff));
  CU(ctx_alloc(ctx, &m.zbuf, n, 0xff));  // kept cleared by k_splat_resolve from here on
  // as if the tags had just run out: before the first pass re-arms it, no key carries the tag (0) fuse and clean look for
  CU(ctx_alloc(ctx, &m.index_keys, n, 0xff));
  ctx->index.pass = 255;
  ctx->index.keys_only = false;
  ctx->index.vis_pending = false;
  // look-back tile states: the clean pass walks capacity + n surfels in tiles of CC_TILE, the image-sized compactions
  // (first-frame feedback, new surfels, the tracker's candidate list) <= 2 n items in tiles of at least 128
  const size_t max_items = cap + n;
  const size_t tiles = (max_items + CC_TILE - 1) / CC_TILE + (2 * n + 127) / 128 + 2;
  CU(ctx_alloc(ctx, &B->scan.state, tiles, 0));
  CU(ctx_alloc(ctx, &B->scan.counter, 4, 0));
  CU(ctx_alloc(ctx, &m.clean_ctl, 4));
  CU(cudaMemsetAsync(m.clean_ctl, 0, 8, ctx->stream));
  CU(cudaMemsetAsync(m.clean_ctl + 2, 0xff, 8, ctx->stream));
  CU(ctx_alloc(ctx, &m.vis_list, cap));
  CU(ctx_alloc(ctx, &m.vis_count, 4, 0));
  CU(ctx_alloc(ctx, &m.keep_mask, ((max_items + CC_TILE - 1) / CC_TILE) * CC_WORDS));
  CU(ctx_alloc(ctx, &B->totals, 4, 0));
  CU(ctx_alloc(ctx, &B->fb_off_raw, n));
  CU(ctx_alloc(ctx, &B->fb_off_filt, n));
  CU(ctx_alloc(ctx, &B->fb_flag_raw, n));
  CU(ctx_alloc(ctx, &B->fb_flag_filt, n));
  CU(ctx_alloc(ctx, &m.pose, 1));
  CU(ctx_alloc(ctx, &m.view_pose, 1));
  CU(ctx_alloc(ctx, &m.dense_count, 4, 0));
  CU(ctx_alloc(ctx, &m.tick, 4));
  CU(ctx_alloc(ctx, &m.nodes, (size_t)MAX_GRAPH_NODES * 16));
  CU(ctx_alloc(ctx, &m.loop, 1, 0));
  m.loop_capacity = loop_constraint_capacity(c.width, c.height);
  CU(ctx_alloc(ctx, &m.loop_src, (size_t)m.loop_capacity * 3));
  CU(ctx_alloc(ctx, &m.loop_dst, (size_t)m.loop_capacity * 3));
  CU(ctx_alloc(ctx, &m.loop_times, (size_t)m.loop_capacity));
  if (c.close_loops == 2) {
    CU(ctx_alloc(ctx, &m.graph, (size_t)MAX_GRAPH_NODES - 1, 0));
    CU(ctx_alloc(ctx, &m.graph_n, 1, 0));
  }
  B->scan.epoch = 0;
  B->scan.bytes = tiles * 8;
  const int one = 1;
  CU(cudaMemcpyAsync(m.tick, &one, 4, cudaMemcpyHostToDevice, ctx->stream));
  CU(cudaStreamSynchronize(ctx->stream));
  return 0;
}

static int scan_slot_of(EfContext* ctx, ScanTiles& S, ScanSlot* out) {
  RC(next_scan_epoch(ctx, S));
  out->state = S.state;
  out->counter = S.counter;
  out->epoch = S.epoch;
  return 0;
}
int scan_slot(EfContext* ctx, ScanSlot* out) { return scan_slot_of(ctx, mb(ctx).scan, out); }
int scan_slot(EfContext* ctx, ScanTiles& tiles, ScanSlot* out) { return scan_slot_of(ctx, tiles, out); }

static int run_scan(EfContext* ctx, const uint8_t* flags, const int* n_a, const int* n_b, size_t max_items, int* offsets, int* total) {
  const size_t tiles = (max_items + SCAN_TILE - 1) / SCAN_TILE + 1;
  ScanSlot sc;
  RC(scan_slot(ctx, &sc));
  EF_LAUNCH(ctx, k_scan_flags, wave_blocks(ctx, tiles, 4, 1), SCAN_THREADS, 0, flags, n_a, n_b, offsets, sc.state, sc.counter, total, sc.epoch);
  CHECK_LAST();
  return 0;
}

// T == nullptr: use the tracker's device-resident pose
int map_update_pose_async(EfContext* ctx, const double* T_host) {
  const double* src = ctx->odom[0].gn->T_wc;
  if (T_host) {
    CU(cudaStreamSynchronize(ctx->stream));
    memcpy(ctx->pin_small->map_pose, T_host, sizeof(double) * 16);
    CU(cudaMemcpyAsync(ctx->dev_small->map_pose, ctx->pin_small->map_pose, sizeof(double) * 16, cudaMemcpyHostToDevice, ctx->stream));
    src = ctx->dev_small->map_pose;
  }
  return map_pose_record_async(ctx, ctx->map.pose, src);
}

int map_pose_record_async(EfContext* ctx, MapPose* mp, const double* T_dev) {
  EF_LAUNCH(ctx, k_update_pose, 1, 32, 0, mp, T_dev);
  CHECK_LAST();
  return 0;
}

int map_initialise_async(EfContext* ctx) {
  MapDev& m = ctx->map;
  MapBuffers& B = mb(ctx);
  const int n = m.rows * m.cols;
  EF_LAUNCH(ctx, k_feedback_flags, wave_blocks(ctx, n), 256, 0, ctx->tex.depth_metric, ctx->tex.depth_metric_filtered, m.rows, m.cols,
            ctx->max_depth_processed, B.fb_flag_raw, B.fb_flag_filt);
  // device-resident element count for the scans: reuse new_count as "n pixels"
  EF_LAUNCH(ctx, k_set_int, 1, 32, 0, m.new_count, n);
  RC(run_scan(ctx, B.fb_flag_raw, m.new_count, nullptr, n, B.fb_off_raw, B.totals + 0));
  RC(run_scan(ctx, B.fb_flag_filt, m.new_count, nullptr, n, B.fb_off_filt, B.totals + 1));
  CU(cudaMemsetAsync(m.norm_rad, 0, (size_t)(n < m.capacity ? n : m.capacity) * sizeof(float4), ctx->stream));
  EF_LAUNCH(ctx, k_init_scatter, wave_blocks(ctx, n), 256, 0, ctx->tex.rgb, ctx->tex.depth_metric, ctx->tex.depth_metric_filtered, m.rows, m.cols,
            cam_of(ctx), ctx->tick, B.fb_flag_raw, B.fb_flag_filt, B.fb_off_raw, B.fb_off_filt, B.totals + 0, m.capacity, m.pos_conf,
            m.color_time, m.norm_rad, m.count);
  EF_LAUNCH(ctx, k_set_int, 1, 32, 0, m.new_count, 0);
  CHECK_LAST();
  return 0;
}

MapTarget map_frame_target(EfContext* ctx) {
  MapDev& m = ctx->map;
  Textures& x = ctx->tex;
  MapTarget t = {};
  t.rows = m.rows;
  t.cols = m.cols;
  t.cx = ctx->cfg.cx;
  t.cy = ctx->cfg.cy;
  t.fx = ctx->cfg.fx;
  t.fy = ctx->cfg.fy;
  t.rgb = x.rgb;
  t.depth_metric = x.depth_metric;
  t.depth_metric_filtered = x.depth_metric_filtered;
  t.synth_depth = x.synth_depth;
  t.pose = m.pose;
  t.weighting = &ctx->odom[0].gn->weighting;
  t.index_keys = m.index_keys;
  t.key_texels = (size_t)m.rows * m.cols;
  t.index = x.index;
  t.vert_conf = x.vert_conf;
  t.color_time = x.color_time;
  t.norm_rad = x.norm_rad;
  t.ix = &ctx->index;
  t.assoc_id = m.assoc_id;
  t.new_pos = m.new_pos;
  t.new_col = m.new_col;
  t.new_nr = m.new_nr;
  t.new_count = m.new_count;
  t.keep_mask = m.keep_mask;
  t.clean_ctl = m.clean_ctl;
  t.clean_total = mb(ctx).totals + 3;
  t.scan = &mb(ctx).scan;
  return t;
}

static IndexMap index_map(const MapTarget& t) {
  IndexMap ix;
  ix.keys = t.index_keys;
  ix.tag = 0xffu - (unsigned int)t.ix->pass;
  ix.index = t.index;
  ix.vert_conf = t.vert_conf;
  ix.col_time = t.color_time;
  ix.norm_rad = t.norm_rad;
  return ix;
}

// vis_mode 0: plain (stage API, fuse views), textures written. 1: also record the surfels that reach the z-buffer (first pass of
// a frame). 2: visit only those (second pass of the frame, same arguments, only fuse in between). The frame's passes (1, 2) leave
// the textures to the frame's clean, which also re-arms the list.
int map_predict_indices_async(EfContext* ctx, const MapTarget& t, int time, float max_depth, int time_delta, int vis_mode) {
  MapDev& m = ctx->map;
  IndexState& st = *t.ix;
  const int n = t.rows * t.cols;
  const bool in_frame = vis_mode != 0;
  if (!ctx->visible_list) vis_mode = 0;
  const int grid = ctx->num_sms * 5;
  if (vis_mode == 1 && st.vis_pending) CU(cudaMemsetAsync(m.vis_count, 0, 4, ctx->stream));  // (a frame that failed before its clean)
  if (vis_mode == 2 && !st.vis_pending) vis_mode = 0;
  if (vis_mode == 1) st.vis_pending = true;
  if (st.pass == 255) {  // the tags have run out: every key becomes stale
    CU(cudaMemsetAsync(t.index_keys, 0xff, t.key_texels * sizeof(unsigned long long), ctx->stream));
    st.pass = 0;
  }
  st.pass++;
  const IndexMap ix = index_map(t);
  const auto scatter = vis_mode == 1 ? k_index_scatter<1> : vis_mode == 2 ? k_index_scatter<2> : k_index_scatter<0>;  // (mode 0 never reads the list)
  EF_LAUNCH(ctx, scatter, grid, 256, 0, m.pos_conf, m.color_time, m.count, t.pose, time, max_depth, time_delta, t.rows, t.cols, cam_of(t),
            t.index_keys, ix.tag, m.vis_list, m.vis_count, m.capacity);
  st.keys_only = in_frame;
  if (!in_frame) EF_LAUNCH(ctx, k_index_textures, wave_blocks(ctx, n), 256, 0, ix, m.pos_conf, m.color_time, m.norm_rad, t.pose, n);
  CHECK_LAST();
  return 0;
}

int map_index_textures_async(EfContext* ctx, const MapTarget& t) {
  if (!t.ix->keys_only) return 0;
  MapDev& m = ctx->map;
  const int n = t.rows * t.cols;
  EF_LAUNCH(ctx, k_index_textures, wave_blocks(ctx, n), 256, 0, index_map(t), m.pos_conf, m.color_time, m.norm_rad, t.pose, n);
  t.ix->keys_only = false;
  CHECK_LAST();
  return 0;
}

static FuseArgs fuse_args(const MapTarget& t, int time, float max_depth) {
  FuseArgs a;
  a.rgb = t.rgb;
  a.depth_raw = t.depth_metric;
  a.depth_filt = t.depth_metric_filtered;
  a.ix = index_map(t);
  a.rows = t.rows;
  a.cols = t.cols;
  a.c = cam_of(t);
  a.time = time;
  a.max_depth = max_depth;
  return a;
}

// weighting < 0: the device-resident one *t.weighting holds (the frame's: computed by the tracker)
int map_fuse_async(EfContext* ctx, const MapTarget& t, int time, float max_depth, float weighting) {
  MapDev& m = ctx->map;
  if (weighting >= 0) {
    CU(cudaStreamSynchronize(ctx->stream));
    ctx->pin_small->weighting = weighting;
    CU(cudaMemcpyAsync(t.weighting, &ctx->pin_small->weighting, 4, cudaMemcpyHostToDevice, ctx->stream));
  }
  FuseArgs a = fuse_args(t, time, max_depth);
  const Quarter Q = quarter_of(time, t.rows, t.cols);
  const int nq = Q.ni * Q.nj;
  const auto associate = t.ix->keys_only ? k_fuse_associate<false> : k_fuse_associate<true>;
  EF_LAUNCH(ctx, associate, wave_blocks(ctx, nq, 16, 128), 128, 0, a, t.pose, m.pos_conf, m.norm_rad, m.count, t.assoc_id, m.pending);
  ScanSlot sc;
  RC(scan_slot_of(ctx, *t.scan, &sc));
  EF_LAUNCH(ctx, k_fuse_update, wave_blocks(ctx, nq, 16, FU_THREADS), FU_THREADS, 0, a, t.pose, (const float*)t.weighting, m.count, t.assoc_id,
            m.pending, m.pos_conf, m.color_time, m.norm_rad, t.new_pos, t.new_col, t.new_nr, t.new_count, sc.state, sc.counter, sc.epoch);
  CHECK_LAST();
  return 0;
}

// n_nodes > 0: the deformation graph previously stored by map_set_graph is applied to every kept surfel
int map_clean_async(EfContext* ctx, const MapTarget& t, int time, float conf_threshold, int time_delta, float max_depth, int n_nodes,
                    bool is_fern) {
  MapDev& m = ctx->map;
  IndexState& st = *t.ix;
  CleanArgs a;
  a.ix = index_map(t);
  a.rows = t.rows;
  a.cols = t.cols;
  a.c = cam_of(t);
  a.time = time;
  a.conf_threshold = conf_threshold;
  a.time_delta = time_delta;
  a.nodes = m.nodes;
  a.n_nodes = n_nodes;
  a.depth = t.synth_depth;
  a.max_depth = max_depth;
  a.is_fern = is_fern ? 1 : 0;
  // test (parallel) -> order-preserving in-place compaction + append of the new surfels + count publication (movers only)
  const size_t max_items = (size_t)m.capacity + (size_t)t.rows * t.cols;
  const size_t tiles = (max_items + CC_TILE - 1) / CC_TILE;
  RC(next_scan_epoch(ctx, *t.scan));
  // grids never depend on a surfel count the host would have to read back: the test strides over the tiles, the movers draw
  // tiles from a dispenser (one resident wave: four 49 KB CTAs per SM)
  const int write_tex = st.keys_only ? 1 : 0;
  int* reset_count = st.vis_pending ? m.vis_count : nullptr;
  const auto flags = st.keys_only ? k_clean_flags<false> : k_clean_flags<true>;
  EF_LAUNCH(ctx, flags, wave_blocks(ctx, tiles, 2, 1), CF_THREADS, 0, a, t.pose, m.pos_conf, m.color_time, m.norm_rad, m.count, t.new_pos,
            t.new_col, t.new_nr, t.new_count, t.keep_mask, t.clean_ctl, write_tex, reset_count);
  st.keys_only = false;
  st.vis_pending = false;
  const auto move = n_nodes > 0 ? k_clean_move<true> : k_clean_move<false>;
  EF_LAUNCH(ctx, move, wave_blocks(ctx, tiles, 4, 1), CC_THREADS, sizeof(CcShared), a, t.pose, m.pos_conf, m.color_time, m.norm_rad, m.count,
            t.new_pos, t.new_col, t.new_nr, t.new_count, m.capacity, t.keep_mask, t.scan->state, t.clean_ctl, t.clean_total, t.scan->epoch);
  CHECK_LAST();
  return 0;
}

static FillOut fill_out(EfContext* ctx, bool pass_geom, bool pass_img) {
  const Textures& t = ctx->tex;
  FillOut f = {};
  f.raw_depth = t.depth_filtered;
  f.rgb = t.rgb;
  f.pass_geom = pass_geom ? 1 : 0;
  f.pass_img = pass_img ? 1 : 0;
  f.vertex = t.fill_vertex;
  f.normal = t.fill_normal;
  f.image = t.fill_image;
  f.dense_count = ctx->map.dense_count;
  return f;
}

int map_raycast_async(EfContext* ctx, float max_depth, float conf_threshold, int time, int max_time, int time_delta, int mode, int fill_in) {
  MapDev& m = ctx->map;
  const int n = m.rows * m.cols;
  RayArgs a;
  a.rows = m.rows;
  a.cols = m.cols;
  a.c = cam_of(ctx);
  a.max_depth = max_depth;
  a.conf_threshold = conf_threshold;
  a.time = time;
  a.max_time = max_time;
  a.time_delta = time_delta;
  // mode 0 keeps the lit-sample count of denseEnough in step with the predicted image
  EF_LAUNCH(ctx, k_splat_scatter, ctx->num_sms * 4, SPLAT_THREADS, 0, a, m.pose, m.pos_conf, m.color_time, m.norm_rad, m.count, m.zbuf,
            mode == 0 ? m.dense_count : (int*)nullptr);
  // mode 0: the predicted model, 1: the old model (loop closure), 2: the synthesised depth alone
  Textures& t = ctx->tex;
  struct Out {
    uchar4* image;
    float4 *vertex, *normal;
    uint16_t* time;
    float* depth;
  };
  const Out o = mode == 0 ? Out{t.image, t.vertex, t.normal, t.time, nullptr}
              : mode == 1 ? Out{t.old_image, t.old_vertex, t.old_normal, t.old_time, nullptr}
                          : Out{nullptr, nullptr, nullptr, nullptr, t.synth_depth};
  FillOut f = {};
  if (mode == 0) {
    f.dense_count = m.dense_count;
    if (fill_in >= 0) f = fill_out(ctx, false, fill_in == 1);
  }
  EF_LAUNCH(ctx, k_splat_resolve, wave_blocks(ctx, n), 256, 0, a, m.pose, m.pos_conf, m.color_time, m.norm_rad, m.zbuf, o.image, o.vertex, o.normal,
            o.time, o.depth, f);
  CHECK_LAST();
  return 0;
}

// a view's pose into MapDev::view_pose and, weighting >= 0, its fusion weighting into DevStaging::view_weighting. The pinned slots
// are rewritten once the previous view's copies have read them (not the whole stream: the call stays asynchronous).
static int stage_view_pose(EfContext* ctx, const double* T_wc, float weighting) {
  PinStaging* pin = ctx->pin_small;
  DevStaging* dev = ctx->dev_small;
  CU(cudaEventSynchronize(ctx->view_pose_sent));
  memcpy(pin->view_pose, T_wc, sizeof(double) * 16);
  CU(cudaMemcpyAsync(dev->view_pose, pin->view_pose, sizeof(double) * 16, cudaMemcpyHostToDevice, ctx->stream));
  if (weighting >= 0) {
    pin->view_weighting = weighting;
    CU(cudaMemcpyAsync(&dev->view_weighting, &pin->view_weighting, sizeof(float), cudaMemcpyHostToDevice, ctx->stream));
  }
  CU(cudaEventRecord(ctx->view_pose_sent, ctx->stream));
  EF_LAUNCH(ctx, k_update_pose, 1, 32, 0, ctx->map.view_pose, (const double*)dev->view_pose);
  CHECK_LAST();
  return 0;
}

// the raycast above at a camera of its own and the pose record `pose`, on the off-frame z-buffer; f: its dense count and fill-in;
// depth given: the synthesised depth alone
static int predict_offframe(EfContext* ctx, const RayArgs& a, const MapPose* pose, uchar4* image, float4* vertex, float4* normal, uint16_t* time,
                            const FillOut& f, float* depth = nullptr) {
  MapDev& m = ctx->map;
  const size_t n = (size_t)a.rows * a.cols;
  unsigned long long* zbuf = nullptr;
  RC(offframe_zbuf(ctx, n, &zbuf));
  EF_LAUNCH(ctx, k_splat_scatter, ctx->num_sms * 4, SPLAT_THREADS, 0, a, pose, m.pos_conf, m.color_time, m.norm_rad, m.count, zbuf, f.dense_count);
  EF_LAUNCH(ctx, k_splat_resolve, wave_blocks(ctx, n), 256, 0, a, pose, m.pos_conf, m.color_time, m.norm_rad, zbuf, image, vertex, normal, time,
            depth, f);
  CHECK_LAST();
  return 0;
}

static RayArgs ray_args(int rows, int cols, const Cam& c, float max_depth, float conf_threshold, int time, int max_time, int time_delta) {
  RayArgs a;
  a.rows = rows;
  a.cols = cols;
  a.c = c;
  a.max_depth = max_depth;
  a.conf_threshold = conf_threshold;
  a.time = time;
  a.max_time = max_time;
  a.time_delta = time_delta;
  return a;
}

// at the view's own pose, camera and size, with no fill-in; the dense count only when asked for (a track view's)
int map_predict_view_async(EfContext* ctx, const EfModelView* v, uint8_t* image, float* vertex, float* normal, uint16_t* time, int* dense_count) {
  RC(stage_view_pose(ctx, v->T_wc, -1.0f));
  FillOut f = {};
  f.dense_count = dense_count;
  return predict_offframe(ctx, ray_args(v->height, v->width, Cam{v->cx, v->cy, v->fx, v->fy}, v->max_depth, v->conf_threshold, v->time,
                                        v->max_time, v->time_delta),
                          ctx->map.view_pose, reinterpret_cast<uchar4*>(image), reinterpret_cast<float4*>(vertex),
                          reinterpret_cast<float4*>(normal), time, f);
}

int map_predict_target_async(EfContext* ctx, const PredictTarget& t, float max_depth, float conf_threshold, int time, int max_time, int time_delta) {
  FillOut f = {};
  f.dense_count = t.dense_count;
  if (t.fill_vertex) {
    f.raw_depth = t.fill_depth;
    f.rgb = t.fill_rgb;
    f.pass_img = t.fill_pass_img;
    f.vertex = t.fill_vertex;
    f.normal = t.fill_normal;
    f.image = t.fill_image;
  }
  return predict_offframe(ctx, ray_args(t.rows, t.cols, Cam{t.cx, t.cy, t.fx, t.fy}, max_depth, conf_threshold, time, max_time, time_delta),
                          t.pose, t.image, t.vertex, t.normal, t.time, f, t.depth);
}

// ---- fuse view (ef_map_fuse_view*): its own inputs, index map and scratch, in one allocation grown to the largest view ----
struct FuseViewBuffers {
  void* block;
  size_t px;  // pixels the block was carved for
  uint8_t* rgb;
  uint16_t* depth_raw;
  float *depth_metric, *depth_metric_filtered;
  unsigned long long* index_keys;
  uint32_t* index;
  float4 *vert_conf, *color_time, *norm_rad;
  uint32_t* assoc_id;
  float4 *new_pos, *new_col, *new_nr;
  int *new_count, *clean_total;
  unsigned int* clean_ctl;
  uint32_t* keep_mask;
  IndexState ix;
  ScanTiles scan;
};

// carves the buffers of a px-pixel view out of `base` (nullptr: only sizes them); returns the bytes needed
static size_t fuse_view_layout(FuseViewBuffers& V, uint8_t* base, size_t px, size_t capacity) {
  size_t off = 0;
  auto take = [&](auto** p, size_t bytes) {
    off = (off + 255) & ~(size_t)255;
    *p = base ? reinterpret_cast<std::remove_pointer_t<decltype(p)>>(base + off) : nullptr;
    off += bytes;
  };
  const size_t clean_tiles = (capacity + px + CC_TILE - 1) / CC_TILE;
  take(&V.rgb, px * 3);
  take(&V.depth_raw, px * 2);
  take(&V.depth_metric, px * 4);
  take(&V.depth_metric_filtered, px * 4);
  take(&V.index_keys, px * 8);
  take(&V.index, px * 4);
  take(&V.vert_conf, px * 16);
  take(&V.color_time, px * 16);
  take(&V.norm_rad, px * 16);
  take(&V.assoc_id, px * 4);
  take(&V.new_pos, px * 16);
  take(&V.new_col, px * 16);
  take(&V.new_nr, px * 16);
  take(&V.new_count, 4);
  take(&V.clean_total, 4);
  take(&V.clean_ctl, 16);
  take(&V.keep_mask, clean_tiles * CC_WORDS * 4);
  take(&V.scan.counter, 8);
  V.scan.bytes = (clean_tiles + (px + FU_THREADS - 1) / FU_THREADS + 2) * 8;  // the clean's tiles, or fuse's (at most px pixels)
  take(&V.scan.state, V.scan.bytes);
  return off;
}

// the buffers of a px-pixel view in `block` (fuse_view_layout's bytes), as a fresh view finds them: every key stale, no new surfels,
// clean's dispenser and tickets at zero and no first mover, no published tile state
static int arm_view_buffers(EfContext* ctx, FuseViewBuffers& V, void* block, size_t px) {
  V.block = block;
  fuse_view_layout(V, (uint8_t*)block, px, (size_t)ctx->map.capacity);
  V.px = px;
  CU(cudaMemsetAsync(V.index_keys, 0xff, px * sizeof(unsigned long long), ctx->stream));
  CU(cudaMemsetAsync(V.new_count, 0, 4, ctx->stream));
  CU(cudaMemsetAsync(V.clean_ctl, 0, 8, ctx->stream));
  CU(cudaMemsetAsync(V.clean_ctl + 2, 0xff, 8, ctx->stream));
  CU(cudaMemsetAsync(V.scan.counter, 0, 8, ctx->stream));
  CU(cudaMemsetAsync(V.scan.state, 0, V.scan.bytes, ctx->stream));
  V.scan.epoch = 0;
  V.ix.pass = 0;
  V.ix.keys_only = false;
  V.ix.vis_pending = false;
  return 0;
}

// the target of a rows x cols view on V's buffers; its pose record and weighting are the caller's to set
static MapTarget view_target(FuseViewBuffers& V, int rows, int cols, float fx, float fy, float cx, float cy) {
  MapTarget t = {};
  t.rows = rows;
  t.cols = cols;
  t.cx = cx;
  t.cy = cy;
  t.fx = fx;
  t.fy = fy;
  t.rgb = V.rgb;
  t.depth_metric = V.depth_metric;
  t.depth_metric_filtered = V.depth_metric_filtered;
  t.synth_depth = nullptr;
  t.index_keys = V.index_keys;
  t.key_texels = V.px;
  t.index = V.index;
  t.vert_conf = V.vert_conf;
  t.color_time = V.color_time;
  t.norm_rad = V.norm_rad;
  t.ix = &V.ix;
  t.assoc_id = V.assoc_id;
  t.new_pos = V.new_pos;
  t.new_col = V.new_col;
  t.new_nr = V.new_nr;
  t.new_count = V.new_count;
  t.keep_mask = V.keep_mask;
  t.clean_ctl = V.clean_ctl;
  t.clean_total = V.clean_total;
  t.scan = &V.scan;
  return t;
}

int map_fuse_view_target(EfContext* ctx, const EfFuseView* v, MapTarget* out, uint8_t** rgb, uint16_t** depth_raw) {
  if (!ctx->fuse_view) {
    FuseViewBuffers* nv = new (std::nothrow) FuseViewBuffers();
    if (!nv) return EF_ENOMEM;
    ctx->fuse_view = nv;
  }
  FuseViewBuffers& V = *static_cast<FuseViewBuffers*>(ctx->fuse_view);
  const size_t px = (size_t)v->width * v->height;
  if (px > V.px) {
    CU(cudaStreamSynchronize(ctx->stream));  // the previous view may still read the old block
    if (V.block) CU(cudaFree(V.block));
    V.block = nullptr;
    V.px = 0;
    void* block = nullptr;
    if (cudaMalloc(&block, fuse_view_layout(V, nullptr, px, (size_t)ctx->map.capacity)) != cudaSuccess) {
      cudaGetLastError();  // (an allocation failure is not sticky: the context stays usable)
      return EF_ENOMEM;
    }
    RC(arm_view_buffers(ctx, V, block, px));
  }
  RC(stage_view_pose(ctx, v->T_wc, v->weighting));
  MapTarget t = view_target(V, v->height, v->width, v->fx, v->fy, v->cx, v->cy);
  t.pose = ctx->map.view_pose;
  t.weighting = &ctx->dev_small->view_weighting;
  *out = t;
  *rgb = V.rgb;
  *depth_raw = V.depth_raw;
  return 0;
}

int map_camera_target(EfContext* ctx, Arena& arena, int rows, int cols, float fx, float fy, float cx, float cy, void** state, MapTarget* out,
                      uint8_t** rgb, uint16_t** depth_raw) {
  FuseViewBuffers* V = new (std::nothrow) FuseViewBuffers();
  if (!V) return EF_ENOMEM;
  *state = V;
  const size_t px = (size_t)rows * cols;
  uint8_t* block = nullptr;
  CU(arena_alloc(ctx, arena, &block, fuse_view_layout(*V, nullptr, px, (size_t)ctx->map.capacity)));
  RC(arm_view_buffers(ctx, *V, block, px));
  *out = view_target(*V, rows, cols, fx, fy, cx, cy);
  *rgb = V->rgb;
  *depth_raw = V->depth_raw;
  return 0;
}

void map_camera_target_free(void* state) { delete static_cast<FuseViewBuffers*>(state); }

void map_fuse_view_free(EfContext* ctx) {
  FuseViewBuffers* V = static_cast<FuseViewBuffers*>(ctx->fuse_view);
  if (!V) return;
  if (V->block) cudaFree(V->block);
  delete V;
  ctx->fuse_view = nullptr;
}

int map_fill_in_async(EfContext* ctx, bool pass_geom, bool pass_img) {
  MapDev& m = ctx->map;
  Textures& t = ctx->tex;
  const int n = m.rows * m.cols;
  EF_LAUNCH(ctx, k_fill_in, wave_blocks(ctx, n), 256, 0, t.vertex, t.normal, t.image, m.rows, m.cols, cam_of(ctx), fill_out(ctx, pass_geom, pass_img));
  CHECK_LAST();
  return 0;
}

int map_dense_enough_async(EfContext* ctx) {
  MapDev& m = ctx->map;
  EF_LAUNCH(ctx, k_dense_enough, 1, 256, 0, ctx->tex.image, m.rows, m.cols, m.dense_count);
  CHECK_LAST();
  return 0;
}

int map_download(EfContext* ctx, const float4* a, const float4* b, const float4* c, int n, float* out) {
  MapBuffers& B = mb(ctx);
  if (n <= 0) return 0;
  RC(aos_reserve(B, (size_t)n * 48));
  EF_LAUNCH(ctx, k_pack_aos, wave_blocks(ctx, n), 256, 0, a, b, c, n, B.aos);
  CU(cudaMemcpyAsync(out, B.aos, (size_t)n * 48, cudaMemcpyDeviceToHost, ctx->stream));
  CU(cudaStreamSynchronize(ctx->stream));
  return 0;
}

int map_upload(EfContext* ctx, const float* in, int n) {
  MapDev& m = ctx->map;
  MapBuffers& B = mb(ctx);
  if (n > m.capacity) return EF_EINVAL;
  if (n > 0) {
    RC(aos_reserve(B, (size_t)n * 48));
    CU(cudaMemcpyAsync(B.aos, in, (size_t)n * 48, cudaMemcpyHostToDevice, ctx->stream));
    EF_LAUNCH(ctx, k_unpack_aos, wave_blocks(ctx, n), 256, 0, (const float4*)B.aos, n, m.pos_conf, m.color_time, m.norm_rad);
  }
  EF_LAUNCH(ctx, k_set_int, 1, 32, 0, m.count, n);
  CU(cudaStreamSynchronize(ctx->stream));
  ctx->host_count = n;
  return 0;
}

// overwrites surfels [first, first + n) of the resident map (count unchanged; the range must lie inside it)
int map_upload_range(EfContext* ctx, const float* in, int first, int n) {
  MapDev& m = ctx->map;
  MapBuffers& B = mb(ctx);
  int cnt = 0;
  CU(cudaMemcpyAsync(&cnt, m.count, 4, cudaMemcpyDeviceToHost, ctx->stream));
  CU(cudaStreamSynchronize(ctx->stream));
  if ((long long)first + n > cnt) return EF_EINVAL;
  RC(aos_reserve(B, (size_t)n * 48));
  CU(cudaMemcpyAsync(B.aos, in, (size_t)n * 48, cudaMemcpyHostToDevice, ctx->stream));
  EF_LAUNCH(ctx, k_unpack_aos, wave_blocks(ctx, n), 256, 0, (const float4*)B.aos, n, m.pos_conf + first, m.color_time + first, m.norm_rad + first);
  CU(cudaStreamSynchronize(ctx->stream));
  return 0;
}

// Resize::image / vertex / time (Resize.cpp:50-159, resize.frag): the source sampled at the centres of a (cols/factor) x
// (rows/factor) grid with nearest filtering. elem: bytes per texel (4 RGBA8, 16 RGBA32F, 2 R16UI); out: device, tightly packed.
__global__ void k_resize_nearest(const uint8_t* __restrict__ src, int rows, int cols, int factor, int elem, uint8_t* __restrict__ out) {
  pdl_enter();
  const int drows = rows / factor, dcols = cols / factor, n = drows * dcols;
  for (int q = blockIdx.x * blockDim.x + threadIdx.x; q < n; q += gridDim.x * blockDim.x) {
    const int j = q / dcols, i = q - j * dcols;
    const int sx = texel(((float)i + 0.5f) / (float)dcols, cols), sy = texel(((float)j + 0.5f) / (float)drows, rows);
    const uint8_t* s = src + ((size_t)sy * cols + sx) * elem;
    uint8_t* d = out + (size_t)q * elem;
    if (elem == 16)
      *reinterpret_cast<float4*>(d) = *reinterpret_cast<const float4*>(s);
    else if (elem == 4)
      *reinterpret_cast<uint32_t*>(d) = *reinterpret_cast<const uint32_t*>(s);
    else
      *reinterpret_cast<uint16_t*>(d) = *reinterpret_cast<const uint16_t*>(s);
  }
}
int map_resize_to_host(EfContext* ctx, const void* src_dev, int elem, int factor, void* host_out) {
  MapDev& m = ctx->map;
  MapBuffers& B = mb(ctx);
  if (factor < 1 || m.rows / factor < 1 || m.cols / factor < 1) return EF_EINVAL;
  const size_t n = (size_t)(m.rows / factor) * (m.cols / factor);
  RC(aos_reserve(B, n * elem));
  EF_LAUNCH(ctx, k_resize_nearest, wave_blocks(ctx, n), 256, 0, (const uint8_t*)src_dev, m.rows, m.cols, factor, elem, (uint8_t*)B.aos);
  CU(cudaMemcpyAsync(host_out, B.aos, n * elem, cudaMemcpyDeviceToHost, ctx->stream));
  CU(cudaStreamSynchronize(ctx->stream));
  return 0;
}

// deformation graph for the next clean (GlobalModel.cpp:542-546: glTexSubImage2D of the node texture); nodes: HOST, 16 floats each
int map_set_graph(EfContext* ctx, const float* nodes16, int n_nodes) {
  MapDev& m = ctx->map;
  if (n_nodes < 0 || n_nodes >= MAX_GRAPH_NODES) return EF_EINVAL;  // assert(graph.size() / 16 < MAX_NODES), GlobalModel.cpp:540
  if (n_nodes == 0) return 0;
  CU(cudaStreamSynchronize(ctx->stream));
  CU(cudaMemcpyAsync(m.nodes, nodes16, (size_t)n_nodes * 16 * sizeof(float), cudaMemcpyHostToDevice, ctx->stream));
  CU(cudaStreamSynchronize(ctx->stream));  // nodes16 is caller memory
  return 0;
}
// the same from a device buffer (the device solve's hand-over), stream-ordered
int map_set_graph_device(EfContext* ctx, const float* nodes16_dev, int n_nodes) {
  if (n_nodes < 0 || n_nodes >= MAX_GRAPH_NODES) return EF_EINVAL;
  if (n_nodes > 0)
    CU(cudaMemcpyAsync(ctx->map.nodes, nodes16_dev, (size_t)n_nodes * 16 * sizeof(float), cudaMemcpyDeviceToDevice, ctx->stream));
  return 0;
}

// Deformation::sampleGraphModel (Deformation.cpp:248-303, sample.geom): position and colorTime.z (init time) of surfels 0, 5000,
// 10000, ... The graph is replaced only when more than k = 4 nodes come out (:284); otherwise the previous one stays. The
// reference's transform-feedback buffer holds 1024 nodes and keeps the oldest ones (Deformation.cpp:27); here the cap is 1023,
// the largest graph clean accepts (GlobalModel.cpp:540 asserts fewer than MAX_NODES = 1024), so maps of more than 5 110 000
// surfels sample one node fewer than the reference does.
__global__ void k_sample_graph(const float4* __restrict__ pos_conf, const float4* __restrict__ color_time, const int* __restrict__ count,
                               float4* __restrict__ graph, int* __restrict__ graph_n) {
  pdl_enter();
  const int sampled = (*count + 4999) / 5000;
  if (sampled <= 4) return;
  const int n = min(sampled, MAX_GRAPH_NODES - 1);
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const float4 p = pos_conf[(size_t)i * 5000];
    graph[i] = make_float4(p.x, p.y, p.z, color_time[(size_t)i * 5000].z);
  }
  if (blockIdx.x == 0 && threadIdx.x == 0) *graph_n = n;
}
int map_sample_graph_async(EfContext* ctx) {
  MapDev& m = ctx->map;
  EF_LAUNCH(ctx, k_sample_graph, 4, 256, 0, (const float4*)m.pos_conf, (const float4*)m.color_time, (const int*)m.count, m.graph, m.graph_n);
  CHECK_LAST();
  return 0;
}

// ---- local loop closure front half, last step (ElasticFusion.cpp:473-505): acceptance test on the model-to-model result and
// the constraint pairs sampled on the W/20 x H/20 grid (Resize::vertex / Resize::time = nearest sampling at texel centres).
// src / dst / times hold `capacity` constraints, one per grid cell; the bound check only guards against a caller that sized
// them for another frame
// One camera's grid, by one CTA of 256 threads: its constraints (src = T_curr v, dst = T_est v, the INACTIVE time stamp) are appended
// from *s_base on, which ends advanced by their number; s_warp: 8 ints of shared scratch
__device__ __forceinline__ void loop_sample_grid(const double* __restrict__ T_curr, const double* __restrict__ T_est,
                                                 const float4* __restrict__ vertex, const uint16_t* __restrict__ old_time, int rows, int cols,
                                                 float max_depth, double* __restrict__ src, double* __restrict__ dst, int* __restrict__ times,
                                                 int capacity, int& s_base, int* s_warp) {
  const int dcols = cols / 20, drows = rows / 20, n = dcols * drows;
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  for (int q0 = 0; q0 < n; q0 += 256) {  // order: i (columns) outer, j (rows) inner, as the reference's loops
    const int q = q0 + threadIdx.x;
    bool ok = false;
    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
    int t = 0;
    if (q < n) {
      const int i = q / drows, j = q - i * drows;
      const int sx = texel(((float)i + 0.5f) / (float)dcols, cols), sy = texel(((float)j + 0.5f) / (float)drows, rows);
      v = vertex[(size_t)sy * cols + sx];
      t = old_time[(size_t)sy * cols + sx];
      ok = v.z > 0 && v.z < max_depth && t > 0;
    }
    const unsigned int b = __ballot_sync(0xffffffffu, ok);
    if (lane == 0) s_warp[wid] = __popc(b);
    __syncthreads();
    int off = s_base;
    for (int w = 0; w < wid; ++w) off += s_warp[w];
    const int o = off + __popc(b & ((1u << lane) - 1u));
    if (ok && o < capacity) {
      const double x = v.x, y = v.y, z = v.z;
#pragma unroll
      for (int r = 0; r < 3; ++r) {
        src[o * 3 + r] = T_curr[r * 4 + 0] * x + T_curr[r * 4 + 1] * y + T_curr[r * 4 + 2] * z + T_curr[r * 4 + 3];
        dst[o * 3 + r] = T_est[r * 4 + 0] * x + T_est[r * 4 + 1] * y + T_est[r * 4 + 2] * z + T_est[r * 4 + 3];
      }
      times[o] = t;
    }
    __syncthreads();
    if (threadIdx.x == 0) {
      int tot = 0;
      for (int w = 0; w < 8; ++w) tot += s_warp[w];
      s_base += tot;
    }
    __syncthreads();
  }
}
// the acceptance test's covariance half (lastA.lu().inverse(), RGBDOdometry.cpp:573-575): every diagonal entry within cov_thresh
__device__ __forceinline__ bool loop_cov_ok(const double* lastA, float cov_thresh, LoopDev* out) {
  double cov[36];
  efm::inv_n<6>(lastA, cov);
  bool covOk = true;
  for (int i = 0; i < 6; ++i) {
    out->cov_diag[i] = cov[i * 6 + i];
    if (cov[i * 6 + i] > (double)cov_thresh) covOk = false;
  }
  return covOk;
}

__global__ void __launch_bounds__(256) k_loop_constraints(const GNState* __restrict__ gn_curr, const GNState* __restrict__ gn_est,
                                                          const float4* __restrict__ vertex, const uint16_t* __restrict__ old_time, int rows,
                                                          int cols, float max_depth, int count_thresh, float err_thresh, float cov_thresh,
                                                          LoopDev* out, double* __restrict__ src, double* __restrict__ dst,
                                                          int* __restrict__ times, int capacity) {
  pdl_enter();
  if (blockIdx.x != 0) return;
  __shared__ int s_accept, s_base, s_warp[8];
  if (threadIdx.x == 0) {
    const bool covOk = loop_cov_ok(gn_est->lastA, cov_thresh, out);
    out->lastICPError = gn_est->lastICPError;
    out->lastICPCount = gn_est->lastICPCount;
    for (int k = 0; k < 16; ++k) out->T_wc_est[k] = gn_est->T_wc[k];
    const int ok = (covOk && gn_est->lastICPCount > (float)count_thresh && gn_est->lastICPError < err_thresh) ? 1 : 0;
    out->ran = 1;
    out->accepted = ok;
    s_accept = ok;
    s_base = 0;
  }
  __syncthreads();
  if (!s_accept) {
    if (threadIdx.x == 0) out->n_constraints = 0;
    return;
  }
  loop_sample_grid(gn_curr->T_wc, gn_est->T_wc, vertex, old_time, rows, cols, max_depth, src, dst, times, capacity, s_base, s_warp);
  if (threadIdx.x == 0) out->n_constraints = s_base < capacity ? s_base : capacity;
}

// A closing rig's acceptance test and constraints after its joint model-to-model registration. The covariance is that of the joint
// system (member 0's loop tracker's lastA); count and error are those of the members' last-iteration ICP residuals summed in member
// order: count = sum res1, error = sqrtf(sum res0) / count. Accepted, every member's grid is sampled as k_loop_constraints samples it,
// concatenated in member order. For one member this is k_loop_constraints.
__global__ void __launch_bounds__(256) k_rig_loop_constraints(const __grid_constant__ RigLoopArgs a, int count_thresh, float err_thresh,
                                                              float cov_thresh) {
  pdl_enter();
  if (blockIdx.x != 0) return;
  __shared__ int s_accept, s_base, s_warp[8];
  LoopDev* out = a.loop;
  if (threadIdx.x == 0) {
    const bool covOk = loop_cov_ok(a.est[0]->lastA, cov_thresh, out);
    float res0 = a.dev->res[0][0], res1 = a.dev->res[0][1];
    for (int m = 1; m < a.n; ++m) {
      res0 += a.dev->res[m][0];
      res1 += a.dev->res[m][1];
    }
    const float err = sqrtf(res0) / res1;
    out->lastICPError = err;
    out->lastICPCount = res1;
    for (int k = 0; k < 16; ++k) {
      out->T_wc_est[k] = a.est[0]->T_wc[k];
      a.rec->T_wc_curr[k] = a.curr[0]->T_wc[k];
    }
    const int ok = (covOk && res1 > (float)count_thresh && err < err_thresh) ? 1 : 0;
    out->ran = 1;
    out->accepted = ok;
    s_accept = ok;
    s_base = 0;
  }
  __syncthreads();
  if (!s_accept) {
    if (threadIdx.x == 0) {
      out->n_constraints = 0;
      for (int m = 0; m < EF_MAX_CAMERAS; ++m) a.rec->member_n[m] = 0;
    }
    return;
  }
  for (int m = 0; m < a.n; ++m) {
    const int first = s_base;
    loop_sample_grid(a.curr[m]->T_wc, a.est[m]->T_wc, a.vertex[m], a.old_time[m], a.rows[m], a.cols[m], a.max_depth[m], a.src, a.dst, a.times,
                     a.capacity, s_base, s_warp);
    if (threadIdx.x == 0) a.rec->member_n[m] = min(s_base, a.capacity) - min(first, a.capacity);
  }
  if (threadIdx.x == 0) out->n_constraints = s_base < a.capacity ? s_base : a.capacity;
}

__global__ void k_loop_reset(LoopDev* out) {
  pdl_enter();
  if (blockIdx.x == 0 && threadIdx.x == 0) {
    out->ran = 0;
    out->accepted = 0;
    out->n_constraints = 0;
  }
}
// T_wc of tracker `dst` = T_wc of tracker `src` (modelToModel starts from T_wc_curr: Sophus::SE3d T_wc_est = T_wc_curr)
__global__ void k_copy_pose(GNState* dst, const GNState* src) {
  pdl_enter();
  if (blockIdx.x == 0 && threadIdx.x < 16) dst->T_wc[threadIdx.x] = src->T_wc[threadIdx.x];
}

int map_loop_constraints_async(EfContext* ctx, const LoopSide& s) {
  const EfConfig& c = ctx->cfg;
  EF_LAUNCH(ctx, k_loop_constraints, 1, 256, 0, (const GNState*)ctx->odom[s.curr].gn, (const GNState*)ctx->odom[s.est].gn, s.vertex, s.old_time,
            s.rows, s.cols, s.max_depth, c.count_thresh, c.err_thresh, c.cov_thresh, s.loop, s.src, s.dst, s.times, s.capacity);
  CHECK_LAST();
  return 0;
}
int map_rig_loop_constraints_async(EfContext* ctx, const RigLoopArgs& a) {
  const EfConfig& c = ctx->cfg;
  EF_LAUNCH(ctx, k_rig_loop_constraints, 1, 256, 0, a, c.count_thresh, c.err_thresh, c.cov_thresh);
  CHECK_LAST();
  return 0;
}
int map_loop_reset_async(EfContext* ctx, LoopDev* loop) {
  EF_LAUNCH(ctx, k_loop_reset, 1, 32, 0, loop);
  CHECK_LAST();
  return 0;
}
int odom_copy_pose_async(EfContext* ctx, int dst, int src) {
  EF_LAUNCH(ctx, k_copy_pose, 1, 32, 0, ctx->odom[dst].gn, (const GNState*)ctx->odom[src].gn);
  CHECK_LAST();
  return 0;
}

void map_free_host(EfContext* ctx) {
  MapBuffers* B = reinterpret_cast<MapBuffers*>(ctx->map_host);
  if (B) {
    if (B->aos) cudaFree(B->aos);
    delete B;
    ctx->map_host = nullptr;
  }
}

}  // namespace ef
