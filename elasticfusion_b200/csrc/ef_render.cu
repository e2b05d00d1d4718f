// Render of the surfel map from any viewpoint: the reference viewer's global-surface pass, draw_global_surface.{vert,geom,frag}
// and draw_global_surface_phong.frag (GlobalModel::renderPointCloud, GlobalModel.cpp:286-350; the colour pass of GUI::drawFXAA,
// Tools/GUI.h:273-345), as two kernels over the resident map. Pinned by running those shader files on Mesa llvmpipe
// (oracle/gl, tests/golden/ref_render_*.npz).
//
// The geometry shader emits each surfel as a 4-vertex strip with texcoords (-1,-1), (1,-1), (-1,1), (1,1), and the fragment shader
// discards dot(tc, tc) > 1. The disc lies inside the quad, and both triangles lie on one plane with one affine map from texcoord to
// position, so the coverage of the two triangles reduces to the disc test on the plane's perspective-correct interpolants. Those
// come from the homogeneous barycentrics of the strip's first triangle at the pixel centre (2D homogeneous rasterisation), which
// also clip against the near and far planes (-w <= z <= w, w > 0) without building clipped polygons: a quad that crosses the near
// plane, or has a corner behind the eye, renders the part in front.
//
// Depth test: atomicMin of (d24 << 32 | id), GL_LESS against the cleared depth 1.0 with the lower id (earlier in draw order) winning
// ties; the resolve re-arms the z-buffer, so no pass clears it.
#include <float.h>
#include <stddef.h>

#include "ef_device.cuh"
#include "ef_internal.h"

using namespace ef;

namespace {

constexpr unsigned long long kEmptyKey = ~0ull;
constexpr int RENDER_THREADS = 256;

// the buffers of the passes outside the frame (this render and the model view, ef_map.cu), grown to the largest view requested
// (ef_destroy frees them)
struct RenderBuffers {
  unsigned long long* zbuf = nullptr;  // kept at kEmptyKey between passes by k_render_resolve / k_splat_resolve
  uint8_t* staging = nullptr;          // device outputs of a call that returns them to the host
  size_t zbuf_bytes = 0, staging_bytes = 0;
};

struct RenderQuad {
  float X[3], Y[3], Z[3], W[3];  // clip coordinates of strip vertices 0, 1, 2
  float rad;
  bool unstable;
};
struct RenderFrag {
  float b[3];  // homogeneous barycentrics of strip vertices 0, 1, 2
  float u, v;  // texcoord
  float zw;    // window depth (gl_FragCoord.z)
};

__device__ __forceinline__ float clipc(const float* m, int r, const f3& p) { return ((m[r] * p.x + m[4 + r] * p.y) + m[8 + r] * p.z) + m[12 + r]; }

// draw_global_surface.vert's test and .geom's strip: corners p+x, p+y, p-y, p-x in clip space (C4) and world space (P4)
__device__ __forceinline__ bool render_quad(const EfRenderView& v, const float4& pc, const float4& nr, float (&C4)[4][4], f3 (&P4)[4]) {
  if (!(pc.w > v.threshold || v.unstable == 1)) return false;
  const f3 p = mk3(pc.x, pc.y, pc.z), n = mk3(nr.x, nr.y, nr.z);
  const f3 x = normalized(mk3(n.y - n.z, -n.x, n.x)) * nr.w * 1.41421356f;
  const f3 y = cross(n, x);
  P4[0] = p + x;
  P4[1] = p + y;
  P4[2] = p - y;
  P4[3] = p - x;
#pragma unroll
  for (int k = 0; k < 4; ++k)
#pragma unroll
    for (int r = 0; r < 4; ++r) C4[k][r] = clipc(v.mvp, r, P4[k]);
  return true;
}

// pixel range of a quad; false if nothing of it can be visible. All w > 0: the corners' window bounding box with one pixel of slack
// each side; w changes sign: the whole view.
__device__ __forceinline__ bool render_bounds(const float (&C4)[4][4], int w, int h, int& x0, int& x1, int& y0, int& y1) {
  int pos = 0, behind_near = 0, beyond_far = 0;
  float xmin = FLT_MAX, xmax = -FLT_MAX, ymin = FLT_MAX, ymax = -FLT_MAX;
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    const float W = C4[k][3];
    pos += W > 0.f;
    behind_near += C4[k][2] < -W;
    beyond_far += C4[k][2] > W;
    if (W > 0.f) {
      const float xw = ((C4[k][0] / W) * 0.5f + 0.5f) * (float)w, yw = ((C4[k][1] / W) * 0.5f + 0.5f) * (float)h;
      xmin = fminf(xmin, xw);
      xmax = fmaxf(xmax, xw);
      ymin = fminf(ymin, yw);
      ymax = fmaxf(ymax, yw);
    }
  }
  if (pos == 0 || behind_near == 4 || beyond_far == 4) return false;
  if (pos < 4) {
    x0 = 0, x1 = w - 1, y0 = 0, y1 = h - 1;
    return true;
  }
  // (clamped in float first: a corner close to w = 0 projects far outside the int range)
  xmin = fmaxf(xmin, -2.f), ymin = fmaxf(ymin, -2.f), xmax = fminf(xmax, (float)w + 2.f), ymax = fminf(ymax, (float)h + 2.f);
  x0 = max((int)floorf(xmin - 0.5f) - 1, 0), x1 = min((int)floorf(xmax - 0.5f) + 1, w - 1);
  y0 = max((int)floorf(ymin - 0.5f) - 1, 0), y1 = min((int)floorf(ymax - 0.5f) + 1, h - 1);
  return x0 <= x1 && y0 <= y1;
}

// the quad's plane at the centre of pixel (px, py): false if no fragment (the plane is seen edge-on, lies behind the eye there, is
// clipped by the near or far plane, or the disc test discards it)
__device__ __forceinline__ bool render_frag(const RenderQuad& q, int px, int py, int w, int h, RenderFrag& f) {
  const float xn = (float)(2 * px + 1 - w) / (float)w, yn = (float)(2 * py + 1 - h) / (float)h;
  float ax[3], ay[3];
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    ax[k] = q.X[k] - xn * q.W[k];
    ay[k] = q.Y[k] - yn * q.W[k];
  }
  const float e0 = ax[1] * ay[2] - ay[1] * ax[2], e1 = ax[2] * ay[0] - ay[2] * ax[0], e2 = ax[0] * ay[1] - ay[0] * ax[1];
  const float S = (e0 + e1) + e2;
  if (!(S != 0.f)) return false;
  f.b[0] = e0 / S, f.b[1] = e1 / S, f.b[2] = e2 / S;
  f.u = (f.b[1] - f.b[0]) - f.b[2];
  f.v = (f.b[2] - f.b[0]) - f.b[1];
  const float Wp = (f.b[0] * q.W[0] + f.b[1] * q.W[1]) + f.b[2] * q.W[2];
  const float Zp = (f.b[0] * q.Z[0] + f.b[1] * q.Z[1]) + f.b[2] * q.Z[2];
  if (!(Wp > 0.f) || !(Zp >= -Wp) || !(Zp <= Wp)) return false;
  if (f.u * f.u + f.v * f.v > 1.0f) return false;
  f.zw = (Zp / Wp) * 0.5f + 0.5f;
  return true;
}

// 24-bit window depth as the project's depth24 quantises it (ef_map.cu), the fragment shader's push of unstable surfels included
__device__ __forceinline__ unsigned int render_d24(const RenderQuad& q, const RenderFrag& f) {
  float zw = q.unstable ? f.zw + q.rad : f.zw;
  if (!(zw > 0.f)) zw = 0.f;
  if (zw > 1.f) zw = 1.f;
  return (unsigned int)rintf(zw * 16777215.0f);
}

__device__ __forceinline__ RenderQuad quad_of(const float (&C4)[4][4], const float4& pc, const float4& nr, float threshold) {
  RenderQuad q;
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    q.X[k] = C4[k][0];
    q.Y[k] = C4[k][1];
    q.Z[k] = C4[k][2];
    q.W[k] = C4[k][3];
  }
  q.rad = nr.w;
  q.unstable = pc.w <= threshold;
  return q;
}

// One warp's surviving quads, rasterised as one fragment list (the scheme of k_splat_scatter in ef_map.cu). That kernel's walk is
// not shared: its sprites are at most 2047^2 pixels, so its fragment prefix fits 32 bits, whereas a surfel here may cover the whole
// view (16384^2 at most), so this prefix is 64-bit; making the shared walk 64-bit would change k_splat_scatter's code in the
// frame's hot path for no gain there.
struct RenderWarp {
  float4 xy[32][3];          // X, Y, Z, W of strip vertex k
  float2 rad_unstable[32];
  int4 box[32];              // x0, y0, width, surfel id
  long long start[33];       // exclusive prefix of the fragment counts
};

__global__ void __launch_bounds__(RENDER_THREADS) k_render_scatter(const EfRenderView v, const float4* __restrict__ pos_conf,
                                                                   const float4* __restrict__ norm_rad, const int* __restrict__ count,
                                                                   unsigned long long* __restrict__ zbuf) {
  pdl_enter();
  __shared__ RenderWarp rw_all[RENDER_THREADS / 32];
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  RenderWarp& R = rw_all[wid];
  const int n = *count, w = v.width, h = v.height;
  const int gw = blockIdx.x * (RENDER_THREADS / 32) + wid, nw = gridDim.x * (RENDER_THREADS / 32);
  for (long long base = (long long)gw * 32; base < n; base += (long long)nw * 32) {
    const int id = (int)base + lane;
    int x0 = 0, y0 = 0, bw = 0;
    long long nfrag = 0;
    float C4[4][4];
    f3 P4[4];
    float4 pc = make_float4(0.f, 0.f, 0.f, 0.f), nr = pc;
    if (id < n) {
      pc = pos_conf[id];
      if (pc.w > v.threshold || v.unstable == 1) nr = norm_rad[id];
    }
    int x1, y1;
    if (id < n && render_quad(v, pc, nr, C4, P4) && render_bounds(C4, w, h, x0, x1, y0, y1)) {
      bw = x1 - x0 + 1;
      nfrag = (long long)bw * (long long)(y1 - y0 + 1);
    }
    if (!__any_sync(0xffffffffu, nfrag > 0)) continue;
    long long incl = nfrag;
#pragma unroll
    for (int off = 1; off < 32; off <<= 1) {
      const long long t = __shfl_up_sync(0xffffffffu, incl, off);
      if (lane >= off) incl += t;
    }
    const long long total = __shfl_sync(0xffffffffu, incl, 31);
    R.start[lane] = incl - nfrag;
    if (lane == 31) R.start[32] = total;
    if (nfrag > 0) {
#pragma unroll
      for (int k = 0; k < 3; ++k) R.xy[lane][k] = make_float4(C4[k][0], C4[k][1], C4[k][2], C4[k][3]);
      R.rad_unstable[lane] = make_float2(nr.w, pc.w <= v.threshold ? 1.f : 0.f);
      R.box[lane] = make_int4(x0, y0, bw, id);
    }
    __syncwarp();
    for (long long f = lane; f < total; f += 32) {
      // quad of fragment f: the last s with start[s] <= f (quads without fragments share their successor's start)
      int s = 0;
#pragma unroll
      for (int step = 16; step > 0; step >>= 1)
        if (R.start[s + step] <= f) s += step;
      const int4 bx = R.box[s];
      const long long local = f - R.start[s];
      const int ry = (int)(local / bx.z);
      const int px = bx.x + (int)(local - (long long)ry * bx.z), py = bx.y + ry;
      RenderQuad q;
#pragma unroll
      for (int k = 0; k < 3; ++k) {
        const float4 c = R.xy[s][k];
        q.X[k] = c.x, q.Y[k] = c.y, q.Z[k] = c.z, q.W[k] = c.w;
      }
      const float2 ru = R.rad_unstable[s];
      q.rad = ru.x;
      q.unstable = ru.y != 0.f;
      RenderFrag fr;
      if (!render_frag(q, px, py, w, h, fr)) continue;
      const unsigned int d24 = render_d24(q, fr);
      if (d24 >= 16777215u) continue;  // GL_LESS against the cleared depth 1.0
      const unsigned long long key = ((unsigned long long)d24 << 32) | (unsigned int)bx.w;
      unsigned long long* slot = &zbuf[(size_t)py * w + px];
      if (__ldcg(slot) <= key) continue;  // cannot win: the slot only ever decreases
      atomicMin(slot, key);
    }
    __syncwarp();
  }
}

__device__ __forceinline__ unsigned char unorm8(float x) {
  if (!(x > 0.f)) x = 0.f;
  if (x > 1.f) x = 1.f;
  return (unsigned char)(int)rintf(x * 255.0f);
}

__device__ __forceinline__ f3 decode_color(float c) {  // color.glsl:27-34
  const int ci = (int)c;
  return mk3((float)(ci >> 16 & 0xFF) / 255.0f, (float)(ci >> 8 & 0xFF) / 255.0f, (float)(ci & 0xFF) / 255.0f);
}

// draw_global_surface.geom's vColor0: colour types 0..3 and the drawWindow dimming
__device__ __forceinline__ f3 render_colour(const EfRenderView& v, const float4& ct, const float4& nr) {
  const f3 n = mk3(nr.x, nr.y, nr.z);
  f3 c;
  if (v.color_type == 1) {
    c = n;
  } else if (v.color_type == 2) {
    c = decode_color(ct.x);
  } else if (v.color_type == 3) {  // (time <= 1 divides by zero, as the shader does)
    const float ratio = (2.0f * (ct.z - 1.0f)) / ((float)v.time - 1.0f);
    c.x = gmax(0.f, 1.f - ratio);
    c.y = gmax(0.f, ratio - 1.f);
    c.z = (1.0f - c.x) - c.y;
    const float k = fabsf(dot(n, mk3(1.f, 1.f, 1.f))) + 0.1f;
    c = mk3(c.x * k, c.y * k, c.z * k);
  } else {
    const float k = 0.5f * fabsf(dot(n, mk3(1.f, 1.f, 1.f))) + 0.1f;
    c = mk3(k, k, k);
  }
  if (v.draw_window == 1 && (float)v.time - ct.w > (float)v.time_delta) c = c * 0.25f;
  return c;
}

// draw_global_surface_phong.frag at world position p: lightpos is the model-view translation and the view vector is -p, as written
__device__ __forceinline__ f3 render_phong(const EfRenderView& v, const f3& col, const f3& nrm, const f3& p) {
  const f3 n = nrm * v.sign_mult;
  const f3 light = normalized(mk3(v.mv[12], v.mv[13], v.mv[14]) - p);
  const float NdotL = dot(n, light);
  f3 out = col * 0.3f;
  if (NdotL > 0.0f) out = out + col * NdotL;
  const f3 r = normalized((n * 2.0f) * NdotL - light);
  const float RdotV = dot(r, normalized(mk3(-p.x, -p.y, -p.z)));
  if (RdotV > 0.0f) {
    float s = RdotV * RdotV;  // RdotV^32 by five squarings
    s = s * s, s = s * s, s = s * s, s = s * s;
    out = out + mk3(s, s, s);
  }
  return out;
}

__global__ void k_render_resolve(const EfRenderView v, const float4* __restrict__ pos_conf, const float4* __restrict__ color_time,
                                 const float4* __restrict__ norm_rad, unsigned long long* __restrict__ zbuf, uchar4* __restrict__ out) {
  pdl_enter();
  const int w = v.width, n_px = v.width * v.height;
  for (int p = blockIdx.x * blockDim.x + threadIdx.x; p < n_px; p += gridDim.x * blockDim.x) {
    const unsigned long long key = zbuf[p];
    if (key == kEmptyKey) {
      out[p] = make_uchar4(0, 0, 0, 0);
      continue;
    }
    zbuf[p] = kEmptyKey;
    const uint32_t id = (uint32_t)(key & 0xffffffffull);
    const float4 nr = norm_rad[id];
    f3 col = render_colour(v, color_time[id], nr);
    if (v.phong) {
      const float4 pc = pos_conf[id];
      float C4[4][4];
      f3 P4[4];
      render_quad(v, pc, nr, C4, P4);
      const RenderQuad q = quad_of(C4, pc, nr, v.threshold);
      RenderFrag f;
      render_frag(q, p % w, p / w, w, v.height, f);
      const f3 pos = (P4[0] * f.b[0] + P4[1] * f.b[1]) + P4[2] * f.b[2];
      col = render_phong(v, col, mk3(nr.x, nr.y, nr.z), pos);
    }
    out[p] = make_uchar4(unorm8(col.x), unorm8(col.y), unorm8(col.z), 255);
  }
}

RenderBuffers* buffers(EfContext* ctx) {
  if (!ctx->render) ctx->render = new RenderBuffers();
  return static_cast<RenderBuffers*>(ctx->render);
}

// grows *p to at least `bytes` (never shrinks); true if it was reallocated
template <typename T>
int grow(EfContext* ctx, T** p, size_t& have, size_t bytes, bool* grown) {
  *grown = bytes > have;
  if (!*grown) return 0;
  // (waits for the pass in flight that may still use the old buffer)
  CU(cudaStreamSynchronize(ctx->stream));
  if (*p) CU(cudaFree(*p));
  *p = nullptr;
  have = 0;
  CU(cudaMalloc((void**)p, bytes));
  have = bytes;
  return 0;
}

}  // namespace

namespace ef {

int offframe_zbuf(EfContext* ctx, size_t n, unsigned long long** out) {
  RenderBuffers* b = buffers(ctx);
  bool grown = false;
  RC(grow(ctx, &b->zbuf, b->zbuf_bytes, n * sizeof(unsigned long long), &grown));
  if (grown) CU(cudaMemsetAsync(b->zbuf, 0xff, b->zbuf_bytes, ctx->stream));
  *out = b->zbuf;
  return 0;
}

int offframe_staging(EfContext* ctx, size_t bytes, uint8_t** out) {
  RenderBuffers* b = buffers(ctx);
  bool grown = false;
  RC(grow(ctx, &b->staging, b->staging_bytes, bytes, &grown));
  *out = b->staging;
  return 0;
}

int render_map_async(EfContext* ctx, const EfRenderView* v, uint8_t* rgba_dev) {
  const size_t n = (size_t)v->width * v->height;
  unsigned long long* zbuf = nullptr;
  RC(offframe_zbuf(ctx, n, &zbuf));
  uchar4* out = reinterpret_cast<uchar4*>(rgba_dev);
  const MapDev& m = ctx->map;
  EF_LAUNCH(ctx, k_render_scatter, ctx->num_sms * 4, RENDER_THREADS, 0, *v, m.pos_conf, m.norm_rad, m.count, zbuf);
  EF_LAUNCH(ctx, k_render_resolve, wave_blocks(ctx, n), 256, 0, *v, m.pos_conf, m.color_time, m.norm_rad, zbuf, out);
  CHECK_LAST();
  return 0;
}

void render_free(EfContext* ctx) {
  RenderBuffers* b = static_cast<RenderBuffers*>(ctx->render);
  if (!b) return;
  if (b->zbuf) cudaFree(b->zbuf);
  if (b->staging) cudaFree(b->staging);
  delete b;
  ctx->render = nullptr;
}

}  // namespace ef
