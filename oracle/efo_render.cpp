// TEST INFRASTRUCTURE ONLY — CPU oracle of the global-surface render (libef_render_oracle.so, built by oracle/ef_render_oracle.py):
// draw_global_surface.{vert,geom,frag} / draw_global_surface_phong.frag as GlobalModel::renderPointCloud (GlobalModel.cpp:286-350)
// and the colour pass of GUI::drawFXAA (Tools/GUI.h:273-345) run them. PARITY PINNED against those shader files executed unmodified
// on Mesa llvmpipe (oracle/gl/ref_gl_render.cpp -> tests/golden/ref_render_*.npz, compared in tests/test_render_golden.py).
// Conventions as oracle/efo_map.cpp: IEEE fp32, no contraction (-ffp-contract=off), mat4 * vec4 accumulated left to right,
// window depth quantised as round(z * (2^24 - 1)), GL_LESS with the earlier primitive winning ties.
#include <stdint.h>

#include <algorithm>
#include <cfloat>
#include <vector>

#include "efo_common.h"

using namespace efo;

extern "C" {
/* the layout of EfRenderView (include/efusion_b200.h) */
typedef struct {
  int32_t width, height;
  float mvp[16];
  float mv[16];
  float threshold;
  int32_t color_type, unstable, draw_window, time, time_delta, phong;
  float sign_mult;
} EfoRenderView;
}

namespace {
// color.glsl:27-34
inline f3 decode_color(float c) {
  int ci = (int)c;
  return mk3((float)(ci >> 16 & 0xFF) / 255.0f, (float)(ci >> 8 & 0xFF) / 255.0f, (float)(ci & 0xFF) / 255.0f);
}
inline uint32_t depth24(float zw) {
  if (!(zw > 0.f)) zw = 0.f;
  if (zw > 1.f) zw = 1.f;
  return (uint32_t)rintf(zw * 16777215.0f);
}
inline void atomic_min_u64(uint64_t* addr, uint64_t v) {
  uint64_t old = __atomic_load_n(addr, __ATOMIC_RELAXED);
  while (v < old && !__atomic_compare_exchange_n(addr, &old, v, true, __ATOMIC_RELAXED, __ATOMIC_RELAXED)) {
  }
}
const uint64_t kEmptyKey = ~0ull;
}  // namespace

// The geometry shader emits each surfel as a 4-vertex strip (two triangles) with texcoords (-1,-1), (1,-1), (-1,1), (1,1) and the
// fragment shader discards dot(tc, tc) > 1. The disc lies inside the quad and both triangles lie on one plane with one affine map
// from texcoord to position, so the two triangles' coverage reduces to the disc test on the plane's perspective-correct
// interpolants. Those come from the homogeneous barycentrics of the first triangle at the pixel centre, which also clip against the
// near and far planes (-w <= z <= w, w > 0) without building clipped polygons. Same float formulation as ef_render.cu.
namespace {
struct RenderQuad {
  float X[3], Y[3], Z[3], W[3];  // clip coordinates of strip vertices 0, 1, 2
  f3 P[3];                       // their world positions
  float rad;
  bool unstable;
};
inline float clipc(const float* m, int r, const f3& p) { return ((m[r] * p.x + m[4 + r] * p.y) + m[8 + r] * p.z) + m[12 + r]; }
// draw_global_surface.geom: the strip's corners (p+x, p+y, p-y, p-x) in clip space. False: culled by the vertex shader.
inline bool render_quad(const float* s, const EfoRenderView* v, RenderQuad& q, float (&C4)[4][4]) {
  if (!(s[3] > v->threshold || v->unstable == 1)) return false;
  const f3 p = mk3(s[0], s[1], s[2]), n = mk3(s[8], s[9], s[10]);
  const f3 x = normalized(mk3(n.y - n.z, -n.x, n.x)) * s[11] * 1.41421356f;
  const f3 y = cross(n, x);
  const f3 P4[4] = {p + x, p + y, p - y, p - x};
  for (int k = 0; k < 4; ++k)
    for (int r = 0; r < 4; ++r) C4[k][r] = clipc(v->mvp, r, P4[k]);
  for (int k = 0; k < 3; ++k) {
    q.X[k] = C4[k][0];
    q.Y[k] = C4[k][1];
    q.Z[k] = C4[k][2];
    q.W[k] = C4[k][3];
    q.P[k] = P4[k];
  }
  q.rad = s[11];
  q.unstable = s[3] <= v->threshold;
  return true;
}
// pixel range of the quad, false if nothing of it can be visible. All w > 0: the corners' window bounding box, one pixel of slack
// each side; w changes sign: the whole view.
inline bool render_bounds(const float (&C4)[4][4], int w, int h, int& x0, int& x1, int& y0, int& y1) {
  int pos = 0, behind_near = 0, beyond_far = 0;
  float xmin = FLT_MAX, xmax = -FLT_MAX, ymin = FLT_MAX, ymax = -FLT_MAX;
  for (int k = 0; k < 4; ++k) {
    const float W = C4[k][3];
    pos += W > 0.f;
    behind_near += C4[k][2] < -W;
    beyond_far += C4[k][2] > W;
    if (W > 0.f) {
      const float xw = ((C4[k][0] / W) * 0.5f + 0.5f) * (float)w, yw = ((C4[k][1] / W) * 0.5f + 0.5f) * (float)h;
      xmin = std::min(xmin, xw);
      xmax = std::max(xmax, xw);
      ymin = std::min(ymin, yw);
      ymax = std::max(ymax, yw);
    }
  }
  if (pos == 0 || behind_near == 4 || beyond_far == 4) return false;
  if (pos < 4) {
    x0 = 0, x1 = w - 1, y0 = 0, y1 = h - 1;
    return true;
  }
  // (clamped in float first: a corner close to w = 0 projects far outside the int range)
  xmin = std::max(xmin, -2.f), ymin = std::max(ymin, -2.f), xmax = std::min(xmax, (float)w + 2.f), ymax = std::min(ymax, (float)h + 2.f);
  x0 = std::max((int)floorf(xmin - 0.5f) - 1, 0), x1 = std::min((int)floorf(xmax - 0.5f) + 1, w - 1);
  y0 = std::max((int)floorf(ymin - 0.5f) - 1, 0), y1 = std::min((int)floorf(ymax - 0.5f) + 1, h - 1);
  return x0 <= x1 && y0 <= y1;
}
struct RenderFrag {
  float b[3];  // homogeneous barycentrics of strip vertices 0, 1, 2
  float u, v;  // texcoord
  float Wp, Zp;  // clip w and z
  float zw;      // window depth (gl_FragCoord.z)
};
// the quad's plane at the centre of pixel (px, py); false: no fragment (behind the eye or clipped by the near / far plane). f.u,
// f.v are set whenever the plane projects to the pixel, so the caller applies the disc test.
inline bool render_frag(const RenderQuad& q, int px, int py, int w, int h, RenderFrag& f) {
  const float xn = (float)(2 * px + 1 - w) / (float)w, yn = (float)(2 * py + 1 - h) / (float)h;
  float ax[3], ay[3];
  for (int k = 0; k < 3; ++k) {
    ax[k] = q.X[k] - xn * q.W[k];
    ay[k] = q.Y[k] - yn * q.W[k];
  }
  const float e0 = ax[1] * ay[2] - ay[1] * ax[2], e1 = ax[2] * ay[0] - ay[2] * ax[0], e2 = ax[0] * ay[1] - ay[0] * ax[1];
  const float S = (e0 + e1) + e2;
  if (!(S != 0.f)) {  // the plane is seen edge-on
    f.Wp = 0.f;
    return false;
  }
  f.b[0] = e0 / S, f.b[1] = e1 / S, f.b[2] = e2 / S;
  f.u = (f.b[1] - f.b[0]) - f.b[2];
  f.v = (f.b[2] - f.b[0]) - f.b[1];
  f.Wp = (f.b[0] * q.W[0] + f.b[1] * q.W[1]) + f.b[2] * q.W[2];
  f.Zp = (f.b[0] * q.Z[0] + f.b[1] * q.Z[1]) + f.b[2] * q.Z[2];
  if (!(f.Wp > 0.f) || !(f.Zp >= -f.Wp) || !(f.Zp <= f.Wp)) return false;
  f.zw = (f.Zp / f.Wp) * 0.5f + 0.5f;
  return true;
}
inline bool render_disc(const RenderFrag& f) { return !(f.u * f.u + f.v * f.v > 1.0f); }
// 24-bit window depth of a fragment, the fragment shader's push of unstable surfels included; >= 0xFFFFFF never passes GL_LESS
inline uint32_t render_d24(const RenderQuad& q, const RenderFrag& f) { return depth24(q.unstable ? f.zw + q.rad : f.zw); }
inline uint8_t unorm8(float x) {
  if (!(x > 0.f)) x = 0.f;
  if (x > 1.f) x = 1.f;
  return (uint8_t)(int)rintf(x * 255.0f);
}
// the geometry shader's vColor0 (colour types 0..3 and the drawWindow dimming)
inline f3 render_colour(const float* s, const EfoRenderView* v) {
  const f3 n = mk3(s[8], s[9], s[10]);
  f3 c;
  if (v->color_type == 1) {
    c = n;
  } else if (v->color_type == 2) {
    c = decode_color(s[4]);
  } else if (v->color_type == 3) {
    const float ratio = (2.0f * (s[6] - 1.0f)) / ((float)v->time - 1.0f);
    c.x = std::max(0.f, 1.f - ratio);
    c.y = std::max(0.f, ratio - 1.f);
    c.z = (1.0f - c.x) - c.y;
    const float k = fabsf(dot(n, mk3(1.f, 1.f, 1.f))) + 0.1f;
    c = mk3(c.x * k, c.y * k, c.z * k);
  } else {
    const float k = 0.5f * fabsf(dot(n, mk3(1.f, 1.f, 1.f))) + 0.1f;
    c = mk3(k, k, k);
  }
  if (v->draw_window == 1 && (float)v->time - s[7] > (float)v->time_delta) c = c * 0.25f;
  return c;
}
// draw_global_surface_phong.frag at world position p (lightpos = the model-view translation; the view vector is -p, as written)
inline f3 render_phong(const f3& col, const f3& nrm, const f3& p, const EfoRenderView* v) {
  const f3 n = nrm * v->sign_mult;
  const f3 light = normalized(mk3(v->mv[12], v->mv[13], v->mv[14]) - p);
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
}  // namespace

// keys (optional): the winning key per pixel, (d24 << 32) | id, ~0 where nothing was drawn
extern "C" void efo_render(const float* map, int count, const EfoRenderView* v, uint8_t* rgba, uint64_t* keys) {
  const int w = v->width, h = v->height;
  const size_t n = (size_t)w * h;
  std::vector<uint64_t> zbuf(n, kEmptyKey);
#pragma omp parallel for schedule(dynamic, 1024)
  for (int id = 0; id < count; ++id) {
    RenderQuad q;
    float C4[4][4];
    int x0, x1, y0, y1;
    if (!render_quad(map + (size_t)id * 12, v, q, C4) || !render_bounds(C4, w, h, x0, x1, y0, y1)) continue;
    for (int py = y0; py <= y1; ++py)
      for (int px = x0; px <= x1; ++px) {
        RenderFrag f;
        if (!render_frag(q, px, py, w, h, f) || !render_disc(f)) continue;
        const uint32_t d24 = render_d24(q, f);
        if (d24 >= 16777215u) continue;
        atomic_min_u64(&zbuf[(size_t)py * w + px], ((uint64_t)d24 << 32) | (uint32_t)id);
      }
  }
#pragma omp parallel for schedule(static)
  for (int p = 0; p < (int)n; ++p) {
    uint8_t* o = rgba + (size_t)p * 4;
    if (keys) keys[p] = zbuf[p];
    if (zbuf[p] == kEmptyKey) {
      o[0] = o[1] = o[2] = o[3] = 0;
      continue;
    }
    const uint32_t id = (uint32_t)(zbuf[p] & 0xffffffffu);
    const float* s = map + (size_t)id * 12;
    f3 col = render_colour(s, v);
    if (v->phong) {
      RenderQuad q;
      float C4[4][4];
      RenderFrag f;
      render_quad(s, v, q, C4);
      render_frag(q, p % w, p / w, w, h, f);
      const f3 pos = (q.P[0] * f.b[0] + q.P[1] * f.b[1]) + q.P[2] * f.b[2];
      col = render_phong(col, mk3(s[8], s[9], s[10]), pos, v);
    }
    o[0] = unorm8(col.x);
    o[1] = unorm8(col.y);
    o[2] = unorm8(col.z);
    o[3] = 255;
  }
}

// What tells a pixel's disagreement with another rasteriser apart, per pixel over every fragment of every surfel whose plane reaches
// the pixel centre with dot(tc, tc) <= 1 + slack: rim = min |dot(tc, tc) - 1| (the disc test decided by rounding); edge = the least
// distance in texcoord units to the strip's diagonal or to the quad's border, or in NDC depth to the near or far plane (the triangle
// set-up or the clipper decided); runner = the least key of a surfel other than the winner's (a depth tie decided by rounding).
extern "C" void efo_render_margins(const float* map, int count, const EfoRenderView* v, const uint64_t* keys, float slack, float* rim,
                                   float* edge, uint64_t* runner) {
  const int w = v->width, h = v->height;
  const size_t n = (size_t)w * h;
  for (size_t p = 0; p < n; ++p) rim[p] = edge[p] = FLT_MAX, runner[p] = kEmptyKey;
  for (int id = 0; id < count; ++id) {
    RenderQuad q;
    float C4[4][4];
    int x0, x1, y0, y1;
    if (!render_quad(map + (size_t)id * 12, v, q, C4) || !render_bounds(C4, w, h, x0, x1, y0, y1)) continue;
    for (int py = y0; py <= y1; ++py)
      for (int px = x0; px <= x1; ++px) {
        const size_t p = (size_t)py * w + px;
        RenderFrag f;
        const bool ok = render_frag(q, px, py, w, h, f);
        if (!(f.Wp > 0.f)) continue;
        const float r2 = f.u * f.u + f.v * f.v;
        if (!ok) {  // clipped by the near or far plane: its distance to the plane is an edge margin as well
          if (r2 <= 1.f + slack) edge[p] = std::min(edge[p], std::min(fabsf(f.Zp / f.Wp + 1.f), fabsf(f.Zp / f.Wp - 1.f)));
          continue;
        }
        if (r2 > 1.f + slack) continue;
        rim[p] = std::min(rim[p], fabsf(r2 - 1.f));
        const float ndc = f.zw * 2.f - 1.f;
        const float e = std::min(std::min(fabsf(f.u + f.v) * 0.70710678f, std::min(1.f - fabsf(f.u), 1.f - fabsf(f.v))),
                                 std::min(fabsf(ndc + 1.f), fabsf(ndc - 1.f)));
        edge[p] = std::min(edge[p], e);
        if (!render_disc(f)) continue;
        const uint32_t d24 = render_d24(q, f);
        if (d24 >= 16777215u || (keys[p] != kEmptyKey && (uint32_t)(keys[p] & 0xffffffffu) == (uint32_t)id)) continue;
        runner[p] = std::min(runner[p], ((uint64_t)d24 << 32) | (uint32_t)id);
      }
  }
}
