// Depth preprocess: ElasticFusion::filterDepth + metriciseDepth of the reference
// (Core/ElasticFusion.cpp:655-673; Core/Shaders/depth_bilateral.frag:30-75, depth_metric.frag:28-39) as ONE launch:
// the 13x13 bilateral filter on raw uint16 millimetres plus both metric conversions (raw and filtered), instead of three
// full-screen GL passes each followed by glFinish.
#include "ef_device.cuh"
#include "ef_internal.h"

using namespace ef;

namespace {
constexpr int TILE_X = 32, TILE_Y = 8, R = 6;
constexpr int SM_W = TILE_X + 2 * R, SM_H = TILE_Y + 2 * R;
}  // namespace

__global__ void __launch_bounds__(TILE_X* TILE_Y) k_preprocess_depth(const uint16_t* __restrict__ depth, int rows, int cols, float maxD,
                                                                      uint16_t* __restrict__ filtered, float* __restrict__ metric,
                                                                      float* __restrict__ metric_filtered) {
  pdl_enter();
  // stage the (32+12) x (8+12) neighbourhood once per CTA; out-of-image taps are never read (the window is clipped)
  __shared__ float tile[SM_H][SM_W + 1];
  const int x0 = blockIdx.x * TILE_X - R, y0 = blockIdx.y * TILE_Y - R;
  for (int i = threadIdx.y * TILE_X + threadIdx.x; i < SM_W * SM_H; i += TILE_X * TILE_Y) {
    const int ty = i / SM_W, tx = i - ty * SM_W;
    const int gx = x0 + tx, gy = y0 + ty;
    tile[ty][tx] = (gx >= 0 && gy >= 0 && gx < cols && gy < rows) ? (float)depth[(size_t)gy * cols + gx] : 0.f;
  }
  __syncthreads();
  const int x = blockIdx.x * TILE_X + threadIdx.x, y = blockIdx.y * TILE_Y + threadIdx.y;
  if (x >= cols || y >= rows) return;
  const size_t p = (size_t)y * cols + x;
  const unsigned int hi = (unsigned int)(maxD * 1000.0f);
  const unsigned int value = depth[p];
  const bool gated = (value > hi || value < 300U);
  if (metric) metric[p] = gated ? 0.f : (float)value / 1000.0f;
  unsigned int out = 0;
  if (!gated) {
    const float sigma_space2_inv_half = 0.024691358f;
    const float sigma_color2_inv_half = 0.000555556f;
    const int D = R * 2 + 1;
    const int tx = min(x - D / 2 + D, cols);
    const int ty = min(y - D / 2 + D, rows);
    float sum1 = 0, sum2 = 0;
    const float fv = (float)value;
    for (int cy = max(y - D / 2, 0); cy < ty; ++cy) {
      const float dy = (float)y - (float)cy;
      const float* trow = tile[cy - y0];
      for (int cx = max(x - D / 2, 0); cx < tx; ++cx) {
        const float tmp = trow[cx - x0];
        const float dx = (float)x - (float)cx;
        const float space2 = dx * dx + dy * dy;
        const float color2 = (fv - tmp) * (fv - tmp);
        const float weight = expf(-(space2 * sigma_space2_inv_half + color2 * sigma_color2_inv_half));
        sum1 += tmp * weight;
        sum2 += weight;
      }
    }
    out = (unsigned int)roundf(sum1 / sum2);
  }
  if (filtered) filtered[p] = (uint16_t)out;
  if (metric_filtered) metric_filtered[p] = (out > hi || out < 300U) ? 0.f : (float)out / 1000.0f;
}

// GL_RGB upload into the RGBA8 texture the tracker samples (alpha = 255)
__global__ void k_rgb_to_rgba(const uint8_t* __restrict__ rgb, uchar4* __restrict__ rgba, size_t n) {
  pdl_enter();
  for (size_t p = (size_t)blockIdx.x * blockDim.x + threadIdx.x; p < n; p += (size_t)gridDim.x * blockDim.x)
    rgba[p] = make_uchar4(rgb[p * 3 + 0], rgb[p * 3 + 1], rgb[p * 3 + 2], 255);
}

namespace ef {
int preprocess_depth(EfContext* ctx, int rows, int cols, const uint16_t* raw, float cutoff, uint16_t* filtered, float* metric,
                     float* metric_filtered) {
  dim3 grid((cols + TILE_X - 1) / TILE_X, (rows + TILE_Y - 1) / TILE_Y), block(TILE_X, TILE_Y);
  EF_LAUNCH(ctx, k_preprocess_depth, grid, block, 0, raw, rows, cols, cutoff, filtered, metric, metric_filtered);
  CHECK_LAST();
  return 0;
}
int rgb_to_rgba(EfContext* ctx, int rows, int cols, const uint8_t* rgb, uint8_t* rgba) {
  const size_t n = (size_t)rows * cols;
  EF_LAUNCH(ctx, k_rgb_to_rgba, wave_blocks(ctx, n), 256, 0, rgb, (uchar4*)rgba, n);
  CHECK_LAST();
  return 0;
}
}  // namespace ef
