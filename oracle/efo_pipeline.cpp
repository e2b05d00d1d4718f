// TEST INFRASTRUCTURE ONLY — CPU oracle, whole-frame pipeline.
// Restates ElasticFusion::processFrame / predict / filterDepth / metriciseDepth (Core/ElasticFusion.cpp:270-673)
// for the open-loop configuration (closeLoops == false, reloc == false): Ferns, deformation graphs and the
// INACTIVE model-to-model branch are out of scope (SURVEY.md §8).
#include "ef_oracle.h"
#include "efo_common.h"
#include "efo_linalg.h"

#include <chrono>
#include <cstdio>
#include <vector>

namespace {
double now_s() {
  return std::chrono::duration<double>(std::chrono::steady_clock::now().time_since_epoch()).count();
}
}  // namespace

struct EfoFusion {
  EfoConfig cfg;
  EfoOdometry* frameToModel;
  int rows, cols;
  float cam4[4];
  int tick;
  double T_wc[16];
  float maxDepthProcessed;

  std::vector<uint8_t> rgb, rgba;
  std::vector<uint16_t> depthRaw, depthFiltered;
  std::vector<float> depthMetric, depthMetricFiltered;

  std::vector<float> map, mapTmp, newUnstable, rawFb, filtFb;
  int count;

  std::vector<uint32_t> indexTex;
  std::vector<float> vertConf, colorTime, normRad;

  std::vector<uint8_t> imageTex, fillImage;
  std::vector<float> vertexTex, normalTex, fillVertex, fillNormal;
  std::vector<uint16_t> timeTex;

  // local loop closure front half (ElasticFusion.cpp:447-505)
  EfoOdometry* modelToModel;
  bool closeLoops;
  int icpCountThresh;
  float icpErrThresh, covThresh;
  std::vector<uint8_t> oldImage;
  std::vector<float> oldVertex, oldNormal, synthDepth;
  std::vector<uint16_t> oldTime;
  EfoLoopResult loop;
  std::vector<double> consSrc, consDst;
  std::vector<int32_t> consTime;

  double timers[4];
  float lastWeighting;
  EfoTrackerBackend ext;
  bool has_ext;
};

extern "C" EfoFusion* efo_fusion_create(const EfoConfig* cfg) {
  EfoFusion* f = new EfoFusion();
  f->cfg = *cfg;
  f->rows = cfg->height;
  f->cols = cfg->width;
  f->cam4[0] = cfg->cx;
  f->cam4[1] = cfg->cy;
  f->cam4[2] = cfg->fx;
  f->cam4[3] = cfg->fy;
  // RGBDOdometry defaults: distThresh 0.10, angleThresh sin(20*3.14159254/180) (RGBDOdometry.h:41-42)
  f->frameToModel = efo_odom_create(cfg->width, cfg->height, cfg->cx, cfg->cy, cfg->fx, cfg->fy, 0.10f,
                                    sinf(20.f * 3.14159254f / 180.f));
  f->modelToModel = efo_odom_create(cfg->width, cfg->height, cfg->cx, cfg->cy, cfg->fx, cfg->fy, 0.10f, sinf(20.f * 3.14159254f / 180.f));
  f->closeLoops = false;
  f->icpCountThresh = 35000;
  f->icpErrThresh = 5e-05f;
  f->covThresh = 1e-05f;
  memset(&f->loop, 0, sizeof(f->loop));
  f->tick = 1;
  for (int i = 0; i < 16; ++i) f->T_wc[i] = (i % 5 == 0) ? 1.0 : 0.0;
  f->maxDepthProcessed = 20.0f;
  const size_t n = (size_t)f->rows * f->cols;
  f->rgb.assign(n * 3, 0);
  f->rgba.assign(n * 4, 0);
  f->depthRaw.assign(n, 0);
  f->depthFiltered.assign(n, 0);
  f->depthMetric.assign(n, 0.f);
  f->depthMetricFiltered.assign(n, 0.f);
  f->map.assign(((size_t)cfg->capacity + n) * 12, 0.f);
  f->mapTmp.assign(((size_t)cfg->capacity + n) * 12, 0.f);  // clean may emit count + new surfels before the capacity cut
  f->newUnstable.assign(n * 12, 0.f);
  f->rawFb.assign(n * 12, 0.f);
  f->filtFb.assign(n * 12, 0.f);
  f->count = 0;
  f->indexTex.assign(n, 0);
  f->vertConf.assign(n * 4, 0.f);
  f->colorTime.assign(n * 4, 0.f);
  f->normRad.assign(n * 4, 0.f);
  f->imageTex.assign(n * 4, 0);
  f->fillImage.assign(n * 4, 0);
  f->vertexTex.assign(n * 4, 0.f);
  f->normalTex.assign(n * 4, 0.f);
  f->fillVertex.assign(n * 4, 0.f);
  f->fillNormal.assign(n * 4, 0.f);
  f->timeTex.assign(n, 0);
  f->oldImage.assign(n * 4, 0);
  f->oldVertex.assign(n * 4, 0.f);
  f->oldNormal.assign(n * 4, 0.f);
  f->oldTime.assign(n, 0);
  f->synthDepth.assign(n, 0.f);
  for (int i = 0; i < 4; ++i) f->timers[i] = 0;
  f->lastWeighting = 0;
  f->has_ext = false;
  return f;
}

extern "C" void efo_fusion_destroy(EfoFusion* f) {
  efo_odom_destroy(f->frameToModel);
  efo_odom_destroy(f->modelToModel);
  delete f;
}

// ElasticFusion::predict, ElasticFusion.cpp:621-653 (lastFrameRecovery == false, lost == false)
static void predict(EfoFusion* f) {
  efo_combined_predict(f->map.data(), f->count, f->T_wc, f->maxDepthProcessed, f->cfg.confidence, f->tick, f->tick,
                       f->cfg.time_delta, f->rows, f->cols, f->cam4, f->imageTex.data(), f->vertexTex.data(),
                       f->normalTex.data(), f->timeTex.data(), nullptr, 0);
  efo_fill_vertex(f->vertexTex.data(), f->depthFiltered.data(), 0, f->rows, f->cols, f->cam4, f->fillVertex.data());
  efo_fill_normal(f->normalTex.data(), f->depthFiltered.data(), 0, f->rows, f->cols, f->cam4, f->fillNormal.data());
  efo_fill_image(f->imageTex.data(), f->rgb.data(), f->cfg.frame_to_frame_rgb ? 1 : 0, f->rows, f->cols,
                 f->fillImage.data());
}

// ElasticFusion.cpp:447-505 (the branch taken when no fern matched: always, here). Resize::vertex / Resize::time sample
// the W/20 x H/20 grid at texel centres with nearest filtering (Resize.cpp:81-159, resize.frag); the time texture is an integer
// texture read through a float sampler in the reference (formally undefined) — restated as the integer value.
static void local_loop_front_half(EfoFusion* f) {
  EfoLoopResult& L = f->loop;
  memset(&L, 0, sizeof(L));
  f->consSrc.clear();
  f->consDst.clear();
  f->consTime.clear();
  L.ran = 1;
  const int td = f->cfg.time_delta;
  efo_combined_predict(f->map.data(), f->count, f->T_wc, f->maxDepthProcessed, f->cfg.confidence, 0, f->tick - td, td, f->rows,
                       f->cols, f->cam4, f->oldImage.data(), f->oldVertex.data(), f->oldNormal.data(), f->oldTime.data(), nullptr, 0);
  // WARNING initICP* must be called before initRGB* (ElasticFusion.cpp:461-467)
  efo_odom_init_icp_model(f->modelToModel, f->oldVertex.data(), f->oldNormal.data(), f->T_wc);
  efo_odom_init_rgb_model(f->modelToModel, f->oldImage.data());
  efo_odom_init_icp_pred(f->modelToModel, f->vertexTex.data(), f->normalTex.data());
  efo_odom_init_rgb(f->modelToModel, f->imageTex.data());
  memcpy(L.T_wc_est, f->T_wc, sizeof(L.T_wc_est));
  efo_odom_track(f->modelToModel, L.T_wc_est, 0, 10.f, f->cfg.pyramid, f->cfg.fast_odom, 0, nullptr, 0);
  double cov[36];
  efo_odom_covariance(f->modelToModel, cov);
  bool covOk = true;
  for (int i = 0; i < 6; i++) {
    L.cov_diag[i] = cov[i * 6 + i];
    if (cov[i * 6 + i] > f->covThresh) covOk = false;
  }
  float st[8];
  efo_odom_stats(f->modelToModel, st);
  L.lastICPError = st[0];
  L.lastICPCount = st[1];
  if (covOk && st[1] > (float)f->icpCountThresh && st[0] < f->icpErrThresh) {
    L.accepted = 1;
    const int dcols = f->cols / 20, drows = f->rows / 20;
    for (int i = 0; i < dcols; i++)
      for (int j = 0; j < drows; j++) {
        const int sx = std::min(f->cols - 1, (int)floorf((((float)i + 0.5f) / (float)dcols) * (float)f->cols));
        const int sy = std::min(f->rows - 1, (int)floorf((((float)j + 0.5f) / (float)drows) * (float)f->rows));
        const float* v = f->vertexTex.data() + ((size_t)sy * f->cols + sx) * 4;
        const uint16_t t = f->oldTime[(size_t)sy * f->cols + sx];
        if (v[2] > 0 && v[2] < f->maxDepthProcessed && t > 0) {
          for (int pass = 0; pass < 2; ++pass) {
            const double* T = pass == 0 ? f->T_wc : L.T_wc_est;
            std::vector<double>& dst = pass == 0 ? f->consSrc : f->consDst;
            for (int r = 0; r < 3; ++r) dst.push_back(T[r * 4 + 0] * (double)v[0] + T[r * 4 + 1] * (double)v[1] + T[r * 4 + 2] * (double)v[2] + T[r * 4 + 3]);
          }
          f->consTime.push_back((int32_t)t);
        }
      }
    L.n_constraints = (int)f->consTime.size();
  }
}

extern "C" void efo_fusion_set_loop_closure(EfoFusion* f, int enabled, int count_thresh, float err_thresh, float cov_thresh) {
  f->closeLoops = enabled != 0;
  f->icpCountThresh = count_thresh;
  f->icpErrThresh = err_thresh;
  f->covThresh = cov_thresh;
}
extern "C" int efo_fusion_loop_result(const EfoFusion* f, EfoLoopResult* out, double* src3, double* dst3, int32_t* times, int max_constraints) {
  if (out) *out = f->loop;
  const int n = std::min((int)f->consTime.size(), max_constraints);
  if (src3) memcpy(src3, f->consSrc.data(), sizeof(double) * 3 * n);
  if (dst3) memcpy(dst3, f->consDst.data(), sizeof(double) * 3 * n);
  if (times) memcpy(times, f->consTime.data(), sizeof(int32_t) * n);
  return n;
}

extern "C" void efo_fusion_process_frame(EfoFusion* f, const uint8_t* rgb, const uint16_t* depth, int64_t timestamp,
                                         float weightMultiplier, const double* in_T_wc) {
  efo_fusion_process_frame_deform(f, rgb, depth, timestamp, weightMultiplier, in_T_wc, nullptr, nullptr, 0, 0);
}

extern "C" void efo_fusion_process_frame_deform(EfoFusion* f, const uint8_t* rgb, const uint16_t* depth, int64_t timestamp,
                                                float weightMultiplier, const double* in_T_wc, const double* T_override,
                                                const float* nodes, int n_nodes, int fern_accepted) {
  (void)timestamp;
  const size_t n = (size_t)f->rows * f->cols;
  double t0 = now_s();
  memcpy(f->rgb.data(), rgb, n * 3);
  memcpy(f->depthRaw.data(), depth, n * 2);
  for (size_t i = 0; i < n; ++i) {  // GL_RGB upload into an RGBA8 texture: alpha = 255
    f->rgba[i * 4 + 0] = rgb[i * 3 + 0];
    f->rgba[i * 4 + 1] = rgb[i * 3 + 1];
    f->rgba[i * 4 + 2] = rgb[i * 3 + 2];
    f->rgba[i * 4 + 3] = 255;
  }
  // filterDepth + metriciseDepth, ElasticFusion.cpp:284-285,655-673
  efo_bilateral(f->depthRaw.data(), f->rows, f->cols, f->cfg.depth_cutoff, f->depthFiltered.data());
  efo_metric(f->depthRaw.data(), f->rows, f->cols, f->cfg.depth_cutoff, f->depthMetric.data());
  efo_metric(f->depthFiltered.data(), f->rows, f->cols, f->cfg.depth_cutoff, f->depthMetricFiltered.data());
  double t1 = now_s();
  f->timers[0] += t1 - t0;

  if (f->tick == 1) {
    // ElasticFusion.cpp:290-296
    int rawN = efo_feedback_buffer(f->rgb.data(), f->depthMetric.data(), f->rows, f->cols, f->cam4, f->tick,
                                   f->maxDepthProcessed, f->rawFb.data());
    int filtN = efo_feedback_buffer(f->rgb.data(), f->depthMetricFiltered.data(), f->rows, f->cols, f->cam4, f->tick,
                                    f->maxDepthProcessed, f->filtFb.data());
    f->count = efo_map_initialise(f->rawFb.data(), rawN, f->filtFb.data(), filtN, (int)n, f->map.data());
    if (f->count > f->cfg.capacity) f->count = f->cfg.capacity;
    if (f->has_ext)
      f->ext.init_first_rgb(f->ext.handle, f->rgba.data());
    else
      efo_odom_init_first_rgb(f->frameToModel, f->rgba.data());
    f->timers[2] += now_s() - t1;
  } else {
    double T_prev[16];
    memcpy(T_prev, f->T_wc, sizeof(T_prev));
    if (!in_T_wc) {
      // ElasticFusion.cpp:302-323
      bool shouldFillIn = !efo_dense_enough(f->imageTex.data(), f->rows, f->cols, 20);
      const float* mv = shouldFillIn ? f->fillVertex.data() : f->vertexTex.data();
      const float* mn = shouldFillIn ? f->fillNormal.data() : f->normalTex.data();
      const uint8_t* mi = (shouldFillIn || f->cfg.frame_to_frame_rgb) ? f->fillImage.data() : f->imageTex.data();
      if (f->has_ext) {
        f->ext.init_icp_model(f->ext.handle, mv, mn, f->T_wc);
        f->ext.init_rgb_model(f->ext.handle, mi);
        f->ext.init_icp_depth(f->ext.handle, f->depthFiltered.data(), f->maxDepthProcessed);
        f->ext.init_rgb(f->ext.handle, f->rgba.data());
        f->ext.track(f->ext.handle, f->T_wc, f->cfg.rgb_only, f->cfg.icp_weight, f->cfg.pyramid, f->cfg.fast_odom, f->cfg.so3,
                     nullptr, 0);
      } else {
        efo_odom_init_icp_model(f->frameToModel, mv, mn, f->T_wc);
        efo_odom_init_rgb_model(f->frameToModel, mi);
        efo_odom_init_icp_depth(f->frameToModel, f->depthFiltered.data(), f->maxDepthProcessed);
        efo_odom_init_rgb(f->frameToModel, f->rgba.data());
        efo_odom_track(f->frameToModel, f->T_wc, f->cfg.rgb_only, f->cfg.icp_weight, f->cfg.pyramid, f->cfg.fast_odom,
                       f->cfg.so3, nullptr, 0);
      }
    } else {
      memcpy(f->T_wc, in_T_wc, sizeof(f->T_wc));
    }
    double t2 = now_s();
    f->timers[1] += t2 - t1;

    // velocity weighting, ElasticFusion.cpp:369-383
    double inv[16], T_curr_prev[16];
    la::se3_inverse(f->T_wc, inv);
    la::mul4(inv, T_prev, T_curr_prev);
    double tn = std::sqrt(T_curr_prev[3] * T_curr_prev[3] + T_curr_prev[7] * T_curr_prev[7] + T_curr_prev[11] * T_curr_prev[11]);
    double ln = la::se3_log_norm(T_curr_prev);
    float weighting = (float)std::max(tn, ln);
    float largest = 0.01f, minWeight = 0.5f;
    if (weighting > largest) weighting = largest;
    weighting = std::max(1.0f - (weighting / largest), minWeight) * weightMultiplier;
    f->lastWeighting = weighting;

    // ElasticFusion.cpp:387 — the mid-frame predict(): its outputs are only consumed by loop closure and are
    // overwritten by the predict() at :599, but the reference pays for it, so the timed baseline does too.
    predict(f);
    f->loop.ran = 0;
    if (f->closeLoops) local_loop_front_half(f);
    if (T_override) memcpy(f->T_wc, T_override, sizeof(f->T_wc));  // T_wc_curr = T_wc_est (ElasticFusion.cpp:524)
    double t3 = now_s();
    f->timers[3] += t3 - t2;

    if (!f->cfg.rgb_only) {
      // ElasticFusion.cpp:536-585
      efo_predict_indices(f->map.data(), f->count, f->T_wc, f->tick, f->maxDepthProcessed, f->cfg.time_delta, f->rows,
                          f->cols, f->cam4, f->indexTex.data(), f->vertConf.data(), f->colorTime.data(),
                          f->normRad.data());
      int newN = efo_fuse(f->map.data(), f->count, f->T_wc, f->tick, f->rgb.data(), f->depthMetric.data(),
                          f->depthMetricFiltered.data(), f->indexTex.data(), f->vertConf.data(), f->colorTime.data(),
                          f->normRad.data(), f->maxDepthProcessed, weighting, f->rows, f->cols, f->cam4,
                          f->newUnstable.data());
      efo_predict_indices(f->map.data(), f->count, f->T_wc, f->tick, f->maxDepthProcessed, f->cfg.time_delta, f->rows,
                          f->cols, f->cam4, f->indexTex.data(), f->vertConf.data(), f->colorTime.data(),
                          f->normRad.data());
      // Transform feedback into a full buffer stops recording primitives (GL 4.x spec, "Transform Feedback": primitives that
      // do not fit are not written and not counted): the map keeps the first `capacity` surfels clean emits, in order.
      if (n_nodes > 0 && !fern_accepted)  // ElasticFusion.cpp:559-569
        efo_combined_predict(f->map.data(), f->count, f->T_wc, f->maxDepthProcessed, f->cfg.confidence, f->tick, f->tick - f->cfg.time_delta,
                             65535, f->rows, f->cols, f->cam4, nullptr, nullptr, nullptr, nullptr, f->synthDepth.data(), 1);
      f->count = efo_clean_deform(f->map.data(), f->count, f->newUnstable.data(), newN, f->T_wc, f->tick, f->indexTex.data(),
                                  f->vertConf.data(), f->colorTime.data(), f->cfg.confidence, f->cfg.time_delta, f->maxDepthProcessed,
                                  f->rows, f->cols, f->cam4, nodes, n_nodes, f->synthDepth.data(), fern_accepted, f->mapTmp.data());
      if (f->count > f->cfg.capacity) f->count = f->cfg.capacity;
      f->map.swap(f->mapTmp);
    }
    f->timers[2] += now_s() - t3;
  }

  double t4 = now_s();
  predict(f);  // ElasticFusion.cpp:599
  f->timers[3] += now_s() - t4;
  f->tick++;
}

// Replaces the model by n surfels (at most `capacity`) and re-renders the model view with predict(), as a caller that loads a map
// after the first frame would; the frame inputs predict() fills in from (filtered depth, colour) stay those of the last frame.
extern "C" void efo_fusion_set_map(EfoFusion* f, const float* surfels12, int n) {
  f->count = std::max(0, std::min(n, f->cfg.capacity));
  if (f->count > 0) memcpy(f->map.data(), surfels12, sizeof(float) * 12 * (size_t)f->count);
  predict(f);
}

extern "C" void efo_fusion_set_tracker(EfoFusion* f, const EfoTrackerBackend* b) {
  f->has_ext = b != nullptr;
  if (b) f->ext = *b;
}
extern "C" void efo_fusion_pose(const EfoFusion* f, double* T) { memcpy(T, f->T_wc, sizeof(f->T_wc)); }
extern "C" int efo_fusion_count(const EfoFusion* f) { return f->count; }
extern "C" int efo_fusion_tick(const EfoFusion* f) { return f->tick; }
extern "C" const float* efo_fusion_map(const EfoFusion* f) { return f->map.data(); }
extern "C" EfoOdometry* efo_fusion_odometry(EfoFusion* f) { return f->frameToModel; }
extern "C" const void* efo_fusion_buffer(const EfoFusion* f, int which) {
  switch (which) {
    case 0: return f->imageTex.data();
    case 1: return f->vertexTex.data();
    case 2: return f->normalTex.data();
    case 3: return f->timeTex.data();
    case 4: return f->fillImage.data();
    case 5: return f->fillVertex.data();
    case 6: return f->fillNormal.data();
    case 7: return f->depthFiltered.data();
    case 8: return f->depthMetric.data();
    case 9: return f->depthMetricFiltered.data();
    case 10: return f->indexTex.data();
    case 11: return f->vertConf.data();
    case 12: return f->colorTime.data();
    case 13: return f->normRad.data();
  }
  return nullptr;
}
extern "C" void efo_fusion_timers(const EfoFusion* f, double* out4) { memcpy(out4, f->timers, sizeof(f->timers)); }
