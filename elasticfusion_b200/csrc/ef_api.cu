// C ABI of libefusion.so (include/efusion_b200.h): context management, named buffers, the RGBDOdometry stage API and
// the whole-frame orchestration that mirrors ElasticFusion::processFrame (reference Core/ElasticFusion.cpp:270-607).
#include <math.h>
#include <stddef.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <new>
#include <utility>
#include <vector>

#include "ef_dmath.cuh"
#include "ef_internal.h"

using namespace ef;

extern "C" void ef_default_config(EfConfig* c, int width, int height, float fx, float fy, float cx, float cy) {
  memset(c, 0, sizeof(*c));
  c->width = width;
  c->height = height;
  c->fx = fx;
  c->fy = fy;
  c->cx = cx;
  c->cy = cy;
  // ElasticFusion ctor defaults, reference Core/ElasticFusion.h:42-58
  c->time_delta = 200;
  c->count_thresh = 35000;
  c->err_thresh = 5e-05f;
  c->cov_thresh = 1e-05f;
  c->close_loops = 0;
  c->iclnuim = 0;
  c->reloc = 0;
  c->photo_thresh = 115;
  c->confidence = 10;
  c->depth_cutoff = 3;
  c->icp_weight = 10;
  c->fast_odom = 0;
  c->fern_thresh = 0.3095f;
  c->so3 = 1;
  c->frame_to_frame_rgb = 0;
  c->capacity = 3072 * 3072;  // GlobalModel::MAX_VERTICES, reference Core/GlobalModel.cpp:22-24
  c->device = 0;
  c->skip_mid_predict = 1;
}

extern "C" const char* ef_error_string(int code) {
  if (code == 0) return "ok";
  if (code == EF_EINVAL) return "invalid argument";
  if (code == EF_ENOMEM) return "out of memory";
  if (code == EF_ESTATE) return "invalid state";
  if (code > 0) return cudaGetErrorString((cudaError_t)code);
  return "unknown error";
}

namespace ef {
int alloc_odom(EfContext* ctx, Arena& arena, int which, int width, int height, float fx, float fy, float cx, float cy) {
  OdomDev& od = ctx->odom[which];
  memset(&od, 0, sizeof(od));
  od.width = width;
  od.height = height;
  const float cam[4] = {fx, fy, cx, cy};
  memcpy(ctx->odom_cam[which], cam, sizeof(cam));
  // RGBDOdometry ctor, reference Core/Utils/RGBDOdometry.cpp:22-117 and RGBDOdometry.h:41-42
  od.distThres = 0.10f;
  od.angleThres = sinf(20.f * 3.14159254f / 180.f);
  od.sobelScale = (float)(1.0 / pow(2.0, 3));
  od.maxDepthDeltaRGB = 0.07f;
  od.maxDepthRGB = 6.0f;
  od.minGrad[0] = 5;
  od.minGrad[1] = 3;
  od.minGrad[2] = 1;
  for (int i = 0; i < NUM_PYRS; ++i) {
    od.minScale[i] = (float)(pow((double)od.minGrad[i], 2.0) / pow((double)od.sobelScale, 2.0));
    od.rows[i] = height >> i;
    od.cols[i] = width >> i;
    const size_t n = (size_t)od.rows[i] * od.cols[i];
    // the reference's cudaMalloc'd maps start uninitialised; NaN / zero fill keeps every first read defined
    CU(arena_alloc(ctx, arena, &od.depth_tmp[i], n, 0));
    CU(arena_alloc(ctx, arena, &od.vmap_g_prev[i], 3 * n, 0xff));
    CU(arena_alloc(ctx, arena, &od.nmap_g_prev[i], 3 * n, 0xff));
    CU(arena_alloc(ctx, arena, &od.vmap_c_prev[i], 3 * n, 0xff));
    CU(arena_alloc(ctx, arena, &od.nmap_c_prev[i], 3 * n, 0xff));
    CU(arena_alloc(ctx, arena, &od.vmap_curr[i], 3 * n, 0xff));
    CU(arena_alloc(ctx, arena, &od.nmap_curr[i], 3 * n, 0xff));
    CU(arena_alloc(ctx, arena, &od.lastDepth[i], n, 0xff));
    CU(arena_alloc(ctx, arena, &od.nextDepth[i], n, 0xff));
    CU(arena_alloc(ctx, arena, &od.lastImage[i], n, 0));
    CU(arena_alloc(ctx, arena, &od.nextImage[i], n, 0));
    CU(arena_alloc(ctx, arena, &od.lastNextImage[i], n, 0));
    CU(arena_alloc(ctx, arena, &od.dIdx[i], n, 0));
    CU(arena_alloc(ctx, arena, &od.dIdy[i], n, 0));
    CU(arena_alloc(ctx, arena, &od.corres[i], n, 0));
  }
  const size_t n0 = (size_t)width * height;
  CU(arena_alloc(ctx, arena, &od.vmaps_tmp, 4 * n0, 0));
  CU(arena_alloc(ctx, arena, &od.gn, 1));
  od.cand_base = reinterpret_cast<const int*>(reinterpret_cast<const char*>(od.gn) + offsetof(GNState, cand_base));
  od.intr0 = reinterpret_cast<const float*>(reinterpret_cast<const char*>(od.gn) + offsetof(GNState, fx));
  od.K_levels = reinterpret_cast<const double*>(reinterpret_cast<const char*>(od.gn) + offsetof(GNState, Kd));
  CU(arena_alloc(ctx, arena, &od.so3s, 1, 0));
  // one slot per CTA of k_so3_step, whose grid red_blocks() caps at MAX_RED_BLOCKS (254 CTAs at 1920x1080 on an H100)
  // (the reductions read whole 32-float rows of the partials; the kernels write the 29 / 11 terms of a system, so the padding
  // lanes are defined once here)
  CU(arena_alloc(ctx, arena, &od.so3_partials, (size_t)MAX_RED_BLOCKS * PARTIAL_STRIDE, 0));
  CU(arena_alloc(ctx, arena, &od.so3_counter, 4, 0));
  CU(arena_alloc(ctx, arena, &od.partials, (size_t)MAX_RED_BLOCKS * PARTIAL_STRIDE, 0));
  CU(arena_alloc(ctx, arena, &od.partials_rgb, (size_t)MAX_RGB_BLOCKS * 32, 0));
  CU(arena_alloc(ctx, arena, &od.partials2, (size_t)MAX_RGB_BLOCKS * 32, 0));
  {
    size_t flat = 0;
    for (int i = 0; i < NUM_PYRS; ++i) {
      od.level_start[i] = (int)flat;
      flat += (size_t)od.rows[i] * od.cols[i];
    }
    od.level_start[NUM_PYRS] = (int)flat;
    CU(arena_alloc(ctx, arena, &od.cand, flat, 0));
    CU(arena_alloc(ctx, arena, &od.terms, flat, 0));
  }
  CU(arena_alloc(ctx, arena, &od.partials_i, (size_t)MAX_RED_BLOCKS * 2));
  CU(arena_alloc(ctx, arena, &od.counter, 4, 0));
  CU(arena_alloc(ctx, arena, &od.trace, MAX_TRACE, 0));
  GNState g;
  gn_initial_state(&g, width, height, fx, fy, cx, cy);
  CU(cudaMemcpyAsync(od.gn, &g, sizeof(g), cudaMemcpyHostToDevice, ctx->stream));
  CU(cudaStreamSynchronize(ctx->stream));
  ctx->maps_dirty[which] = true;
  return 0;
}
}  // namespace ef

// every buffer, stream and event of a context, in order; returns on the first error (ef_destroy frees whatever was made)
static int create_buffers(EfContext* ctx) {
  const EfConfig& c = ctx->cfg;
  for (int w = 0; w < 2; ++w) RC(alloc_odom(ctx, ctx->arena, w, c.width, c.height, c.fx, c.fy, c.cx, c.cy));
  const size_t n = (size_t)ctx->cfg.width * ctx->cfg.height;
  Textures& t = ctx->tex;
  memset(&t, 0, sizeof(t));
  CU(ctx_alloc(ctx, &t.rgb, n * 3, 0));
  CU(ctx_alloc(ctx, &t.rgba, n * 4, 0));
  CU(ctx_alloc(ctx, &t.depth_raw, n, 0));
  CU(ctx_alloc(ctx, &t.depth_filtered, n, 0));
  CU(ctx_alloc(ctx, &t.depth_metric, n, 0));
  CU(ctx_alloc(ctx, &t.depth_metric_filtered, n, 0));
  CU(ctx_alloc(ctx, &t.index, n, 0));
  CU(ctx_alloc(ctx, &t.vert_conf, n, 0));
  CU(ctx_alloc(ctx, &t.color_time, n, 0));
  CU(ctx_alloc(ctx, &t.norm_rad, n, 0));
  CU(ctx_alloc(ctx, &t.image, n, 0));
  CU(ctx_alloc(ctx, &t.old_image, n, 0));
  CU(ctx_alloc(ctx, &t.fill_image, n, 0));
  CU(ctx_alloc(ctx, &t.vertex, n, 0));
  CU(ctx_alloc(ctx, &t.normal, n, 0));
  CU(ctx_alloc(ctx, &t.old_vertex, n, 0));
  CU(ctx_alloc(ctx, &t.old_normal, n, 0));
  CU(ctx_alloc(ctx, &t.fill_vertex, n, 0));
  CU(ctx_alloc(ctx, &t.fill_normal, n, 0));
  CU(ctx_alloc(ctx, &t.time, n, 0));
  CU(ctx_alloc(ctx, &t.old_time, n, 0));
  CU(ctx_alloc(ctx, &t.synth_depth, n, 0));
  // spare input-side set + side stream of the frame look-ahead
  Lookahead& la = ctx->la;
  memset(&la, 0, sizeof(la));
  CU(ctx_alloc(ctx, &la.rgb, n * 3, 0));
  CU(ctx_alloc(ctx, &la.rgba, n * 4, 0));
  CU(ctx_alloc(ctx, &la.depth_raw, n, 0));
  CU(ctx_alloc(ctx, &la.depth_filtered, n, 0));
  CU(ctx_alloc(ctx, &la.depth_metric, n, 0));
  CU(ctx_alloc(ctx, &la.depth_metric_filtered, n, 0));
  for (int i = 0; i < NUM_PYRS; ++i) {
    const size_t ni = (size_t)ctx->odom[0].rows[i] * ctx->odom[0].cols[i];
    CU(ctx_alloc(ctx, &la.depth_tmp[i], ni, 0));
    CU(ctx_alloc(ctx, &la.vmap_curr[i], 3 * ni, 0xff));
    CU(ctx_alloc(ctx, &la.nmap_curr[i], 3 * ni, 0xff));
    CU(ctx_alloc(ctx, &la.image[i], ni, 0));
  }
  CU(ctx_alloc(ctx, &la.so3s, 1, 0));
  CU(ctx_alloc(ctx, &la.so3_partials, (size_t)MAX_RED_BLOCKS * PARTIAL_STRIDE, 0));
  CU(ctx_alloc(ctx, &la.so3_counter, 4, 0));
  CU(cudaStreamCreateWithFlags(&la.stream, cudaStreamNonBlocking));
  CU(cudaEventCreateWithFlags(&la.ready, cudaEventDisableTiming));
  CU(cudaEventCreateWithFlags(&la.spare_free, cudaEventDisableTiming));
  CU(cudaEventCreateWithFlags(&la.h2d_done, cudaEventDisableTiming));
  CU(cudaEventCreateWithFlags(&la.image_ready, cudaEventDisableTiming));
  CU(cudaEventCreateWithFlags(&la.track_started, cudaEventDisableTiming));
  CU(cudaEventCreateWithFlags(&ctx->view_pose_sent, cudaEventDisableTiming));
  if (ctx->stage_timing) {
    CU(cudaEventCreate(&la.timing[0]));
    CU(cudaEventCreate(&la.timing[1]));
  }
  CU(cudaMallocHost((void**)&la.pin_rgb, n * 3));
  CU(cudaMallocHost((void**)&la.pin_depth, n * 2));
  RC(alloc_map(ctx));
  CU(cudaMallocHost((void**)&ctx->pin_rgb, n * 3));
  CU(cudaMallocHost((void**)&ctx->pin_depth, n * 2));
  CU(cudaMallocHost((void**)&ctx->pin_small, sizeof(PinStaging)));
  CU(cudaMalloc((void**)&ctx->dev_small, sizeof(DevStaging)));
  CU(cudaEventRecord(la.spare_free, ctx->stream));
  CU(cudaEventRecord(la.h2d_done, la.stream));
  CU(cudaEventRecord(la.image_ready, ctx->stream));
  CU(cudaStreamSynchronize(ctx->stream));
  return 0;
}

extern "C" int ef_create(const EfConfig* cfg, void* stream, EfContext** out) {
  if (!cfg || !out || cfg->width <= 0 || cfg->height <= 0 || cfg->capacity <= 0) return EF_EINVAL;
  // close_loops = 1 runs the LOCAL loop closure front half every frame (ElasticFusion.cpp:447-505; results through
  // ef_local_loop_result); 2 also samples, solves and applies the deformation graph inside the frame (frame_local_deform).
  // Ferns / relocalisation stay outside this library (SURVEY.md §8).
  if (cfg->close_loops < 0 || cfg->close_loops > 2) return EF_EINVAL;
  if (cfg->reloc) return EF_EINVAL;
  if ((cfg->width >> 2) < 8 || (cfg->height >> 2) < 8) return EF_EINVAL;
  CU(cudaSetDevice(cfg->device));
  EfContext* ctx = new (std::nothrow) EfContext();
  if (!ctx) return EF_ENOMEM;
  ctx->cfg = *cfg;
  ctx->device = cfg->device;
  {
    int sms = 0;
    cudaError_t e = cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, cfg->device);
    ctx->num_sms = sms;
    ctx->own_stream = false;
    if (e == cudaSuccess) {
      if (stream) {
        ctx->stream = (cudaStream_t)stream;
      } else {
        e = cudaStreamCreateWithFlags(&ctx->stream, cudaStreamNonBlocking);
        ctx->own_stream = (e == cudaSuccess);
      }
    }
    if (e != cudaSuccess) {  // nothing else has been allocated yet
      delete ctx;
      return (int)e;
    }
  }
  ctx->launches = 0;
  ctx->so3_ready = false;
  {
    const char* e = getenv("EF_NO_PDL");
    ctx->pdl = !(e && e[0] == '1');
    ctx->plain_next = false;
    for (bool& d : ctx->maps_dirty) d = true;
    // Gauss-Newton iterations of the coarse pyramid levels inside one thread-block cluster (k_gn_cluster): EF_GN_CLUSTER = wanted
    // cluster size (16 default, 8, or 0 = off), EF_GN_CLUSTER_LEVELS = how many levels from the top of the pyramid (default 1: the 160x120
    // level; 16 SMs are too few for the dense pass of the finer levels)
    e = getenv("EF_VISIBLE_LIST");
    ctx->visible_list = !(e && e[0] == '0');
    e = getenv("EF_GN_CLUSTER");
    ctx->gn_cluster = odom_cluster_size(e ? atoi(e) : 16);
    e = getenv("EF_GN_CLUSTER_LEVELS");
    ctx->gn_cluster_levels = e ? atoi(e) : 1;
    if (ctx->gn_cluster_levels < 0) ctx->gn_cluster_levels = 0;
    if (ctx->gn_cluster_levels > NUM_PYRS) ctx->gn_cluster_levels = NUM_PYRS;
    e = getenv("EF_STAGE_TIMING");
    ctx->stage_timing = (e && e[0] == '1');
    ctx->stage_n = 0;
    if (ctx->stage_timing)
      for (int i = 0; i < 16; ++i) cudaEventCreate(&ctx->stage_ev[i]);
    // the look-ahead's side stream starts after the frame's coarse-level cluster (default) or, EF_LA_AFTER_TRACK=0, at frame start
    e = getenv("EF_LA_AFTER_TRACK");
    ctx->la_after_track = !(e && e[0] == '0');
  }
  ctx->tick = 1;
  for (int k = 0; k < 16; ++k) ctx->T_wc[k] = (k % 5 == 0) ? 1.0 : 0.0;
  ctx->rgb_only = false;
  ctx->icp_weight = cfg->icp_weight;
  ctx->pyramid = true;
  ctx->fast_odom = cfg->fast_odom != 0;
  ctx->so3 = cfg->so3 != 0;
  ctx->frame_to_frame_rgb = cfg->frame_to_frame_rgb != 0;
  ctx->confidence = cfg->confidence;
  ctx->depth_cutoff = cfg->depth_cutoff;
  ctx->max_depth_processed = 20.0f;  // reference Core/ElasticFusion.cpp:83
  ctx->host_count = 0;
  ctx->frame_open = false;

  if (int rc = create_buffers(ctx)) {
    ef_destroy(ctx);
    return rc;
  }
  *out = ctx;
  return 0;
}

extern "C" int ef_destroy(EfContext* ctx) {
  if (!ctx) return EF_EINVAL;
  cudaSetDevice(ctx->device);
  cudaStreamSynchronize(ctx->stream);
  if (ctx->la.stream) {
    cudaStreamSynchronize(ctx->la.stream);
    cudaStreamDestroy(ctx->la.stream);
  }
  if (ctx->la.ready) cudaEventDestroy(ctx->la.ready);
  if (ctx->la.spare_free) cudaEventDestroy(ctx->la.spare_free);
  if (ctx->la.h2d_done) cudaEventDestroy(ctx->la.h2d_done);
  if (ctx->la.image_ready) cudaEventDestroy(ctx->la.image_ready);
  if (ctx->la.track_started) cudaEventDestroy(ctx->la.track_started);
  if (ctx->view_pose_sent) cudaEventDestroy(ctx->view_pose_sent);
  for (cudaEvent_t ev : ctx->la.timing)
    if (ev) cudaEventDestroy(ev);
  if (ctx->la.pin_rgb) cudaFreeHost(ctx->la.pin_rgb);
  if (ctx->la.pin_depth) cudaFreeHost(ctx->la.pin_depth);
  map_free_host(ctx);
  deform_free(ctx);
  render_free(ctx);
  map_fuse_view_free(ctx);
  track_view_free(ctx);
  for (EfCamera* cam : ctx->cameras)
    if (cam) camera_destroy(ctx, cam);
  ctx->arena.release();
  if (ctx->pin_rgb) cudaFreeHost(ctx->pin_rgb);
  if (ctx->pin_depth) cudaFreeHost(ctx->pin_depth);
  if (ctx->pin_small) cudaFreeHost(ctx->pin_small);
  if (ctx->dev_small) cudaFree(ctx->dev_small);
  if (ctx->own_stream) cudaStreamDestroy(ctx->stream);
  delete ctx;
  return 0;
}

extern "C" void* ef_stream(EfContext* ctx) { return ctx ? (void*)ctx->stream : nullptr; }
extern "C" int ef_sync(EfContext* ctx) {
  if (!ctx) return EF_EINVAL;
  CU(cudaStreamSynchronize(ctx->stream));
  CU(cudaStreamSynchronize(ctx->la.stream));
  return 0;
}
extern "C" int ef_launch_count(EfContext* ctx, int64_t* n) {
  if (!ctx || !n) return EF_EINVAL;
  *n = ctx->launches;
  return 0;
}

// ---------------------------------------------------------------------------------------------------------------
// named buffers
// ---------------------------------------------------------------------------------------------------------------
// pyramid buffer `base` (EF_BUF_VMAP_CURR ..) of a tracker at `level`; n: its level-0 pixels
static int odom_buffer(const OdomDev& od, int base, int level, size_t n, void** p, size_t* b) {
  if (level < 0 || level >= NUM_PYRS) return EF_EINVAL;
  const size_t nl = (size_t)od.rows[level] * od.cols[level];
  switch (base) {
    case EF_BUF_VMAP_CURR: *p = od.vmap_curr[level]; *b = nl * 12; break;
    case EF_BUF_NMAP_CURR: *p = od.nmap_curr[level]; *b = nl * 12; break;
    case EF_BUF_VMAP_G_PREV: *p = od.vmap_g_prev[level]; *b = nl * 12; break;
    case EF_BUF_NMAP_G_PREV: *p = od.nmap_g_prev[level]; *b = nl * 12; break;
    case EF_BUF_LAST_DEPTH: *p = od.lastDepth[level]; *b = nl * 4; break;
    case EF_BUF_NEXT_DEPTH: *p = od.nextDepth[level]; *b = nl * 4; break;
    case EF_BUF_LAST_IMAGE: *p = od.lastImage[level]; *b = nl; break;
    case EF_BUF_NEXT_IMAGE: *p = od.nextImage[level]; *b = nl; break;
    case EF_BUF_LAST_NEXT_IMAGE: *p = od.lastNextImage[level]; *b = nl; break;
    case EF_BUF_DIDX: *p = od.dIdx[level]; *b = nl * 2; break;
    case EF_BUF_DIDY: *p = od.dIdy[level]; *b = nl * 2; break;
    case EF_BUF_DEPTH_TMP: *p = od.depth_tmp[level]; *b = nl * 2; break;
    case EF_BUF_CORRES: *p = od.corres[level]; *b = nl * 16; break;
    case EF_BUF_VMAPS_TMP: *p = od.vmaps_tmp; *b = n * 16; break;
    default: return EF_EINVAL;
  }
  return 0;
}

extern "C" int ef_buffer(EfContext* ctx, int32_t id, int32_t level, void** dev_ptr, size_t* bytes) {
  if (!ctx) return EF_EINVAL;
  const size_t n = (size_t)ctx->cfg.width * ctx->cfg.height;
  void* p = nullptr;
  size_t b = 0;
  Textures& t = ctx->tex;
  if (id < 40) {
    switch (id) {
      case EF_BUF_RGB: p = t.rgb; b = n * 3; break;
      case EF_BUF_RGBA: p = t.rgba; b = n * 4; break;
      case EF_BUF_DEPTH_RAW: p = t.depth_raw; b = n * 2; break;
      case EF_BUF_DEPTH_FILTERED: p = t.depth_filtered; b = n * 2; break;
      case EF_BUF_DEPTH_METRIC: p = t.depth_metric; b = n * 4; break;
      case EF_BUF_DEPTH_METRIC_FILTERED: p = t.depth_metric_filtered; b = n * 4; break;
      case EF_BUF_INDEX: p = t.index; b = n * 4; break;
      case EF_BUF_VERT_CONF: p = t.vert_conf; b = n * 16; break;
      case EF_BUF_COLOR_TIME: p = t.color_time; b = n * 16; break;
      case EF_BUF_NORM_RAD: p = t.norm_rad; b = n * 16; break;
      case EF_BUF_IMAGE: p = t.image; b = n * 4; break;
      case EF_BUF_VERTEX: p = t.vertex; b = n * 16; break;
      case EF_BUF_NORMAL: p = t.normal; b = n * 16; break;
      case EF_BUF_TIME: p = t.time; b = n * 2; break;
      case EF_BUF_OLD_IMAGE: p = t.old_image; b = n * 4; break;
      case EF_BUF_OLD_VERTEX: p = t.old_vertex; b = n * 16; break;
      case EF_BUF_OLD_NORMAL: p = t.old_normal; b = n * 16; break;
      case EF_BUF_OLD_TIME: p = t.old_time; b = n * 2; break;
      case EF_BUF_SYNTH_DEPTH: p = t.synth_depth; b = n * 4; break;
      case EF_BUF_FILL_IMAGE: p = t.fill_image; b = n * 4; break;
      case EF_BUF_FILL_VERTEX: p = t.fill_vertex; b = n * 16; break;
      case EF_BUF_FILL_NORMAL: p = t.fill_normal; b = n * 16; break;
      default: return EF_EINVAL;
    }
  } else {
    const int which = id / 100;
    if (which < 0 || which > 1) return EF_EINVAL;
    RC(odom_buffer(ctx->odom[which], id % 100, level, n, &p, &b));
  }
  if (dev_ptr) *dev_ptr = p;
  if (bytes) *bytes = b;
  return 0;
}

extern "C" int ef_resize(EfContext* ctx, int32_t id, int32_t factor, void* host_out, size_t bytes) {
  if (!ctx || !host_out || factor < 1) return EF_EINVAL;
  void* p;
  size_t b;
  RC(ef_buffer(ctx, id, 0, &p, &b));
  if (id >= 40) return EF_EINVAL;  // full-resolution image attachments only
  const size_t n = (size_t)ctx->cfg.width * ctx->cfg.height;
  const int elem = (int)(b / n);
  if (elem != 2 && elem != 4 && elem != 16) return EF_EINVAL;
  if (bytes < (size_t)(ctx->cfg.width / factor) * (ctx->cfg.height / factor) * elem) return EF_EINVAL;
  return map_resize_to_host(ctx, p, elem, factor, host_out);
}
extern "C" int ef_upload(EfContext* ctx, int32_t id, int32_t level, const void* host, size_t bytes) {
  void* p;
  size_t b;
  RC(ef_buffer(ctx, id, level, &p, &b));
  if (bytes > b || !host) return EF_EINVAL;
  CU(cudaMemcpyAsync(p, host, bytes, cudaMemcpyHostToDevice, ctx->stream));
  if (id == EF_BUF_IMAGE) RC(map_dense_enough_async(ctx));  // the next frame's fill-in choice follows the uploaded image
  if (id == EF_BUF_INDEX || id == EF_BUF_VERT_CONF || id == EF_BUF_COLOR_TIME || id == EF_BUF_NORM_RAD) ctx->index.keys_only = false;  // (only the frame path leaves them unwritten)
  CU(cudaStreamSynchronize(ctx->stream));
  return 0;
}
extern "C" int ef_download(EfContext* ctx, int32_t id, int32_t level, void* host, size_t bytes) {
  void* p;
  size_t b;
  RC(ef_buffer(ctx, id, level, &p, &b));
  if (bytes > b || !host) return EF_EINVAL;
  CU(cudaMemcpyAsync(host, p, bytes, cudaMemcpyDeviceToHost, ctx->stream));
  CU(cudaStreamSynchronize(ctx->stream));
  return 0;
}

// ---------------------------------------------------------------------------------------------------------------
// tracker stage API
// ---------------------------------------------------------------------------------------------------------------
static int upload_gn(EfContext* ctx, int which, size_t offset, const void* src, size_t bytes) {
  CU(cudaMemcpyAsync((char*)ctx->odom[which].gn + offset, src, bytes, cudaMemcpyHostToDevice, ctx->stream));
  return 0;
}
static int download_gn(EfContext* ctx, int which, GNState* g) {
  CU(cudaMemcpyAsync(g, ctx->odom[which].gn, sizeof(GNState), cudaMemcpyDeviceToHost, ctx->stream));
  CU(cudaStreamSynchronize(ctx->stream));
  return 0;
}
#define WHICH_OK(w) ((w) == 0 || (w) == 1)

extern "C" int ef_odom_init_icp_depth(EfContext* ctx, int which, const uint16_t* depth_dev, float cutoff) {
  if (!ctx || !WHICH_OK(which) || !depth_dev) return EF_EINVAL;
  return odom_init_icp_depth(ctx, which, depth_dev, cutoff);
}
extern "C" int ef_odom_init_icp_pred(EfContext* ctx, int which, const float* vtx4, const float* nrm4) {
  if (!ctx || !WHICH_OK(which) || !vtx4 || !nrm4) return EF_EINVAL;
  return odom_init_icp_pred(ctx, which, vtx4, nrm4);
}
extern "C" int ef_odom_init_icp_model(EfContext* ctx, int which, const float* vtx4, const float* nrm4, const double* T) {
  if (!ctx || !WHICH_OK(which) || !vtx4 || !nrm4) return EF_EINVAL;
  if (T) {
    RC(upload_gn(ctx, which, offsetof(GNState, T_wc), T, sizeof(double) * 16));
    CU(cudaStreamSynchronize(ctx->stream));  // T is caller memory
  }
  return odom_init_icp_model(ctx, which, vtx4, nrm4);
}
extern "C" int ef_odom_init_rgb(EfContext* ctx, int which, const uint8_t* rgba) {
  if (!ctx || !WHICH_OK(which) || !rgba) return EF_EINVAL;
  OdomDev& od = ctx->odom[which];
  return odom_populate(ctx, which, rgba, od.nextDepth, od.nextImage, true);
}
extern "C" int ef_odom_init_rgb_model(EfContext* ctx, int which, const uint8_t* rgba) {
  if (!ctx || !WHICH_OK(which) || !rgba) return EF_EINVAL;
  OdomDev& od = ctx->odom[which];
  return odom_populate(ctx, which, rgba, od.lastDepth, od.lastImage, true);
}
extern "C" int ef_odom_init_first_rgb(EfContext* ctx, int which, const uint8_t* rgba) {
  if (!ctx || !WHICH_OK(which) || !rgba) return EF_EINVAL;
  OdomDev& od = ctx->odom[which];
  return odom_populate(ctx, which, rgba, nullptr, od.lastNextImage, false);
}

extern "C" int ef_odom_track(EfContext* ctx, int which, double* T_wc, int32_t rgb_only, float icp_weight, int32_t pyramid,
                             int32_t fast_odom, int32_t so3, EfSolveTrace* trace, int32_t max_trace, int32_t* n_trace) {
  if (!ctx || !WHICH_OK(which) || !T_wc) return EF_EINVAL;
  RC(upload_gn(ctx, which, offsetof(GNState, T_wc), T_wc, sizeof(double) * 16));
  CU(cudaStreamSynchronize(ctx->stream));
  RC(odom_track_async(ctx, which, rgb_only != 0, icp_weight, pyramid != 0, fast_odom != 0, so3 != 0));
  RC(odom_finish_async(ctx, which, 1.0f, true, which == 0 ? ctx->map.pose : nullptr));
  GNState g;
  RC(download_gn(ctx, which, &g));
  memcpy(T_wc, g.T_wc, sizeof(double) * 16);
  if (n_trace) *n_trace = g.trace_n < max_trace ? g.trace_n : max_trace;
  if (trace && max_trace > 0) {
    const int n = g.trace_n < max_trace ? g.trace_n : max_trace;
    CU(cudaMemcpyAsync(trace, ctx->odom[which].trace, sizeof(EfSolveTrace) * n, cudaMemcpyDeviceToHost, ctx->stream));
    CU(cudaStreamSynchronize(ctx->stream));
  }
  return 0;
}

extern "C" int ef_odom_stats(EfContext* ctx, int which, EfOdomStats* out) {
  if (!ctx || !WHICH_OK(which) || !out) return EF_EINVAL;
  GNState g;
  RC(download_gn(ctx, which, &g));
  out->lastICPError = g.lastICPError;
  out->lastICPCount = g.lastICPCount;
  out->lastRGBError = g.lastRGBError;
  out->lastRGBCount = g.lastRGBCount;
  out->lastSO3Error = g.lastSO3Error;
  out->lastSO3Count = g.lastSO3Count;
  memcpy(out->lastA, g.lastA, sizeof(g.lastA));
  memcpy(out->lastb, g.lastb, sizeof(g.lastb));
  return 0;
}

extern "C" int ef_odom_covariance(EfContext* ctx, int which, double* cov36) {
  if (!ctx || !WHICH_OK(which) || !cov36) return EF_EINVAL;
  GNState g;
  RC(download_gn(ctx, which, &g));
  efm::inv_n<6>(g.lastA, cov36);  // lastA.lu().inverse(), reference RGBDOdometry.cpp:573-575
  return 0;
}

extern "C" int ef_icp_step_async(EfContext* ctx, int which, int level, const float* Rcurr, const float* tcurr, const float* Rprev_inv,
                                 const float* tprev) {
  if (!ctx || !WHICH_OK(which) || level < 0 || level >= NUM_PYRS) return EF_EINVAL;
  if (Rcurr) {
    float* s = ctx->pin_small->icp_inputs;
    CU(cudaStreamSynchronize(ctx->stream));  // the H2D copies of the previous call may still be reading the staging buffer
    memcpy(s, Rcurr, 36);
    memcpy(s + 9, tcurr, 12);
    memcpy(s + 12, Rprev_inv, 36);
    memcpy(s + 21, tprev, 12);
    RC(upload_gn(ctx, which, offsetof(GNState, Rcurr), s, 36));
    RC(upload_gn(ctx, which, offsetof(GNState, tcurr), s + 9, 12));
    RC(upload_gn(ctx, which, offsetof(GNState, Rprev_inv), s + 12, 36));
    RC(upload_gn(ctx, which, offsetof(GNState, tprev), s + 21, 12));
    // the kernel works in the previous camera's frame: M = R_prev^-1 R_curr, t' = R_prev^-1 (t_curr - t_prev)
    float* M = s + 24;
    for (int r = 0; r < 3; ++r) {
      for (int c = 0; c < 3; ++c)
        M[r * 3 + c] = Rprev_inv[r * 3 + 0] * Rcurr[0 * 3 + c] + Rprev_inv[r * 3 + 1] * Rcurr[1 * 3 + c] + Rprev_inv[r * 3 + 2] * Rcurr[2 * 3 + c];
      M[9 + r] = Rprev_inv[r * 3 + 0] * (tcurr[0] - tprev[0]) + Rprev_inv[r * 3 + 1] * (tcurr[1] - tprev[1]) + Rprev_inv[r * 3 + 2] * (tcurr[2] - tprev[2]);
    }
    RC(upload_gn(ctx, which, offsetof(GNState, Mcp), M, 48));
  }
  return launch_se3_step_raw(ctx, which, level, true, false, 0.f);
}

extern "C" int ef_icp_dense_pass_async(EfContext* ctx, int which, int level) {
  if (!ctx || !WHICH_OK(which) || level < 0 || level >= NUM_PYRS) return EF_EINVAL;
  return launch_icp_dense_only(ctx, which, level);
}

extern "C" int ef_icp_step(EfContext* ctx, int which, int level, const float* Rcurr, const float* tcurr, const float* Rprev_inv,
                           const float* tprev, float* A36, float* b6, float* residual2) {
  if (!Rcurr || !tcurr || !Rprev_inv || !tprev || !A36 || !b6 || !residual2) return EF_EINVAL;
  RC(ef_icp_step_async(ctx, which, level, Rcurr, tcurr, Rprev_inv, tprev));
  GNState g;
  RC(download_gn(ctx, which, &g));
  efm::unpack_normal_eq<6>(g.sum_icp, A36, b6);
  residual2[0] = g.sum_icp[27];
  residual2[1] = g.sum_icp[28];
  return 0;
}

extern "C" int ef_rgb_residual(EfContext* ctx, int which, int level, const float* krkinv, const float* kt, int32_t* sigma_sum,
                               int32_t* count) {
  if (!ctx || !WHICH_OK(which) || level < 0 || level >= NUM_PYRS || !krkinv || !kt) return EF_EINVAL;
  RC(upload_gn(ctx, which, offsetof(GNState, krkinv), krkinv, 36));
  RC(upload_gn(ctx, which, offsetof(GNState, kt), kt, 12));
  CU(cudaStreamSynchronize(ctx->stream));
  RC(launch_sobel(ctx, which));
  RC(launch_rgb_residual_raw(ctx, which, level));
  GNState g;
  RC(download_gn(ctx, which, &g));
  if (count) *count = g.sum_res[0];
  if (sigma_sum) *sigma_sum = g.sum_res[1];
  return 0;
}

extern "C" int ef_rgb_step(EfContext* ctx, int which, int level, float sigma, float* A36, float* b6) {
  if (!ctx || !WHICH_OK(which) || level < 0 || level >= NUM_PYRS || !A36 || !b6) return EF_EINVAL;
  RC(launch_se3_step_raw(ctx, which, level, false, true, sigma));
  GNState g;
  RC(download_gn(ctx, which, &g));
  efm::unpack_normal_eq<6>(g.sum_rgb, A36, b6);
  return 0;
}

extern "C" int ef_so3_step(EfContext* ctx, int which, const float* image_basis, const float* kinv, const float* krlr, float* A9, float* b3,
                           float* residual2) {
  if (!ctx || !WHICH_OK(which) || !image_basis || !kinv || !krlr || !A9 || !b3 || !residual2) return EF_EINVAL;
  char* sdev = (char*)ctx->odom[which].so3s;
  CU(cudaMemcpyAsync(sdev + offsetof(So3State, imageBasis), image_basis, 36, cudaMemcpyHostToDevice, ctx->stream));
  CU(cudaMemcpyAsync(sdev + offsetof(So3State, kinv), kinv, 36, cudaMemcpyHostToDevice, ctx->stream));
  CU(cudaMemcpyAsync(sdev + offsetof(So3State, krlr), krlr, 36, cudaMemcpyHostToDevice, ctx->stream));
  CU(cudaStreamSynchronize(ctx->stream));
  RC(launch_so3_raw(ctx, which));
  struct {
    float sum_so3[12];
  } g;
  CU(cudaMemcpyAsync(g.sum_so3, sdev + offsetof(So3State, sum_so3), sizeof(g.sum_so3), cudaMemcpyDeviceToHost, ctx->stream));
  CU(cudaStreamSynchronize(ctx->stream));
  efm::unpack_normal_eq<3>(g.sum_so3, A9, b3);
  residual2[0] = g.sum_so3[9];
  residual2[1] = g.sum_so3[10];
  return 0;
}

extern "C" int ef_preprocess_depth(EfContext* ctx, const uint16_t* raw, float cutoff, uint16_t* filtered, float* metric,
                                   float* metric_filtered) {
  if (!ctx || !raw) return EF_EINVAL;
  return preprocess_depth(ctx, ctx->cfg.height, ctx->cfg.width, raw, cutoff, filtered, metric, metric_filtered);
}

// ---------------------------------------------------------------------------------------------------------------
// setters / getters
// ---------------------------------------------------------------------------------------------------------------
extern "C" int ef_get_pose(EfContext* ctx, double* T) {
  if (!ctx || !T) return EF_EINVAL;
  CU(cudaMemcpyAsync(T, (char*)ctx->odom[0].gn + offsetof(GNState, T_wc), sizeof(double) * 16, cudaMemcpyDeviceToHost, ctx->stream));
  CU(cudaStreamSynchronize(ctx->stream));
  memcpy(ctx->T_wc, T, sizeof(double) * 16);
  return 0;
}
extern "C" int ef_set_pose(EfContext* ctx, const double* T) {
  if (!ctx || !T) return EF_EINVAL;
  RC(upload_gn(ctx, 0, offsetof(GNState, T_wc), T, sizeof(double) * 16));
  CU(cudaStreamSynchronize(ctx->stream));
  memcpy(ctx->T_wc, T, sizeof(double) * 16);
  return 0;
}
extern "C" int ef_get_tick(EfContext* ctx, int32_t* tick) {
  if (!ctx || !tick) return EF_EINVAL;
  *tick = ctx->tick;
  return 0;
}
extern "C" int ef_set_tick(EfContext* ctx, int32_t tick) {
  if (!ctx) return EF_EINVAL;
  ctx->tick = tick;
  CU(cudaMemcpyAsync(ctx->map.tick, &ctx->tick, 4, cudaMemcpyHostToDevice, ctx->stream));
  CU(cudaStreamSynchronize(ctx->stream));
  return 0;
}
extern "C" int ef_set_rgb_only(EfContext* ctx, int32_t v) { if (!ctx) return EF_EINVAL; ctx->rgb_only = v != 0; return 0; }
extern "C" int ef_set_icp_weight(EfContext* ctx, float v) { if (!ctx) return EF_EINVAL; ctx->icp_weight = v; return 0; }
extern "C" int ef_set_pyramid(EfContext* ctx, int32_t v) { if (!ctx) return EF_EINVAL; ctx->pyramid = v != 0; return 0; }
extern "C" int ef_set_fast_odom(EfContext* ctx, int32_t v) { if (!ctx) return EF_EINVAL; ctx->fast_odom = v != 0; return 0; }
extern "C" int ef_set_so3(EfContext* ctx, int32_t v) { if (!ctx) return EF_EINVAL; ctx->so3 = v != 0; return 0; }
extern "C" int ef_set_frame_to_frame_rgb(EfContext* ctx, int32_t v) { if (!ctx) return EF_EINVAL; ctx->frame_to_frame_rgb = v != 0; return 0; }
extern "C" int ef_set_confidence_threshold(EfContext* ctx, float v) { if (!ctx) return EF_EINVAL; ctx->confidence = v; return 0; }
extern "C" int ef_set_depth_cutoff(EfContext* ctx, float v) { if (!ctx) return EF_EINVAL; ctx->depth_cutoff = v; return 0; }

// ---------------------------------------------------------------------------------------------------------------
// map stage API
// ---------------------------------------------------------------------------------------------------------------
static int read_count(EfContext* ctx, const int* dev, int* out) {
  CU(cudaMemcpyAsync(out, dev, 4, cudaMemcpyDeviceToHost, ctx->stream));
  CU(cudaStreamSynchronize(ctx->stream));
  return 0;
}

extern "C" int ef_map_initialise(EfContext* ctx) {
  if (!ctx) return EF_EINVAL;
  return map_initialise_async(ctx);
}
extern "C" int ef_map_predict_indices(EfContext* ctx, const double* T, int32_t time, float max_depth, int32_t time_delta) {
  if (!ctx) return EF_EINVAL;
  RC(map_update_pose_async(ctx, T));
  return map_predict_indices_async(ctx, map_frame_target(ctx), time, max_depth, time_delta);
}
extern "C" int ef_map_fuse(EfContext* ctx, const double* T, int32_t time, float max_depth, float weighting) {
  if (!ctx) return EF_EINVAL;
  RC(map_update_pose_async(ctx, T));
  return map_fuse_async(ctx, map_frame_target(ctx), time, max_depth, weighting);
}
extern "C" int ef_map_clean(EfContext* ctx, const double* T, int32_t time, float conf_threshold, int32_t time_delta, float max_depth) {
  if (!ctx) return EF_EINVAL;
  RC(map_update_pose_async(ctx, T));
  return map_clean_async(ctx, map_frame_target(ctx), time, conf_threshold, time_delta, max_depth);
}
extern "C" int ef_map_clean_deform(EfContext* ctx, const double* T, int32_t time, float conf_threshold, int32_t time_delta, float max_depth,
                                   const float* graph_nodes16, int32_t n_nodes, int32_t is_fern) {
  if (!ctx || n_nodes < 0 || (n_nodes > 0 && !graph_nodes16)) return EF_EINVAL;
  RC(map_set_graph(ctx, graph_nodes16, n_nodes));
  RC(map_update_pose_async(ctx, T));
  return map_clean_async(ctx, map_frame_target(ctx), time, conf_threshold, time_delta, max_depth, n_nodes, is_fern != 0);
}
extern "C" int ef_map_raycast(EfContext* ctx, const double* T, float max_depth, float conf_threshold, int32_t time, int32_t max_time,
                              int32_t time_delta, int32_t mode) {
  if (!ctx || mode < 0 || mode > 2) return EF_EINVAL;
  RC(map_update_pose_async(ctx, T));
  return map_raycast_async(ctx, max_depth, conf_threshold, time, max_time, time_delta, mode);
}
extern "C" int ef_map_fill_in(EfContext* ctx, int32_t pass_geom, int32_t pass_img) {
  if (!ctx) return EF_EINVAL;
  return map_fill_in_async(ctx, pass_geom != 0, pass_img != 0);
}
extern "C" int ef_dense_enough(EfContext* ctx, int32_t* out) {
  if (!ctx || !out) return EF_EINVAL;
  int lit = 0;  // counted by the mode-0 raycast (or the upload) that wrote the predicted image
  RC(read_count(ctx, ctx->map.dense_count, &lit));
  *out = dense_enough_of(lit, ctx->map.rows, ctx->map.cols) ? 1 : 0;
  return 0;
}
extern "C" int ef_map_count(EfContext* ctx, int32_t* count) {
  if (!ctx || !count) return EF_EINVAL;
  RC(read_count(ctx, ctx->map.count, count));
  ctx->host_count = *count;
  return 0;
}
extern "C" int ef_map_download(EfContext* ctx, float* out12, int32_t max_surfels, int32_t* count) {
  if (!ctx || !out12) return EF_EINVAL;
  int n = 0;
  RC(read_count(ctx, ctx->map.count, &n));
  ctx->host_count = n;
  if (count) *count = n;
  if (n > max_surfels) n = max_surfels;
  return map_download(ctx, ctx->map.pos_conf, ctx->map.color_time, ctx->map.norm_rad, n, out12);
}
extern "C" int ef_map_download_new(EfContext* ctx, float* out12, int32_t max_surfels, int32_t* count) {
  if (!ctx || !out12) return EF_EINVAL;
  int n = 0;
  RC(read_count(ctx, ctx->map.new_count, &n));
  if (count) *count = n;
  if (n > max_surfels) n = max_surfels;
  return map_download(ctx, ctx->map.new_pos, ctx->map.new_col, ctx->map.new_nr, n, out12);
}
extern "C" int ef_map_upload_range(EfContext* ctx, const float* in12, int32_t first, int32_t count) {
  if (!ctx || !in12 || first < 0 || count <= 0) return EF_EINVAL;
  return map_upload_range(ctx, in12, first, count);
}
extern "C" int ef_map_upload(EfContext* ctx, const float* in12, int32_t count) {
  if (!ctx || (!in12 && count > 0) || count < 0) return EF_EINVAL;
  return map_upload(ctx, in12, count);
}

// ---------------------------------------------------------------------------------------------------------------
// global-surface render (ef_render.cu)
// ---------------------------------------------------------------------------------------------------------------
template <typename T>
static bool finite_all(const T* a, int n) {
  for (int i = 0; i < n; ++i)
    if (!isfinite(a[i])) return false;
  return true;
}
static bool render_view_ok(const EfRenderView* v) {
  return v && v->width >= 1 && v->width <= 16384 && v->height >= 1 && v->height <= 16384 && v->color_type >= 0 && v->color_type <= 3 &&
         finite_all(v->mvp, 16) && (!v->phong || finite_all(v->mv, 16));
}
extern "C" int ef_render_map_device(EfContext* ctx, const EfRenderView* view, uint8_t* rgba_dev) {
  if (!ctx || !rgba_dev || !render_view_ok(view)) return EF_EINVAL;
  CU(cudaSetDevice(ctx->device));
  return render_map_async(ctx, view, rgba_dev);
}
extern "C" int ef_render_map(EfContext* ctx, const EfRenderView* view, uint8_t* rgba_host) {
  if (!ctx || !rgba_host || !render_view_ok(view)) return EF_EINVAL;
  CU(cudaSetDevice(ctx->device));
  const size_t bytes = (size_t)view->width * view->height * 4;
  uint8_t* dev = nullptr;
  RC(offframe_staging(ctx, bytes, &dev));
  RC(render_map_async(ctx, view, dev));
  CU(cudaMemcpyAsync(rgba_host, dev, bytes, cudaMemcpyDeviceToHost, ctx->stream));
  CU(cudaStreamSynchronize(ctx->stream));
  return 0;
}
extern "C" int ef_render_camera(const double* T_wc16, float fx, float fy, float cx, float cy, int32_t width, int32_t height, float z_near,
                                float z_far, float* mvp16, float* mv16) {
  if (!T_wc16 || !mvp16 || !mv16 || width < 1 || width > 16384 || height < 1 || height > 16384) return EF_EINVAL;
  for (int i = 0; i < 16; ++i)
    if (!isfinite(T_wc16[i])) return EF_EINVAL;
  if (!isfinite(fx) || !isfinite(fy) || !isfinite(cx) || !isfinite(cy) || fx == 0.f || fy == 0.f || !isfinite(z_near) || !isfinite(z_far) ||
      !(z_near > 0.f) || !(z_far > z_near))
    return EF_EINVAL;
  // mv = T_wc^-1 (rigid), row-major
  double mv[16] = {0};
  for (int r = 0; r < 3; ++r) {
    for (int c = 0; c < 3; ++c) mv[r * 4 + c] = T_wc16[c * 4 + r];
    mv[r * 4 + 3] = -(T_wc16[0 * 4 + r] * T_wc16[3] + T_wc16[1 * 4 + r] * T_wc16[7] + T_wc16[2 * 4 + r] * T_wc16[11]);
  }
  mv[15] = 1.0;
  // camera looks down +z; window x = fx x/z + cx, window y = fy y/z + cy (the image's own rows: window row j is image row j), so
  // window pixel (i, j) samples the ray through image pixel centre (i + 0.5, j + 0.5); depth -1 at z_near, +1 at z_far
  const double W = width, H = height, n = z_near, f = z_far;
  const double P[16] = {2.0 * fx / W, 0, 2.0 * cx / W - 1.0, 0, 0, 2.0 * fy / H, 2.0 * cy / H - 1.0, 0,
                        0, 0, (f + n) / (f - n), -2.0 * f * n / (f - n), 0, 0, 1, 0};
  for (int r = 0; r < 4; ++r)
    for (int c = 0; c < 4; ++c) {
      double acc = 0;
      for (int k = 0; k < 4; ++k) acc += P[r * 4 + k] * mv[k * 4 + c];
      mvp16[c * 4 + r] = (float)acc;  // column-major
      mv16[c * 4 + r] = (float)mv[r * 4 + c];
    }
  return 0;
}

// ---------------------------------------------------------------------------------------------------------------
// model view: combinedPredict at any camera (ef_map.cu, on the render's z-buffer)
// ---------------------------------------------------------------------------------------------------------------
static bool model_view_ok(const EfModelView* v) {
  if (!v || v->width < 1 || v->width > 16384 || v->height < 1 || v->height > 16384) return false;
  for (int i = 0; i < 16; ++i)
    if (!isfinite(v->T_wc[i])) return false;
  return isfinite(v->fx) && isfinite(v->fy) && v->fx != 0.f && v->fy != 0.f && isfinite(v->cx) && isfinite(v->cy) && isfinite(v->max_depth) &&
         v->max_depth > 0.f && isfinite(v->conf_threshold);
}
static bool aligned(const void* p, size_t a) { return ((uintptr_t)p & (a - 1)) == 0; }
extern "C" int ef_map_predict_view_device(EfContext* ctx, const EfModelView* v, uint8_t* image4, float* vertex4, float* normal4, uint16_t* time) {
  if (!ctx || !model_view_ok(v) || (!image4 && !vertex4 && !normal4 && !time)) return EF_EINVAL;
  if (!aligned(image4, 4) || !aligned(vertex4, 16) || !aligned(normal4, 16) || !aligned(time, 2)) return EF_EINVAL;
  CU(cudaSetDevice(ctx->device));
  return map_predict_view_async(ctx, v, image4, vertex4, normal4, time);
}
extern "C" int ef_map_predict_view(EfContext* ctx, const EfModelView* v, uint8_t* image4, float* vertex4, float* normal4, uint16_t* time) {
  if (!ctx || !model_view_ok(v) || (!image4 && !vertex4 && !normal4 && !time)) return EF_EINVAL;
  CU(cudaSetDevice(ctx->device));
  // device staging of the requested outputs, the 16-byte ones first so that every part stays aligned
  const size_t n = (size_t)v->width * v->height;
  struct Part {
    void* host;
    size_t bytes;
    uint8_t* dev;
  } parts[4] = {{vertex4, n * 16, nullptr}, {normal4, n * 16, nullptr}, {image4, n * 4, nullptr}, {time, n * 2, nullptr}};
  size_t total = 0;
  for (Part& p : parts)
    if (p.host) total += p.bytes;
  uint8_t* dev = nullptr;
  RC(offframe_staging(ctx, total, &dev));
  for (Part& p : parts)
    if (p.host) {
      p.dev = dev;
      dev += p.bytes;
    }
  RC(map_predict_view_async(ctx, v, parts[2].dev, (float*)parts[0].dev, (float*)parts[1].dev, (uint16_t*)parts[3].dev));
  for (const Part& p : parts)
    if (p.host) CU(cudaMemcpyAsync(p.host, p.dev, p.bytes, cudaMemcpyDeviceToHost, ctx->stream));
  CU(cudaStreamSynchronize(ctx->stream));
  return 0;
}

// ---------------------------------------------------------------------------------------------------------------
// fuse view: the map half of a frame at any camera (ef_map.cu, on the view's own buffers)
// ---------------------------------------------------------------------------------------------------------------
static bool fuse_view_ok(const EfFuseView* v) {
  if (!v || v->width < 1 || v->width > 16384 || v->height < 1 || v->height > 16384) return false;
  for (int i = 0; i < 16; ++i)
    if (!isfinite(v->T_wc[i])) return false;
  return isfinite(v->fx) && isfinite(v->fy) && v->fx != 0.f && v->fy != 0.f && isfinite(v->cx) && isfinite(v->cy) &&
         isfinite(v->depth_cutoff) && v->depth_cutoff > 0.f && isfinite(v->max_depth) && v->max_depth > 0.f && isfinite(v->weighting) &&
         v->weighting >= 0.f && isfinite(v->conf_threshold) && v->time >= 0 && v->time_delta >= 0;
}
// before the first frame the map is not initialised (that frame would overwrite the view's surfels); between ef_process_frame_begin
// and _end the frame's map half is still to come
static int fuse_view_state(const EfContext* ctx) { return (ctx->tick <= 1 || ctx->frame_open) ? EF_ESTATE : 0; }

// upload (host inputs), bilateral filter + metric depth, predictIndices, fuse, predictIndices, clean: ElasticFusion.cpp:536-584 with
// no graph, at the view's camera
static int fuse_view_async(EfContext* ctx, const EfFuseView* v, const uint8_t* rgb, const uint16_t* depth, bool from_host) {
  MapTarget t;
  uint8_t* rgb_buf = nullptr;
  uint16_t* depth_buf = nullptr;
  RC(map_fuse_view_target(ctx, v, &t, &rgb_buf, &depth_buf));
  const size_t n = (size_t)v->width * v->height;
  if (from_host) {
    CU(cudaMemcpyAsync(rgb_buf, rgb, n * 3, cudaMemcpyHostToDevice, ctx->stream));
    CU(cudaMemcpyAsync(depth_buf, depth, n * 2, cudaMemcpyHostToDevice, ctx->stream));
    depth = depth_buf;
  } else {
    t.rgb = rgb;
  }
  RC(preprocess_depth(ctx, t.rows, t.cols, depth, v->depth_cutoff, nullptr, t.depth_metric, t.depth_metric_filtered));
  RC(map_predict_indices_async(ctx, t, v->time, v->max_depth, v->time_delta));
  RC(map_fuse_async(ctx, t, v->time, v->max_depth, -1.0f));  // (the view's weighting is staged with its pose)
  RC(map_predict_indices_async(ctx, t, v->time, v->max_depth, v->time_delta));
  return map_clean_async(ctx, t, v->time, v->conf_threshold, v->time_delta, v->max_depth);
}

extern "C" int ef_map_fuse_view_device(EfContext* ctx, const EfFuseView* v, const uint8_t* rgb_dev, const uint16_t* depth_dev) {
  if (!ctx || !fuse_view_ok(v) || !rgb_dev || !depth_dev || !aligned(depth_dev, 2)) return EF_EINVAL;
  RC(fuse_view_state(ctx));
  CU(cudaSetDevice(ctx->device));
  return fuse_view_async(ctx, v, rgb_dev, depth_dev, false);
}
extern "C" int ef_map_fuse_view(EfContext* ctx, const EfFuseView* v, const uint8_t* rgb, const uint16_t* depth) {
  if (!ctx || !fuse_view_ok(v) || !rgb || !depth) return EF_EINVAL;
  RC(fuse_view_state(ctx));
  CU(cudaSetDevice(ctx->device));
  RC(fuse_view_async(ctx, v, rgb, depth, true));
  return ef_map_count(ctx, &ctx->host_count);  // (synchronises)
}

// ---------------------------------------------------------------------------------------------------------------
// track view: the frame's tracking recipe at any camera (ef_track.cu, on the view's own buffers and tracker slot)
// ---------------------------------------------------------------------------------------------------------------
// the size rule of ef_create (every pyramid level at least 8 pixels on each side), capped at 4096 to bound the view's memory
static bool track_view_ok(const EfTrackView* v) {
  if (!v || !model_view_ok(&v->model)) return false;
  const int w = v->model.width, h = v->model.height;
  return w >= 32 && w <= 4096 && h >= 32 && h <= 4096 && (w >> 2) >= 8 && (h >> 2) >= 8 && isfinite(v->depth_cutoff) &&
         v->depth_cutoff > 0.f && isfinite(v->icp_weight) && v->icp_weight >= 0.f;
}

extern "C" int ef_track_view_device(EfContext* ctx, const EfTrackView* v, const uint8_t* rgb_dev, const uint16_t* depth_dev, EfTrackResult* out_dev) {
  if (!ctx || !track_view_ok(v) || !rgb_dev || !depth_dev || !out_dev || !aligned(depth_dev, 2) || !aligned(out_dev, 8)) return EF_EINVAL;
  CU(cudaSetDevice(ctx->device));
  return track_view_async(ctx, v, rgb_dev, depth_dev, false, out_dev);
}
extern "C" int ef_track_view(EfContext* ctx, const EfTrackView* v, const uint8_t* rgb, const uint16_t* depth, EfTrackResult* out,
                             EfSolveTrace* trace, int32_t max_trace, int32_t* n_trace) {
  if (!ctx || !track_view_ok(v) || !rgb || !depth || !out || max_trace < 0 || (max_trace > 0 && !trace)) return EF_EINVAL;
  CU(cudaSetDevice(ctx->device));
  RC(track_view_async(ctx, v, rgb, depth, true, nullptr));
  GNState g;
  int lit = 0;
  RC(track_view_read(ctx, &g, &lit));
  memcpy(out->T_wc, g.T_wc, sizeof(g.T_wc));
  EfOdomStats& s = out->stats;
  s.lastICPError = g.lastICPError;
  s.lastICPCount = g.lastICPCount;
  s.lastRGBError = g.lastRGBError;
  s.lastRGBCount = g.lastRGBCount;
  s.lastSO3Error = g.lastSO3Error;
  s.lastSO3Count = g.lastSO3Count;
  memcpy(s.lastA, g.lastA, sizeof(g.lastA));
  memcpy(s.lastb, g.lastb, sizeof(g.lastb));
  efm::inv_n<6>(g.lastA, out->covariance);  // as ef_odom_covariance
  out->dense_enough = dense_enough_of(lit, v->model.height, v->model.width) ? 1 : 0;
  const int n = g.trace_n < max_trace ? g.trace_n : max_trace;
  if (n_trace) *n_trace = n;
  if (n > 0) {
    CU(cudaMemcpyAsync(trace, ctx->odom[VIEW_TRACKER].trace, sizeof(EfSolveTrace) * n, cudaMemcpyDeviceToHost, ctx->stream));
    CU(cudaStreamSynchronize(ctx->stream));
  }
  return 0;
}

// ---------------------------------------------------------------------------------------------------------------
// cameras: processFrame for a sensor of the context's map (ef_track.cu, on the camera's own buffers and tracker slot)
// ---------------------------------------------------------------------------------------------------------------
// the track view's size rule
static bool camera_config_ok(const EfCameraConfig* c) {
  if (!c) return false;
  const int w = c->width, h = c->height;
  return w >= 32 && w <= 4096 && h >= 32 && h <= 4096 && isfinite(c->fx) && isfinite(c->fy) && c->fx != 0.f && c->fy != 0.f &&
         isfinite(c->cx) && isfinite(c->cy) && isfinite(c->depth_cutoff) && c->depth_cutoff > 0.f && isfinite(c->max_depth) &&
         c->max_depth > 0.f && isfinite(c->conf_threshold) && c->time_delta >= 0 && isfinite(c->icp_weight) && c->icp_weight >= 0.f;
}
static bool camera_of(const EfContext* ctx, const EfCamera* cam) {
  if (!ctx || !cam) return false;
  for (const EfCamera* c : ctx->cameras)
    if (c == cam) return true;
  return false;
}
static bool camera_frame_ok(const EfCameraFrame* f) {
  if (!f || f->time < 0 || !isfinite(f->weight_multiplier) || f->weight_multiplier < 0.f) return false;
  if (f->has_pose && !finite_all(f->T_wc, 16)) return false;
  return true;
}
// the first frame sets the pose; fuse follows ef_map_fuse_view's rule; a rig's member runs only in its rig's frames
static int camera_frame_state(const EfContext* ctx, const EfCamera* cam, const EfCameraFrame* f) {
  if (cam->rig || (!cam->has_frame && !f->has_pose)) return EF_ESTATE;
  return f->fuse ? fuse_view_state(ctx) : 0;
}

extern "C" int ef_camera_create(EfContext* ctx, const EfCameraConfig* cfg, EfCamera** out) {
  if (!ctx || !out || !camera_config_ok(cfg)) return EF_EINVAL;
  // a closing camera shares the graph and Deformation's bookkeeping of the context's in-frame closures
  if (cfg->close_loops != 0 && (cfg->close_loops != 1 || ctx->cfg.close_loops != 2)) return EF_EINVAL;
  CU(cudaSetDevice(ctx->device));
  return camera_create(ctx, cfg, out);
}
extern "C" int ef_camera_destroy(EfContext* ctx, EfCamera* cam) {
  if (!camera_of(ctx, cam)) return EF_EINVAL;
  CU(cudaSetDevice(ctx->device));
  camera_destroy(ctx, cam);
  return 0;
}
extern "C" int ef_camera_frame_device(EfContext* ctx, EfCamera* cam, const EfCameraFrame* f, const uint8_t* rgb_dev, const uint16_t* depth_dev,
                                      EfCameraResult* out_dev) {
  if (!camera_of(ctx, cam) || !camera_frame_ok(f) || !rgb_dev || !depth_dev || !out_dev || !aligned(depth_dev, 2) || !aligned(out_dev, 8))
    return EF_EINVAL;
  RC(camera_frame_state(ctx, cam, f));
  CU(cudaSetDevice(ctx->device));
  return camera_frame_async(ctx, cam, f, rgb_dev, depth_dev, false, out_dev);
}
extern "C" int ef_camera_frame(EfContext* ctx, EfCamera* cam, const EfCameraFrame* f, const uint8_t* rgb, const uint16_t* depth, EfCameraResult* out,
                               EfSolveTrace* trace, int32_t max_trace, int32_t* n_trace) {
  if (!camera_of(ctx, cam) || !camera_frame_ok(f) || !rgb || !depth || !out || max_trace < 0 || (max_trace > 0 && !trace)) return EF_EINVAL;
  RC(camera_frame_state(ctx, cam, f));
  CU(cudaSetDevice(ctx->device));
  RC(camera_frame_async(ctx, cam, f, rgb, depth, true, nullptr));
  RC(camera_read(ctx, cam, out, trace, max_trace, n_trace));  // (synchronises)
  return ef_map_count(ctx, &ctx->host_count);
}
extern "C" int ef_camera_buffer(EfContext* ctx, EfCamera* cam, int32_t id, int32_t level, void** dev_ptr, size_t* bytes) {
  if (!camera_of(ctx, cam)) return EF_EINVAL;
  const size_t n = (size_t)cam->cfg.width * cam->cfg.height;
  void* p = nullptr;
  size_t b = 0;
  if (id < 40) {
    switch (id) {
      case EF_BUF_RGB: p = cam->rgb; b = n * 3; break;
      case EF_BUF_RGBA: p = cam->rgba; b = n * 4; break;
      case EF_BUF_DEPTH_RAW: p = cam->depth_raw; b = n * 2; break;
      case EF_BUF_DEPTH_FILTERED: p = cam->depth_filtered; b = n * 2; break;
      case EF_BUF_DEPTH_METRIC: p = cam->target.depth_metric; b = n * 4; break;
      case EF_BUF_DEPTH_METRIC_FILTERED: p = cam->target.depth_metric_filtered; b = n * 4; break;
      case EF_BUF_IMAGE: p = cam->image; b = n * 4; break;
      case EF_BUF_VERTEX: p = cam->vertex; b = n * 16; break;
      case EF_BUF_NORMAL: p = cam->normal; b = n * 16; break;
      case EF_BUF_TIME: p = cam->time; b = n * 2; break;
      case EF_BUF_FILL_IMAGE: p = cam->fill_image; b = n * 4; break;
      case EF_BUF_FILL_VERTEX: p = cam->fill_vertex; b = n * 16; break;
      case EF_BUF_FILL_NORMAL: p = cam->fill_normal; b = n * 16; break;
      default: return EF_EINVAL;
    }
  } else {
    RC(odom_buffer(ctx->odom[cam->slot], id, level, n, &p, &b));
  }
  if (dev_ptr) *dev_ptr = p;
  if (bytes) *bytes = b;
  return 0;
}

// ---------------------------------------------------------------------------------------------------------------
// rigs: cameras tracked as one rigid body (ef_track.cu, on the members' buffers and tracker slots)
// ---------------------------------------------------------------------------------------------------------------
// rigid and finite: |R^T R - I| <= 1e-6 entrywise and a last row of 0 0 0 1
static bool rigid(const double* T) {
  if (!finite_all(T, 16) || T[12] != 0.0 || T[13] != 0.0 || T[14] != 0.0 || T[15] != 1.0) return false;
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) {
      double d = 0;
      for (int k = 0; k < 3; ++k) d += T[k * 4 + i] * T[k * 4 + j];
      if (fabs(d - (i == j ? 1.0 : 0.0)) > 1e-6) return false;
    }
  return true;
}
static bool rig_config_ok(const EfContext* ctx, const EfRigConfig* cfg) {
  if (!cfg || cfg->n < 1 || cfg->n > EF_MAX_CAMERAS || (cfg->joint_so3 != 0 && cfg->joint_so3 != 1)) return false;
  const EfCamera* c0 = cfg->cameras[0];
  for (int m = 0; m < cfg->n; ++m) {
    const EfCamera* c = cfg->cameras[m];
    if (!camera_of(ctx, c) || c->rig || !rigid(cfg->T_0i[m])) return false;
    for (int j = 0; j < m; ++j)
      if (cfg->cameras[j] == c) return false;
    const EfCameraConfig& k = c->cfg;
    if (k.close_loops != c0->cfg.close_loops || k.rgb_only || k.icp_weight != c0->cfg.icp_weight || k.pyramid != c0->cfg.pyramid || k.fast_odom != c0->cfg.fast_odom ||
        k.so3 != c0->cfg.so3 || (cfg->joint_so3 && !k.so3))
      return false;
  }
  for (int k = 0; k < 16; ++k)
    if (cfg->T_0i[0][k] != ((k % 5 == 0) ? 1.0 : 0.0)) return false;
  return true;
}
static bool rig_of(const EfContext* ctx, const EfRig* rig) {
  if (!ctx || !rig) return false;
  for (const EfRig* r : ctx->rigs)
    if (r == rig) return true;
  return false;
}
// the camera frame's rules, once for the rig
static int rig_frame_args(const EfContext* ctx, const EfRig* rig, const EfRigFrame* f, const void* const* rgb, const void* const* depth) {
  if (!rig_of(ctx, rig) || !rgb || !depth) return EF_EINVAL;
  EfCameraFrame cf = {};
  if (f) {
    cf.time = f->time;
    cf.weight_multiplier = f->weight_multiplier;
    cf.has_pose = f->has_pose;
    memcpy(cf.T_wc, f->T_wc, sizeof(cf.T_wc));
    cf.fuse = f->fuse;
  }
  if (!camera_frame_ok(f ? &cf : nullptr)) return EF_EINVAL;
  for (int m = 0; m < rig->n; ++m)
    if (!rgb[m] || !depth[m]) return EF_EINVAL;
  if (!rig->has_frame && !f->has_pose) return EF_ESTATE;
  return f->fuse ? fuse_view_state(ctx) : 0;
}

extern "C" int ef_rig_create(EfContext* ctx, const EfRigConfig* cfg, EfRig** out) {
  if (!ctx || !out || !rig_config_ok(ctx, cfg)) return EF_EINVAL;
  CU(cudaSetDevice(ctx->device));
  return rig_create(ctx, cfg, out);
}
extern "C" int ef_rig_destroy(EfContext* ctx, EfRig* rig) {
  if (!rig_of(ctx, rig)) return EF_EINVAL;
  CU(cudaSetDevice(ctx->device));
  rig_destroy(ctx, rig);
  return 0;
}
extern "C" int ef_rig_frame_device(EfContext* ctx, EfRig* rig, const EfRigFrame* f, const uint8_t* const* rgb_dev, const uint16_t* const* depth_dev,
                                   EfCameraResult* members_dev, EfRigResult* out_dev) {
  const int rc = rig_frame_args(ctx, rig, f, (const void* const*)rgb_dev, (const void* const*)depth_dev);
  if (rc == EF_EINVAL || !members_dev || !out_dev || !aligned(members_dev, 8) || !aligned(out_dev, 8)) return EF_EINVAL;
  for (int m = 0; m < rig->n; ++m)
    if (!aligned(depth_dev[m], 2)) return EF_EINVAL;
  RC(rc);
  CU(cudaSetDevice(ctx->device));
  return rig_frame_async(ctx, rig, f, rgb_dev, depth_dev, false, members_dev, out_dev);
}
extern "C" int ef_rig_frame(EfContext* ctx, EfRig* rig, const EfRigFrame* f, const uint8_t* const* rgb, const uint16_t* const* depth,
                            EfCameraResult* members, EfRigResult* out, EfSolveTrace* trace, int32_t max_trace, int32_t* n_trace) {
  const int rc = rig_frame_args(ctx, rig, f, (const void* const*)rgb, (const void* const*)depth);
  if (rc == EF_EINVAL || !members || !out || max_trace < 0 || (max_trace > 0 && !trace)) return EF_EINVAL;
  RC(rc);
  CU(cudaSetDevice(ctx->device));
  RC(rig_frame_async(ctx, rig, f, rgb, depth, true, nullptr, nullptr));
  RC(rig_read(ctx, rig, members, out, trace, max_trace, n_trace));  // (synchronises)
  return ef_map_count(ctx, &ctx->host_count);
}

// ---------------------------------------------------------------------------------------------------------------
// whole frame
// ---------------------------------------------------------------------------------------------------------------
// ElasticFusion::predict, reference Core/ElasticFusion.cpp:621-653 (lost == false, lastFrameRecovery == false)
static int predict_async(EfContext* ctx) {
  return map_raycast_async(ctx, ctx->max_depth_processed, ctx->confidence, ctx->tick, ctx->tick, ctx->cfg.time_delta, 0,
                           ctx->frame_to_frame_rgb ? 1 : 0);
}

extern "C" int ef_predict(EfContext* ctx) {
  if (!ctx) return EF_EINVAL;
  RC(map_update_pose_async(ctx, nullptr));
  return predict_async(ctx);
}

// Input side of a frame: everything that depends neither on the map nor on the pose (ElasticFusion.cpp:278-285 and the
// live half of RGBDOdometry::initICP / initRGB). Runs on ctx->stream into the live buffer set.
static int frame_input_side(EfContext* ctx, const uint8_t* rgb_dev, const uint16_t* depth_dev) {
  const size_t n = (size_t)ctx->cfg.width * ctx->cfg.height;
  Textures& t = ctx->tex;
  // texture uploads, reference ElasticFusion.cpp:278-280
  if (rgb_dev != t.rgb) CU(cudaMemcpyAsync(t.rgb, rgb_dev, n * 3, cudaMemcpyDeviceToDevice, ctx->stream));
  if (depth_dev != t.depth_raw) CU(cudaMemcpyAsync(t.depth_raw, depth_dev, n * 2, cudaMemcpyDeviceToDevice, ctx->stream));
  RC(rgb_to_rgba(ctx, ctx->cfg.height, ctx->cfg.width, t.rgb, t.rgba));
  // filterDepth + metriciseDepth, ElasticFusion.cpp:284-285
  RC(preprocess_depth(ctx, ctx->cfg.height, ctx->cfg.width, t.depth_raw, ctx->depth_cutoff, t.depth_filtered, t.depth_metric,
                      t.depth_metric_filtered));
  if (ctx->stream != ctx->la.stream) ef_stage(ctx, 1);  // (stage events live on the main stream only)
  // frameToModel.initICP(filtered depth) and the intensity half of initRGB, ElasticFusion.cpp:318-319
  RC(odom_init_icp_depth(ctx, 0, t.depth_filtered, ctx->max_depth_processed));
  RC(odom_populate(ctx, 0, t.rgba, nullptr, ctx->odom[0].nextImage, false));
  // SO(3) pre-alignment (RGBDOdometry.cpp:305-368): needs only this intensity pyramid and the previous frame's
  // (lastNextImage), so it belongs to the input side. Not for the first frame (nothing is tracked, ElasticFusion.cpp:290).
  ctx->so3_ready = false;
  if (ctx->so3 && ctx->tick > 1) {
    RC(odom_so3_async(ctx, 0));
    ctx->so3_ready = true;
  }
  CU(cudaEventRecord(ctx->la.image_ready, ctx->stream));  // this pyramid is the next frame's lastNextImage
  return 0;
}

static void swap_sides(EfContext* ctx) {
  Lookahead& la = ctx->la;
  Textures& t = ctx->tex;
  OdomDev& od = ctx->odom[0];
  std::swap(t.rgb, la.rgb);
  std::swap(t.rgba, la.rgba);
  std::swap(t.depth_raw, la.depth_raw);
  std::swap(t.depth_filtered, la.depth_filtered);
  std::swap(t.depth_metric, la.depth_metric);
  std::swap(t.depth_metric_filtered, la.depth_metric_filtered);
  for (int i = 0; i < NUM_PYRS; ++i) {
    std::swap(od.depth_tmp[i], la.depth_tmp[i]);
    std::swap(od.vmap_curr[i], la.vmap_curr[i]);
    std::swap(od.nmap_curr[i], la.nmap_curr[i]);
    std::swap(od.nextImage[i], la.image[i]);
  }
  std::swap(od.so3s, la.so3s);
  std::swap(od.so3_partials, la.so3_partials);
  std::swap(od.so3_counter, la.so3_counter);
  std::swap(ctx->so3_ready, la.so3_ready);
}

// rgb/depth: device pointers, or pinned host staging when from_host
static int prefetch_common(EfContext* ctx, const uint8_t* rgb, const uint16_t* depth, bool from_host) {
  Lookahead& la = ctx->la;
  if (la.pending) return EF_ESTATE;
  const size_t n = (size_t)ctx->cfg.width * ctx->cfg.height;
  cudaStream_t main_stream = ctx->stream;
  swap_sides(ctx);  // the helpers below write the live pointers: make the spare set live while enqueueing
  ctx->stream = la.stream;
  int rc = 0;
  cudaError_t e = cudaStreamWaitEvent(la.stream, la.spare_free, 0);
  if (e == cudaSuccess) e = cudaStreamWaitEvent(la.stream, la.image_ready, 0);  // previous frame's intensity pyramid (SO(3) input)
  if (e == cudaSuccess && la.track_marked) e = cudaStreamWaitEvent(la.stream, la.track_started, 0);
  la.track_marked = false;
  if (e == cudaSuccess && ctx->stage_timing) e = cudaEventRecord(la.timing[0], la.stream);
  if (e == cudaSuccess && from_host) {
    e = cudaMemcpyAsync(ctx->tex.rgb, rgb, n * 3, cudaMemcpyHostToDevice, la.stream);
    if (e == cudaSuccess) e = cudaMemcpyAsync(ctx->tex.depth_raw, depth, n * 2, cudaMemcpyHostToDevice, la.stream);
    if (e == cudaSuccess) e = cudaEventRecord(la.h2d_done, la.stream);
    rgb = ctx->tex.rgb;
    depth = ctx->tex.depth_raw;
  }
  if (e != cudaSuccess) rc = (int)e;
  if (!rc) rc = frame_input_side(ctx, rgb, depth);
  if (!rc) {
    e = cudaEventRecord(la.ready, la.stream);
    if (e == cudaSuccess && ctx->stage_timing) e = cudaEventRecord(la.timing[1], la.stream);
    if (e != cudaSuccess) rc = (int)e;
  }
  ctx->stream = main_stream;
  swap_sides(ctx);
  if (!rc) la.pending = true;
  return rc;
}

extern "C" int ef_prefetch_frame_device(EfContext* ctx, const uint8_t* rgb_dev, const uint16_t* depth_dev) {
  if (!ctx || !rgb_dev || !depth_dev) return EF_EINVAL;
  return prefetch_common(ctx, rgb_dev, depth_dev, false);
}

extern "C" int ef_prefetch_frame(EfContext* ctx, const uint8_t* rgb, const uint16_t* depth) {
  if (!ctx || !rgb || !depth) return EF_EINVAL;
  if (ctx->la.pending) return EF_ESTATE;
  const size_t n = (size_t)ctx->cfg.width * ctx->cfg.height;
  CU(cudaEventSynchronize(ctx->la.h2d_done));  // the staging buffers of the previous prefetch have been read
  memcpy(ctx->la.pin_rgb, rgb, n * 3);
  memcpy(ctx->la.pin_depth, depth, n * 2);
  return prefetch_common(ctx, ctx->la.pin_rgb, ctx->la.pin_depth, true);
}

// The frame's side of the local loop closure: trackers 0 and 1, the context's textures and MapDev's loop buffers
static LoopSide frame_loop_side(EfContext* ctx) {
  const Textures& t = ctx->tex;
  const MapDev& m = ctx->map;
  LoopSide s = {};
  s.curr = 0;
  s.est = 1;
  s.rows = m.rows;
  s.cols = m.cols;
  s.max_depth = ctx->max_depth_processed;
  s.pyramid = ctx->pyramid;
  s.fast_odom = ctx->fast_odom;
  s.vertex = t.vertex;
  s.normal = t.normal;
  s.image = t.image;
  s.old_vertex = t.old_vertex;
  s.old_normal = t.old_normal;
  s.old_image = t.old_image;
  s.old_time = t.old_time;
  s.loop = m.loop;
  s.src = m.loop_src;
  s.dst = m.loop_dst;
  s.times = m.loop_times;
  s.capacity = m.loop_capacity;
  return s;
}

namespace ef {
// Local loop closure front half (ElasticFusion.cpp:447-505, the branch taken when no fern matched) once its INACTIVE prediction is
// made: modelToModel in the reference's order (initICPModel -> initRGBModel -> initICP(pred, pred) -> initRGB, App. A-2),
// getIncrementalTransformation(rgbOnly = false, icpWeight = 10, so3 = false), acceptance test and constraint sampling.
// Everything stays on the device (LoopDev); nothing is applied to the map or the pose.
int loop_tracker_inputs(EfContext* ctx, const LoopSide& s) {
  OdomDev& od = ctx->odom[s.est];
  RC(odom_copy_pose_async(ctx, s.est, s.curr));
  RC(odom_init_icp_model(ctx, s.est, (const float*)s.old_vertex, (const float*)s.old_normal, false));
  RC(odom_populate(ctx, s.est, (const uint8_t*)s.old_image, od.lastDepth, od.lastImage, true));
  RC(odom_init_icp_pred(ctx, s.est, (const float*)s.vertex, (const float*)s.normal));
  return odom_populate(ctx, s.est, (const uint8_t*)s.image, od.nextDepth, od.nextImage, true);
}

int loop_front_half(EfContext* ctx, const LoopSide& s) {
  RC(loop_tracker_inputs(ctx, s));
  RC(odom_track_async(ctx, s.est, false, 10.0f, s.pyramid, s.fast_odom, false));
  RC(odom_finish_async(ctx, s.est, 1.0f, true, nullptr));
  return map_loop_constraints_async(ctx, s);
}

// The closure itself once the front half ran (ElasticFusion.cpp:505-526; no fern matched). One small record is read back: whether
// it accepted, its constraint count and the node count of the graph sampled at the end of the previous frame or camera call. A
// graph exists once some call sampled more than 4 nodes (Deformation::def.isInit()). On an accepted closure with a graph and at
// least one constraint, the graph is solved on the device (pinned while nothing has been deformed, nodes up to lastDeformTime
// fixed, constraint source time `time`) and the solve's result is read back. Its nodes go to the clean and T_wc_est becomes the
// pose of tracker s.curr and of pose_record, whatever the solve's stop rule (the reference applies the graph unconditionally without
// a fern match), except stop 6, where nothing was solved; then Deformation's bookkeeping, which the frame and every closing camera
// share.
int loop_solve_apply(EfContext* ctx, const LoopSide& s, int time, MapPose* pose_record, DeformOutcome* out, int* n_nodes) {
  memset(out, 0, sizeof(*out));
  *n_nodes = 0;
  MapDev& m = ctx->map;
  PinStaging* p = ctx->pin_small;
  CU(cudaMemcpyAsync(p->loop_record, &s.loop->accepted, 2 * sizeof(int), cudaMemcpyDeviceToHost, ctx->stream));
  CU(cudaMemcpyAsync(p->loop_record + 2, m.graph_n, sizeof(int), cudaMemcpyDeviceToHost, ctx->stream));
  CU(cudaStreamSynchronize(ctx->stream));
  const int accepted = p->loop_record[0], n_cons = p->loop_record[1], graph_n = p->loop_record[2];
  if (!accepted || graph_n <= 0 || n_cons <= 0) return 0;
  const float* nodes16 = nullptr;
  RC(deform_solve_local(ctx, m.graph, graph_n, s.src, s.dst, s.times, n_cons, ctx->deforms == 0, time, ctx->last_deform_time,
                        &p->deform_result, &nodes16));
  out->solved = true;
  out->result = p->deform_result;
  if (out->result.stop == 6) return 0;
  // ef_process_frame_end(T_wc_est, graph): the pose, the map kernels' copy of it and the nodes the clean reads
  double* T = ctx->odom[s.curr].gn->T_wc;
  CU(cudaMemcpyAsync(T, s.loop->T_wc_est, sizeof(double) * 16, cudaMemcpyDeviceToDevice, ctx->stream));
  RC(map_pose_record_async(ctx, pose_record, T));
  RC(map_set_graph_device(ctx, nodes16, graph_n));
  *n_nodes = graph_n;
  out->applied = true;
  ctx->deforms += 1;             // ElasticFusion.cpp:518
  ctx->last_deform_time = time;  // Deformation.cpp:191-193
  return 0;
}
}  // namespace ef

// the frame's front half: the INACTIVE prediction into the old textures, then the shared steps
static int local_loop_async(EfContext* ctx) {
  RC(map_raycast_async(ctx, ctx->max_depth_processed, ctx->confidence, 0, ctx->tick - ctx->cfg.time_delta, ctx->cfg.time_delta, 1));
  return loop_front_half(ctx, frame_loop_side(ctx));
}

// First half of processFrame (ElasticFusion.cpp:270-534): input side, first-frame map / tracking, velocity weighting, the
// mid-frame predict() and the local loop closure front half. Asynchronous.
static int frame_begin_device(EfContext* ctx, const uint8_t* rgb_dev, const uint16_t* depth_dev, float weight_multiplier, const double* in_T_wc) {
  Textures& t = ctx->tex;
  Lookahead& la = ctx->la;
  if (ctx->frame_open) return EF_ESTATE;  // ef_process_frame_end has not been called for the previous frame
  ef_stage(ctx, 0);
  if (!rgb_dev) {
    // consume the prefetched frame: its buffer set becomes live, the previous live set becomes the spare one
    if (!la.pending) return EF_ESTATE;
    swap_sides(ctx);
    CU(cudaEventRecord(la.spare_free, ctx->stream));
    CU(cudaStreamWaitEvent(ctx->stream, la.ready, 0));
    la.pending = false;
  } else {
    if (la.pending) return EF_ESTATE;  // a prefetched frame must be consumed first (pass NULL, NULL)
    RC(frame_input_side(ctx, rgb_dev, depth_dev));
  }
  ef_stage(ctx, 2);
  ctx->frame_open = true;
  if (ctx->cfg.close_loops) RC(map_loop_reset_async(ctx, ctx->map.loop));

  if (ctx->tick == 1) {
    // ElasticFusion.cpp:290-296; initFirstRGB: the intensity pyramid of the first frame is the SO(3) "last" image
    RC(map_initialise_async(ctx));
    for (int i = 0; i < NUM_PYRS; ++i) std::swap(ctx->odom[0].nextImage[i], ctx->odom[0].lastNextImage[i]);
    return 0;
  }
  OdomDev& od = ctx->odom[0];
  if (!in_T_wc) {
    // ElasticFusion.cpp:302-323. The fill-in decision stays on the device: both candidate inputs are handed to the
    // pyramid kernels together with the lit-sample count that the raycast writing the image (or its upload) left.
    RC(map_select_model_inputs(ctx));
    // initRGB's depth half (populateRGBDData -> verticesToDepth(vmaps_tmp), RGBDOdometry.cpp:212-222) reads the SAME
    // vmaps_tmp initICPModel just filled, so in frame-to-model mode nextDepth is identical to lastDepth: alias it for
    // the tracking call instead of building the pyramid twice.
    float* saved[NUM_PYRS];
    const bool alias = !ctx->frame_to_frame_rgb;
    if (alias) {
      for (int i = 0; i < NUM_PYRS; ++i) {
        saved[i] = od.nextDepth[i];
        od.nextDepth[i] = od.lastDepth[i];
      }
    } else {
      RC(odom_populate(ctx, 0, t.rgba, od.nextDepth, od.nextImage, true, false));
    }
    ef_stage(ctx, 3);
    int rc = odom_track_async(ctx, 0, ctx->rgb_only, ctx->icp_weight, ctx->pyramid, ctx->fast_odom, ctx->so3);
    if (alias)
      for (int i = 0; i < NUM_PYRS; ++i) od.nextDepth[i] = saved[i];
    RC(rc);
    RC(odom_finish_async(ctx, 0, weight_multiplier, true, ctx->map.pose));
  } else {
    CU(cudaStreamSynchronize(ctx->stream));
    memcpy(ctx->pin_small->T_wc, in_T_wc, sizeof(double) * 16);
    CU(cudaMemcpyAsync(ctx->dev_small->T_wc, ctx->pin_small->T_wc, sizeof(double) * 16, cudaMemcpyHostToDevice, ctx->stream));
    ctx->so3_ready = false;  // no tracking for this frame: the SO(3) result of its input side is not used
    RC(odom_set_pose_async(ctx, 0, ctx->dev_small->T_wc));
    RC(odom_finish_async(ctx, 0, weight_multiplier, false, ctx->map.pose));
  }
  // (k_gn_finish also refreshed the map kernels' float pose + inverse from the new T_wc)
  ef_stage(ctx, 6);
  // ElasticFusion.cpp:387: only loop closure reads this prediction
  if (!ctx->cfg.skip_mid_predict || ctx->cfg.close_loops) RC(predict_async(ctx));
  if (ctx->cfg.close_loops && !ctx->rgb_only) RC(local_loop_async(ctx));
  return 0;
}

// Second half of processFrame (ElasticFusion.cpp:536-607): index map, fuse, index map, clean (with the deformation graph stored by
// ef_set_deformation_graph when n_nodes > 0), predict, tick++.
static int frame_map_device(EfContext* ctx, int n_nodes, bool fern_accepted) {
  const MapTarget t = map_frame_target(ctx);
  RC(map_predict_indices_async(ctx, t, ctx->tick, ctx->max_depth_processed, ctx->cfg.time_delta, 1));
  ef_stage(ctx, 7);
  RC(map_fuse_async(ctx, t, ctx->tick, ctx->max_depth_processed, -1.0f));
  ef_stage(ctx, 8);
  RC(map_predict_indices_async(ctx, t, ctx->tick, ctx->max_depth_processed, ctx->cfg.time_delta, 2));
  ef_stage(ctx, 9);
  if (n_nodes > 0 && !fern_accepted)  // ElasticFusion.cpp:559-569: the time-stamp refresh of deformed surfels reads this depth
    RC(map_raycast_async(ctx, ctx->max_depth_processed, ctx->confidence, ctx->tick, ctx->tick - ctx->cfg.time_delta, 65535, 2));
  RC(map_clean_async(ctx, t, ctx->tick, ctx->confidence, ctx->cfg.time_delta, ctx->max_depth_processed, n_nodes, fern_accepted));
  ef_stage(ctx, 10);
  return 0;
}

static int frame_end_device(EfContext* ctx, int n_nodes, bool fern_accepted) {
  if (!ctx->frame_open) return EF_ESTATE;
  if (ctx->tick > 1 && !ctx->rgb_only) {
    if (int rc = frame_map_device(ctx, n_nodes, fern_accepted)) {
      map_index_textures_async(ctx, map_frame_target(ctx));  // a pass whose clean did not run still leaves its textures, as the stage API's passes do
      return rc;
    }
  }
  if (ctx->tick == 1) RC(map_update_pose_async(ctx, nullptr));  // later frames: done by k_gn_finish, pose unchanged since
  RC(predict_async(ctx));  // ElasticFusion.cpp:599
  ef_stage(ctx, 11);
  ctx->tick++;
  ctx->frame_open = false;
  return 0;
}

// close_loops = 2: the rest of a frame whose first half frame_begin_device has enqueued, with the local loop closure closed inside it
// (ElasticFusion.cpp:505-534, 536-593; no fern matched): when the front half ran, loop_solve_apply; then the second half of the
// frame and, after clean as at :593, the graph for the next frame is sampled.
static int frame_local_deform(EfContext* ctx) {
  memset(&ctx->deform_out, 0, sizeof(ctx->deform_out));
  int n_nodes = 0;
  if (ctx->tick > 1 && !ctx->rgb_only)  // the front half ran (frame_begin_device)
    RC(loop_solve_apply(ctx, frame_loop_side(ctx), ctx->tick, ctx->map.pose, &ctx->deform_out, &n_nodes));
  RC(frame_end_device(ctx, n_nodes, false));
  return map_sample_graph_async(ctx);  // (predict, which frame_end_device ran after clean, leaves the surfels as they are)
}

extern "C" int ef_process_frame_device(EfContext* ctx, const uint8_t* rgb_dev, const uint16_t* depth_dev, int64_t timestamp,
                                       float weight_multiplier, const double* in_T_wc) {
  (void)timestamp;
  if (!ctx || ((rgb_dev == nullptr) != (depth_dev == nullptr))) return EF_EINVAL;
  RC(frame_begin_device(ctx, rgb_dev, depth_dev, weight_multiplier, in_T_wc));
  if (ctx->cfg.close_loops == 2) return frame_local_deform(ctx);
  return frame_end_device(ctx, 0, false);
}

// host frame -> pinned staging -> the live input textures, on ctx->stream
static int stage_host_frame(EfContext* ctx, const uint8_t* rgb, const uint16_t* depth) {
  const size_t n = (size_t)ctx->cfg.width * ctx->cfg.height;
  CU(cudaStreamSynchronize(ctx->stream));  // the staging buffers may still be in flight from the previous frame
  memcpy(ctx->pin_rgb, rgb, n * 3);
  memcpy(ctx->pin_depth, depth, n * 2);
  CU(cudaMemcpyAsync(ctx->tex.rgb, ctx->pin_rgb, n * 3, cudaMemcpyHostToDevice, ctx->stream));
  CU(cudaMemcpyAsync(ctx->tex.depth_raw, ctx->pin_depth, n * 2, cudaMemcpyHostToDevice, ctx->stream));
  return 0;
}

// processFrame split at the point where the reference hands control to its CPU deformation solver (ElasticFusion.cpp:505-526):
// begin = everything up to and including the local loop closure front half, end = fuse / clean / predict. Between the two
// the host may read ef_local_loop_result, run Deformation::constrain (unchanged reference code) and hand its output back:
// T_wc_override (T_wc_curr = T_wc_est) and the graph nodes applied inside clean.
extern "C" int ef_process_frame_begin(EfContext* ctx, const uint8_t* rgb, const uint16_t* depth, int64_t timestamp, float weight_multiplier,
                                      const double* in_T_wc) {
  (void)timestamp;
  if (!ctx || !rgb || !depth) return EF_EINVAL;
  if (ctx->la.pending || ctx->frame_open || ctx->cfg.close_loops == 2) return EF_ESTATE;  // mode 2 closes its loops itself
  RC(stage_host_frame(ctx, rgb, depth));
  RC(frame_begin_device(ctx, ctx->tex.rgb, ctx->tex.depth_raw, weight_multiplier, in_T_wc));
  return ef_finish_frame(ctx);  // pose (and the loop-closure result) are final on return
}

extern "C" int ef_process_frame_end(EfContext* ctx, const double* T_wc_override, const float* graph_nodes16, int32_t n_nodes, int32_t fern_accepted) {
  if (!ctx || n_nodes < 0 || (n_nodes > 0 && !graph_nodes16)) return EF_EINVAL;
  if (!ctx->frame_open || ctx->cfg.close_loops == 2) return EF_ESTATE;
  if (T_wc_override) {
    RC(ef_set_pose(ctx, T_wc_override));
    RC(map_update_pose_async(ctx, nullptr));
  }
  RC(map_set_graph(ctx, graph_nodes16, n_nodes));
  RC(frame_end_device(ctx, n_nodes, fern_accepted != 0));
  return ef_finish_frame(ctx);
}

// one side's last closure, the shared bookkeeping and the current graph (ef_local_deform_result, ef_camera_deform_result)
static int deform_report(EfContext* ctx, const DeformOutcome& d, EfLocalDeform* out, float* nodes4, int32_t max_nodes, int32_t* n_out) {
  int n = 0;
  RC(read_count(ctx, ctx->map.graph_n, &n));
  out->solved = d.solved;
  out->applied = d.applied;
  out->result = d.result;
  out->deforms = ctx->deforms;
  out->last_deform_time = ctx->last_deform_time;
  out->n_nodes = n;
  if (n > max_nodes) n = max_nodes;
  if (n_out) *n_out = n;
  if (n > 0) {
    CU(cudaMemcpyAsync(nodes4, ctx->map.graph, sizeof(float) * 4 * n, cudaMemcpyDeviceToHost, ctx->stream));
    CU(cudaStreamSynchronize(ctx->stream));
  }
  return 0;
}

extern "C" int ef_local_deform_result(EfContext* ctx, EfLocalDeform* out, float* nodes4, int32_t max_nodes, int32_t* n_out) {
  if (!ctx || !out || max_nodes < 0 || (max_nodes > 0 && !nodes4)) return EF_EINVAL;
  if (ctx->cfg.close_loops != 2) return EF_ESTATE;
  return deform_report(ctx, ctx->deform_out, out, nodes4, max_nodes, n_out);
}

extern "C" int ef_camera_deform_result(EfContext* ctx, EfCamera* cam, EfLocalDeform* out, float* nodes4, int32_t max_nodes, int32_t* n_out) {
  if (!camera_of(ctx, cam) || !out || max_nodes < 0 || (max_nodes > 0 && !nodes4)) return EF_EINVAL;
  if (!cam->cfg.close_loops || cam->rig) return EF_ESTATE;
  CU(cudaSetDevice(ctx->device));
  return deform_report(ctx, cam->deform_out, out, nodes4, max_nodes, n_out);
}

extern "C" int ef_rig_deform_result(EfContext* ctx, EfRig* rig, EfLocalDeform* out, float* nodes4, int32_t max_nodes, int32_t* n_out) {
  if (!rig_of(ctx, rig) || !out || max_nodes < 0 || (max_nodes > 0 && !nodes4)) return EF_EINVAL;
  if (!rig->closing) return EF_ESTATE;
  CU(cudaSetDevice(ctx->device));
  return deform_report(ctx, rig->deform_out, out, nodes4, max_nodes, n_out);
}

extern "C" int ef_rig_loop_result(EfContext* ctx, EfRig* rig, EfRigLoopResult* out, double* src3, double* dst3, int32_t* times,
                                  int32_t max_constraints, int32_t* n_out) {
  if (!rig_of(ctx, rig) || !out || max_constraints < 0) return EF_EINVAL;
  if (!rig->closing) return EF_ESTATE;
  CU(cudaSetDevice(ctx->device));
  LoopDev h;
  RigLoopDev rec;
  CU(cudaMemcpyAsync(&h, rig->loop, sizeof(h), cudaMemcpyDeviceToHost, ctx->stream));
  CU(cudaMemcpyAsync(&rec, rig->loop_rec, sizeof(rec), cudaMemcpyDeviceToHost, ctx->stream));
  CU(cudaStreamSynchronize(ctx->stream));
  memset(out, 0, sizeof(*out));
  out->ran = h.ran;
  out->accepted = h.accepted;
  out->n_constraints = h.n_constraints;
  for (int m = 0; m < EF_MAX_CAMERAS; ++m) out->member_constraints[m] = rec.member_n[m];
  out->lastICPError = h.lastICPError;
  out->lastICPCount = h.lastICPCount;
  memcpy(out->cov_diag, h.cov_diag, sizeof(h.cov_diag));
  memcpy(out->T_wc_curr, rec.T_wc_curr, sizeof(rec.T_wc_curr));
  memcpy(out->T_wc_est, h.T_wc_est, sizeof(h.T_wc_est));
  int n = h.n_constraints < max_constraints ? h.n_constraints : max_constraints;
  if (n > rig->capacity) n = rig->capacity;
  if (n_out) *n_out = n;
  if (n > 0) {
    if (src3) CU(cudaMemcpyAsync(src3, rig->src, sizeof(double) * 3 * n, cudaMemcpyDeviceToHost, ctx->stream));
    if (dst3) CU(cudaMemcpyAsync(dst3, rig->dst, sizeof(double) * 3 * n, cudaMemcpyDeviceToHost, ctx->stream));
    if (times) CU(cudaMemcpyAsync(times, rig->times, sizeof(int) * n, cudaMemcpyDeviceToHost, ctx->stream));
    CU(cudaStreamSynchronize(ctx->stream));
  }
  return 0;
}

extern "C" int ef_local_loop_result(EfContext* ctx, EfLoopResult* out, double* src3, double* dst3, int32_t* times, int32_t max_constraints,
                                    int32_t* n_out) {
  if (!ctx || !out || max_constraints < 0) return EF_EINVAL;
  const MapDev& m = ctx->map;
  LoopDev h;
  CU(cudaMemcpyAsync(&h, m.loop, sizeof(h), cudaMemcpyDeviceToHost, ctx->stream));
  CU(cudaStreamSynchronize(ctx->stream));
  out->ran = h.ran;
  out->accepted = h.accepted;
  out->n_constraints = h.n_constraints;
  out->lastICPError = h.lastICPError;
  out->lastICPCount = h.lastICPCount;
  memcpy(out->cov_diag, h.cov_diag, sizeof(h.cov_diag));
  memcpy(out->T_wc_est, h.T_wc_est, sizeof(h.T_wc_est));
  int n = h.n_constraints < max_constraints ? h.n_constraints : max_constraints;
  if (n > m.loop_capacity) n = m.loop_capacity;
  if (n_out) *n_out = n;
  if (n > 0) {
    if (src3) CU(cudaMemcpyAsync(src3, m.loop_src, sizeof(double) * 3 * n, cudaMemcpyDeviceToHost, ctx->stream));
    if (dst3) CU(cudaMemcpyAsync(dst3, m.loop_dst, sizeof(double) * 3 * n, cudaMemcpyDeviceToHost, ctx->stream));
    if (times) CU(cudaMemcpyAsync(times, m.loop_times, sizeof(int) * n, cudaMemcpyDeviceToHost, ctx->stream));
    CU(cudaStreamSynchronize(ctx->stream));
  }
  return 0;
}

// Deformation::constrain for a local loop closure (Deformation.cpp:73-207) on host inputs: constraints are expanded to
// [c0, pin0, c1, pin1, ...] when `pin` is set (addConstraint, :73-86), then weighted, solved and handed over on the device.
extern "C" int ef_deform_solve(EfContext* ctx, const double* node_pos3, const int32_t* node_times, int32_t n_nodes, const double* src3,
                               const double* dst3, const int32_t* src_times, const int32_t* dst_times, int32_t n_constraints, int32_t pin,
                               int32_t last_deform_time, float* nodes16, double* rt12, int32_t* cons_nodes4, double* cons_weights4,
                               EfDeformResult* out) {
  if (!ctx || !out || !node_pos3 || !node_times || !src3 || !dst3 || !src_times || (pin && !dst_times)) return EF_EINVAL;
  if (n_nodes < 5 || n_nodes >= MAX_GRAPH_NODES || n_constraints < 1 || last_deform_time < 0) return EF_EINVAL;
  for (int i = 0; i < n_nodes; ++i)  // the graph is sampled in time order (Deformation.cpp:294-296)
    if (node_times[i] < 0 || (i > 0 && node_times[i] < node_times[i - 1])) return EF_EINVAL;
  const int m = pin ? 2 * n_constraints : n_constraints;
  std::vector<double> s(3 * (size_t)m), d(3 * (size_t)m);
  std::vector<int32_t> t(m);
  for (int i = 0, o = 0; i < n_constraints; ++i) {
    if (src_times[i] < 0 || (pin && dst_times[i] < 0)) return EF_EINVAL;
    memcpy(&s[3 * o], src3 + 3 * i, sizeof(double) * 3);
    memcpy(&d[3 * o], dst3 + 3 * i, sizeof(double) * 3);
    t[o++] = src_times[i];
    if (pin) {  // (target, target, targetTime, targetTime)
      memcpy(&s[3 * o], dst3 + 3 * i, sizeof(double) * 3);
      memcpy(&d[3 * o], dst3 + 3 * i, sizeof(double) * 3);
      t[o++] = dst_times[i];
    }
  }
  CU(cudaSetDevice(ctx->device));
  return deform_solve(ctx, node_pos3, node_times, n_nodes, s.data(), d.data(), t.data(), m, last_deform_time, nodes16, rt12,
                      cons_nodes4, cons_weights4, out);
}

// Makes the main stream wait for the side stream's staged frame (a no-op without a pending frame): after this call every
// kernel enqueued so far, on either stream, precedes whatever the caller records on ef_stream() next.
extern "C" int ef_join_lookahead(EfContext* ctx) {
  if (!ctx) return EF_EINVAL;
  if (ctx->la.pending) CU(cudaStreamWaitEvent(ctx->stream, ctx->la.ready, 0));
  return 0;
}

// Completes the frame enqueued by ef_process_frame_device: pose and surfel count are read back and final on return.
extern "C" int ef_finish_frame(EfContext* ctx) {
  if (!ctx) return EF_EINVAL;
  PinStaging* s = ctx->pin_small;
  CU(cudaMemcpyAsync(s->finish_T_wc, ctx->odom[0].gn->T_wc, sizeof(double) * 16, cudaMemcpyDeviceToHost, ctx->stream));
  CU(cudaMemcpyAsync(&s->finish_count, ctx->map.count, 4, cudaMemcpyDeviceToHost, ctx->stream));
  CU(cudaStreamSynchronize(ctx->stream));
  memcpy(ctx->T_wc, s->finish_T_wc, sizeof(double) * 16);
  ctx->host_count = s->finish_count;
  return 0;
}

extern "C" int ef_process_frame(EfContext* ctx, const uint8_t* rgb, const uint16_t* depth, int64_t timestamp, float weight_multiplier,
                                const double* in_T_wc) {
  if (!ctx || ((rgb == nullptr) != (depth == nullptr))) return EF_EINVAL;
  if (!rgb) {
    RC(ef_process_frame_device(ctx, nullptr, nullptr, timestamp, weight_multiplier, in_T_wc));  // prefetched frame
    return ef_finish_frame(ctx);
  }
  if (ctx->la.pending) return EF_ESTATE;  // a prefetched frame must be consumed first; nothing has been touched yet
  RC(stage_host_frame(ctx, rgb, depth));
  RC(ef_process_frame_device(ctx, ctx->tex.rgb, ctx->tex.depth_raw, timestamp, weight_multiplier, in_T_wc));
  // results the caller can observe (get_T_wc, counts) are final on return
  return ef_finish_frame(ctx);
}

// debug exports (phase profiling builds)
// EF_STAGE_TIMING=1: milliseconds between consecutive stage events of the last frame (0 start, 1 upload + RGBA + bilateral/metric,
// 2 live pyramids + SO(3) loop, 3 model pyramids, 4 sobel + candidates + begin, 5 Gauss-Newton loop, 6 finish, 7 index map, 8 fuse,
// 9 index map, 10 clean, 11 predict); returns the event count. Stages 2..6 are what the reference does inside
// RGBDOdometry::init* + getIncrementalTransformation.
extern "C" int ef_debug_stage_ms(EfContext* ctx, float* out) {
  if (!ctx || !ctx->stage_timing) return 0;
  cudaStreamSynchronize(ctx->stream);
  int prev = -1;
  for (int i = 0; i < 16; ++i) {
    out[i] = 0.f;
    if (!(ctx->stage_n >> i & 1)) continue;
    if (prev >= 0) cudaEventElapsedTime(&out[i], ctx->stage_ev[prev], ctx->stage_ev[i]);
    prev = i;
  }
  return 12;
}
// EF_STAGE_TIMING=1: milliseconds from the start of the frame in flight during the last prefetch (stage event 0) to the start of
// the side stream's work (once its waits are met) and to its end; returns 2, or 0 without a timed prefetch.
extern "C" int ef_debug_lookahead_ms(EfContext* ctx, float* out2) {
  if (!ctx || !out2 || !ctx->stage_timing || !(ctx->stage_n & 1)) return 0;
  if (cudaStreamSynchronize(ctx->la.stream) != cudaSuccess) return 0;
  for (int i = 0; i < 2; ++i)
    if (cudaEventElapsedTime(&out2[i], ctx->stage_ev[0], ctx->la.timing[i]) != cudaSuccess) return 0;
  return 2;
}
extern "C" void* ef_debug_gn(EfContext* ctx, int which) { return ctx ? (void*)ctx->odom[which].gn : nullptr; }
extern "C" int ef_debug_gn_size() { return (int)sizeof(GNState); }
extern "C" int ef_debug_dbg_offset() { return (int)offsetof(GNState, dbg); }
