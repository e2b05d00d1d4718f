// Internal context layout of libefusion.so (not part of the ABI).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/efusion_b200.h"

namespace ef {

constexpr int NUM_PYRS = 3;          // RGBDOdometry::NUM_PYRS (reference Core/Utils/RGBDOdometry.h:114)
constexpr int RED_THREADS = 256;     // threads per reduction CTA
constexpr int MAX_RED_BLOCKS = 1184; // 8 resident 256-thread CTAs per SM on up to 148 SMs (H100: 132)
constexpr int PARTIAL_STRIDE = 64;   // floats per CTA partial: [0,29) geometric system, [32,61) photometric system
constexpr int MAX_TRACE = 48;
constexpr int MAX_RGB_BLOCKS = 160;

// reference DataTerm (Core/Cuda/types.cuh:79-84): 16 bytes, bool widened to int32
struct DataTerm {
  short zero_x, zero_y;
  short one_x, one_y;
  float diff;
  int valid;
};

// Device-resident state of one getIncrementalTransformation call: everything the reference keeps in host
// locals between kernel launches (RGBDOdometry.cpp:259-571) lives here so no iteration needs the host.
struct GNState {
  double T_wc[16];
  float lastICPError, lastICPCount, lastRGBError, lastRGBCount, lastSO3Error, lastSO3Count;
  double lastA[36], lastb[6];

  float Rprev[9], tprev[3], Rprev_inv[9];
  float Rcurr[9], tcurr[3];
  float Mcp[9], tcp[3];  // current camera -> previous camera: R_prev^-1 R_curr, R_prev^-1 (t_curr - t_prev) (= the inverse increment)
  double resultRt[16];
  int break_level;  // rgbOnly early exit of one pyramid level's loop (-1: none)

  float krkinv[9], kt[3];                  // inputs of the next photometric residual pass
  float sigmaVal;
  int rgbSize, sigma;

  float sum_icp[32], sum_rgb[32];  // last reduced systems (reference JtJJtrSE3 order)
  int sum_res[2];                               // last {count, sigma} of the residual pass
  unsigned int res_acc[2];                      // accumulators of the running residual pass (re-armed by k_iter2)

  int rgbOnly, icp, rgb, so3;
  float icpWeight;
  float fx, fy, cx, cy;
  double Kd[NUM_PYRS][9], Kinvd[NUM_PYRS][9];  // per-level K (float intrinsics / 2^level, widened) and its inverse
  int trace_n;
  int cand_base[NUM_PYRS + 1];  // photometric candidates of level L live in cand[cand_base[L], cand_base[L+1])
  int flat_n;                   // total pixels over the three levels
  float rgbErrBuf[2];           // rgbError of the previous / current iteration (double-buffered across CTAs)
  float weighting;  // velocity weighting for fusion (ElasticFusion.cpp:369-383)
  long long dbg[40];  // phase timestamps (%globaltimer) of levels 0 and 1 when built with -DEF_PROFILE_PHASES
};

// State of the SO(3) pre-alignment loop (RGBDOdometry.cpp:305-368). The loop depends only on the two intensity pyramids
// (previous and current frame, level 2) -- not on the map, not on the pose -- so it has its own block, one per buffer set,
// and runs with the rest of the frame's input side (on the look-ahead stream when the frame was prefetched).
constexpr int SO3_MAX_ITER = 10;
struct So3State {
  double resultR[9], lastResultR[9];
  float R_lr[9];
  float imageBasis[9], kinv[9], krlr[9];  // inputs of the next pass
  float so3_lastError, so3_lastCount;
  int so3_done;
  float sum_so3[12];                      // last reduced system (reference JtJJtrSO3 order)
  float lastSO3Error, lastSO3Count;
  int trace_n;
  EfSolveTrace trace[SO3_MAX_ITER];
};

// pose matrices consumed by the map kernels (float, as the reference's shader uniforms)
struct MapPose {
  float pose[16];   // T_wc
  float t_inv[16];  // T_cw
};

struct OdomDev {
  int width, height;
  int rows[NUM_PYRS], cols[NUM_PYRS];
  float distThres, angleThres;
  float sobelScale, maxDepthDeltaRGB, maxDepthRGB;
  float minGrad[NUM_PYRS];
  float minScale[NUM_PYRS];  // (minGrad/sobelScale)^2, reference RGBDOdometry.cpp:425

  uint16_t* depth_tmp[NUM_PYRS];
  float* vmaps_tmp;  // float4 AoS, level 0
  float *vmap_g_prev[NUM_PYRS], *nmap_g_prev[NUM_PYRS], *vmap_curr[NUM_PYRS], *nmap_curr[NUM_PYRS];
  float *vmap_c_prev[NUM_PYRS], *nmap_c_prev[NUM_PYRS];  // model maps in the previous camera's frame (what the ICP kernel reads)
  float *lastDepth[NUM_PYRS], *nextDepth[NUM_PYRS];
  uint8_t *lastImage[NUM_PYRS], *nextImage[NUM_PYRS], *lastNextImage[NUM_PYRS];
  int16_t *dIdx[NUM_PYRS], *dIdy[NUM_PYRS];
  DataTerm* corres[NUM_PYRS];
  // photometric candidates: pixels that pass every pose-independent gate of computeRgbResidual (reference reduce.cu:641-660),
  // compacted once per frame; {pixel index, nextDepth bits, dIdx | dIdy << 16, nextImage}
  int4* cand;
  const int* cand_base;   // = gn->cand_base (device address): bounds of each level's candidates; like `cand`, final before the loop starts
  const float* intr0;     // = &gn->fx (device address): level-0 {fx, fy, cx, cy}, written once at context creation
  const double* K_levels; // = gn->Kd (device address): K of each level, then K^-1 of each level (gn->Kinvd); written once as well
  int4* terms;            // per candidate and iteration: {zero_x | zero_y << 16 (or -1), diff bits, dIdx | dIdy << 16, lastDepth[zero] bits}
  int level_start[NUM_PYRS + 1];  // flat pixel offset of each level

  GNState* gn;
  So3State* so3s;             // SO(3) loop state + its own partials / ticket (it may run concurrently with the GN loop of
  float* so3_partials;        // the previous frame); MAX_RED_BLOCKS * PARTIAL_STRIDE, one slot per CTA of k_so3_step
  unsigned int* so3_counter;
  float* partials;        // MAX_RED_BLOCKS * PARTIAL_STRIDE (geometric system, one slot per CTA of the dense pass)
  double* partials2;      // MAX_RGB_BLOCKS * 32: second-level sums of `partials`, one slot per CTA of the candidate pass
  float* partials_rgb;    // MAX_RGB_BLOCKS * 32 (photometric system, one slot per CTA of the candidate pass)
  int* partials_i;        // MAX_RED_BLOCKS * 2
  unsigned int* counter;  // last-block ticket
  EfSolveTrace* trace;    // MAX_TRACE records (device)
};

constexpr int MAX_GRAPH_NODES = 1024;  // GlobalModel::MAX_NODES = 16384 / 16 (GlobalModel.cpp:25-26)

// device-resident result of the local loop closure front half (ElasticFusion.cpp:447-505); the constraint pairs themselves
// live in MapDev::loop_src / loop_dst / loop_times, sized from the frame
struct LoopDev {
  int ran, accepted, n_constraints;
  float lastICPError, lastICPCount;
  double cov_diag[6];
  double T_wc_est[16];
};

// constraints of one local loop closure: at most one per cell of the (W/20) x (H/20) sample grid (ElasticFusion.cpp:487-503;
// the reference keeps them in a std::vector): 768 at 640x480, 5184 at 1920x1080
inline int loop_constraint_capacity(int width, int height) { return (width / 20) * (height / 20); }

struct MapDev {
  int rows, cols;
  float cx, cy, fx, fy;
  int capacity;
  // surfel map, SoA of float4: pos+conf | colour,unused,initTime,lastTime | normal+radius
  float4 *pos_conf, *color_time, *norm_rad;
  int* count;             // device-resident surfel count
  // unstable surfels of the current frame (reference newUnstableVbo)
  float4 *new_pos, *new_col, *new_nr;
  int* new_count;
  // per-pixel association scratch for fuse
  uint32_t* assoc_id;     // W*H: matched surfel id (or 0xffffffff none / 0xfffffffe new)
  uint32_t* pending;      // capacity: lowest draw index that chose this surfel (0xffffffff idle)
  // z-buffers
  unsigned long long* zbuf;  // W*H
  // scan scratch
  int* scan_tile_state;   // decoupled look-back
  unsigned int* scan_counter;
  uint32_t* vis_list;        // surfels that reached the z-buffer in the frame's first index-map pass (k_index_scatter<1>)
  int* vis_count;
  unsigned int* clean_ctl;   // [0] tile dispenser, [1] exit tickets, [2] first tile that moves (k_clean_flags -> k_clean_move)
  uint32_t* keep_mask;       // one warp ballot per 32 surfels: the clean test's verdicts
  uint8_t* flags;         // capacity + W*H
  // first-frame feedback buffers
  float4 *fb_raw[3], *fb_filt[3];
  int* fb_count;          // [2]
  MapPose* pose;          // device
  int* dense_flag;        // device: 1 if the predicted image is dense enough (no fill-in)
  int* tick;              // device-resident tick
  float* nodes;           // deformation graph of the current frame, 16 floats per node
  LoopDev* loop;
  int loop_capacity;      // loop_constraint_capacity(cols, rows)
  double *loop_src, *loop_dst;  // loop_capacity x 3: vert_w_curr / vert_w_est of each constraint
  int* loop_times;              // loop_capacity: the INACTIVE view's time stamp of each constraint
};

struct Textures {
  uint8_t* rgb;      // W*H*3
  uint8_t* rgba;     // W*H*4
  uint16_t* depth_raw;
  uint16_t* depth_filtered;
  float* depth_metric;
  float* depth_metric_filtered;
  // IndexMap
  uint32_t* index;
  float4 *vert_conf, *color_time, *norm_rad;
  uchar4 *image, *old_image, *fill_image;
  float4 *vertex, *normal, *old_vertex, *old_normal, *fill_vertex, *fill_normal;
  uint16_t *time, *old_time;
  float* synth_depth;
};

// Look-ahead ("prefetch") of the next frame: everything of a frame that does not depend on the map or the pose -- upload,
// RGBA expansion, bilateral filter + metric depth, depth pyramid + vertex/normal maps, intensity pyramid -- can run on a
// side stream while the previous frame is still in its (latency-bound) Gauss-Newton loop. The products live in a spare
// set of buffers that is swapped with the live pointers of Textures / OdomDev when the frame is consumed.
struct Lookahead {
  cudaStream_t stream;
  cudaEvent_t ready;       // side stream: the spare set is complete
  cudaEvent_t spare_free;  // main stream: every reader of the spare set precedes this point
  cudaEvent_t h2d_done;    // side stream: the pinned staging buffers may be rewritten
  cudaEvent_t image_ready; // whichever stream built the newest intensity pyramid (the next frame's SO(3) loop reads it)
  cudaEvent_t track_started;  // main stream: the frame's coarse-level cluster (or k_gn_begin) has been enqueued before this
  bool track_marked;          // track_started was recorded by the frame in flight and the next prefetch has not waited on it
  cudaEvent_t timing[2];   // EF_STAGE_TIMING=1: start (after its waits) and end of the side stream's work of the last prefetch
  bool pending;            // a prefetched frame is waiting to be consumed
  uint8_t *rgb, *rgba;
  uint16_t *depth_raw, *depth_filtered;
  float *depth_metric, *depth_metric_filtered;
  uint16_t* depth_tmp[NUM_PYRS];
  float *vmap_curr[NUM_PYRS], *nmap_curr[NUM_PYRS];
  uint8_t* image[NUM_PYRS];
  So3State* so3s;
  float* so3_partials;
  unsigned int* so3_counter;
  bool so3_ready;          // the spare set holds a finished SO(3) loop for its frame
  uint8_t* pin_rgb;
  uint16_t* pin_depth;
};

}  // namespace ef

struct EfContext {
  EfConfig cfg;
  int device;
  int num_sms;
  cudaStream_t stream;
  bool own_stream;
  int64_t launches;
  bool stage_timing;            // EF_STAGE_TIMING=1: record an event after every stage of ef_process_frame_device
  cudaEvent_t stage_ev[16];
  int stage_n;
  bool pdl;  // programmatic dependent launch on every kernel (default on; EF_NO_PDL=1 disables)
  bool vis_pending;      // the first pass of a frame has filled the visible list and the second has not consumed it yet
  bool visible_list;      // second index-map pass of a frame visits only the surfels the first one rasterised; EF_VISIBLE_LIST=0 disables
  int gn_cluster;         // CTAs of the clusters that run the SO(3) loop and the coarse-level Gauss-Newton iterations (0: plain launches everywhere)
  int gn_cluster_levels;  // pyramid levels, from the coarsest, whose iterations run in that cluster
  bool la_after_track;    // the look-ahead's side stream starts after the frame's coarse-level cluster (EF_LA_AFTER_TRACK=0: at frame start)
  bool plain_next;     // the next ef_launch omits the programmatic-serialisation attribute (EF_PLAIN_NEXT)
  bool maps_dirty[2];  // a kernel that writes tracker w's pyramids may still be in flight ahead of the next stage launch

  ef::OdomDev odom[2];
  ef::MapDev map;
  ef::Textures tex;
  ef::Lookahead la;
  bool so3_ready;  // the live set of odom[0] holds a finished SO(3) loop for the frame about to be tracked

  // host mirrors
  int tick;
  double T_wc[16];
  bool rgb_only;
  float icp_weight;
  bool pyramid, fast_odom, so3, frame_to_frame_rgb;
  float confidence, depth_cutoff, max_depth_processed;
  int host_count;  // last count read back
  bool frame_open; // ef_process_frame_begin has run, ef_process_frame_end has not

  // pinned staging
  uint8_t* pin_rgb;
  uint16_t* pin_depth;
  void* pin_small;   // results read-back
  void* dev_small;   // upload area for per-call parameters
  void* map_host;    // host-side bookkeeping of the surfel buffers (ef_map.cu)
  void* deform;      // workspace of the deformation-graph solve (ef_deform.cu), allocated by its first call
};

// launch bookkeeping
inline void ef_stage(EfContext* ctx, int i) {
  if (ctx->stage_timing) {
    cudaEventRecord(ctx->stage_ev[i], ctx->stream);
    if (i == 0) ctx->stage_n = 0;  // bit mask of the events recorded for this frame
    ctx->stage_n |= 1 << i;
  }
}
// Every kernel is launched with programmatic stream serialisation allowed (see pdl_enter() in ef_device.cuh); set
// EF_NO_PDL=1 in the environment to fall back to plain stream-ordered launches (A/B measurements).
template <typename... KArgs, typename... Args>
inline void ef_launch(EfContext* ctx, void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, Args&&... args) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = ctx->stream;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = (ctx->pdl && !ctx->plain_next) ? 1 : 0;
  ctx->plain_next = false;
  cudaLaunchKernelEx(&cfg, kernel, static_cast<KArgs>(args)...);
  ctx->launches++;
}
#define EF_LAUNCH(ctx, kernel, grid, block, smem, ...) ef_launch((ctx), kernel, dim3(grid), dim3(block), (smem), __VA_ARGS__)
// the next launch is a plain stream-ordered one: it starts only after everything enqueued before it has completed, so no
// kernel launched after it can become resident while earlier work is still running (a full barrier in the PDL chain)
#define EF_PLAIN_NEXT(ctx) ((ctx)->plain_next = true)
