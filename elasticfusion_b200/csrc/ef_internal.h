// Internal context layout of libefusion.so (not part of the ABI) and the host-side plumbing every translation unit shares:
// allocation, error macros, the launch helper and the entry points one .cu file calls in another.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <string.h>

#include <vector>

#include "../../include/efusion_b200.h"

namespace ef {

constexpr int NUM_PYRS = 3;          // RGBDOdometry::NUM_PYRS (reference Core/Utils/RGBDOdometry.h:114)
constexpr int RED_THREADS = 256;     // threads per reduction CTA
constexpr int MAX_RED_BLOCKS = 1184; // 8 resident 256-thread CTAs per SM on up to 148 SMs (H100: 132)
constexpr int PARTIAL_STRIDE = 64;   // floats per CTA partial: [0,29) geometric system, [32,61) photometric system
constexpr int MAX_TRACE = 48;
// tracker slots of EfContext::odom: 0 frameToModel, 1 modelToModel (both sized for the context's camera), the tracker of
// ef_track_view*, whose buffers are sized for the largest view so far, one per live EfCamera, sized for its camera, and the
// modelToModel tracker of each camera that closes loops (CAMERA_LOOP_TRACKER0 + the camera's index)
constexpr int VIEW_TRACKER = 2;
constexpr int CAMERA_TRACKER0 = 3;
constexpr int CAMERA_LOOP_TRACKER0 = CAMERA_TRACKER0 + EF_MAX_CAMERAS;
constexpr int NUM_TRACKERS = CAMERA_LOOP_TRACKER0 + EF_MAX_CAMERAS;
constexpr int DENSE_FACTOR = 20;  // ElasticFusion::denseEnough decimates the predicted image by 20 (ElasticFusion.cpp:258)

// ElasticFusion::denseEnough (ElasticFusion.cpp:256-268) from the number of lit samples of the decimated image
__host__ __device__ inline bool dense_enough_of(int lit, int rows, int cols) {
  return (float)lit / (float)((rows / DENSE_FACTOR) * (cols / DENSE_FACTOR)) > 0.75f;
}
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
  float rgbErrBuf[2];           // rgbError of the previous / current iteration (double-buffered across CTAs)
  float weighting;  // velocity weighting for fusion (ElasticFusion.cpp:369-383)
  long long dbg[40];  // phase timestamps (%globaltimer) of levels 0 and 1 when built with -DEF_PROFILE_PHASES
};

// What a tracker's GNState holds before its first call (RGBDOdometry ctor, RGBDOdometry.cpp:22-117): identity pose, whole-image
// counts, the level-0 intrinsics and K / K^-1 of every level. Written by alloc_odom on the host and, before every track view, on the
// device, so that a view's result never depends on an earlier call.
__host__ __device__ inline void gn_initial_state(GNState* g, int width, int height, float fx, float fy, float cx, float cy) {
  memset(g, 0, sizeof(*g));
  for (int k = 0; k < 16; ++k) g->T_wc[k] = (k % 5 == 0) ? 1.0 : 0.0;
  g->lastICPCount = g->lastRGBCount = g->lastSO3Count = (float)(width * height);
  g->fx = fx;
  g->fy = fy;
  g->cx = cx;
  g->cy = cy;
  for (int lv = 0; lv < NUM_PYRS; ++lv) {
    const int div = 1 << lv;  // CameraModel::operator()(level), reference Core/Cuda/types.cuh:92-95
    const double lfx = (double)(fx / div), lfy = (double)(fy / div), lcx = (double)(cx / div), lcy = (double)(cy / div);
    const double K[9] = {lfx, 0, lcx, 0, lfy, lcy, 0, 0, 1};
    const double ifx = 1.0 / lfx, ify = 1.0 / lfy;
    const double Ki[9] = {ifx, 0, -lcx * ifx, 0, ify, -lcy * ify, 0, 0, 1};
    for (int k = 0; k < 9; ++k) {
      g->Kd[lv][k] = K[k];
      g->Kinvd[lv][k] = Ki[k];
    }
  }
  g->break_level = -1;
  g->weighting = 1.0f;
}

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
// live in MapDev::loop_src / loop_dst / loop_times, sized from the frame (a closing camera's in LoopBuffers of its own)
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
  uint32_t* pending;      // capacity: lowest draw index that chose this surfel (0xffffffff idle; every fuse leaves it so)
  // z-buffers
  unsigned long long* zbuf;        // W*H: the raycast's (k_splat_scatter / k_splat_resolve)
  unsigned long long* index_keys;  // W*H: the index map's tagged keys (IndexMap in ef_map.cu)
  uint32_t* vis_list;        // surfels that reached the z-buffer in the frame's first index-map pass (k_index_scatter<1>)
  int* vis_count;
  unsigned int* clean_ctl;   // [0] tile dispenser, [1] exit tickets, [2] first tile that moves (k_clean_flags -> k_clean_move)
  uint32_t* keep_mask;       // one warp ballot per 32 surfels: the clean test's verdicts
  MapPose* pose;         // device
  MapPose* view_pose;    // device: the pose of ef_map_predict_view* and ef_map_fuse_view*, so that a view never touches the frame's `pose`
  int* dense_count;       // device: lit samples of the predicted image's decimation (dense_enough_of gives the flag)
  int* tick;              // device-resident tick
  float* nodes;           // deformation graph of the current frame, 16 floats per node
  LoopDev* loop;
  int loop_capacity;      // loop_constraint_capacity(cols, rows)
  double *loop_src, *loop_dst;  // loop_capacity x 3: vert_w_curr / vert_w_est of each constraint
  int* loop_times;              // loop_capacity: the INACTIVE view's time stamp of each constraint
  // close_loops = 2 only: the deformation graph sampled at the end of the last frame (Deformation::rawSampledNodes_w: xyz and
  // init time of every 5000th surfel, at most MAX_GRAPH_NODES - 1) and its node count (0 until a frame sampled more than 4)
  float4* graph;
  int* graph_n;
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

// Device buffers owned by one context (or one workspace), freed together. Every block has 256 bytes of slack.
struct Arena {
  std::vector<void*> blocks;
  template <typename T>
  cudaError_t alloc(T** p, size_t n) {
    void* q = nullptr;
    cudaError_t e = cudaMalloc(&q, n * sizeof(T) + 256);
    if (e != cudaSuccess) return e;
    blocks.push_back(q);
    *p = (T*)q;
    return cudaSuccess;
  }
  void release() {
    for (void* p : blocks) cudaFree(p);
    blocks.clear();
  }
};

// Layout of the pinned staging block (EfContext::pin_small): host values on their way to the device and results on their way
// back. A slot is rewritten only after a cudaStreamSynchronize, since a copy enqueued by the previous call may still read it.
struct PinStaging {
  float icp_inputs[36];  // ef_icp_step_async: Rcurr, tcurr, Rprev_inv, tprev, then M = R_prev^-1 R_curr, t' (9 + 3 each)
  double map_pose[16];   // map_update_pose_async: T_wc of a stage-API map call
  float weighting;       // map_fuse_async: fusion weighting of a stage-API fuse
  double T_wc[16];       // frame_begin_device: the caller's pose for a frame that is not tracked
  double finish_T_wc[16];  // ef_finish_frame: pose and surfel count read back
  int finish_count;
  int loop_record[3];              // loop_solve_apply: LoopDev::accepted, LoopDev::n_constraints, MapDev::graph_n
  EfDeformResult deform_result;    // loop_solve_apply: the deformation solve of the frame or a closing camera
  double view_pose[16];  // stage_view_pose: T_wc of a model or fuse view (rewritten after EfContext::view_pose_sent, not a sync)
  float view_weighting;  // stage_view_pose: fusion weighting of a fuse view (same guard)
};
// Layout of the device staging block (EfContext::dev_small): where the kernels read the pinned slots above.
struct DevStaging {
  double map_pose[16];
  double T_wc[16];
  double view_pose[16];
  float view_weighting;
};
static_assert(sizeof(PinStaging) <= 65536 && sizeof(DevStaging) <= 65536, "staging blocks stay within 64 KiB");

// Look-back tile states of order-preserving compactions (lookback_prefix) and their dispenser; each compaction takes a fresh epoch
struct ScanTiles {
  unsigned long long* state;
  unsigned int* counter;
  size_t bytes;
  unsigned int epoch;
};

// Host-side state of one index map, kept across calls
struct IndexState {
  int pass;          // index-map passes since the keys were last re-armed: the current pass's tag is 0xff - pass
  bool keys_only;    // the last index pass was a frame's: fuse and clean read its keys, the frame's clean writes its textures
  bool vis_pending;  // the first pass of a frame has filled the visible list and no clean has re-armed it yet
};

// What the map's write side -- preprocess, index map, fuse, clean -- works on besides the surfels: a camera, its inputs, its index
// map and the scratch sized by its pixels. The frame's (map_frame_target, rebuilt per call: the look-ahead swaps the input
// buffers) or a fuse view's (map_fuse_view_target).
struct MapTarget {
  int rows, cols;
  float cx, cy, fx, fy;
  const uint8_t* rgb;  // W*H*3
  float *depth_metric, *depth_metric_filtered;
  const float* synth_depth;  // read by the clean's time-stamp refresh under a deformation graph (the frame's or a closing camera's)
  MapPose* pose;
  float* weighting;          // device: fuse's confidence weighting
  // index map: tagged keys (key_texels of them, all re-armed when the tags run out) and the four textures
  unsigned long long* index_keys;
  size_t key_texels;
  uint32_t* index;
  float4 *vert_conf, *color_time, *norm_rad;
  IndexState* ix;
  // fuse: association per pixel and the unstable surfels it adds; clean: verdicts, control words and the kept count
  uint32_t* assoc_id;
  float4 *new_pos, *new_col, *new_nr;
  int* new_count;
  uint32_t* keep_mask;
  unsigned int* clean_ctl;
  int* clean_total;
  ScanTiles* scan;  // covers the clean's capacity + W*H surfels and fuse's W*H pixels
};

// What combinedPredict at a device pose record writes for a camera of its own (ef_camera_frame*): the model view (any output may be
// null), the lit samples of its decimation (null: not counted) and, fill_vertex given, the fill-in of predict() from the camera's
// filtered depth and RGB in the same pass (ElasticFusion.cpp:621-653)
struct PredictTarget {
  int rows, cols;
  float cx, cy, fx, fy;
  const MapPose* pose;
  uchar4* image;
  float4 *vertex, *normal;
  uint16_t* time;
  float* depth;                // given: the synthesised depth alone (synthesizeDepth), and none of the outputs above
  int* dense_count;
  const uint16_t* fill_depth;  // W*H filtered millimetres
  const uint8_t* fill_rgb;     // W*H*3
  int fill_pass_img;           // frameToFrameRGB: the fill-in image is the live RGB everywhere
  uchar4* fill_image;
  float4 *fill_vertex, *fill_normal;
};

// What the local loop closure of one camera works on (ElasticFusion.cpp:447-534): the frame's (tracker 0 and modelToModel tracker 1,
// MapDev's loop buffers, Textures' predictions) or a closing camera's (its tracker, its loop tracker and LoopBuffers)
struct LoopSide {
  int curr, est;             // tracker slots: the camera's (T_wc_curr) and its modelToModel tracker
  int rows, cols;
  float max_depth;
  bool pyramid, fast_odom;
  const float4 *vertex, *normal;  // the ACTIVE prediction of the mid-frame predict()
  const uchar4* image;
  const float4 *old_vertex, *old_normal;  // the INACTIVE prediction
  const uchar4* old_image;
  const uint16_t* old_time;
  LoopDev* loop;
  double *src, *dst;
  int* times;
  int capacity;
};

// A closing camera's buffers of the local loop closure, at its size (ef_camera_* with close_loops = 1)
struct LoopBuffers {
  uchar4* old_image;  // INACTIVE prediction at (0, time - time_delta, time_delta)
  float4 *old_vertex, *old_normal;
  uint16_t* old_time;
  float* synth_depth;  // the deformed clean's depth-only prediction
  LoopDev* loop;
  double *src, *dst;
  int* times;
  int capacity;
  ScanTiles scan;      // look-back tile states of the loop tracker's candidate compaction
};

// A rig's extrinsics on the device (ef_rig_*), written once at creation: T_0i (camera i -> member 0's camera), its inverse T_i0 and
// Ad(T_i0), the adjoint that maps member 0's increment to member i's in the reference's (t, w) order: [[R, [p]x R], [0, R]], row-major.
// res: each member's ICP residual sum and inlier count of the last iteration (res0, res1 of gn_gather), written by k_rig_update.
struct RigDev {
  double T_0i[EF_MAX_CAMERAS][16], T_i0[EF_MAX_CAMERAS][16];
  double Ad[EF_MAX_CAMERAS][36];
  float res[EF_MAX_CAMERAS][2];
};
// What the rig kernels (k_rig_seed, k_rig_update, k_rig_finish) work on: each member's tracker state, trace, per-level K / K^-1
// (OdomDev::K_levels) and map pose record (null: none), in member order
struct RigArgs {
  int n;
  GNState* gn[EF_MAX_CAMERAS];
  EfSolveTrace* trace[EF_MAX_CAMERAS];
  const double* K_levels[EF_MAX_CAMERAS];
  MapPose* pose[EF_MAX_CAMERAS];
  RigDev* dev;
};
// What a rig's joint SO(3) pre-alignment (k_rig_so3_begin, k_rig_so3_step) works on: each member's SO(3) state, the GNState whose
// level-2 K its homography uses, its level-2 image pair and size and its partials; member m's CTAs are [cta0[m], cta0[m + 1]). The
// extrinsics are the rig's; the ticket, the rig's own, replaces the members' so3_counter.
struct RigSo3Args {
  int n;
  So3State* so3[EF_MAX_CAMERAS];
  const GNState* gn[EF_MAX_CAMERAS];
  const uint8_t* last[EF_MAX_CAMERAS];
  const uint8_t* next[EF_MAX_CAMERAS];
  int rows[EF_MAX_CAMERAS], cols[EF_MAX_CAMERAS];
  float* partials[EF_MAX_CAMERAS];
  int cta0[EF_MAX_CAMERAS + 1];
  const RigDev* dev;
  unsigned int* ticket;
};

// A closing rig's record of its last front half besides its LoopDev: each member's constraint count and member 0's T_wc_curr
struct RigLoopDev {
  int member_n[EF_MAX_CAMERAS];
  double T_wc_curr[16];
};
// What k_rig_loop_constraints works on: each member's tracker (T_wc_curr) and loop tracker after the joint model-to-model
// registration (T_wc_est; member 0's lastA is the joint system), its ACTIVE prediction and INACTIVE time stamps at its size, the
// members' residuals (RigDev::res) and the rig's record and constraint buffers (capacity: the sum of the members' grids)
struct RigLoopArgs {
  int n;
  const GNState* curr[EF_MAX_CAMERAS];
  const GNState* est[EF_MAX_CAMERAS];
  const float4* vertex[EF_MAX_CAMERAS];
  const uint16_t* old_time[EF_MAX_CAMERAS];
  int rows[EF_MAX_CAMERAS], cols[EF_MAX_CAMERAS];
  float max_depth[EF_MAX_CAMERAS];
  const RigDev* dev;
  LoopDev* loop;
  RigLoopDev* rec;
  double *src, *dst;
  int* times;
  int capacity;
};

// The outcome of the last local closure of one side (the frame, or a closing camera)
struct DeformOutcome {
  bool solved, applied;
  EfDeformResult result;
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
  bool visible_list;      // second index-map pass of a frame visits only the surfels the first one rasterised; EF_VISIBLE_LIST=0 disables
  int gn_cluster;         // CTAs of the clusters that run the SO(3) loop and the coarse-level Gauss-Newton iterations (0: plain launches everywhere)
  int gn_cluster_levels;  // pyramid levels, from the coarsest, whose iterations run in that cluster
  bool la_after_track;    // the look-ahead's side stream starts after the frame's coarse-level cluster (EF_LA_AFTER_TRACK=0: at frame start)
  bool plain_next;     // the next ef_launch omits the programmatic-serialisation attribute (EF_PLAIN_NEXT)
  bool maps_dirty[ef::NUM_TRACKERS];  // a kernel that writes tracker w's pyramids may still be in flight ahead of the next stage launch
  ef::IndexState index;  // the frame's index map (MapDev::index_keys, Textures::index ...)

  ef::OdomDev odom[ef::NUM_TRACKERS];
  float odom_cam[ef::NUM_TRACKERS][4];  // level-0 {fx, fy, cx, cy} of tracker w: the host's copy of what its GNState holds
  ef::ScanTiles* odom_tiles[ef::NUM_TRACKERS];  // tile states of tracker w's candidate compaction (null: the context's own)
  EfCamera* cameras[EF_MAX_CAMERAS];           // live cameras, by tracker slot (CAMERA_TRACKER0 + i)
  EfRig* rigs[EF_MAX_CAMERAS];                 // live rigs (each holds at least one camera)
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
  // close_loops = 2: Deformation's bookkeeping (ElasticFusion::deforms, Deformation::lastDeformTime), shared with the closing cameras,
  // and the last frame's outcome
  int deforms, last_deform_time;
  ef::DeformOutcome deform_out;

  // pinned staging
  uint8_t* pin_rgb;
  uint16_t* pin_depth;
  ef::PinStaging* pin_small;  // per-call parameters and results read-back
  ef::DevStaging* dev_small;  // device side of the per-call parameters
  void* map_host;    // host-side bookkeeping of the surfel buffers (ef_map.cu)
  void* deform;      // workspace of the deformation-graph solve (ef_deform.cu), allocated by its first call
  void* render;      // z-buffer and output staging of ef_render_map* and ef_map_predict_view* (ef_render.cu), allocated by the first
                     // call and grown with the view
  void* fuse_view;   // input, index-map and scratch buffers of ef_map_fuse_view* (ef_map.cu), allocated by the first call and grown
                     // with the view
  void* track_view;  // inputs, prediction and tracker buffers (odom[VIEW_TRACKER]) of ef_track_view* (ef_track.cu), allocated by the
                     // first call and grown with the view
  cudaEvent_t view_pose_sent;  // ctx->stream: the last view's pose and weighting have been copied out of PinStaging
  ef::Arena arena;   // every device buffer of the context
};

// A camera of a context (ef_camera_*): its tracker slot, inputs, prediction, fill-in and map-write buffers, all at its own size
struct EfCamera {
  int slot;                // tracker slot in ctx->odom (CAMERA_TRACKER0 + its index in ctx->cameras)
  EfCameraConfig cfg;
  bool has_frame;          // a first frame has set its pose and previous intensity pyramid
  ef::Arena arena;         // every device buffer below and those of ctx->odom[slot]
  uint8_t *rgb, *rgba;     // its inputs (rgb and depth_raw are the map target's, which fuse reads)
  uint16_t *depth_raw, *depth_filtered;
  uchar4* image;           // predict(): the model its next frame tracks against, and the fill-in
  float4 *vertex, *normal;
  uint16_t* time;
  uchar4* fill_image;
  float4 *fill_vertex, *fill_normal;
  int* dense_count;        // lit samples of the prediction's decimation
  ef::ScanTiles scan;      // look-back tile states of its candidate compaction
  ef::MapPose* pose;       // its pose record, written by k_gn_finish
  ef::MapTarget target;    // its map-write side (pose record and tracker weighting set)
  void* target_state;      // map_camera_target's
  EfCameraResult* result;  // device: the result of its last frame (the host call reads it back)
  ef::LoopBuffers loop;    // close_loops = 1: its local loop closure (tracker slot loop_slot)
  int loop_slot;
  ef::DeformOutcome deform_out;  // close_loops = 1: its last frame's closure
  double* pin_T;           // pinned staging of a frame's has_pose T_wc, rewritten after pose_sent
  double* dev_T;
  cudaEvent_t pose_sent;
  EfRig* rig;              // the rig it is a member of (null: none); its own frames are refused meanwhile
};

// A rig of cameras tracked as one rigid body (ef_rig_*): its members in order (member 0's camera frame is the rig body), their
// extrinsics and the device block the rig kernels read
struct EfRig {
  int n;
  EfCamera* cams[EF_MAX_CAMERAS];
  double T_0i[EF_MAX_CAMERAS][16];  // row-major, camera i -> member 0's camera
  bool has_frame;                   // a first frame has set the rig's pose
  ef::Arena arena;                  // dev, result and a closing rig's loop buffers
  ef::RigDev* dev;
  EfRigResult* result;              // device: the rig result of its last frame (the host call reads it back)
  // every member has close_loops = 1: the rig closes local loops as one body (its members' loop trackers and LoopBuffers, and these)
  bool closing;
  ef::LoopDev* loop;
  ef::RigLoopDev* loop_rec;
  double *src, *dst;                // the members' constraints, concatenated in member order
  int* times;
  int capacity;                     // the sum of the members' loop_constraint_capacity
  ef::DeformOutcome deform_out;     // its last frame's closure
  // joint_so3: one SO(3) pre-alignment over every member's image pair instead of member 0's; the ticket of its reduction
  bool joint_so3;
  unsigned int* so3_ticket;
};

// error propagation of the host entry points: a CUDA error code, or the code of a failed internal call
#define CU(x)                                  \
  do {                                         \
    cudaError_t e__ = (x);                     \
    if (e__ != cudaSuccess) return (int)e__;   \
  } while (0)
#define RC(x)              \
  do {                     \
    int rc__ = (x);        \
    if (rc__) return rc__; \
  } while (0)
#define CHECK_LAST() CU(cudaGetLastError())

namespace ef {
// n elements of T from `arena`; fill >= 0: every byte set to `fill` on ctx->stream
template <typename T>
inline cudaError_t arena_alloc(EfContext* ctx, Arena& arena, T** p, size_t n, int fill = -1) {
  cudaError_t e = arena.alloc(p, n);
  if (e != cudaSuccess || fill < 0) return e;
  return cudaMemsetAsync(*p, fill, n * sizeof(T), ctx->stream);
}
// the same from the context's arena
template <typename T>
inline cudaError_t ctx_alloc(EfContext* ctx, T** p, size_t n, int fill = -1) {
  return arena_alloc(ctx, ctx->arena, p, n, fill);
}
}  // namespace ef

// launch bookkeeping
inline void ef_stage(EfContext* ctx, int i) {
  if (ctx->stage_timing) {
    cudaEventRecord(ctx->stage_ev[i], ctx->stream);
    if (i == 0) ctx->stage_n = 0;  // bit mask of the events recorded for this frame
    ctx->stage_n |= 1 << i;
  }
}
inline cudaLaunchAttribute cluster_attr(int cluster) {
  cudaLaunchAttribute a;
  a.id = cudaLaunchAttributeClusterDimension;
  a.val.clusterDim.x = cluster;
  a.val.clusterDim.y = 1;
  a.val.clusterDim.z = 1;
  return a;
}
// Every kernel is launched with programmatic stream serialisation allowed (see pdl_enter() in ef_device.cuh); set
// EF_NO_PDL=1 in the environment to fall back to plain stream-ordered launches (A/B measurements).
// cluster > 0: the grid runs as thread-block clusters of that many CTAs.
template <typename... KArgs, typename... Args>
inline void ef_launch(EfContext* ctx, void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, int cluster, Args&&... args) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = ctx->stream;
  cudaLaunchAttribute attr[2];
  int n = 0;
  if (cluster > 0) attr[n++] = cluster_attr(cluster);
  if (ctx->pdl && !ctx->plain_next) {
    attr[n].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[n++].val.programmaticStreamSerializationAllowed = 1;
  }
  cfg.attrs = attr;
  cfg.numAttrs = n;
  ctx->plain_next = false;
  cudaLaunchKernelEx(&cfg, kernel, static_cast<KArgs>(args)...);
  ctx->launches++;
}
#define EF_LAUNCH(ctx, kernel, grid, block, smem, ...) ef_launch((ctx), kernel, dim3(grid), dim3(block), (smem), 0, __VA_ARGS__)
// the next launch is a plain stream-ordered one: it starts only after everything enqueued before it has completed, so no
// kernel launched after it can become resident while earlier work is still running (a full barrier in the PDL chain)
#define EF_PLAIN_NEXT(ctx) ((ctx)->plain_next = true)

// grid of a grid-stride kernel over n items: ceil(n / threads) CTAs, at least one, at most one wave of per_sm per SM
inline int wave_blocks(const EfContext* ctx, size_t n, int per_sm = 8, int threads = 256) {
  size_t b = (n + threads - 1) / threads, cap = (size_t)ctx->num_sms * per_sm;
  return (int)(b < cap ? (b ? b : 1) : cap);
}

// ---- host entry points one translation unit calls in another; default arguments live here only -------------------
namespace ef {
// ef_api.cu: the buffers and initial state of tracker slot `which` (RGBDOdometry's constructor) for a width x height camera, from
// `arena`; synchronises ctx->stream
int alloc_odom(EfContext* ctx, Arena& arena, int which, int width, int height, float fx, float fy, float cx, float cy);

// ef_api.cu: the local loop closure of one side. loop_front_half: the front half after its INACTIVE prediction (ElasticFusion.cpp:
// 457-505); loop_solve_apply: the read-back, solve and hand-over (:505-526) at `time`, the pose going to tracker s.curr and pose_record;
// *n_nodes: the graph the clean applies (0: none)
int loop_front_half(EfContext* ctx, const LoopSide& s);
// its first steps: tracker s.est at the pose of s.curr with the INACTIVE prediction as its model and the ACTIVE one as its input
int loop_tracker_inputs(EfContext* ctx, const LoopSide& s);
int loop_solve_apply(EfContext* ctx, const LoopSide& s, int time, MapPose* pose_record, DeformOutcome* out, int* n_nodes);

// ef_track.cu: the tracker's input pyramids
int odom_init_icp_depth(EfContext* ctx, int which, const uint16_t* depth_dev, float cutoff);
int odom_init_icp_pred(EfContext* ctx, int which, const float* vtx4, const float* nrm4);
int odom_init_icp_model(EfContext* ctx, int which, const float* vtx4, const float* nrm4, bool with_global = true);
int odom_populate(EfContext* ctx, int which, const uint8_t* rgba, float** destDepths, uint8_t** destImages, bool with_depth,
                  bool with_image = true);
int map_select_model_inputs(EfContext* ctx);
int launch_sobel(EfContext* ctx, int which);
// ef_track_view* (include/efusion_b200.h): host inputs when from_host (then out_dev may be null), device inputs otherwise; the
// result packed into out_dev when given. The view tracker's state stays on the device for the host call to read.
int track_view_async(EfContext* ctx, const EfTrackView* v, const uint8_t* rgb, const uint16_t* depth, bool from_host, EfTrackResult* out_dev);
// the view tracker's GNState and the view's dense-sample count into host memory (synchronises)
int track_view_read(EfContext* ctx, GNState* g, int* lit);
void track_view_free(EfContext* ctx);
// ef_camera_* (include/efusion_b200.h): a camera's buffers and tracker slot (EF_ENOMEM / EF_ESTATE as the ABI says); one camera frame
// (host inputs when from_host, the result into out_dev when given, else into the camera's own result); that own result and the trace
// of its last frame (synchronises); and its release
int camera_create(EfContext* ctx, const EfCameraConfig* cfg, EfCamera** out);
int camera_frame_async(EfContext* ctx, EfCamera* cam, const EfCameraFrame* f, const uint8_t* rgb, const uint16_t* depth, bool from_host,
                       EfCameraResult* out_dev);
int camera_read(EfContext* ctx, EfCamera* cam, EfCameraResult* out, EfSolveTrace* trace, int max_trace, int* n_trace);
void camera_destroy(EfContext* ctx, EfCamera* cam);
// ef_rig_* (include/efusion_b200.h), arguments checked by the caller: a rig of existing cameras, one rig frame (host inputs when
// from_host; results into members_dev / out_dev when given, else into the members' and the rig's own), those own results and the
// members' traces of its last frame (synchronises), and its release (the members stay)
int rig_create(EfContext* ctx, const EfRigConfig* cfg, EfRig** out);
int rig_frame_async(EfContext* ctx, EfRig* rig, const EfRigFrame* f, const uint8_t* const* rgb, const uint16_t* const* depth, bool from_host,
                    EfCameraResult* members_dev, EfRigResult* out_dev);
int rig_read(EfContext* ctx, EfRig* rig, EfCameraResult* members, EfRigResult* out, EfSolveTrace* trace, int max_trace, int* n_trace);
void rig_destroy(EfContext* ctx, EfRig* rig);

// ef_reduce.cu: SO(3) loop, Gauss-Newton schedule and the stage API's reductions
int odom_cluster_size(int want);
int odom_so3_async(EfContext* ctx, int which);
int odom_track_async(EfContext* ctx, int which, bool rgbOnly, float icpWeight, bool pyramid, bool fastOdom, bool so3);
// pose_record: the map pose record the finished pose is written to as well (null: none)
int odom_finish_async(EfContext* ctx, int which, float weightMultiplier, bool have_track, MapPose* pose_record);
int odom_set_pose_async(EfContext* ctx, int which, const double* T_dev);
int launch_se3_step_raw(EfContext* ctx, int which, int level, bool do_icp, bool do_rgb, float sigma);
int launch_rgb_residual_raw(EfContext* ctx, int which, int level);
int launch_icp_dense_only(EfContext* ctx, int which, int level);
int launch_so3_raw(EfContext* ctx, int which);

// ef_reduce.cu: a rig's joint Gauss-Newton loop over the trackers slots[0..R.n) (ef_rig_frame*; every member's model inputs, and initRGB's
// depth half, in place), and its finish with the weighting times weightMultiplier into each member's pose record. so3_ticket (the
// rig's, zero between launches): the SO(3) pre-alignment is the joint one over every member (null: member 0's)
int rig_track_async(EfContext* ctx, const int* slots, const RigArgs& R, float icpWeight, bool pyramid, bool fastOdom, bool so3,
                    unsigned int* so3_ticket);
int rig_finish_async(EfContext* ctx, const RigArgs& R, float weightMultiplier);
// after a closure set member 0's pose: member i's T_wc = T_w0 * T_0i in double, and its pose record
int rig_apply_pose_async(EfContext* ctx, const RigArgs& R);

// ef_preprocess.cu: filtered / metric / metric_filtered may be null
int preprocess_depth(EfContext* ctx, int rows, int cols, const uint16_t* raw, float cutoff, uint16_t* filtered, float* metric,
                     float* metric_filtered);
int rgb_to_rgba(EfContext* ctx, int rows, int cols, const uint8_t* rgb, uint8_t* rgba);

// ef_map.cu: the surfel map
int alloc_map(EfContext* ctx);
void map_free_host(EfContext* ctx);
// look-back tile states, tile dispenser and a fresh epoch for one order-preserving compaction on ctx->stream (lookback_prefix)
struct ScanSlot {
  unsigned long long* state;
  unsigned int* counter;
  unsigned int epoch;
};
int scan_slot(EfContext* ctx, ScanSlot* out);
// the same from a buffer set's own tile states
int scan_slot(EfContext* ctx, ScanTiles& tiles, ScanSlot* out);
int map_initialise_async(EfContext* ctx);
int map_update_pose_async(EfContext* ctx, const double* T_host_or_null);
// the frame's camera, inputs and buffers as they are now
MapTarget map_frame_target(EfContext* ctx);
// a fuse view's buffers, grown to the view (EF_ENOMEM if they cannot be: the context stays usable), with its pose and weighting
// staged and uploaded to MapDev::view_pose; rgb / depth_raw: where its inputs may be uploaded (W*H*3, W*H)
int map_fuse_view_target(EfContext* ctx, const EfFuseView* view, MapTarget* out, uint8_t** rgb, uint16_t** depth_raw);
// a camera's own map-write buffers, as a fuse view's of its size, from `arena` (ef_camera_*): its inputs, index map and scratch. pose and
// weighting are left to the caller; *state keeps the index state and tile states the target points to (map_camera_target_free)
int map_camera_target(EfContext* ctx, Arena& arena, int rows, int cols, float fx, float fy, float cx, float cy, void** state, MapTarget* out,
                      uint8_t** rgb, uint16_t** depth_raw);
void map_camera_target_free(void* state);
int map_predict_indices_async(EfContext* ctx, const MapTarget& t, int time, float max_depth, int time_delta, int vis_mode = 0);
// the textures of a frame's index pass that no clean has written yet (nothing to do otherwise)
int map_index_textures_async(EfContext* ctx, const MapTarget& t);
// weighting < 0: the one *t.weighting already holds
int map_fuse_async(EfContext* ctx, const MapTarget& t, int time, float max_depth, float weighting_or_neg);
int map_clean_async(EfContext* ctx, const MapTarget& t, int time, float conf_threshold, int time_delta, float max_depth, int n_nodes = 0,
                    bool is_fern = false);
int map_set_graph(EfContext* ctx, const float* nodes16, int n_nodes);
int map_set_graph_device(EfContext* ctx, const float* nodes16_dev, int n_nodes);
int map_sample_graph_async(EfContext* ctx);
// mode 0 also recounts dense_count; fill_in >= 0 (mode 0 only) also runs the fill-in in the same pass, with pass_img = fill_in
int map_raycast_async(EfContext* ctx, float max_depth, float conf_threshold, int time, int max_time, int time_delta, int mode, int fill_in = -1);
int map_fill_in_async(EfContext* ctx, bool passthrough_geometry, bool passthrough_image);
// combinedPredict at the view's pose, camera and size into the given device outputs (any may be null); touches no frame state.
// dense_count: where the lit samples of the predicted image's decimation are counted (null: not counted)
int map_predict_view_async(EfContext* ctx, const EfModelView* view, uint8_t* image4, float* vertex4, float* normal4, uint16_t* time,
                           int* dense_count = nullptr);
// the same at t.pose (device), writing t's outputs, dense count and fill-in
int map_predict_target_async(EfContext* ctx, const PredictTarget& t, float max_depth, float conf_threshold, int time, int max_time, int time_delta);
int map_dense_enough_async(EfContext* ctx);
// the acceptance test and the constraints of side s's front half, with the context's thresholds
int map_loop_constraints_async(EfContext* ctx, const LoopSide& s);
// the same for a closing rig: one joint acceptance test and every member's grid, concatenated in member order
int map_rig_loop_constraints_async(EfContext* ctx, const RigLoopArgs& a);
int map_loop_reset_async(EfContext* ctx, LoopDev* loop);
// the map kernels' pose record `mp` from a device T_wc
int map_pose_record_async(EfContext* ctx, MapPose* mp, const double* T_dev);
int odom_copy_pose_async(EfContext* ctx, int dst, int src);
int map_download(EfContext* ctx, const float4* a, const float4* b, const float4* c, int n, float* out);
int map_upload(EfContext* ctx, const float* in, int n);
int map_upload_range(EfContext* ctx, const float* in, int first, int n);
int map_resize_to_host(EfContext* ctx, const void* src_dev, int elem, int factor, void* host_out);
void map_fuse_view_free(EfContext* ctx);

// ef_deform.cu: the deformation-graph solve
int deform_solve(EfContext* ctx, const double* node_pos3, const int32_t* node_times, int n, const double* src3, const double* dst3,
                 const int32_t* src_times, int m, int last_deform_time, float* nodes16_host, double* rt12_host,
                 int32_t* cons_nodes4, double* cons_weights4, EfDeformResult* out);
int deform_solve_local(EfContext* ctx, const float4* graph, int n, const double* src3, const double* dst3, const int* dst_times, int n_cons,
                       bool pin, int src_time, int last_deform_time, EfDeformResult* out, const float** nodes16_dev);
void deform_free(EfContext* ctx);

// ef_render.cu: the global-surface render, and the buffers of every pass outside the frame (the render and the model view), grown
// to the largest view and freed by render_free
int render_map_async(EfContext* ctx, const EfRenderView* view, uint8_t* rgba_dev);
// n z-buffer keys, all kEmptyKey (~0) between passes: each pass's resolve re-arms the pixels its scatter may have written
int offframe_zbuf(EfContext* ctx, size_t n, unsigned long long** out);
// device staging of at least `bytes` (256-byte aligned) for a call that returns its outputs to the host
int offframe_staging(EfContext* ctx, size_t bytes, uint8_t** out);
void render_free(EfContext* ctx);
}  // namespace ef
