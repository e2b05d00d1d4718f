/* efusion_b200.h — C ABI of libefusion.so, the H100-native (sm_90a) implementation of ElasticFusion's per-frame
 * tracking + surfel fuse/predict hot path.
 *
 * This is the drop-in boundary (SURVEY.md §8b): plain pointers and sizes, no C++/torch types. Each entry point
 * names the reference interface it replaces (paths relative to the reference tree). The C++ classes in
 * include/efusion/ (ElasticFusion, RGBDOdometry, GlobalModel, IndexMap) are thin wrappers over these calls.
 *
 * Conventions
 *  - every function returns 0 on success, a cudaError_t value (>0) on a CUDA failure, or a negative EF_E* code.
 *    (The reference prints and exit(0)s on CUDA errors, Core/Cuda/convenience.cuh:64-70; the C++ wrappers keep
 *    that policy, the C ABI reports instead.)
 *  - one EfContext == one device + one CUDA stream; contexts on different devices may be driven from different
 *    host threads concurrently. Host buffers are borrowed only for the duration of a call.
 *  - poses are row-major double[16] camera-to-world (Sophus::SE3d::matrix()); 3x3 matrices row-major float[9].
 *  - all device work is asynchronous on the context's stream; calls that return results to host memory
 *    synchronise that stream before returning.
 */
#ifndef EFUSION_B200_H_
#define EFUSION_B200_H_
#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define EF_OK 0
#define EF_EINVAL (-1)
#define EF_ENOMEM (-2)
#define EF_ESTATE (-3)

typedef struct EfContext EfContext;

/* Constructor arguments of ElasticFusion (Core/ElasticFusion.h:42-58) plus what the reference keeps in the
 * Resolution / Intrinsics singletons (Core/Utils/Resolution.h, Intrinsics.h) and a runtime surfel capacity
 * (the reference hard-codes 3072^2, Core/GlobalModel.cpp:22-24). */
typedef struct {
  int32_t width, height;
  float fx, fy, cx, cy;
  int32_t time_delta;     /* 200 */
  int32_t count_thresh;   /* 35000  (loop closure only; kept for API parity) */
  float err_thresh;       /* 5e-05  (loop closure only) */
  float cov_thresh;       /* 1e-05  (loop closure only) */
  int32_t close_loops;    /* 0: open loop. 1: run the local loop closure front half every frame (results: ef_local_loop_result);
                             the deformation solve stays with the host (ef_process_frame_begin / _end). 2: close local loops
                             inside the frame as well -- sample, solve and apply the deformation graph (ef_local_deform_result).
                             Other values: EF_EINVAL. Ferns stay outside this library (SURVEY.md §8) */
  int32_t iclnuim;
  int32_t reloc;          /* must be 0 */
  float photo_thresh;     /* 115 (ferns only) */
  float confidence;       /* 10 */
  float depth_cutoff;     /* 3 */
  float icp_weight;       /* 10 */
  int32_t fast_odom;      /* 0 */
  float fern_thresh;      /* 0.3095 (ferns only) */
  int32_t so3;            /* 1 */
  int32_t frame_to_frame_rgb; /* 0 */
  int32_t capacity;       /* max surfels resident in HBM (48 B each) */
  int32_t device;         /* CUDA device ordinal */
  int32_t skip_mid_predict; /* 1: skip the predict() at Core/ElasticFusion.cpp:387 whose outputs only loop closure reads */
} EfConfig;

void ef_default_config(EfConfig* cfg, int width, int height, float fx, float fy, float cx, float cy);

/* ElasticFusion::ElasticFusion / ~ElasticFusion (Core/ElasticFusion.cpp:22-163). `stream` is a cudaStream_t
 * (NULL: the context creates its own non-blocking stream). */
int ef_create(const EfConfig* cfg, void* stream, EfContext** out);
int ef_destroy(EfContext* ctx);
void* ef_stream(EfContext* ctx);
const char* ef_error_string(int code);

/* ---- whole frame: ElasticFusion::processFrame (Core/ElasticFusion.cpp:270-607) ------------------------------- */
/* rgb: uint8 RGB row-major W*H*3, depth: uint16 millimetres W*H (HOST memory, consumed before return);
 * in_T_wc may be NULL (track) or a pose to use instead of tracking. Returns after get_T_wc-observable state is final. */
int ef_process_frame(EfContext* ctx, const uint8_t* rgb, const uint16_t* depth, int64_t timestamp,
                     float weight_multiplier, const double* in_T_wc);
/* same with inputs already resident in HBM; fully asynchronous (no host sync) — call ef_sync before reading results. Except
 * with cfg.close_loops = 2: then the host reads a 12-byte record once the loop closure front half has run, and on a frame that
 * solves a deformation graph it also waits for the solve (see ef_local_deform_result) */
int ef_process_frame_device(EfContext* ctx, const uint8_t* rgb_dev, const uint16_t* depth_dev, int64_t timestamp,
                            float weight_multiplier, const double* in_T_wc);
int ef_sync(EfContext* ctx);
/* Frame look-ahead (no reference counterpart: the reference uploads and filters a frame inside processFrame, each GL
 * pass followed by glFinish — Core/ElasticFusion.cpp:278-285). Everything of the NEXT frame that depends neither on the
 * map nor on the pose (upload, RGBA expansion, bilateral filter + metric depth, depth pyramid + vertex/normal maps,
 * intensity pyramid) is enqueued on a side stream into a spare buffer set, so it overlaps the Gauss-Newton loop and the
 * map update of the frame in flight. One frame may be pending; it is consumed by passing rgb = depth = NULL to
 * ef_process_frame / ef_process_frame_device (EF_ESTATE if none is pending, or if a frame is passed while one is).
 * Results are identical to the non-prefetched call. Typical loop:
 *   ef_prefetch_frame(f0); for (i...) { ef_process_frame_device(NULL, NULL, ts[i], ...); ef_prefetch_frame(f[i+1]);
 *   ef_finish_frame(); }                                                                                          */
int ef_prefetch_frame(EfContext* ctx, const uint8_t* rgb, const uint16_t* depth);                /* HOST buffers   */
int ef_prefetch_frame_device(EfContext* ctx, const uint8_t* rgb_dev, const uint16_t* depth_dev); /* DEVICE buffers */
/* orders the main stream after the side stream's staged frame (so an event recorded on ef_stream() afterwards covers the
 * look-ahead work too); no-op when nothing is staged */
int ef_join_lookahead(EfContext* ctx);
/* waits for the frame enqueued by ef_process_frame_device and refreshes the host mirrors (pose, surfel count) */
int ef_finish_frame(EfContext* ctx);
/* processFrame split where the reference hands control to its CPU deformation solver (Core/ElasticFusion.cpp:505-526).
 * ef_process_frame_begin: upload, filter, track, velocity weighting, mid-frame predict and -- with cfg.close_loops -- the local
 * loop closure FRONT HALF (:447-505: INACTIVE prediction, modelToModel registration, acceptance test, constraint sampling);
 * results are final on return. ef_process_frame_end: optional pose override (T_wc_curr = T_wc_est, :524) and deformation graph
 * (16 floats per node: position 3, rotation 9 column-major, translation 3, time -- Core/Deformation.cpp:175-189) applied inside
 * clean (Core/Shaders/copy_unstable.vert:132-322), then index map / fuse / index map / clean / predict, tick++.
 * ef_process_frame == begin + end(NULL, NULL, 0, 0). EF_ESTATE if the calls are not paired, and with cfg.close_loops = 2, which
 * runs the solve inside ef_process_frame. */
int ef_process_frame_begin(EfContext* ctx, const uint8_t* rgb, const uint16_t* depth, int64_t timestamp, float weight_multiplier,
                           const double* in_T_wc);
int ef_process_frame_end(EfContext* ctx, const double* T_wc_override, const float* graph_nodes16, int32_t n_nodes,
                         int32_t fern_accepted);
/* result of the last frame's local loop closure front half (cfg.close_loops = 1); src3 / dst3: vert_w_curr / vert_w_est of
 * each constraint (what localDeformation.addConstraint receives, ElasticFusion.cpp:493-503), times: the INACTIVE view's stamp */
typedef struct {
  int32_t ran;            /* 0: first frame, rgbOnly, or close_loops off */
  int32_t accepted;       /* covariance diagonal <= cov_thresh && lastICPCount > count_thresh && lastICPError < err_thresh */
  int32_t n_constraints;
  float lastICPError, lastICPCount;
  double cov_diag[6];
  double T_wc_est[16];
} EfLoopResult;
int ef_local_loop_result(EfContext* ctx, EfLoopResult* out, double* src3, double* dst3, int32_t* times, int32_t max_constraints,
                         int32_t* n_out);
/* Embedded-deformation solve of a local loop closure: Deformation::constrain with fernMatch = relaxGraph = false
 * (Core/Deformation.cpp:73-207, Core/Utils/DeformationGraph.cpp). HOST inputs: the graph (node positions x3 and times, in
 * non-decreasing time order, 5 <= n_nodes < 1024, R = I and t = 0 at the start) and the constraints (src3 = vert_w_curr at
 * src_times, dst3 = vert_w_est at dst_times). pin != 0 adds the pin constraint (target, target, dst_time, dst_time) after each
 * one, as the reference does while it has not deformed yet (Core/Deformation.cpp:73-86). Nodes with time <= last_deform_time
 * are held fixed. Constraint weighting, at most 3 Gauss-Newton iterations on the normal equations (fp64, block-band
 * Cholesky) and the hand-over run in one launch on the device. Outputs (HOST, any may be NULL except out): nodes16, 16
 * floats per node as ef_process_frame_end takes them; rt12, the fp64 rotation (column-major) and translation of each node
 * (12 doubles per node); cons_nodes4 / cons_weights4, the 4 nodes (ascending id) and weights
 * of each expanded constraint. Results are deterministic: two calls on the same inputs are bit-identical. */
typedef struct {
  int32_t n_nodes, n_enabled, n_constraints;  /* n_constraints counts pin constraints too */
  int32_t iterations;  /* Gauss-Newton iterations run (1..3) */
  int32_t stop;        /* rule that ended the loop (DeformationGraph.cpp:473): 0 none (3 iterations), 1 error > lastError,
                          2 |delta| < 1e-2, 3 error < 1e-3, 4 |errorDiff| < 1e-5 error; 5: the normal equations were not
                          positive definite and the last delta was not applied (the reference would apply CHOLMOD's output);
                          6: two coupled nodes lie more than 19 apart, so the band cannot hold the system and nothing was
                          solved (the 20-node weighting window rules this out) */
  int32_t bandwidth;   /* largest distance between two coupled enabled nodes (<= 19; 20 with stop 6) */
  float error;         /* final squared residual norm */
  float meanConsErr;   /* nonRelativeConstraintError after the solve */
} EfDeformResult;
int ef_deform_solve(EfContext* ctx, const double* node_pos3, const int32_t* node_times, int32_t n_nodes, const double* src3,
                    const double* dst3, const int32_t* src_times, const int32_t* dst_times, int32_t n_constraints, int32_t pin,
                    int32_t last_deform_time, float* nodes16, double* rt12, int32_t* cons_nodes4, double* cons_weights4,
                    EfDeformResult* out);
/* cfg.close_loops = 2: the local loop closure closed inside ef_process_frame / ef_process_frame_device (Core/ElasticFusion.cpp:
 * 447-534 and 593 without ferns, Core/Deformation.cpp). After each frame the graph is sampled from the map: position and init time
 * of surfels 0, 5000, 10000, ... (sample.geom), at most 1023 nodes (the reference keeps 1024: maps of more than 5 110 000 surfels
 * get one node fewer), kept from the previous frame when 4 or fewer come out. When the front half of a later frame accepts, has at
 * least one constraint and a graph exists, the graph is solved as ef_deform_solve solves it (pin = (deforms == 0), constraint
 * source time = the frame's tick, last_deform_time) and, unless the solve stopped with code 6, applied: T_wc = T_wc_est and the
 * nodes go to the frame's clean, as ef_process_frame_end(T_wc_est, nodes) does; then deforms += 1, last_deform_time = tick. */
typedef struct {
  int32_t solved;            /* the last frame ran the solve */
  int32_t applied;           /* ... and applied its graph and pose */
  EfDeformResult result;     /* that solve's result; all zero when !solved */
  int32_t deforms;           /* closures applied since ef_create (ElasticFusion::getDeforms), a closing camera's included */
  int32_t last_deform_time;  /* tick (a closing camera's: time) of the last applied closure (Deformation::lastDeformTime); 0 before
                                the first */
  int32_t n_nodes;           /* nodes of the current graph (0: none sampled yet) */
} EfLocalDeform;
/* nodes4 (HOST, may be NULL when max_nodes = 0): the current graph, x y z and time per node (Deformation::rawSampledNodes_w);
 * n_out: how many were written. EF_ESTATE unless cfg.close_loops = 2. */
int ef_local_deform_result(EfContext* ctx, EfLocalDeform* out, float* nodes4, int32_t max_nodes, int32_t* n_out);
/* ElasticFusion::predict (Core/ElasticFusion.cpp:621-653) */
int ef_predict(EfContext* ctx);

/* getters/setters of ElasticFusion (Core/ElasticFusion.h:120-213) */
int ef_get_pose(EfContext* ctx, double* T_wc16);             /* get_T_wc */
int ef_set_pose(EfContext* ctx, const double* T_wc16);
int ef_get_tick(EfContext* ctx, int32_t* tick);              /* getTick */
int ef_set_tick(EfContext* ctx, int32_t tick);               /* setTick */
int ef_set_rgb_only(EfContext* ctx, int32_t v);              /* setRgbOnly */
int ef_set_icp_weight(EfContext* ctx, float v);              /* setIcpWeight */
int ef_set_pyramid(EfContext* ctx, int32_t v);               /* setPyramid */
int ef_set_fast_odom(EfContext* ctx, int32_t v);             /* setFastOdom */
int ef_set_so3(EfContext* ctx, int32_t v);                   /* setSo3 */
int ef_set_frame_to_frame_rgb(EfContext* ctx, int32_t v);    /* setFrameToFrameRGB */
int ef_set_confidence_threshold(EfContext* ctx, float v);    /* setConfidenceThreshold */
int ef_set_depth_cutoff(EfContext* ctx, float v);            /* setDepthCutoff */

/* ---- tracker: RGBDOdometry (Core/Utils/RGBDOdometry.h:31-79) and the free functions of
 *      Core/Cuda/cudafuncs.cuh:61-169 it drives -------------------------------------------------------------- */
typedef struct {
  int32_t kind;  /* 0 SE3 Gauss-Newton iteration, 1 SO3 pre-alignment iteration */
  int32_t level, iter;
  int32_t rgb_count, rgb_sigma;
  float sigma_val;
  float A_icp[36], b_icp[6], icp_residual[2];
  float A_rgb[36], b_rgb[6];
  float A_so3[9], b_so3[3], so3_residual[2];
  double lastA[36], lastb[6], result[6];
} EfSolveTrace;

/* public result fields of RGBDOdometry (RGBDOdometry.h:71-79) */
typedef struct {
  float lastICPError, lastICPCount, lastRGBError, lastRGBCount, lastSO3Error, lastSO3Count;
  double lastA[36], lastb[6];
} EfOdomStats;

/* which tracker instance: 0 = frameToModel (the only one driven by ef_process_frame), 1 = modelToModel */
/* RGBDOdometry::initICP(GPUTexture* filteredDepth, depthCutoff) — RGBDOdometry.cpp:121-147. depth: DEVICE u16 */
int ef_odom_init_icp_depth(EfContext* ctx, int which, const uint16_t* depth_dev, float depth_cutoff);
/* RGBDOdometry::initICP(predictedVertices, predictedNormals) — RGBDOdometry.cpp:149-169. DEVICE float4 maps */
int ef_odom_init_icp_pred(EfContext* ctx, int which, const float* vtx4_dev, const float* nrm4_dev);
/* RGBDOdometry::initICPModel — RGBDOdometry.cpp:171-210 */
int ef_odom_init_icp_model(EfContext* ctx, int which, const float* vtx4_dev, const float* nrm4_dev,
                           const double* T_wc16);
/* RGBDOdometry::initRGB / initRGBModel / initFirstRGB — RGBDOdometry.cpp:212-257. DEVICE RGBA8 image */
int ef_odom_init_rgb(EfContext* ctx, int which, const uint8_t* rgba_dev);
int ef_odom_init_rgb_model(EfContext* ctx, int which, const uint8_t* rgba_dev);
int ef_odom_init_first_rgb(EfContext* ctx, int which, const uint8_t* rgba_dev);
/* RGBDOdometry::getIncrementalTransformation — RGBDOdometry.cpp:259-571. The whole SO3 + 3-level Gauss-Newton loop
 * runs on the device with no host round trip; trace (HOST, may be NULL) receives one record per iteration. */
int ef_odom_track(EfContext* ctx, int which, double* T_wc16, int32_t rgb_only, float icp_weight, int32_t pyramid,
                  int32_t fast_odom, int32_t so3, EfSolveTrace* trace, int32_t max_trace, int32_t* n_trace);
int ef_odom_stats(EfContext* ctx, int which, EfOdomStats* out);
/* RGBDOdometry::getCovariance — RGBDOdometry.cpp:573-575 */
int ef_odom_covariance(EfContext* ctx, int which, double* cov36);

/* single reduction steps on the tracker's current pyramids, with explicit poses and HOST results, exactly the
 * argument meaning of the reference's free functions (used by the parity tests and the roofline bench):
 * icpStep (Core/Cuda/reduce.cu:333-401), computeRgbResidual (:723-787), rgbStep (:502-550), so3Step (:919-973) */
int ef_icp_step(EfContext* ctx, int which, int level, const float* Rcurr9, const float* tcurr3,
                const float* Rprev_inv9, const float* tprev3, float* A36, float* b6, float* residual2);
int ef_rgb_residual(EfContext* ctx, int which, int level, const float* krkinv9, const float* kt3,
                    int32_t* sigma_sum, int32_t* count);
int ef_rgb_step(EfContext* ctx, int which, int level, float sigma, float* A36, float* b6);
int ef_so3_step(EfContext* ctx, int which, const float* image_basis9, const float* kinv9, const float* krlr9,
                float* A9, float* b3, float* residual2);
/* asynchronous variant for benchmarking the ICP reduction: result stays on the device. Poses may be NULL (reuse the last ones).
 * ef_icp_dense_pass_async launches only the dense residual+Jacobian+per-CTA reduction kernel (k_iter1), without the 1-CTA
 * final sum — the launch bench.py's roofline object times. */
int ef_icp_step_async(EfContext* ctx, int which, int level, const float* Rcurr9, const float* tcurr3,
                      const float* Rprev_inv9, const float* tprev3);
int ef_icp_dense_pass_async(EfContext* ctx, int which, int level);

/* ---- depth preprocess: ElasticFusion::filterDepth + metriciseDepth (Core/ElasticFusion.cpp:655-673,
 *      Core/Shaders/depth_bilateral.frag, depth_metric.frag). DEVICE in/out, any out may be NULL ------------- */
int ef_preprocess_depth(EfContext* ctx, const uint16_t* depth_raw_dev, float depth_cutoff, uint16_t* filtered_dev,
                        float* metric_dev, float* metric_filtered_dev);

/* ---- surfel map: GlobalModel (Core/GlobalModel.h:34-89), IndexMap (Core/IndexMap.h:33-142),
 *      FillIn (Core/Shaders/FillIn.h), Resize (Core/Shaders/Resize.h) -------------------------------------- */
/* GlobalModel::initialise + FeedbackBuffer::compute (GlobalModel.cpp:229-284, FeedbackBuffer.cpp:81-138): builds the
 * first-frame map from the context's current RGB / metric depth textures */
int ef_map_initialise(EfContext* ctx);
/* IndexMap::predictIndices — IndexMap.cpp:190-258 */
int ef_map_predict_indices(EfContext* ctx, const double* T_wc16, int32_t time, float max_depth, int32_t time_delta);
/* GlobalModel::fuse — GlobalModel.cpp:356-525 (uses the context's RGB, metric depth and index-map textures) */
int ef_map_fuse(EfContext* ctx, const double* T_wc16, int32_t time, float max_depth, float weighting);
/* GlobalModel::clean — GlobalModel.cpp:527-671 (no deformation graph) */
int ef_map_clean(EfContext* ctx, const double* T_wc16, int32_t time, float conf_threshold, int32_t time_delta,
                 float max_depth);
/* GlobalModel::clean with a deformation graph (GlobalModel.cpp:527-671, graph.size() > 0; copy_unstable.vert:132-322); the
 * time-stamp refresh reads EF_BUF_SYNTH_DEPTH (ef_map_raycast mode 2). graph_nodes16: HOST, 16 floats per node. */
int ef_map_clean_deform(EfContext* ctx, const double* T_wc16, int32_t time, float conf_threshold, int32_t time_delta,
                        float max_depth, const float* graph_nodes16, int32_t n_nodes, int32_t is_fern);
/* IndexMap::combinedPredict (mode 0 ACTIVE, 1 INACTIVE) / synthesizeDepth (mode 2) — IndexMap.cpp:293-476 */
int ef_map_raycast(EfContext* ctx, const double* T_wc16, float max_depth, float conf_threshold, int32_t time,
                   int32_t max_time, int32_t time_delta, int32_t mode);
/* FillIn::vertex/normal/image — FillIn.cpp:62-191 */
int ef_map_fill_in(EfContext* ctx, int32_t passthrough_geometry, int32_t passthrough_image);
/* Resize::image + ElasticFusion::denseEnough — Resize.cpp:50-79, ElasticFusion.cpp:256-268 — of the predicted image as the last
   mode-0 ef_map_raycast / ef_predict / frame or ef_upload of EF_BUF_IMAGE left it */
int ef_dense_enough(EfContext* ctx, int32_t* out);
/* GlobalModel::lastCount / downloadMap (GlobalModel.cpp:673-706): out = count*12 floats, reference Vertex layout
 * (Core/Shaders/Vertex.cpp:22-41) */
int ef_map_count(EfContext* ctx, int32_t* count);
int ef_map_download(EfContext* ctx, float* out12, int32_t max_surfels, int32_t* count);
int ef_map_upload(EfContext* ctx, const float* in12, int32_t count);
/* overwrites surfels [first, first+count) of the resident map in place (count unchanged; EF_EINVAL if the range leaves it).
 * No reference counterpart (the reference never edits its VBO from the host); used to build large maps piecewise. */
int ef_map_upload_range(EfContext* ctx, const float* in12, int32_t first, int32_t count);
/* unstable surfels appended by the last ef_map_fuse (the reference's newUnstableVbo) */
int ef_map_download_new(EfContext* ctx, float* out12, int32_t max_surfels, int32_t* count);

/* ---- map render: the global-surface pass of the reference's viewer, GlobalModel::renderPointCloud (Core/GlobalModel.cpp:286-350,
 *      drawPoints = false) and the colour pass of GUI::drawFXAA (Tools/GUI.h:273-345): every surfel drawn as a screen-facing disc by
 *      draw_global_surface.{vert,geom,frag} / draw_global_surface_phong.frag, depth-tested GL_LESS against a 24-bit depth buffer.
 *      The render has its own z-buffer and output staging, shared with the model view below (allocated by the first call, grown to
 *      the largest view, freed by ef_destroy), and touches neither the frame's textures nor its pose state, so it may run between
 *      any two frames, also while a frame is staged by the look-ahead or in flight between ef_process_frame_device and
 *      ef_finish_frame (it renders the map that frame leaves).
 *
 *      Output: RGBA8, W*H*4 bytes, in glReadPixels order: row 0 is window y = 0. Pixels no surfel covers are (0,0,0,0), so alpha is
 *      coverage. colour_type 3 at time <= 1 divides by zero as the reference's geometry shader does; that output is not pinned. */
typedef struct {
  int32_t width, height;     /* 1..16384 */
  float mvp[16];             /* column-major, the MVP uniform (pangolin::OpenGlMatrix cast to float, as Uniform does) */
  float mv[16];              /* column-major model-view; read only when phong = 1 (lightpos = its translation) */
  float threshold;           /* confidence threshold */
  int32_t color_type;        /* 0 grey, 1 normals, 2 colours, 3 times: renderPointCloud's drawNormals/drawColors/drawTimes */
  int32_t unstable, draw_window, time, time_delta;
  int32_t phong;             /* 0: draw_global_surface.frag (renderPointCloud); 1: draw_global_surface_phong.frag (drawFXAA's colour pass) */
  float sign_mult;           /* phong only; the GUI passes iclnuim ? 1 : -1 */
} EfRenderView;
/* EF_EINVAL for a size out of range, colour_type outside 0..3 or a non-finite matrix. Synchronises. */
int ef_render_map(EfContext* ctx, const EfRenderView* view, uint8_t* rgba_host);
/* same into DEVICE memory (W*H*4 bytes), asynchronous on ef_stream() */
int ef_render_map_device(EfContext* ctx, const EfRenderView* view, uint8_t* rgba_dev);
/* mvp16 / mv16 (column-major) of a pinhole camera at pose T_wc16 (row-major camera-to-world): mv = T_wc^-1, and a projection under
 * which window pixel (i, j) samples the ray through image pixel centre (i + 0.5, j + 0.5) with rows as ef_map_raycast has them, so
 * a render from the tracked pose with the frame's intrinsics lines up with the input image, top row first. Window depth 0 at
 * z_near, 1 at z_far. EF_EINVAL for a size outside 1..16384, non-finite input, fx or fy = 0, or not 0 < z_near < z_far. No device
 * work. */
int ef_render_camera(const double* T_wc16, float fx, float fy, float cx, float cy, int32_t width, int32_t height, float z_near,
                     float z_far, float* mvp16, float* mv16);

/* ---- model view: IndexMap::combinedPredict (splat.vert + combo_splat.frag, Core/IndexMap.cpp:293-476) at any pose, intrinsics and
 *      size. The outputs mean what EF_BUF_IMAGE / VERTEX / NORMAL / TIME mean after ef_map_raycast with the same arguments: row 0 is
 *      the top image row, pixels no surfel covers are all zero, the depth is vertex.z. There is no fill-in (it needs the live frame,
 *      which exists only at the frame's camera). A view touches no frame texture, pose record, z-buffer, index map or tracker state,
 *      and uses the render's z-buffer (grown to the largest view, freed by ef_destroy), so like the render it may run between any two
 *      frames, also while a frame is staged by the look-ahead or in flight between ef_process_frame_device and ef_finish_frame (it
 *      predicts the map that frame leaves). */
typedef struct {
  double T_wc[16];                      /* row-major camera-to-world, as every pose in this ABI */
  float fx, fy, cx, cy;
  int32_t width, height;                /* 1..16384, as ef_render_map */
  float max_depth, conf_threshold;
  int32_t time, max_time, time_delta;   /* combinedPredict's window: ACTIVE = (tick, tick, td), INACTIVE = (0, tick - td, td) */
} EfModelView;
/* HOST outputs (W*H*4 B RGBA8, W*H*16 B float4 vertex + confidence, W*H*16 B float4 normal + radius, W*H*2 B time), synchronises.
 * Any output may be NULL, but not all four. EF_EINVAL for all-NULL outputs, a size outside 1..16384, a non-finite pose entry, a
 * non-finite or zero fx / fy, a non-finite cx / cy, max_depth not finite and > 0, or a non-finite conf_threshold. */
int ef_map_predict_view(EfContext* ctx, const EfModelView* view, uint8_t* image4, float* vertex4, float* normal4, uint16_t* time);
/* same into DEVICE memory, asynchronous on ef_stream(); EF_EINVAL also for an output not aligned to its element (4, 16, 16, 2 B) */
int ef_map_predict_view_device(EfContext* ctx, const EfModelView* view, uint8_t* image4, float* vertex4, float* normal4, uint16_t* time);

/* ---- fuse view: an RGB-D frame from any camera fused into the map, the map half of processFrame without a deformation graph
 *      (Core/ElasticFusion.cpp:536-584) at a pose, intrinsics and size of the caller's choosing: upload, bilateral filter + metric
 *      depth (depth_cutoff), predictIndices, fuse (weighting), predictIndices, clean (conf_threshold, time_delta), all at `time`
 *      and max_depth. The map is byte-identical, order and count included, to what a context built for the view's camera (same
 *      capacity) makes of the same map with ef_preprocess_depth, ef_map_predict_indices, ef_map_fuse, ef_map_predict_indices and
 *      ef_map_clean with these arguments. A full map behaves as the frame's clean at capacity.
 *
 *      A view writes nothing but the surfels and their count: not the pose or tick, the frame's pose record or the tracker's
 *      weighting, any EF_BUF_* texture, the denseEnough count, the unstable list of ef_map_download_new, the look-ahead's staged
 *      frame or the loop-closure graph. Its inputs, index map and scratch are its own (allocated by the first call, grown to the
 *      largest view, freed by ef_destroy). It does not refresh the predicted model: call ef_predict if the next frame should
 *      track against the view's surfels.
 *
 *      For the second camera of a rig, `time` is the tick of the tracked frame the view accompanies (ef_get_tick() - 1 after it).
 *      EF_ESTATE before the first frame (which initialises the map) and between ef_process_frame_begin and _end. Allowed while the
 *      look-ahead holds a staged frame and between ef_process_frame_device and ef_finish_frame: the view is stream-ordered and
 *      fuses into the map that frame leaves. */
typedef struct {
  double T_wc[16];           /* row-major camera-to-world */
  float fx, fy, cx, cy;
  int32_t width, height;     /* 1..16384 */
  float depth_cutoff;        /* metric gate of the preprocess, metres (the frame uses cfg.depth_cutoff) */
  float max_depth;           /* maxDepthProcessed (the frame uses 20) */
  float weighting;           /* >= 0: fuse's confidence weighting, as ef_map_fuse takes it */
  float conf_threshold;
  int32_t time, time_delta;  /* the tick the view's surfels are stamped with; the index map's and clean's window */
} EfFuseView;
/* HOST inputs: RGB8 (W*H*3 B) and uint16 millimetres (W*H), as ef_process_frame takes them; synchronises. EF_EINVAL for a NULL
 * input, a size outside 1..16384, a non-finite pose entry, a non-finite or zero fx / fy, a non-finite cx / cy, depth_cutoff or
 * max_depth not finite and > 0, a negative or non-finite weighting, a non-finite conf_threshold, or time / time_delta < 0.
 * EF_ENOMEM when the view's buffers cannot be grown (the context stays usable). */
int ef_map_fuse_view(EfContext* ctx, const EfFuseView* view, const uint8_t* rgb, const uint16_t* depth);
/* same from DEVICE inputs, asynchronous on ef_stream() (the inputs are read when the stream gets there); EF_EINVAL also for a depth
 * pointer not aligned to 2 bytes */
int ef_map_fuse_view_device(EfContext* ctx, const EfFuseView* view, const uint8_t* rgb_dev, const uint16_t* depth_dev);

/* ---- track view: an RGB-D frame from any camera tracked against the map, the frame-to-model recipe of processFrame
 *      (Core/ElasticFusion.cpp:309-323) run by an RGBDOdometry of the view's camera (RGBDOdometry.cpp:22-117), from a pose guess of
 *      the caller's: upload, RGBA, bilateral filter (depth_cutoff), the live depth pyramid and vertex / normal maps (initICP at
 *      model.max_depth) and intensity pyramid, combinedPredict of `model` at the guess (no fill-in), initICPModel + initRGBModel
 *      from it, Sobel and the photometric candidates, and getIncrementalTransformation(guess, rgb_only, icp_weight, pyramid,
 *      fast_odom, so3 = false). As in the frame, initRGB's depth pyramid is the model's (quirk A.2). The result is byte-identical to
 *      what a context built for the view's camera gives with ef_map_predict_view_device, ef_odom_init_icp_model(0, vertex, normal,
 *      guess), ef_odom_init_rgb_model(0, image), ef_preprocess_depth, ef_odom_init_icp_depth(0, filtered, max_depth),
 *      ef_odom_init_rgb(0, rgba) and ef_odom_track(0, guess, ..., so3 = 0), then ef_odom_stats and ef_odom_covariance.
 *
 *      There is no SO(3) pre-alignment and no fill-in: both need the previous live frame of the same camera, and a one-off view has
 *      none (the reference's own trackers that are not the frame's, modelToModel and the fern tracker, also run with so3 = false).
 *      dense_enough says how well the map covers the view, as ElasticFusion::denseEnough would decide for its predicted image.
 *
 *      A view only reads the map. It writes none of: the pose, tick or weighting of the frame, any EF_BUF_* buffer (the pyramids of
 *      trackers 0 and 1 included), ef_odom_stats(0 / 1), the SO(3) state or staged frame of the look-ahead, the loop-closure state,
 *      the denseEnough count, ef_debug_stage_ms's events or the map. Its inputs, prediction and tracker buffers are its own
 *      (allocated by the first call, grown to the bounding box of the views so far, freed by ef_destroy): 243 B per pixel of that
 *      box, plus 8 B per pixel for the z-buffer it shares with the render and the model view, and about 1 MB besides: 78 MB at
 *      640x480, 521 MB at 1920x1080 and 4.2 GB at 4096x4096. It returns no EF_ESTATE: it may run before the first
 *      frame (on a map from ef_map_upload), between ef_process_frame_begin and _end, while the look-ahead holds a staged frame and
 *      between ef_process_frame_device and ef_finish_frame (stream-ordered: it tracks against the map that frame leaves).
 *
 *      On an empty map, or where the view sees no surfel, the call still returns 0 with whatever the recipe gives: no term is valid,
 *      every system is zero, the pose is the guess as the tracker's finish rebuilds it from its float rotation, both counts are 0,
 *      lastICPError is 0/0 (NaN), the covariance (the inverse of the zero lastA) is not finite and dense_enough is 0. */
typedef struct {
  EfModelView model;         /* the prediction tracked against, as ef_map_predict_view takes it. model.T_wc is the initial guess;
                                model.max_depth is also initICP's cutoff (the frame uses 20 for both). width, height: 32..4096 */
  float depth_cutoff;        /* > 0: the bilateral filter's maxD, metres (the frame uses cfg.depth_cutoff) */
  float icp_weight;          /* >= 0 (the frame uses 10; >= 100: ICP only) */
  int32_t rgb_only, pyramid, fast_odom;  /* as ef_odom_track takes them (the frame uses 0, 1, cfg.fast_odom) */
} EfTrackView;
typedef struct {
  double T_wc[16];           /* tracked pose, row-major camera-to-world */
  EfOdomStats stats;         /* as ef_odom_stats reports them */
  double covariance[36];     /* lastA^-1, as ef_odom_covariance (RGBDOdometry::getCovariance) */
  int32_t dense_enough;      /* ElasticFusion::denseEnough of the view's predicted image, at the view's size */
} EfTrackResult;
/* HOST inputs: RGB8 (W*H*3 B) and uint16 millimetres (W*H); synchronises. trace (HOST, may be NULL when max_trace = 0) receives one
 * record per Gauss-Newton iteration, as ef_odom_track's. EF_EINVAL for a NULL input or output, a negative max_trace, each bad
 * `model` field as ef_map_predict_view checks it, a size outside 32..4096, a non-finite or non-positive depth_cutoff, or a
 * non-finite or negative icp_weight. EF_ENOMEM when the view's buffers cannot be grown (the context stays usable). */
int ef_track_view(EfContext* ctx, const EfTrackView* view, const uint8_t* rgb, const uint16_t* depth, EfTrackResult* out,
                  EfSolveTrace* trace, int32_t max_trace, int32_t* n_trace);
/* same from DEVICE inputs into a DEVICE result, asynchronous on ef_stream() (the inputs are read when the stream gets there); the
 * covariance is computed on the device. EF_EINVAL also for a depth pointer not aligned to 2 bytes or out_dev not aligned to 8 */
int ef_track_view_device(EfContext* ctx, const EfTrackView* view, const uint8_t* rgb_dev, const uint16_t* depth_dev,
                         EfTrackResult* out_dev);

/* ---- camera: a second RGB-D sensor run frame after frame against the context's map, as ElasticFusion::processFrame
 *      (Core/ElasticFusion.cpp:270-607, closeLoops = false, reloc = false) runs the context's own camera. A camera belongs to one
 *      context and has its own tracker (RGBDOdometry of its camera), previous frame, pose, prediction and fill-in; it writes into the
 *      context's map. One ef_camera_frame runs, at the camera's intrinsics and size:
 *        1. upload, RGBA, bilateral filter (depth_cutoff) + metric depth, initICP at max_depth and the intensity pyramid (:278-285);
 *        2. unless has_pose: initICPModel + initRGBModel from the camera's own prediction of its previous call, or from its fill-in
 *           when that prediction is not dense enough (decided on the device, :302-315; frame_to_frame_rgb takes the fill-in image
 *           always), the SO(3) pre-alignment against the previous frame's intensity pyramid (so3) and
 *           getIncrementalTransformation(rgb_only, icp_weight, pyramid, fast_odom, so3);
 *           with has_pose: the pose is set (processFrame's in_T_wc) and nothing is tracked;
 *        3. the velocity weighting from the camera's previous pose, times weight_multiplier (:369-383);
 *        4. fuse and not rgb_only: predictIndices, fuse, predictIndices, clean at `time`, with no graph (:536-585);
 *        5. predict(): combinedPredict ACTIVE at (time, time, time_delta), then the fill-in from this frame's filtered depth and RGB
 *           (:621-653) -- the model the camera's next frame tracks against.
 *      The first frame of a camera must have has_pose (EF_ESTATE otherwise); its intensity pyramid becomes the previous one of the
 *      next frame (initFirstRGB) and, if it fuses, its weighting is weight_multiplier.
 *
 *      A camera writes the surfels and their count, nothing else of the context: not the frame's pose, tick, weighting or pose record,
 *      any EF_BUF_* buffer, the frame's prediction, fill-in or denseEnough count, the SO(3) or staged frame of the look-ahead, the
 *      loop-closure state or ef_debug_stage_ms's events. The frame does not re-predict after a camera fused (call ef_predict if it
 *      should). For a rig: frame A with ef_process_frame*, then the camera with time = ef_get_tick() - 1.
 *
 *      With close_loops = 1 (a context with cfg.close_loops = 2 only), a camera's frames close local loops as the frame does in that
 *      mode (Core/ElasticFusion.cpp:387, 447-534, 559-569 and 593), at the camera's intrinsics, size and `time` in place of the tick:
 *        - on a fused, not rgb_only frame after the camera's first (has_pose frames too): after step 3, predict() ACTIVE at (time, time,
 *          time_delta), the INACTIVE prediction at (0, time - time_delta, time_delta), model-to-model tracking in a second tracker of the
 *          camera, the acceptance test with the context's count_thresh / err_thresh / cov_thresh and the constraints on its
 *          (W/20) x (H/20) grid; on an accepted front half with a graph and a constraint, the solve of ef_local_deform_result
 *          (pin = (deforms == 0), source time `time`) and, unless it stops with code 6, its pose becomes T_wc_est and step 4's clean
 *          deforms the map with the nodes (its time-stamp refresh reads a depth-only prediction at (time, time - time_delta, 65535));
 *          then deforms += 1 and last_deform_time = time;
 *        - at the end of every call, the graph is sampled from the map (fuse = 0 and first calls too).
 *      EfCameraResult.T_wc is then the pose after the closure; the weighting is the one computed before it. Besides the surfels and
 *      their count, a closing camera writes the context's graph, deforms and last_deform_time (none of the frame's other loop-closure
 *      results: see ef_camera_deform_result). ef_camera_frame_device then waits for the host once for the front half's record and, on a
 *      frame that solves, once more for the solve (as ef_process_frame_device does with cfg.close_loops = 2). The side that did not
 *      deform the map keeps tracking against the prediction it made before the closure.
 *
 *      fuse = 1 returns EF_ESTATE before the context's first frame and between ef_process_frame_begin and _end (as ef_map_fuse_view);
 *      fuse = 0 may also run before the first frame, on a map from ef_map_upload. Both may run while the look-ahead holds a staged frame
 *      and between ef_process_frame_device and ef_finish_frame (stream-ordered). At most EF_MAX_CAMERAS cameras are live per context. */
#define EF_MAX_CAMERAS 4
typedef struct EfCamera EfCamera;
typedef struct {
  int32_t width, height;          /* 32..4096 */
  float fx, fy, cx, cy;
  float depth_cutoff, max_depth;  /* the bilateral filter's maxD (cfg.depth_cutoff); maxDepthProcessed (20), also the map passes' */
  float conf_threshold;           /* confidenceThreshold of the prediction and the clean (cfg.confidence) */
  int32_t time_delta;             /* >= 0 (cfg.time_delta) */
  float icp_weight;               /* >= 0 (10; >= 100: ICP only) */
  int32_t rgb_only, pyramid, fast_odom, so3, frame_to_frame_rgb;  /* the frame's setters (0, 1, cfg.fast_odom, cfg.so3, ...) */
  int32_t close_loops;            /* 0: open loop. 1: its frames close local loops on the context's graph (cfg.close_loops = 2 only) */
} EfCameraConfig;
typedef struct {
  int32_t time;                   /* >= 0: the tick this frame's surfels are stamped with and its prediction is made at */
  float weight_multiplier;        /* finite, >= 0 */
  int32_t has_pose;               /* set the pose T_wc instead of tracking (processFrame's in_T_wc) */
  double T_wc[16];                /* row-major camera-to-world, read when has_pose */
  int32_t fuse;                   /* 0: track and predict only (localise in a fixed map) */
} EfCameraFrame;
typedef struct {
  double T_wc[16];                /* the camera's pose after the frame */
  EfOdomStats stats;              /* its tracker's, as ef_odom_stats reports them */
  double covariance[36];          /* lastA^-1, as ef_odom_covariance */
  int32_t tracked;                /* 0 when the pose came from has_pose */
  int32_t dense_enough;           /* denseEnough of the prediction this frame tracked against (0: the fill-in was used) */
  float weighting;                /* the fusion weighting (ElasticFusion.cpp:369-383) */
} EfCameraResult;
/* EF_EINVAL for a NULL argument or a bad field (a size outside 32..4096, a zero or non-finite fx / fy, a non-finite cx / cy,
 * depth_cutoff or max_depth not finite and > 0, a non-finite conf_threshold, a negative time_delta, a non-finite or negative
 * icp_weight, close_loops other than 0 or 1, or 1 on a context whose cfg.close_loops is not 2); EF_ESTATE when EF_MAX_CAMERAS cameras are live; EF_ENOMEM when its buffers cannot be allocated (the context stays
 * usable). Memory: see INTEGRATION.md. Synchronises. */
int ef_camera_create(EfContext* ctx, const EfCameraConfig* cfg, EfCamera** out);
/* frees the camera (ef_destroy frees those still live); EF_EINVAL for a camera of another context. Synchronises. */
int ef_camera_destroy(EfContext* ctx, EfCamera* cam);
/* HOST inputs RGB8 (W*H*3 B) and uint16 millimetres (W*H); synchronises. trace (HOST, may be NULL when max_trace = 0) receives one
 * record per Gauss-Newton iteration of a tracked frame. EF_EINVAL for a NULL argument, a camera of another context, a negative time,
 * a bad weight_multiplier, a non-finite pose entry with has_pose, or a negative max_trace. */
int ef_camera_frame(EfContext* ctx, EfCamera* cam, const EfCameraFrame* frame, const uint8_t* rgb, const uint16_t* depth,
                    EfCameraResult* out, EfSolveTrace* trace, int32_t max_trace, int32_t* n_trace);
/* same from DEVICE inputs into a DEVICE result, asynchronous on ef_stream(); EF_EINVAL also for a depth pointer not aligned to 2
 * bytes or out_dev not aligned to 8 */
int ef_camera_frame_device(EfContext* ctx, EfCamera* cam, const EfCameraFrame* frame, const uint8_t* rgb_dev, const uint16_t* depth_dev,
                           EfCameraResult* out_dev);
/* device pointer + byte size of a buffer of the camera, at its size: EF_BUF_RGB, RGBA, DEPTH_* (its inputs), IMAGE, VERTEX, NORMAL,
 * TIME (its prediction), FILL_* (its fill-in) and the tracker ids 40..53 without the 100*which (its pyramids, `level`). Any other id:
 * EF_EINVAL. */
int ef_camera_buffer(EfContext* ctx, EfCamera* cam, int32_t id, int32_t level, void** dev_ptr, size_t* bytes);
/* close_loops = 1: ef_local_deform_result for the camera's last frame. solved, applied and result are the camera's; deforms,
 * last_deform_time and the graph (nodes4, n_out as there) are the context's, which the frame and its closing cameras share.
 * EF_EINVAL for a NULL out, a negative max_nodes, NULL nodes4 with max_nodes > 0 or a camera of another context; EF_ESTATE for a
 * camera with close_loops = 0. Synchronises. */
int ef_camera_deform_result(EfContext* ctx, EfCamera* cam, EfLocalDeform* out, float* nodes4, int32_t max_nodes, int32_t* n_out);

/* ---- rig: cameras bolted together at known extrinsics, tracked as one rigid body. A rig is built from cameras of one context that
 *      all have close_loops = 0 (an open-loop rig) or all close_loops = 1 (a closing rig); member 0's camera frame is the rig body. One
 *      ef_rig_frame runs ef_camera_frame's steps for every member, except that the pose is one joint estimate:
 *        1. each member's input side and model inputs (its own fill-in choice and frame_to_frame_rgb);
 *        2. with has_pose, member 0's pose is T_wc and member i's T_wc * T_0i; nothing is tracked. Otherwise one Gauss-Newton loop:
 *           the SO(3) pre-alignment seeds every member (resultRt_i = T_i0 * resultRt_0 * T_0i), then per iteration each member's systems are reduced, combined (rgb + w^2 icp), mapped into member 0's parameters through
 *           the adjoint Ad(T_i0) (A += Ad^T A_i Ad, b += Ad^T b_i, in the (t, w) order of the update), summed and solved once; member 0
 *           takes the update as getIncrementalTransformation would and member i is set to T_i0 * resultRt_0 * T_0i, so the rig stays
 *           rigid at every iteration. The pre-alignment is member 0's alone, or with joint_so3 one loop for the whole body: member
 *           0's loop state is the body's and member i's rotation is R_i0 * R_0 * R_0i; per iteration each member reduces its own
 *           level-2 image pair at its own homography, member i's 3x3 system enters the joint one as R_0i A_i R_0i^T, R_0i b_i (sums
 *           in double, then float), the error is sqrt(sum of res0) / sum of res1 and the count the sum of res1, and the reference's
 *           convergence and divergence tests and update act on these for member 0 (on divergence every member keeps its last
 *           rotation); every member reports the joint SO(3) error and count. A one-member joint rig computes what its camera computes
 *           with gn_cluster off, except for the joint fields of its SO(3) trace records;
 *        3. the finish: if any member's translation jumped by more than 0.3 m, every member keeps its previous pose; otherwise member 0
 *           is orthogonalised as the tracker does and member i's pose is T_w0 * T_0i. Each member gets its own velocity weighting times
 *           weight_multiplier;
 *        4. with fuse, every member's map half in member order at `time`; then every member's predict() with fill-in. So each member's
 *           next model holds the surfels the whole rig fused in this frame, which calling the cameras one after another does not give.
 *      A one-member rig computes what ef_camera_frame computes for its camera with the context's gn_cluster off (EF_GN_CLUSTER=0); the
 *      rig never runs the coarse levels in the cluster launch, nor the SO(3) pre-alignment when it is joint. Not covered: rgb_only
 *      members, the C++ drop-in classes and the command line.
 *
 *      A closing rig closes local loops as one body, on the context's graph (T_x_i = T_x_0 * T_0i throughout):
 *        - on a fused frame after the rig's first (has_pose frames too), after step 3: each member's predict() ACTIVE at (time, time,
 *          time_delta) and INACTIVE prediction at (0, time - time_delta, time_delta), as a closing camera makes them; each member's loop
 *          tracker at its pose, with the INACTIVE prediction as its model; one joint model-to-model registration over the members' loop
 *          trackers (step 2's solve with rgb_only = 0, icp_weight = 10, no SO(3)) and step 3's finish, so T_est_i = T_est_0 * T_0i;
 *        - one acceptance test: every diagonal entry of the joint system's inverse within cov_thresh, count > count_thresh and
 *          error < err_thresh, where count is the ICP inlier count SUMMED over the members and error = sqrt(sum of their ICP
 *          residuals) / count (for one member, the camera's test);
 *        - accepted, each member's (W_i/20) x (H_i/20) grid is sampled as a closing camera samples its own (src = T_curr_i v,
 *          dst = T_est_i v, time = its INACTIVE stamp), concatenated in member order; with a graph and a constraint, one solve of
 *          them all (pin = (deforms == 0), source time `time`) and, unless it stops with code 6, member 0's pose becomes T_est_0 and
 *          member i's T_est_0 * T_0i; only member 0's clean in step 4 deforms the map (the map is deformed once); then deforms += 1
 *          and last_deform_time = time;
 *        - at the end of every call, the graph is sampled from the map (fuse = 0 and first calls too).
 *      The members' EfCameraResult.T_wc and EfRigResult.T_wc are then the closed poses; the weighting is the one computed before the
 *      closure. ef_rig_frame_device waits for the host once for the front half's record and, on a frame that solves, once more for
 *      the solve (as a closing camera does). Results: ef_rig_loop_result and ef_rig_deform_result. A one-member closing rig computes
 *      what its closing camera computes with gn_cluster off.
 *      While a camera is a member, ef_camera_frame* and ef_camera_deform_result on it return EF_ESTATE (ef_camera_buffer still works);
 *      after ef_rig_destroy its members run alone again (a closing camera closes its own loops). ef_camera_destroy of a member
 *      and ef_destroy free the rig first. fuse and the first frame follow the camera rules: fuse = 1 needs the context past its first
 *      frame and not between ef_process_frame_begin and _end, and the rig's first frame must have has_pose (EF_ESTATE otherwise). A rig
 *      may run while the look-ahead holds a staged frame and between ef_process_frame_device and ef_finish_frame (stream-ordered). */
typedef struct EfRig EfRig;
typedef struct {
  int32_t n;                                /* 1..EF_MAX_CAMERAS */
  EfCamera* cameras[EF_MAX_CAMERAS];        /* cameras of the context, each in at most one rig, with rgb_only = 0 and the same
                                               close_loops, icp_weight, pyramid, fast_odom and so3 */
  double T_0i[EF_MAX_CAMERAS][16];          /* row-major, camera i -> member 0's camera: rigid (|R^T R - I| <= 1e-6 entrywise, last row
                                               0 0 0 1, finite); T_0i[0] is the identity */
  int32_t joint_so3;                        /* 0: member 0's SO(3) pre-alignment seeds the rig; 1 (members with so3 = 1): one joint
                                               SO(3) pre-alignment over every member's image pair (see step 2) */
} EfRigConfig;
typedef struct {                            /* as EfCameraFrame, once for the rig */
  int32_t time;                             /* >= 0 */
  float weight_multiplier;                  /* finite, >= 0 */
  int32_t has_pose;
  double T_wc[16];                          /* member 0's pose, read when has_pose */
  int32_t fuse;
} EfRigFrame;
typedef struct {
  double T_wc[16];                          /* member 0's pose = the rig's */
  double lastA[36], lastb[6];               /* the joint system of the last iteration, in member 0's parameters (of the last tracked
                                               frame when this one has has_pose) */
  double covariance[36];                    /* lastA^-1 */
  int32_t tracked;                          /* 0 when the pose came from has_pose */
} EfRigResult;
/* EF_EINVAL for a NULL argument, n outside 1..EF_MAX_CAMERAS, a camera of another context or listed twice, one already in a rig, a
 * member with rgb_only set, members whose close_loops, icp_weight, pyramid, fast_odom or so3 differ, a T_0i that is not rigid or
 * finite, T_0i[0] not the identity, a joint_so3 other than 0 and 1, or joint_so3 = 1 with members whose so3 = 0. EF_ENOMEM when a closing rig's buffers cannot be allocated (the context stays usable).
 * Synchronises. */
int ef_rig_create(EfContext* ctx, const EfRigConfig* cfg, EfRig** out);
/* frees the rig; its cameras stay and may run alone again. EF_EINVAL for a rig of another context. Synchronises. */
int ef_rig_destroy(EfContext* ctx, EfRig* rig);
/* HOST inputs rgb[i] (RGB8, W_i*H_i*3 B) and depth[i] (uint16 millimetres) of member i; members: n results, member i's stats and
 * covariance its own (member 0's lastA / lastb are the joint system's); synchronises. trace (HOST, may be NULL when max_trace = 0):
 * n blocks of max_trace records, member i's at trace + i * max_trace, one per iteration of a tracked frame (member 0's SO(3) records
 * first, or with joint_so3 every member's own: its A_so3 / b_so3 / so3_residual, the joint 3x3 system in lastA[0..8] / lastb[0..2]
 * and the joint update in result[0..2], 0 on the iteration that stops the loop) with its own A_icp / A_rgb / b_icp / b_rgb, its own
 * combined lastA / lastb and the joint result; n_trace (may be NULL): the
 * n record counts. EF_EINVAL for a NULL argument, a rig of another context, a negative time, a bad weight_multiplier, a non-finite
 * pose entry with has_pose, or a negative max_trace. */
int ef_rig_frame(EfContext* ctx, EfRig* rig, const EfRigFrame* frame, const uint8_t* const* rgb, const uint16_t* const* depth,
                 EfCameraResult* members, EfRigResult* out, EfSolveTrace* trace, int32_t max_trace, int32_t* n_trace);
/* same from DEVICE inputs into DEVICE results (members_dev: n EfCameraResult), asynchronous on ef_stream(); EF_EINVAL also for a
 * depth pointer not aligned to 2 bytes or a result not aligned to 8 */
int ef_rig_frame_device(EfContext* ctx, EfRig* rig, const EfRigFrame* frame, const uint8_t* const* rgb_dev, const uint16_t* const* depth_dev,
                        EfCameraResult* members_dev, EfRigResult* out_dev);
/* a closing rig's front half of its last frame, as EfLoopResult reports the frame's */
typedef struct {
  int32_t ran;                                   /* 0: no front half ran (a first or fuse = 0 call) */
  int32_t accepted;                              /* the joint test (see above) */
  int32_t n_constraints;                         /* the sum of member_constraints */
  int32_t member_constraints[EF_MAX_CAMERAS];    /* each member's, at most its (W_i/20) x (H_i/20) grid (0 beyond n) */
  float lastICPError, lastICPCount;              /* the joint error and the summed count the test compared */
  double cov_diag[6];                            /* of the joint system's inverse */
  double T_wc_curr[16];                          /* member 0's pose before the closure */
  double T_wc_est[16];                           /* member 0's pose after the joint registration */
} EfRigLoopResult;
/* ef_local_loop_result for a closing rig's last frame: src3 / dst3 / times (HOST, any may be NULL) receive the concatenated
 * constraints, at most max_constraints; n_out (may be NULL) their number. EF_EINVAL for a NULL out, a negative max_constraints or a
 * rig of another context; EF_ESTATE for an open-loop rig. Synchronises. */
int ef_rig_loop_result(EfContext* ctx, EfRig* rig, EfRigLoopResult* out, double* src3, double* dst3, int32_t* times, int32_t max_constraints,
                       int32_t* n_out);
/* ef_camera_deform_result for a closing rig's last frame: solved, applied and result are the rig's; deforms, last_deform_time and the
 * graph the context's. EF_EINVAL for a NULL out, a negative max_nodes, NULL nodes4 with max_nodes > 0 or a rig of another context;
 * EF_ESTATE for an open-loop rig. Synchronises. */
int ef_rig_deform_result(EfContext* ctx, EfRig* rig, EfLocalDeform* out, float* nodes4, int32_t max_nodes, int32_t* n_out);

/* ---- named device buffers (the reference's GPUTexture / DeviceArray handles) ------------------------------ */
enum {
  /* input / preprocess textures (ElasticFusion::textures, GPUTexture.cpp:22-27) */
  EF_BUF_RGB = 0,                 /* u8 x3  */
  EF_BUF_DEPTH_RAW = 1,           /* u16    */
  EF_BUF_DEPTH_FILTERED = 2,      /* u16    */
  EF_BUF_DEPTH_METRIC = 3,        /* f32    */
  EF_BUF_DEPTH_METRIC_FILTERED = 4,
  EF_BUF_RGBA = 5,                /* u8 x4: the RGB texture as CUDA sees it */
  /* IndexMap attachments (IndexMap.h:74-142) */
  EF_BUF_INDEX = 10,              /* u32    */
  EF_BUF_VERT_CONF = 11,          /* f32 x4 */
  EF_BUF_COLOR_TIME = 12,
  EF_BUF_NORM_RAD = 13,
  EF_BUF_IMAGE = 14,              /* u8 x4  */
  EF_BUF_VERTEX = 15,             /* f32 x4 */
  EF_BUF_NORMAL = 16,
  EF_BUF_TIME = 17,               /* u16    */
  EF_BUF_OLD_IMAGE = 18,
  EF_BUF_OLD_VERTEX = 19,
  EF_BUF_OLD_NORMAL = 20,
  EF_BUF_OLD_TIME = 21,
  EF_BUF_SYNTH_DEPTH = 22,        /* f32    */
  /* FillIn textures */
  EF_BUF_FILL_IMAGE = 30,
  EF_BUF_FILL_VERTEX = 31,
  EF_BUF_FILL_NORMAL = 32,
  /* RGBDOdometry pyramids: id + 100*which, `level` selects the pyramid level */
  EF_BUF_VMAP_CURR = 40,          /* f32, 3 planes stacked ((3*rows) x cols) */
  EF_BUF_NMAP_CURR = 41,
  EF_BUF_VMAP_G_PREV = 42,
  EF_BUF_NMAP_G_PREV = 43,
  EF_BUF_LAST_DEPTH = 44,         /* f32 */
  EF_BUF_NEXT_DEPTH = 45,
  EF_BUF_LAST_IMAGE = 46,         /* u8 */
  EF_BUF_NEXT_IMAGE = 47,
  EF_BUF_LAST_NEXT_IMAGE = 48,
  EF_BUF_DIDX = 49,               /* i16 */
  EF_BUF_DIDY = 50,
  EF_BUF_DEPTH_TMP = 51,          /* u16 */
  EF_BUF_CORRES = 52,             /* DataTerm 16 B */
  EF_BUF_VMAPS_TMP = 53           /* f32 x4, level 0 only */
};
/* device pointer + byte size of a named buffer (id + 100*which for tracker buffers) */
int ef_buffer(EfContext* ctx, int32_t id, int32_t level, void** dev_ptr, size_t* bytes);
int ef_upload(EfContext* ctx, int32_t id, int32_t level, const void* host, size_t bytes);
int ef_download(EfContext* ctx, int32_t id, int32_t level, void* host, size_t bytes);
/* Resize::image / vertex / time (Core/Shaders/Resize.cpp:50-159): the named full-resolution attachment (RGBA8, RGBA32F or
 * R16UI) sampled on the (W/factor) x (H/factor) grid of texel centres with nearest filtering, into HOST memory, tightly packed. */
int ef_resize(EfContext* ctx, int32_t id, int32_t factor, void* host_out, size_t bytes);
/* number of kernels launched by this context since creation (bench.py's gpu_launches) */
int ef_launch_count(EfContext* ctx, int64_t* n);
/* EF_STAGE_TIMING=1 in the environment at ef_create: milliseconds between the stage events of the last frame, out[16]:
 * [1] upload + RGBA + bilateral/metric, [2] live pyramids + SO(3), [3] model pyramids, [4] sobel + candidates, [5] Gauss-Newton
 * loop, [6] finish, [7] index map, [8] fuse, [9] index map, [10] clean, [11] predict. Returns the number of slots (0 if off). */
int ef_debug_stage_ms(EfContext* ctx, float* out16);
/* EF_STAGE_TIMING=1: milliseconds from the start of the frame in flight during the last ef_prefetch_frame* call to the start
 * of the side stream's work (once it may begin) and to its end, out[2]. Returns 2, or 0 without a timed prefetch. */
int ef_debug_lookahead_ms(EfContext* ctx, float* out2);

#ifdef __cplusplus
}
#endif
#endif /* EFUSION_B200_H_ */
