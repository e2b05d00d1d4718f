/* TEST INFRASTRUCTURE ONLY — CPU oracle (C ABI) for the ElasticFusion hot path.
 *
 * A single-precision CPU restatement of the reference's per-frame tracking (CUDA half,
 * Core/Cuda/{reduce,cudafuncs}.cu + Core/Utils/RGBDOdometry.cpp) and mapping (GLSL half,
  * Core/Shaders + Core/{GlobalModel,IndexMap,ElasticFusion}.cpp). Every function cites the
 * reference file:line it follows.  Nothing here is linked into the product.
 *
 * PARITY PIN STATUS: the reference ships no tests, golden vectors or fixtures (SURVEY.md §4).
 *  - tracking half: pinned against the reference's own CUDA kernels compiled unmodified
 *    from the reference tree into oracle/_ref/ (run on the GPU; tests/test_gpu_ref_pin.py).
 *  - mapping half (GLSL): pinned against the reference's own shader files, executed unmodified
 *    on Mesa 18 llvmpipe (the software libGL bundled with Nsight Compute in this image) by
 *    oracle/gl/ref_gl_harness.cpp; the outputs are committed as tests/golden/ref_mapping_160x120.npz
 *    (generator tests/golden/make_gl_golden.py) and tests/test_gl_golden.py compares every pass.
 *    The reference's application (Pangolin window, NVIDIA GL) itself cannot be built here.
 *
 * Conventions: all images row-major, no pitch. SoA vertex/normal maps are 3 planes stacked
 * vertically ((3*rows) x cols) exactly as the reference's DeviceArray2D<float> maps.
 * float4 maps are AoS [rows][cols][4]. 3x3 matrices are row-major float[9]; poses are
 * row-major double[16] (4x4).
 */
#ifndef EF_ORACLE_H_
#define EF_ORACLE_H_
#include <stdint.h>
#ifdef __cplusplus
extern "C" {
#endif

typedef struct {
  int16_t zero_x, zero_y; /* pixel in the model ("last") image  */
  int16_t one_x, one_y;   /* pixel in the live ("next") image   */
  float diff;
  int32_t valid;          /* reference: bool + padding, 16 bytes */
} EfoDataTerm;

/* ---------------- image kernels: Core/Cuda/cudafuncs.cu ---------------- */
void efo_pyr_down_u16(const uint16_t* src, int srows, int scols, uint16_t* dst);
void efo_create_vmap(const uint16_t* depth, int rows, int cols, float fx, float fy, float cx, float cy,
                     float depth_cutoff, float* vmap);
void efo_create_nmap(const float* vmap, int rows, int cols, float* nmap);
void efo_transform_maps(float* vmap, float* nmap, int rows, int cols, const float* R, const float* t);
void efo_copy_maps(const float* vtx4, const float* nrm4, int rows, int cols, float* vmaps_tmp, float* vmap,
                   float* nmap);
void efo_resize_map(const float* in, int srows, int scols, float* out, int normalize);
void efo_pyr_down_gauss_f(const float* src, int srows, int scols, float* dst);
void efo_pyr_down_u8(const uint8_t* src, int srows, int scols, uint8_t* dst);
void efo_vertices_to_depth(const float* vmaps_tmp, int rows, int cols, float cutoff, float* dst);
void efo_rgba_to_intensity(const uint8_t* rgba, int rows, int cols, uint8_t* dst);
void efo_sobel(const uint8_t* src, int rows, int cols, int16_t* dx, int16_t* dy);
void efo_project_points(const float* depth, int rows, int cols, float fx, float fy, float cx, float cy,
                        float* cloud3);

/* ---------------- reductions: Core/Cuda/reduce.cu ---------------- */
void efo_icp_step(const float* Rcurr, const float* tcurr, const float* vmap_curr, const float* nmap_curr,
                  const float* Rprev_inv, const float* tprev, float fx, float fy, float cx, float cy,
                  const float* vmap_g_prev, const float* nmap_g_prev, float dist_thres, float angle_thres, int rows,
                  int cols, float* A36, float* b6, float* residual2);
void efo_rgb_residual(float min_scale, const int16_t* dIdx, const int16_t* dIdy, const float* last_depth,
                      const float* next_depth, const uint8_t* last_image, const uint8_t* next_image,
                      EfoDataTerm* corres, float max_depth_delta, const float* kt3, const float* krkinv9, int rows,
                      int cols, int* sigma_sum, int* count);
void efo_rgb_step(const EfoDataTerm* corres, float sigma, const float* cloud3, float fx, float fy,
                  const int16_t* dIdx, const int16_t* dIdy, float sobel_scale, int rows, int cols, float* A36,
                  float* b6);
void efo_so3_step(const uint8_t* last_image, const uint8_t* next_image, const float* image_basis9,
                  const float* kinv9, const float* krlr9, int rows, int cols, float* A9, float* b3,
                  float* residual2);

/* ---------------- tracker host logic: Core/Utils/RGBDOdometry.cpp ---------------- */
typedef struct EfoOdometry EfoOdometry;

typedef struct {
  int32_t kind;  /* 0 = SE3 Gauss-Newton iteration, 1 = SO3 pre-alignment iteration */
  int32_t level; /* pyramid level */
  int32_t iter;
  int32_t rgb_count;
  int32_t rgb_sigma;
  float sigma_val;
  float A_icp[36], b_icp[6], icp_residual[2];
  float A_rgb[36], b_rgb[6];
  float A_so3[9], b_so3[3], so3_residual[2];
  double lastA[36], lastb[6], result[6];
} EfoTrace;

EfoOdometry* efo_odom_create(int width, int height, float cx, float cy, float fx, float fy, float dist_thresh,
                             float angle_thresh);
void efo_odom_destroy(EfoOdometry* o);
void efo_odom_init_icp_depth(EfoOdometry* o, const uint16_t* filtered_depth, float depth_cutoff);
void efo_odom_init_icp_pred(EfoOdometry* o, const float* vtx4, const float* nrm4);
void efo_odom_init_icp_model(EfoOdometry* o, const float* vtx4, const float* nrm4, const double* T_wc16);
void efo_odom_init_rgb(EfoOdometry* o, const uint8_t* rgba);
void efo_odom_init_rgb_model(EfoOdometry* o, const uint8_t* rgba);
void efo_odom_init_first_rgb(EfoOdometry* o, const uint8_t* rgba);
/* returns the number of trace records written (<= max_trace); T_wc16 is updated in place */
int efo_odom_track(EfoOdometry* o, double* T_wc16, int rgb_only, float icp_weight, int pyramid, int fast_odom,
                   int so3, EfoTrace* trace, int max_trace);
/* out8: lastICPError, lastICPCount, lastRGBError, lastRGBCount, lastSO3Error, lastSO3Count, 0, 0 */
void efo_odom_stats(const EfoOdometry* o, float* out8);
void efo_odom_last_system(const EfoOdometry* o, double* A36, double* b6);
void efo_odom_covariance(const EfoOdometry* o, double* cov36);
/* buffer access for stage tests: which = 0 vmap_curr,1 nmap_curr,2 vmap_g_prev,3 nmap_g_prev (float, 3*rows*cols)
 * 4 lastDepth, 5 nextDepth (float rows*cols), 6 lastImage, 7 nextImage, 8 lastNextImage (u8),
 * 9 dIdx, 10 dIdy (int16), 11 depth_tmp (u16) */
const void* efo_odom_buffer(const EfoOdometry* o, int which, int level);

/* ---------------- preprocess: depth_bilateral.frag / depth_metric.frag ---------------- */
void efo_bilateral(const uint16_t* depth, int rows, int cols, float max_d, uint16_t* out);
void efo_metric(const uint16_t* depth, int rows, int cols, float max_d, float* out);

/* ---------------- surfel map: GlobalModel / IndexMap / FillIn / Resize ---------------- */
/* surfels are AoS 12 floats: pos.xyz conf | colour(24-bit as float) unused initTime lastTime | normal.xyz radius
 * (Core/Shaders/Vertex.cpp:22-41) */
int efo_feedback_buffer(const uint8_t* rgb, const float* depth_metric, int rows, int cols, const float* cam4,
                        int time, float max_depth, float* out_surfels);
int efo_map_initialise(const float* raw_fb, int raw_count, const float* filt_fb, int filt_count, int cap_pixels,
                       float* map);
void efo_predict_indices(const float* map, int count, const double* T_wc16, int time, float max_depth,
                         int time_delta, int rows, int cols, const float* cam4, uint32_t* index, float* vert_conf4,
                         float* color_time4, float* norm_rad4);
/* fuse: updates map in place; writes new unstable surfels to new_unstable (capacity rows*cols); returns their count */
int efo_fuse(float* map, int count, const double* T_wc16, int time, const uint8_t* rgb, const float* depth_raw,
             const float* depth_filt, const uint32_t* index, const float* vert_conf4, const float* color_time4,
             const float* norm_rad4, float max_depth, float weighting, int rows, int cols, const float* cam4,
             float* new_unstable);
/* clean: stable compaction of map followed by new_unstable into out; returns new count */
int efo_clean(const float* map, int count, const float* new_unstable, int new_count, const double* T_wc16,
              int time, const uint32_t* index, const float* vert_conf4, const float* color_time4,
              const float* norm_rad4, float conf_threshold, int time_delta, float max_depth, int rows, int cols,
              const float* cam4, float* out);
/* clean with a deformation graph (copy_unstable.vert:132-322): nodes = 16 floats each (position 3, rotation 9 column-major,
 * translation 3, time — Deformation.cpp:175-189), depth = IndexMap::depthTex() (synthesizeDepth). n_nodes == 0: efo_clean. */
int efo_clean_deform(const float* map, int count, const float* new_unstable, int new_count, const double* T_wc16, int time,
                     const uint32_t* index, const float* vert_conf4, const float* color_time4, float conf_threshold,
                     int time_delta, float max_depth, int rows, int cols, const float* cam4, const float* nodes, int n_nodes,
                     const float* depth, int is_fern, float* out);
/* combinedPredict: image RGBA8, vertex float4, normal float4, time u16; depth_only!=0 -> depth_out (float) only */
void efo_combined_predict(const float* map, int count, const double* T_wc16, float max_depth, float conf_threshold,
                          int time, int max_time, int time_delta, int rows, int cols, const float* cam4,
                          uint8_t* image4, float* vertex4, float* normal4, uint16_t* time_out, float* depth_out,
                          int depth_only);
void efo_fill_vertex(const float* existing4, const uint16_t* raw_depth, int passthrough, int rows, int cols,
                     const float* cam4, float* out4);
void efo_fill_normal(const float* existing4, const uint16_t* raw_depth, int passthrough, int rows, int cols,
                     const float* cam4, float* out4);
void efo_fill_image(const uint8_t* existing4, const uint8_t* rgb, int passthrough, int rows, int cols,
                    uint8_t* out4);
int efo_dense_enough(const uint8_t* image4, int rows, int cols, int factor);

/* ---------------- whole pipeline: Core/ElasticFusion.cpp processFrame (open loop) ---------------- */
typedef struct EfoFusion EfoFusion;
typedef struct {
  int width, height;
  float fx, fy, cx, cy;
  int time_delta;      /* ElasticFusion ctor timeDelta (200; INT_MAX/2 in open loop) */
  float confidence;    /* 10 */
  float depth_cutoff;  /* 3 */
  float icp_weight;    /* 10 */
  int fast_odom, so3, frame_to_frame_rgb, pyramid, rgb_only;
  int capacity;        /* max surfels */
} EfoConfig;
EfoFusion* efo_fusion_create(const EfoConfig* cfg);
/* Local loop closure FRONT HALF (ElasticFusion.cpp:447-505): INACTIVE prediction, model-to-model registration, acceptance
 * test, constraint sampling. Enabled per frame by efo_fusion_set_loop_closure; the deformation solve is out of scope, so
 * nothing is applied to the map or pose — the results of the last frame are read with efo_fusion_loop_result. */
typedef struct {
  int32_t ran;            /* the front half ran for the last frame (tick > 1, not rgbOnly) */
  int32_t accepted;       /* covOk && lastICPCount > icpCountThresh && lastICPError < icpErrThresh */
  int32_t n_constraints;
  float lastICPError, lastICPCount;
  double cov_diag[6];
  double T_wc_est[16];
} EfoLoopResult;
void efo_fusion_set_loop_closure(EfoFusion* f, int enabled, int count_thresh, float err_thresh, float cov_thresh);
/* src / dst: 3 doubles per constraint (vert_w_curr, vert_w_est), times: the INACTIVE view's time stamp; returns the count */
int efo_fusion_loop_result(const EfoFusion* f, EfoLoopResult* out, double* src3, double* dst3, int32_t* times, int max_constraints);
/* second-half variant: processFrame with a deformation graph applied in clean and an optional pose override after tracking
 * (what the reference does when localDeformation.constrain() succeeded: ElasticFusion.cpp:519-526, 559-586) */
void efo_fusion_process_frame_deform(EfoFusion* f, const uint8_t* rgb, const uint16_t* depth, int64_t timestamp,
                                     float weight_multiplier, const double* in_T_wc16, const double* T_override16,
                                     const float* nodes, int n_nodes, int fern_accepted);
void efo_fusion_destroy(EfoFusion* f);
void efo_fusion_process_frame(EfoFusion* f, const uint8_t* rgb, const uint16_t* depth, int64_t timestamp,
                              float weight_multiplier, const double* in_T_wc16);
void efo_fusion_pose(const EfoFusion* f, double* T_wc16);
int efo_fusion_count(const EfoFusion* f);
int efo_fusion_tick(const EfoFusion* f);
const float* efo_fusion_map(const EfoFusion* f);
EfoOdometry* efo_fusion_odometry(EfoFusion* f);
/* which: 0 image4(u8) 1 vertex4 2 normal4 3 time(u16) 4 fill image4 5 fill vertex4 6 fill normal4
 * 7 depth filtered (u16) 8 metric raw 9 metric filtered 10 index (u32) 11 vertConf 12 colorTime 13 normRad */
const void* efo_fusion_buffer(const EfoFusion* f, int which);
/* Optional external tracker backend (used by bench.py --impl reference to drive the REFERENCE's own CUDA tracking
 * kernels from oracle/_ref/libef_ref.so inside this pipeline). All pointers are host memory. */
typedef struct {
  void* handle;
  void (*init_icp_model)(void*, const float* vtx4, const float* nrm4, const double* T_wc16);
  void (*init_rgb_model)(void*, const uint8_t* rgba);
  void (*init_icp_depth)(void*, const uint16_t* depth, float cutoff);
  void (*init_rgb)(void*, const uint8_t* rgba);
  void (*init_first_rgb)(void*, const uint8_t* rgba);
  int (*track)(void*, double* T_wc16, int rgb_only, float icp_weight, int pyramid, int fast_odom, int so3, void* trace,
               int max_trace);
} EfoTrackerBackend;
void efo_fusion_set_tracker(EfoFusion* f, const EfoTrackerBackend* backend);
/* wall-clock seconds spent per stage since creation: preprocess, tracking, mapping(fuse+clean+index), predict */
void efo_fusion_timers(const EfoFusion* f, double* out4);

#ifdef __cplusplus
}
#endif
#endif
