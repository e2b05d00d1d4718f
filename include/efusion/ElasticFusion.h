// Source-level drop-in for the reference's Core/ElasticFusion.h on top of the C ABI of libefusion.so
// (include/efusion_b200.h). A program written against the reference API
//
//     #include <ElasticFusion.h>
//     Resolution::getInstance(640, 480);
//     Intrinsics::getInstance(528, 528, 320, 240);
//     ElasticFusion eFusion;
//     eFusion.processFrame(rgb, depth, timestamp, weightMultiplier);
//     const auto& T = eFusion.get_T_wc();
//
// (reference README.md:74-100, MainController.cpp:178-243) compiles and runs unchanged, minus OpenGL display: there is
// no GL context to create, GPUTexture wraps a CUDA device buffer, and model() returns an opaque handle.
// Relocalisation and global (fern) loop closures are outside this library's scope: the constructor refuses reloc. Local loop
// closures: closeLoops runs the front half on the device; with the trailing deviceLoopClosure = true processFrame also
// samples, solves and applies the deformation graph (ef_create with close_loops = 2).
//
// If <sophus/se3.hpp> is on the include path the pose types are Sophus::SE3d exactly as in the reference; otherwise a
// minimal ef::SE3d with the members the reference API uses (matrix(), translation(), rotationMatrix(), inverse()).
#ifndef EFUSION_B200_ELASTICFUSION_H_
#define EFUSION_B200_ELASTICFUSION_H_

#include <cmath>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <fstream>
#include <iomanip>
#include <map>
#include <memory>
#include <sstream>
#include <string>
#include <utility>
#include <vector>

#include "../efusion_b200.h"
#include "Utils/Intrinsics.h"
#include "Utils/Resolution.h"

#if defined(__has_include)
#if __has_include(<sophus/se3.hpp>)
#include <sophus/se3.hpp>
#define EFUSION_HAVE_SOPHUS 1
#endif
#endif

namespace ef {
#ifndef EFUSION_HAVE_SOPHUS
struct Mat4d {
  double m[16];
  double operator()(int r, int c) const { return m[r * 4 + c]; }
  const double* data() const { return m; }
};
struct Vec3d {
  double v[3];
  double operator()(int i) const { return v[i]; }
  double operator[](int i) const { return v[i]; }
};
struct Mat3d {
  double m[9];
  double operator()(int r, int c) const { return m[r * 3 + c]; }
};
class SE3d {
 public:
  SE3d() {
    for (int i = 0; i < 16; ++i) T_[i] = (i % 5 == 0) ? 1.0 : 0.0;
  }
  explicit SE3d(const double* rowMajor16) {
    for (int i = 0; i < 16; ++i) T_[i] = rowMajor16[i];
  }
  Mat4d matrix() const {
    Mat4d r;
    for (int i = 0; i < 16; ++i) r.m[i] = T_[i];
    return r;
  }
  Vec3d translation() const { return Vec3d{{T_[3], T_[7], T_[11]}}; }
  Mat3d rotationMatrix() const { return Mat3d{{T_[0], T_[1], T_[2], T_[4], T_[5], T_[6], T_[8], T_[9], T_[10]}}; }
  SE3d inverse() const {
    double r[16] = {0};
    for (int i = 0; i < 3; ++i)
      for (int j = 0; j < 3; ++j) r[i * 4 + j] = T_[j * 4 + i];
    for (int i = 0; i < 3; ++i) r[i * 4 + 3] = -(r[i * 4 + 0] * T_[3] + r[i * 4 + 1] * T_[7] + r[i * 4 + 2] * T_[11]);
    r[15] = 1;
    return SE3d(r);
  }
  const double* rowMajor() const { return T_; }

 private:
  double T_[16];
};
inline void toRowMajor(const SE3d& T, double* out) {
  for (int i = 0; i < 16; ++i) out[i] = T.rowMajor()[i];
}
inline SE3d fromRowMajor(const double* in) { return SE3d(in); }
#else
using SE3d = Sophus::SE3d;
inline void toRowMajor(const SE3d& T, double* out) {
  const Eigen::Matrix4d M = T.matrix();
  for (int r = 0; r < 4; ++r)
    for (int c = 0; c < 4; ++c) out[r * 4 + c] = M(r, c);
}
inline SE3d fromRowMajor(const double* in) {
  Eigen::Matrix3d R;
  for (int r = 0; r < 3; ++r)
    for (int c = 0; c < 3; ++c) R(r, c) = in[r * 4 + c];
  SE3d T;
  T.setRotationMatrix(R);
  T.translation() = Eigen::Vector3d(in[3], in[7], in[11]);
  return T;
}
#endif

// The reference prints and exits on CUDA errors (Core/Cuda/convenience.cuh:64-70, with status 0); the wrappers keep the
// print-and-terminate policy but report failure to the parent process (status 1).
inline void check(int rc, const char* what) {
  if (rc != 0) {
    std::fprintf(stderr, "Error: %s: %s\n", ef_error_string(rc), what);
    std::exit(1);
  }
}
}  // namespace ef

// GPUTexture (reference Core/GPUTexture.h): same name and role — a named image the pipeline produces or consumes — but
// backed by a CUDA device buffer of the owning context instead of a GL texture + cudaGraphicsResource.
class GPUTexture {
 public:
  static constexpr const char* RGB = "RGB";
  static constexpr const char* DEPTH_RAW = "DEPTH";
  static constexpr const char* DEPTH_FILTERED = "DEPTH_FILTERED";
  static constexpr const char* DEPTH_METRIC = "DEPTH_METRIC";
  static constexpr const char* DEPTH_METRIC_FILTERED = "DEPTH_METRIC_FILTERED";
  static constexpr const char* DEPTH_NORM = "DEPTH_NORM";
  GPUTexture(EfContext* ctx, int bufferId) : ctx_(ctx), id_(bufferId) {}
  void* devicePtr() const {
    void* p = nullptr;
    size_t n = 0;
    ef::check(ef_buffer(ctx_, id_, 0, &p, &n), "ef_buffer");
    return p;
  }
  size_t bytes() const {
    void* p = nullptr;
    size_t n = 0;
    ef::check(ef_buffer(ctx_, id_, 0, &p, &n), "ef_buffer");
    return n;
  }
  void download(void* host) const { ef::check(ef_download(ctx_, id_, 0, host, bytes()), "ef_download"); }
  int id() const { return id_; }
  EfContext* context() const { return ctx_; }

 private:
  EfContext* ctx_;
  int id_;
};

// RGBDOdometry (reference Core/Utils/RGBDOdometry.h:31-79)
class RGBDOdometry {
 public:
  RGBDOdometry(EfContext* ctx, int which) : ctx_(ctx), which_(which) { refresh(); }
  void initICP(GPUTexture* filteredDepth, const float depthCutoff) {
    ef::check(ef_odom_init_icp_depth(ctx_, which_, (const uint16_t*)filteredDepth->devicePtr(), depthCutoff), "initICP");
  }
  void initICP(GPUTexture* predictedVertices, GPUTexture* predictedNormals) {
    ef::check(ef_odom_init_icp_pred(ctx_, which_, (const float*)predictedVertices->devicePtr(), (const float*)predictedNormals->devicePtr()), "initICP");
  }
  void initICPModel(GPUTexture* predictedVertices, GPUTexture* predictedNormals, const ef::SE3d& T_wc) {
    double T[16];
    ef::toRowMajor(T_wc, T);
    ef::check(ef_odom_init_icp_model(ctx_, which_, (const float*)predictedVertices->devicePtr(), (const float*)predictedNormals->devicePtr(), T),
              "initICPModel");
  }
  void initRGB(GPUTexture* rgb) { ef::check(ef_odom_init_rgb(ctx_, which_, (const uint8_t*)rgb->devicePtr()), "initRGB"); }
  void initRGBModel(GPUTexture* rgb) { ef::check(ef_odom_init_rgb_model(ctx_, which_, (const uint8_t*)rgb->devicePtr()), "initRGBModel"); }
  void initFirstRGB(GPUTexture* rgb) { ef::check(ef_odom_init_first_rgb(ctx_, which_, (const uint8_t*)rgb->devicePtr()), "initFirstRGB"); }
  void getIncrementalTransformation(ef::SE3d& T_wc, const bool& rgbOnly, const float& icpWeight, const bool& pyramid, const bool& fastOdom,
                                    const bool& so3) {
    double T[16];
    ef::toRowMajor(T_wc, T);
    ef::check(ef_odom_track(ctx_, which_, T, rgbOnly, icpWeight, pyramid, fastOdom, so3, nullptr, 0, nullptr), "getIncrementalTransformation");
    T_wc = ef::fromRowMajor(T);
    refresh();
  }
  // lastA.lu().inverse(), row-major 6x6
  std::vector<double> getCovariance() {
    std::vector<double> c(36);
    ef::check(ef_odom_covariance(ctx_, which_, c.data()), "getCovariance");
    return c;
  }
  void refresh() {
    EfOdomStats s;
    if (ef_odom_stats(ctx_, which_, &s) != 0) return;
    lastICPError = s.lastICPError;
    lastICPCount = s.lastICPCount;
    lastRGBError = s.lastRGBError;
    lastRGBCount = s.lastRGBCount;
    lastSO3Error = s.lastSO3Error;
    lastSO3Count = s.lastSO3Count;
    for (int i = 0; i < 36; ++i) lastA[i] = s.lastA[i];
    for (int i = 0; i < 6; ++i) lastb[i] = s.lastb[i];
  }
  float lastICPError = 0, lastICPCount = 0, lastRGBError = 0, lastRGBCount = 0, lastSO3Error = 0, lastSO3Count = 0;
  double lastA[36] = {0}, lastb[6] = {0};

 private:
  EfContext* ctx_;
  int which_;
};

// IndexMap (reference Core/IndexMap.h:33-142)
class IndexMap {
 public:
  enum Prediction { ACTIVE, INACTIVE };
  static const int FACTOR = 1;
  explicit IndexMap(EfContext* ctx)
      : ctx_(ctx), index_(ctx, EF_BUF_INDEX), vertConf_(ctx, EF_BUF_VERT_CONF), colorTime_(ctx, EF_BUF_COLOR_TIME), normalRad_(ctx, EF_BUF_NORM_RAD),
        depth_(ctx, EF_BUF_SYNTH_DEPTH), image_(ctx, EF_BUF_IMAGE), vertex_(ctx, EF_BUF_VERTEX), normal_(ctx, EF_BUF_NORMAL), time_(ctx, EF_BUF_TIME),
        oldImage_(ctx, EF_BUF_OLD_IMAGE), oldVertex_(ctx, EF_BUF_OLD_VERTEX), oldNormal_(ctx, EF_BUF_OLD_NORMAL), oldTime_(ctx, EF_BUF_OLD_TIME) {}
  void predictIndices(const ef::SE3d& T_wc, const int& time, const std::pair<uint32_t, uint32_t>&, const float depthCutoff, const int timeDelta) {
    double T[16];
    ef::toRowMajor(T_wc, T);
    ef::check(ef_map_predict_indices(ctx_, T, time, depthCutoff, timeDelta), "predictIndices");
  }
  void combinedPredict(const ef::SE3d& T_wc, const std::pair<uint32_t, uint32_t>&, const float depthCutoff, const float confThreshold, const int time,
                       const int maxTime, const int timeDelta, Prediction predictionType) {
    double T[16];
    ef::toRowMajor(T_wc, T);
    ef::check(ef_map_raycast(ctx_, T, depthCutoff, confThreshold, time, maxTime, timeDelta, predictionType == ACTIVE ? 0 : 1), "combinedPredict");
  }
  void synthesizeDepth(const ef::SE3d& T_wc, const std::pair<uint32_t, uint32_t>&, const float depthCutoff, const float confThreshold, const int time,
                       const int maxTime, const int timeDelta) {
    double T[16];
    ef::toRowMajor(T_wc, T);
    ef::check(ef_map_raycast(ctx_, T, depthCutoff, confThreshold, time, maxTime, timeDelta, 2), "synthesizeDepth");
  }
  GPUTexture* indexTex() { return &index_; }
  GPUTexture* vertConfTex() { return &vertConf_; }
  GPUTexture* colorTimeTex() { return &colorTime_; }
  GPUTexture* normalRadTex() { return &normalRad_; }
  GPUTexture* depthTex() { return &depth_; }
  GPUTexture* imageTex() { return &image_; }
  GPUTexture* vertexTex() { return &vertex_; }
  GPUTexture* normalTex() { return &normal_; }
  GPUTexture* timeTex() { return &time_; }
  GPUTexture* oldImageTex() { return &oldImage_; }
  GPUTexture* oldVertexTex() { return &oldVertex_; }
  GPUTexture* oldNormalTex() { return &oldNormal_; }
  GPUTexture* oldTimeTex() { return &oldTime_; }

 private:
  EfContext* ctx_;
  GPUTexture index_, vertConf_, colorTime_, normalRad_, depth_, image_, vertex_, normal_, time_, oldImage_, oldVertex_, oldNormal_, oldTime_;
};

// GlobalModel (reference Core/GlobalModel.h:34-89). The surfel map is a device-resident structure of arrays owned by the
// context; model() returns an opaque handle for signature compatibility.
class GlobalModel {
 public:
  explicit GlobalModel(EfContext* ctx) : ctx_(ctx), handle_(0u, 0u) {}
  const std::pair<uint32_t, uint32_t>& model() { return handle_; }
  void fuse(const ef::SE3d& T_wc, const int& time, GPUTexture*, GPUTexture*, GPUTexture*, GPUTexture*, GPUTexture*, GPUTexture*, GPUTexture*,
            const float depthCutoff, const float weighting) {
    double T[16];
    ef::toRowMajor(T_wc, T);
    ef::check(ef_map_fuse(ctx_, T, time, depthCutoff, weighting), "fuse");
  }
  void clean(const ef::SE3d& T_wc, const int& time, GPUTexture*, GPUTexture*, GPUTexture*, GPUTexture*, GPUTexture*, const float confThreshold,
             std::vector<float>& graph, const int timeDelta, const float maxDepth, const bool isFern) {
    double T[16];
    ef::toRowMajor(T_wc, T);
    // graph: 16 floats per node as Deformation::constrain writes them (Core/Deformation.cpp:175-189); the time-stamp refresh of
    // deformed surfels reads IndexMap::depthTex(), i.e. the last synthesizeDepth
    ef::check(ef_map_clean_deform(ctx_, T, time, confThreshold, timeDelta, maxDepth, graph.empty() ? nullptr : graph.data(), (int32_t)(graph.size() / 16),
                                  isFern ? 1 : 0),
              "clean");
  }
  uint32_t lastCount() {
    int32_t n = 0;
    ef::check(ef_map_count(ctx_, &n), "lastCount");
    return (uint32_t)n;
  }
  // 3 x float4 per surfel in the reference Vertex layout (Core/Shaders/Vertex.cpp:22-41); caller delete[]s, as in the
  // reference. (The reference copies from the stale ping-pong half, SURVEY App. A-24; this returns the current map.)
  float* downloadMap() {
    const uint32_t n = lastCount();
    float* out = new float[(size_t)(n ? n : 1) * 12];
    int32_t cnt = 0;
    ef::check(ef_map_download(ctx_, out, (int32_t)n, &cnt), "downloadMap");
    return out;
  }
  // GlobalModel::renderPointCloud (GlobalModel.cpp:286-350) with the reference's arguments, drawn into `rgba` (width * height * 4
  // bytes, RGBA8, row 0 = window y 0, (0,0,0,0) where no surfel is drawn) instead of the bound framebuffer. mvp: column-major
  // float[16], as the MVP uniform receives it. drawPoints (the draw_feedback point program) is outside this library's scope.
  void renderPointCloud(const float* mvp, const float threshold, const bool drawUnstable, const bool drawNormals, const bool drawColors,
                        const bool drawPoints, const bool drawWindow, const bool drawTimes, const int time, const int timeDelta, const int width,
                        const int height, std::vector<uint8_t>& rgba) {
    if (drawPoints) {
      std::fprintf(stderr, "GlobalModel(b200): renderPointCloud with drawPoints (draw_feedback) is outside this library's scope.\n");
      std::exit(1);
    }
    render(mvp, nullptr, threshold, drawUnstable, drawNormals, drawColors, drawWindow, drawTimes, time, timeDelta, false, false, width, height, rgba);
  }
  // The colour pass of GUI::drawFXAA (Tools/GUI.h:273-345): draw_global_surface_phong.frag, lit from the model-view's translation;
  // invertNormals is the GUI's iclnuim flag (signMult = invertNormals ? 1 : -1). mv: column-major float[16].
  void renderPhong(const float* mvp, const float* mv, const float threshold, const int time, const int timeDelta, const bool invertNormals,
                   const bool drawUnstable, const bool drawNormals, const bool drawColors, const bool drawWindow, const bool drawTimes,
                   const int width, const int height, std::vector<uint8_t>& rgba) {
    render(mvp, mv, threshold, drawUnstable, drawNormals, drawColors, drawWindow, drawTimes, time, timeDelta, true, invertNormals, width, height, rgba);
  }

 private:
  void render(const float* mvp, const float* mv, float threshold, bool drawUnstable, bool drawNormals, bool drawColors, bool drawWindow,
              bool drawTimes, int time, int timeDelta, bool phong, bool invertNormals, int width, int height, std::vector<uint8_t>& rgba) {
    EfRenderView v = {};
    v.width = width;
    v.height = height;
    for (int i = 0; i < 16; ++i) {
      v.mvp[i] = mvp[i];
      v.mv[i] = mv ? mv[i] : 0.f;
    }
    v.threshold = threshold;
    v.color_type = drawNormals ? 1 : drawColors ? 2 : drawTimes ? 3 : 0;
    v.unstable = drawUnstable;
    v.draw_window = drawWindow;
    v.time = time;
    v.time_delta = timeDelta;
    v.phong = phong;
    v.sign_mult = invertNormals ? 1.f : -1.f;
    rgba.resize((size_t)(width > 0 ? width : 0) * (height > 0 ? height : 0) * 4);
    ef::check(ef_render_map(ctx_, &v, rgba.data()), phong ? "renderPhong" : "renderPointCloud");
  }

  EfContext* ctx_;
  std::pair<uint32_t, uint32_t> handle_;
};

class ElasticFusion {
 public:
  ElasticFusion(const int timeDelta = 200, const int countThresh = 35000, const float errThresh = 5e-05, const float covThresh = 1e-05,
                const bool closeLoops = true, const bool iclnuim = false, const bool reloc = false, const float photoThresh = 115,
                const float confidence = 10, const float depthCut = 3, const float icpThresh = 10, const bool fastOdom = false,
                const float fernThresh = 0.3095, const bool so3 = true, const bool frameToFrameRGB = false, const std::string fileName = "",
                const int surfelCapacity = 3072 * 3072, const int device = 0, const bool deviceLoopClosure = false)
      : saveFilename(fileName), iclnuim_(iclnuim), confidenceThreshold_(confidence), maxDepthProcessed_(20.0f), timeDelta_(timeDelta),
        deviceLoopClosure_(closeLoops && deviceLoopClosure) {
    if (reloc) {
      std::fprintf(stderr,
                   "ElasticFusion(b200): relocalisation (Ferns) is outside this library's scope; construct with reloc=false.\n");
      std::exit(1);
    }
    if (closeLoops && !deviceLoopClosure_)
      std::fprintf(stderr,
                   "ElasticFusion(b200): closeLoops=true runs the LOCAL loop closure front half on the device every frame (registration of "
                   "the active against the inactive model view, acceptance test, constraint sampling: getLocalLoopClosure()); the "
                   "deformation solve (Deformation::constrain) and Ferns are not part of this library, so the map stays open-loop unless "
                   "the caller feeds processFrameEnd() a graph, or deviceLoopClosure=true lets processFrame() close local loops itself.\n");
    EfConfig cfg;
    ef_default_config(&cfg, Resolution::getInstance().width(), Resolution::getInstance().height(), Intrinsics::getInstance().fx(),
                      Intrinsics::getInstance().fy(), Intrinsics::getInstance().cx(), Intrinsics::getInstance().cy());
    cfg.time_delta = timeDelta;
    cfg.count_thresh = countThresh;
    cfg.err_thresh = errThresh;
    cfg.cov_thresh = covThresh;
    cfg.close_loops = deviceLoopClosure_ ? 2 : closeLoops ? 1 : 0;  // 2: sample, solve and apply the deformation graph in the frame
    cfg.iclnuim = iclnuim;
    cfg.photo_thresh = photoThresh;
    cfg.confidence = confidence;
    cfg.depth_cutoff = depthCut;
    cfg.icp_weight = icpThresh;
    cfg.fast_odom = fastOdom;
    cfg.fern_thresh = fernThresh;
    cfg.so3 = so3;
    cfg.frame_to_frame_rgb = frameToFrameRGB;
    cfg.capacity = surfelCapacity;
    cfg.device = device;
    ef::check(ef_create(&cfg, nullptr, &ctx_), "ef_create");
    indexMap_.reset(new IndexMap(ctx_));
    globalModel_.reset(new GlobalModel(ctx_));
    frameToModel_.reset(new RGBDOdometry(ctx_, 0));
    modelToModel_.reset(new RGBDOdometry(ctx_, 1));
    textures_[GPUTexture::RGB] = new GPUTexture(ctx_, EF_BUF_RGBA);
    textures_[GPUTexture::DEPTH_RAW] = new GPUTexture(ctx_, EF_BUF_DEPTH_RAW);
    textures_[GPUTexture::DEPTH_FILTERED] = new GPUTexture(ctx_, EF_BUF_DEPTH_FILTERED);
    textures_[GPUTexture::DEPTH_METRIC] = new GPUTexture(ctx_, EF_BUF_DEPTH_METRIC);
    textures_[GPUTexture::DEPTH_METRIC_FILTERED] = new GPUTexture(ctx_, EF_BUF_DEPTH_METRIC_FILTERED);
    std::ofstream file((fileName + ".freiburg").c_str(), std::fstream::out);  // truncated at start, as the reference does
  }

  virtual ~ElasticFusion() {
    if (iclnuim_) savePly();
    // pose log in TUM format `t x y z qx qy qz qw` (reference Core/ElasticFusion.cpp:107-139)
    std::ofstream f((saveFilename + ".freiburg").c_str(), std::fstream::out);
    for (size_t i = 0; i < poseLog_.size(); i++) {
      std::stringstream strs;
      if (iclnuim_)
        strs << std::setprecision(6) << std::fixed << (double)poseLogTimes_[i] << " ";
      else
        strs << std::setprecision(6) << std::fixed << (double)poseLogTimes_[i] / 1000000.0 << " ";
      const double* T = poseLog_[i].data();
      double q[4];
      rotToQuat(T, q);
      f << strs.str() << T[3] << " " << T[7] << " " << T[11] << " " << q[0] << " " << q[1] << " " << q[2] << " " << q[3] << "\n";
    }
    f.close();
    for (auto& kv : textures_) delete kv.second;
    ef_destroy(ctx_);
  }

  // Reference signature (Core/ElasticFusion.h:62-75) plus an optional look-ahead: when the caller already holds the NEXT
  // frame (a log reader does), passing it as nextRgb / nextDepth stages its upload, depth preprocess and pyramids on a side
  // stream while this frame is tracked and fused (ef_prefetch_frame). The next call must then be for that frame (its
  // rgb / depth arguments are not read again). Results are identical with or without look-ahead.
  void processFrame(const uint8_t* rgb, const uint16_t* depth, const int64_t& timestamp, const float weightMultiplier,
                    const ef::SE3d* in_T_wc = 0, const uint8_t* nextRgb = 0, const uint16_t* nextDepth = 0) {
    double T[16];
    if (in_T_wc) ef::toRowMajor(*in_T_wc, T);
    if (!staged_ && !(nextRgb && nextDepth)) {
      ef::check(ef_process_frame(ctx_, rgb, depth, timestamp, weightMultiplier, in_T_wc ? T : nullptr), "processFrame");
    } else {
      if (!staged_) ef::check(ef_prefetch_frame(ctx_, rgb, depth), "processFrame (stage)");
      ef::check(ef_process_frame_device(ctx_, nullptr, nullptr, timestamp, weightMultiplier, in_T_wc ? T : nullptr), "processFrame");
      staged_ = false;
      if (nextRgb && nextDepth) {
        ef::check(ef_prefetch_frame(ctx_, nextRgb, nextDepth), "processFrame (look-ahead)");
        staged_ = true;
      }
      ef::check(ef_finish_frame(ctx_), "processFrame (finish)");
    }
    ef::check(ef_get_pose(ctx_, T), "get_T_wc");
    T_wc_curr_ = ef::fromRowMajor(T);
    poseLog_.emplace_back(T, T + 16);
    poseLogTimes_.push_back((uint64_t)timestamp);
    frameToModel_->refresh();
  }
  void predict() { ef::check(ef_predict(ctx_), "predict"); }

  // Additions for closed-loop hosts. The reference runs its CPU deformation solver in the middle of processFrame
  // (Core/ElasticFusion.cpp:505-526); a host that owns that solver splits the frame instead:
  //   processFrameBegin(...); c = getLocalLoopClosure(); <Deformation::constrain on c> ; processFrameEnd(&T_wc_est, graph, n)
  struct LocalLoopClosure {
    bool ran = false, accepted = false;
    float lastICPError = 0, lastICPCount = 0;
    double covDiag[6] = {0, 0, 0, 0, 0, 0};
    ef::SE3d T_wc_est;
    std::vector<double> src, dst;  // 3 per constraint: vert_w_curr, vert_w_est (ElasticFusion.cpp:493-503)
    std::vector<int> times;        // the INACTIVE view's time stamp of each constraint
  };
  void processFrameBegin(const uint8_t* rgb, const uint16_t* depth, const int64_t& timestamp, const float weightMultiplier,
                         const ef::SE3d* in_T_wc = 0) {
    double T[16];
    if (in_T_wc) ef::toRowMajor(*in_T_wc, T);
    ef::check(ef_process_frame_begin(ctx_, rgb, depth, timestamp, weightMultiplier, in_T_wc ? T : nullptr), "processFrameBegin");
    pendingTimestamp_ = timestamp;
  }
  void processFrameEnd(const ef::SE3d* T_wc_override = 0, const float* graphNodes16 = 0, int numNodes = 0, bool fernAccepted = false) {
    double T[16];
    if (T_wc_override) ef::toRowMajor(*T_wc_override, T);
    ef::check(ef_process_frame_end(ctx_, T_wc_override ? T : nullptr, graphNodes16, numNodes, fernAccepted ? 1 : 0), "processFrameEnd");
    ef::check(ef_get_pose(ctx_, T), "get_T_wc");
    T_wc_curr_ = ef::fromRowMajor(T);
    poseLog_.emplace_back(T, T + 16);
    poseLogTimes_.push_back((uint64_t)pendingTimestamp_);
    frameToModel_->refresh();
  }
  LocalLoopClosure getLocalLoopClosure() {
    LocalLoopClosure c;
    EfLoopResult r;
    const int cap = (Resolution::getInstance().width() / 20) * (Resolution::getInstance().height() / 20);
    c.src.resize((size_t)cap * 3);
    c.dst.resize((size_t)cap * 3);
    c.times.resize((size_t)cap);
    int32_t n = 0;
    ef::check(ef_local_loop_result(ctx_, &r, c.src.data(), c.dst.data(), c.times.data(), cap, &n), "getLocalLoopClosure");
    c.ran = r.ran != 0;
    c.accepted = r.accepted != 0;
    c.lastICPError = r.lastICPError;
    c.lastICPCount = r.lastICPCount;
    for (int i = 0; i < 6; ++i) c.covDiag[i] = r.cov_diag[i];
    c.T_wc_est = ef::fromRowMajor(r.T_wc_est);
    c.src.resize((size_t)n * 3);
    c.dst.resize((size_t)n * 3);
    c.times.resize((size_t)n);
    return c;
  }

  IndexMap& getIndexMap() { return *indexMap_; }
  GlobalModel& getGlobalModel() { return *globalModel_; }
  std::map<std::string, GPUTexture*>& getTextures() { return textures_; }
  const RGBDOdometry& getModelToModel() { return *modelToModel_; }
  RGBDOdometry& getFrameToModel() { return *frameToModel_; }
  const float& getConfidenceThreshold() { return confidenceThreshold_; }
  void setRgbOnly(const bool& val) { ef::check(ef_set_rgb_only(ctx_, val), "setRgbOnly"); }
  void setIcpWeight(const float& val) { ef::check(ef_set_icp_weight(ctx_, val), "setIcpWeight"); }
  void setPyramid(const bool& val) { ef::check(ef_set_pyramid(ctx_, val), "setPyramid"); }
  void setFastOdom(const bool& val) { ef::check(ef_set_fast_odom(ctx_, val), "setFastOdom"); }
  void setSo3(const bool& val) { ef::check(ef_set_so3(ctx_, val), "setSo3"); }
  void setFrameToFrameRGB(const bool& val) { ef::check(ef_set_frame_to_frame_rgb(ctx_, val), "setFrameToFrameRGB"); }
  void setConfidenceThreshold(const float& val) {
    confidenceThreshold_ = val;
    ef::check(ef_set_confidence_threshold(ctx_, val), "setConfidenceThreshold");
  }
  void setFernThresh(const float&) {}  // ferns are out of scope; kept for source compatibility
  void setDepthCutoff(const float& val) { ef::check(ef_set_depth_cutoff(ctx_, val), "setDepthCutoff"); }
  const bool& getLost() { return lost_; }
  const int& getTick() {
    int32_t t = 0;
    ef::check(ef_get_tick(ctx_, &t), "getTick");
    tick_ = t;
    return tick_;
  }
  const int& getTimeDelta() { return timeDelta_; }
  void setTick(const int& val) { ef::check(ef_set_tick(ctx_, val), "setTick"); }
  const float& getMaxDepthProcessed() { return maxDepthProcessed_; }
  const ef::SE3d& get_T_wc() { return T_wc_curr_; }
  // local loop closures applied so far; they happen inside processFrame only with deviceLoopClosure
  const int& getDeforms() {
    if (deviceLoopClosure_) {
      EfLocalDeform d;
      ef::check(ef_local_deform_result(ctx_, &d, nullptr, 0, nullptr), "getDeforms");
      deforms_ = d.deforms;
    }
    return deforms_;
  }
  const int& getFernDeforms() { return zero_; }

  // binary little-endian PLY, x y z r g b nx ny nz radius, normals negated, only surfels above the confidence threshold
  // (reference Core/ElasticFusion.cpp:684-781)
  void savePly() {
    const std::string filename = saveFilename + ".ply";
    float* mapData = globalModel_->downloadMap();
    const uint32_t count = globalModel_->lastCount();
    int validCount = 0;
    for (uint32_t i = 0; i < count; i++)
      if (mapData[i * 12 + 3] > confidenceThreshold_) validCount++;
    std::ofstream fs(filename.c_str());
    fs << "ply\nformat binary_little_endian 1.0\nelement vertex " << validCount
       << "\nproperty float x\nproperty float y\nproperty float z\nproperty uchar red\nproperty uchar green\nproperty uchar blue"
          "\nproperty float nx\nproperty float ny\nproperty float nz\nproperty float radius\nend_header\n";
    fs.close();
    std::ofstream fpout(filename.c_str(), std::ios::app | std::ios::binary);
    for (uint32_t i = 0; i < count; i++) {
      const float* s = mapData + (size_t)i * 12;
      if (s[3] > confidenceThreshold_) {
        fpout.write(reinterpret_cast<const char*>(s), 12);
        const int c = (int)s[4];
        unsigned char rgb[3] = {(unsigned char)(c >> 16 & 0xFF), (unsigned char)(c >> 8 & 0xFF), (unsigned char)(c & 0xFF)};
        fpout.write(reinterpret_cast<const char*>(rgb), 3);
        const float n[4] = {-s[8], -s[9], -s[10], s[11]};
        fpout.write(reinterpret_cast<const char*>(n), 16);
      }
    }
    fpout.close();
    delete[] mapData;
  }

  EfContext* context() { return ctx_; }

 private:
  static void rotToQuat(const double* T, double* q) {  // Eigen::Quaterniond(rot): x y z w
    const double m00 = T[0], m01 = T[1], m02 = T[2], m10 = T[4], m11 = T[5], m12 = T[6], m20 = T[8], m21 = T[9], m22 = T[10];
    const double tr = m00 + m11 + m22;
    double w, x, y, z;
    if (tr > 0) {
      double s = std::sqrt(tr + 1.0) * 2;
      w = 0.25 * s;
      x = (m21 - m12) / s;
      y = (m02 - m20) / s;
      z = (m10 - m01) / s;
    } else if (m00 > m11 && m00 > m22) {
      double s = std::sqrt(1.0 + m00 - m11 - m22) * 2;
      w = (m21 - m12) / s;
      x = 0.25 * s;
      y = (m01 + m10) / s;
      z = (m02 + m20) / s;
    } else if (m11 > m22) {
      double s = std::sqrt(1.0 + m11 - m00 - m22) * 2;
      w = (m02 - m20) / s;
      x = (m01 + m10) / s;
      y = 0.25 * s;
      z = (m12 + m21) / s;
    } else {
      double s = std::sqrt(1.0 + m22 - m00 - m11) * 2;
      w = (m10 - m01) / s;
      x = (m02 + m20) / s;
      y = (m12 + m21) / s;
      z = 0.25 * s;
    }
    q[0] = x;
    q[1] = y;
    q[2] = z;
    q[3] = w;
  }

  EfContext* ctx_ = nullptr;
  std::unique_ptr<IndexMap> indexMap_;
  std::unique_ptr<GlobalModel> globalModel_;
  std::unique_ptr<RGBDOdometry> frameToModel_, modelToModel_;
  std::map<std::string, GPUTexture*> textures_;
  const std::string saveFilename;
  ef::SE3d T_wc_curr_;
  std::vector<std::vector<double>> poseLog_;
  std::vector<uint64_t> poseLogTimes_;
  bool iclnuim_;
  float confidenceThreshold_;
  float maxDepthProcessed_;
  int timeDelta_;
  int tick_ = 1;
  int zero_ = 0;
  int deforms_ = 0;
  const bool deviceLoopClosure_;  // close_loops = 2
  bool lost_ = false;
  bool staged_ = false;  // a look-ahead frame is waiting in the library (ef_prefetch_frame)
  int64_t pendingTimestamp_ = 0;
};

#endif  // EFUSION_B200_ELASTICFUSION_H_
