// Headless ElasticFusion driver on libefusion.so: the reference application's command line (MainController.cpp:32-104,
// README.md:40-72) without the GUI, sensors or Pangolin. It reads a .klg log (raw, zlib depth, JPEG colour), runs
// ElasticFusion::processFrame over it and leaves <log>.freiburg (always) and <log>.ply (-icl or -ply) behind, like the
// reference's destructor / "save" button do.
//
//   -cal <file>  calibration: one line "fx fy cx cy"            -l <log.klg>   (required: no live cameras here)
//   -p <poses>   ground-truth poses to use instead of tracking   -c -d -i -ie -cv -pt -ft -t -ic -s -e   as the reference
//   -icl  -o  -rl(refused)  -fs  -q(implied)  -fo  -nso  -f  -ftf  -r(ignored: nothing to watch)
// additions: -w <width> -h <height> (default 640 480), -cap <surfels>, -dev <cuda device>, -ply (write the map at the end),
//            -nola (no frame look-ahead), -v (per-frame line), -dlc (without -o: close local loops inside processFrame, i.e.
//            sample, solve and apply the deformation graph on the device; prints the number of closures applied),
//            -render N (every N frames and after the last one, write <log>.render.<tick>.ppm: the map drawn as the reference's viewer
//            draws it -- GlobalModel::renderPointCloud -- from the tracked pose at the input intrinsics and resolution, so it lines up
//            with the input image), -rt T (its colour type: 0 grey, 1 normals, 2 colours (default), 3 times)
#include <ElasticFusion.h>
#include <Tools/RawLogReader.h>

#include <chrono>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <fstream>
#include <limits>
#include <map>
#include <string>

namespace {

// <log>.render.<tick>.ppm: the map from the current pose, as GlobalModel::renderPointCloud draws it (stable surfels only)
void writeRender(ElasticFusion& eFusion, const std::string& logFile, int colorType, float confidence, int timeDelta) {
  const int w = Resolution::getInstance().width(), h = Resolution::getInstance().height();
  const Intrinsics& K = Intrinsics::getInstance();
  double T[16];
  ef::toRowMajor(eFusion.get_T_wc(), T);
  float mvp[16], mv[16];
  ef::check(ef_render_camera(T, K.fx(), K.fy(), K.cx(), K.cy(), w, h, 0.1f, 1000.0f, mvp, mv), "render camera");
  std::vector<uint8_t> rgba;
  eFusion.getGlobalModel().renderPointCloud(mvp, confidence, false, colorType == 1, colorType == 2, false, false, colorType == 3,
                                            eFusion.getTick(), timeDelta, w, h, rgba);
  const std::string path = logFile + ".render." + std::to_string(eFusion.getTick()) + ".ppm";
  std::ofstream f(path, std::ios::binary);
  f << "P6\n" << w << " " << h << "\n255\n";
  for (size_t p = 0; p < (size_t)w * h; ++p) f.write(reinterpret_cast<const char*>(&rgba[p * 4]), 3);  // row 0 = the image's top row
}

int findArg(int argc, char** argv, const char* name) {
  for (int i = 1; i < argc; ++i)
    if (std::strcmp(argv[i], name) == 0) return i;
  return -1;
}
template <typename T>
void getArg(int argc, char** argv, const char* name, T& v);
template <>
void getArg<std::string>(int argc, char** argv, const char* name, std::string& v) {
  const int i = findArg(argc, argv, name);
  if (i > 0 && i + 1 < argc) v = argv[i + 1];
}
template <>
void getArg<float>(int argc, char** argv, const char* name, float& v) {
  const int i = findArg(argc, argv, name);
  if (i > 0 && i + 1 < argc) v = (float)std::atof(argv[i + 1]);
}
template <>
void getArg<int>(int argc, char** argv, const char* name, int& v) {
  const int i = findArg(argc, argv, name);
  if (i > 0 && i + 1 < argc) v = std::atoi(argv[i + 1]);
}

// Tools/GroundTruthOdometry.cpp:28-88: "utime,x,y,z,qx,qy,qz,qw" lines in the iSAM basis; the first query defines the origin
class GroundTruthOdometry {
 public:
  explicit GroundTruthOdometry(const std::string& file) {
    std::ifstream f(file.c_str());
    std::string line;
    while (std::getline(f, line)) {
      unsigned long long t;
      float x, y, z, qx, qy, qz, qw;
      if (std::sscanf(line.c_str(), "%llu,%f,%f,%f,%f,%f,%f,%f", &t, &x, &y, &z, &qx, &qy, &qz, &qw) != 8) continue;
      Pose p;
      const float n = std::sqrt(qx * qx + qy * qy + qz * qz + qw * qw);
      qx /= n, qy /= n, qz /= n, qw /= n;
      const float R[9] = {1 - 2 * (qy * qy + qz * qz), 2 * (qx * qy - qz * qw),     2 * (qx * qz + qy * qw),
                          2 * (qx * qy + qz * qw),     1 - 2 * (qx * qx + qz * qz), 2 * (qy * qz - qx * qw),
                          2 * (qx * qz - qy * qw),     2 * (qy * qz + qx * qw),     1 - 2 * (qx * qx + qy * qy)};
      for (int r = 0; r < 3; ++r) {
        for (int c = 0; c < 3; ++c) p.m[r * 4 + c] = R[r * 3 + c];
        p.m[r * 4 + 3] = r == 0 ? x : (r == 1 ? y : z);
      }
      traj_[t] = p;
    }
  }
  bool ok() const { return !traj_.empty(); }
  // pose = M^-1 * T(timestamp) * M with the basis change M of the reference; identity for the first frame
  bool get(uint64_t ts, double* T16) {
    for (int k = 0; k < 16; ++k) T16[k] = (k % 5 == 0) ? 1.0 : 0.0;
    auto it = traj_.find(ts);
    if (it == traj_.end()) return first_ ? false : true;
    if (first_) {
      first_ = false;
      return true;
    }
    static const float M[16] = {0, 0, 1, 0, -1, 0, 0, 0, 0, -1, 0, 0, 0, 0, 0, 1};
    static const float Mi[16] = {0, -1, 0, 0, 0, 0, -1, 0, 1, 0, 0, 0, 0, 0, 0, 1};
    float a[16], b[16];
    mul(Mi, it->second.m, a);
    mul(a, M, b);
    for (int k = 0; k < 16; ++k) T16[k] = b[k];
    return true;
  }

 private:
  struct Pose {
    float m[16] = {1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1};
  };
  static void mul(const float* a, const float* b, float* c) {
    for (int i = 0; i < 4; ++i)
      for (int j = 0; j < 4; ++j) {
        float s = 0;
        for (int k = 0; k < 4; ++k) s += a[i * 4 + k] * b[k * 4 + j];
        c[i * 4 + j] = s;
      }
  }
  std::map<uint64_t, Pose> traj_;
  bool first_ = true;
};

}  // namespace

int main(int argc, char** argv) {
  std::string logFile, calibrationFile, poseFile;
  getArg(argc, argv, "-l", logFile);
  if (logFile.empty() || findArg(argc, argv, "--help") > 0) {
    std::fprintf(stderr, "usage: %s -l <log.klg> [-cal <file>] [-w W -h H] [-o] [-icl] [-fo] [-nso] [-f] [-ftf] [-c conf] [-d depth] [-i icp] "
                         "[-t timeDelta] [-s start] [-e end] [-p poses] [-cap surfels] [-dev n] [-ply] [-nola] [-v] [-dlc] [-render N] [-rt T]\n", argv[0]);
    return 2;
  }
  int width = 640, height = 480;
  getArg(argc, argv, "-w", width);
  getArg(argc, argv, "-h", height);
  Resolution::getInstance(width, height);
  getArg(argc, argv, "-cal", calibrationFile);
  if (!calibrationFile.empty()) {
    std::ifstream f(calibrationFile.c_str());
    std::string line;
    std::getline(f, line);
    double fx, fy, cx, cy;
    if (std::sscanf(line.c_str(), "%lg %lg %lg %lg", &fx, &fy, &cx, &cy) != 4) {
      std::fprintf(stderr, "Ooops, your calibration file should contain a single line with fx fy cx cy!\n");
      return 1;
    }
    Intrinsics::getInstance((float)fx, (float)fy, (float)cx, (float)cy);
  } else {
    Intrinsics::getInstance(528.f * width / 640.f, 528.f * height / 480.f, 320.f * width / 640.f, 240.f * height / 480.f);
  }
  const bool iclnuim = findArg(argc, argv, "-icl") > 0, flip = findArg(argc, argv, "-f") > 0;
  float confidence = 10.0f, depth = 3.0f, icp = 10.0f, icpErrThresh = 4e-05f, covThresh = 1e-05f, photoThresh = 115, fernThresh = 0.3095f;
  int timeDelta = 200, icpCountThresh = 40000, start = 1, end = std::numeric_limits<uint16_t>::max();
  int capacity = 3072 * 3072, device = 0;
  getArg(argc, argv, "-c", confidence);
  getArg(argc, argv, "-d", depth);
  getArg(argc, argv, "-i", icp);
  getArg(argc, argv, "-ie", icpErrThresh);
  getArg(argc, argv, "-cv", covThresh);
  getArg(argc, argv, "-pt", photoThresh);
  getArg(argc, argv, "-ft", fernThresh);
  getArg(argc, argv, "-t", timeDelta);
  getArg(argc, argv, "-ic", icpCountThresh);
  getArg(argc, argv, "-s", start);
  getArg(argc, argv, "-e", end);
  getArg(argc, argv, "-cap", capacity);
  getArg(argc, argv, "-dev", device);
  getArg(argc, argv, "-p", poseFile);
  GroundTruthOdometry* gt = poseFile.empty() ? nullptr : new GroundTruthOdometry(poseFile);
  if (gt && !gt->ok()) {
    std::fprintf(stderr, "no poses in %s\n", poseFile.c_str());
    return 1;
  }
  const bool openLoop = !gt && findArg(argc, argv, "-o") > 0;
  const bool reloc = findArg(argc, argv, "-rl") > 0, frameskip = findArg(argc, argv, "-fs") > 0, fastOdom = findArg(argc, argv, "-fo") > 0;
  const bool so3 = !(findArg(argc, argv, "-nso") > 0), frameToFrameRGB = findArg(argc, argv, "-ftf") > 0;
  const bool lookahead = !(findArg(argc, argv, "-nola") > 0) && !frameskip, verbose = findArg(argc, argv, "-v") > 0;
  const bool deviceLoopClosure = !openLoop && findArg(argc, argv, "-dlc") > 0;
  int renderEvery = 0, renderType = 2;
  getArg(argc, argv, "-render", renderEvery);
  getArg(argc, argv, "-rt", renderType);
  if (renderType < 0 || renderType > 3) {
    std::fprintf(stderr, "-rt: colour type 0..3\n");
    return 1;
  }
  const int renderTimeDelta = openLoop ? std::numeric_limits<int>::max() / 2 : timeDelta;
  int lastRendered = -1;

  RawLogReader reader(logFile, flip);
  ElasticFusion eFusion(openLoop ? std::numeric_limits<int>::max() / 2 : timeDelta, icpCountThresh, icpErrThresh, covThresh, !openLoop, iclnuim, reloc,
                        photoThresh, confidence, depth, icp, fastOdom, fernThresh, so3, frameToFrameRGB, reader.getFile(), capacity, device,
                        deviceLoopClosure);
  int framesToSkip = 0, processed = 0;
  const auto t0 = std::chrono::steady_clock::now();
  while (reader.hasMore() && eFusion.getTick() < end) {
    reader.getNext();
    if (eFusion.getTick() < start) {
      eFusion.setTick(start);
      reader.fastForward(start);
    }
    const float weightMultiplier = (float)(framesToSkip + 1);
    if (framesToSkip > 0) {
      eFusion.setTick(eFusion.getTick() + framesToSkip);
      reader.fastForward(reader.currentFrame + framesToSkip);
      framesToSkip = 0;
    }
    double T[16];
    ef::SE3d T_in;
    const bool havePose = gt && gt->get((uint64_t)reader.timestamp, T);
    if (havePose) T_in = ef::fromRowMajor(T);
    const auto f0 = std::chrono::steady_clock::now();
    if (lookahead && !havePose && !gt && reader.peekNext())
      eFusion.processFrame(reader.rgb, reader.depth, reader.timestamp, weightMultiplier, nullptr, reader.nextRgb(), reader.nextDepth());
    else
      eFusion.processFrame(reader.rgb, reader.depth, reader.timestamp, weightMultiplier, havePose ? &T_in : nullptr);
    const double ms = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - f0).count();
    if (frameskip && ms > 1000.0 / 30.0) framesToSkip = (int)(ms / (1000.0 / 30.0));
    ++processed;
    if (verbose) {
      const auto M = eFusion.get_T_wc().matrix();
      std::printf("frame %d tick %d t %.4f %.4f %.4f surfels %u %.3f ms\n", reader.currentFrame, eFusion.getTick(), (double)M(0, 3), (double)M(1, 3),
                  (double)M(2, 3), eFusion.getGlobalModel().lastCount(), ms);
    }
    if (renderEvery > 0 && processed % renderEvery == 0) {
      writeRender(eFusion, logFile, renderType, confidence, renderTimeDelta);
      lastRendered = processed;
    }
  }
  if (renderEvery > 0 && processed > 0 && lastRendered != processed) writeRender(eFusion, logFile, renderType, confidence, renderTimeDelta);
  const double s = std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
  std::printf("%d frames in %.3f s (%.1f frames/s incl. log decode), %u surfels, tick %d\n", processed, s, processed / (s > 0 ? s : 1),
              eFusion.getGlobalModel().lastCount(), eFusion.getTick());
  if (deviceLoopClosure) std::printf("deforms %d\n", eFusion.getDeforms());
  if (findArg(argc, argv, "-ply") > 0 && !iclnuim) eFusion.savePly();
  delete gt;
  return 0;  // ~ElasticFusion writes <log>.freiburg (and <log>.ply with -icl)
}
