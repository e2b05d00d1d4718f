// TEST INFRASTRUCTURE ONLY — harness around the REFERENCE's own CUDA tracking half.
//
// Built by oracle/Makefile (target `ref`) together with the reference's Core/Cuda/reduce.cu, cudafuncs.cu and
// containers/device_memory.cpp, compiled UNMODIFIED from the reference tree for sm_90a, into oracle/_ref/libef_ref.so.
// Purpose: (1) pin the CPU oracle against the real reference kernels on the GPU box, (2) time the reference's
// tracking path exactly as the reference drives it (two launches + cudaDeviceSynchronize + blocking D2H per step).
//
// The class below re-implements the HOST side of Core/Utils/RGBDOdometry.cpp:22-575 (that file itself cannot be
// compiled here: it includes GPUTexture.h -> Pangolin -> OpenGL) on top of the reference's free functions declared
// in Core/Cuda/cudafuncs.cuh:61-169, using the reference's vendored Eigen for the same host math. GL textures are
// replaced by cudaArrays filled from host memory; everything else goes through the reference code paths.
#include <cuda_runtime.h>

#include <Eigen/Core>
#include <Eigen/Dense>
#include <chrono>
#include <cstdio>
#include <cstring>
#include <limits>
#include <vector>

#include "cudafuncs.cuh"

namespace {

using M3f = Eigen::Matrix<float, 3, 3, Eigen::RowMajor>;
using M3d = Eigen::Matrix<double, 3, 3, Eigen::RowMajor>;
using M4d = Eigen::Matrix<double, 4, 4, Eigen::RowMajor>;
using M6f = Eigen::Matrix<float, 6, 6, Eigen::RowMajor>;
using M6d = Eigen::Matrix<double, 6, 6, Eigen::RowMajor>;
using V6f = Eigen::Matrix<float, 6, 1>;
using V6d = Eigen::Matrix<double, 6, 1>;

struct Trace {  // same layout as EfoTrace / EfSolveTrace
  int32_t kind, level, iter, rgb_count, rgb_sigma;
  float sigma_val;
  float A_icp[36], b_icp[6], icp_residual[2];
  float A_rgb[36], b_rgb[6];
  float A_so3[9], b_so3[3], so3_residual[2];
  double lastA[36], lastb[6], result[6];
};

constexpr int NP = 3;

mat33 to_mat33(const M3f& e) {  // types.cuh only offers this constructor to non-nvcc translation units
  mat33 m;
  memcpy(m.data, e.data(), sizeof(mat33));
  return m;
}

M3d rodrigues(const Eigen::Vector3d& w) {  // OdometryProvider::rodrigues semantics
  M3d R = M3d::Identity();
  const double th = w.norm();
  if (th >= std::numeric_limits<double>::epsilon()) {
    const Eigen::Vector3d k = w / th;
    M3d Kx;
    Kx << 0, -k.z(), k.y(), k.z(), 0, -k.x(), -k.y(), k.x(), 0;
    R = std::cos(th) * M3d::Identity() + (1.0 - std::cos(th)) * (k * k.transpose()) + std::sin(th) * Kx;
  }
  return R;
}

struct RefOdom {
  int W, H;
  CameraModel intr;
  float distThres, angleThres, sobelScale, maxDepthDeltaRGB, maxDepthRGB;
  float minGrad[NP];
  std::vector<DeviceArray2D<uint16_t>> depth_tmp;
  DeviceArray<float> vmaps_tmp;
  std::vector<DeviceArray2D<float>> vmaps_g_prev, nmaps_g_prev, vmaps_curr, nmaps_curr;
  DeviceArray2D<float> lastDepth[NP], nextDepth[NP];
  DeviceArray2D<uint8_t> lastImage[NP], nextImage[NP], lastNextImage[NP];
  DeviceArray2D<int16_t> dIdx[NP], dIdy[NP];
  DeviceArray2D<DataTerm> corres[NP];
  DeviceArray2D<float3> clouds[NP];
  DeviceArray<JtJJtrSE3> sumSE3, outSE3;
  DeviceArray<JtJJtrSO3> sumSO3, outSO3;
  DeviceArray<int2> sumRes;
  cudaArray_t arrV = nullptr, arrN = nullptr, arrC = nullptr;
  float stats[6] = {0, 0, 0, 0, 0, 0};
  M6d lastA = M6d::Zero();
  V6d lastb = V6d::Zero();
  double t_init = 0, t_track = 0;  // accumulated wall seconds

  RefOdom(int w, int h, float cx, float cy, float fx, float fy) : W(w), H(h), intr(fx, fy, cx, cy) {
    distThres = 0.10f;
    angleThres = sinf(20.f * 3.14159254f / 180.f);
    sobelScale = (float)(1.0 / pow(2.0, 3));
    maxDepthDeltaRGB = 0.07f;
    maxDepthRGB = 6.0f;
    minGrad[0] = 5;
    minGrad[1] = 3;
    minGrad[2] = 1;
    depth_tmp.resize(NP);
    vmaps_g_prev.resize(NP);
    nmaps_g_prev.resize(NP);
    vmaps_curr.resize(NP);
    nmaps_curr.resize(NP);
    for (int i = 0; i < NP; ++i) {
      const int r = h >> i, c = w >> i;
      depth_tmp[i].create(r, c);
      vmaps_g_prev[i].create(r * 3, c);
      nmaps_g_prev[i].create(r * 3, c);
      vmaps_curr[i].create(r * 3, c);
      nmaps_curr[i].create(r * 3, c);
      lastDepth[i].create(r, c);
      nextDepth[i].create(r, c);
      lastImage[i].create(r, c);
      nextImage[i].create(r, c);
      lastNextImage[i].create(r, c);
      dIdx[i].create(r, c);
      dIdy[i].create(r, c);
      corres[i].create(r, c);
      clouds[i].create(r, c);
      // the reference leaves these uninitialised; NaN-fill the maps so stale y/z reads are defined (SURVEY App. A-6)
      cudaMemset2D(vmaps_g_prev[i].ptr(), vmaps_g_prev[i].step(), 0xff, c * sizeof(float), r * 3);
      cudaMemset2D(nmaps_g_prev[i].ptr(), nmaps_g_prev[i].step(), 0xff, c * sizeof(float), r * 3);
      cudaMemset2D(vmaps_curr[i].ptr(), vmaps_curr[i].step(), 0xff, c * sizeof(float), r * 3);
      cudaMemset2D(nmaps_curr[i].ptr(), nmaps_curr[i].step(), 0xff, c * sizeof(float), r * 3);
      cudaMemset2D(lastNextImage[i].ptr(), lastNextImage[i].step(), 0, c, r);
    }
    vmaps_tmp.create((size_t)h * 4 * w);
    sumSE3.create(MAX_THREADS);
    outSE3.create(1);
    sumRes.create(MAX_THREADS);
    sumSO3.create(MAX_THREADS);
    outSO3.create(1);
    cudaChannelFormatDesc f4 = cudaCreateChannelDesc<float4>();
    cudaChannelFormatDesc u4 = cudaCreateChannelDesc<uchar4>();
    cudaMallocArray(&arrV, &f4, w, h);
    cudaMallocArray(&arrN, &f4, w, h);
    cudaMallocArray(&arrC, &u4, w, h);
    cudaDeviceSynchronize();
  }
  ~RefOdom() {
    cudaFreeArray(arrV);
    cudaFreeArray(arrN);
    cudaFreeArray(arrC);
  }

  void load_maps(const float* v4, const float* n4) {
    cudaMemcpy2DToArray(arrV, 0, 0, v4, W * 16, W * 16, H, cudaMemcpyHostToDevice);
    cudaMemcpy2DToArray(arrN, 0, 0, n4, W * 16, W * 16, H, cudaMemcpyHostToDevice);
  }
  void load_rgba(const uint8_t* rgba) { cudaMemcpy2DToArray(arrC, 0, 0, rgba, W * 4, W * 4, H, cudaMemcpyHostToDevice); }

  void initICPDepth(const uint16_t* depth, float cutoff) {
    depth_tmp[0].upload(depth, W * 2, H, W);
    for (int i = 1; i < NP; ++i) pyrDown(depth_tmp[i - 1], depth_tmp[i]);
    for (int i = 0; i < NP; ++i) {
      createVMap(intr(i), depth_tmp[i], vmaps_curr[i], cutoff);
      createNMap(vmaps_curr[i], nmaps_curr[i]);
    }
    cudaDeviceSynchronize();
  }
  void initICPPred(const float* v4, const float* n4) {
    load_maps(v4, n4);
    copyMaps(arrV, arrN, W, H, vmaps_tmp, vmaps_curr[0], nmaps_curr[0]);
    for (int i = 1; i < NP; ++i) {
      resizeVMap(vmaps_curr[i - 1], vmaps_curr[i]);
      resizeNMap(nmaps_curr[i - 1], nmaps_curr[i]);
    }
    cudaDeviceSynchronize();
  }
  void initICPModel(const float* v4, const float* n4, const double* T) {
    load_maps(v4, n4);
    copyMaps(arrV, arrN, W, H, vmaps_tmp, vmaps_g_prev[0], nmaps_g_prev[0]);
    for (int i = 1; i < NP; ++i) {
      resizeVMap(vmaps_g_prev[i - 1], vmaps_g_prev[i]);
      resizeNMap(nmaps_g_prev[i - 1], nmaps_g_prev[i]);
    }
    M3f R;
    Eigen::Vector3f t;
    for (int r = 0; r < 3; ++r) {
      for (int c = 0; c < 3; ++c) R(r, c) = (float)T[r * 4 + c];
      t(r) = (float)T[r * 4 + 3];
    }
    mat33 dR = to_mat33(R);
    float3 dt = *reinterpret_cast<float3*>(t.data());
    for (int i = 0; i < NP; ++i) tranformMaps(vmaps_g_prev[i], nmaps_g_prev[i], dR, dt, vmaps_g_prev[i], nmaps_g_prev[i]);
    cudaDeviceSynchronize();
  }
  void populate(const uint8_t* rgba, DeviceArray2D<float>* dd, DeviceArray2D<uint8_t>* di, bool depth) {
    load_rgba(rgba);
    if (depth) {
      verticesToDepth(vmaps_tmp, dd[0], maxDepthRGB);
      for (int i = 0; i + 1 < NP; ++i) pyrDownGaussF(dd[i], dd[i + 1]);
    }
    imageBGRToIntensity(arrC, di[0]);
    for (int i = 0; i + 1 < NP; ++i) pyrDownUcharGauss(di[i], di[i + 1]);
    cudaDeviceSynchronize();
  }

  int track(double* Tio, bool rgbOnly, float icpWeight, bool pyramid, bool fastOdom, bool so3, Trace* trace, int maxTrace) {
    int nt = 0;
    const bool icp = !rgbOnly && icpWeight > 0, rgb = rgbOnly || icpWeight < 100;
    M3f Rprev;
    Eigen::Vector3f tprev;
    for (int r = 0; r < 3; ++r) {
      for (int c = 0; c < 3; ++c) Rprev(r, c) = (float)Tio[r * 4 + c];
      tprev(r) = (float)Tio[r * 4 + 3];
    }
    M3f Rcurr = Rprev;
    Eigen::Vector3f tcurr = tprev;
    if (rgb)
      for (int i = 0; i < NP; ++i) computeDerivativeImages(nextImage[i], dIdx[i], dIdy[i]);
    M3d resultR = M3d::Identity();
    if (so3) {
      const int L = 2;
      M3f R_lr = M3f::Identity();
      M3d K = M3d::Zero();
      K(0, 0) = intr(L).fx;
      K(1, 1) = intr(L).fy;
      K(0, 2) = intr(L).cx;
      K(1, 2) = intr(L).cy;
      K(2, 2) = 1;
      float lastError = std::numeric_limits<float>::max() / 2, lastCount = std::numeric_limits<float>::max() / 2;
      M3d lastResultR = M3d::Identity();
      for (int i = 0; i < 10; ++i) {
        M3f jtj;
        Eigen::Matrix<float, 3, 1> jtr;
        M3d Hm = K * resultR * K.inverse(), Kinv = K.inverse(), KR = K * resultR;
        mat33 ib, ki, kr;
        memcpy(&ib.data[0], Hm.cast<float>().eval().data(), sizeof(mat33));
        memcpy(&ki.data[0], Kinv.cast<float>().eval().data(), sizeof(mat33));
        memcpy(&kr.data[0], KR.cast<float>().eval().data(), sizeof(mat33));
        float residual[2];
        so3Step(lastNextImage[L], nextImage[L], ib, ki, kr, sumSO3, outSO3, jtj.data(), jtr.data(), residual);
        if (trace && nt < maxTrace) {
          Trace& t = trace[nt++];
          memset(&t, 0, sizeof(t));
          t.kind = 1;
          t.level = L;
          t.iter = i;
          memcpy(t.A_so3, jtj.data(), 36);
          memcpy(t.b_so3, jtr.data(), 12);
          t.so3_residual[0] = residual[0];
          t.so3_residual[1] = residual[1];
        }
        stats[4] = sqrt(residual[0]) / residual[1];
        stats[5] = residual[1];
        if (stats[4] < lastError && lastCount == stats[5]) break;
        if (stats[4] > lastError + 0.001) {
          stats[4] = lastError;
          stats[5] = lastCount;
          resultR = lastResultR;
          break;
        }
        lastError = stats[4];
        lastCount = stats[5];
        lastResultR = resultR;
        Eigen::Vector3f delta = jtj.ldlt().solve(jtr);
        M3d up = rodrigues(delta.cast<double>());
        R_lr = up.cast<float>() * R_lr;
        for (int x = 0; x < 3; ++x)
          for (int y = 0; y < 3; ++y) resultR(x, y) = R_lr(x, y);
      }
    }
    const int iters[NP] = {fastOdom ? 3 : 10, pyramid ? 5 : 0, pyramid ? 4 : 0};
    M3f Rprev_inv = Rprev.inverse();
    mat33 dRprev_inv = to_mat33(Rprev_inv);
    float3 dtprev = *reinterpret_cast<float3*>(tprev.data());
    M4d resultRt = M4d::Identity();
    if (so3)
      for (int x = 0; x < 3; ++x)
        for (int y = 0; y < 3; ++y) resultRt(x, y) = resultR(x, y);
    for (int i = NP - 1; i >= 0; --i) {
      if (rgb) projectToPointCloud(lastDepth[i], clouds[i], intr, i);
      M3d K = M3d::Zero();
      K(0, 0) = intr(i).fx;
      K(1, 1) = intr(i).fy;
      K(0, 2) = intr(i).cx;
      K(1, 2) = intr(i).cy;
      K(2, 2) = 1;
      stats[2] = std::numeric_limits<float>::max();
      for (int j = 0; j < iters[i]; ++j) {
        M4d Rt = resultRt.inverse();
        M3d R = Rt.topLeftCorner(3, 3);
        M3d KRK = K * R * K.inverse();
        mat33 krk;
        memcpy(&krk.data[0], KRK.cast<float>().eval().data(), sizeof(mat33));
        Eigen::Vector3d Kt = Rt.topRightCorner(3, 1);
        Kt = K * Kt;
        float3 kt = {(float)Kt(0), (float)Kt(1), (float)Kt(2)};
        int sigma = 0, rgbSize = 0;
        if (rgb)
          computeRgbResidual(pow(minGrad[i], 2.0) / pow(sobelScale, 2.0), dIdx[i], dIdy[i], lastDepth[i], nextDepth[i], lastImage[i],
                             nextImage[i], corres[i], sumRes, maxDepthDeltaRGB, kt, krk, sigma, rgbSize);
        float sigmaVal = std::sqrt((float)sigma / rgbSize == 0 ? 1 : rgbSize);
        float rgbError = std::sqrt(sigma) / (rgbSize == 0 ? 1 : rgbSize);
        if (rgbOnly && rgbError > stats[2]) break;
        stats[2] = rgbError;
        stats[3] = rgbSize;
        if (rgbOnly) sigmaVal = -1;
        M6f A_icp = M6f::Zero(), A_rgb = M6f::Zero();
        V6f b_icp = V6f::Zero(), b_rgb = V6f::Zero();
        mat33 dRcurr = to_mat33(Rcurr);
        float3 dtcurr = *reinterpret_cast<float3*>(tcurr.data());
        float residual[2] = {0, 0};
        if (icp)
          icpStep(dRcurr, dtcurr, vmaps_curr[i], nmaps_curr[i], dRprev_inv, dtprev, intr(i), vmaps_g_prev[i], nmaps_g_prev[i], distThres,
                  angleThres, sumSE3, outSE3, A_icp.data(), b_icp.data(), residual);
        stats[0] = sqrt(residual[0]) / residual[1];
        stats[1] = residual[1];
        if (rgb)
          rgbStep(corres[i], sigmaVal, clouds[i], intr(i).fx, intr(i).fy, dIdx[i], dIdy[i], sobelScale, sumSE3, outSE3, A_rgb.data(),
                  b_rgb.data());
        V6d result;
        M6d dA_rgb = A_rgb.cast<double>(), dA_icp = A_icp.cast<double>();
        V6d db_rgb = b_rgb.cast<double>(), db_icp = b_icp.cast<double>();
        if (icp && rgb) {
          const double w = icpWeight;
          lastA = dA_rgb + w * w * dA_icp;
          lastb = db_rgb + w * db_icp;
        } else if (icp) {
          lastA = dA_icp;
          lastb = db_icp;
        } else {
          lastA = dA_rgb;
          lastb = db_rgb;
        }
        result = lastA.ldlt().solve(lastb);
        if (trace && nt < maxTrace) {
          Trace& t = trace[nt++];
          memset(&t, 0, sizeof(t));
          t.level = i;
          t.iter = j;
          t.rgb_count = rgbSize;
          t.rgb_sigma = sigma;
          t.sigma_val = sigmaVal;
          memcpy(t.A_icp, A_icp.data(), 144);
          memcpy(t.b_icp, b_icp.data(), 24);
          t.icp_residual[0] = residual[0];
          t.icp_residual[1] = residual[1];
          memcpy(t.A_rgb, A_rgb.data(), 144);
          memcpy(t.b_rgb, b_rgb.data(), 24);
          memcpy(t.lastA, lastA.data(), 288);
          memcpy(t.lastb, lastb.data(), 48);
          memcpy(t.result, result.data(), 48);
        }
        // OdometryProvider::computeUpdateSE3 semantics
        M4d upd = M4d::Identity();
        upd.topLeftCorner(3, 3) = rodrigues(Eigen::Vector3d(result(3), result(4), result(5)));
        upd(0, 3) = result(0);
        upd(1, 3) = result(1);
        upd(2, 3) = result(2);
        resultRt = upd * resultRt;
        Eigen::Isometry3f odom;
        odom.setIdentity();
        M3d rotation = resultRt.topLeftCorner(3, 3);
        odom.rotate(rotation.cast<float>().eval());
        odom.translation() = resultRt.cast<float>().eval().topRightCorner(3, 1);
        Eigen::Isometry3f cur;
        cur.setIdentity();
        cur.rotate(Rprev);
        cur.translation() = tprev;
        cur = cur * odom.inverse();
        tcurr = cur.translation();
        Rcurr = cur.rotation();
      }
    }
    if (rgb && (tcurr - tprev).norm() > 0.3) {
      Rcurr = Rprev;
      tcurr = tprev;
    }
    if (so3)
      for (int i = 0; i < NP; ++i) std::swap(lastNextImage[i], nextImage[i]);
    Eigen::JacobiSVD<Eigen::Matrix3d> svd(Rcurr.cast<double>(), Eigen::ComputeFullU | Eigen::ComputeFullV);
    Eigen::Matrix3d Ro = svd.matrixU() * svd.matrixV().transpose();
    for (int r = 0; r < 3; ++r) {
      for (int c = 0; c < 3; ++c) Tio[r * 4 + c] = Ro(r, c);
      Tio[r * 4 + 3] = (double)tcurr(r);
    }
    Tio[12] = Tio[13] = Tio[14] = 0;
    Tio[15] = 1;
    return nt;
  }
};

double now_s() { return std::chrono::duration<double>(std::chrono::steady_clock::now().time_since_epoch()).count(); }

template <typename T>
void download2d(const DeviceArray2D<T>& a, void* host) {
  a.download(host, a.cols() * sizeof(T));
}

}  // namespace

extern "C" {

void* efr_create(int w, int h, float cx, float cy, float fx, float fy) { return new RefOdom(w, h, cx, cy, fx, fy); }
void efr_destroy(void* p) { delete (RefOdom*)p; }
void efr_init_icp_depth(void* p, const uint16_t* depth, float cutoff) {
  double t0 = now_s();
  ((RefOdom*)p)->initICPDepth(depth, cutoff);
  ((RefOdom*)p)->t_init += now_s() - t0;
}
void efr_init_icp_pred(void* p, const float* v4, const float* n4) { ((RefOdom*)p)->initICPPred(v4, n4); }
void efr_init_icp_model(void* p, const float* v4, const float* n4, const double* T) {
  double t0 = now_s();
  ((RefOdom*)p)->initICPModel(v4, n4, T);
  ((RefOdom*)p)->t_init += now_s() - t0;
}
void efr_init_rgb(void* p, const uint8_t* rgba) {
  RefOdom* o = (RefOdom*)p;
  double t0 = now_s();
  o->populate(rgba, o->nextDepth, o->nextImage, true);
  o->t_init += now_s() - t0;
}
void efr_init_rgb_model(void* p, const uint8_t* rgba) {
  RefOdom* o = (RefOdom*)p;
  double t0 = now_s();
  o->populate(rgba, o->lastDepth, o->lastImage, true);
  o->t_init += now_s() - t0;
}
void efr_init_first_rgb(void* p, const uint8_t* rgba) {
  RefOdom* o = (RefOdom*)p;
  o->populate(rgba, nullptr, o->lastNextImage, false);
}
int efr_track(void* p, double* T, int rgbOnly, float icpWeight, int pyramid, int fastOdom, int so3, void* trace, int maxTrace) {
  RefOdom* o = (RefOdom*)p;
  double t0 = now_s();
  int n = o->track(T, rgbOnly != 0, icpWeight, pyramid != 0, fastOdom != 0, so3 != 0, (Trace*)trace, maxTrace);
  o->t_track += now_s() - t0;
  return n;
}
void efr_stats(void* p, float* out6) { memcpy(out6, ((RefOdom*)p)->stats, 24); }
void efr_timers(void* p, double* out2) {
  out2[0] = ((RefOdom*)p)->t_init;
  out2[1] = ((RefOdom*)p)->t_track;
}

// which: 0 vmap_curr 1 nmap_curr 2 vmap_g_prev 3 nmap_g_prev 4 lastDepth 5 nextDepth 6 lastImage 7 nextImage
//        8 lastNextImage 9 dIdx 10 dIdy 11 depth_tmp 12 corres
void efr_download(void* p, int which, int level, void* host) {
  RefOdom* o = (RefOdom*)p;
  switch (which) {
    case 0: download2d(o->vmaps_curr[level], host); break;
    case 1: download2d(o->nmaps_curr[level], host); break;
    case 2: download2d(o->vmaps_g_prev[level], host); break;
    case 3: download2d(o->nmaps_g_prev[level], host); break;
    case 4: download2d(o->lastDepth[level], host); break;
    case 5: download2d(o->nextDepth[level], host); break;
    case 6: download2d(o->lastImage[level], host); break;
    case 7: download2d(o->nextImage[level], host); break;
    case 8: download2d(o->lastNextImage[level], host); break;
    case 9: download2d(o->dIdx[level], host); break;
    case 10: download2d(o->dIdy[level], host); break;
    case 11: download2d(o->depth_tmp[level], host); break;
    case 12: download2d(o->corres[level], host); break;
  }
}

// single reference steps with explicit parameters
void efr_icp_step(void* p, int level, const float* Rcurr, const float* tcurr, const float* Rprev_inv, const float* tprev, float* A, float* b,
                  float* residual) {
  RefOdom* o = (RefOdom*)p;
  mat33 rc, rp;
  memcpy(&rc, Rcurr, 36);
  memcpy(&rp, Rprev_inv, 36);
  float3 tc = {tcurr[0], tcurr[1], tcurr[2]}, tp = {tprev[0], tprev[1], tprev[2]};
  icpStep(rc, tc, o->vmaps_curr[level], o->nmaps_curr[level], rp, tp, o->intr(level), o->vmaps_g_prev[level], o->nmaps_g_prev[level],
          o->distThres, o->angleThres, o->sumSE3, o->outSE3, A, b, residual);
}
void efr_rgb_residual(void* p, int level, const float* krkinv, const float* kt, int* sigma, int* count) {
  RefOdom* o = (RefOdom*)p;
  computeDerivativeImages(o->nextImage[level], o->dIdx[level], o->dIdy[level]);
  mat33 kk;
  memcpy(&kk, krkinv, 36);
  float3 k3 = {kt[0], kt[1], kt[2]};
  computeRgbResidual(pow(o->minGrad[level], 2.0) / pow(o->sobelScale, 2.0), o->dIdx[level], o->dIdy[level], o->lastDepth[level],
                     o->nextDepth[level], o->lastImage[level], o->nextImage[level], o->corres[level], o->sumRes, o->maxDepthDeltaRGB, k3, kk,
                     *sigma, *count);
}
void efr_rgb_step(void* p, int level, float sigma, float* A, float* b) {
  RefOdom* o = (RefOdom*)p;
  projectToPointCloud(o->lastDepth[level], o->clouds[level], o->intr, level);
  rgbStep(o->corres[level], sigma, o->clouds[level], o->intr(level).fx, o->intr(level).fy, o->dIdx[level], o->dIdy[level], o->sobelScale,
          o->sumSE3, o->outSE3, A, b);
}
void efr_so3_step(void* p, const float* ib, const float* ki, const float* kr, float* A, float* b, float* residual) {
  RefOdom* o = (RefOdom*)p;
  mat33 a, c, d;
  memcpy(&a, ib, 36);
  memcpy(&c, ki, 36);
  memcpy(&d, kr, 36);
  so3Step(o->lastNextImage[2], o->nextImage[2], a, c, d, o->sumSO3, o->outSO3, A, b, residual);
}

// wall-clock milliseconds per icpStep() call exactly as the reference issues it (2 launches + device sync + D2H)
double efr_time_icp_step(void* p, int level, const float* Rcurr, const float* tcurr, const float* Rprev_inv, const float* tprev, int reps) {
  float A[36], b[6], r[2];
  efr_icp_step(p, level, Rcurr, tcurr, Rprev_inv, tprev, A, b, r);
  cudaDeviceSynchronize();
  double t0 = now_s();
  for (int i = 0; i < reps; ++i) efr_icp_step(p, level, Rcurr, tcurr, Rprev_inv, tprev, A, b, r);
  return (now_s() - t0) * 1000.0 / reps;
}

}  // extern "C"
