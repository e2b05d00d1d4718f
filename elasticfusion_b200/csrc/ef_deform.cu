// Embedded-deformation solve of the local loop closure (reference Core/Deformation.cpp:88-207,
// Core/Utils/DeformationGraph.cpp:239-956): constraint weighting, Gauss-Newton on the sparse normal equations and the
// hand-over of the graph as 16 floats per node, all on the device in one single-CTA launch.
//
// The reference materialises the Jacobian and lets CHOLMOD factorise JᵀJ under a fill-reducing permutation. Here JᵀJ and
// Jᵀr are assembled directly from the row definitions of sparseJacobian / sparseResidual (:494-887), in fp64, each output
// entry summed by one thread in a fixed order (two runs are bit-identical; no atomics). In time order JᵀJ is block-banded:
// regularisation couples nodes at most 4 apart and a constraint's k nodes lie in one 20-node window, so a block-band
// Cholesky (12x12 node blocks, at most 19 sub-diagonal blocks) needs no permutation. Results differ from the reference in
// rounding only.
#include <math.h>
#include <string.h>

#include "ef_device.cuh"
#include "ef_internal.h"

namespace ef {

namespace {

constexpr int KNN = 4;         // DeformationGraph::k (Deformation.cpp:23)
constexpr int LOOKBACK = 20;   // weightVerticesSeq window (DeformationGraph.cpp:269)
constexpr int NV = 12;         // numVariables: rotation column-major, then translation (applyDeltaSparse, :896-923)
constexpr int NB = 4;          // neighbours per node (connectGraphSeq with k = 4, :239-266)
constexpr int MAXBW = 19;      // largest block distance between two coupled nodes
constexpr int THREADS = 1024;
constexpr int MAX_ITER = 3;    // optimiseGraphSparse (:460)

struct DeformWork {
  int cap_nodes = 0, cap_cons = 0;
  double *pos = nullptr, *src = nullptr, *dst = nullptr;  // node positions, constraint source / target points (x3)
  int *ntime = nullptr, *ctime = nullptr;                 // node times, constraint source times
  double *R = nullptr, *t = nullptr;                      // node rotation (column-major) and translation
  int* cnode = nullptr;                                   // KNN nodes of each constraint, ascending id
  double* cw = nullptr;                                   // their normalised weights
  int *list_off = nullptr, *list = nullptr;               // constraints touching each node, ascending
  double *res_rot = nullptr, *res_reg = nullptr, *res_con = nullptr;
  double* cerr = nullptr;                                 // |position - target| of each constraint
  double *band = nullptr, *linv = nullptr, *x = nullptr;  // JᵀJ lower block band, inverse diagonal factors, rhs / delta
  float* nodes16 = nullptr;
  double* rt12 = nullptr;                                 // R (column-major) and t of each node, fp64
  EfDeformResult* out = nullptr;
  Arena arena;  // every buffer above
};

struct Args {
  int n, m, last_deform_time;
  double *pos, *src, *dst;
  const int *ntime, *ctime;
  double *R, *t;
  int* cnode;
  double* cw;
  int *list_off, *list;
  double *res_rot, *res_reg, *res_con;
  double* cerr;
  double *band, *linv, *x;
  float* nodes16;
  double* rt12;
  EfDeformResult* out;
};

// s-th neighbour of node x in a graph of n >= 5 nodes (connectGraphSeq): the first and last k/2 nodes connect to the
// other k of the first / last k+1 nodes, every other node to x-1, x+1, x-2, x+2
__device__ __forceinline__ int nbr(int x, int s, int n) {
  if (x < KNN / 2) return s < x ? s : s + 1;
  if (x >= n - KNN / 2) {
    const int v = n - (KNN + 1) + s;
    return v < x ? v : v + 1;
  }
  return (s & 1) ? x + (s >> 1) + 1 : x - (s >> 1) - 1;
}

// component (row of a 3-row residual block) that variable v of a node enters: R.data()[v] is R(v % 3, v / 3)
__device__ __forceinline__ int comp(int v) { return v < 9 ? v % 3 : v - 9; }

// coefficient of rotation variable v (< 9) in rotation row r of a node (sparseJacobian, :518-549)
__device__ __forceinline__ double jrot(int r, int v, const double* R) {
  const int c = v / 3, i = v % 3;
  switch (r) {
    case 0: return c == 0 ? R[3 + i] : c == 1 ? R[i] : 0.0;      // c0 . c1
    case 1: return c == 0 ? R[6 + i] : c == 2 ? R[i] : 0.0;      // c0 . c2
    case 2: return c == 1 ? R[6 + i] : c == 2 ? R[3 + i] : 0.0;  // c1 . c2
    default: return c == r - 3 ? 2 * R[v] : 0.0;                  // |ci|^2 - 1
  }
}

__device__ __forceinline__ double dnorm3(double x, double y, double z) { return sqrt(x * x + y * y + z * z); }

// deterministic sum over the CTA (every thread passes its own partial; fixed tree)
__device__ double block_sum(double v, double* red) {
  red[threadIdx.x] = v;
  __syncthreads();
  for (int s = THREADS / 2; s > 0; s >>= 1) {
    if ((int)threadIdx.x < s) red[threadIdx.x] += red[threadIdx.x + s];
    __syncthreads();
  }
  const double r = red[0];
  __syncthreads();
  return r;
}

__device__ int block_max(int v, int* redi) {
  redi[threadIdx.x] = v;
  __syncthreads();
  for (int s = THREADS / 2; s > 0; s >>= 1) {
    if ((int)threadIdx.x < s) redi[threadIdx.x] = max(redi[threadIdx.x], redi[threadIdx.x + s]);
    __syncthreads();
  }
  const int r = redi[0];
  __syncthreads();
  return r;
}

// computeVertexPosition (:925-942) of constraint l's source point
__device__ void vertex_position(const Args& A, int l, double* p) {
  const double* s = A.src + 3 * l;
  p[0] = p[1] = p[2] = 0;
  for (int i = 0; i < KNN; ++i) {
    const int j = A.cnode[KNN * l + i];
    const double w = A.cw[KNN * l + i];
    const double* P = A.pos + 3 * j;
    const double* R = A.R + 9 * j;
    const double d0 = s[0] - P[0], d1 = s[1] - P[1], d2 = s[2] - P[2];
    for (int q = 0; q < 3; ++q) {
      const double rd = R[q] * d0 + R[3 + q] * d1 + R[6 + q] * d2;
      p[q] += w * (rd + P[q] + A.t[3 * j + q]);
    }
  }
}

// weightVerticesSeq (:268-373) for one constraint point: nearest node in time (the reference's imin/imid/imax rule), a
// 20-node window backwards then forwards, sorted by float distance; the k nearest weighted by (1 - d/dMax)^2 with dMax the
// (k+1)-th distance, normalised, ordered by node id
__device__ void weight_point(const Args& A, int l) {
  const int n = A.n;
  const int vt = A.ctime[l];
  const double* p = A.src + 3 * l;
  int imin = 0, imax = n - 1, imid = (imin + imax) / 2;
  while (imax >= imin) {
    imid = (imin + imax) / 2;
    if (A.ntime[imid] < vt) imin = imid + 1;
    else if (A.ntime[imid] > vt) imax = imid - 1;
    else break;
  }
  imin = min(imin, n - 1);
  const long long di = llabs((long long)A.ntime[imin] - vt), dm = llabs((long long)A.ntime[imid] - vt);
  // imax < 0 only when vt precedes every node; the reference then reads outside its vector, but whichever of node 0 or
  // "node -1" it picks, the window below is nodes 0..19 in the same order
  const long long dx = imax >= 0 ? llabs((long long)A.ntime[imax] - vt) : -1;
  int found;
  if (di <= dm && (imax < 0 || di <= dx)) found = imin;
  else if (dm <= di && (imax < 0 || dm <= dx)) found = imid;
  else found = imax < 0 ? 0 : imax;

  float dist[LOOKBACK];
  int id[LOOKBACK];
  int cnt = 0;
  for (int j = found; j >= 0 && cnt < LOOKBACK; --j, ++cnt) {
    id[cnt] = j;
    dist[cnt] = (float)dnorm3(A.pos[3 * j] - p[0], A.pos[3 * j + 1] - p[1], A.pos[3 * j + 2] - p[2]);
  }
  for (int j = found + 1; j < n && cnt < LOOKBACK; ++j, ++cnt) {
    id[cnt] = j;
    dist[cnt] = (float)dnorm3(A.pos[3 * j] - p[0], A.pos[3 * j + 1] - p[1], A.pos[3 * j + 2] - p[2]);
  }
  // stable insertion sort by float distance (the reference's std::sort leaves exact ties in an unspecified order)
  for (int i = 1; i < cnt; ++i) {
    const float d = dist[i];
    const int k = id[i];
    int j = i - 1;
    while (j >= 0 && dist[j] > d) {
      dist[j + 1] = dist[j];
      id[j + 1] = id[j];
      --j;
    }
    dist[j + 1] = d;
    id[j + 1] = k;
  }
  const double dMax = dist[KNN];
  double w[KNN];
  int nid[KNN];
  double sum = 0;
  for (int i = 0; i < KNN; ++i) {
    const int j = id[i];
    const double r = 1.0 - dnorm3(p[0] - A.pos[3 * j], p[1] - A.pos[3 * j + 1], p[2] - A.pos[3 * j + 2]) / dMax;
    w[i] = r * r;
    nid[i] = j;
    sum += w[i];
  }
  for (int i = 0; i < KNN; ++i) w[i] /= sum;
  for (int i = 1; i < KNN; ++i)  // ids are distinct: plain insertion sort gives VertexWeightMap::sort's order
    for (int j = i; j > 0 && nid[j - 1] > nid[j]; --j) {
      const int ti = nid[j]; nid[j] = nid[j - 1]; nid[j - 1] = ti;
      const double tw = w[j]; w[j] = w[j - 1]; w[j - 1] = tw;
    }
  for (int i = 0; i < KNN; ++i) {
    A.cnode[KNN * l + i] = nid[i];
    A.cw[KNN * l + i] = w[i];
  }
}

// value of variable v of node j in its 3-row regularisation block towards `delta` = pos_nb - pos_j (:579-592)
__device__ __forceinline__ double reg_coef(int v, const double* delta, double sReg) {
  return v < 9 ? delta[v / 3] * sReg : 1.0 * sReg;
}

// value of variable v of constraint l's i-th node in the constraint's 3-row block (:754-778)
__device__ __forceinline__ double con_coef(const Args& A, int l, int i, int v, double sCon) {
  const int j = A.cnode[KNN * l + i];
  const double w = A.cw[KNN * l + i];
  if (v >= 9) return w * sCon;
  const int m = v / 3;
  return ((A.src[3 * l + m] - A.pos[3 * j + m]) * w) * sCon;
}

// sparseResidual (:791-887) into res_rot / res_reg / res_con; returns the squared norm of the rows the reference keeps
__device__ double residuals(const Args& A, int e0, double* red) {
  const double sReg = sqrt(10.0), sCon = sqrt(100.0);
  const int n = A.n;
  double acc = 0;
  for (int j = threadIdx.x; j < n; j += THREADS) {
    const double* R = A.R + 9 * j;
    double* r = A.res_rot + 6 * j;
    r[0] = R[0] * R[3] + R[1] * R[4] + R[2] * R[5];
    r[1] = R[0] * R[6] + R[1] * R[7] + R[2] * R[8];
    r[2] = R[3] * R[6] + R[4] * R[7] + R[5] * R[8];
    r[3] = (R[0] * R[0] + R[1] * R[1] + R[2] * R[2]) - 1.0;
    r[4] = (R[3] * R[3] + R[4] * R[4] + R[5] * R[5]) - 1.0;
    r[5] = (R[6] * R[6] + R[7] * R[7] + R[8] * R[8]) - 1.0;
    if (j >= e0)
      for (int i = 0; i < 6; ++i) acc += r[i] * r[i];
    for (int s = 0; s < NB; ++s) {
      const int b = nbr(j, s, n);
      const double* Pj = A.pos + 3 * j;
      const double* Pb = A.pos + 3 * b;
      const double d0 = Pb[0] - Pj[0], d1 = Pb[1] - Pj[1], d2 = Pb[2] - Pj[2];
      double* g = A.res_reg + 3 * (NB * j + s);
      for (int q = 0; q < 3; ++q) {
        const double rd = R[q] * d0 + R[3 + q] * d1 + R[6 + q] * d2;
        g[q] = (((rd + Pj[q]) + A.t[3 * j + q]) - (Pb[q] + A.t[3 * b + q])) * sReg;
      }
      if (j >= e0 || b >= e0)
        for (int q = 0; q < 3; ++q) acc += g[q] * g[q];
    }
  }
  for (int l = threadIdx.x; l < A.m; l += THREADS) {
    double p[3];
    vertex_position(A, l, p);
    const double* T = A.dst + 3 * l;
    double* g = A.res_con + 3 * l;
    for (int q = 0; q < 3; ++q) g[q] = (p[q] - T[q]) * sCon;
    A.cerr[l] = dnorm3(p[0] - T[0], p[1] - T[1], p[2] - T[2]);
    if (A.cnode[KNN * l + KNN - 1] >= e0)
      for (int q = 0; q < 3; ++q) acc += g[q] * g[q];
  }
  return block_sum(acc, red);
}

// nonRelativeConstraintError (:944-956): a float running sum in constraint order, each fp64 norm added before rounding
__device__ float mean_cons_err(const Args& A) {
  float r = 0;
  for (int l = 0; l < A.m; ++l) r = (float)((double)r + A.cerr[l]);
  return r / (float)A.m;
}

__global__ void __launch_bounds__(THREADS) k_deform_solve(Args A) {
  pdl_enter();
  __shared__ double red[THREADS];
  __shared__ double panel[MAXBW * 144];  // L_{k+i,k}, i = 1..bw, of the current block column
  __shared__ double Ld[144];             // diagonal block being factorised
  __shared__ double yk[NV], part[MAXBW * NV];
  __shared__ int s_fail;
  int* redi = (int*)red;
  const int tid = threadIdx.x;
  const int n = A.n, m = A.m;
  const double sReg = sqrt(10.0), sCon = sqrt(100.0);

  // enabled nodes (time > lastDeformTime, :436-443) form a suffix [e0, n) because times ascend
  int e0 = n;
  {
    int first = n;
    for (int j = tid; j < n; j += THREADS)
      if (A.ntime[j] > A.last_deform_time && (j == 0 || A.ntime[j - 1] <= A.last_deform_time)) first = j;
    e0 = n - block_max(n - first, redi);
  }
  const int N = n - e0;

  // graph state: R = I, t = 0 (initialiseGraph, :69-81)
  for (int j = tid; j < n; j += THREADS) {
    for (int i = 0; i < 9; ++i) A.R[9 * j + i] = (i % 4 == 0) ? 1.0 : 0.0;
    for (int i = 0; i < 3; ++i) A.t[3 * j + i] = 0.0;
  }
  for (int l = tid; l < m; l += THREADS) weight_point(A, l);
  __syncthreads();

  // constraints touching each enabled node, in constraint order (count, scan, fill; one thread per node)
  {
    int c = 0;
    const int a = e0 + tid;
    if (a < n)
      for (int l = 0; l < m; ++l)
        for (int i = 0; i < KNN; ++i) c += A.cnode[KNN * l + i] == a;
    redi[tid] = c;
    __syncthreads();
    if (tid == 0) {
      int s = 0;
      for (int i = 0; i <= N; ++i) {
        const int v = i < N ? redi[i] : 0;
        A.list_off[i] = s;
        s += v;
      }
    }
    __syncthreads();
    if (a < n) {
      int o = A.list_off[tid];
      for (int l = 0; l < m; ++l)
        for (int i = 0; i < KNN; ++i)
          if (A.cnode[KNN * l + i] == a) A.list[o++] = l;
    }
  }
  // block half-bandwidth actually used: largest distance between two coupled enabled nodes
  int bw;
  {
    int b = 0;
    for (int j = e0 + tid; j < n; j += THREADS)
      for (int s = 0; s < NB; ++s) {
        const int q = nbr(j, s, n);
        if (q >= e0) b = max(b, abs(q - j));
      }
    for (int l = tid; l < m; l += THREADS) {
      const int hi = A.cnode[KNN * l + KNN - 1];
      if (hi >= e0) b = max(b, hi - max(A.cnode[KNN * l], e0));
    }
    bw = block_max(b, redi);
  }
  // the band holds MAXBW sub-diagonal blocks; the window rule bounds the coupling by 19, so a wider one is reported, not solved
  const bool too_wide = bw > MAXBW;
  if (too_wide) bw = 0;

  float error = (float)residuals(A, e0, red);
  double lastError = error;
  int iter = 0, stop = too_wide ? 6 : 0;
  if (tid == 0) s_fail = 0;
  __syncthreads();

  while (!too_wide && iter++ < MAX_ITER) {
    // ---- normal equations: lower block band of JᵀJ and x = -Jᵀr
    const int nb_row = (bw + 1) * 144;
    for (int e = tid; e < N * nb_row; e += THREADS) {
      const int i = e / nb_row, d = (e / 144) % (bw + 1), v = (e % 144) / NV, u = e % NV;
      double* dstp = A.band + ((size_t)i * (MAXBW + 1) + d) * 144 + v * NV + u;
      if (d > i) continue;
      const int a = e0 + i, b = a - d;
      double sum = 0;
      if (d == 0) {
        if (v < 9 && u < 9)
          for (int r = 0; r < 6; ++r) sum += jrot(r, v, A.R + 9 * a) * jrot(r, u, A.R + 9 * a);
        for (int s = 0; s < NB; ++s) {  // rows of a's own edges
          const int q = nbr(a, s, n);
          if (comp(v) == comp(u)) {
            const double dl[3] = {A.pos[3 * q] - A.pos[3 * a], A.pos[3 * q + 1] - A.pos[3 * a + 1], A.pos[3 * q + 2] - A.pos[3 * a + 2]};
            sum += reg_coef(v, dl, sReg) * reg_coef(u, dl, sReg);
          }
        }
        if (v >= 9 && v == u)  // rows of the edges that end at a: -sqrt(wReg) on a's translation
          for (int x = max(0, a - 4); x <= min(n - 1, a + 4); ++x)
            for (int s = 0; s < NB; ++s)
              if (x != a && nbr(x, s, n) == a) sum += (-1.0 * sReg) * (-1.0 * sReg);
      } else {
        for (int s = 0; s < NB; ++s) {
          if (nbr(a, s, n) == b && u >= 9 && comp(v) == u - 9) {  // edge a -> b
            const double dl[3] = {A.pos[3 * b] - A.pos[3 * a], A.pos[3 * b + 1] - A.pos[3 * a + 1], A.pos[3 * b + 2] - A.pos[3 * a + 2]};
            sum += reg_coef(v, dl, sReg) * (-1.0 * sReg);
          }
          if (nbr(b, s, n) == a && v >= 9 && comp(u) == v - 9) {  // edge b -> a
            const double dl[3] = {A.pos[3 * a] - A.pos[3 * b], A.pos[3 * a + 1] - A.pos[3 * b + 1], A.pos[3 * a + 2] - A.pos[3 * b + 2]};
            sum += (-1.0 * sReg) * reg_coef(u, dl, sReg);
          }
        }
      }
      if (comp(v) == comp(u))
        for (int o = A.list_off[i]; o < A.list_off[i + 1]; ++o) {
          const int l = A.list[o];
          int ia = -1, ib = -1;
          for (int k = 0; k < KNN; ++k) {
            if (A.cnode[KNN * l + k] == a) ia = k;
            if (A.cnode[KNN * l + k] == b) ib = k;
          }
          if (ib >= 0) sum += con_coef(A, l, ia, v, sCon) * con_coef(A, l, ib, u, sCon);
        }
      *dstp = sum;
    }
    for (int e = tid; e < N * NV; e += THREADS) {
      const int i = e / NV, v = e % NV, a = e0 + i, q = comp(v);
      double g = 0;
      if (v < 9)
        for (int r = 0; r < 6; ++r) g += jrot(r, v, A.R + 9 * a) * A.res_rot[6 * a + r];
      for (int s = 0; s < NB; ++s) {
        const int b = nbr(a, s, n);
        const double dl[3] = {A.pos[3 * b] - A.pos[3 * a], A.pos[3 * b + 1] - A.pos[3 * a + 1], A.pos[3 * b + 2] - A.pos[3 * a + 2]};
        g += reg_coef(v, dl, sReg) * A.res_reg[3 * (NB * a + s) + q];
      }
      if (v >= 9)
        for (int x = max(0, a - 4); x <= min(n - 1, a + 4); ++x)
          for (int s = 0; s < NB; ++s)
            if (x != a && nbr(x, s, n) == a) g += (-1.0 * sReg) * A.res_reg[3 * (NB * x + s) + q];
      for (int o = A.list_off[i]; o < A.list_off[i + 1]; ++o) {
        const int l = A.list[o];
        int ia = 0;
        for (int k = 0; k < KNN; ++k)
          if (A.cnode[KNN * l + k] == a) ia = k;
        g += con_coef(A, l, ia, v, sCon) * A.res_con[3 * l + q];
      }
      A.x[e] = -g;
    }
    __syncthreads();

    // ---- right-looking block-band Cholesky, JᵀJ = L Lᵀ; the inverse of every diagonal factor is kept for the solves
    for (int k = 0; k < N; ++k) {
      const int w = min(bw, N - 1 - k);
      double* Akk = A.band + (size_t)k * (MAXBW + 1) * 144;
      if (tid < 144) Ld[tid] = Akk[tid];
      __syncthreads();
      if (tid < 32) {
        for (int c = 0; c < NV; ++c) {
          if (tid == c) {
            const double p = Ld[c * NV + c];
            if (!(p > 0)) s_fail = 1;
            Ld[c * NV + c] = sqrt(p);
          }
          __syncwarp();
          if (tid > c && tid < NV) Ld[tid * NV + c] /= Ld[c * NV + c];
          __syncwarp();
          if (tid > c && tid < NV)
            for (int j = c + 1; j <= tid; ++j) Ld[tid * NV + j] -= Ld[tid * NV + c] * Ld[j * NV + c];
          __syncwarp();
        }
        if (tid < NV) {  // column tid of L_kk^-1 by forward substitution
          double col[NV];
          for (int r = 0; r < NV; ++r) {
            if (r < tid) { col[r] = 0; continue; }
            double s = (r == tid) ? 1.0 : 0.0;
            for (int j = tid; j < r; ++j) s -= Ld[r * NV + j] * col[j];
            col[r] = s / Ld[r * NV + r];
          }
          for (int r = 0; r < NV; ++r) A.linv[(size_t)k * 144 + r * NV + tid] = col[r];
        }
      }
      __syncthreads();
      const double* Li = A.linv + (size_t)k * 144;
      for (int e = tid; e < w * 144; e += THREADS) {  // L_{k+i,k} = A_{k+i,k} L_kk^-T
        const int i = e / 144 + 1, r = (e % 144) / NV, c = e % NV;
        const double* Aik = A.band + ((size_t)(k + i) * (MAXBW + 1) + i) * 144;
        double s = 0;
        for (int j = 0; j <= c; ++j) s += Aik[r * NV + j] * Li[c * NV + j];
        panel[e] = s;
      }
      __syncthreads();
      for (int e = tid; e < w * 144; e += THREADS) {
        const int i = e / 144 + 1;
        A.band[((size_t)(k + i) * (MAXBW + 1) + i) * 144 + e % 144] = panel[e];
      }
      const int nup = w * (w + 1) / 2 * 144;
      for (int e = tid; e < nup; e += THREADS) {  // A_{k+i,k+j} -= L_{k+i,k} L_{k+j,k}ᵀ, 1 <= j <= i <= w
        int p = e / 144, i = 1;
        while (p >= i) { p -= i; ++i; }
        const int j = p + 1, r = (e % 144) / NV, c = e % NV;
        const double* Pi = panel + (i - 1) * 144 + r * NV;
        const double* Pj = panel + (j - 1) * 144 + c * NV;
        double s = 0;
        for (int q = 0; q < NV; ++q) s += Pi[q] * Pj[q];
        A.band[((size_t)(k + i) * (MAXBW + 1) + (i - j)) * 144 + r * NV + c] -= s;
      }
      __syncthreads();
    }
    // ---- L y = -Jᵀr, then Lᵀ delta = y (in place in x)
    for (int k = 0; k < N; ++k) {
      const int w = min(bw, N - 1 - k);
      const double* Li = A.linv + (size_t)k * 144;
      if (tid < NV) {
        double s = 0;
        for (int j = 0; j <= tid; ++j) s += Li[tid * NV + j] * A.x[k * NV + j];
        yk[tid] = s;
      }
      __syncthreads();
      if (tid < NV) A.x[k * NV + tid] = yk[tid];
      for (int e = tid; e < w * NV; e += THREADS) {
        const int i = e / NV + 1, r = e % NV;
        const double* L = A.band + ((size_t)(k + i) * (MAXBW + 1) + i) * 144 + r * NV;
        double s = 0;
        for (int j = 0; j < NV; ++j) s += L[j] * yk[j];
        A.x[(k + i) * NV + r] -= s;
      }
      __syncthreads();
    }
    for (int k = N - 1; k >= 0; --k) {
      const int w = min(bw, N - 1 - k);
      for (int e = tid; e < w * NV; e += THREADS) {
        const int i = e / NV + 1, c = e % NV;
        const double* L = A.band + ((size_t)(k + i) * (MAXBW + 1) + i) * 144;
        double s = 0;
        for (int r = 0; r < NV; ++r) s += L[r * NV + c] * A.x[(k + i) * NV + r];
        part[e] = s;
      }
      __syncthreads();
      if (tid < NV) {
        double s = A.x[k * NV + tid];
        for (int i = 0; i < w; ++i) s -= part[i * NV + tid];
        yk[tid] = s;
      }
      __syncthreads();
      if (tid < NV) {
        const double* Li = A.linv + (size_t)k * 144;
        double s = 0;
        for (int r = tid; r < NV; ++r) s += Li[r * NV + tid] * yk[r];
        A.x[k * NV + tid] = s;
      }
      __syncthreads();
    }
    if (s_fail) {  // JᵀJ not positive definite: leave the graph as it is
      stop = 5;
      break;
    }

    // ---- applyDeltaSparse, new residual, stop rules (:463-476)
    double dsq = 0;
    for (int e = tid; e < N * NV; e += THREADS) {
      const int a = e0 + e / NV, v = e % NV;
      const double dv = A.x[e];
      if (v < 9) A.R[9 * a + v] += dv;
      else A.t[3 * a + v - 9] += dv;
      dsq += dv * dv;
    }
    const double dnorm = sqrt(block_sum(dsq, red));
    error = (float)residuals(A, e0, red);
    const double errorDiff = error - lastError;
    if (error > lastError) stop = 1;
    else if (dnorm < 1e-2) stop = 2;
    else if (error < 1e-3) stop = 3;
    else if (fabs(errorDiff) < 1e-5 * error) stop = 4;
    if (stop) break;
    lastError = error;
  }
  if (iter > MAX_ITER) iter = MAX_ITER;
  if (too_wide) bw = MAXBW + 1;
  __syncthreads();

  // ---- hand-over: 16 floats per node (Deformation.cpp:175-189)
  for (int j = tid; j < n; j += THREADS) {
    float* o = A.nodes16 + 16 * j;
    for (int i = 0; i < 3; ++i) o[i] = (float)A.pos[3 * j + i];
    for (int i = 0; i < 9; ++i) o[3 + i] = (float)A.R[9 * j + i];
    for (int i = 0; i < 3; ++i) o[12 + i] = (float)A.t[3 * j + i];
    o[15] = (float)A.ntime[j];
    for (int i = 0; i < 9; ++i) A.rt12[12 * j + i] = A.R[9 * j + i];
    for (int i = 0; i < 3; ++i) A.rt12[12 * j + 9 + i] = A.t[3 * j + i];
  }
  if (tid == 0) {
    EfDeformResult r;
    r.n_nodes = n;
    r.n_enabled = N;
    r.n_constraints = m;
    r.iterations = iter;
    r.stop = stop;
    r.bandwidth = bw;
    r.error = error;
    r.meanConsErr = mean_cons_err(A);
    *A.out = r;
  }
}

// (re)allocates the workspace for n nodes and m constraints; never shrinks
int reserve(DeformWork* w, int n, int m) {
  if (n <= w->cap_nodes && m <= w->cap_cons) return 0;
  w->arena.release();
  n = n > w->cap_nodes ? n : w->cap_nodes;
  m = m > w->cap_cons ? m : w->cap_cons;
  CU(w->arena.alloc(&w->pos, 3 * n));
  CU(w->arena.alloc(&w->ntime, n));
  CU(w->arena.alloc(&w->R, 9 * n));
  CU(w->arena.alloc(&w->t, 3 * n));
  CU(w->arena.alloc(&w->src, 3 * m));
  CU(w->arena.alloc(&w->dst, 3 * m));
  CU(w->arena.alloc(&w->ctime, m));
  CU(w->arena.alloc(&w->cnode, KNN * m));
  CU(w->arena.alloc(&w->cw, KNN * m));
  CU(w->arena.alloc(&w->list_off, n + 1));
  CU(w->arena.alloc(&w->list, KNN * m));
  CU(w->arena.alloc(&w->res_rot, 6 * n));
  CU(w->arena.alloc(&w->res_reg, 3 * NB * n));
  CU(w->arena.alloc(&w->res_con, 3 * m));
  CU(w->arena.alloc(&w->cerr, m));
  CU(w->arena.alloc(&w->band, (size_t)n * (MAXBW + 1) * 144));
  CU(w->arena.alloc(&w->linv, (size_t)n * 144));
  CU(w->arena.alloc(&w->x, (size_t)n * NV));
  CU(w->arena.alloc(&w->nodes16, 16 * n));
  CU(w->arena.alloc(&w->rt12, 12 * n));
  CU(w->arena.alloc(&w->out, 1));
  w->cap_nodes = n;
  w->cap_cons = m;
  return 0;
}

}  // namespace

void deform_free(EfContext* ctx) {
  DeformWork* w = static_cast<DeformWork*>(ctx->deform);
  if (!w) return;
  w->arena.release();
  delete w;
  ctx->deform = nullptr;
}

static DeformWork* work(EfContext* ctx) {
  if (!ctx->deform) ctx->deform = new DeformWork();
  return static_cast<DeformWork*>(ctx->deform);
}

// the one solve launch: n nodes (pos, ntime) and m constraints (src, dst, ctime) already in the workspace
static int launch_solve(EfContext* ctx, DeformWork* w, int n, int m, int last_deform_time) {
  Args a;
  a.n = n;
  a.m = m;
  a.last_deform_time = last_deform_time;
  a.pos = w->pos; a.src = w->src; a.dst = w->dst;
  a.ntime = w->ntime; a.ctime = w->ctime;
  a.R = w->R; a.t = w->t;
  a.cnode = w->cnode; a.cw = w->cw;
  a.list_off = w->list_off; a.list = w->list;
  a.res_rot = w->res_rot; a.res_reg = w->res_reg; a.res_con = w->res_con;
  a.cerr = w->cerr;
  a.band = w->band; a.linv = w->linv; a.x = w->x;
  a.nodes16 = w->nodes16;
  a.rt12 = w->rt12;
  a.out = w->out;
  EF_LAUNCH(ctx, k_deform_solve, 1, THREADS, 0, a);
  CHECK_LAST();
  return 0;
}

// Device-side inputs are uploaded from `host` (pinned by the caller or pageable); the solve itself is one launch.
int deform_solve(EfContext* ctx, const double* node_pos3, const int32_t* node_times, int n, const double* src3, const double* dst3,
                 const int32_t* src_times, int m, int last_deform_time, float* nodes16_host, double* rt12_host,
                 int32_t* cons_nodes4, double* cons_weights4, EfDeformResult* out) {
  DeformWork* w = work(ctx);
  RC(reserve(w, n, m));
  cudaStream_t st = ctx->stream;
  CU(cudaMemcpyAsync(w->pos, node_pos3, sizeof(double) * 3 * n, cudaMemcpyHostToDevice, st));
  CU(cudaMemcpyAsync(w->ntime, node_times, sizeof(int) * n, cudaMemcpyHostToDevice, st));
  CU(cudaMemcpyAsync(w->src, src3, sizeof(double) * 3 * m, cudaMemcpyHostToDevice, st));
  CU(cudaMemcpyAsync(w->dst, dst3, sizeof(double) * 3 * m, cudaMemcpyHostToDevice, st));
  CU(cudaMemcpyAsync(w->ctime, src_times, sizeof(int) * m, cudaMemcpyHostToDevice, st));
  RC(launch_solve(ctx, w, n, m, last_deform_time));
  CU(cudaMemcpyAsync(out, w->out, sizeof(EfDeformResult), cudaMemcpyDeviceToHost, st));
  if (nodes16_host) CU(cudaMemcpyAsync(nodes16_host, w->nodes16, sizeof(float) * 16 * n, cudaMemcpyDeviceToHost, st));
  if (rt12_host) CU(cudaMemcpyAsync(rt12_host, w->rt12, sizeof(double) * 12 * n, cudaMemcpyDeviceToHost, st));
  if (cons_nodes4) CU(cudaMemcpyAsync(cons_nodes4, w->cnode, sizeof(int) * KNN * m, cudaMemcpyDeviceToHost, st));
  if (cons_weights4) CU(cudaMemcpyAsync(cons_weights4, w->cw, sizeof(double) * KNN * m, cudaMemcpyDeviceToHost, st));
  CU(cudaStreamSynchronize(st));
  return 0;
}

// Solve inputs of an in-frame local closure, what Deformation::sampleGraphFrom / addConstraint / constrain hand the graph
// (Deformation.cpp:73-86, 119-132, 306-330): node positions widened to fp64 and times truncated to integers; constraint i is
// (src, dst) at time src_time, followed by its pin (dst, dst) at dst_times[i] when `pin` is set.
__global__ void k_deform_inputs(const float4* __restrict__ graph, int n, const double* __restrict__ src3, const double* __restrict__ dst3,
                                const int* __restrict__ dst_times, int n_cons, int pin, int src_time, double* __restrict__ pos,
                                int* __restrict__ ntime, double* __restrict__ src, double* __restrict__ dst, int* __restrict__ ctime) {
  pdl_enter();
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < max(n, n_cons); i += gridDim.x * blockDim.x) {
    if (i < n) {
      const float4 g = graph[i];
      pos[3 * i] = g.x;
      pos[3 * i + 1] = g.y;
      pos[3 * i + 2] = g.z;
      ntime[i] = (int)g.w;
    }
    if (i < n_cons) {
      const int o = pin ? 2 * i : i;
      for (int q = 0; q < 3; ++q) {
        src[3 * o + q] = src3[3 * i + q];
        dst[3 * o + q] = dst3[3 * i + q];
      }
      ctime[o] = src_time;
      if (pin) {
        for (int q = 0; q < 3; ++q) src[3 * (o + 1) + q] = dst[3 * (o + 1) + q] = dst3[3 * i + q];
        ctime[o + 1] = dst_times[i];
      }
    }
  }
}

// Deformation::constrain of a local closure inside the frame: inputs gathered on the device, the same solve as deform_solve,
// then the solve's result read back into `out` (pinned). *nodes16_dev: the hand-over, valid until the next solve.
int deform_solve_local(EfContext* ctx, const float4* graph, int n, const double* src3, const double* dst3, const int* dst_times, int n_cons,
                       bool pin, int src_time, int last_deform_time, EfDeformResult* out, const float** nodes16_dev) {
  DeformWork* w = work(ctx);
  const int m = pin ? 2 * n_cons : n_cons;
  RC(reserve(w, n, m));
  EF_LAUNCH(ctx, k_deform_inputs, 4, 256, 0, graph, n, src3, dst3, dst_times, n_cons, pin ? 1 : 0, src_time, w->pos, w->ntime, w->src, w->dst,
            w->ctime);
  CHECK_LAST();
  RC(launch_solve(ctx, w, n, m, last_deform_time));
  CU(cudaMemcpyAsync(out, w->out, sizeof(EfDeformResult), cudaMemcpyDeviceToHost, ctx->stream));
  CU(cudaStreamSynchronize(ctx->stream));
  *nodes16_dev = w->nodes16;
  return 0;
}

}  // namespace ef
