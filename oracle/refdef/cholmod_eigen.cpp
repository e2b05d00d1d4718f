// TEST INFRASTRUCTURE ONLY. The cholmod_* calls of cholmod.h on top of Eigen's SimplicialLLT (natural ordering).
// A is stored as CHOLMOD stores Jᵀ for CholeskyDecomp.cpp: nrow = unknowns, ncol = Jacobian rows, column-compressed, so
// cholmod_factorize(A) factorises A·Aᵀ = JᵀJ.
#include "cholmod.h"

#include <Eigen/Sparse>
#include <Eigen/SparseCholesky>
#include <string.h>

namespace {
using Sp = Eigen::SparseMatrix<double>;
using LLT = Eigen::SimplicialLLT<Sp, Eigen::Lower, Eigen::NaturalOrdering<int>>;

Sp as_eigen(const cholmod_sparse* A) {
  const int* p = (const int*)A->p;
  const int* i = (const int*)A->i;
  const double* x = (const double*)A->x;
  std::vector<Eigen::Triplet<double>> t;
  for (size_t c = 0; c < A->ncol; ++c)
    for (int k = p[c]; k < p[c + 1]; ++k) t.emplace_back(i[k], (int)c, x[k]);
  Sp m((Eigen::Index)A->nrow, (Eigen::Index)A->ncol);
  m.setFromTriplets(t.begin(), t.end());
  return m;
}

cholmod_factor* new_factor(size_t n) {
  cholmod_factor* L = new cholmod_factor;
  L->n = n;
  int* perm = new int[n ? n : 1];
  for (size_t k = 0; k < n; ++k) perm[k] = (int)k;
  L->Perm = perm;
  L->impl = nullptr;
  return L;
}
}  // namespace

int cholmod_start(cholmod_common* c) {
  c->n_factorize = 0;
  return 1;
}
int cholmod_finish(cholmod_common*) { return 1; }

cholmod_sparse* cholmod_allocate_sparse(size_t nrow, size_t ncol, size_t nzmax, int sorted, int packed, int stype, int xtype,
                                        cholmod_common*) {
  cholmod_sparse* A = new cholmod_sparse;
  A->nrow = nrow;
  A->ncol = ncol;
  A->nzmax = nzmax;
  A->p = new int[ncol + 1]();
  A->i = new int[nzmax ? nzmax : 1];
  A->x = new double[nzmax ? nzmax : 1];
  A->stype = stype;
  A->xtype = xtype;
  A->sorted = sorted;
  A->packed = packed;
  return A;
}

int cholmod_free_sparse(cholmod_sparse** A, cholmod_common*) {
  if (!A || !*A) return 1;
  delete[](int*)(*A)->p;
  delete[](int*)(*A)->i;
  delete[](double*)(*A)->x;
  delete *A;
  *A = nullptr;
  return 1;
}

cholmod_factor* cholmod_analyze(cholmod_sparse* A, cholmod_common*) { return new_factor(A->nrow); }

cholmod_factor* cholmod_copy_factor(cholmod_factor* L, cholmod_common*) { return new_factor(L->n); }

int cholmod_factorize(cholmod_sparse* A, cholmod_factor* L, cholmod_common* c) {
  c->n_factorize++;
  const Sp J = as_eigen(A);
  const Sp AtA = (J * J.transpose()).pruned(0.0);
  LLT* f = new LLT();
  if (L->n > 0) f->compute(AtA);
  delete (LLT*)L->impl;
  L->impl = f;
  return 1;
}

int cholmod_change_factor(int, int, int, int, int, cholmod_factor*, cholmod_common*) { return 1; }

int cholmod_free_factor(cholmod_factor** L, cholmod_common*) {
  if (!L || !*L) return 1;
  delete (LLT*)(*L)->impl;
  delete[](int*)(*L)->Perm;
  delete *L;
  *L = nullptr;
  return 1;
}

cholmod_dense* cholmod_zeros(size_t nrow, size_t ncol, int xtype, cholmod_common*) {
  cholmod_dense* X = new cholmod_dense;
  X->nrow = nrow;
  X->ncol = ncol;
  X->nzmax = X->d = nrow;
  X->nzmax = nrow * ncol;
  X->x = new double[nrow * ncol ? nrow * ncol : 1]();
  X->xtype = xtype;
  return X;
}

int cholmod_free_dense(cholmod_dense** X, cholmod_common*) {
  if (!X || !*X) return 1;
  delete[](double*)(*X)->x;
  delete *X;
  *X = nullptr;
  return 1;
}

// Y = alpha A X + beta Y (transpose = 0 only)
int cholmod_sdmult(cholmod_sparse* A, int transpose, double alpha[2], double beta[2], cholmod_dense* X, cholmod_dense* Y,
                   cholmod_common*) {
  if (transpose) return 0;
  const Sp M = as_eigen(A);
  Eigen::Map<const Eigen::VectorXd> x((const double*)X->x, (Eigen::Index)X->nrow);
  Eigen::Map<Eigen::VectorXd> y((double*)Y->x, (Eigen::Index)Y->nrow);
  const Eigen::VectorXd r = M * x;
  y = alpha[0] * r + beta[0] * y;
  return 1;
}

cholmod_dense* cholmod_solve(int sys, cholmod_factor* L, cholmod_dense* B, cholmod_common* c) {
  cholmod_dense* X = cholmod_zeros(B->nrow, 1, CHOLMOD_REAL, c);
  Eigen::Map<const Eigen::VectorXd> b((const double*)B->x, (Eigen::Index)B->nrow);
  Eigen::Map<Eigen::VectorXd> x((double*)X->x, (Eigen::Index)X->nrow);
  const LLT* f = (const LLT*)L->impl;
  if (sys == CHOLMOD_P || B->nrow == 0) x = b;  // identity permutation
  else if (sys == CHOLMOD_L) x = f->matrixL().solve(b);
  else if (sys == CHOLMOD_Lt) x = f->matrixU().solve(b);
  else x = f->solve(b);
  return X;
}
