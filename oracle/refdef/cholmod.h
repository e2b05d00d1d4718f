// TEST INFRASTRUCTURE ONLY. Stand-in for the part of SuiteSparse CHOLMOD's API that the reference's
// Core/Utils/CholeskyDecomp.cpp calls, so that file compiles unmodified without SuiteSparse. Behind it is Eigen's
// simplicial LLᵀ in natural (identity) ordering; the permutation the reference applies is therefore the identity.
// Only real, double, packed matrices and the calls CholeskyDecomp.cpp makes are supported.
#pragma once
#include <stddef.h>

#define CHOLMOD_REAL 1
#define CHOLMOD_A 0
#define CHOLMOD_P 7
#define CHOLMOD_L 4
#define CHOLMOD_Lt 5

typedef struct cholmod_common_struct {
  int n_factorize;  // factorisations since cholmod_start (the harness reads it: one per Gauss-Newton iteration)
} cholmod_common;

typedef struct cholmod_sparse_struct {
  size_t nrow, ncol, nzmax;
  void *p, *i, *x;
  int stype, xtype, sorted, packed;
} cholmod_sparse;

typedef struct cholmod_dense_struct {
  size_t nrow, ncol, nzmax, d;
  void* x;
  int xtype;
} cholmod_dense;

typedef struct cholmod_factor_struct {
  size_t n;
  void* Perm;  // int[n], identity
  void* impl;  // the Eigen factor
} cholmod_factor;

int cholmod_start(cholmod_common* c);
int cholmod_finish(cholmod_common* c);
cholmod_sparse* cholmod_allocate_sparse(size_t nrow, size_t ncol, size_t nzmax, int sorted, int packed, int stype, int xtype,
                                        cholmod_common* c);
int cholmod_free_sparse(cholmod_sparse** A, cholmod_common* c);
cholmod_factor* cholmod_analyze(cholmod_sparse* A, cholmod_common* c);
cholmod_factor* cholmod_copy_factor(cholmod_factor* L, cholmod_common* c);
int cholmod_factorize(cholmod_sparse* A, cholmod_factor* L, cholmod_common* c);
int cholmod_change_factor(int to_xtype, int to_ll, int to_super, int to_packed, int to_monotonic, cholmod_factor* L,
                          cholmod_common* c);
int cholmod_free_factor(cholmod_factor** L, cholmod_common* c);
cholmod_dense* cholmod_zeros(size_t nrow, size_t ncol, int xtype, cholmod_common* c);
int cholmod_free_dense(cholmod_dense** X, cholmod_common* c);
int cholmod_sdmult(cholmod_sparse* A, int transpose, double alpha[2], double beta[2], cholmod_dense* X, cholmod_dense* Y,
                   cholmod_common* c);
cholmod_dense* cholmod_solve(int sys, cholmod_factor* L, cholmod_dense* B, cholmod_common* c);
