// HSL_MA97 C-interface shim over the b200ldlt handle (SURVEY.md 8b' / 8f-3).
//
// Stock Ipopt binaries load their HSL solvers at run time: with  linear_solver=ma97  and  hsllib=<this library>  the
// reference's Ma97SolverInterface dlopen()s the library and resolves exactly seven symbols
// (reference src/Algorithm/LinearSolvers/IpMa97SolverInterface.cpp:303-314):
//   ma97_default_control_d, ma97_analyse_d, ma97_factor_d, ma97_factor_solve_d, ma97_solve_d, ma97_finalise_d,
//   ma97_free_akeep_d
// with the prototypes and the ma97_control_d / ma97_info_d layouts of reference
// src/Algorithm/LinearSolvers/hsl_ma97d.h:67-178.  This file exports those seven entry points on top of the GPU
// backend, so an UNMODIFIED Ipopt (AMPL ipopt, cyipopt, ...) runs its KKT factorisations on the GPU with an options-file
// change only.  How the adapter uses them: :473-608 (analyse: CSC lower triangle, 1-based when f_arrays != 0, values may
// be NULL), :610-800 (factor with matrix_type 4 = real symmetric indefinite, then solve job 0; info.num_neg is the
// inertia; info.flag 7 / -7 = singular), :802-860 (IncreaseQuality raises control.u and re-factors).
#include <cmath>
#include <cstdio>
#include <cstring>
#include <vector>

#include "../../include/b200ldlt.h"

extern "C" {

// ---- ABI structs: field order / types as in hsl_ma97d.h:67-134 (double precision interface) ----------------------
struct ma97_control_d {
  int f_arrays;
  int action;
  int nemin;
  double multiplier;
  int ordering;
  int print_level;
  int scaling;
  double small_;             /* "small" in the reference header (a macro on some platforms) */
  double u;
  int unit_diagnostics;
  int unit_error;
  int unit_warning;
  long factor_min;
  int solve_blas3;
  long solve_min;
  int solve_mf;
  double consist_tol;
  int ispare[5];
  double rspare[10];
};

struct ma97_info_d {
  int flag;
  int flag68;
  int flag77;
  int matrix_dup;
  int matrix_rank;
  int matrix_outrange;
  int matrix_missing_diag;
  int maxdepth;
  int maxfront;
  int num_delay;
  long num_factor;
  long num_flops;
  int num_neg;
  int num_sup;
  int num_two;
  int ordering;
  int stat;
  int maxsupernode;
  int ispare[4];
  double rspare[10];
};

}  // extern "C"

namespace {

struct Keep {                 // what *akeep (and *fkeep) point to
  b200ldlt_handle h = nullptr;
  int n = 0;
  long nnz = 0;
  double u = -1.0;
  bool factored = false;
};

void fill_info(Keep* K, ma97_info_d* info) {
  memset(info, 0, sizeof(*info));
  if (!K || !K->h) { info->flag = -1; return; }
  b200ldlt_info bi;
  if (b200ldlt_get_info(K->h, &bi) != B200LDLT_SUCCESS) { info->flag = -1; return; }
  info->matrix_rank = K->n - bi.num_tiny;
  info->maxdepth = bi.nlevels;
  info->maxfront = bi.max_front;
  info->maxsupernode = bi.max_pivots;
  info->num_delay = 0;                    // static fronts: no delayed pivots (forced pivots are reported by b200ldlt_info)
  info->num_factor = (long)bi.nnz_L;
  info->num_flops = (long)(bi.flops_panel + bi.flops_schur);
  info->num_neg = bi.num_neg;
  info->num_sup = bi.nsupernodes;
  info->num_two = bi.num_2x2;
  info->ordering = 3;                     // nested dissection (METIS)
}

}  // namespace

extern "C" {

void ma97_free_akeep_d(void** akeep);

void ma97_default_control_d(ma97_control_d* c) {
  memset(c, 0, sizeof(*c));
  c->f_arrays = 0;          // C numbering by default (hsl_ma97d.h: "Use C or Fortran numbering")
  c->action = 1;
  c->nemin = 8;
  c->multiplier = 1.1;
  c->ordering = 5;
  c->print_level = 0;
  c->scaling = 0;
  c->small_ = 1e-20;
  c->u = 0.01;
  c->unit_diagnostics = 6; c->unit_error = 6; c->unit_warning = 6;
  c->factor_min = 20000000; c->solve_blas3 = 0; c->solve_min = 100000; c->solve_mf = 0;
  c->consist_tol = 2.220446049250313e-16;
}

// sparse column entry (lower triangle): ptr[n+1], row[ptr[n]-base]; check is ignored (the backend sums duplicates and
// accepts either triangle); order (user ordering) must be NULL
void ma97_analyse_d(int check, int n, const int ptr[], const int row[], double val[], void** akeep,
                    const ma97_control_d* control, ma97_info_d* info, int order[]) {
  (void)check; (void)val;
  memset(info, 0, sizeof(*info));
  if (!akeep || n <= 0 || !ptr || !row || order != nullptr) { info->flag = -1; return; }
  const int base = control && control->f_arrays ? 1 : 0;
  const long nnz = (long)ptr[n] - base;
  if (nnz < 0 || nnz > 2147483647L) { info->flag = -1; return; }
  std::vector<int> irn((size_t)nnz), jcn((size_t)nnz);
  for (int j = 0; j < n; ++j)
    for (long p = (long)ptr[j] - base; p < (long)ptr[j + 1] - base; ++p) {
      irn[(size_t)p] = row[p] - base + 1;      // the C ABI takes 1-based triplets
      jcn[(size_t)p] = j + 1;
    }
  if (*akeep) ma97_free_akeep_d(akeep);      // re-analysis on a live handle (delayed analyse, IpMa97SolverInterface.cpp:654-677)
  Keep* K = new Keep();
  b200ldlt_options o;
  b200ldlt_default_options(&o);
  if (control && control->u > 0.0) { o.pivtol = control->u; o.pivtolmax = std::fmax(o.pivtolmax, control->u); }
  K->h = b200ldlt_create(&o);
  if (!K->h) { delete K; info->flag = -1; return; }   // no CUDA device: fail loudly (message printed by b200ldlt_create)
  if (b200ldlt_analyse(K->h, n, (int)nnz, irn.data(), jcn.data()) != B200LDLT_SUCCESS) {
    fprintf(stderr, "[b200ldlt/ma97 shim] analyse failed: %s\n", b200ldlt_last_error(K->h));
    b200ldlt_destroy(K->h); delete K; info->flag = -1; return;
  }
  K->n = n; K->nnz = nnz;
  *akeep = K;
  info->flag = 0;
  info->ordering = 3;
  // predicted factor size / flops are only known after the (lazy, value-dependent) ordering; report the matrix size so a
  // caller comparing two orderings (ma97_order=auto, IpMa97SolverInterface.cpp:510-548) sees a tie and keeps either
  info->num_factor = nnz; info->num_flops = nnz; info->maxfront = 0;
}

void ma97_factor_d(int matrix_type, const int ptr[], const int row[], const double val[], void** akeep, void** fkeep,
                   const ma97_control_d* control, ma97_info_d* info, double scale[]) {
  (void)ptr; (void)row; (void)scale;
  memset(info, 0, sizeof(*info));
  Keep* K = akeep ? (Keep*)*akeep : nullptr;
  if (!K || !K->h || !val || (matrix_type != 4 && matrix_type != 3)) { info->flag = -1; return; }
  if (control && control->u > 0.0 && control->u != K->u) {
    b200ldlt_set_pivtol(K->h, control->u, std::fmax(control->u, 1e-4));
    K->u = control->u;
  }
  memcpy(b200ldlt_values_ptr(K->h), val, (size_t)K->nnz * sizeof(double));   // same order as the CSC entries
  int neg = -1;
  const int st = b200ldlt_factor(K->h, 0, 0, &neg);
  fill_info(K, info);
  if (st == B200LDLT_SINGULAR) { info->flag = (control && control->action) ? 7 : -7; K->factored = false; }
  else if (st != B200LDLT_SUCCESS) { info->flag = -1; K->factored = false; }
  else { info->flag = 0; K->factored = true; }
  if (fkeep) *fkeep = K;
}

void ma97_solve_d(int job, int nrhs, double x[], int ldx, void** akeep, void** fkeep, const ma97_control_d* control,
                  ma97_info_d* info) {
  (void)control; (void)fkeep;
  memset(info, 0, sizeof(*info));
  Keep* K = akeep ? (Keep*)*akeep : nullptr;
  if (!K || !K->h || !K->factored || job != 0 || nrhs < 0) { info->flag = -1; return; }
  if (nrhs == 0) return;
  int st;
  if (ldx == K->n) st = b200ldlt_solve(K->h, nrhs, x);
  else {
    st = B200LDLT_SUCCESS;
    for (int c = 0; c < nrhs && st == B200LDLT_SUCCESS; ++c) st = b200ldlt_solve(K->h, 1, x + (size_t)c * ldx);
  }
  fill_info(K, info);
  info->flag = (st == B200LDLT_SUCCESS) ? 0 : -1;
}

void ma97_factor_solve_d(int matrix_type, const int ptr[], const int row[], const double val[], int nrhs, double x[], int ldx,
                         void** akeep, void** fkeep, const ma97_control_d* control, ma97_info_d* info, double scale[]) {
  ma97_factor_d(matrix_type, ptr, row, val, akeep, fkeep, control, info, scale);
  if (info->flag != 0) return;
  ma97_info_d i2;
  ma97_solve_d(0, nrhs, x, ldx, akeep, fkeep, control, &i2);
  if (i2.flag != 0) info->flag = i2.flag;
}

void ma97_free_akeep_d(void** akeep) {
  if (!akeep || !*akeep) return;
  Keep* K = (Keep*)*akeep;
  if (K->h) b200ldlt_destroy(K->h);
  delete K;
  *akeep = nullptr;
}

void ma97_free_fkeep_d(void** fkeep) { if (fkeep) *fkeep = nullptr; }   // the factors live in the handle behind akeep

void ma97_finalise_d(void** akeep, void** fkeep) {
  if (fkeep) *fkeep = nullptr;
  ma97_free_akeep_d(akeep);
}

}  // extern "C"
