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
//
// Beyond what Ipopt resolves, the shim also serves the other MA97 callers of the same library:
//   ma97_solve_d job 1..4  the partial solves (b200ldlt_solve_partial: L, D, L^T on their own, in pivot order);
//   ma97_enquire_indef_d   the pivot order and D^-1 (b200ldlt_enquire_indef), declared at hsl_ma97d.h:158-160;
//   scale[]                of ma97_factor_d / ma97_factor_solve_d: the equilibration factors of that factorisation;
//   ma97_lmultiply_d       multiplication by S^-1 P L or its transpose (b200ldlt_lmultiply), hsl_ma97d.h:169-171;
//   ma97_alter_d           writes D^-1 back in the layout ma97_enquire_indef_d returns (b200ldlt_alter_d);
//   ma97_enquire_posdef_d  the diagonal of the Cholesky factor L D^1/2 when every pivot is a positive 1x1 pivot;
//   ma97_sparse_fwd_solve_d  job 1 of a sparse right-hand side, swept over the fronts it reaches only
//                          (b200ldlt_sparse_fwd_solve), declared at hsl_ma97d.h:173-176;
//   control->action        != 0 keeps the factors of a singular matrix whose zero pivots are all rounding noise
//                          (b200ldlt_set_singular_action): flag 7 with factors, D^+ at the zero pivots;
//   ma97_solve_fredholm_d  the Fredholm alternative on those factors (b200ldlt_solve_fredholm), hsl_ma97d.h:164-167.
// Not provided: the 64-bit variants.
// The conventions of the inspection calls (enquire_indef / enquire_posdef / alter / lmultiply / sparse_fwd_solve /
// solve_fredholm) are our reading of the reference header; they have not been checked against the HSL user documentation.
#include <cuda_runtime_api.h>

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

// the start of the entry points on an analysed matrix: info cleared, then the Keep behind *akeep, or nullptr when there
// is none or, with need_factors, it holds no factors (the caller then sets flag -1)
Keep* keep_of(void** akeep, ma97_info_d* info, bool need_factors = true) {
  memset(info, 0, sizeof(*info));
  Keep* K = akeep ? (Keep*)*akeep : nullptr;
  return K && K->h && (K->factored || !need_factors) ? K : nullptr;
}

// scale[] of the factor calls: the n equilibration factors of the factorisation just done (device_ptr "scale")
bool copy_scale(Keep* K, double* scale) {
  const void* d = b200ldlt_device_ptr(K->h, "scale");
  return d && cudaMemcpy(scale, d, (size_t)K->n * sizeof(double), cudaMemcpyDeviceToHost) == cudaSuccess;
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
  (void)ptr; (void)row;
  Keep* K = keep_of(akeep, info, false);
  if (!K || !val || (matrix_type != 4 && matrix_type != 3)) { info->flag = -1; return; }
  if (control && control->u > 0.0 && control->u != K->u) {
    b200ldlt_set_pivtol(K->h, control->u, std::fmax(control->u, 1e-4));
    K->u = control->u;
  }
  memcpy(b200ldlt_values_ptr(K->h), val, (size_t)K->nnz * sizeof(double));   // same order as the CSC entries
  const bool keep = control && control->action;
  b200ldlt_set_singular_action(K->h, keep ? 1 : 0);
  int neg = -1;
  const int st = b200ldlt_factor(K->h, 0, 0, &neg);
  fill_info(K, info);
  if (st == B200LDLT_SINGULAR) {
    // action != 0: continue on singularity -- flag 7, with the factors (D^+) when they were kept (only zero pivots)
    int nz = 0;
    K->factored = keep && b200ldlt_enquire_zero_pivots(K->h, &nz, nullptr) == B200LDLT_SUCCESS;
    info->flag = keep ? 7 : -7;
  }
  else if (st != B200LDLT_SUCCESS) { info->flag = -1; K->factored = false; }
  else { info->flag = 0; K->factored = true; }
  if (K->factored && scale && !copy_scale(K, scale)) info->flag = -1;
  if (fkeep) *fkeep = K;
}

// job 0: A x = b; 1: P L x = S b; 2: D x = b; 3: (P L)^T S^-1 x = b; 4: D (P L)^T S^-1 x = b, i.e. the jobs of
// b200ldlt_solve_partial (include/b200ldlt.h) -- intermediate vectors in pivot order
void ma97_solve_d(int job, int nrhs, double x[], int ldx, void** akeep, void** fkeep, const ma97_control_d* control,
                  ma97_info_d* info) {
  (void)control; (void)fkeep;
  Keep* K = keep_of(akeep, info);
  if (!K || job < 0 || job > 4 || nrhs < 0) { info->flag = -1; return; }
  if (nrhs == 0) return;
  int st;
  if (ldx == K->n) st = b200ldlt_solve_partial(K->h, job, nrhs, x);
  else {
    st = B200LDLT_SUCCESS;
    for (int c = 0; c < nrhs && st == B200LDLT_SUCCESS; ++c) st = b200ldlt_solve_partial(K->h, job, 1, x + (size_t)c * ldx);
  }
  fill_info(K, info);
  info->flag = (st == B200LDLT_SUCCESS) ? 0 : -1;
}

// piv_order[i] (variable i, 0-based index; values 1-based): the position of variable i in the pivot order, negative for
// both variables of a 2x2 pivot.  d[2p] / d[2p+1]: diagonal / off-diagonal (p, p+1) entry of D^-1 at pivot position p,
// the off-diagonal 0 unless p opens a 2x2 pivot.  Either output may be NULL.  This is our reading of MA97's documented
// convention; the HSL user documentation was not available to check it against, so callers that depend on the exact
// signs or on D^-1 versus D should verify it with their HSL version.
void ma97_enquire_indef_d(void** akeep, void** fkeep, const ma97_control_d* control, ma97_info_d* info, int piv_order[],
                          double d[]) {
  (void)fkeep; (void)control;
  Keep* K = keep_of(akeep, info);
  if (!K) { info->flag = -1; return; }
  std::vector<int> var, ty;
  if (piv_order) { var.resize(K->n); ty.resize(K->n); }
  if (b200ldlt_enquire_indef(K->h, piv_order ? var.data() : nullptr, piv_order ? ty.data() : nullptr, d) != B200LDLT_SUCCESS) {
    info->flag = -1;
    return;
  }
  if (piv_order)
    for (int p = 0; p < K->n; ++p) piv_order[var[p]] = ty[p] == 1 ? p + 1 : -(p + 1);
  fill_info(K, info);
  info->flag = 0;
}

// y = (S^-1 P L) x for trans = 0, its transpose for trans = 1: the operator of job 1 inverted (b200ldlt_lmultiply).
// k columns; ldx / ldy != n: column by column, as ma97_solve_d does.  k = 0 does nothing.
void ma97_lmultiply_d(int trans, int k, const double x[], int ldx, double y[], int ldy, void** akeep, void** fkeep,
                      const ma97_control_d* control, ma97_info_d* info) {
  (void)control; (void)fkeep;
  Keep* K = keep_of(akeep, info);
  if (!K || k < 0 || (trans != 0 && trans != 1) || ldx < K->n || ldy < K->n) { info->flag = -1; return; }
  if (k == 0) return;
  int st;
  if (ldx == K->n && ldy == K->n) st = b200ldlt_lmultiply(K->h, trans, k, x, y);
  else {
    st = B200LDLT_SUCCESS;
    for (int c = 0; c < k && st == B200LDLT_SUCCESS; ++c)
      st = b200ldlt_lmultiply(K->h, trans, 1, x + (size_t)c * ldx, y + (size_t)c * ldy);
  }
  fill_info(K, info);
  info->flag = (st == B200LDLT_SUCCESS) ? 0 : -1;
}

// d[2p] / d[2p+1]: the new diagonal / off-diagonal entry of D^-1 at pivot position p -- the convention of
// ma97_enquire_indef_d, so that enquire followed by alter changes nothing.  Refused (flag -1, D unchanged) for a
// non-finite entry or a non-zero off-diagonal entry where no 2x2 pivot opens.  Lasts until the next factorisation.
void ma97_alter_d(const double d[], void** akeep, void** fkeep, const ma97_control_d* control, ma97_info_d* info) {
  (void)fkeep; (void)control;
  Keep* K = keep_of(akeep, info);
  if (!K || !d) { info->flag = -1; return; }
  const int st = b200ldlt_alter_d(K->h, d);
  fill_info(K, info);
  info->flag = (st == B200LDLT_SUCCESS) ? 0 : -1;
}

// d[p] = sqrt(D_pp), pivot order: the diagonal of the Cholesky factor L D^1/2 of the scaled matrix.  Defined only when
// every pivot is a positive 1x1 pivot (a positive-definite factorisation); otherwise flag -1 and d untouched.
void ma97_enquire_posdef_d(void** akeep, void** fkeep, const ma97_control_d* control, ma97_info_d* info, double d[]) {
  (void)fkeep; (void)control;
  Keep* K = keep_of(akeep, info);
  if (!K || !d) { info->flag = -1; return; }
  std::vector<int> ty(K->n);
  std::vector<double> dinv2(2 * (size_t)K->n);
  if (b200ldlt_enquire_indef(K->h, nullptr, ty.data(), dinv2.data()) != B200LDLT_SUCCESS) { info->flag = -1; return; }
  for (int p = 0; p < K->n; ++p)
    if (ty[p] != 1 || !(dinv2[2 * (size_t)p] > 0.0)) { fill_info(K, info); info->flag = -1; return; }
  for (int p = 0; p < K->n; ++p) d[p] = std::sqrt(1.0 / dinv2[2 * (size_t)p]);
  fill_info(K, info);
  info->flag = 0;
}

// x = L^-1 P^T S b (job 1, pivot order) for a sparse b.  Our reading of the convention: b is a dense n-vector indexed by
// variable, its entries b[bindex[i]]; x is a dense n-vector in pivot order, written whole (the solve at xindex[0..*nxi),
// zeros elsewhere); bindex / xindex are 0- or 1-based as control->f_arrays says (as for ma97_analyse_d); order is ignored
// (the shim's analyse takes no user ordering).  flag -1, with nothing written, for the refusals of
// b200ldlt_sparse_fwd_solve (an index out of range or repeated, no factors).  Not checked against the HSL documentation.
void ma97_sparse_fwd_solve_d(int nbi, const int bindex[], const double b[], const int order[], int* nxi, int xindex[],
                             double x[], void** akeep, void** fkeep, const ma97_control_d* control, ma97_info_d* info) {
  (void)fkeep; (void)order;
  Keep* K = keep_of(akeep, info);
  if (!K || nbi < 0 || nbi > K->n || !nxi || !xindex || !x || (nbi > 0 && (!bindex || !b))) { info->flag = -1; return; }
  const int base = control && control->f_arrays ? 1 : 0;
  std::vector<int> bi(nbi), xi(K->n);
  std::vector<double> bv(nbi), xv(K->n);
  for (int i = 0; i < nbi; ++i) {
    bi[i] = bindex[i] - base;
    if (bi[i] < 0 || bi[i] >= K->n) { info->flag = -1; return; }
    bv[i] = b[bi[i]];
  }
  int nx = 0;
  const int st = b200ldlt_sparse_fwd_solve(K->h, nbi, bi.data(), bv.data(), &nx, xi.data(), xv.data());
  fill_info(K, info);
  if (st != B200LDLT_SUCCESS) { info->flag = -1; return; }
  memset(x, 0, (size_t)K->n * sizeof(double));
  for (int j = 0; j < nx; ++j) { x[xi[j]] = xv[j]; xindex[j] = xi[j] + base; }
  *nxi = nx;
  info->flag = 0;
}

void ma97_factor_solve_d(int matrix_type, const int ptr[], const int row[], const double val[], int nrhs, double x[], int ldx,
                         void** akeep, void** fkeep, const ma97_control_d* control, ma97_info_d* info, double scale[]) {
  ma97_factor_d(matrix_type, ptr, row, val, akeep, fkeep, control, info, scale);
  if (info->flag != 0 && info->flag != 7) return;   // flag 7 comes with factors (kept D^+)
  ma97_info_d i2;
  ma97_solve_d(0, nrhs, x, ldx, akeep, fkeep, control, &i2);
  if (i2.flag != 0) info->flag = i2.flag;
}

// Fredholm alternative (b200ldlt_solve_fredholm) of the kept factors of a singular matrix.  Our reading of the convention:
// x is ldx x 2 nrhs; on entry x(:, i) holds b_i, on exit the D^+ solution; flag_out[i] = 1 when column i is consistent
// within control->consist_tol (max over the zero pivots of |L^-1 P^T S b| <= consist_tol * its max over all pivots),
// else 0, and then x(:, nrhs + i) holds f_i with A f_i = 0 and b_i^T f_i > 0; for consistent columns x(:, nrhs + i) is
// left untouched.  ldx != n: column by column, as ma97_solve_d does.  Neither this convention nor the scaling of
// consist_tol has been checked against the HSL documentation; with MA97's default consist_tol (machine epsilon) only
// columns whose components on the zero pivots are exactly zero count as consistent.
void ma97_solve_fredholm_d(int nrhs, int flag_out[], double x[], int ldx, void** akeep, void** fkeep,
                           const ma97_control_d* control, ma97_info_d* info) {
  (void)fkeep;
  Keep* K = keep_of(akeep, info);
  if (!K || nrhs < 0 || ldx < K->n || (nrhs > 0 && (!x || !flag_out))) { info->flag = -1; return; }
  if (nrhs == 0) return;
  const double tol = control ? control->consist_tol : 2.220446049250313e-16;
  const size_t n = (size_t)K->n;
  const bool whole = ldx == K->n;
  const int cols = whole ? nrhs : 1;
  std::vector<double> buf(n * 2 * (size_t)cols);
  std::vector<int> cons((size_t)cols);
  int st = B200LDLT_SUCCESS;
  for (int c0 = 0; c0 < nrhs && st == B200LDLT_SUCCESS; c0 += cols) {
    for (int i = 0; i < cols; ++i) memcpy(buf.data() + i * n, x + (size_t)(c0 + i) * ldx, n * sizeof(double));
    st = b200ldlt_solve_fredholm(K->h, cols, tol, buf.data(), cons.data());
    if (st != B200LDLT_SUCCESS) break;
    for (int i = 0; i < cols; ++i) {
      memcpy(x + (size_t)(c0 + i) * ldx, buf.data() + i * n, n * sizeof(double));
      flag_out[c0 + i] = cons[i];
      if (!cons[i]) memcpy(x + (size_t)(nrhs + c0 + i) * ldx, buf.data() + (cols + i) * n, n * sizeof(double));
    }
  }
  fill_info(K, info);
  info->flag = (st == B200LDLT_SUCCESS) ? 0 : -1;
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
