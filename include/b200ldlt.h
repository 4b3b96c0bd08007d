/* b200ldlt -- C ABI of the H100-native sparse symmetric-indefinite LDL^T backend.
 *
 * This is the drop-in boundary: one entry point per virtual of Ipopt's
 * SparseSymLinearSolverInterface (reference file
 * src/Algorithm/LinearSolvers/IpSparseSymLinearSolverInterface.hpp:98-256), so the
 * reference-side binding (ipopt_b200/plugin/B200LdltSolverInterface.cpp, shown in
 * INTEGRATION.md) is a 1:1 forwarding adapter, exactly like the reference's own
 * vendor adapters (e.g. IpMumpsSolverInterface.cpp:247-306).
 *
 * Plain C types only; no C++/torch types cross this boundary.  All calls on one
 * handle must come from one thread at a time (the reference's caller is
 * single-threaded per solver instance); different handles are independent.
 * The library FAILS LOUDLY (B200LDLT_FATAL_ERROR + message) when no CUDA device is
 * usable -- there is no CPU fallback.
 */
#ifndef B200LDLT_H
#define B200LDLT_H
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* == Ipopt::ESymSolverStatus, src/Algorithm/LinearSolvers/IpSymLinearSolver.hpp:19-33 (same order) */
enum {
  B200LDLT_SUCCESS = 0,
  B200LDLT_SINGULAR = 1,
  B200LDLT_WRONG_INERTIA = 2,
  B200LDLT_CALL_AGAIN = 3,
  B200LDLT_FATAL_ERROR = 4
};

typedef struct b200ldlt_s* b200ldlt_handle;

typedef struct b200ldlt_options {
  int device;          /* CUDA ordinal; -1 = current device */
  void* stream;        /* cudaStream_t to enqueue on; NULL = library-owned stream */
  int ordering;        /* 0 = METIS nested dissection on the pair-compressed graph, 1 = natural */
  int pair_saddle;     /* 1 = match zero-diagonal rows to a primal neighbour (2x2 pivots stay in-supernode) */
  int leaf_k;          /* merge elimination subtrees of <= leaf_k columns into one front */
  double relax_frac;   /* relaxed amalgamation: tolerated fraction of explicit zeros */
  int scaling;         /* 0 = none, >0 = number of symmetric inf-norm equilibration sweeps (power-of-two factors) */
  double pivtol;       /* threshold u of the 1x1/2x2 pivot test; cf. MA57 default 1e-8 (IpMa57TSolverInterface.cpp) */
  double pivtolmax;    /* cap for increase_quality; cf. ma57_pivtolmax 1e-4 */
  double tiny;         /* |pivot| below this (after scaling) is treated as zero -> SINGULAR */
  int smem_front_max;  /* fronts of order <= this are factored by one CTA in shared memory */
  int use_graph;       /* 1 = replay the factorisation from a CUDA graph; any other value = plain launches */
  int verbose;
  int tc_schur_min_r;  /* fronts with >= this many contribution rows form their Schur complement on the tensor cores
                          (wgmma int8 Ozaki split, csrc/schur_tc.cu); 0 = off (FP64 DFMA tiles everywhere) */
} b200ldlt_options;

/* statistics of the last analyse/factor/solve (algorithmic work per SURVEY.md section 8d) */
typedef struct b200ldlt_info {
  int n;
  int64_t nnz_in, nnz_unique;
  int nsupernodes, nlevels, max_front, max_pivots;
  int n_saddle, n_pairs;
  int64_t nnz_L;            /* sum k(k+1)/2 + k r over fronts (stored L incl. amalgamation zeros) */
  int64_t nnz_L_true;       /* column counts before amalgamation */
  int64_t L_bytes, cb_bytes; /* device storage */
  double flops_panel;       /* sum k^3/3 + k^2 r */
  double flops_schur;       /* sum k r (r+1) */
  double t_order_s, t_symbolic_s;
  /* last factorisation */
  int num_neg, num_forced, num_tiny, num_growth, num_2x2;
  float ms_factor_gpu, ms_solve_gpu;   /* CUDA-event time of the last factor / solve (device part only) */
  int launches_factor, launches_solve; /* kernel launches enqueued by the last factor / solve */
} b200ldlt_info;

void b200ldlt_default_options(b200ldlt_options* opt);

/* Create a solver instance. Returns NULL (and prints the reason to stderr) when no CUDA device is usable. */
b200ldlt_handle b200ldlt_create(const b200ldlt_options* opt);
void b200ldlt_destroy(b200ldlt_handle h);
const char* b200ldlt_last_error(b200ldlt_handle h);

/* <-> InitializeStructure(dim, nonzeros, ia, ja) (IpSparseSymLinearSolverInterface.hpp:139-144).
 * Triplets are 1-based, either triangle, duplicates are summed. The pattern is copied. The
 * ordering/symbolic phase runs lazily at the first factor call (it looks at the values of the
 * first matrix to pair saddle rows), like MUMPS job=1 in IpMumpsSolverInterface.cpp:385-446. */
int b200ldlt_analyse(b200ldlt_handle h, int dim, int nonzeros, const int* irn, const int* jcn);

/* <-> GetValuesArrayPtr() (hpp:155): pinned host array of >= nonzeros doubles, owned by the handle. */
double* b200ldlt_values_ptr(b200ldlt_handle h);

/* <-> MultiSolve(new_matrix=true, ..., check_NegEVals, numberOfNegEVals) part 1 (hpp:190-198):
 * numeric LDL^T of the values currently in values_ptr (H2D copy inside). *num_neg is always set.
 * Returns SUCCESS, SINGULAR, WRONG_INERTIA (only if check_inertia) or FATAL_ERROR. */
int b200ldlt_factor(b200ldlt_handle h, int check_inertia, int expected_neg, int* num_neg);
/* Same, values already resident in device memory (nonzeros doubles). */
int b200ldlt_factor_device(b200ldlt_handle h, const double* d_vals, int check_inertia, int expected_neg, int* num_neg);

/* <-> MultiSolve part 2: rhs is dim x nrhs column-major, overwritten with the solution (host memory).
 * nrhs > 1: the columns are solved in blocks of up to 8 (environment B200_SOLVE_BLOCK=n at b200ldlt_create caps the
 * width, 1 = one solve per column), one forward and one backward sweep per block; every column is bit-identical to a
 * solve of that column alone.  The first such call after an analysis allocates per-column device state for the full width
 * (before its timing starts); if that allocation fails, the columns are solved one by one.  Refusals, timing and
 * calls without columns: see the head of the next section. */
int b200ldlt_solve(b200ldlt_handle h, int nrhs, double* rhs);
/* Same with a device-resident rhs/solution. */
int b200ldlt_solve_device(b200ldlt_handle h, int nrhs, double* d_rhs);

/* ---- partial solves and factor inspection (cf. MA57 / HSL_MA97 job 1-4, Pardiso phases 331-333) ---------------------
 * The calls that read the factors -- solve and the calls below -- share three rules:
 *   refusals : FATAL_ERROR with "<call>: <reason>" in last_error and nothing written, first for the call's own
 *              arguments (listed with each call), then without factors (never factorised, after a SINGULAR factorisation
 *              outside keep mode, after a lifted zero), on a sharded handle -- solve, enquire_indef and
 *              enquire_zero_pivots accept a sharded handle -- and in Schur mode ("<call>: Schur mode", see
 *              b200ldlt_set_schur; solve_refine_device too), where only the Schur calls read the factors;
 *   timing   : info.launches_solve counts the call's kernel launches and info.ms_solve_gpu is its device time (host entry
 *              point: with its copies); per-analysis state a call builds at its first use is built before its timing
 *              starts (alter_d, enquire_indef and enquire_zero_pivots are not timed and leave both as they are);
 *   no columns: nrhs <= 0 for solve, solve_partial and lmultiply, nrhs = 0 for solve_fredholm and nbi = 0 for
 *              sparse_fwd_solve succeed, write nothing to the caller's arrays, launch nothing and set launches_solve and
 *              ms_solve_gpu to 0.
 * Host entry points copy through pinned staging owned by the handle, which grows to the largest call and is freed by
 * the next analysis.
 * The factor call computes  S A S = P L D L^T P^T :  S the diagonal (power-of-two) equilibration of that call
 * (device_ptr "scale"), P the fill-reducing permutation composed with the pivoting inside the supernodes, L unit lower
 * triangular, D block diagonal with 1x1 and 2x2 blocks.  Intermediate vectors are indexed by PIVOT POSITION p = 0..n-1.
 *   job 0 : x = A^-1 b                      (= b200ldlt_solve)
 *   job 1 : x = L^-1 P^T S b                original -> pivot order
 *   job 2 : x = D^-1 b                      pivot -> pivot
 *   job 3 : x = S P L^-T b                  pivot -> original
 *   job 4 : x = S P L^-T D^-1 b             pivot -> original
 * job 3 . 2 . 1 = job 4 . 1 = job 0, bit for bit: the parts run the arithmetic of the full solve.  nrhs > 1 is blocked
 * like b200ldlt_solve, and every column is bit-identical to a partial solve of that column alone.  Kernel launches per
 * block: job 1, 3, 4: 5 and job 2: 1 (job 0: 8) -- with the default B200_SOLVE_DIRECT=2; in general job 1, 3, 4 take
 * 3 + D and job 0 takes 4 + 2 D for D direct levels.  Refused: a job outside 0..4.  With info.num_forced > 0, D holds
 * the lifted pivots: the parts describe the perturbed matrix. */
int b200ldlt_solve_partial(b200ldlt_handle h, int job, int nrhs, double* rhs);
int b200ldlt_solve_partial_device(b200ldlt_handle h, int job, int nrhs, double* d_rhs);
/* Per pivot position p (any pointer may be NULL): pivot_var[p] = the 0-based original variable; pivot_type[p] = 1 (1x1),
 * 2 (first of a 2x2), 3 (second of a 2x2); dinv2[2p] = diagonal entry of D^-1, dinv2[2p+1] = off-diagonal entry
 * (p, p+1) of D^-1 when p opens a 2x2 pivot, else 0.  D^-1 is that of the scaled matrix S A S. */
int b200ldlt_enquire_indef(b200ldlt_handle h, int* pivot_var, int* pivot_type, double* dinv2);
/* Sparse forward solve (cf. HSL_MA97 ma97_sparse_fwd_solve): job 1 for a right-hand side b with few non-zeros, at a cost
 * that follows the non-zeros instead of the whole elimination tree.  bindex[0..nbi) are the distinct 0-based original
 * variables where b is non-zero, b[i] the value at bindex[i] (compact: nbi values).  The non-zeros of L^-1 P^T S b lie in
 * the REACH: the fronts on the tree paths from the fronts of those variables to the root.  On return *nxi is the number
 * of pivot positions of the reach, xindex[0..nxi) those positions in ascending order (position p belongs to front s when
 * sn_start[s] <= p < sn_start[s+1]) and x[i] the entry of job 1's vector at xindex[i]; every entry of job 1's vector
 * outside xindex is zero.  The forward sweep runs job 1's own front routines over the lists of the full solve pruned to
 * the fronts of the reach (and the fronts that share a work item with one), so x[i] equals job 1 on the dense b at
 * that position as a value (they may differ in the sign of a zero), and repeated calls give the same bits.
 * Device entry point: only the values are device memory -- d_b (nbi doubles) and d_x (room for n doubles); bindex,
 * nxi and xindex are host memory in both entry points (the pruned work lists are built on the host from the pattern).
 * Kernel launches: 2 + d + t, where d is the number of the B200_SOLVE_DIRECT bottom tree levels that hold a front of
 * the reach solved by the direct kernel, and t = 1 when the reach has a front above those levels (always, unless the
 * whole tree is made of direct fronts), else 0.
 * Memory of the three calls that prune sweeps (this one, b200ldlt_sparse_solve and b200ldlt_inverse_entries): the first
 * of them after an analysis builds, before its timing starts, host-side indices into the solve's forward and backward
 * work lists and the marks of a pruned sweep (ints per front, per variable and per top task).  Each call stages its
 * pruned lists and position lists in one pinned and device staging that the three calls share, which grows to the
 * largest call and is freed by the next analysis.  A handle that never makes such a call allocates none of it.  Here the
 * staging holds the pruned lists, 8 bytes per position of the run set and 4 per position of the reach; the host entry
 * point copies b in and x out through the staging of the other host entry points.
 * Refused (nothing written to nxi, xindex or x): nbi < 0 or nbi > n, a NULL pointer with nbi > 0, an index out of range
 * or repeated.  nbi = 0 sets *nxi = 0. */
int b200ldlt_sparse_fwd_solve(b200ldlt_handle h, int nbi, const int* bindex, const double* b, int* nxi, int* xindex, double* x);
int b200ldlt_sparse_fwd_solve_device(b200ldlt_handle h, int nbi, const int* bindex, const double* d_b, int* nxi, int* xindex,
                                     double* d_x);

/* ---- sparse solve: chosen entries of A^-1 b for a sparse b (cf. Pardiso iparm(31), MUMPS ICNTL(20)) -------------------
 * nrhs columns b_c that share one pattern, and the entries of x_c = M b_c at chosen variables; M as for selected inversion
 * below (A^-1, the perturbed matrix's inverse with info.num_forced > 0, D^+ on kept singular factors, the altered D after
 * alter_d): the operator of job 0.  Column c of b is compact: b[c*nbi + i] is its value at variable bindex[i], and it is
 * zero elsewhere.  On return x[c*nxs + i] is entry xsel[i] of x_c.  The indices are 0-based original variables in host
 * memory for both entry points; bindex entries are distinct, xsel entries may repeat and come in any order.
 *   bindex == NULL (nbi = n): b is dense (b[c*n + v] at variable v); the forward stage is job 0's;
 *   xsel == NULL (nxs = n):   every entry (x[c*n + v]); the backward stage and the output are job 0's;
 *   both NULL:                the call IS b200ldlt_solve on b: the same launches and the same bits.
 * x_c = S P L^-T D^-1 L^-1 P^T S b_c.  L^-1 P^T S b_c is non-zero only on the REACH of bindex (sparse_fwd_solve), and the
 * entries at xsel need L^-T only on the reach of xsel: the fronts on the tree paths from their fronts to the root.  The
 * forward sweep runs job 0's front routines (D^-1 applied as the fused sweep applies it) over the run set R_f of bindex
 * -- the work lists of the full solve pruned to the reach and the fronts that share a work item with one, as in
 * sparse_fwd_solve -- and the backward sweep runs job 0's over the run set R_b of xsel, pruned the same way over the
 * backward lists.  The fronts of R_b outside R_f start the backward sweep from zero.  Both run sets are built once per
 * call and shared by every column, with a check that refuses, before anything is launched, a pruned sweep that could
 * wait forever.
 * Values: every returned entry equals job 0 on the dense b as a value (the two may differ in the sign of a zero, as
 * sparse_fwd_solve allows).  Repeated calls, both entry points and any B200_SOLVE_BLOCK give the same bits, and every
 * column is bit-identical to a call on that column alone.
 * Kernel launches per block of up to B200_SOLVE_BLOCK columns (blocked as b200ldlt_solve is):
 *   1 (input) + d_f + t_f + 1 (between the sweeps) + d_b + t_b + 1 (output)
 * with d_f and t_f counted as for sparse_fwd_solve on the reach of bindex (d_f: the B200_SOLVE_DIRECT bottom levels that
 * hold a direct front of R_f, t_f = 1 when R_f has a front above them), d_b and t_b the same counts for R_b; a dense b
 * gives d_f = D and t_f = 1, a full selection d_b = D and t_b = 1 (D = the direct levels that hold any front).  With both
 * NULL: job 0's 4 + 2 D.  nbi = 0 is a zero b: d_f = t_f = 0.
 * Memory: as stated at b200ldlt_sparse_fwd_solve for the three calls that prune sweeps; here the staging holds both
 * pruned lists and the position lists (4 bytes per position of R_f twice, per zeroed position and per selected
 * entry).  symbolic_array "sparse_solve_fwd_run_set" and "sparse_solve_bwd_run_set" return the run sets of the last call
 * (every front for a dense b / a full selection), ascending; the call leaves "sparse_run_set", "inverse_run_set", the
 * factors, D and every later solve as they were.
 * Refused (FATAL_ERROR with "sparse_solve: <reason>", nothing written to x): nrhs < 0, nbi < 0 or nbi > n, nxs < 0; a
 * NULL b with nrhs, nbi > 0 or a NULL x with nrhs, nxs > 0; a NULL bindex with nbi != n or a NULL xsel with nxs != n; an
 * index out of range or a repeated bindex entry; the failed dependency check; a failed staging allocation.
 * nrhs = 0 or nxs = 0 is the no-columns case.  Device entry point: d_b (nrhs*nbi doubles) and d_x (nrhs*nxs) are
 * device memory. */
int b200ldlt_sparse_solve(b200ldlt_handle h, int nrhs, int nbi, const int* bindex, const double* b, int nxs, const int* xsel,
                          double* x);
int b200ldlt_sparse_solve_device(b200ldlt_handle h, int nrhs, int nbi, const int* bindex, const double* d_b, int nxs,
                                 const int* xsel, double* d_x);

/* ---- multiplication by the factors and alteration of D (cf. HSL_MA97 ma97_lmultiply / ma97_alter) --------------------
 * Same conventions as the partial solves (S A S = P L D L^T P^T, vectors in pivot order indexed by pivot position p):
 *   trans = 0 :  y = S^-1 P L x        x in pivot order, y in original order   (the inverse of job 1)
 *   trans = 1 :  y = L^T P^T S^-1 x    x in original order, y in pivot order   (the inverse of job 3)
 * x and y are n x nrhs column-major; they may be the same array (in place), otherwise they must not overlap.  L is read
 * as the factorisation left it, so  lmultiply(0, D lmultiply(1, v))  =  A v  up to rounding (with
 * info.num_forced > 0: the perturbed matrix).  Results are bit-reproducible; nrhs > 1 runs in blocks of up to 8 columns
 * (B200_SOLVE_BLOCK, as for the solves), L streamed once per block, every column bit-identical to a call on that column
 * alone.  Kernel launches: 2 per block (trans 0: multiply + gather; trans 1: copy-in + multiply).  The first call after
 * an analysis builds the work lists and slot map (about 8 bytes per panel row and column chunk: 9 MB per column at
 * MBndryCntrl1 N=400); a handle that never multiplies allocates none of it.  Refused: trans other than 0 / 1. */
int b200ldlt_lmultiply(b200ldlt_handle h, int trans, int nrhs, const double* x, double* y);
int b200ldlt_lmultiply_device(b200ldlt_handle h, int trans, int nrhs, const double* d_x, double* d_y);
/* Replace D^-1 by the caller's, 2n doubles in the layout of enquire_indef (dinv2[2p] diagonal, dinv2[2p+1] off-diagonal
 * (p, p+1), host memory); the pivot types stay.  Refused -- and D left exactly as it was -- for a NULL dinv2, and when
 * an entry is not finite or an off-diagonal entry is non-zero at a p that does not open a 2x2 pivot.  Every later
 * solve, partial solve and enquire_indef use the new D until the next factor or refactor call, which computes D afresh.
 * num_neg and b200ldlt_info keep describing the factorisation, not the altered D. */
int b200ldlt_alter_d(b200ldlt_handle h, const double* dinv2);

/* ---- singular matrices: zero pivots and the Fredholm alternative (cf. HSL_MA97 action, ma97_solve_fredholm) ----------
 * A ZERO PIVOT is a 1x1 pivot that every threshold test rejected (it is forced) and whose whole remaining front column,
 * diagonal included, is <= 1e-12 in the scaled matrix: rounding noise.  The factorisation replaces it by +-1.5e-8 (its L
 * column is the noise over 1.5e-8, |l| <~ 7e-5), so with D_pp = 0 instead the factors are those of a singular matrix within
 * about 1e-12 (scaled max norm) of S A S.  A LIFTED ZERO is a forced pivot with |d| <= tiny under a column that is NOT
 * noise: its L column is that column over 1.5e-8, and D_pp = 0 would describe a matrix far from A.  Either makes the
 * factor call return SINGULAR (info.num_tiny counts them).
 * Keep mode (b200ldlt_set_singular_action(h, 1); default 0, from the next factor / refactor / factor_device call on; a
 * sharded handle ignores it): a SINGULAR factorisation whose forced zeros are all zero pivots still returns SINGULAR -- the
 * status describes the matrix -- but KEEPS its factors, with D^-1 = 0 at the zero pivots Z (D^+: D with its zero pivots
 * left at zero, inverted elsewhere).  *num_neg and info.num_neg then leave the zero pivots out, info.num_tiny = |Z| =
 * n - rank, and last_error says what happened.  Every solve, partial solve, sparse_fwd_solve, lmultiply, alter_d,
 * enquire_indef (D^-1 = 0 at Z) and solve_refine_device work on kept factors unchanged; job 0 is then the D^+ solve.  A
 * factorisation with a lifted zero keeps no factors in any mode (last_error names the pivot).  A non-singular
 * factorisation is the same, bit for bit and launch for launch, in both modes.  keep must be 0 or 1. */
int b200ldlt_set_singular_action(b200ldlt_handle h, int keep);
/* *nzero = |Z| and, unless pos is NULL, pos[0..|Z|) = the pivot positions of Z in ascending order (0 for a factorisation
 * without zero pivots).  Refused: a NULL nzero. */
int b200ldlt_enquire_zero_pivots(b200ldlt_handle h, int* nzero, int* pos);
/* The Fredholm alternative for nrhs columns b_i.  x is n x 2 nrhs, column-major: on entry columns 0..nrhs-1 hold the b_i;
 * on exit column i holds x_i and column nrhs + i holds f_i, and consistent[i] is 1 or 0.  With y = L^-1 P^T S b (job 1) and
 * z = y on Z, 0 elsewhere:
 *   consistent  iff  max_{p in Z} |y_p| <= tol * max_p |y_p|   (max-norms: exact, whatever the reduction order);
 *   x = S P L^-T D^+ y   (job 4 after job 1 with D^+ = job 0 with D^+, bit for bit): A x = b - S^-1 P L z exactly in the
 *                        factored matrix, so x solves A x = b when the column is consistent;
 *   f = S P L^-T z       (job 3 on z): A f = S^-1 P L D z = 0 and b^T f = y^T z = sum_Z y_p^2 > 0 for an inconsistent
 *                        column -- a certificate that b is not in the range of A.
 * f is formed for every column whenever Z is non-empty; with Z empty x is job 0, f = 0 and every column is consistent.
 * Z is that of the factorisation; D is read from D^-1 as it stands (alter_d may overwrite the zeros at Z).  Every column
 * is bit-identical to a call on that column alone.  Kernel launches, D direct levels (B200_SOLVE_DIRECT, default 2):
 * with the blocked state (B200_SOLVE_BLOCK >= 2), blocks of up to B200_SOLVE_BLOCK / 2 columns (4 by default) with x
 * and f through ONE backward sweep of twice the width: 5 + 2 D per block (9 by default); with B200_SOLVE_BLOCK = 1, two
 * backward sweeps per column: 8 + 3 D per column (14); with Z empty, job 0's count.  The first call with Z non-empty
 * allocates the blocked state as a blocked solve does.  Refused: nrhs < 0, tol < 0 or NaN, a NULL pointer with
 * nrhs > 0.  Device entry point: the columns d_x are device memory, consistent host memory. */
int b200ldlt_solve_fredholm(b200ldlt_handle h, int nrhs, double tol, double* x, int* consistent);
int b200ldlt_solve_fredholm_device(b200ldlt_handle h, int nrhs, double tol, double* d_x, int* consistent);

/* ---- selected inversion: the diagonal of A^-1 and A^-1 on the pattern of A (cf. MUMPS entries of A^-1, PSelInv) --------
 * M = S P L^-T D^-1 L^-1 P^T S, the matrix job 0 applies: A^-1 for a non-singular factorisation, the inverse of the
 * perturbed matrix with info.num_forced > 0, the D^+ pseudo-inverse on kept singular factors, and the altered D after
 * alter_d.  diag[i] = M_ii (n doubles, original order); vals[t] = M at (irn[t], jcn[t]) (nonzeros doubles, one per triplet
 * given to b200ldlt_analyse, the order of values_ptr): either triangle, and duplicates read the same stored entry, so they
 * are bit-equal, and the diagonal triplets equal diag bit for bit.  Either pointer may be NULL, not both.  Z = L^-T D^-1
 * L^-1 is computed on the pattern of L by the supernodal Takahashi recurrences, from the root down the elimination tree,
 * every entry as one fixed-order sum: the results are bit-reproducible, and both entry points give the same bits.
 * Kernel launches:  2 + sum over tree levels l of ( g_l + s_l + m_l + 2 b_l + c_l )
 * with, for the fronts of level l (order f = pivots k + rows r): g_l = 1 if one has r > 0, s_l = 1 if one has f <= 96,
 * m_l = 1 if one has 96 < f <= 256, b_l = 1 if one has f > 96 and r > 0, c_l = 1 if one has f > 96; else 0.
 * The first call after an analysis allocates the Z panels (nnz_L doubles: info.L_bytes), L11^-1 of the fronts of order
 * 97..256, the work lists and the output staging; a handle that never calls allocates none of it.  The call uses the
 * contribution blocks and the W scratch of the factorisation as its own scratch (no factorisation reads them before
 * writing them) and leaves the factors, D, the solves and the counters untouched.  Refused: both pointers NULL.
 * Device entry point: d_diag and d_vals are device memory. */
int b200ldlt_selected_inverse(b200ldlt_handle h, double* diag, double* vals);
int b200ldlt_selected_inverse_device(b200ldlt_handle h, double* d_diag, double* d_vals);

/* ---- entries of A^-1 at chosen positions (cf. MUMPS ICNTL(30), sIPOPT's reduced Hessian) ------------------------------
 * vals[t] = M(irow[t], jcol[t]) for t < nent, M as for selected inversion (A^-1, the perturbed matrix's inverse with
 * info.num_forced > 0, D^+ on kept singular factors, the altered D after alter_d).  irow and jcol are 0-based original
 * indices in host memory for both entry points; entries come in any order, repeats and both (i, j) and (j, i) allowed.
 *   M_ij = y_i^T D^-1 y_j ,   y_k = L^-1 P^T S e_k   (job 1 of e_k = sparse_fwd_solve({k}, {1.0}))
 * y_k is non-zero only on the reach of k, the path from its front to the root; fronts are numbered in postorder, so its
 * positions ascend along the path, and y_i and y_j share exactly the path from the lowest common ancestor of their fronts
 * to the root: a common SUFFIX of m positions.  Each entry is one dot over that suffix with D^-1 between (a 2x2 pivot
 * never straddles a front); i and j in different trees of the forest give exactly +0.
 * The columns (the distinct indices of irow and jcol) are sorted by pivot position and swept in blocks of up to
 * B200_SOLVE_BLOCK columns (the blocked state of the solves, allocated as a blocked solve does; B200_SOLVE_BLOCK=1 or
 * a failed allocation: one column per block), each block by the forward stage of sparse_fwd_solve on its unit columns,
 * pruned to the union of their reaches (the same run sets, work lists and dependency check, which refuses a sweep that
 * could wait forever before anything is launched).
 * Summation order, pinned (every operation rounded on its own, no FMA): with a = y_i and b = y_j on the suffix, the TERM
 * at suffix offset o is d (a_o b_o) for a 1x1 pivot (d = D^-1 there), (d1 (a_o b_o) + d2 (a_o+1 b_o+1)) + e ((a_o b_o+1)
 * + (a_o+1 b_o)) for a 2x2 pivot opening at o (d1, d2 its diagonal and e its off-diagonal entry of D^-1), none at the
 * second position of a 2x2.  Partial sum l = 0..31 adds, from +0 in ascending o, the terms at o = l (mod 32); then
 * s_l += s_(l xor k) for k = 16, 8, 4, 2, 1; the entry is s_0.  So (i, j) and (j, i) and repeats give the same bits,
 * repeated calls and both entry points the same bits, and a float64 replay on y from sparse_fwd_solve and D^-1 from
 * enquire_indef reproduces every entry; an entry equals the same entry requested alone, whatever B200_SOLVE_BLOCK, as a
 * value (the y of a column swept in a block may differ from its y swept alone in the sign of a zero).
 * Kernel launches: sum over blocks b of (1 + d_b + t_b + 1), plus 1, with d_b and t_b counted as for sparse_fwd_solve on
 * the block's columns.  Memory: as stated at b200ldlt_sparse_fwd_solve for the three calls that prune sweeps; here a
 * call needs 12 bytes per element of the y store (sum over the columns of the pivots on their paths to the root), 24
 * bytes per entry, 8 w^2 bytes for the identity of the block width w, and per block its pruned lists and 8 bytes per
 * position of its run set, in the shared staging and a device y store that grows to the largest call and is freed by
 * the next analysis.  symbolic_array "inverse_run_set" returns the union
 * of the run sets the last call swept.  The call leaves the factors, D, every later solve and "sparse_run_set" as they
 * were.  Refused (nothing written): nent < 0, a NULL pointer with nent > 0, an index out of range, and (FATAL_ERROR with
 * a message) a failed allocation of the staging or the y store.  nent = 0 is the no-columns case.
 * Device entry point: d_vals (nent doubles) is device memory. */
int b200ldlt_inverse_entries(b200ldlt_handle h, int nent, const int* irow, const int* jcol, double* vals);
int b200ldlt_inverse_entries_device(b200ldlt_handle h, int nent, const int* irow, const int* jcol, double* d_vals);

/* ---- partial factorisation with an explicit Schur complement (cf. MUMPS ICNTL(19) / ICNTL(26), Pardiso iparm(36)) -----
 * S = vars[0..m) are the caller's Schur variables (distinct 0-based original indices), E the other n - m.  In Schur mode
 * the analysis orders E alone and places S last, in the caller's order, as one root front; the factor calls (factor,
 * factor_device, refactor) eliminate E only and leave
 *   S_c = A_SS - A_SE A_EE^-1 A_ES
 * in a handle-owned device buffer of m x m doubles: unscaled (the equilibration factors are powers of two, so exactly),
 * row / column i = vars[i], both triangles written from one, so S_c is bit-symmetric.  That root front is assembled by the
 * big-front kernels and not factored.  *num_neg, info.num_neg and the inertia check (check_inertia, expected_neg)
 * describe A_EE; by Haynsworth, inertia(A) = inertia(A_EE) + inertia(S_c).  Zero and lifted pivots inside E behave as
 * outside Schur mode, except that a SINGULAR factorisation keeps neither factors nor S_c, whatever the keep mode (keep
 * mode combined with Schur mode is not supported).  Pivots are never delayed from E into S.  Factor launches: those of
 * the fronts of E, plus 4 (5 when some front of E is a child of the root): the root's zeroing, assembly and extend-add,
 * the copy-out of S_c and the identity pivot block that replaces the root's factor state.
 * Every other call that reads the factors is refused in Schur mode (see the rules of the partial solves). */
/* Schur mode on vars[0..m) (m = 0: off).  Call it after b200ldlt_analyse, which clears Schur mode (a new pattern makes
 * the indices meaningless); it invalidates the factors, and the next factor call re-analyses with S last.  The set
 * persists through the re-analyses of increase_quality.  After m = 0 the handle's factors, solutions and launch counts
 * are those of a handle that never called it, bit for bit.  Refused (FATAL_ERROR, "set_schur: <reason>", state
 * unchanged): before b200ldlt_analyse, m < 0, m >= n, a NULL vars with m > 0, an index out of range or repeated, a
 * sharded handle.  A handle in Schur mode refuses b200ldlt_shard_setup. */
int b200ldlt_set_schur(b200ldlt_handle h, int m, const int* vars);
/* S_c of the last Schur-mode factorisation, m x m column-major (host / device memory).  Not a launch: one copy.
 * Refused: a NULL sc, a handle not in Schur mode ("<call>: not in Schur mode") or without its factors. */
int b200ldlt_schur_complement(b200ldlt_handle h, double* sc);
int b200ldlt_schur_complement_device(b200ldlt_handle h, double* d_sc);
/* The reduced right-hand side  y = b_S - A_SE A_EE^-1 b_E  (b: n x nrhs, y: m x nrhs, column-major, row i = vars[i]).
 * Job 1's forward sweep (the root's identity pivot block leaves the scaled y in the Schur positions), then one gather:
 * 3 + D kernel launches per block (5 by default), D direct levels (B200_SOLVE_DIRECT). */
int b200ldlt_schur_reduce(b200ldlt_handle h, int nrhs, const double* b, double* y);
int b200ldlt_schur_reduce_device(b200ldlt_handle h, int nrhs, const double* d_b, double* d_y);
/* The expansion of the caller's Schur solution xs (m x nrhs):  x_S = xs,  x_E = A_EE^-1 (b_E - A_ES xs)  (x: n x nrhs).
 * With S_c xs = schur_reduce(b), A x = b.  Job 1's forward sweep on b, a kernel that writes the scaled xs into the
 * Schur positions and applies D^-1 to E, then job 4's backward sweep, which leaves the Schur positions as they are, so
 * x_E has job 0's arithmetic: 5 + 2 D launches per block (9 by default).  x may be b (in place).
 * Both calls: blocks of up to B200_SOLVE_BLOCK columns like the other solves, every column bit-identical to a call on
 * that column alone; nrhs = 0 is the no-columns case; refused for nrhs < 0, a NULL pointer with nrhs > 0, a handle not in
 * Schur mode or without its factors. */
int b200ldlt_schur_expand(b200ldlt_handle h, int nrhs, const double* b, const double* xs, double* x);
int b200ldlt_schur_expand_device(b200ldlt_handle h, int nrhs, const double* d_b, const double* d_xs, double* d_x);

/* ---- error analysis and condition estimation (cf. MUMPS ICNTL(11) / RINFOG(4..11), LAPACK xSYCON) --------------------
 * How far to trust a solution x of A x = b, per column, with componentwise measures (the rows of a KKT system differ in
 * scale by orders of magnitude, so a normwise residual says little about the rows that matter).
 *   A   the matrix of the last factor call: its values (device_ptr "vals", unscaled) with duplicate triplets summed in
 *       triplet order, as the factorisation sums them, BEFORE absolute values are taken;
 *   M   the operator job 0 applies (as for selected inversion): A^-1, the inverse of the perturbed matrix with
 *       info.num_forced > 0, the matrix with the altered D after alter_d.
 * For each column, with r = b - A x, s = |A| |x|, a_i = max_j |a_ij|, eps = 2^-52 and
 * tau_i = 1000 n eps (a_i ||x||_inf + |b_i|):
 *   I2 = { i : s_i + |b_i| <= tau_i },  I1 the other rows;
 *   omega1 = max_{i in I1} |r_i| / (s_i + |b_i|),   omega2 = max_{i in I2} |r_i| / (s_i + a_i ||x||_inf)
 *            (a term with r_i = 0 counts as 0; a zero denominator occurs only then), 0 for an empty set;
 *   w1 = s + |b| on I1, 0 elsewhere;  w2 = s + a ||x||_inf on I2, 0 elsewhere;
 *   cond_k = est || M diag(w_k) ||_inf / ||x||_inf = est || diag(w_k) M ||_1 / ||x||_inf (M is symmetric), estimated through
 *            the products B v = w_k o (M v) and B^T v = M (w_k o v); an empty set gives cond_k = 0 and runs no estimator;
 *   ferr   = omega1 cond1 + omega2 cond2, an estimated bound on ||x - x*||_inf / ||x||_inf (first order);
 *   ||x||_inf = 0 runs no estimator: cond1 = cond2 = ferr = 0 if b = 0, +inf otherwise.
 * The estimator is Higham's 1-norm estimator exactly as LAPACK dlacn2 runs it: start from x = e/n; sign(y) = +1 for
 * y >= 0 (-0 included); j = the first index of max |z|; stop on a repeated sign vector, on est <= est_old, when
 * z_jlast = |z_j| or after 5 iterations; finish with x_i = (-1)^i (1 + i/(n-1)) (i = 0..n-1) and the test 2 ||y||_1 / (3n)
 * > est.  At most 11 products per estimator.
 * cond = 0 (cheap, as MUMPS ICNTL(11) = 2): the norms, omega1, omega2 and n_i2 only; no solve runs, cond1 = cond2 = ferr
 * = -1 ("not computed").  Kept singular factors (zero pivots, keep mode): omega1 and omega2 as usual, cond1 = cond2 =
 * ferr = +inf, no estimator runs.
 * Every column's struct is bit-identical to a call on that column alone, under any B200_SOLVE_BLOCK, between the two entry
 * points and across calls: maxima are exact (atomicMax on bit patterns), |I2| an integer count and every sum (r, s, the
 * row sums of |A|, ||y||_1) has a fixed order.  The call leaves the factors, D, the solves and their bits as they were.
 * Kernel launches, with L0 = job 0's launches per block (4 + 2 D, 8 by default): cond = 0: 3 (the unique values, the row
 * pass, the row classes); cond = 1: 3 + (2 + L0) T, where T is the number of estimator steps: each step is one input
 * kernel, one job-0 solve of the block's unfinished estimators and one reduction kernel.  The two estimators of a column
 * take two columns of the blocked solve state, so blocks of up to B200_SOLVE_BLOCK / 2 columns (4 by default) step in
 * lockstep and T = the sum over the blocks of the largest product count of an estimator in the block; with
 * B200_SOLVE_BLOCK = 1 (or without the blocked state) every estimator runs alone and T = the sum of nprod.
 * The first call after an analysis builds |A| by rows (about 4 (n + 1 + 2 m) bytes, m the entries of both triangles,
 * 2 nnz_unique - the diagonal ones) and its buffers: 8 (nnz_unique + n) bytes, 16 n bytes per right-hand side (grown to
 * the largest call) and, with cond = 1, 9 n bytes per column of the solve state it uses.  b and x are n x nrhs,
 * column-major, and are not modified; out is nrhs structs in host memory for both entry points.  Refused (nothing
 * written to out): nrhs < 0, cond other than 0 or 1, a NULL pointer with nrhs > 0.  nrhs = 0 is the no-columns case. */
typedef struct b200ldlt_errors {
  double anorm;          /* ||A||_inf = max_i sum_j |a_ij|   (= ||A||_1, A symmetric)                                  */
  double xnorm, rnorm;   /* ||x||_inf, ||r||_inf with r = b - A x                                                   */
  double omega1, omega2; /* componentwise backward errors on I1 and I2 (Arioli, Demmel, Duff)                       */
  double cond1, cond2;   /* estimated condition numbers for the two row sets                                        */
  double ferr;           /* omega1 cond1 + omega2 cond2: estimated bound on ||x - x*||_inf / ||x||_inf               */
  int n_i2;              /* |I2|                                                                                    */
  int nprod;             /* products with M the column's estimators took (0 when cond == 0)                         */
} b200ldlt_errors;
int b200ldlt_error_analysis(b200ldlt_handle h, int nrhs, const double* b, const double* x, int cond, b200ldlt_errors* out);
int b200ldlt_error_analysis_device(b200ldlt_handle h, int nrhs, const double* d_b, const double* d_x, int cond,
                                   b200ldlt_errors* out);
/* kappa1 = ||A||_1 est ||M||_1 (1 / LAPACK's rcond): one estimator with w = 1 through the single-column solve state.
 * anorm1 (||A||_1), ainv1 (est ||M||_1) and nprod (products taken, <= 11) may be NULL.  Kept singular factors: kappa1 =
 * ainv1 = +inf, no estimator runs.  Kernel launches: 2 + (2 + L0) nprod.  Refused: a NULL kappa1. */
int b200ldlt_condest(b200ldlt_handle h, double* kappa1, double* anorm1, double* ainv1, int* nprod);

/* ---- iterative refinement by the componentwise backward error (cf. MUMPS ICNTL(10) / CNTL(2), MA57 job 2..4, LAPACK
 * xSYRFS / xSYRFSX) ------------------------------------------------------------------------------------------------------
 * Solves A x = b for nrhs columns and refines each x until its componentwise backward error omega (Arioli, Demmel, Duff)
 * is small, stops improving, or max_steps corrections are taken.  The residual is accumulated in double-double, so omega
 * can fall to about eps even where cond(A) eps is large -- e.g. after lifted pivots (info.num_forced > 0), where job 0
 * solves a perturbed matrix.  A, M, s = |A| |x|, a_i, tau_i, I1, I2, omega1 and omega2 are those of
 * b200ldlt_error_analysis above, bit for bit given r; only r differs.
 *   Iterates:  x_0 = job 0 on b (bit-identical to b200ldlt_solve);  x_{k+1} = x_k (+) d_k,  d_k = job 0 on r_k, one
 *              rounded add (__dadd_rn) per entry.
 *   Residual:  r_k = b - A x_k.  Row i is one warp over the row's entries of |A|'s row structure (both triangles of the
 *              unique entries, columns ascending); lane l takes entries l, l + 32, ... in order.  Every operation below is
 *              one correctly rounded IEEE operation (nothing is contracted); TwoSum(a, c) = (s, t) with s = a (+) c,
 *              v = s (-) a, t = (a (-) (s (-) v)) (+) (c (-) v).
 *                lane 0 starts from (h, l) = (b_i, 0), the other lanes from (0, 0);
 *                per entry: p = (-a_ij) (*) x_j, e = fma(-a_ij, x_j, -p); (h, t) = TwoSum(h, p); l = l (+) (t (+) e);
 *                then for o = 16, 8, 4, 2, 1 with (h', l') of lane l xor o: (h, t) = TwoSum(h, h'); l = (l (+) l') (+) t;
 *                r_i = h (+) l (lane 0's).
 *              Barring overflow and underflow, with m_i the entries of row i and E_i the exact residual:
 *                |r_i - E_i| <= 2^-53 |E_i| + (m_i + 32)^2 2^-105 (|b_i| + sum_j |a_ij x_j|),
 *              so each reported omega is within 2^-51 w + (m + 32)^2 2^-103 of the value w it has with exact residuals
 *              (same s, classes and weights), m the longest row.
 *   Omega:     omega_k = omega1 + omega2 of x_k (one rounded add).
 *   Stopping:  on each iterate k = 0, 1, ..., in this order:
 *                1. omega_k not finite: the result is the last iterate with a finite omega, status 3 (x_0 itself when
 *                   k = 0, with its omega1 and omega2 as computed, so omega_first = +inf);
 *                2. omega_k <= tol: x_k, status 0;
 *                3. k >= 1 and omega_k > omega_{k-1} / 2: x_k if omega_k < omega_{k-1}, else x_{k-1}; status 1;
 *                4. k = max_steps: x_k, status 2;
 *              otherwise the column takes the next correction.  So the returned omega never exceeds omega_first, and
 *              max_steps = 0 returns job 0 with its omega.  An inconsistent column (kept singular factors) ends by
 *              stagnation.  A column with b = 0 returns x = 0 at k = 0, status 0.
 *   Blocks:    columns run in blocks of up to B200_SOLVE_BLOCK (8 by default) in lockstep; each step solves only the
 *              block's unfinished columns, packed into consecutive solve slots, and a finished column that returns
 *              x_{k-1} gets it back from a copy.  Without the blocked state (B200_SOLVE_BLOCK = 1 or no memory for it)
 *              the columns run one by one.  Every column's x and struct are bit-identical to a call on that column alone,
 *              under any B200_SOLVE_BLOCK, between the two entry points and across calls.
 * Kernel launches, with L0 = job 0's launches per block (4 + 2 D, 8 by default): 1 (the unique values) + per block
 * E (L0 + 3) - 1, where E is the largest nres of the block's columns: x_0 (L0), per iterate the row pass and the row
 * classes (2), per correction job 0 and the update kernel (L0 + 1).  One column: nres (L0 + 3).  Each iterate ends in one
 * small D2H and a host decision, and the call synchronises per iterate.
 * Memory: the state of b200ldlt_error_analysis (|A| by rows at the first call after an analysis, its 16 n bytes per
 * column) for the block width, plus 16 n bytes per column of the block for the solve slots and the rollback copies
 * (grown to the largest call, kept until the next analysis), and the blocked solve state if nrhs > 1 allocates it first.
 * The host entry point stages 2 n nrhs doubles (x and a copy of b).
 * b and x are n x nrhs, column-major; b is not modified and x may not be b; out is nrhs structs in host memory for both
 * entry points.  Timing (info.ms_solve_gpu, launches_solve) and refusals follow the solve family: no factors, a sharded
 * handle, Schur mode; and nrhs < 0, max_steps < 0, tol < 0 or NaN, a NULL pointer with nrhs > 0, x == b.  Nothing is
 * written on a refusal; nrhs = 0 is the no-columns case.  The call leaves the factors, D, later solves and the results
 * of b200ldlt_error_analysis as they were. */
typedef struct b200ldlt_refined {
  double omega_first;    /* omega1 + omega2 of x_0, the plain job-0 solution                                        */
  double omega1, omega2; /* componentwise backward errors of the returned x                                         */
  int steps;             /* corrections contained in the returned x                                                  */
  int status;            /* 0 converged (omega <= tol), 1 stagnated, 2 max_steps reached, 3 non-finite omega          */
  int nres;              /* residuals evaluated (iterates 0 .. nres - 1; steps + 1, or steps + 2 after a rollback)    */
} b200ldlt_refined;
int b200ldlt_solve_refined(b200ldlt_handle h, int nrhs, const double* b, double* x, int max_steps, double tol,
                           b200ldlt_refined* out);
int b200ldlt_solve_refined_device(b200ldlt_handle h, int nrhs, const double* d_b, double* d_x, int max_steps,
                                  double tol, b200ldlt_refined* out);

/* ---- FGMRES preconditioned by the factors (cf. Arioli, Duff, Gratton and Pralet, SIAM J. Sci. Comput. 29 (2007);
 * Carson and Higham's GMRES-IR; Pardiso iparm(4)) -----------------------------------------------------------------------
 * Solves A_op x = b for nrhs columns by restarted, right-preconditioned flexible GMRES with M = job 0 as preconditioner,
 * stopped by the componentwise backward error as b200ldlt_solve_refined stops.  M A_op = I + M (A_op - A_M), A_M the
 * matrix job 0 inverts: with lifted pivots (info.num_forced > 0) or an altered D the difference has low rank, and with
 * other values it is what the new values change, so GMRES converges where classical refinement (x <- x + M r, which
 * needs the spectral radius of I - M A_op below 1) stagnates or diverges.
 *   A_op   vals: nonzeros doubles in the triplet order given to b200ldlt_analyse, duplicates summed in triplet order as
 *          the factorisation sums them (0.0 + v_0 + v_1 ...); vals == NULL is the matrix of the last factor call, bit for
 *          bit the same as passing its values.  vals is in the memory of its entry point: host memory for
 *          b200ldlt_solve_gmres (staged with b), device memory for _device.  A_op is not kept: the factors, the values
 *          b200ldlt_refactor reuses and every other call are unaffected.
 *   M      job 0's operator, as in the selected-inversion and error-analysis blocks above.
 *   Omega: omega1, omega2, I1, I2, s, a_i, tau_i and the weights are those of b200ldlt_error_analysis with A := A_op;
 *          r = b - A_op x is the double-double residual of b200ldlt_solve_refined, in its order.
 *   Iterates: x_0 = job 0 on b (bit-identical to b200ldlt_solve).  The stopping rule of b200ldlt_solve_refined is applied
 *          to each iterate x_k = x_0, x_1, ... exactly as stated there, with max_cycles in place of max_steps (status 0
 *          converged, 1 stagnated with x_k or x_{k-1}, 2 max_cycles, 3 non-finite omega).  When the column goes on, one
 *          restart cycle runs on A_op d = r_k (r_k the residual of the rule's iterate):
 *            beta^2 = <r_k, r_k>, beta = sqrt(beta^2), v_0 = r_k (/) beta (per entry), g_0 = beta;
 *            per step j = 0, 1, ...: z_j = job 0 on v_j (kept); w = A_op z_j (row i: lane l of a warp takes the row's
 *              entries l, l + 32, ... of |A|'s row structure in order, t = t (+) (a_ij (*) z_j) from t = 0, then for
 *              o = 16, 8, 4, 2, 1: t = t (+) t' of lane l xor o; w_i = lane 0's t);
 *              CGS2: h1_q = <v_q, w> (q = 0..j), w_i = w_i (-) (h1_q (*) v_q,i) for q = 0..j in order;
 *                    h2_q = <v_q, w> with that w, w_i = w_i (-) (h2_q (*) v_q,i) likewise;
 *              h_q,j = h1_q (+) h2_q (q <= j), h_{j+1,j} = sqrt(<w, w>), v_{j+1} = w (/) h_{j+1,j} (per entry);
 *            <a, b> is the fixed sum over P = min(ceil(n / 256), 264) CTAs of 256 threads: thread t of CTA p adds
 *              a_i (*) b_i for i = 256 p + t, + 256 P, ... in order from 0.0; each warp a shuffle-xor tree (o = 16 .. 1,
 *              t = t (+) t'); the CTA's 8 warps in order (t = w_0, t = t (+) w_k); the CTAs' partials in order from 0.0.
 *            The host then rotates the column (every operation one rounded double operation, no FMA, no hypot):
 *              for i < j with the earlier rotations (c_i, s_i): t = c_i h_i + s_i h_{i+1}, h_{i+1} = c_i h_{i+1} - s_i h_i,
 *              h_i = t;  rho = sqrt(h_j h_j + h_{j+1} h_{j+1}), c_j = h_j / rho, s_j = h_{j+1} / rho, R_ij = h_i (i < j),
 *              R_jj = rho;  g_{j+1} = -(s_j g_j), g_j = c_j g_j.
 *            A step in which any h_{i,j} (i <= j + 1) or rho is not finite, or rho = 0, is a breakdown that is dropped:
 *              the cycle ends with the steps before it.  Otherwise the step is kept, and the cycle ends after it when
 *              h_{j+1,j} = 0 (a breakdown that is kept), |g_{j+1}| <= inner_tol (*) beta, or j + 1 = restart.  A beta that
 *              is 0 or not finite (|r| beyond the range of its square) ends the cycle before its first step.
 *            With m steps kept: y_i = (g_i (-) sum_{l = i+1}^{m-1} R_il y_l) (/) R_ii for i = m - 1 down to 0, the sum
 *              subtracted term by term in ascending l;  d_i = 0 (+) y_0 z_0,i (+) ... (+) y_{m-1} z_{m-1},i in order,
 *              each product rounded;  x_{k+1} = x_k (+) d, x_k kept for the rule's rollback.
 *          So the returned omega never exceeds omega_first, and max_cycles = 0 returns job 0 with its omega.  In exact
 *          arithmetic a cycle with M A_op = I + (rank k) ends within k + 1 steps.
 *   Blocks: columns run in blocks of up to B200_SOLVE_BLOCK (8 by default) in lockstep by cycle and by Arnoldi step; each
 *          iterate and each step works on the block's columns still active, packed into consecutive solve slots, as
 *          b200ldlt_solve_refined packs them.  Every column's x and struct are bit-identical to a call on that column
 *          alone, under any B200_SOLVE_BLOCK, between the two entry points and across calls.
 * Kernel launches, with L0 = job 0's launches per block (4 + 2 D, 8 by default): 1 (the unique values of A_op) + per
 * block L0 (x_0) + 3 E (per iterate: the row pass, the row classes and beta^2) + 2 (E - 1) (per cycle: v_0 and the
 * update of x) + (L0 + 6) T (per Arnoldi step: job 0, the product with A_op, two dot and two update kernels, and the
 * normalisation), where E is the largest nres of the block's columns and T the sum over the block's cycles of the most
 * steps a column of the block took in that cycle.  One column: 1 + L0 + 5 nres - 2 + (L0 + 6) iters.  The call
 * synchronises once per iterate (one D2H of the maxima and beta^2) and once per Arnoldi step (one D2H of the Hessenberg
 * columns for the host's rotations and stopping decisions).
 * Memory: that of b200ldlt_solve_refined for the block width, plus V (restart + 1 vectors) and Z (restart vectors) per
 * column of the block, (2 restart + 1) 8 n bytes, and about 1.1 MB of reduction scratch; grown to the largest call and
 * freed by the next analysis.  A failed allocation is a refusal with a message.  The host entry point stages
 * 2 n nrhs doubles (x and a copy of b), plus nonzeros doubles when vals is given.
 * b and x are n x nrhs, column-major; b and vals are not modified and x may not be b; out is nrhs structs in host memory
 * for both entry points.  Timing (info.ms_solve_gpu, launches_solve) and refusals follow the solve family: no factors, a
 * sharded handle, Schur mode; and nrhs < 0, restart < 1 or > 64, max_cycles < 0, tol or inner_tol < 0 or NaN, a NULL
 * b, x or out with nrhs > 0, x == b.  Nothing is written on a refusal; nrhs = 0 is the no-columns case.  With kept
 * singular factors the call runs and obeys the rule.  The call leaves the factors, D, the device values of the last
 * factor call, later solves and the results of b200ldlt_error_analysis and b200ldlt_solve_refined as they were. */
typedef struct b200ldlt_gmres {
  double omega_first;    /* omega1 + omega2 of x_0 (job 0 on b) against A_op                                        */
  double omega1, omega2; /* of the returned x                                                                        */
  int cycles;            /* corrections (restart cycles) contained in the returned x                                 */
  int iters;             /* Arnoldi steps (job-0 applications after x_0) the column took, rolled-back cycle included */
  int status;            /* as b200ldlt_refined: 0 converged, 1 stagnated, 2 max_cycles, 3 non-finite omega          */
  int nres;              /* residuals evaluated (cycles + 1, or cycles + 2 after a rollback)                         */
} b200ldlt_gmres;
int b200ldlt_solve_gmres(b200ldlt_handle h, int nrhs, const double* b, double* x, const double* vals, int restart,
                         int max_cycles, double tol, double inner_tol, b200ldlt_gmres* out);
int b200ldlt_solve_gmres_device(b200ldlt_handle h, int nrhs, const double* d_b, double* d_x, const double* d_vals,
                                int restart, int max_cycles, double tol, double inner_tol, b200ldlt_gmres* out);

/* <-> NumberOfNegEVals() (hpp:207) */
int b200ldlt_num_neg(b200ldlt_handle h);
/* <-> IncreaseQuality() (hpp:220): pivtol <- min(pivtolmax, pivtol^0.75); returns 0 if already at max.
 * If the last factorisation had to LIFT pivots (info.num_forced) or saw growth beyond 1/u (info.num_growth), the
 * first request instead schedules a re-analysis (saddle pairing + ordering) on the values of the next factor call.
 * With num_forced > 0 the factors and the inertia are those of a matrix perturbed by <= 1e-8 |column| in the lifted pivots.
 * The values of the last matrix are kept on the device, so the next factor call may pass new or old values. */
int b200ldlt_increase_quality(b200ldlt_handle h);
/* Re-run the numeric factorisation on the values kept on the device from the last factor call
 * (used after increase_quality instead of the reference's CALL_AGAIN round trip,
 *  IpMumpsSolverInterface.cpp:265-278). */
int b200ldlt_refactor(b200ldlt_handle h, int check_inertia, int expected_neg, int* num_neg);

/* (Re)set the pivot threshold and its cap, e.g. when a kept handle starts a new optimisation
 * (warm_start_same_structure: the reference adapters re-read pivtol in every InitializeImpl,
 *  IpMumpsSolverInterface.cpp:191-245). */
int b200ldlt_set_pivtol(b200ldlt_handle h, double pivtol, double pivtolmax);

int b200ldlt_get_info(b200ldlt_handle h, b200ldlt_info* info);
/* Copy a named array of the symbolic analysis ("perm","sn_start","sn_parent","rows_ptr","rows","rel",
 * "L_off","cb_off","u_dst64","uent_ptr","t2u","sn_level","level_ptr","level_sn") as int64 into out (cap entries).
 * Returns the array length, or -1 for an unknown name. Runs the lazy analysis (pattern only) if needed.
 * "sparse_run_set": the fronts the last b200ldlt_sparse_fwd_solve swept, ascending (empty before the first one);
 * "inverse_run_set": the union of the fronts the last b200ldlt_inverse_entries swept, ascending (empty before the first). */
int64_t b200ldlt_symbolic_array(b200ldlt_handle h, const char* name, int64_t* out, int64_t cap);
/* Force the symbolic phase now; vals may be NULL (no saddle pairing then). */
int b200ldlt_analyse_now(b200ldlt_handle h, const double* vals);

/* Fused residual helper on the device: r = b - A x for the matrix of the last factor call
 * (original, unscaled values), returns max-norms. Used by tests/bench for parity checks. */
int b200ldlt_residual(b200ldlt_handle h, const double* x, const double* b, double* r_inf, double* x_inf, double* b_inf);

/* ---- device-side callers of the path (SURVEY.md 8f-1) ----------------------------------------------------------------
 * What TSymLinearSolver does on the host around every MultiSolve -- fill the values array from the blocks of the augmented
 * system (TripletHelper::FillValues, IpTripletHelper.cpp:805-873, on the CompoundSymMatrix StdAugSystemSolver builds,
 * IpStdAugSystemSolver.cpp:232-430) and the iterative refinement of the solve (IpPDFullSpaceSolver.cpp:241-346) -- for
 * callers that keep W, J, Sigma and the right-hand sides in device memory: no 8*nnz H2D per factorisation, one D2H of
 * the refined solution per solve. */
typedef struct b200ldlt_augsys {
  int n_x, n_s, n_c, n_d;          /* block dimensions (n_d == n_s) */
  int nnz_w, nnz_jc, nnz_jd;       /* triplet counts of W (lower triangle), J_c, J_d as delivered at analyse time */
  const double* W;  double W_factor;   /* DEVICE pointers; NULL W = "no Hessian" (the block values are 0) */
  const double* D_x; double delta_x;   /* diagonal of the (1,1) block: D_x + delta_x   (NULL D: delta only) */
  const double* D_s; double delta_s;   /* (2,2): D_s + delta_s */
  const double* J_c;                   /* (3,1) */
  const double* D_c; double delta_c;   /* (3,3): D_c - delta_c */
  const double* J_d;                   /* (4,1) */
  const double* D_d; double delta_d;   /* (4,4): D_d - delta_d ; the (4,2) block is -I */
} b200ldlt_augsys;
/* Writes the handle's DEVICE value array in exactly the order FillValues produces for that CompoundSymMatrix:
 *   [W_factor*W | D_x+delta_x | D_s+delta_s | J_c | D_c-delta_c | J_d | -1 (n_s times) | D_d-delta_d]
 * (bit-identical: one multiply / one add per entry like the reference).  Follow with b200ldlt_refactor(). */
int b200ldlt_assemble_augsys_device(b200ldlt_handle h, const b200ldlt_augsys* a);
/* Solve with iterative refinement entirely on the device: d_rhs (dim doubles, DEVICE) holds b on entry and the refined x
 * on exit.  After the first solve, steps of  r = b - A x ; x += solve(r)  are taken while step < min_steps or the
 * residual ratio  ||r||_inf / (min(||x||_inf, 1e6 ||b||_inf) + ||b||_inf)  (IpPDFullSpaceSolver.cpp:795-820) exceeds tol,
 * at most max_steps.  A is the matrix of the last factor call (its values on the device). */
int b200ldlt_solve_refine_device(b200ldlt_handle h, double* d_rhs, int min_steps, int max_steps, double tol,
                                 int* steps_done, double* residual_ratio);

/* ---- multi-GPU elimination-tree sharding (one process / handle per GPU; SURVEY.md section 8e) -----------------
 * The exchange itself (contribution blocks of the cut -> rank 0, update vectors, top solution back) is done by the
 * caller with NCCL send/recv on the device pointers below; ipopt_b200/sharded.py is the reference orchestration. */
int b200ldlt_shard_setup(b200ldlt_handle h, int rank, int world);
/* "owner" (per supernode: owning rank, -1 = top part on rank 0), "cut_roots", "top_fronts" */
int64_t b200ldlt_shard_array(b200ldlt_handle h, const char* name, int64_t* out, int64_t cap);
/* device arrays of the handle: "CB" (contribution blocks, offsets cb_off; after b200ldlt_selected_inverse it holds that
 * call's scratch until the next factorisation), "cbv" (update vectors, offsets rows_ptr),
 * "x" (permuted solution vector), "counters" (8 ints), "vals" (triplet values), "scale" (the n equilibration factors
 * S of the last factor call, original order) */
void* b200ldlt_device_ptr(b200ldlt_handle h, const char* name);
int b200ldlt_shard_factor(b200ldlt_handle h, int phase, int from_host);
int b200ldlt_shard_factor_finish(b200ldlt_handle h, const int* counters_total, int check_inertia, int expected_neg, int* num_neg);
int b200ldlt_shard_solve(b200ldlt_handle h, int phase, double* d_rhs);

#ifdef __cplusplus
}
#endif
#endif
