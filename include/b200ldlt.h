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
  int use_graph;       /* 1 = replay numeric phases from CUDA graphs */
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

/* <-> MultiSolve part 2: rhs is dim x nrhs column-major, overwritten with the solution (host memory). */
int b200ldlt_solve(b200ldlt_handle h, int nrhs, double* rhs);
/* Same with a device-resident rhs/solution. */
int b200ldlt_solve_device(b200ldlt_handle h, int nrhs, double* d_rhs);

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
 * Returns the array length, or -1 for an unknown name. Runs the lazy analysis (pattern only) if needed. */
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
/* device arrays of the handle: "CB" (contribution blocks, offsets cb_off), "cbv" (update vectors, offsets rows_ptr),
 * "x" (permuted solution vector), "counters" (8 ints), "vals" (triplet values) */
void* b200ldlt_device_ptr(b200ldlt_handle h, const char* name);
int b200ldlt_shard_factor(b200ldlt_handle h, int phase, int from_host);
int b200ldlt_shard_factor_finish(b200ldlt_handle h, const int* counters_total, int check_inertia, int expected_neg, int* num_neg);
int b200ldlt_shard_solve(b200ldlt_handle h, int phase, double* d_rhs);

#ifdef __cplusplus
}
#endif
#endif
