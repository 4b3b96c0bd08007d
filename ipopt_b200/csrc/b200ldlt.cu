// Host orchestration + extern "C" shim of the GPU LDL^T backend (see include/b200ldlt.h), H100 / sm_90a.
// One translation unit: the kernels are included so nvcc sees launch sites and definitions together.
#include "../../include/b200ldlt.h"
#include "../../include/b200vec.h"

#include <cuda_runtime.h>

#include <algorithm>
#include <climits>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <iterator>
#include <string>
#include <memory>
#include <vector>

#include "factor_kernels.cu"
#include "solve_kernels.cu"
#include "solve_dataflow.cu"
#include "lmul_kernels.cu"
#include "schur_tc.cu"
#include "selinv_kernels.cu"
#include "sc_kernels.cu"
#include "ea_kernels.cu"
#include "gmres_kernels.cu"
#include "symbolic.hpp"

namespace b200 {

template <class T>
struct DevBuf {
  T* p = nullptr;
  size_t n = 0;
  DevBuf() = default;
  DevBuf(const DevBuf&) = delete;              // one owner per allocation
  DevBuf& operator=(const DevBuf&) = delete;
  ~DevBuf() { release(); }
  void release() { if (p) cudaFree(p); p = nullptr; n = 0; }
  // n is the size only once the memory is there: a failed allocation leaves the buffer released (p null, n 0)
  cudaError_t alloc(size_t count) {
    release();
    if (count == 0) return cudaSuccess;
    const cudaError_t e = cudaMalloc((void**)&p, count * sizeof(T));
    if (e == cudaSuccess) n = count; else p = nullptr;
    return e;
  }
  template <class U>
  cudaError_t upload(const std::vector<U>& v, cudaStream_t st) {
    std::vector<T> tmp(v.begin(), v.end());
    cudaError_t e = alloc(tmp.size());
    if (e != cudaSuccess || tmp.empty()) return e;
    e = cudaMemcpyAsync(p, tmp.data(), tmp.size() * sizeof(T), cudaMemcpyHostToDevice, st);
    if (e != cudaSuccess) return e;
    return cudaStreamSynchronize(st);  // tmp dies here
  }
};

// work lists of the explicit L11 inverses of the big fronts (k_linv_diag / k_linv_gemm, solve_dataflow.cu)
struct LinvPlan {
  DevBuf<int> d_diag;                      // (front, 64-block) pairs
  int ndiag = 0;
  std::vector<std::unique_ptr<DevBuf<LinvItem>>> d_g;   // per recursion level: the tile items (same list for both passes ...
  std::vector<std::unique_ptr<DevBuf<LinvItem>>> d_g2;  // ... up to the k-range)
  std::vector<int> ng, ng2;                // items per level (pass 1, pass 2: the chunking differs)
  long long part_tiles = 0;                // scratch tiles (= counters) the chunked items of one launch need (max over launches)
};

// triangular-solve work of a set of fronts (solve_dataflow.cu): subtrees for k_solve_sub + task lists for k_solve_top
struct SolvePlan {
  // host copies of the lists as uploaded, one-element placeholders included (the pruned sweeps prune them)
  std::vector<SolveTask> tf, tb;
  std::vector<int2> pairs;
  std::vector<SubDesc> subs;
  std::vector<int> meta, bundle;
  std::vector<std::vector<int>> direct;
  DevBuf<SolveTask> d_tf, d_tb;
  DevBuf<int> d_bundle, d_sub_meta, d_ccnt, d_subrow;
  DevBuf<SubDesc> d_subs;
  DevBuf<int2> d_subpair;
  DevBuf<int> d_sub_Loff;
  std::vector<std::unique_ptr<DevBuf<int>>> d_direct;   // per bottom level: the fronts k_solve_direct owns
  std::vector<int> direct_cnt;
  DevBuf<double> d_part;
  int nsub = 0, npair = 0, ntf = 0, ntb = 0;
  long long sub_bytes = 0;
};

// what the solve sweeps write, for `width` columns: column c of each array at its base + c * its stride in M.  The chunk
// partials and counters belong to a plan (a counter counts modulo its task's nq, so plans must not share them): one column
// uses those of the plan it sweeps, a block (width > 1) has its own copies of the handle's in d_part / d_ccnt.
struct SweepState {
  int width = 0;
  DevBuf<double> d_x, d_cbv, d_bigv, d_bigy, d_part;
  DevBuf<int> d_done_f, d_done_b, d_bflag_f, d_bflag_b, d_bcnt, d_bcnt_b, d_ccnt;
  DevBuf<unsigned long long> d_ticket;   // [0] fwd, [1] bwd (monotonic)
  unsigned long long ticket_f = 0, ticket_b = 0;   // their values when the next sweep starts
  MultiStride M;
  int grid = 0;                          // CTAs of the persistent sweep kernel
};

// multiplication by the factors (lmul_kernels.cu): the work lists and the slot map of k_lmul_n / k_lmul_gather, built at
// the first lmultiply call after an analysis (a handle that never multiplies allocates nothing), and a scratch of `width`
// columns of `ld` doubles (the slots for trans = 0, w for trans = 1)
struct LmulPlan {
  DevBuf<LmulItem> d_items_n;
  DevBuf<int2> d_items_t;
  DevBuf<int> d_pcol0, d_own_ptr, d_own, d_desc_ptr, d_desc;
  DevBuf<double> d_scr;
  long long ld = 0;
  int width = 0;
};

struct Solver;

// Pinned -> device staging of the lists of a call (ListStaging::reserve / upload): h the pinned copy, d the device copy of
// the same layout, ev the last copy out of h.  Grows to the largest call and lasts until the next analysis.
struct ListStaging {
  char* h = nullptr;
  DevBuf<char> d;
  cudaEvent_t ev = nullptr;
  int reserve(Solver* sv, const char* call, size_t bytes);
  int upload(Solver* sv, size_t bytes);
  ~ListStaging() {
    if (h) cudaFreeHost(h);
    if (ev) cudaEventDestroy(ev);
  }
};

// The calls that run pruned sweeps (b200ldlt_sparse_fwd_solve, b200ldlt_inverse_entries, b200ldlt_sparse_solve): per
// front its indices into the host copies of the full plan's lists and, per direction, its top tasks; the marks of one
// pruned sweep; each call's last run sets; the inverse entries' tree depths and path lengths and their y store; and the
// one list staging the three calls share (each call ends in the synchronise of timed_call on the handle's one stream).
// Built at the first such call after an analysis, before that call's timing starts; a handle that never makes one
// allocates none of it.
struct PrunedPlan {
  std::vector<int> dlev, didx;                 // by front: its direct level and index there, or -1
  std::vector<int> item_of, sub_of;            // by front: the subtree item / the subtree that walks it, or -1
  std::vector<int> item_ptr, item_fr;          // by subtree item (CSR): the fronts its subtrees walk
  std::vector<int> iperm, sn_of;               // variable -> permuted column; position -> front
  std::vector<int> pos_bi;                     // position -> index into the compact b during a call, else -1
  std::vector<int> depth, pathlen;             // by front: depth in the tree, pivots on its path to the root
  std::vector<int> col_of;                     // inverse entries: variable -> its column in the current call, else -1
  struct Dir {                                 // [0] forward (SolvePlan::tf), [1] backward (SolvePlan::tb)
    std::vector<int> task_ptr, task_idx;       // by front (CSR): its top tasks, ascending
    std::vector<unsigned> m_task;
  } dir[2];
  std::vector<unsigned> m_reach, m_run, m_fr, m_item;   // marks of the current sweep (== stamp)
  std::vector<int> ord0, ord1;                 // per sweep: first / last slot of a run front in the pruned order
  unsigned stamp = 0;
  // the run sets of each call's last run, ascending (symbolic_array "sparse_run_set", "inverse_run_set",
  // "sparse_solve_fwd_run_set", "sparse_solve_bwd_run_set"); a call leaves the others' untouched
  std::vector<int> last_sfs, last_inv, last_fwd, last_bwd;
  ListStaging stg;
  DevBuf<double> d_y;                          // inverse entries: the y store, grown to the largest call
};

// selected inversion (b200ldlt_selected_inverse, selinv_kernels.cu): per tree level the fronts of each launch and the tile
// items of the fronts above SI_SMALL, the Z panels, the L11^-1 of the fronts of order (SI_SMALL, SI_MID] and the index
// maps of the output.  Built at the first call after an analysis, before its timing starts; a handle that never makes
// the call allocates none of it.
struct SelInvPlan {
  struct Level {
    int g_off = 0, g_cnt = 0;      // k_si_gather items (32-row column segments of the G of the fronts with r > 0)
    int s_off = 0, s_cnt = 0;      // fronts of order <= SI_SMALL (k_si_small), their largest f^2 + k^2 doubles in smem
    int m_off = 0, m_cnt = 0;      // fronts of order (SI_SMALL, SI_MID] (k_si_linv)
    size_t smem = 0;
    int t_off[3] = {0, 0, 0}, t_cnt[3] = {0, 0, 0};   // k_si_tile<PASS> items
  };
  std::vector<Level> lev;
  DevBuf<double> d_Z, d_E, d_diag, d_vals;   // Z (layout of L), L11^-1 (ld k), staging of the host entry point
  DevBuf<int> d_fronts, d_iperm, d_sn_of, d_lpinv, d_t2u;
  DevBuf<long long> d_eoff;
  DevBuf<SiItem> d_items;
  DevBuf<SiGather> d_gather;
};

// error analysis and condition estimation (b200ldlt_error_analysis / b200ldlt_condest, ea_kernels.cu): |A| by rows
// (d_ptr / d_col / d_uid: both triangles of the unique entries, grouped by original row, columns ascending), the unique
// values of the call (k_sum_dups of d_vals: d_uval is scaled in place by the factorisation) and the row maxima a_i; per
// right-hand side r and s, overwritten by w1 and w2, and the reduced norms (grown to the largest call); the estimators'
// input / product vectors and sign vectors (one column per estimator of a block) and the reduction scratch of
// k_ea_post; for the refinement (b200ldlt_solve_refined) the solve slots of a block (r, then d) and the rollback copies
// of its x; for FGMRES (b200ldlt_solve_gmres) the Krylov vectors V and Z of each column of a block (grown to the largest
// call), its Hessenberg columns, y, and the reduction scratch of the dots and norms.  Built at the first call after an
// analysis, before its timing starts; a handle that never makes the calls allocates none of it.
struct EaPlan {
  DevBuf<int> d_ptr, d_col, d_uid;
  DevBuf<double> d_uval, d_amax, d_rs, d_v, d_rf_d, d_rf_old;
  DevBuf<double> d_gm_kv, d_gm_h, d_gm_y, d_gm_part;
  DevBuf<unsigned> d_gm_cnt;
  DevBuf<unsigned long long> d_nrm;
  DevBuf<signed char> d_xi;
  DevBuf<EaPart> d_part;
  DevBuf<EaRes> d_res;
  DevBuf<unsigned> d_cnt;
};

struct LevelPlan {
  // big fronts of the level: [big_off, big_off+big_cnt) in front_list
  int big_off = 0, big_cnt = 0, big_kmax = 0, big_fmax = 0, big_rmax = 0, big_chmax = 0;
  long long big_entmax = 0, big_zero_max = 0;
  struct Bucket { int off, cnt, fmax, kmax, threads; size_t smem; int kind = 0; };   // kind 2: k_front_warp2 (order 33..64, <= 32 pivots)
  std::vector<Bucket> small;
  // Schur complements of the level's big fronts: tensor-core (Ozaki int8, schur_tc.cu) for r >= tc_min_r, DFMA tiles else
  int tc_f_off = 0, tc_f_cnt = 0, tc_t_off = 0, tc_t_cnt = 0, tc_rmax = 0;
  int df_off = 0, df_cnt = 0, df_rmax = 0;
};

// device lists behind LevelPlan::tc_* / df_* of one plan set
struct SchurLists {
  DevBuf<TcFront> d_f;
  DevBuf<TcTile> d_t;
  DevBuf<int> d_dfl;
  std::vector<TcFront> f;
  std::vector<TcTile> t;
  std::vector<int> dfl;
  long long dig_bytes = 0, exp_ints = 0;   // scratch needed by the largest level
};

// what one set of fronts needs (build_front_plan): the factorisation's level plans, Schur lists and device front list,
// the explicit L11^-1 work of the whole set and, when filled, the same work split by tree level (issued behind each
// level's chain), and the triangular-solve plan
struct FrontPlan {
  std::vector<LevelPlan> levels;
  SchurLists schur;
  DevBuf<int> d_fl;
  LinvPlan linv;
  std::vector<std::unique_ptr<LinvPlan>> linv_level;
  SolvePlan solve;
};

// environment switches for profiling / A-B runs, read ONCE at b200ldlt_create (never on the enqueue path)
struct DebugSwitches {
  bool one_stream = false;        // B200_ONE_STREAM=1: big-front pipeline on a single stream
  bool cb_at_end = false;         // B200_CB_AT_END=1: Schur complements as one GEMM per level (k_big_schur84) instead of per-panel updates
  int solve_direct = 2;           // B200_SOLVE_DIRECT=D: the D lowest tree levels are solved by k_solve_direct (0 = all inside the subtrees)
  bool solve_nopair = false;      // B200_SOLVE_NOPAIR=1: one subtree per CTA in the solve sweeps (no side-by-side pairs)
  int solve_block = MS_NB_MAX;    // B200_SOLVE_BLOCK=n: nrhs > 1 solved in blocks of at most n columns (1 = one solve per column)
  bool no_warp2 = false;          // B200_NO_WARP2=1: fronts of order 33..64 by the shared-memory kernel (one CTA each) instead of k_front_warp2
  bool no_pdl = false;            // B200_NO_PDL=1: chain kernels launched without programmatic dependent launch
  void read() {
    one_stream = getenv("B200_ONE_STREAM") != nullptr;
    cb_at_end = getenv("B200_CB_AT_END") != nullptr;
    solve_nopair = getenv("B200_SOLVE_NOPAIR") != nullptr;
    if (const char* e = getenv("B200_SOLVE_DIRECT")) solve_direct = atoi(e);
    if (const char* e = getenv("B200_SOLVE_BLOCK")) solve_block = std::min(std::max(atoi(e), 1), MS_NB_MAX);
    no_pdl = getenv("B200_NO_PDL") != nullptr;
    no_warp2 = getenv("B200_NO_WARP2") != nullptr;
  }
};

// Everything one analysis derives: the symbolic structure and its device copies, the factor and contribution-block
// storage, the plans and sweep states, the per-call plans built at their first call, the shard plan, the captured
// factorisation and the staging of the host entry points.  A new analysis replaces it whole and a failed one leaves
// none, so nothing sized by an old analysis can outlive it.
struct Analysis {
  Symbolic S;
  FrontPlan fronts;                  // factorisation: all fronts but the Schur root; solves: all fronts
  bool factored = false;
  DevBuf<int8_t> d_tc_dig;           // digit scratch of the tensor-core Schur path (largest level)
  DevBuf<int> d_tc_exp;
  DevBuf<int> d_sn_start, d_sn_parent, d_rows, d_rel, d_child_ptr, d_child_idx, d_perm;
  DevBuf<int> d_useg_src, d_u_row, d_u_col, d_irn, d_jcn;
  DevBuf<long long> d_rows_ptr, d_uent_ptr, d_u_dst64, d_L_off, d_cb_off, d_useg_ptr;
  DevBuf<unsigned> d_u_dst;
  DevBuf<double> d_uval, d_L, d_W, d_CB, d_dinv, d_doff, d_scale, d_res, d_colmax;
  DevBuf<int> d_ptype, d_lperm, d_bperm, d_counters, d_einv;
  DevBuf<long long> d_einv_off;
  DevBuf<unsigned long long> d_rmax;
  DevSym DS;
  DevNum DN;
  // solve (solve_dataflow.cu): per-front tables, sweep states + one plan per front set
  SweepState sweep;                 // one column: every single-column solve (also the sharded one), device_ptr "x" / "cbv"
  std::unique_ptr<SweepState> blk;  // blocked solve: B200_SOLVE_BLOCK columns, allocated at the first nrhs > 1 solve
                                    // (width 0: the column loop)
  DevBuf<int> d_boff;
  DevBuf<long long> d_bigv_off;
  DevBuf<long long> d_piv_big;      // n : per pivot position, its index in bigv (pivots of big fronts) or -1 (partial solves)
  std::unique_ptr<LmulPlan> lmul;   // lmultiply: built at its first call
  std::unique_ptr<PrunedPlan> pruned;   // sparse forward solve / inverse entries / sparse solve: built at the first such call
  std::unique_ptr<SelInvPlan> selinv;   // selected inversion: built at its first call
  std::unique_ptr<EaPlan> ea;       // error analysis / condest: built at the first such call
  // zero pivots (b200ldlt_set_singular_action): the factor kernels append every forced zero pivot to d_zlist; with
  // keep_singular a factorisation whose zero pivots are all noise pivots keeps its factors, with dinv = 0 at zpos
  DevBuf<int> d_zlist, d_zpos;
  DevBuf<unsigned char> d_zflag;    // n : 1 at the zero pivots of the kept factors
  std::vector<int> zpos;            // the zero pivots of the kept factors, ascending (empty otherwise)
  DevBuf<double> d_fred_z;          // solve_fredholm without a blocked state: z of one column, pivot order
  // Schur mode: an analysis with the handle's Schur variables makes supernode sc_root (the last one) their root front,
  // which the factorisation assembles but does not factor; d_sc then holds S_c (m x m, column-major)
  int sc_root = -1, sc_nch = 0;
  long long sc_nent = 0, sc_linv_off = 0;   // its unique entries; its L11^-1 block in d_linv (order > 256)
  DevBuf<int> d_sc_vars, d_sc_root;
  DevBuf<double> d_sc;
  DevBuf<double> d_linv;
  DevBuf<double> d_linv_part;       // partial tiles of the chunked k_linv_gemm items (one launch at a time uses it)
  DevBuf<int> d_linv_cnt;           // their arrival counters (self-resetting)
  DevBuf<long long> d_linv_off, d_gmap_off;
  std::vector<long long> linv_off;  // per supernode: its L11^-1 block in d_linv (order > 256), else -1
  DevBuf<FrontDesc> d_fdesc;
  DevBuf<int> d_gmap;
  std::vector<char> solve_direct_front;   // per supernode: solved by k_solve_direct (see build_solve_tables)
  int solve_epoch = 0;
  struct Shard {
    bool active = false;
    int rank = 0, world = 1, nsub = 0;
    std::vector<int> owner, cut_roots, top_fronts;
    FrontPlan part[2];                       // [0] my subtrees, [1] top part
    DevBuf<int> d_mark_cut, d_mark_top;
  } shard;
  cudaGraph_t fgraph = nullptr;
  cudaGraphExec_t fgraph_exec = nullptr;
  double fgraph_u = -1.0;
  int fgraph_launches = 0;
  double* h_rhs = nullptr;          // pinned staging of the host entry points: d_rhs.n doubles, like d_rhs (staged_call)
  DevBuf<double> d_rhs;

  ~Analysis() {
    if (fgraph_exec) cudaGraphExecDestroy(fgraph_exec);
    if (fgraph) cudaGraphDestroy(fgraph);
    if (h_rhs) cudaFreeHost(h_rhs);
  }
};

struct Solver {
  b200ldlt_options opt;
  DebugSwitches dbg;
  std::string err;
  int dev = 0;
  cudaStream_t stream = nullptr;
  cudaStream_t stream2 = nullptr;      // bulk (trsm / trailing update) stream of the big-front pipeline
  cudaStream_t stream3 = nullptr;      // explicit L11 inverses of a level's big fronts (trail behind the chain)
  cudaStream_t side[4] = {nullptr, nullptr, nullptr, nullptr};   // the shared-memory front classes of a level run side by side
  std::vector<cudaEvent_t> ev_pool;
  size_t ev_next = 0;
  bool own_stream = false;
  cudaEvent_t ev0 = nullptr, ev1 = nullptr, ev_zero = nullptr;
  cudaEvent_t ev_chunk[4] = {nullptr, nullptr, nullptr, nullptr};   // D2H chunks of staged_call

  int n = 0, nnz = 0;
  std::vector<int> irn, jcn;
  double* h_vals = nullptr;      // pinned
  int* h_counters = nullptr;     // pinned
  DevBuf<double> d_vals;         // the values on the device (nnz): allocated at the first need, released with the pattern
  bool have_dev_vals = false;
  b200vec_ctx vec = nullptr;       // vector kernels on the handle's stream (device-side refinement)
  b200vec_tmat amat = nullptr;     // the matrix as a symmetric triplet operator (residuals)
  DevBuf<double> d_ref_b, d_ref_r;
  int tc_min_r = 0;                // fronts with r >= this use the tensor-core Schur path (0 = off)
  bool reanalyse = false;          // set by increase_quality after forced pivots: next factor re-runs the analysis on its values
  int n_reanalysed = 0;
  bool reanalysed_since_raise = false;
  std::unique_ptr<Analysis> an;    // null: not analysed (none yet, a new pattern, or the last analysis failed)
  b200ldlt_info info;
  int num_neg = 0;
  double pivtol = 1e-8;
  int launches = 0;
  DevBuf<double> d_alter;           // alter_d: the caller's 2n entries of D^-1 (allocated at the first call)
  DevBuf<int> d_alter_bad;
  bool keep_singular = false;       // b200ldlt_set_singular_action (see Analysis::zpos)
  DevBuf<unsigned long long> d_fred_nrm;   // solve_fredholm: the two max-norms per column
  // Schur mode (b200ldlt_set_schur): the caller's Schur variables, given to every analysis until b200ldlt_analyse or
  // set_schur(0) clears them
  std::vector<int> sc_vars;
  int num_sms = 132;

  ~Solver() {
    an.reset();   // (its graph and pinned buffers before the streams and events)
    if (amat) b200vec_tmat_destroy(amat);
    if (vec) b200vec_destroy(vec);
    if (h_vals) cudaFreeHost(h_vals);
    if (h_counters) cudaFreeHost(h_counters);
    if (ev0) cudaEventDestroy(ev0);
    if (ev1) cudaEventDestroy(ev1);
    for (cudaEvent_t e : ev_chunk) if (e) cudaEventDestroy(e);
    for (cudaEvent_t e : ev_pool) cudaEventDestroy(e);
    if (stream2) cudaStreamDestroy(stream2);
    if (stream3) cudaStreamDestroy(stream3);
    for (auto& q : side) if (q) cudaStreamDestroy(q);
    if (own_stream && stream) cudaStreamDestroy(stream);
  }
  cudaEvent_t next_event() {
    if (ev_next == ev_pool.size()) { cudaEvent_t e; cudaEventCreateWithFlags(&e, cudaEventDisableTiming); ev_pool.push_back(e); }
    return ev_pool[ev_next++];
  }
};

#define CU(call)                                                                         \
  do {                                                                                   \
    cudaError_t e__ = (call);                                                            \
    if (e__ != cudaSuccess) {                                                            \
      sv->err = std::string(#call) + ": " + cudaGetErrorString(e__);                     \
      if (sv->opt.verbose) fprintf(stderr, "[b200ldlt] CUDA error: %s\n", sv->err.c_str()); \
      return B200LDLT_FATAL_ERROR;                                                       \
    }                                                                                    \
  } while (0)

// per level: big fronts first, then the shared-memory classes by descending front order; only fronts with take[s]
static void build_level_plans(const Symbolic& S, int smax, const std::vector<char>& take, std::vector<int>& fl,
                              std::vector<LevelPlan>& plan, SchurLists& SL, int tc_min_r,
                              bool use_warp2) {
  SL.f.clear(); SL.t.clear(); SL.dfl.clear(); SL.dig_bytes = 0; SL.exp_ints = 0;
  fl.clear();
  fl.reserve(S.nsn);
  plan.assign(S.nlevels, LevelPlan());
  for (int l = 0; l < S.nlevels; ++l) {
    LevelPlan& P = plan[l];
    P.big_off = (int)fl.size();
    for (int q = S.level_ptr[l]; q < S.level_ptr[l + 1]; ++q) {
      int s = S.level_sn[q];
      if (!take[s]) continue;
      if (S.f(s) > smax) {
        fl.push_back(s);
        P.big_cnt++;
        P.big_kmax = std::max(P.big_kmax, S.k(s));
        P.big_fmax = std::max(P.big_fmax, S.f(s));
        P.big_rmax = std::max(P.big_rmax, S.r(s));
        P.big_chmax = std::max(P.big_chmax, S.child_ptr[s + 1] - S.child_ptr[s]);
        P.big_entmax = std::max<long long>(P.big_entmax, S.uent_ptr[s + 1] - S.uent_ptr[s]);
        P.big_zero_max = std::max<long long>(P.big_zero_max, (long long)S.f(s) * S.k(s) + (long long)S.r(s) * S.r(s));
      }
    }
    // Schur complements of the big fronts of this level
    {
      P.tc_f_off = (int)SL.f.size(); P.tc_t_off = (int)SL.t.size(); P.df_off = (int)SL.dfl.size();
      long long dig = 0, ex = 0;
      for (int q = 0; q < P.big_cnt; ++q) {
        const int s = fl[P.big_off + q];
        const int r = S.r(s), k = S.k(s);
        if (r <= 0) continue;
        if (tc_min_r > 0 && r >= tc_min_r && k >= 32) {
          TcFront F;
          F.s = s; F.nks = (k + TC_BK - 1) / TC_BK;
          const int nra = (r + TC_BM - 1) / TC_BM, nrb = (r + TC_BN - 1) / TC_BN;
          F.a_off = dig; dig += (long long)nra * F.nks * TC_A_UNIT;
          F.b_off = dig; dig += (long long)nrb * F.nks * TC_B_UNIT;
          F.e_off = ex; ex += 2LL * r;
          const int fi = (int)SL.f.size() - P.tc_f_off;
          SL.f.push_back(F);
          for (int ti = 0; ti < nra; ++ti)
            for (int tj = 0; tj < nrb && tj * TC_BN <= ti * TC_BM + TC_BM - 1; ++tj) SL.t.push_back(TcTile{fi, ti, tj});
          P.tc_rmax = std::max(P.tc_rmax, r);
        } else {
          SL.dfl.push_back(s);
          P.df_rmax = std::max(P.df_rmax, r);
        }
      }
      P.tc_f_cnt = (int)SL.f.size() - P.tc_f_off; P.tc_t_cnt = (int)SL.t.size() - P.tc_t_off; P.df_cnt = (int)SL.dfl.size() - P.df_off;
      SL.dig_bytes = std::max(SL.dig_bytes, dig); SL.exp_ints = std::max(SL.exp_ints, ex);
    }
    // small fronts (level_sn is sorted by f descending inside a level)
    // Size classes: (64, smax] 256 threads, (32, 64] 128 threads, <= 32 one warp per front.  Inside a class the
    // fronts are split again at the soft limits below (shared memory per CTA follows the largest front of a launch,
    // so finer buckets raise the number of resident CTAs per SM); a soft split only happens once the current bucket
    // holds enough fronts to fill the GPU.  Soft limits at 48 and 96: the classes of a level run side by side, so a finer
    // split costs no serial launches (H100 SXM, 700 W, factorisation at N=400 / 800: {96} and {32,64,96} within 0.4 %).
    const int kSoft[] = {48, 96};
    const int kMinBucket = 296;
    auto threads_of = [](int f) { return f > 64 ? 256 : (f > 32 ? 128 : 64); };
    LevelPlan::Bucket cur{(int)fl.size(), 0, 0, 0, 256, 0};
    int cur_lo = 1 << 30;   // the current bucket accepts f > cur_lo ... (set when the bucket gets its first front)
    std::vector<int> w2;    // order 33..64 with <= 32 pivot columns: register kernel, two rows per lane
    for (int q = S.level_ptr[l]; q < S.level_ptr[l + 1]; ++q) {
      int s = S.level_sn[q];
      int f = S.f(s);
      if (!take[s] || f > smax) continue;
      if (use_warp2 && f > 32 && f <= 64 && S.k(s) <= 32) { w2.push_back(s); continue; }
      bool split = false;
      if (cur.cnt) {
        if (threads_of(f) != cur.threads) split = true;
        else if (cur.cnt >= kMinBucket && f <= cur_lo) split = true;
      }
      if (split) { P.small.push_back(cur); cur = LevelPlan::Bucket{(int)fl.size(), 0, 0, 0, 256, 0}; }
      if (cur.cnt == 0) cur.off = (int)fl.size();
      if (cur.cnt == 0) {
        cur.threads = threads_of(f);
        cur_lo = 0;
        for (int v : kSoft) if (v < f) cur_lo = std::max(cur_lo, v);
      }
      fl.push_back(s);
      cur.cnt++;
      cur.fmax = std::max(cur.fmax, f);
      cur.kmax = std::max(cur.kmax, S.k(s));
    }
    if (cur.cnt) P.small.push_back(cur);
    for (auto& bk : P.small) {
      size_t ld = (size_t)(bk.fmax | 1);
      bk.smem = (ld * bk.fmax + 2 * (size_t)bk.fmax) * sizeof(double) + (2 * (size_t)bk.kmax + 8) * sizeof(int);
    }
    if (!w2.empty()) {
      LevelPlan::Bucket bk{(int)fl.size(), (int)w2.size(), 64, 32, 128, 4 * (size_t)S2_SMEM_PER_WARP};
      bk.kind = 2;
      for (int s : w2) fl.push_back(s);
      P.small.insert(P.small.begin(), bk);     // the most numerous class first (it gets the main stream when there are no big fronts)
    }
  }
}

static const int kSolveMidMax = 256;   // fronts above this order are "big" in the solve (block tasks + explicit L11 inverse)

static int build_linv_plan(Solver* sv, Analysis& A, const std::vector<char>& take, LinvPlan& LP, cudaStream_t st) {
  const Symbolic& S = A.S;
  std::vector<int> pairs;
  int maxkb = 0;
  for (int s = 0; s < S.nsn; ++s) if (take[s] && S.f(s) > kSolveMidMax) {
    const int nkb = (S.k(s) + DF_BLK - 1) / DF_BLK;
    maxkb = std::max(maxkb, nkb);
    for (int b = 0; b < nkb; ++b) { pairs.push_back(s); pairs.push_back(b); }
  }
  LP.ndiag = (int)pairs.size() / 2;
  if (pairs.empty()) pairs.push_back(0);
  CU(LP.d_diag.upload(pairs, st));
  LP.d_g.clear(); LP.d_g2.clear(); LP.ng.clear(); LP.ng2.clear(); LP.part_tiles = 0;
  for (int Bt = 1; Bt < maxkb; Bt *= 2) {   // merge neighbouring blocks of Bt tiles
    std::vector<LinvItem> g1, g2;
    for (int s = 0; s < S.nsn; ++s) if (take[s] && S.f(s) > kSolveMidMax) {
      const int nkb = (S.k(s) + DF_BLK - 1) / DF_BLK;
      for (int a0 = 0; a0 + Bt < nkb; a0 += 2 * Bt) {
        const int a1 = a0 + Bt, b1 = std::min(a1 + Bt, nkb);   // first block [a0,a1), second [a1,b1)
        for (int ib = a1; ib < b1; ++ib)
          for (int jb = a0; jb < a1; ++jb) {
            g1.push_back(LinvItem{s, ib, jb, jb, a1, 1, 0, 0});        // T[ib,jb]    =  sum_{m=jb..a1-1} L[ib,m] Inv11[m,jb]
            g2.push_back(LinvItem{s, ib, jb, a1, ib + 1, 1, 0, 0});    // Linv[ib,jb] = -sum_{m=a1..ib}   Inv22[ib,m] T[m,jb]
          }
      }
    }
    // long k-ranges -> chunks of LINV_KCHUNK tiles (partial sums combined by the last chunk to arrive, in chunk order)
    auto split = [&](std::vector<LinvItem>& g) {
      std::vector<LinvItem> out;
      int base = 0;                          // first scratch tile (and counter index) of the item being cut
      for (const LinvItem& it : g) {
        const int K = it.m1 - it.m0, nch = (K + LINV_KCHUNK - 1) / LINV_KCHUNK;
        if (nch <= 1) { out.push_back(it); continue; }
        for (int c = 0; c < nch; ++c)
          out.push_back(LinvItem{it.s, it.ib, it.jb, it.m0 + c * LINV_KCHUNK, std::min(it.m1, it.m0 + (c + 1) * LINV_KCHUNK), nch, c, base});
        base += nch;
      }
      LP.part_tiles = std::max<long long>(LP.part_tiles, base);
      g.swap(out);
    };
    split(g1);
    split(g2);
    LP.ng.push_back((int)g1.size());
    if (g1.empty()) { g1.push_back(LinvItem{0, 0, 0, 0, 0, 1, 0, 0}); g2.push_back(LinvItem{0, 0, 0, 0, 0, 1, 0, 0}); }
    LP.ng2.push_back((int)g2.size());
    LP.d_g.emplace_back(new DevBuf<LinvItem>());
    LP.d_g2.emplace_back(new DevBuf<LinvItem>());
    CU(LP.d_g.back()->upload(g1, st));
    CU(LP.d_g2.back()->upload(g2, st));
  }
  if ((size_t)LP.part_tiles > A.d_linv_cnt.n) {     // (analysis time: never inside a captured graph)
    CU(cudaStreamSynchronize(st));
    CU(A.d_linv_part.alloc((size_t)LP.part_tiles * 4096));
    CU(A.d_linv_cnt.alloc((size_t)LP.part_tiles));
    CU(cudaMemset(A.d_linv_cnt.p, 0, A.d_linv_cnt.n * sizeof(int)));
  }
  return B200LDLT_SUCCESS;
}

static int enqueue_linv(Solver* sv, const LinvPlan& LP, cudaStream_t st);

// Triangular-solve plan of the fronts in take[] (see solve_dataflow.cu).
//  * Subtrees: maximal subtrees whose fronts are all taken, of order <= DF_MIDMAX, and whose whole working set (SubLayout)
//    fits the dynamic shared memory of k_solve_sub -> one CTA each, largest first.  Supernodes are numbered in postorder,
//    so a subtree is the contiguous range [root - size + 1, root] and so are its panels, columns, row lists, child lists.
//  * Everything else -> topologically sorted task lists for k_solve_top (forward: levels ascending; backward: descending).
static int build_solve_plan(Solver* sv, const Analysis& A, const std::vector<char>& take, SolvePlan& SP, cudaStream_t st) {
  const Symbolic& S = A.S;
  const int nsn = S.nsn;
  std::vector<int> size(nsn, 1), ntaken(nsn, 0), subF(nsn, 0);
  for (int s = 0; s < nsn; ++s) {   // children precede parents
    ntaken[s] += take[s] ? 1 : 0; subF[s] = std::max(subF[s], S.f(s));
    const int p = S.sn_parent[s];
    if (p >= 0) { size[p] += size[s]; ntaken[p] += ntaken[s]; subF[p] = std::max(subF[p], subF[s]); }
  }
  const std::vector<char>& direct = A.solve_direct_front;
  // compact panel bytes of the fronts of [s0, s] that are walked inside a subtree (not owned by the direct kernel)
  std::vector<long long> ownL(nsn + 1, 0);   // prefix sums over supernodes
  std::vector<int> ownN(nsn + 1, 0);
  for (int q = 0; q < nsn; ++q) {
    ownL[q + 1] = ownL[q] + (direct[q] ? 0 : S.L_off[q + 1] - S.L_off[q]);
    ownN[q + 1] = ownN[q] + (direct[q] ? 0 : 1);
  }
  auto layout_of = [&](int s) {
    const int s0 = s - size[s] + 1;
    SubLayout L;
    L.nL = ownL[s + 1] - ownL[s0];
    L.ncol = S.sn_start[s + 1] - S.sn_start[s0];
    L.nrt = (int)(S.rows_ptr[s + 1] - S.rows_ptr[s0]);
    L.rroot = S.r(s);
    L.nchi = S.child_ptr[s + 1] - S.child_ptr[s0];
    L.nfront = size[s];
    L.nmeta = 2 * (S.sn_level[s] + 1) + 1 + size[s];   // upper bound (levels <= height of the root + 1)
    return L;
  };
  auto ok = [&](int s) {
    if (!take[s] || ntaken[s] != size[s] || subF[s] > DF_MIDMAX || size[s] > 4096) return false;
    if (s - size[s] + 1 < 0) return false;
    if (direct[s]) return false;        // (then the whole subtree is direct: nothing to walk)
    return layout_of(s).bytes() <= (long long)DF_DYN_SMEM;
  };
  std::vector<char> okv(nsn);
  for (int s = 0; s < nsn; ++s) okv[s] = ok(s) ? 1 : 0;
  std::vector<int> roots;
  std::vector<char> insub(nsn, 0);
  for (int s = nsn - 1; s >= 0; --s) {
    if (!okv[s]) continue;
    const int p = S.sn_parent[s];
    if (p >= 0 && okv[p]) continue;
    roots.push_back(s);
    for (int q = s - size[s] + 1; q <= s; ++q) insub[q] = 1;
  }
  // largest subtree (bytes of L) first
  std::stable_sort(roots.begin(), roots.end(), [&](int a, int b) {
    return ownL[a + 1] - ownL[a - size[a] + 1] > ownL[b + 1] - ownL[b - size[b] + 1];
  });
  std::vector<int> subLoff(std::max(nsn, 1), 0);
  const int nsub = (int)roots.size();
  std::vector<SubDesc> subs(std::max(nsub, 1), SubDesc{});
  std::vector<int> meta;
  SP.sub_bytes = 0;
  for (int u = 0; u < nsub; ++u) {
    const int sR = roots[u], s0 = sR - size[sR] + 1;
    SP.sub_bytes += (ownL[sR + 1] - ownL[s0]) * 8;
    std::vector<int> M;
    for (int q = s0; q <= sR; ++q) {
      subLoff[q] = (int)(ownL[q] - ownL[s0]);
      if (!direct[q]) M.push_back(q);
    }
    // by (level, small first, larger first)
    std::stable_sort(M.begin(), M.end(), [&](int a, int b) {
      if (S.sn_level[a] != S.sn_level[b]) return S.sn_level[a] < S.sn_level[b];
      const bool sa = S.f(a) <= 64, sb = S.f(b) <= 64;
      if (sa != sb) return sa;
      return S.f(a) > S.f(b);
    });
    std::vector<int> lvl(1, 0), nsm;
    for (size_t q = 0; q < M.size();) {
      size_t e = q; int ns = 0;
      while (e < M.size() && S.sn_level[M[e]] == S.sn_level[M[q]]) { if (S.f(M[e]) <= 64) ++ns; ++e; }
      lvl.push_back((int)e); nsm.push_back(ns);
      q = e;
    }
    {
      SubDesc d{};
      d.s0 = s0; d.sR = sR; d.moff = (int)meta.size(); d.nlv = (int)nsm.size();
      d.col0 = S.sn_start[s0]; d.ncol = S.sn_start[sR + 1] - S.sn_start[s0];
      d.nrt = (int)(S.rows_ptr[sR + 1] - S.rows_ptr[s0]); d.rroot = S.r(sR);
      d.ch00 = S.child_ptr[s0]; d.nchi = S.child_ptr[sR + 1] - S.child_ptr[s0];
      d.parent = S.sn_parent[sR];
      d.nL = ownL[sR + 1] - ownL[s0]; d.ro0 = S.rows_ptr[s0]; d.nown = (int)M.size();
      d.sbytes = (int)((layout_of(sR).bytes() + 127) / 128 * 128);
      subs[u] = d;
    }
    meta.insert(meta.end(), lvl.begin(), lvl.end());
    meta.insert(meta.end(), nsm.begin(), nsm.end());
    meta.insert(meta.end(), M.begin(), M.end());
  }
  // Work items of the subtree phase.  The walk of one subtree is latency-bound (a few fronts per level, dependent
  // shuffle chains) and most subtrees need less than half of the shared memory, so two of them share a CTA whenever their
  // layouts fit together: the largest unpaired subtree takes the smallest one that still fits (both halves of the CTA
  // work independently).  Items are issued by decreasing panel bytes (the hardware scheduler then does LPT).
  std::vector<int2> pairs;
  {
    int lo = 0, hi = nsub - 1;      // subs[] is sorted by decreasing panel size
    const bool pairing = !sv->dbg.solve_nopair;
    while (lo <= hi) {
      if (pairing && lo < hi && (long long)subs[lo].sbytes + subs[hi].sbytes <= (long long)DF_DYN_SMEM) {
        pairs.push_back(make_int2(lo, hi)); ++lo; --hi;
      } else {
        pairs.push_back(make_int2(lo, -1)); ++lo;
      }
    }
    std::stable_sort(pairs.begin(), pairs.end(), [&](const int2& a, const int2& b) {
      const long long wa = subs[a.x].nL + (a.y >= 0 ? subs[a.y].nL : 0), wb = subs[b.x].nL + (b.y >= 0 ? subs[b.y].nL : 0);
      return wa > wb;
    });
  }
  SP.npair = (int)pairs.size();
  if (pairs.empty()) pairs.push_back(make_int2(0, -1));
  CU(SP.d_subpair.upload(pairs, st));
  // backward addresses of the contribution rows of the subtree fronts: a row inside the subtree's column range is a local
  // index into its x slice (>= 0); a row above it is one of the ROOT's contribution rows (every row of a descendant
  // beyond the root's columns is in the root's row list): -(1 + position there)
  std::vector<int> subrow(std::max<size_t>(S.rows.size(), 1), 0);
  for (int u = 0; u < nsub; ++u) {
    const int sR = roots[u], s0 = sR - size[sR] + 1;
    const int col0 = S.sn_start[s0], col1 = S.sn_start[sR + 1];
    const int* rr = S.rows.data() + S.rows_ptr[sR];
    const int nr = S.r(sR);
    for (long long e = S.rows_ptr[s0]; e < S.rows_ptr[sR + 1]; ++e) {
      const int g = S.rows[e];
      if (g < col1) subrow[e] = g - col0;
      else {
        const int* it = std::lower_bound(rr, rr + nr, g);
        if (it == rr + nr || *it != g) { sv->err = "solve plan: row of a subtree front missing from the root's row list"; return B200LDLT_FATAL_ERROR; }
        subrow[e] = -(1 + (int)(it - rr));
      }
    }
  }
  CU(SP.d_subrow.upload(subrow, st));
  // top task lists
  std::vector<SolveTask> tf, tb;
  std::vector<int> bundle;
  int ncidx = 0;
  long long npart = 0;
  auto chunked = [&](std::vector<SolveTask>& T, int type, int s, int blk, int t0, int t1) {
    const int ntile = t1 - t0;
    const int nq = std::max(1, (ntile + DF_CH - 1) / DF_CH);
    for (int q = 0; q < nq; ++q) {
      SolveTask k{type, s, blk, t0 + q * DF_CH, std::min(t1, t0 + (q + 1) * DF_CH), q, nq, (int)npart, ncidx, 0};
      if (ntile <= 0) { k.t0 = t0; k.t1 = t0; }
      T.push_back(k);
    }
    npart += nq; ncidx += 1;
  };
  for (int pass = 0; pass < 2; ++pass) {
    std::vector<SolveTask>& T = pass == 0 ? tf : tb;
    for (int li = 0; li < S.nlevels; ++li) {
      const int l = pass == 0 ? li : S.nlevels - 1 - li;
      std::vector<int> smalls;
      for (int phase = 0; phase < 2; ++phase)
        for (int q = S.level_ptr[l]; q < S.level_ptr[l + 1]; ++q) {
          const int s = S.level_sn[q];
          if (!take[s] || insub[s] || direct[s] || S.f(s) <= DF_MIDMAX) continue;
          const int nkb = (S.k(s) + DF_BLK - 1) / DF_BLK, ncb = (S.r(s) + DF_BLK - 1) / DF_BLK;
          if (pass == 0 && phase == 0) for (int b = nkb - 1; b >= 0; --b) chunked(T, ST_FP, s, b, 0, b + 1);
          if (pass == 0 && phase == 1) for (int j = 0; j < ncb; ++j) chunked(T, ST_FC, s, j, 0, nkb);
          if (pass == 1 && phase == 0) for (int b = 0; b < nkb; ++b) chunked(T, ST_BT, s, b, 0, ncb);
          if (pass == 1 && phase == 1) for (int b = 0; b < nkb; ++b) chunked(T, ST_BX, s, b, b, nkb);
        }
      for (int q = S.level_ptr[l]; q < S.level_ptr[l + 1]; ++q) {
        const int s = S.level_sn[q];
        if (!take[s] || insub[s] || direct[s] || S.f(s) > DF_MIDMAX) continue;
        if (S.f(s) > 64) T.push_back(SolveTask{ST_MID, s, 0, 0, 0, 0, 1, 0, 0, 0});
        else smalls.push_back(s);
      }
      for (size_t q = 0; q < smalls.size(); q += 8) {
        const int cnt = (int)std::min<size_t>(8, smalls.size() - q);
        T.push_back(SolveTask{ST_SMALL, (int)bundle.size(), cnt, 0, 0, 0, 1, 0, 0, 0});
        for (int w = 0; w < cnt; ++w) bundle.push_back(smalls[q + w]);
      }
    }
  }
  // the bottom levels owned by k_solve_direct, one list per level
  SP.d_direct.clear(); SP.direct_cnt.clear(); SP.direct.clear();
  long long ndirect = 0, direct_nnz = 0;
  for (int l = 0; l < S.nlevels && l < sv->dbg.solve_direct; ++l) {
    std::vector<int> lst;
    for (int q = S.level_ptr[l]; q < S.level_ptr[l + 1]; ++q) {
      const int s = S.level_sn[q];
      if (take[s] && direct[s]) { lst.push_back(s); direct_nnz += S.L_off[s + 1] - S.L_off[s]; }
    }
    ndirect += (long long)lst.size();
    SP.direct_cnt.push_back((int)lst.size());
    SP.d_direct.emplace_back(new DevBuf<int>());
    if (lst.empty()) lst.push_back(0);
    CU(SP.d_direct.back()->upload(lst, st));
    SP.direct.push_back(std::move(lst));
  }
  CU(SP.d_sub_Loff.upload(subLoff, st));
  if (sv->opt.verbose)
    fprintf(stderr, "[b200ldlt] solve plan: %lld fronts (%.1f MB of L) on %d bottom levels by the direct kernel\n", ndirect,
            direct_nnz * 8 / 1e6, (int)SP.direct_cnt.size());
  SP.nsub = nsub; SP.ntf = (int)tf.size(); SP.ntb = (int)tb.size();
  if (sv->opt.verbose)
    fprintf(stderr, "[b200ldlt] solve plan: %d subtrees in %d work items (%.1f MB of L, largest %.0f KB), top: %d fwd / %d bwd tasks, %lld partial slots\n",
            nsub, SP.npair, SP.sub_bytes / 1e6, nsub ? (ownL[roots[0] + 1] - ownL[roots[0] - size[roots[0]] + 1]) * 8 / 1e3 : 0.0, SP.ntf, SP.ntb, npart);
  if (tf.empty()) tf.push_back(SolveTask{ST_SMALL, 0, 0, 0, 0, 0, 1, 0, 0, 0});
  if (tb.empty()) tb.push_back(SolveTask{ST_SMALL, 0, 0, 0, 0, 0, 1, 0, 0, 0});
  if (bundle.empty()) bundle.push_back(0);
  if (meta.empty()) meta.push_back(0);
  CU(SP.d_tf.upload(tf, st)); CU(SP.d_tb.upload(tb, st));
  CU(SP.d_bundle.upload(bundle, st));
  CU(SP.d_subs.upload(subs, st)); CU(SP.d_sub_meta.upload(meta, st));
  CU(SP.d_ccnt.alloc(std::max(ncidx, 1)));
  CU(cudaMemsetAsync(SP.d_ccnt.p, 0, SP.d_ccnt.n * sizeof(int), st));
  CU(SP.d_part.alloc(std::max<long long>(npart, 1) * 64));
  SP.tf = std::move(tf); SP.tb = std::move(tb); SP.pairs = std::move(pairs); SP.subs = std::move(subs);
  SP.meta = std::move(meta); SP.bundle = std::move(bundle);
  return B200LDLT_SUCCESS;
}

// per-front records shared by every solve plan: descriptors, gather maps of the big fronts, backward row addresses
static int build_solve_tables(Solver* sv, Analysis& A, cudaStream_t st) {
  const Symbolic& S = A.S;
  const int nsn = S.nsn;
  // fronts owned by k_solve_direct: on the lowest levels, order <= 64, all children of the same kind (children precede parents)
  A.solve_direct_front.assign(nsn, 0);
  for (int s = 0; s < nsn; ++s) {
    if (S.sn_level[s] >= sv->dbg.solve_direct || S.f(s) > 64) continue;
    bool all = true;
    for (int q = S.child_ptr[s]; q < S.child_ptr[s + 1]; ++q) all = all && A.solve_direct_front[S.child_idx[q]];
    A.solve_direct_front[s] = all ? 1 : 0;
  }
  std::vector<FrontDesc> fd(nsn);
  for (int s = 0; s < nsn; ++s) {
    FrontDesc& d = fd[s];
    d.c0 = S.sn_start[s]; d.k = (unsigned short)S.k(s); d.r = (unsigned short)S.r(s);
    d.ch0 = S.child_ptr[s];
    const int nch = S.child_ptr[s + 1] - S.child_ptr[s];
    if (nch > 65535) { sv->err = "front with more than 65535 children"; return B200LDLT_FATAL_ERROR; }
    d.nch = (unsigned short)nch; d.direct = (unsigned short)A.solve_direct_front[s];
    d.L_off = S.L_off[s]; d.ro = S.rows_ptr[s];
  }
  CU(A.d_fdesc.upload(fd, st));
  // gather maps of the big fronts: for child slot q and parent row j, the index into cbv (or -1)
  {
    std::vector<long long> goff(nsn, 0);
    long long tot = 0;
    for (int s = 0; s < nsn; ++s) if (S.f(s) > DF_MIDMAX) {
      goff[s] = tot; tot += (long long)S.f(s) * (S.child_ptr[s + 1] - S.child_ptr[s]);
    }
    if (S.rows.size() >= (size_t)1 << 31) { sv->err = "row structure too large for 32-bit gather maps"; return B200LDLT_FATAL_ERROR; }
    std::vector<int> gm((size_t)std::max<long long>(tot, 1), -1);
    for (int s = 0; s < nsn; ++s) if (S.f(s) > DF_MIDMAX) {
      const int f = S.f(s);
      for (int q = S.child_ptr[s]; q < S.child_ptr[s + 1]; ++q) {
        const int c = S.child_idx[q];
        const long long ro = S.rows_ptr[c];
        const int rc = S.r(c);
        int* dst = gm.data() + goff[s] + (long long)(q - S.child_ptr[s]) * f;
        for (int j = 0; j < rc; ++j) dst[S.rel[ro + j]] = (int)(ro + j);
      }
    }
    CU(A.d_gmap_off.upload(goff, st));
    CU(A.d_gmap.upload(gm, st));
  }
  return B200LDLT_SUCCESS;
}

static int upload_schur_lists(Solver* sv, Analysis& A, SchurLists& SL, cudaStream_t st) {
  std::vector<TcFront> f = SL.f; std::vector<TcTile> t = SL.t; std::vector<int> d = SL.dfl;
  if (f.empty()) f.push_back(TcFront{0, 0, 0, 0, 0});
  if (t.empty()) t.push_back(TcTile{0, 0, 0});
  if (d.empty()) d.push_back(0);
  CU(SL.d_f.upload(f, st)); CU(SL.d_t.upload(t, st)); CU(SL.d_dfl.upload(d, st));
  if ((long long)A.d_tc_dig.n < SL.dig_bytes) CU(A.d_tc_dig.alloc(SL.dig_bytes));
  if ((long long)A.d_tc_exp.n < SL.exp_ints) CU(A.d_tc_exp.alloc(SL.exp_ints));
  return B200LDLT_SUCCESS;
}

// The plan of the fronts in take_factor (factorisation, L11^-1) and take_solve (triangular solves); FP.linv_level is left
// empty.  Needs the solve tables (build_solve_tables).
static int build_front_plan(Solver* sv, Analysis& A, const std::vector<char>& take_factor,
                            const std::vector<char>& take_solve, FrontPlan& FP) {
  const Symbolic& S = A.S;
  cudaStream_t st = sv->stream;
  std::vector<int> fl;
  build_level_plans(S, sv->opt.smem_front_max, take_factor, fl, FP.levels, FP.schur, sv->tc_min_r, !sv->dbg.no_warp2);
  if (fl.empty()) fl.push_back(0);
  CU(FP.d_fl.upload(fl, st));
  FP.linv_level.clear();
  int rc = upload_schur_lists(sv, A, FP.schur, st);
  if (rc == B200LDLT_SUCCESS) rc = build_linv_plan(sv, A, take_factor, FP.linv, st);
  if (rc == B200LDLT_SUCCESS) rc = build_solve_plan(sv, A, take_solve, FP.solve, st);
  return rc;
}

// the persistent sweep kernel for one column (multi = false) or a block of columns; apply_d = false: the forward sweep
// of the partial solves (L only)
static auto sweep_kernel(bool fwd, bool multi, bool apply_d = true) {
  if (fwd && !apply_d) return multi ? k_solve<true, true, false> : k_solve<true, false, false>;
  return fwd ? (multi ? k_solve<true, true> : k_solve<true, false>) : (multi ? k_solve<false, true> : k_solve<false, false>);
}

// Allocates and zeroes the sweep state of M.nb columns, M giving the per-column sizes, and sizes its sweep grid.
static cudaError_t alloc_sweep_state(Solver* sv, SweepState& W, const MultiStride& M) {
  cudaStream_t st = sv->stream;
  const int nb = M.nb;
  W.width = 0;
  W.M = M;
  cudaError_t e;
  if ((e = W.d_x.alloc(M.x * nb)) != cudaSuccess || (e = W.d_cbv.alloc(M.cbv * nb)) != cudaSuccess ||
      (e = W.d_bigv.alloc(M.bigv * nb)) != cudaSuccess || (e = W.d_bigy.alloc(M.bigv * nb)) != cudaSuccess ||
      (e = W.d_part.alloc(M.part * nb)) != cudaSuccess || (e = W.d_ticket.alloc(2)) != cudaSuccess)
    return e;
  DevBuf<int>* flags[] = {&W.d_done_f, &W.d_done_b, &W.d_bcnt, &W.d_bcnt_b, &W.d_bflag_f, &W.d_bflag_b, &W.d_ccnt};
  const long long per_col[] = {M.nsn, M.nsn, M.nsn, M.nsn, M.nbo, M.nbo, M.nccnt};
  for (int i = 0; i < 7; ++i) {
    if ((e = flags[i]->alloc(per_col[i] * nb)) != cudaSuccess) return e;
    if (flags[i]->n && (e = cudaMemsetAsync(flags[i]->p, 0, flags[i]->n * sizeof(int), st)) != cudaSuccess) return e;
  }
  if ((e = cudaMemsetAsync(W.d_ticket.p, 0, 2 * sizeof(unsigned long long), st)) != cudaSuccess) return e;
  W.ticket_f = W.ticket_b = 0;
  int occ = 1, occ_b = 1, occ_l = 1;
  if ((e = cudaFuncSetAttribute(sweep_kernel(true, nb > 1), cudaFuncAttributeMaxDynamicSharedMemorySize, DF_DYN_SMEM)) != cudaSuccess ||
      (e = cudaFuncSetAttribute(sweep_kernel(false, nb > 1), cudaFuncAttributeMaxDynamicSharedMemorySize, DF_DYN_SMEM)) != cudaSuccess ||
      (e = cudaFuncSetAttribute(sweep_kernel(true, nb > 1, false), cudaFuncAttributeMaxDynamicSharedMemorySize, DF_DYN_SMEM)) != cudaSuccess ||
      (e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, sweep_kernel(true, nb > 1), DF_THREADS, DF_DYN_SMEM)) != cudaSuccess ||
      (e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ_b, sweep_kernel(false, nb > 1), DF_THREADS, DF_DYN_SMEM)) != cudaSuccess ||
      (e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ_l, sweep_kernel(true, nb > 1, false), DF_THREADS, DF_DYN_SMEM)) != cudaSuccess)
    return e;
  // every CTA of a persistent sweep must be resident: the grid fits all three sweep kernels (the same in practice: the
  // launch bounds cap each at 128 registers)
  W.grid = std::max(1, std::min(std::min(occ, occ_b), occ_l)) * sv->num_sms;
  if ((e = cudaStreamSynchronize(st)) != cudaSuccess) return e;
  W.width = nb;
  return cudaSuccess;
}

// A new analysis of the handle's pattern on vals.  The old one (and with it the factors) is released first, so its device
// memory is free before the new one is allocated; the new one becomes the handle's only when all of it is built.
static int run_analysis(Solver* sv, const double* vals) {
  sv->an.reset();
  sv->reanalyse = false;
  std::unique_ptr<Analysis> an(new Analysis());
  Analysis& A = *an;
  AnalyseOptions ao;
  ao.ordering = sv->opt.ordering;
  ao.pair_saddle = sv->opt.pair_saddle;
  ao.leaf_k = sv->opt.leaf_k;
  ao.relax_frac = sv->opt.relax_frac;
  ao.sc_vars = sv->sc_vars;
  std::string e;
  int rc = analyse(sv->n, sv->nnz, sv->irn.data(), sv->jcn.data(), vals, ao, A.S, e);
  if (rc != 0) { sv->err = e; return B200LDLT_FATAL_ERROR; }
  Symbolic& S = A.S;
  cudaStream_t st = sv->stream;
  // Schur mode: the root front of S, factored by none of the plans below; assembled by the big-front kernels (one-entry
  // front list d_sc_root), so its children get inverse row maps whatever its order
  const int m = (int)sv->sc_vars.size();
  if (m > 0) {
    const int rt = S.nsn - 1;
    if (S.sn_start[rt] != S.n - m || S.r(rt) != 0 || S.sn_parent[rt] != -1) {
      sv->err = "internal: the Schur variables do not form the last root front";
      return B200LDLT_FATAL_ERROR;
    }
    A.sc_root = rt;
    A.sc_nch = S.child_ptr[rt + 1] - S.child_ptr[rt];
    A.sc_nent = S.uent_ptr[rt + 1] - S.uent_ptr[rt];
    CU(A.d_sc_vars.upload(sv->sc_vars, st));
    CU(A.d_sc_root.upload(std::vector<int>{rt}, st));
    CU(A.d_sc.alloc((size_t)m * m));
  }
  // the fronts the factorisation factors: all but the Schur root
  std::vector<char> take_f(S.nsn, 1);
  if (A.sc_root >= 0) take_f[A.sc_root] = 0;
  CU(A.d_sn_start.upload(S.sn_start, st));
  CU(A.d_sn_parent.upload(S.sn_parent, st));
  CU(A.d_rows_ptr.upload(S.rows_ptr, st));
  CU(A.d_rows.upload(S.rows, st));
  CU(A.d_rel.upload(S.rel, st));
  CU(A.d_child_ptr.upload(S.child_ptr, st));
  CU(A.d_child_idx.upload(S.child_idx, st));
  CU(A.d_uent_ptr.upload(S.uent_ptr, st));
  CU(A.d_u_dst.upload(S.u_dst, st));
  CU(A.d_u_dst64.upload(S.u_dst64, st));
  CU(A.d_L_off.upload(S.L_off, st));
  CU(A.d_cb_off.upload(S.cb_off, st));
  CU(A.d_useg_ptr.upload(S.useg_ptr, st));
  CU(A.d_useg_src.upload(S.useg_src, st));
  CU(A.d_u_row.upload(S.u_row, st));
  CU(A.d_u_col.upload(S.u_col, st));
  CU(A.d_perm.upload(S.perm, st));
  CU(A.d_irn.upload(sv->irn, st));
  CU(A.d_jcn.upload(sv->jcn, st));
  const int n = S.n;
  if (!sv->d_vals.p) CU(sv->d_vals.alloc(sv->nnz));
  CU(A.d_uval.alloc(S.nnz_u));
  CU(A.d_L.alloc(S.L_off[S.nsn]));
  CU(A.d_W.alloc(S.L_off[S.nsn]));
  CU(A.d_CB.alloc(std::max<int64_t>(S.cb_off[S.nsn], 1)));
  CU(A.d_dinv.alloc(n)); CU(A.d_doff.alloc(n)); CU(A.d_scale.alloc(n));
  CU(A.d_res.alloc(n));
  CU(A.d_ptype.alloc(n)); CU(A.d_lperm.alloc(n)); CU(A.d_bperm.alloc(n));
  CU(A.d_counters.alloc(CNT_N));
  CU(A.d_zlist.alloc(n)); CU(A.d_zflag.alloc(n));
  CU(A.d_colmax.alloc(n));
  CU(A.d_rmax.alloc(n));
  CU(cudaMemsetAsync(A.d_rmax.p, 0, n * sizeof(unsigned long long), st));
  CU(cudaMemsetAsync(A.d_L.p, 0, A.d_L.n * sizeof(double), st));

  DevSym& D = A.DS;
  D.n = n; D.nsn = S.nsn;
  D.sn_start = A.d_sn_start.p; D.sn_parent = A.d_sn_parent.p;
  D.rows_ptr = A.d_rows_ptr.p; D.rows = A.d_rows.p; D.rel = A.d_rel.p;
  D.child_ptr = A.d_child_ptr.p; D.child_idx = A.d_child_idx.p;
  D.uent_ptr = A.d_uent_ptr.p; D.u_dst = A.d_u_dst.p; D.u_dst64 = A.d_u_dst64.p;
  D.L_off = A.d_L_off.p; D.cb_off = A.d_cb_off.p;
  DevNum& N = A.DN;
  N.L = A.d_L.p; N.W = A.d_W.p; N.CB = A.d_CB.p; N.uval = A.d_uval.p;
  N.dinv = A.d_dinv.p; N.doff = A.d_doff.p; N.ptype = A.d_ptype.p;
  N.lperm = A.d_lperm.p; N.bperm = A.d_bperm.p; N.counters = A.d_counters.p; N.colmax = A.d_colmax.p;
  N.zlist = A.d_zlist.p;

  // inverse row maps of the children of the (factorisation-)big fronts, for the one-launch extend-add
  {
    std::vector<long long> eoff(S.nsn, -1);
    long long tot = 0;
    for (int c = 0; c < S.nsn; ++c) {
      const int p = S.sn_parent[c];
      if (p >= 0 && (S.f(p) > sv->opt.smem_front_max || p == A.sc_root)) { eoff[c] = tot; tot += S.f(p); }
    }
    std::vector<int> einv((size_t)std::max<long long>(tot, 1), -1);
    for (int c = 0; c < S.nsn; ++c) if (eoff[c] >= 0) {
      const long long ro = S.rows_ptr[c];
      const int rc = S.r(c);
      for (int j = 0; j < rc; ++j) einv[(size_t)(eoff[c] + S.rel[ro + j])] = j;
    }
    CU(A.d_einv_off.upload(eoff, st));
    CU(A.d_einv.upload(einv, st));
    D.einv_off = A.d_einv_off.p; D.einv = A.d_einv.p;
  }

  CU(cudaFuncSetAttribute(k_tc_schur, cudaFuncAttributeMaxDynamicSharedMemorySize, TC_SMEM_BYTES));
  CU(cudaFuncSetAttribute(k_big_panel, cudaFuncAttributeMaxDynamicSharedMemorySize, CHAIN_SMEM));
  CU(cudaFuncSetAttribute(k_front_warp2, cudaFuncAttributeMaxDynamicSharedMemorySize, 4 * S2_SMEM_PER_WARP));
  CU(cudaFuncSetAttribute(k_front_smem, cudaFuncAttributeMaxDynamicSharedMemorySize, 220 * 1024));
  CU(cudaStreamSynchronize(st));


  // ---- triangular solves: flags, scratch, explicit-inverse work lists, plan ------------------------------
  {
    std::vector<int> boff(S.nsn, 0);
    std::vector<long long> bigv_off(S.nsn, 0);
    long long bv = 0; int bo = 0;
    for (int s = 0; s < S.nsn; ++s) if (S.f(s) > DF_MIDMAX) {
      boff[s] = bo; bo += (S.f(s) + DF_BLK - 1) / DF_BLK;
      bigv_off[s] = bv; bv += S.f(s) + (S.f(s) & 1);
    }
    // explicit inverses of the big fronts' pivot blocks (k_linv_*): K64 x K64 doubles per big front
    {
      std::vector<long long>& linv_off = A.linv_off;
      linv_off.assign(S.nsn, -1);
      long long tot = 0;
      for (int s = 0; s < S.nsn; ++s) if (S.f(s) > DF_MIDMAX) {
        linv_off[s] = tot;
        const long long K64 = (long long)((S.k(s) + DF_BLK - 1) / DF_BLK) * DF_BLK;
        tot += K64 * K64;
      }
      if (A.sc_root >= 0) A.sc_linv_off = std::max(linv_off[A.sc_root], 0LL);
      CU(A.d_linv_off.upload(linv_off, st));
      CU(A.d_linv.alloc(std::max<long long>(tot, 1)));
      CU(cudaMemsetAsync(A.d_linv.p, 0, A.d_linv.n * sizeof(double), st));
    }
    CU(A.d_boff.upload(boff, st));
    CU(A.d_bigv_off.upload(bigv_off, st));
    {
      // partial solves: where a pivot position's value lives between the sweeps (k_piv_out / k_piv_in)
      std::vector<long long> piv_big(n, -1);
      for (int s = 0; s < S.nsn; ++s) if (S.f(s) > DF_MIDMAX)
        for (int t = 0; t < S.k(s); ++t) piv_big[S.sn_start[s] + t] = bigv_off[s] + t;
      CU(A.d_piv_big.upload(piv_big, st));
    }
    CU(cudaDeviceGetAttribute(&sv->num_sms, cudaDevAttrMultiProcessorCount, sv->dev));
    const MultiStride one{1, S.nsn, std::max(bo, 1), 0, n, (long long)std::max<size_t>(S.rows.size(), 1),
                          std::max<long long>(bv, 1), 0};
    CU(alloc_sweep_state(sv, A.sweep, one));
    int rc2 = build_solve_tables(sv, A, st);
    if (rc2 == B200LDLT_SUCCESS) rc2 = build_front_plan(sv, A, take_f, std::vector<char>(S.nsn, 1), A.fronts);
    if (rc2 != B200LDLT_SUCCESS) return rc2;
    // the L11^-1 work once more, split by tree level
    for (int l = 0; l < S.nlevels; ++l) {
      std::vector<char> tl(S.nsn, 0);
      bool any = false;
      for (int q = 0; q < S.nsn; ++q) if (take_f[q] && S.sn_level[q] == l && S.f(q) > kSolveMidMax) { tl[q] = 1; any = true; }
      A.fronts.linv_level.emplace_back(new LinvPlan());
      if (any) { rc2 = build_linv_plan(sv, A, tl, *A.fronts.linv_level.back(), st); if (rc2 != B200LDLT_SUCCESS) return rc2; }
    }
    if (sv->opt.verbose)
      fprintf(stderr, "[b200ldlt] solve: %d big-front blocks, top grid %d x %d thr (%d CTAs per SM)\n",
              bo, A.sweep.grid, DF_THREADS, A.sweep.grid / sv->num_sms);
    CU(cudaStreamSynchronize(st));
  }

  b200ldlt_info& I = sv->info;
  I.n = n; I.nnz_in = S.nnz_in; I.nnz_unique = S.nnz_u;
  I.nsupernodes = S.nsn; I.nlevels = S.nlevels; I.max_front = S.max_front; I.max_pivots = S.max_k;
  I.n_saddle = S.n_saddle; I.n_pairs = S.n_pairs;
  I.nnz_L = S.nnzL; I.nnz_L_true = S.nnzL_true;
  I.L_bytes = (int64_t)A.d_L.n * 8; I.cb_bytes = (int64_t)A.d_CB.n * 8;
  I.flops_panel = S.flops_panel; I.flops_schur = S.flops_schur;
  I.t_order_s = S.t_order; I.t_symbolic_s = S.t_symbolic;
  if (sv->opt.verbose)
    fprintf(stderr,
            "[b200ldlt] analyse: n=%d nnz=%lld uniq=%lld saddle=%d pairs=%d nsn=%d levels=%d maxfront=%d maxk=%d "
            "nnzL=%lld (true %lld) flops panel=%.3g schur=%.3g cb=%.1f MB  order %.2fs symbolic %.2fs\n",
            n, (long long)S.nnz_in, (long long)S.nnz_u, S.n_saddle, S.n_pairs, S.nsn, S.nlevels, S.max_front,
            S.max_k, (long long)S.nnzL, (long long)S.nnzL_true, S.flops_panel, S.flops_schur,
            S.cb_total * 8.0 / 1e6, S.t_order, S.t_symbolic);
  sv->an = std::move(an);
  return B200LDLT_SUCCESS;
}

static inline unsigned cdiv(long long a, long long b) { return (unsigned)((a + b - 1) / b); }

// kernel launch with the programmatic-stream-serialisation attribute (PDL): the kernel may become resident while its
// predecessor on the stream is still running; it synchronises itself with griddepcontrol.wait
template <class... KArgs, class... Args>
static cudaError_t launch_pdl(bool pdl, void (*kern)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st, Args... args) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid; cfg.blockDim = block; cfg.dynamicSmemBytes = smem; cfg.stream = st;
  cudaLaunchAttribute at[1];
  at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  at[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = at; cfg.numAttrs = pdl ? 1 : 0;
  return cudaLaunchKernelEx(&cfg, kern, KArgs(args)...);
}

// enqueue the numeric factorisation of the fronts of FP from the values in d_vals; prologue: first the summing of
// duplicates and the scaling
static int enqueue_factor(Solver* sv, const FrontPlan& FP, bool prologue) {
  Analysis& A = *sv->an;
  const SchurLists& SL = FP.schur;
  Symbolic& S = A.S;
  cudaStream_t st = sv->stream;
  DevSym& D = A.DS;
  DevNum& N = A.DN;
  N.u = sv->pivtol;
  N.tiny = sv->opt.tiny;
  const int n = S.n;
  const long long nu = S.nnz_u;
  const int* fl = FP.d_fl.p;
  const std::vector<LevelPlan>& plan = FP.levels;
  int& L = sv->launches;
  if (prologue) {
  L = 0;
  sv->ev_next = 0;
  CU(cudaMemsetAsync(A.d_counters.p, 0, CNT_N * sizeof(int), st));
  CU(cudaMemsetAsync(A.d_colmax.p, 0, (size_t)n * sizeof(double), st));
  k_sum_dups<<<cdiv(nu, 256), 256, 0, st>>>(nu, A.d_useg_ptr.p, A.d_useg_src.p, sv->d_vals.p, A.d_uval.p); ++L;
  k_fill<<<cdiv(n, 256), 256, 0, st>>>(n, A.d_scale.p, 1.0); ++L;
  for (int sw = 0; sw < sv->opt.scaling; ++sw) {
    k_rowmax<<<cdiv(nu, 256), 256, 0, st>>>(nu, A.d_u_row.p, A.d_u_col.p, A.d_uval.p, A.d_scale.p, A.d_rmax.p); ++L;
    k_scale_update<<<cdiv(n, 256), 256, 0, st>>>(n, A.d_scale.p, A.d_rmax.p); ++L;
  }
  if (sv->opt.scaling > 0) {
    k_apply_scale<<<cdiv(nu, 256), 256, 0, st>>>(nu, A.d_u_row.p, A.d_u_col.p, A.d_scale.p, A.d_uval.p); ++L;
  }
  }  // prologue
  // storage of all big fronts of this plan is cleared up front on the third stream (idle until the first L11 inverse),
  // level by level with one event per level: a level's big fronts wait for THEIR storage only, the leaf levels run next to it
  bool any_big = false;
  for (int l = 0; l < S.nlevels; ++l) any_big = any_big || plan[l].big_cnt > 0;
  std::vector<cudaEvent_t> ev_zero_lvl(S.nlevels, nullptr);
  if (any_big) {
    cudaStream_t sz = sv->dbg.one_stream ? st : sv->stream3;
    cudaEvent_t e0 = sv->next_event();
    CU(cudaEventRecord(e0, st));
    CU(cudaStreamWaitEvent(sz, e0, 0));
    for (int l = 0; l < S.nlevels; ++l) {
      const LevelPlan& P = plan[l];
      if (!P.big_cnt) continue;
      k_big_zero<<<dim3(std::min<unsigned>(cdiv(P.big_zero_max, 1024), 592), P.big_cnt), 256, 0, sz>>>(D, N, fl + P.big_off); ++L;
      // ... and the original entries scattered in (they do not depend on the children either)
      k_big_assemble<<<dim3(std::max(1u, std::min<unsigned>(cdiv(P.big_entmax, 256), 64)), P.big_cnt), 256, 0, sz>>>(D, N, fl + P.big_off); ++L;
      ev_zero_lvl[l] = sv->next_event();
      CU(cudaEventRecord(ev_zero_lvl[l], sz));
    }
  }
  bool linv_forked = false;
  for (int l = 0; l < S.nlevels; ++l) {
    const LevelPlan& P = plan[l];
    if (P.big_cnt) {
      const int* bl = fl + P.big_off;
      if (ev_zero_lvl[l]) CU(cudaStreamWaitEvent(st, ev_zero_lvl[l], 0));
      if (P.big_chmax > 0) {
        k_big_extend_all<<<dim3(cdiv(P.big_fmax, 8), P.big_cnt), 256, 0, st>>>(D, N, bl); ++L;
      }
    }
    unsigned used_side = 0;
    {
      // the front classes of a level are independent: issue them side by side (forked from / joined to the main stream)
      const bool fork = !sv->dbg.one_stream && (P.small.size() + (P.big_cnt ? 1 : 0)) > 1;
      cudaEvent_t e_lvl = nullptr;
      if (fork) { e_lvl = sv->next_event(); CU(cudaEventRecord(e_lvl, st)); }
      int slot = P.big_cnt ? 1 : 0;          // slot 0 = the main stream (busy with the big fronts' assembly if there are any)
      unsigned used = 0;
      for (const auto& bk : P.small) {
        cudaStream_t sq = st;
        if (fork && slot > 0) {
          const int q = (slot - 1) % 4;
          sq = sv->side[q];
          if (!(used & (1u << q))) { CU(cudaStreamWaitEvent(sq, e_lvl, 0)); used |= 1u << q; }
        }
        ++slot;
        if (fork && slot > 4) slot = 0;
        if (bk.kind == 2) {   // order 33..64, <= 32 pivots: one warp per front, two rows per lane
          k_front_warp2<<<cdiv(bk.cnt, 4), 128, bk.smem, sq>>>(D, N, fl + bk.off, bk.cnt); ++L;
        } else if (bk.fmax <= 32) {  // one warp per front (registers), 4 fronts per CTA
          k_front_warp<<<cdiv(bk.cnt, 4), 128, 4 * XS_SMEM_PER_WARP, sq>>>(D, N, fl + bk.off, bk.cnt); ++L;
        } else {
          k_front_smem<<<bk.cnt, bk.threads, bk.smem, sq>>>(D, N, fl + bk.off, bk.cnt); ++L;
        }
      }
      used_side = used;
      // (the side streams are joined at the END of the level: this level's big fronts do not depend on its small fronts,
      //  so the panel chain below runs next to them)
    }
    if (P.big_cnt) {
      const int* bl = fl + P.big_off;
      if (P.big_chmax <= 0) {   // (with children the extend-add kernel has recorded the column maxima of the first panels)
        k_big_colmax0<<<dim3(P.big_cnt, 8), 256, 0, st>>>(D, N, bl); ++L;
      }
      // Panel pipeline on two streams (both inside the captured graph):
      //   chain  (st): k_big_panel(p) = LDL^T of block p+1 (one CTA) + the panel rows below it, which apply the update of
      //                panel p-1 to their own columns first (left-looking by one panel).  Needs k_big_panel(p-1) (stream
      //                order) and k_big_update(p-2).
      //   bulk   (su): k_big_update(p) = rank-32 update of the columns from panel p+2 on.  Needs k_big_panel(p).
      // So the critical path is ONE launch per 32 pivots and the bulk update of a panel has a whole chain step of slack.
      cudaStream_t su = sv->dbg.one_stream ? st : sv->stream2;
      {
        cudaEvent_t e = sv->next_event();
        CU(cudaEventRecord(e, st));
        CU(cudaStreamWaitEvent(su, e, 0));
      }
      const int npan = (P.big_kmax + NB - 1) / NB;
      std::vector<cudaEvent_t> eUB(npan + 2, nullptr);
      // contribution blocks: one rank-32 update per panel, behind that panel's bulk update on the same stream (a second
      // dependent stream per panel measurably delays the launch of the next chain step).  Only when every front of the level
      // takes the DFMA route; with tensor-core Schur fronts in the level the complements are formed at the end of the level.
      const bool cb_panel = !sv->dbg.cb_at_end && !sv->dbg.one_stream && P.tc_t_cnt == 0 && P.df_cnt > 0;
      k_big_panel<<<dim3(1, P.big_cnt), 128, CHAIN_SMEM, st>>>(D, N, bl, -NB, 0); ++L;     // LDL^T of block 0
      for (int p = 0; p < npan; ++p) {
        const int jb = p * NB;
        if (p >= 2 && eUB[p - 2]) CU(cudaStreamWaitEvent(st, eUB[p - 2], 0));
        const int rows_below = P.big_fmax - jb;  // upper bound
        const int nrowblk = std::max(1u, cdiv(rows_below, 128));
        CU(launch_pdl(!sv->dbg.no_pdl, k_big_panel, dim3(1 + nrowblk + cdiv(jb, TRSM_SWAP_COLS), P.big_cnt), dim3(128), CHAIN_SMEM, st,
                      D, N, bl, jb, nrowblk)); ++L;
        const int rem_k = P.big_kmax - jb - 2 * NB;
        if (rem_k > 0 || cb_panel) {
          cudaEvent_t en = sv->next_event();
          CU(cudaEventRecord(en, st));
          CU(cudaStreamWaitEvent(su, en, 0));
        }
        if (rem_k > 0) {
          const unsigned tiles_i = cdiv(P.big_fmax - jb - 2 * NB, TM), tiles_j = cdiv(rem_k, TM);
          k_big_update<<<dim3(tiles_i, tiles_j, P.big_cnt), 256, 0, su>>>(D, N, bl, jb); ++L;
          eUB[p] = sv->next_event();
          CU(cudaEventRecord(eUB[p], su));
        }
        if (cb_panel) {
          k_big_update_cb<<<dim3(cdiv(P.df_rmax, TM), cdiv(P.df_rmax, TM), P.big_cnt), 256, 0, su>>>(D, N, bl, jb); ++L;
        }
      }
      {
        cudaEvent_t e = sv->next_event();
        CU(cudaEventRecord(e, su));
        CU(cudaStreamWaitEvent(st, e, 0));
      }
      if (!FP.linv_level.empty() && !sv->dbg.one_stream && FP.linv_level[l]->ndiag > 0) {
        // explicit L11 inverses of this level's fronts: behind the chain on their own stream, concurrent with the Schur
        // complements and the levels above (they only read the finished pivot blocks; k_linv_gemm<1> uses the top k x k
        // part of W as scratch, which nothing reads after the chain)
        cudaEvent_t e = sv->next_event();
        CU(cudaEventRecord(e, st));
        CU(cudaStreamWaitEvent(sv->stream3, e, 0));
        int rc = enqueue_linv(sv, *FP.linv_level[l], sv->stream3);
        if (rc != B200LDLT_SUCCESS) return rc;
        linv_forked = true;
      }
      // Schur complements CB -= L21 (L21 D)^T: tensor cores (Ozaki int8 digits, schur_tc.cu) for the large fronts,
      // register-blocked DFMA tiles for the rest
      if (P.tc_t_cnt > 0) {
        const TcFront* tf = SL.d_f.p + P.tc_f_off;
        k_tc_slice<<<dim3(cdiv(P.tc_rmax, 8), P.tc_f_cnt), 256, 0, st>>>(D, N, tf, 0, A.d_tc_dig.p, A.d_tc_exp.p); ++L;
        k_tc_slice<<<dim3(cdiv(P.tc_rmax, 8), P.tc_f_cnt), 256, 0, st>>>(D, N, tf, 1, A.d_tc_dig.p, A.d_tc_exp.p); ++L;
        k_tc_schur<<<P.tc_t_cnt, TC_THREADS, TC_SMEM_BYTES, st>>>(D, N, tf, SL.d_t.p + P.tc_t_off, A.d_tc_dig.p, A.d_tc_exp.p); ++L;
      }
      if (!cb_panel && P.df_cnt > 0) {
        k_big_schur84<<<dim3(cdiv(P.df_rmax, TM), cdiv(P.df_rmax, TM), P.df_cnt), 128, 0, st>>>(D, N, SL.d_dfl.p + P.df_off); ++L;
      }
    }
    for (int q = 0; q < 4; ++q) if (used_side & (1u << q)) {     // join the small-front streams of this level
      cudaEvent_t e = sv->next_event();
      CU(cudaEventRecord(e, sv->side[q]));
      CU(cudaStreamWaitEvent(st, e, 0));
    }
  }
  if (A.sc_root >= 0) {
    // Schur mode: the root front of S, once all of its children are done, through the big-front assembly (its panel
    // is m x m, r = 0); S_c out of the assembled panel, then the identity pivot block in its place
    const int m = (int)sv->sc_vars.size(), rt = A.sc_root;
    const long long mm = (long long)m * m;
    const int* rl = A.d_sc_root.p;
    k_big_zero<<<dim3(std::min<unsigned>(cdiv(mm, 1024), 592), 1), 256, 0, st>>>(D, N, rl); ++L;
    k_big_assemble<<<dim3(std::max(1u, std::min<unsigned>(cdiv(A.sc_nent, 256), 64)), 1), 256, 0, st>>>(D, N, rl); ++L;
    if (A.sc_nch > 0) { k_big_extend_all<<<dim3(cdiv(m, 8), 1), 256, 0, st>>>(D, N, rl); ++L; }
    double* P = A.d_L.p + S.L_off[rt];
    k_sc_out<<<cdiv(mm, 256), 256, 0, st>>>(m, P, A.d_sc_vars.p, A.d_scale.p, A.d_sc.p); ++L;
    const bool big = S.f(rt) > DF_MIDMAX;
    const long long k64 = big ? (long long)((m + DF_BLK - 1) / DF_BLK) * DF_BLK : 0;
    k_sc_identity<<<cdiv(std::max(mm, k64 * k64), 256), 256, 0, st>>>(m, n - m, k64, P, A.d_lperm.p, A.d_bperm.p,
        A.d_ptype.p, A.d_dinv.p, A.d_doff.p, big ? A.d_linv.p + A.sc_linv_off : nullptr); ++L;
  }
  if (linv_forked) {
    cudaEvent_t e = sv->next_event();
    CU(cudaEventRecord(e, sv->stream3));
    CU(cudaStreamWaitEvent(st, e, 0));
  } else {
    int rc = enqueue_linv(sv, FP.linv, st);
    if (rc != B200LDLT_SUCCESS) return rc;
  }
  CU(cudaGetLastError());
  return B200LDLT_SUCCESS;
}

// explicit inverses of the pivot blocks of the big fronts in LP (after their numeric factorisation): level 0 for all
// 64x64 diagonal blocks in one launch, then two tile-GEMM launches per doubling level (all fronts and pairs batched)
static int enqueue_linv(Solver* sv, const LinvPlan& LP, cudaStream_t st) {
  if (LP.ndiag <= 0) return B200LDLT_SUCCESS;
  Analysis& A = *sv->an;
  int& L = sv->launches;
  k_linv_diag<<<LP.ndiag, 64, 0, st>>>(A.DS, A.DN, LP.d_diag.p, A.d_linv_off.p, A.d_linv.p); ++L;
  for (size_t l = 0; l < LP.ng.size(); ++l) {
    if (LP.ng[l] <= 0) continue;
    k_linv_gemm<1><<<LP.ng[l], 128, 0, st>>>(A.DS, A.DN, LP.d_g[l]->p, A.d_linv_off.p, A.d_linv.p, A.d_linv_part.p, A.d_linv_cnt.p); ++L;
    k_linv_gemm<2><<<LP.ng2[l], 128, 0, st>>>(A.DS, A.DN, LP.d_g2[l]->p, A.d_linv_off.p, A.d_linv.p, A.d_linv_part.p, A.d_linv_cnt.p); ++L;
  }
  CU(cudaGetLastError());
  return B200LDLT_SUCCESS;
}

// keep mode: D^+ at the zero pivots zpos[0..nz) (dinv = 0; they are 1x1 pivots, doff is already 0) and their flags
__global__ void k_zero_pivots(int nz, const int* __restrict__ zpos, double* __restrict__ dinv, unsigned char* __restrict__ zflag) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < nz) { dinv[zpos[i]] = 0.0; zflag[zpos[i]] = 1; }
}

// The outcome of a factorisation whose stream has drained (ev1 recorded after its last launch), from its counters (CNT_N
// ints; on a sharded handle summed over the ranks): timing, launches and counts into info, the factors offered to the
// solves or not, keep mode's D^+, the inertia and the return code.
static int settle_factor(Solver* sv, const int* counters, int check_inertia, int expected_neg, int* num_neg) {
  Analysis& A = *sv->an;
  cudaStream_t st = sv->stream;
  float ms = 0;
  cudaEventElapsedTime(&ms, sv->ev0, sv->ev1);
  b200ldlt_info& I = sv->info;
  I.ms_factor_gpu = ms;
  I.launches_factor = sv->launches;
  I.num_neg = counters[CNT_NEG];
  I.num_forced = counters[CNT_FORCED];
  I.num_tiny = counters[CNT_TINY];
  I.num_growth = counters[CNT_GROWTH];
  I.num_2x2 = counters[CNT_2X2];
  // Factors of a matrix with a noise pivot (SINGULAR) are not offered to the solves, unless keep mode is on and every such
  // pivot is a zero pivot (its whole column noise): D_pp = 0 then describes the matrix, so dinv[p] is set to 0 (D^+) and
  // the pivot leaves the inertia.  A lifted zero (|pivot| <= tiny under a column that is not noise) never keeps factors.
  // With num_forced > 0 the factors (and the inertia reported) are those of a matrix perturbed by <= 1e-8 |column| in the
  // lifted pivots; the count is surfaced in b200ldlt_info and drives increase_quality (re-analysis with the current values).
  // A sharded handle reads no zero list: its own holds only this rank's entries, while CNT_ZLIST counts all ranks'.
  A.factored = (I.num_tiny == 0);
  A.zpos.clear();
  if (I.num_tiny > 0 && !A.shard.active) {
    const int nz = std::min(counters[CNT_ZLIST], sv->n);
    std::vector<int> zl(nz);
    CU(cudaMemcpy(zl.data(), A.d_zlist.p, nz * sizeof(int), cudaMemcpyDeviceToHost));
    std::sort(zl.begin(), zl.end());
    int lifted = -1, zneg = 0;
    for (int e : zl) {
      if ((e & 2) && lifted < 0) lifted = e >> 2;
      zneg += e & 1;
    }
    if (lifted >= 0) {
      sv->err = "factor: SINGULAR with a lifted zero pivot (|pivot| <= tiny at pivot position " + std::to_string(lifted) +
                ", whose column is not rounding noise): no factors kept";
    } else {
      const bool keep = sv->keep_singular && sv->sc_vars.empty();   // (Schur mode keeps no singular factors)
      sv->err = "factor: SINGULAR: " + std::to_string(nz) + " zero pivot(s)" +
                (keep ? "; factors kept with D^+ (zero pivots left out of the inertia)" : "; no factors kept");
      if (keep && nz == I.num_tiny) {
        for (int e : zl) A.zpos.push_back(e >> 2);
        CU(A.d_zpos.upload(A.zpos, st));
        CU(cudaMemsetAsync(A.d_zflag.p, 0, sv->n, st));
        k_zero_pivots<<<cdiv(nz, 256), 256, 0, st>>>(nz, A.d_zpos.p, A.d_dinv.p, A.d_zflag.p);
        CU(cudaGetLastError());
        CU(cudaStreamSynchronize(st));
        I.launches_factor += 1;
        I.num_neg -= zneg;
        A.factored = true;
      }
    }
  }
  sv->num_neg = I.num_neg;
  if (num_neg) *num_neg = I.num_neg;
  if (sv->opt.verbose > 1)
    fprintf(stderr, "[b200ldlt] factor: %.3f ms, %d launches, neg=%d 2x2=%d forced=%d tiny=%d growth=%d (u=%g)\n", ms,
            sv->launches, I.num_neg, I.num_2x2, I.num_forced, I.num_tiny, I.num_growth, sv->pivtol);
  if (I.num_tiny > 0) return B200LDLT_SINGULAR;
  if (check_inertia && I.num_neg != expected_neg) return B200LDLT_WRONG_INERTIA;
  return B200LDLT_SUCCESS;
}

static int do_factor(Solver* sv, const double* d_vals_ext, bool from_host, int check_inertia, int expected_neg,
                     int* num_neg) {
  if (num_neg) *num_neg = -1;
  if (sv->n <= 0) { sv->err = "factor before analyse"; return B200LDLT_FATAL_ERROR; }
  CU(cudaSetDevice(sv->dev));
  if (!sv->an || sv->reanalyse) {
    if (sv->an) ++sv->n_reanalysed;
    std::vector<double> hv;
    const double* vals = sv->h_vals;
    if (!from_host && d_vals_ext) {
      hv.resize(sv->nnz);
      CU(cudaMemcpy(hv.data(), d_vals_ext, sv->nnz * sizeof(double), cudaMemcpyDeviceToHost));
      vals = hv.data();
    }
    int rc = run_analysis(sv, vals);
    if (rc != B200LDLT_SUCCESS) return rc;
  }
  Analysis& A = *sv->an;
  cudaStream_t st = sv->stream;
  CU(cudaEventRecord(sv->ev0, st));
  if (from_host)
    CU(cudaMemcpyAsync(sv->d_vals.p, sv->h_vals, sv->nnz * sizeof(double), cudaMemcpyHostToDevice, st));
  else if (d_vals_ext && d_vals_ext != sv->d_vals.p)
    CU(cudaMemcpyAsync(sv->d_vals.p, d_vals_ext, sv->nnz * sizeof(double), cudaMemcpyDeviceToDevice, st));
  sv->have_dev_vals = true;
  if (!from_host) CU(cudaEventRecord(sv->ev0, st));  // device-resident timing excludes the staging copy
  int rc;
  if (sv->opt.use_graph == 1) {
    // the launch sequence is fixed by the symbolic structure: capture it once, replay it every factorisation
    if (!A.fgraph_exec || A.fgraph_u != sv->pivtol) {
      if (A.fgraph_exec) { cudaGraphExecDestroy(A.fgraph_exec); A.fgraph_exec = nullptr; }
      if (A.fgraph) { cudaGraphDestroy(A.fgraph); A.fgraph = nullptr; }
      CU(cudaStreamBeginCapture(st, cudaStreamCaptureModeThreadLocal));
      rc = enqueue_factor(sv, A.fronts, true);
      cudaError_t ce = cudaStreamEndCapture(st, &A.fgraph);
      if (rc != B200LDLT_SUCCESS) return rc;
      CU(ce);
      CU(cudaGraphInstantiate(&A.fgraph_exec, A.fgraph, 0));
      A.fgraph_u = sv->pivtol;
      A.fgraph_launches = sv->launches;
    }
    sv->launches = A.fgraph_launches;
    CU(cudaGraphLaunch(A.fgraph_exec, st));
  } else {
    rc = enqueue_factor(sv, A.fronts, true);
    if (rc != B200LDLT_SUCCESS) return rc;
  }
  CU(cudaEventRecord(sv->ev1, st));
  CU(cudaMemcpyAsync(sv->h_counters, A.d_counters.p, CNT_N * sizeof(int), cudaMemcpyDeviceToHost, st));
  CU(cudaStreamSynchronize(st));
  return settle_factor(sv, sv->h_counters, check_inertia, expected_neg, num_neg);
}

__global__ void k_mark_flags(int* flags, const int* __restrict__ list, int n, int value) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) flags[list[i]] = value;
}

// the DevSolve of a sweep: the handle's per-front tables, the plan's work lists, the state's arrays (column 0; the
// kernels find the other columns through MultiStride)
static DevSolve sweep_view(const Solver* sv, const SolvePlan& SP, const SweepState& W) {
  const Analysis& A = *sv->an;
  DevSolve V;
  V.tasks = SP.d_tf.p; V.tasks_bwd = SP.d_tb.p; V.ntasks_fwd = SP.ntf; V.ntasks_bwd = SP.ntb;
  V.bundle = SP.d_bundle.p;
  V.done_f = W.d_done_f.p; V.done_b = W.d_done_b.p;
  V.bflag_f = W.d_bflag_f.p; V.bflag_b = W.d_bflag_b.p; V.bcnt = W.d_bcnt.p; V.bcnt_b = W.d_bcnt_b.p;
  V.boff = A.d_boff.p; V.bigv_off = A.d_bigv_off.p; V.bigv = W.d_bigv.p; V.bigy = W.d_bigy.p;
  V.part = W.width > 1 ? W.d_part.p : SP.d_part.p; V.ccnt = W.width > 1 ? W.d_ccnt.p : SP.d_ccnt.p;
  V.ticket = W.d_ticket.p;
  V.linv = A.d_linv.p; V.linv_off = A.d_linv_off.p;
  V.fdesc = A.d_fdesc.p; V.gmap = A.d_gmap.p; V.gmap_off = A.d_gmap_off.p;
  V.subs = SP.d_subs.p; V.sub_meta = SP.d_sub_meta.p; V.subrow = SP.d_subrow.p; V.nsub = SP.nsub;
  V.subpair = SP.d_subpair.p; V.npair = SP.npair; V.sub_Loff = SP.d_sub_Loff.p;
  V.upper_max = sv->opt.smem_front_max;
  return V;
}

// subsequences of a plan's lists, in their order, on the device (the pruned sweeps): the top tasks of the sweep's
// direction (forward or backward list), the subtree items, the direct fronts of each level
struct PrunedLists {
  const SolveTask* tasks; int ntasks;
  const int2* subpair; int npair;
  const int* direct; std::vector<int> direct_off, direct_cnt;   // direct level l: direct_cnt[l] fronts at direct + direct_off[l]
};

// one sweep of nb columns (nb <= W.width) over the fronts of a plan: the bottom levels one launch each, and ONE persistent
// kernel (forward: bottom levels, then subtrees, then top tasks; backward: the reverse).  apply_d = false: a forward
// sweep that leaves D^-1 out (partial solves).  pruned: the sweep takes those lists instead of SP's
static int launch_sweep(Solver* sv, const SolvePlan& SP, SweepState& W, int nb, bool fwd, bool apply_d = true,
                        const PrunedLists* pruned = nullptr) {
  Analysis& A = *sv->an;
  cudaStream_t st = sv->stream;
  DevSolve V = sweep_view(sv, SP, W);
  if (pruned) {
    if (fwd) { V.tasks = pruned->tasks; V.ntasks_fwd = pruned->ntasks; }
    else { V.tasks_bwd = pruned->tasks; V.ntasks_bwd = pruned->ntasks; }
    V.subpair = pruned->subpair; V.npair = pruned->npair;
  }
  MultiStride M = W.M;
  M.nb = nb;
  const bool multi = nb > 1;
  const long long nt = ((long long)(fwd ? V.ntasks_fwd : V.ntasks_bwd) + V.npair) * nb;
  const int grid = (int)std::min<long long>(W.grid, nt);
  const int nd = (int)SP.direct_cnt.size();
  const auto k_direct = (fwd && !apply_d) ? (multi ? k_solve_direct<true, true, false> : k_solve_direct<true, false, false>)
                        : fwd ? (multi ? k_solve_direct<true, true> : k_solve_direct<true, false>)
                              : (multi ? k_solve_direct<false, true> : k_solve_direct<false, false>);
  const auto k_sweep = sweep_kernel(fwd, multi, apply_d);
  auto direct = [&](int l) {
    const int cnt = pruned ? pruned->direct_cnt[l] : SP.direct_cnt[l];
    if (cnt <= 0) return;
    const int* lst = pruned ? pruned->direct + pruned->direct_off[l] : SP.d_direct[l]->p;
    const unsigned g = cdiv(cnt * nb, DF_THREADS / 32);
    k_direct<<<g, DF_THREADS, 0, st>>>(A.DS, A.DN, V, M, lst, cnt, A.solve_epoch, W.d_x.p, W.d_cbv.p);
    ++sv->launches;
  };
  if (fwd) for (int l = 0; l < nd; ++l) direct(l);
  if (nt > 0) {
    unsigned long long& ticket = fwd ? W.ticket_f : W.ticket_b;
    k_sweep<<<grid, DF_THREADS, DF_DYN_SMEM, st>>>(A.DS, A.DN, V, M, A.solve_epoch, ticket, W.d_x.p, W.d_cbv.p);
    ticket += (unsigned long long)nt + grid;
    ++sv->launches;
  }
  if (!fwd) for (int l = nd - 1; l >= 0; --l) direct(l);
  CU(cudaGetLastError());
  return B200LDLT_SUCCESS;
}

// The two stages every solve over the fronts of SP is built from, for nb <= W.width columns of leading dimension n.  Each
// sweep waits on flags that its own fronts stamp with A.solve_epoch, so each stage takes a new epoch: a flag left by
// an earlier sweep never matches it.  (Backward work waits only on backward flags, so a backward stage may follow a
// forward one under a new epoch.)
// forward: x = P^T S d_in, then the forward sweep; apply_d = false leaves D^-1 out (L only)
static int forward(Solver* sv, const SolvePlan& SP, SweepState& W, const double* d_in, int nb, bool apply_d = true) {
  Analysis& A = *sv->an;
  const int n = sv->n;
  k_rhs_in<<<dim3(cdiv(n, 256), nb), 256, 0, sv->stream>>>(n, A.d_perm.p, A.d_scale.p, d_in, W.d_x.p, W.M.x);
  ++sv->launches;
  A.solve_epoch++;
  return launch_sweep(sv, SP, W, nb, true, apply_d);
}

// backward: the backward sweep, then d_out = S P x unless d_out is null
static int backward(Solver* sv, const SolvePlan& SP, SweepState& W, double* d_out, int nb) {
  Analysis& A = *sv->an;
  A.solve_epoch++;
  const int rc = launch_sweep(sv, SP, W, nb, false);
  if (rc != B200LDLT_SUCCESS || !d_out) return rc;
  const int n = sv->n;
  k_sol_out<<<dim3(cdiv(n, 256), nb), 256, 0, sv->stream>>>(n, A.d_perm.p, A.d_scale.p, W.d_x.p, W.M.x, d_out);
  ++sv->launches;
  CU(cudaGetLastError());
  return B200LDLT_SUCCESS;
}

// columns [0, nrhs) in blocks of at most cap columns: block(c, w) for each, in order
template <class Block>
static int for_blocks(int nrhs, int cap, Block&& block) {
  for (int c = 0; c < nrhs;) {
    const int w = std::min(cap, nrhs - c);
    const int rc = block(c, w);
    if (rc != B200LDLT_SUCCESS) return rc;
    c += w;
  }
  return B200LDLT_SUCCESS;
}

// The solve (job 0) or one part of it (job 1..4, include/b200ldlt.h) for nb columns of d_in -> d_out (leading dimension
// n, in place when they are the same), nb <= W.width.  Job 0 is forward then backward over all fronts; job 1 is its
// forward stage leaving D^-1 out, copied out in pivot order; job 3 its backward stage, fed in pivot order; job 2 (and
// the front of job 4) applies D^-1 through the helper the fused sweep uses.  So job 3 . 2 . 1 and job 4 . 1 reproduce
// job 0 bit for bit.  Launches: job 0: 2 + two sweeps; job 1, 3, 4: 2 + one sweep (the direct levels + 1); job 2: 1.
static int enqueue_solve(Solver* sv, SweepState& W, int job, const double* d_in, double* d_out, int nb) {
  Analysis& A = *sv->an;
  const SolvePlan& SP = A.fronts.solve;
  cudaStream_t st = sv->stream;
  const int n = sv->n;
  const dim3 g(cdiv(n, 256), nb);
  const long long ldx = W.M.x, ldb = W.M.bigv;
  if (job == 0) {
    const int rc = forward(sv, SP, W, d_in, nb);
    return rc != B200LDLT_SUCCESS ? rc : backward(sv, SP, W, d_out, nb);
  }
  if (job == 1) {
    const int rc = forward(sv, SP, W, d_in, nb, false);
    if (rc != B200LDLT_SUCCESS) return rc;
    k_piv_out<<<g, 256, 0, st>>>(n, A.d_piv_big.p, W.d_x.p, ldx, W.d_bigv.p, ldb, d_out); ++sv->launches;
  } else if (job == 2) {
    // (through the sweep state's x: d_in and d_out may be the same array, and k_dinv reads partners from its input)
    k_dinv<<<g, 256, 0, st>>>(n, A.d_ptype.p, A.d_dinv.p, A.d_doff.p, d_in, nullptr, W.d_x.p, n, nullptr, 0); ++sv->launches;
    CU(cudaMemcpyAsync(d_out, W.d_x.p, (size_t)n * nb * sizeof(double), cudaMemcpyDeviceToDevice, st));
  } else {
    if (job == 3) k_piv_in<<<g, 256, 0, st>>>(n, A.d_piv_big.p, d_in, W.d_x.p, ldx, W.d_bigv.p, ldb);
    else k_dinv<<<g, 256, 0, st>>>(n, A.d_ptype.p, A.d_dinv.p, A.d_doff.p, d_in, A.d_piv_big.p, W.d_x.p, ldx, W.d_bigv.p, ldb);
    ++sv->launches;
    return backward(sv, SP, W, d_out, nb);
  }
  CU(cudaGetLastError());
  return B200LDLT_SUCCESS;
}

// The sweep state of the blocked solve, B200_SOLVE_BLOCK columns wide: allocated once per analysis, at the first nrhs > 1
// solve, before that solve's timing starts.  Returns false (and the columns are then solved one by one, as with
// B200_SOLVE_BLOCK=1) when the device memory for it cannot be had.
static bool block_solve_state(Solver* sv) {
  Analysis& A = *sv->an;
  if (A.blk) return A.blk->width > 1;
  const int nb = sv->dbg.solve_block;
  A.blk.reset(new SweepState());   // width 0: not retried before the next analysis
  if (nb < 2) return false;
  SweepState& B = *A.blk;
  MultiStride M = A.sweep.M;
  M.nb = nb;
  M.nccnt = (int)A.fronts.solve.d_ccnt.n;
  M.part = (long long)A.fronts.solve.d_part.n;
  const cudaError_t e = alloc_sweep_state(sv, B, M);
  if (e != cudaSuccess) {
    if (sv->opt.verbose) fprintf(stderr, "[b200ldlt] blocked solve unavailable (%s): one solve per column\n", cudaGetErrorString(e));
    cudaGetLastError();
    A.blk.reset(new SweepState());
    return false;
  }
  if (sv->opt.verbose)
    fprintf(stderr, "[b200ldlt] blocked solve: %d columns, %.1f MB of per-column state, grid %d\n", nb,
            (double)(8 * (B.d_x.n + B.d_cbv.n + B.d_bigv.n + B.d_bigy.n + B.d_part.n) +
                     4 * (B.d_done_f.n + B.d_done_b.n + B.d_bcnt.n + B.d_bcnt_b.n + B.d_bflag_f.n + B.d_bflag_b.n + B.d_ccnt.n)) / 1e6,
            B.grid);
  return true;
}

// nrhs columns of d_rhs (leading dimension n), in place: blocks of up to B200_SOLVE_BLOCK columns through the blocked
// state, single columns through the one-column state.  `blocked`: the result of block_solve_state, called by the entry
// point before its timing starts.  job: as in enqueue_solve.
static int enqueue_solve_columns(Solver* sv, double* d_rhs, int nrhs, bool blocked, int job = 0) {
  Analysis& A = *sv->an;
  return for_blocks(nrhs, blocked ? A.blk->width : 1, [&](int c, int w) {
    double* col = d_rhs + (size_t)c * sv->n;
    return enqueue_solve(sv, w == 1 ? A.sweep : *A.blk, job, col, col, w);
  });
}

// The Fredholm alternative (b200ldlt_solve_fredholm) with zero pivots Z: columns [0, nrhs) of d_x (leading dimension n)
// hold the b's; on exit column i holds x_i = S P L^-T D^+ y_i and column nrhs + i holds f_i = S P L^-T z_i, where
// y_i = L^-1 P^T S b_i and z_i is y_i on Z.  sv->d_fred_nrm receives max |y_i| and max_Z |y_i| per column.  x_i runs
// job 1, then job 4 with D^+ (= job 0 with D^+, bit for bit); f_i runs job 3 on z_i.
//   blocked (a state of width >= 2): blocks of w <= width / 2 columns, x and f through ONE backward sweep of 2w columns:
//     k_rhs_in, forward sweep without D, k_fred, backward sweep, k_fred_out -- 5 + 2 D launches per block;
//   otherwise column by column in the single-column state, z parked in A.d_fred_z, two backward sweeps: k_rhs_in,
//     forward, k_fred, backward, k_sol_out, k_piv_in, backward, k_sol_out -- 8 + 3 D launches per column.
// Every column runs the arithmetic of a single-column call.
static int enqueue_fredholm(Solver* sv, double* d_x, int nrhs, bool blocked) {
  Analysis& A = *sv->an;
  cudaStream_t st = sv->stream;
  const int n = sv->n;
  CU(cudaMemsetAsync(sv->d_fred_nrm.p, 0, 2 * (size_t)nrhs * sizeof(unsigned long long), st));
  const SolvePlan& SP = A.fronts.solve;
  SweepState& W = blocked ? *A.blk : A.sweep;
  const long long ldx = W.M.x, ldb = W.M.bigv;
  const int rc = for_blocks(nrhs, blocked ? W.width / 2 : 1, [&](int c, int w) -> int {
    double* col = d_x + (size_t)c * n;
    const dim3 g(cdiv(n, 256), w);
    int rc2 = forward(sv, SP, W, col, w, false);
    if (rc2 != B200LDLT_SUCCESS) return rc2;
    k_fred<<<g, 256, 0, st>>>(n, A.d_ptype.p, A.d_dinv.p, A.d_doff.p, A.d_zflag.p, A.d_piv_big.p, W.d_x.p, ldx,
                              W.d_bigv.p, ldb, w, blocked ? nullptr : A.d_fred_z.p, sv->d_fred_nrm.p + 2 * (size_t)c);
    ++sv->launches;
    if (blocked) {
      rc2 = backward(sv, SP, W, nullptr, 2 * w);
      if (rc2 != B200LDLT_SUCCESS) return rc2;
      k_fred_out<<<dim3(cdiv(n, 256), 2 * w), 256, 0, st>>>(n, A.d_perm.p, A.d_scale.p, W.d_x.p, ldx, col, w, nrhs);
      ++sv->launches;
      return B200LDLT_SUCCESS;
    }
    rc2 = backward(sv, SP, W, col, 1);
    if (rc2 != B200LDLT_SUCCESS) return rc2;
    k_piv_in<<<g, 256, 0, st>>>(n, A.d_piv_big.p, A.d_fred_z.p, W.d_x.p, ldx, W.d_bigv.p, ldb); ++sv->launches;
    return backward(sv, SP, W, d_x + (size_t)(nrhs + c) * n, 1);
  });
  if (rc != B200LDLT_SUCCESS) return rc;
  CU(cudaGetLastError());
  return B200LDLT_SUCCESS;
}

// The work lists and the slot map of the multiply (lmul_kernels.cu).  The pivot columns of a front are cut into chunks
// of LM_CH; chunk [t0, ..) of front s owns f - t0 slots, one per panel row from t0 on.  Pivot position p (panel row
// i = p - c0 of its front) sums its own front's chunks with t0 <= i (own, by p) and, as permuted column q, the
// contribution rows equal to q of its descendants (desc, by q: fronts ascending, then chunks).  All of it depends on the
// analysis only.
static int build_lmul_plan(Solver* sv, LmulPlan& M) {
  const Symbolic& S = sv->an->S;
  const int n = sv->n;
  cudaStream_t st = sv->stream;
  std::vector<LmulItem> itn;
  std::vector<int2> itt;
  std::vector<int> pcol0(n), own_ptr(n + 1, 0), desc_ptr(n + 1, 0);
  std::vector<long long> cbase;
  long long ns = 0;
  for (int s = 0; s < S.nsn; ++s) {
    const int c0 = S.sn_start[s], k = S.sn_start[s + 1] - c0, r = (int)(S.rows_ptr[s + 1] - S.rows_ptr[s]), f = k + r;
    for (int i = 0; i < k; ++i) { pcol0[c0 + i] = c0; own_ptr[c0 + i + 1] = i / LM_CH + 1; }
    for (int t0 = 0; t0 < k; t0 += LM_CH) {
      cbase.push_back(ns);
      for (int g = 0; 32 * g < f - t0; ++g) itn.push_back(LmulItem{s, t0, g, 0, ns});
      for (int j = 0; j < r; ++j) desc_ptr[S.rows[S.rows_ptr[s] + j] + 1]++;
      ns += f - t0;
    }
    for (int t0 = 0; t0 < k; t0 += LM_CW) itt.push_back(make_int2(s, t0));
  }
  if (ns >= (1ll << 31)) { sv->err = "lmultiply: the factors are too large for the slot map"; return B200LDLT_FATAL_ERROR; }
  for (int p = 0; p < n; ++p) { own_ptr[p + 1] += own_ptr[p]; desc_ptr[p + 1] += desc_ptr[p]; }
  std::vector<int> own(own_ptr[n]), desc(std::max(desc_ptr[n], 1)), fill(desc_ptr.begin(), desc_ptr.end() - 1);
  size_t ci = 0;
  for (int s = 0; s < S.nsn; ++s) {
    const int c0 = S.sn_start[s], k = S.sn_start[s + 1] - c0, r = (int)(S.rows_ptr[s + 1] - S.rows_ptr[s]);
    for (int t0 = 0; t0 < k; t0 += LM_CH, ++ci) {
      const long long b = cbase[ci];
      for (int i = t0; i < k; ++i) own[own_ptr[c0 + i] + t0 / LM_CH] = (int)(b + i - t0);
      for (int j = 0; j < r; ++j) desc[fill[S.rows[S.rows_ptr[s] + j]]++] = (int)(b + k + j - t0);
    }
  }
  CU(M.d_items_n.upload(itn, st));
  CU(M.d_items_t.upload(itt, st));
  CU(M.d_pcol0.upload(pcol0, st));
  CU(M.d_own_ptr.upload(own_ptr, st));
  CU(M.d_own.upload(own, st));
  CU(M.d_desc_ptr.upload(desc_ptr, st));
  CU(M.d_desc.upload(desc, st));
  M.ld = std::max<long long>(ns, n);
  if (sv->opt.verbose)
    fprintf(stderr, "[b200ldlt] lmultiply map: %zu + %zu warp items, %lld slots (%.1f MB per column)\n", itn.size(),
            itt.size(), ns, 8e-6 * (double)M.ld);
  return B200LDLT_SUCCESS;
}

// the multiply's state for calls of nrhs columns (before the call's timing starts): the map at the first call after an
// analysis, the scratch for the widest block the call uses
static int lmul_state(Solver* sv, int nrhs) {
  Analysis& A = *sv->an;
  if (!A.lmul) {
    std::unique_ptr<LmulPlan> M(new LmulPlan());
    const int rc = build_lmul_plan(sv, *M);
    if (rc != B200LDLT_SUCCESS) return rc;
    A.lmul = std::move(M);
  }
  LmulPlan& M = *A.lmul;
  const int w = std::min(nrhs, sv->dbg.solve_block);
  if (w > M.width) {
    M.width = 0;
    CU(M.d_scr.alloc((size_t)M.ld * w));
    M.width = w;
  }
  return B200LDLT_SUCCESS;
}

// nb <= MS_NB_MAX columns (leading dimension n) of d_x -> d_y: two launches
static int enqueue_lmul(Solver* sv, int trans, const double* d_x, double* d_y, int nb) {
  using KN = void (*)(const FrontDesc*, const double*, const LmulItem*, int, const double*, int, double*, long long);
  using KT = void (*)(const FrontDesc*, const double*, const int2*, int, const int*, const int*, const double*, int, double*);
  static_assert(MS_NB_MAX == 8, "one instantiation per block width");
  static const KN kn[8] = {k_lmul_n<1>, k_lmul_n<2>, k_lmul_n<3>, k_lmul_n<4>, k_lmul_n<5>, k_lmul_n<6>, k_lmul_n<7>, k_lmul_n<8>};
  static const KT kt[8] = {k_lmul_t<1>, k_lmul_t<2>, k_lmul_t<3>, k_lmul_t<4>, k_lmul_t<5>, k_lmul_t<6>, k_lmul_t<7>, k_lmul_t<8>};
  const Analysis& A = *sv->an;
  const LmulPlan& M = *A.lmul;
  cudaStream_t st = sv->stream;
  const int n = sv->n;
  const dim3 g(cdiv(n, 256), nb);
  if (trans == 0) {
    const int ni = (int)M.d_items_n.n;
    kn[nb - 1]<<<cdiv(ni, 8), 256, 0, st>>>(A.d_fdesc.p, A.d_L.p, M.d_items_n.p, ni, d_x, n, M.d_scr.p, M.ld);
    k_lmul_gather<<<g, 256, 0, st>>>(n, M.d_pcol0.p, A.d_lperm.p, M.d_own_ptr.p, M.d_own.p, M.d_desc_ptr.p, M.d_desc.p,
                                     A.d_perm.p, A.d_scale.p, M.d_scr.p, M.ld, d_y);
  } else {
    const int ni = (int)M.d_items_t.n;
    k_lmul_in<<<g, 256, 0, st>>>(n, A.d_perm.p, A.d_scale.p, d_x, M.d_scr.p);
    kt[nb - 1]<<<cdiv(ni, 8), 256, 0, st>>>(A.d_fdesc.p, A.d_L.p, M.d_items_t.p, ni, A.d_lperm.p, A.d_rows.p,
                                            M.d_scr.p, n, d_y);
  }
  sv->launches += 2;
  CU(cudaGetLastError());
  return B200LDLT_SUCCESS;
}

// nrhs columns in blocks of up to B200_SOLVE_BLOCK (lmul_state called before)
static int enqueue_lmul_columns(Solver* sv, int trans, int nrhs, const double* d_x, double* d_y) {
  return for_blocks(nrhs, sv->an->lmul->width, [&](int c, int w) {
    return enqueue_lmul(sv, trans, d_x + (size_t)c * sv->n, d_y + (size_t)c * sv->n, w);
  });
}

// ---- pruned sweeps (b200ldlt_sparse_fwd_solve, b200ldlt_inverse_entries, b200ldlt_sparse_solve) ----------------------
// the top tasks T[0..nt) by front (CSR, ascending): a bundle's entry under each of its fronts
static void index_tasks(const SolvePlan& SP, const std::vector<SolveTask>& T, int nt, int nsn, PrunedPlan::Dir& D) {
  std::vector<int>& ptr = D.task_ptr;
  ptr.assign(nsn + 1, 0);
  auto each_front = [&](const SolveTask& K, auto&& fn) {
    if (K.type == ST_SMALL) { for (int w = 0; w < K.blk; ++w) fn(SP.bundle[K.s + w]); }
    else fn(K.s);
  };
  for (int j = 0; j < nt; ++j) each_front(T[j], [&](int s) { ptr[s + 1]++; });
  for (int s = 0; s < nsn; ++s) ptr[s + 1] += ptr[s];
  D.task_idx.resize(ptr[nsn]);
  std::vector<int> fill(ptr.begin(), ptr.end() - 1);
  for (int j = 0; j < nt; ++j) each_front(T[j], [&](int s) { D.task_idx[fill[s]++] = j; });
  D.m_task.assign(std::max(nt, 1), 0);
}

// PrunedPlan at the first pruned call after an analysis, before its timing starts: the per-front indices into the host
// copies of the handle's lists, the marks, and the staging's event.  Fronts are numbered in postorder (a parent after
// its children), so one pass from the last front down gives every front's depth and path length.
static int pruned_state(Solver* sv, const char* call) {
  Analysis& A = *sv->an;
  if (A.pruned) return B200LDLT_SUCCESS;
  const Symbolic& S = A.S;
  const SolvePlan& SP = A.fronts.solve;
  const int nsn = S.nsn, n = sv->n;
  std::unique_ptr<PrunedPlan> Q(new PrunedPlan());
  PrunedPlan& P = *Q;
  P.depth.assign(nsn, 0); P.pathlen.assign(nsn, 0);
  for (int s = nsn - 1; s >= 0; --s) {
    const int p = S.sn_parent[s];
    if (p >= 0 && p <= s) { sv->err = std::string(call) + ": internal: the fronts are not in postorder"; return B200LDLT_FATAL_ERROR; }
    P.depth[s] = p >= 0 ? P.depth[p] + 1 : 0;
    P.pathlen[s] = S.k(s) + (p >= 0 ? P.pathlen[p] : 0);
  }
  P.dlev.assign(nsn, -1); P.didx.assign(nsn, -1); P.item_of.assign(nsn, -1); P.sub_of.assign(nsn, -1);
  for (size_t l = 0; l < SP.direct_cnt.size(); ++l)
    for (int i = 0; i < SP.direct_cnt[l]; ++i) { const int s = SP.direct[l][i]; P.dlev[s] = (int)l; P.didx[s] = i; }
  P.item_ptr.assign(1, 0);
  for (int i = 0; i < SP.npair; ++i) {
    for (const int u : {SP.pairs[i].x, SP.pairs[i].y}) {
      if (u < 0) continue;
      const SubDesc& d = SP.subs[u];
      for (int j = 0; j < d.nown; ++j) {
        const int s = SP.meta[d.moff + 2 * d.nlv + 1 + j];
        P.item_fr.push_back(s); P.item_of[s] = i; P.sub_of[s] = u;
      }
    }
    P.item_ptr.push_back((int)P.item_fr.size());
  }
  index_tasks(SP, SP.tf, SP.ntf, nsn, P.dir[0]);
  index_tasks(SP, SP.tb, SP.ntb, nsn, P.dir[1]);
  P.iperm.resize(n); P.sn_of.resize(n);
  for (int i = 0; i < n; ++i) P.iperm[S.perm[i]] = i;
  for (int s = 0; s < nsn; ++s) for (int p = S.sn_start[s]; p < S.sn_start[s + 1]; ++p) P.sn_of[p] = s;
  P.pos_bi.assign(n, -1);
  P.col_of.assign(n, -1);
  P.m_reach.assign(nsn, 0); P.m_run.assign(nsn, 0); P.m_fr.assign(nsn, 0);
  P.m_item.assign(std::max(SP.npair, 1), 0);
  P.ord0.assign(nsn, 0); P.ord1.assign(nsn, 0);
  CU(cudaEventCreateWithFlags(&P.stg.ev, cudaEventDisableTiming));
  A.pruned = std::move(Q);
  return B200LDLT_SUCCESS;
}

// The staging grown to `bytes` for this call, after the previous call's copy out of h is complete (h is rewritten next).
// FATAL_ERROR with "<call>: ..." when the copy failed or the allocation fails (which leaves both buffers released).
int ListStaging::reserve(Solver* sv, const char* call, size_t bytes) {
  if (cudaEventSynchronize(ev) != cudaSuccess) {
    sv->err = std::string(call) + ": staging copy failed";
    return B200LDLT_FATAL_ERROR;
  }
  if (bytes <= d.n) return B200LDLT_SUCCESS;
  d.release();
  if (h) cudaFreeHost(h);
  h = nullptr;
  if (d.alloc(bytes) != cudaSuccess || cudaHostAlloc((void**)&h, bytes, cudaHostAllocDefault) != cudaSuccess) {
    cudaGetLastError();
    d.release();
    h = nullptr;
    sv->err = std::string(call) + ": cannot allocate the staging of " + std::to_string(bytes) + " bytes";
    return B200LDLT_FATAL_ERROR;
  }
  return B200LDLT_SUCCESS;
}

// the first `bytes` of h to d on the handle's stream, and ev recorded after the copy
int ListStaging::upload(Solver* sv, size_t bytes) {
  CU(cudaMemcpyAsync(d.p, h, bytes, cudaMemcpyHostToDevice, sv->stream));
  CU(cudaEventRecord(ev, sv->stream));
  return B200LDLT_SUCCESS;
}

static inline size_t align8(size_t b) { return (b + 7) & ~(size_t)7; }

// the pivot positions of the fronts
static int npos(const Symbolic& S, const std::vector<int>& fronts) {
  int c = 0;
  for (int s : fronts) c += S.sn_start[s + 1] - S.sn_start[s];
  return c;
}

// one pruned sweep as the host prepares it: the reach (ascending), the run set (the reach first), the subtree items and
// top tasks it runs (ascending), per direct level the indices of its direct fronts (ascending), the frontier
struct PrunedSweep {
  std::vector<int> reach, run, items, tasks, fr;
  std::vector<std::vector<int>> dl;
};

// The run set of a pruned sweep, with stamp m: R's reach, run set, subtree items, top tasks and direct fronts (R.fr
// cleared).  T is the sweep's top-task list, D its entries by front and marks.
static void collect_run_set(PrunedPlan& P, const SolvePlan& SP, const Symbolic& S, const std::vector<SolveTask>& T,
                            PrunedPlan::Dir& D, unsigned m, const int* seed, int nseed, PrunedSweep& R) {
  const int nd = (int)SP.direct_cnt.size();
  std::vector<int>& reach = R.reach;
  std::vector<int>& run = R.run;
  std::vector<int>& items = R.items;
  std::vector<int>& tasks = R.tasks;
  reach.clear(); items.clear(); tasks.clear(); R.fr.clear();
  for (int i = 0; i < nseed; ++i)
    for (int s = P.sn_of[seed[i]]; s >= 0 && P.m_reach[s] != m; s = S.sn_parent[s]) { P.m_reach[s] = m; reach.push_back(s); }
  std::sort(reach.begin(), reach.end());
  run = reach;
  for (int s : reach) P.m_run[s] = m;
  auto add = [&](int s) { if (P.m_run[s] != m) { P.m_run[s] = m; run.push_back(s); } };
  for (size_t q = 0; q < run.size(); ++q) {
    const int s = run[q], it = P.item_of[s];
    if (it >= 0 && P.m_item[it] != m) {
      P.m_item[it] = m; items.push_back(it);
      for (int e = P.item_ptr[it]; e < P.item_ptr[it + 1]; ++e) add(P.item_fr[e]);
    }
    for (int e = D.task_ptr[s]; e < D.task_ptr[s + 1]; ++e) {
      const int t = D.task_idx[e];
      if (D.m_task[t] == m) continue;
      D.m_task[t] = m; tasks.push_back(t);
      if (T[t].type == ST_SMALL) for (int w = 0; w < T[t].blk; ++w) add(SP.bundle[T[t].s + w]);
    }
  }
  std::sort(items.begin(), items.end());
  std::sort(tasks.begin(), tasks.end());
  std::vector<std::vector<int>>& dl = R.dl;
  dl.assign(nd, std::vector<int>());
  for (int s : run) if (P.dlev[s] >= 0) dl[P.dlev[s]].push_back(P.didx[s]);
  for (auto& v : dl) std::sort(v.begin(), v.end());
}

// Host part of a pruned sweep (dir 0: forward over SolvePlan::tf, dir 1: backward over SolvePlan::tb) from the pivot
// positions seed[0..nseed).  The reach (the fronts on the tree paths from the fronts of the seeds to the root) gives the
// run set R: the reach, the fronts walked by a subtree item that walks a reached front, and the fronts of a bundle of
// the direction's list that holds one (items and bundles are kept whole).  The pruned lists take every entry of the
// handle's lists that belongs to a front of R, in list order.  The frontier R.fr: forward, the children of R outside R;
// backward, the parents of R outside R (only item-mates and bundle-mates have one: their backward flags are stamped, so
// those mates read stale x at ancestor positions; their outputs are never returned and nothing in the reach reads them).
// Then the check that the pruned sweep cannot wait forever, before anything is launched: every front of R owns all of
// its top tasks in the lists, each chunked block with all of its chunks, and a big front all of its blocks of both types
// (FP and FC forward, BT and BX backward; the arrival and chunk counters count modulo); and every child (forward) or the
// parent (backward) of a front of R is in the frontier or runs EARLIER in the pruned order -- forward: the direct levels
// from the bottom up, subtree items, top tasks; backward: the reverse (the same subtree walk counts: it is walked level
// by level, from its root down backward).  FATAL_ERROR with "<call>: ..." when the check fails.
static int prune(Solver* sv, const char* call, int dir, const int* seed, int nseed, PrunedSweep& R) {
  Analysis& A = *sv->an;
  PrunedPlan& P = *A.pruned;
  const SolvePlan& SP = A.fronts.solve;
  const Symbolic& S = A.S;
  const bool fwd = dir == 0;
  const std::vector<SolveTask>& T = fwd ? SP.tf : SP.tb;
  PrunedPlan::Dir& D = P.dir[dir];
  const int nd = (int)SP.direct_cnt.size();
  const unsigned m = ++P.stamp;
  collect_run_set(P, SP, S, T, D, m, seed, nseed, R);
  // pruned order: forward, direct level l -> slot l, subtree item i -> nd + i, top task j -> nd + items + j; backward,
  // top task j -> slot j, subtree item i -> tasks + i, direct level l -> tasks + items + nd - 1 - l
  const int nt = (int)R.tasks.size(), ni = (int)R.items.size();
  const int o_item = fwd ? nd : nt, o_task = fwd ? nd + ni : 0;
  auto o_level = [&](int l) { return fwd ? l : nt + ni + nd - 1 - l; };
  for (int s : R.run) { P.ord0[s] = INT_MAX; P.ord1[s] = -1; }
  auto upd = [&](int s, int o) { P.ord0[s] = std::min(P.ord0[s], o); P.ord1[s] = std::max(P.ord1[s], o); };
  for (int l = 0; l < nd; ++l) for (int i : R.dl[l]) upd(SP.direct[l][i], o_level(l));
  for (int i = 0; i < ni; ++i)
    for (int e = P.item_ptr[R.items[i]]; e < P.item_ptr[R.items[i] + 1]; ++e) upd(P.item_fr[e], o_item + i);
  for (int j = 0; j < nt; ++j) {
    const SolveTask& K = T[R.tasks[j]];
    if (K.type == ST_SMALL) for (int w = 0; w < K.blk; ++w) upd(SP.bundle[K.s + w], o_task + j);
    else upd(K.s, o_task + j);
  }
  const int type_a = fwd ? ST_FP : ST_BT, type_b = fwd ? ST_FC : ST_BX;
  for (int s : R.run) {
    bool ok = P.ord1[s] >= 0;
    int na = 0, nb = 0;
    for (int e = D.task_ptr[s]; ok && e < D.task_ptr[s + 1]; ++e) {
      const SolveTask& K = T[D.task_idx[e]];
      ok = D.m_task[D.task_idx[e]] == m;
      if (ok && (K.type == type_a || K.type == type_b) && K.q == 0) {
        ok = e + K.nq <= D.task_ptr[s + 1];
        for (int q = 1; ok && q < K.nq; ++q) {
          const SolveTask& U = T[D.task_idx[e + q]];
          ok = U.type == K.type && U.blk == K.blk && U.cidx == K.cidx && U.q == q && D.m_task[D.task_idx[e + q]] == m;
        }
        (K.type == type_a ? na : nb) += 1;
      }
    }
    if (ok && S.f(s) > DF_MIDMAX && P.dlev[s] < 0 && P.item_of[s] < 0)
      ok = na == (S.k(s) + DF_BLK - 1) / DF_BLK && nb == ((fwd ? S.r(s) : S.k(s)) + DF_BLK - 1) / DF_BLK;
    auto neighbour = [&](int c) {   // c runs earlier in the pruned order, or joins the frontier
      if (P.m_run[c] == m) ok = (P.sub_of[s] >= 0 && P.sub_of[c] == P.sub_of[s]) || P.ord1[c] < P.ord0[s];
      else if (P.m_fr[c] != m) { P.m_fr[c] = m; R.fr.push_back(c); }
    };
    if (fwd) for (int e = S.child_ptr[s]; ok && e < S.child_ptr[s + 1]; ++e) neighbour(S.child_idx[e]);
    else if (ok && S.sn_parent[s] >= 0) neighbour(S.sn_parent[s]);
    if (!ok) {
      sv->err = std::string(call) + (fwd ? ": the pruned sweep" : ": the pruned backward sweep") + " of front " +
                std::to_string(s) + " fails its dependency check (not launched)";
      return B200LDLT_FATAL_ERROR;
    }
  }
  return B200LDLT_SUCCESS;
}

// bytes the pruned lists of R take in a staging (stage_pruned)
static size_t pruned_bytes(const PrunedSweep& R) {
  size_t ndir = 0;
  for (auto& v : R.dl) ndir += v.size();
  return align8(8 * R.items.size()) + align8(sizeof(SolveTask) * R.tasks.size()) + align8(4 * ndir) + align8(4 * R.fr.size());
}

// R's pruned lists to the staging h at offset o (8-aligned; the device copy of the staging is d): subtree items, top
// tasks (entries of T, the sweep's list), direct fronts, frontier.  pl points into d; *o_fr receives the offset of the frontier.  Returns the end offset.
static size_t stage_pruned(const SolvePlan& SP, const std::vector<SolveTask>& T, const PrunedSweep& R, char* h, const char* d,
                           size_t o, PrunedLists& pl, size_t* o_fr) {
  const int nd = (int)SP.direct_cnt.size();
  const size_t o_tf = o + align8(8 * R.items.size());
  const size_t o_dir = o_tf + align8(sizeof(SolveTask) * R.tasks.size());
  int2* hp = reinterpret_cast<int2*>(h + o);
  for (size_t i = 0; i < R.items.size(); ++i) hp[i] = SP.pairs[R.items[i]];
  SolveTask* ht = reinterpret_cast<SolveTask*>(h + o_tf);
  for (size_t j = 0; j < R.tasks.size(); ++j) ht[j] = T[R.tasks[j]];
  int* hd = reinterpret_cast<int*>(h + o_dir);
  pl.direct_off.assign(nd, 0); pl.direct_cnt.assign(nd, 0);
  int j = 0;
  for (int l = 0; l < nd; ++l) {
    pl.direct_off[l] = j; pl.direct_cnt[l] = (int)R.dl[l].size();
    for (int i : R.dl[l]) hd[j++] = SP.direct[l][i];
  }
  *o_fr = o_dir + align8(4 * (size_t)j);
  std::copy(R.fr.begin(), R.fr.end(), reinterpret_cast<int*>(h + *o_fr));
  pl.subpair = reinterpret_cast<const int2*>(d + o); pl.npair = (int)R.items.size();
  pl.tasks = reinterpret_cast<const SolveTask*>(d + o_tf); pl.ntasks = (int)R.tasks.size();
  pl.direct = reinterpret_cast<const int*>(d + o_dir);
  return *o_fr + align8(4 * R.fr.size());
}

// a compact b swept forward over a pruned run set R_f, as staged: R_f's ncol positions and their indices into the
// compact column (offsets o_pos / o_bi), the frontier of nfr fronts and the pruned lists
struct SparseFwd {
  int ncol = 0, nfr = 0;
  size_t o_pos = 0, o_bi = 0, o_fr = 0;
  PrunedLists pl{};
};

// R_f's positions (the fronts of run, in order) to pos, and to bi for each its index into the compact b of nbi entries
// at the pivot positions seed (-1: no entry)
static void stage_positions(PrunedPlan& P, const Symbolic& S, const std::vector<int>& run, const int* seed, int nbi,
                            int* pos, int* bi) {
  for (int i = 0; i < nbi; ++i) P.pos_bi[seed[i]] = i;
  int j = 0;
  for (int s : run) for (int p = S.sn_start[s]; p < S.sn_start[s + 1]; ++p, ++j) { pos[j] = p; bi[j] = P.pos_bi[p]; }
  for (int i = 0; i < nbi; ++i) P.pos_bi[seed[i]] = -1;
}

// The forward stage of w compact columns (column c of b at b + c nbi) over the staged F: k_sps_in (x = P^T S b on R_f,
// the frontier's update vectors and flags) and the forward sweep over the pruned lists, D^-1 applied or not.  The one
// forward stage of the three pruned calls: the sparse forward solve (one column), the sparse solve, and the entries of
// A^-1 (unit columns: b is an identity).  Launches: 1 + the direct levels that hold a front of R_f + 1 when R_f has a
// front outside them.
static int sparse_forward(Solver* sv, SweepState& W, const SparseFwd& F, const double* b, int nbi, int w, bool apply_d) {
  Analysis& A = *sv->an;
  const char* d = A.pruned->stg.d.p;
  A.solve_epoch++;
  const unsigned g = std::max(1u, cdiv(F.ncol, 256) + (unsigned)F.nfr);
  k_sps_in<<<dim3(g, w), 256, 0, sv->stream>>>(F.ncol, reinterpret_cast<const int*>(d + F.o_pos),
                                               reinterpret_cast<const int*>(d + F.o_bi), A.d_perm.p, A.d_scale.p, b, nbi,
                                               W.d_x.p, W.M.x, F.nfr, reinterpret_cast<const int*>(d + F.o_fr),
                                               A.d_rows_ptr.p, W.d_cbv.p, W.M.cbv, W.d_done_f.p, W.M.nsn, A.solve_epoch);
  ++sv->launches;
  return launch_sweep(sv, A.fronts.solve, W, w, true, apply_d, &F.pl);
}

// ---- sparse forward solve (b200ldlt_sparse_fwd_solve) ----------------------------------------------------------------
// one call as prepared on the host: the forward stage of b, and in the staging the output's y-store offsets {0, nxi}
// and its nxi positions (the reach, ascending: xindex)
struct SfsCall {
  int nbi = 0, nxi = 0;
  SparseFwd F;
  size_t o_yoff = 0, o_xi = 0;
};

// Host part (arguments already checked): the pruned forward sweep of b's variables and everything the device needs in
// the list staging.  FATAL_ERROR with a message, nothing written to the caller and nothing launched, for a failed check
// or allocation.
static int sfs_prepare(Solver* sv, int nbi, const int* bindex, SfsCall& C) {
  Analysis& A = *sv->an;
  PrunedPlan& P = *A.pruned;
  const Symbolic& S = A.S;
  std::vector<int> seed(nbi);
  for (int i = 0; i < nbi; ++i) seed[i] = P.iperm[bindex[i]];
  PrunedSweep R;
  { const int rc = prune(sv, "sparse_fwd_solve", 0, seed.data(), nbi, R); if (rc != B200LDLT_SUCCESS) return rc; }
  std::sort(R.run.begin(), R.run.end());
  C.nbi = nbi;
  C.F.ncol = npos(S, R.run); C.F.nfr = (int)R.fr.size();
  C.nxi = npos(S, R.reach);
  // staging layout: the pruned lists, run-set positions and their b indices, the y-store offsets, output positions
  C.F.o_pos = pruned_bytes(R);
  C.F.o_bi = C.F.o_pos + 4 * (size_t)C.F.ncol;
  C.o_yoff = align8(C.F.o_bi + 4 * (size_t)C.F.ncol);
  C.o_xi = C.o_yoff + 16;
  { const int rc = P.stg.reserve(sv, "sparse_fwd_solve", C.o_xi + 4 * (size_t)C.nxi); if (rc != B200LDLT_SUCCESS) return rc; }
  char* h = P.stg.h;
  stage_pruned(A.fronts.solve, A.fronts.solve.tf, R, h, P.stg.d.p, 0, C.F.pl, &C.F.o_fr);
  stage_positions(P, S, R.run, seed.data(), nbi, reinterpret_cast<int*>(h + C.F.o_pos), reinterpret_cast<int*>(h + C.F.o_bi));
  const long long yoff[2] = {0, C.nxi};
  memcpy(h + C.o_yoff, yoff, sizeof(yoff));
  int* xi = reinterpret_cast<int*>(h + C.o_xi);
  for (int s : R.reach) for (int p = S.sn_start[s]; p < S.sn_start[s + 1]; ++p) *xi++ = p;
  P.last_sfs = std::move(R.run);
  return B200LDLT_SUCCESS;
}

// Device part: the staging in, the forward stage of job 1 (D^-1 left out) on the single-column state, and the reached
// positions out through the y-store gather (k_inv_out, one column).  Launches: 2 + the direct levels that hold a front
// of the run set + 1 when the run set has a front outside them.
static int sfs_enqueue(Solver* sv, const SfsCall& C, const double* d_b, double* d_out) {
  Analysis& A = *sv->an;
  PrunedPlan& P = *A.pruned;
  SweepState& W = A.sweep;
  const char* d = P.stg.d.p;
  { const int rc = P.stg.upload(sv, C.o_xi + 4 * (size_t)C.nxi); if (rc != B200LDLT_SUCCESS) return rc; }
  { const int rc = sparse_forward(sv, W, C.F, d_b, C.nbi, 1, false); if (rc != B200LDLT_SUCCESS) return rc; }
  k_inv_out<<<dim3(cdiv(C.nxi, 256), 1), 256, 0, sv->stream>>>(0, reinterpret_cast<const long long*>(d + C.o_yoff),
                                                               reinterpret_cast<const int*>(d + C.o_xi), A.d_piv_big.p,
                                                               W.d_x.p, W.M.x, W.d_bigv.p, W.M.bigv, d_out);
  ++sv->launches;
  CU(cudaGetLastError());
  return B200LDLT_SUCCESS;
}

// ---- entries of A^-1 (b200ldlt_inverse_entries) ---------------------------------------------------------------------
// one block of unit columns: columns [c0, c0 + w) of the call, the longest reach of its columns, and the forward stage
// of its unit columns
struct InvBlock {
  int c0 = 0, w = 0, maxlen = 0;
  SparseFwd F;
};
// one call as prepared on the host: the entry list, the y store's offsets (ncols + 1) and positions, the identity of
// order neye (the compact b of every block: column c of a block is column c of the identity), the blocks
struct InvCall {
  int nent = 0, ncols = 0, neye = 0;
  size_t o_ent = 0, o_yoff = 0, o_ypos = 0, o_eye = 0, staged = 0;
  std::vector<InvBlock> blk;
};

// Host part of b200ldlt_inverse_entries.  The columns are the distinct variables of irow and jcol, sorted by pivot
// position (neighbours in the tree share fronts) and cut into blocks of `width`; each block is one pruned forward sweep
// (prune, its dependency check included) of its unit columns, staged for sparse_forward with a compact b whose seeds are
// the pivot positions of its columns and whose column c is column c of the staged identity.  Column c keeps
// y_c = L^-1 P^T S e_c on its reach, the path from its front to the root (ascending positions), at [yoff[c], yoff[c + 1])
// of the y store.  Entry (i, j) reads the common suffix of y_i and y_j: the path from the lowest common ancestor of
// their fronts to the root, pathlen of that front long (0 in different trees of the forest).  Everything the device
// needs goes to the list staging, each block in a region of its own, so one copy carries the call.  FATAL_ERROR with a message, nothing written and nothing launched,
// for a failed check or allocation.
static int inv_prepare(Solver* sv, int nent, const int* irow, const int* jcol, int width, InvCall& C) {
  Analysis& A = *sv->an;
  PrunedPlan& P = *A.pruned;
  const SolvePlan& SP = A.fronts.solve;
  const Symbolic& S = A.S;
  std::vector<int> cols;
  for (int t = 0; t < nent; ++t)
    for (const int v : {irow[t], jcol[t]})
      if (P.col_of[v] < 0) { P.col_of[v] = 0; cols.push_back(v); }
  std::sort(cols.begin(), cols.end(), [&](int a, int b) { return P.iperm[a] < P.iperm[b]; });
  const int nc = (int)cols.size();
  for (int c = 0; c < nc; ++c) P.col_of[cols[c]] = c;
  auto finish = [&](int rc) { for (const int v : cols) P.col_of[v] = -1; return rc; };   // (col_of back to -1)
  std::vector<long long> yoff(nc + 1, 0);
  for (int c = 0; c < nc; ++c) yoff[c + 1] = yoff[c] + P.pathlen[P.sn_of[P.iperm[cols[c]]]];
  const long long ny = yoff[nc];
  // the blocks, and the staging layout: entries, yoff, ypos, the identity, then per block its pruned lists, run-set
  // positions and their indices into the block's columns
  C.nent = nent; C.ncols = nc; C.neye = std::min(width, nc);
  C.o_ent = 0;
  C.o_yoff = align8(sizeof(InvEnt) * (size_t)nent);
  C.o_ypos = C.o_yoff + 8 * (size_t)(nc + 1);
  C.o_eye = align8(C.o_ypos + 4 * (size_t)ny);
  size_t o = C.o_eye + 8 * (size_t)C.neye * C.neye;
  std::vector<PrunedSweep> R((nc + width - 1) / width);
  std::vector<size_t> o_lst(R.size());
  std::vector<int> seed(width), run_all;
  C.blk.assign(R.size(), InvBlock());
  for (size_t b = 0; b < R.size(); ++b) {
    InvBlock& B = C.blk[b];
    B.c0 = (int)b * width; B.w = std::min(width, nc - B.c0);
    for (int c = 0; c < B.w; ++c) {
      seed[c] = P.iperm[cols[B.c0 + c]];
      B.maxlen = std::max(B.maxlen, (int)(yoff[B.c0 + c + 1] - yoff[B.c0 + c]));
    }
    const int rc = prune(sv, "inverse_entries", 0, seed.data(), B.w, R[b]);
    if (rc != B200LDLT_SUCCESS) return finish(rc);
    B.F.ncol = npos(S, R[b].run);
    B.F.nfr = (int)R[b].fr.size();
    run_all.insert(run_all.end(), R[b].run.begin(), R[b].run.end());
    o_lst[b] = o;
    B.F.o_pos = o + pruned_bytes(R[b]);
    B.F.o_bi = B.F.o_pos + 4 * (size_t)B.F.ncol;
    o = align8(B.F.o_bi + 4 * (size_t)B.F.ncol);
  }
  C.staged = o;
  { const int rc = P.stg.reserve(sv, "inverse_entries", C.staged); if (rc != B200LDLT_SUCCESS) return finish(rc); }
  if ((size_t)ny > P.d_y.n && P.d_y.alloc(ny) != cudaSuccess) {
    cudaGetLastError();
    sv->err = "inverse_entries: cannot allocate the y store of " + std::to_string(ny) + " doubles";
    return finish(B200LDLT_FATAL_ERROR);
  }
  char* h = P.stg.h;
  InvEnt* he = reinterpret_cast<InvEnt*>(h + C.o_ent);
  for (int t = 0; t < nent; ++t) {
    const int ci = P.col_of[irow[t]], cj = P.col_of[jcol[t]];
    int a = P.sn_of[P.iperm[irow[t]]], b = P.sn_of[P.iperm[jcol[t]]];
    while (P.depth[a] > P.depth[b]) a = S.sn_parent[a];
    while (P.depth[b] > P.depth[a]) b = S.sn_parent[b];
    while (a != b) { a = S.sn_parent[a]; b = S.sn_parent[b]; }   // (both -1 at once in different trees)
    const int m = a >= 0 ? P.pathlen[a] : 0;
    he[t] = InvEnt{yoff[ci + 1] - m, yoff[cj + 1] - m, m, 0};
  }
  memcpy(h + C.o_yoff, yoff.data(), 8 * (size_t)(nc + 1));
  int* yp = reinterpret_cast<int*>(h + C.o_ypos);
  for (int c = 0; c < nc; ++c)
    for (int s = P.sn_of[P.iperm[cols[c]]]; s >= 0; s = S.sn_parent[s])
      for (int p = S.sn_start[s]; p < S.sn_start[s + 1]; ++p) *yp++ = p;
  double* eye = reinterpret_cast<double*>(h + C.o_eye);
  std::fill(eye, eye + (size_t)C.neye * C.neye, 0.0);
  for (int c = 0; c < C.neye; ++c) eye[(size_t)c * C.neye + c] = 1.0;
  for (size_t b = 0; b < R.size(); ++b) {
    InvBlock& B = C.blk[b];
    stage_pruned(SP, SP.tf, R[b], h, P.stg.d.p, o_lst[b], B.F.pl, &B.F.o_fr);
    for (int c = 0; c < B.w; ++c) seed[c] = P.iperm[cols[B.c0 + c]];
    stage_positions(P, S, R[b].run, seed.data(), B.w, reinterpret_cast<int*>(h + B.F.o_pos),
                    reinterpret_cast<int*>(h + B.F.o_bi));
  }
  std::sort(run_all.begin(), run_all.end());
  run_all.erase(std::unique(run_all.begin(), run_all.end()), run_all.end());
  P.last_inv = std::move(run_all);
  return finish(B200LDLT_SUCCESS);
}

// Device part: the staging in, then per block the forward stage of job 1 (sparse_forward, D^-1 left out; block width
// w: the blocked state, one column: the single-column state) and k_inv_out into the y store; then k_inv_dot to out.
// Launches: sum over blocks of (2 + the direct levels that hold a front of the block's run set + 1 when the run set has
// a front outside them), + 1.
static int inv_enqueue(Solver* sv, const InvCall& C, double* out) {
  Analysis& A = *sv->an;
  PrunedPlan& P = *A.pruned;
  cudaStream_t st = sv->stream;
  const char* d = P.stg.d.p;
  const long long* yoff = reinterpret_cast<const long long*>(d + C.o_yoff);
  const int* ypos = reinterpret_cast<const int*>(d + C.o_ypos);
  const double* eye = reinterpret_cast<const double*>(d + C.o_eye);
  { const int rc = P.stg.upload(sv, C.staged); if (rc != B200LDLT_SUCCESS) return rc; }
  for (const InvBlock& B : C.blk) {
    SweepState& W = B.w == 1 ? A.sweep : *A.blk;
    const int rc = sparse_forward(sv, W, B.F, eye, C.neye, B.w, false);
    if (rc != B200LDLT_SUCCESS) return rc;
    k_inv_out<<<dim3(cdiv(B.maxlen, 256), B.w), 256, 0, st>>>(B.c0, yoff, ypos, A.d_piv_big.p, W.d_x.p, W.M.x,
                                                              W.d_bigv.p, W.M.bigv, P.d_y.p);
    ++sv->launches;
  }
  k_inv_dot<<<cdiv(C.nent, 8), 256, 0, st>>>(C.nent, reinterpret_cast<const InvEnt*>(d + C.o_ent), P.d_y.p, ypos,
                                             A.d_ptype.p, A.d_dinv.p, A.d_doff.p, out);
  ++sv->launches;
  CU(cudaGetLastError());
  return B200LDLT_SUCCESS;
}

// ---- sparse solve (b200ldlt_sparse_solve) ---------------------------------------------------------------------------
// one sparse solve as prepared on the host: dense b (bindex NULL) / every entry (xsel NULL); the forward stage of a
// sparse b; the nz positions to zero and the nfb fronts of F_b between the sweeps; the staging offsets (bytes) and the
// pruned backward lists on the device
struct SpsCall {
  bool dense_b = false, all_x = false;
  int nbi = 0, nxs = 0, nz = 0, nfb = 0;
  SparseFwd F;
  size_t o_z = 0, o_fb = 0, o_xpos = 0, staged = 0;
  PrunedLists plb{};
};

// Host part of b200ldlt_sparse_solve (arguments already checked): one pruned forward sweep for the pattern of b and one
// pruned backward sweep for the selection (prune), shared by every block of columns; the positions to zero between the
// sweeps (R_b \ R_f with a sparse b; with a full selection everything outside R_f); the output positions; all of it in
// the list staging.  FATAL_ERROR with a message, nothing written and nothing launched, for a failed check or allocation.
static int sps_prepare(Solver* sv, int nbi, const int* bindex, int nxs, const int* xsel, SpsCall& C) {
  Analysis& A = *sv->an;
  PrunedPlan& P = *A.pruned;
  const SolvePlan& SP = A.fronts.solve;
  const Symbolic& S = A.S;
  const int nsn = S.nsn;
  C.dense_b = !bindex; C.all_x = !xsel; C.nbi = nbi; C.nxs = nxs;
  std::vector<int> all;
  if (C.dense_b || C.all_x) { all.resize(nsn); for (int s = 0; s < nsn; ++s) all[s] = s; }
  if (C.dense_b && C.all_x) {   // job 0 itself
    P.last_fwd = all; P.last_bwd = all;
    return B200LDLT_SUCCESS;
  }
  PrunedSweep Rf, Rb;
  std::vector<int> seed;
  if (!C.dense_b) {
    seed.resize(nbi);
    for (int i = 0; i < nbi; ++i) seed[i] = P.iperm[bindex[i]];
    const int rc = prune(sv, "sparse_solve", 0, seed.data(), nbi, Rf);
    if (rc != B200LDLT_SUCCESS) return rc;
  }
  if (!C.all_x) {
    std::vector<int> sb(nxs);
    for (int i = 0; i < nxs; ++i) sb[i] = P.iperm[xsel[i]];
    const int rc = prune(sv, "sparse_solve", 1, sb.data(), nxs, Rb);
    if (rc != B200LDLT_SUCCESS) return rc;
  }
  std::vector<int> runf = C.dense_b ? all : Rf.run, runb = C.all_x ? all : Rb.run;
  std::sort(runf.begin(), runf.end());
  std::sort(runb.begin(), runb.end());
  std::vector<int> zf;   // fronts whose forward result is zeroed between the sweeps
  if (!C.dense_b) std::set_difference(runb.begin(), runb.end(), runf.begin(), runf.end(), std::back_inserter(zf));
  if (!C.dense_b) C.F.ncol = npos(S, runf);
  C.nz = npos(S, zf);
  C.F.nfr = (int)Rf.fr.size(); C.nfb = (int)Rb.fr.size();
  // staging layout: forward pruned lists, backward pruned lists, run-set positions and their b indices, zeroed
  // positions, output positions
  C.F.o_pos = pruned_bytes(Rf) + pruned_bytes(Rb);
  C.F.o_bi = C.F.o_pos + 4 * (size_t)C.F.ncol;
  C.o_z = C.F.o_bi + 4 * (size_t)C.F.ncol;
  C.o_xpos = C.o_z + 4 * (size_t)C.nz;
  C.staged = align8(C.o_xpos + (C.all_x ? 0 : 4 * (size_t)nxs));
  { const int rc = P.stg.reserve(sv, "sparse_solve", C.staged); if (rc != B200LDLT_SUCCESS) return rc; }
  char* h = P.stg.h;
  const char* d = P.stg.d.p;
  size_t o = 0;
  if (!C.dense_b) o = stage_pruned(SP, SP.tf, Rf, h, d, o, C.F.pl, &C.F.o_fr);
  if (!C.all_x) {
    stage_pruned(SP, SP.tb, Rb, h, d, o, C.plb, &C.o_fb);
    int* xp = reinterpret_cast<int*>(h + C.o_xpos);
    for (int i = 0; i < nxs; ++i) xp[i] = P.iperm[xsel[i]];
  }
  if (!C.dense_b)
    stage_positions(P, S, runf, seed.data(), nbi, reinterpret_cast<int*>(h + C.F.o_pos), reinterpret_cast<int*>(h + C.F.o_bi));
  int* zp = reinterpret_cast<int*>(h + C.o_z);
  for (int s : zf) for (int p = S.sn_start[s]; p < S.sn_start[s + 1]; ++p) *zp++ = p;
  P.last_fwd = std::move(runf);
  P.last_bwd = std::move(runb);
  return B200LDLT_SUCCESS;
}

// Device part: the staging in, then per block of w columns (the blocked state, or the single-column state for w = 1):
// the forward stage -- dense b: job 0's (k_rhs_in and the full sweep); sparse b: sparse_forward with D^-1 applied (the
// rounding of the fused sweep) -- then under the backward epoch k_sps_mid, the backward sweep (pruned to R_b unless
// every entry is selected) and the output (k_sol_out for every entry, k_sps_out for a selection).  Launches per block:
// 1 + d_f + t_f + 1 + d_b + t_b + 1; with a dense b and every entry selected the block is job 0 itself (enqueue_solve):
// 4 + 2 D.
static int sps_enqueue(Solver* sv, const SpsCall& C, int nrhs, bool blocked, const double* d_b, double* d_x) {
  Analysis& A = *sv->an;
  PrunedPlan& P = *A.pruned;
  const SolvePlan& SP = A.fronts.solve;
  cudaStream_t st = sv->stream;
  const int n = sv->n;
  const char* d = P.stg.d.p;
  const bool job0 = C.dense_b && C.all_x;
  if (!job0) { const int rc = P.stg.upload(sv, C.staged); if (rc != B200LDLT_SUCCESS) return rc; }
  return for_blocks(nrhs, blocked ? A.blk->width : 1, [&](int c, int w) -> int {
    SweepState& W = w == 1 ? A.sweep : *A.blk;
    const double* b = d_b + (size_t)c * C.nbi;
    double* x = d_x + (size_t)c * C.nxs;
    if (job0) return enqueue_solve(sv, W, 0, b, x, w);
    int rc = C.dense_b ? forward(sv, SP, W, b, w) : sparse_forward(sv, W, C.F, b, C.nbi, w, true);
    if (rc != B200LDLT_SUCCESS) return rc;
    A.solve_epoch++;
    const unsigned g = std::max(1u, cdiv(C.nz, 256) + cdiv(C.nfb, 256));
    k_sps_mid<<<dim3(g, w), 256, 0, st>>>(C.nz, reinterpret_cast<const int*>(d + C.o_z), A.d_piv_big.p, W.d_x.p, W.M.x,
                                          W.d_bigv.p, W.M.bigv, C.nfb, reinterpret_cast<const int*>(d + C.o_fb),
                                          W.d_done_b.p, W.M.nsn, A.solve_epoch);
    ++sv->launches;
    rc = launch_sweep(sv, SP, W, w, false, true, C.all_x ? nullptr : &C.plb);
    if (rc != B200LDLT_SUCCESS) return rc;
    if (C.all_x)
      k_sol_out<<<dim3(cdiv(n, 256), w), 256, 0, st>>>(n, A.d_perm.p, A.d_scale.p, W.d_x.p, W.M.x, x);
    else
      k_sps_out<<<dim3(cdiv(C.nxs, 256), w), 256, 0, st>>>(C.nxs, reinterpret_cast<const int*>(d + C.o_xpos), A.d_perm.p,
                                                            A.d_scale.p, W.d_x.p, W.M.x, x);
    ++sv->launches;
    CU(cudaGetLastError());
    return B200LDLT_SUCCESS;
  });
}

static int shard_setup(Solver* sv, int rank, int world) {
  Analysis& A = *sv->an;
  Symbolic& S = A.S;
  cudaStream_t st = sv->stream;
  Analysis::Shard& H = A.shard;
  H.rank = rank; H.world = world;
  H.nsub = shard_plan(S, world, H.owner);
  H.cut_roots.clear(); H.top_fronts.clear();
  std::vector<char> take[2];
  take[0].assign(S.nsn, 0); take[1].assign(S.nsn, 0);
  for (int s = 0; s < S.nsn; ++s) {
    if (H.owner[s] < 0) { take[1][s] = (rank == 0); H.top_fronts.push_back(s); }
    else {
      take[0][s] = (H.owner[s] == rank);
      const int p = S.sn_parent[s];
      if (p >= 0 && H.owner[p] < 0) H.cut_roots.push_back(s);
    }
  }
  for (int ph = 0; ph < 2; ++ph) {
    const int rc = build_front_plan(sv, A, take[ph], take[ph], H.part[ph]);
    if (rc != B200LDLT_SUCCESS) return rc;
  }
  {
    std::vector<int> mc;
    for (int s : H.cut_roots) if (H.owner[s] != 0) mc.push_back(s);
    size_t cnt = mc.size();
    if (mc.empty()) mc.push_back(0);
    CU(H.d_mark_cut.upload(mc, st));
    H.d_mark_cut.n = cnt;
    std::vector<int> mt = H.top_fronts;
    cnt = mt.size();
    if (mt.empty()) mt.push_back(0);
    CU(H.d_mark_top.upload(mt, st));
    H.d_mark_top.n = cnt;
  }
  H.active = true;
  return B200LDLT_SUCCESS;
}

}  // namespace b200

using namespace b200;

extern "C" {

void b200ldlt_default_options(b200ldlt_options* o) {
  memset(o, 0, sizeof(*o));
  o->device = -1;
  o->stream = nullptr;
  o->ordering = 0;
  o->pair_saddle = 1;
  o->leaf_k = 32;
  o->relax_frac = 0.05;   // 5 % relaxed amalgamation (H100 SXM, 700 W: N=400 5.83 ms vs 6.13 at 0.02, 6.28 at 0.10;
                          // N=800 21.2 ms vs 21.0 at 0.02, 22.8 at 0.10)
  o->scaling = 2;
  o->pivtol = 1e-8;
  o->pivtolmax = 1e-4;
  o->tiny = 1e-15;
  o->smem_front_max = 96;    // fronts of order 65..96 in shared memory, larger ones through the panel pipeline
                             // (H100 SXM, 700 W: 64 and 128 are 1-2.5 % slower at N=400 and N=800)
  o->tc_schur_min_r = 0;
  o->use_graph = 1;   /* 1 = CUDA-graph replay of the factorisation; any other value = plain launches */
  o->verbose = 0;
}

b200ldlt_handle b200ldlt_create(const b200ldlt_options* opt) {
  Solver* sv = new Solver();
  if (opt) sv->opt = *opt; else b200ldlt_default_options(&sv->opt);
  if (sv->opt.smem_front_max > 160) sv->opt.smem_front_max = 160;
  if (sv->opt.smem_front_max < 8) sv->opt.smem_front_max = 8;
  sv->pivtol = sv->opt.pivtol;
  sv->dbg.read();
  sv->tc_min_r = sv->opt.tc_schur_min_r;
  memset(&sv->info, 0, sizeof(sv->info));
  int ndev = 0;
  cudaError_t e = cudaGetDeviceCount(&ndev);
  if (e != cudaSuccess || ndev == 0) {
    fprintf(stderr, "[b200ldlt] FATAL: no usable CUDA device (%s); this backend has no CPU fallback\n",
            e != cudaSuccess ? cudaGetErrorString(e) : "device count is 0");
    delete sv;
    return nullptr;
  }
  if (sv->opt.device >= 0) sv->dev = sv->opt.device; else cudaGetDevice(&sv->dev);
  if (cudaSetDevice(sv->dev) != cudaSuccess) {
    fprintf(stderr, "[b200ldlt] FATAL: cannot select CUDA device %d\n", sv->dev);
    delete sv;
    return nullptr;
  }
  // stream priorities: the chain of the big fronts (main stream) is the critical path of a factorisation; the bulk
  // updates that trail it must never delay one of its launches
  int prio_lo = 0, prio_hi = 0;
  cudaDeviceGetStreamPriorityRange(&prio_lo, &prio_hi);
  if (sv->opt.stream) sv->stream = (cudaStream_t)sv->opt.stream;
  else { cudaStreamCreateWithPriority(&sv->stream, cudaStreamNonBlocking, prio_hi); sv->own_stream = true; }
  cudaStreamCreateWithPriority(&sv->stream2, cudaStreamNonBlocking, std::min(prio_lo, prio_hi + 1));
  cudaStreamCreateWithPriority(&sv->stream3, cudaStreamNonBlocking, prio_lo);
  for (auto& q : sv->side) cudaStreamCreateWithPriority(&q, cudaStreamNonBlocking, prio_lo);
  cudaEventCreate(&sv->ev0);
  cudaEventCreate(&sv->ev1);
  for (auto& e : sv->ev_chunk) cudaEventCreateWithFlags(&e, cudaEventDisableTiming);
  cudaHostAlloc((void**)&sv->h_counters, CNT_N * sizeof(int), cudaHostAllocDefault);
  return (b200ldlt_handle)sv;
}

void b200ldlt_destroy(b200ldlt_handle h) {
  Solver* sv = (Solver*)h;
  if (!sv) return;
  cudaSetDevice(sv->dev);
  if (sv->stream) cudaStreamSynchronize(sv->stream);
  delete sv;
}

const char* b200ldlt_last_error(b200ldlt_handle h) { return h ? ((Solver*)h)->err.c_str() : "null handle"; }

int b200ldlt_analyse(b200ldlt_handle h, int dim, int nonzeros, const int* irn, const int* jcn) {
  Solver* sv = (Solver*)h;
  if (!sv) return B200LDLT_FATAL_ERROR;
  if (dim <= 0 || nonzeros < 0 || (nonzeros > 0 && (!irn || !jcn))) { sv->err = "analyse: bad arguments"; return B200LDLT_FATAL_ERROR; }
  for (int e = 0; e < nonzeros; ++e)
    if (irn[e] < 1 || irn[e] > dim || jcn[e] < 1 || jcn[e] > dim) { sv->err = "analyse: index out of range"; return B200LDLT_FATAL_ERROR; }
  CU(cudaSetDevice(sv->dev));
  sv->n = dim; sv->nnz = nonzeros;
  sv->irn.assign(irn, irn + nonzeros);
  sv->jcn.assign(jcn, jcn + nonzeros);
  if (sv->h_vals) { cudaFreeHost(sv->h_vals); sv->h_vals = nullptr; }
  CU(cudaHostAlloc((void**)&sv->h_vals, std::max<size_t>(nonzeros, 1) * sizeof(double), cudaHostAllocDefault));
  memset(sv->h_vals, 0, std::max<size_t>(nonzeros, 1) * sizeof(double));
  sv->an.reset();
  sv->d_vals.release();
  sv->have_dev_vals = false;
  sv->sc_vars.clear();                // (a new pattern makes the Schur indices meaningless)
  if (sv->amat) { b200vec_tmat_destroy(sv->amat); sv->amat = nullptr; }
  return B200LDLT_SUCCESS;
}

double* b200ldlt_values_ptr(b200ldlt_handle h) { return h ? ((Solver*)h)->h_vals : nullptr; }

int b200ldlt_analyse_now(b200ldlt_handle h, const double* vals) {
  Solver* sv = (Solver*)h;
  if (!sv || sv->n <= 0) return B200LDLT_FATAL_ERROR;
  CU(cudaSetDevice(sv->dev));
  return run_analysis(sv, vals);
}

int b200ldlt_factor(b200ldlt_handle h, int check_inertia, int expected_neg, int* num_neg) {
  Solver* sv = (Solver*)h;
  if (!sv) return B200LDLT_FATAL_ERROR;
  return do_factor(sv, nullptr, true, check_inertia, expected_neg, num_neg);
}

int b200ldlt_factor_device(b200ldlt_handle h, const double* d_vals, int check_inertia, int expected_neg, int* num_neg) {
  Solver* sv = (Solver*)h;
  if (!sv || !d_vals) return B200LDLT_FATAL_ERROR;
  return do_factor(sv, d_vals, false, check_inertia, expected_neg, num_neg);
}

int b200ldlt_refactor(b200ldlt_handle h, int check_inertia, int expected_neg, int* num_neg) {
  Solver* sv = (Solver*)h;
  if (!sv || !sv->have_dev_vals) { if (sv) sv->err = "refactor: no matrix on the device"; return B200LDLT_FATAL_ERROR; }
  return do_factor(sv, sv->d_vals.p, false, check_inertia, expected_neg, num_neg);
}

}  // extern "C"

namespace b200 {
// ---- the calls that read the factors (include/b200ldlt.h, from the partial solves on) -------------------------------
// The state check, after the call's own argument checks: FATAL_ERROR with "<call>: ..." in last_error without factors
// and, unless sharded_ok, on a sharded handle; otherwise the handle's device is selected for what follows.
static int factors_state(Solver* sv, const char* call, bool sharded_ok = false, bool schur_call = false) {
  if (!sv->an || !sv->an->factored)
    sv->err = std::string(call) + ": no factors (factorise first; a SINGULAR factorisation keeps them only in keep mode, "
                                  "see b200ldlt_set_singular_action)";
  else if (sv->an->shard.active && !sharded_ok) sv->err = std::string(call) + ": not available on a sharded handle";
  else if (sv->sc_vars.empty() == schur_call)   // the Schur calls need Schur-mode factors, the others refuse them
    sv->err = std::string(call) + (schur_call ? ": not in Schur mode" : ": Schur mode");
  else { CU(cudaSetDevice(sv->dev)); return B200LDLT_SUCCESS; }
  return B200LDLT_FATAL_ERROR;
}

// a call without columns: succeeds, launches nothing, writes nothing to the caller's arrays
static int no_columns(Solver* sv) {
  sv->info.launches_solve = 0;
  sv->info.ms_solve_gpu = 0.0f;
  return B200LDLT_SUCCESS;
}

// The timed part of a call: enqueue() between the events ev0 and ev1 with the launch count from 0, then drain() (host
// work under the tail of the stream: the copy-out of staged_call) and the synchronise; info.ms_solve_gpu and
// launches_solve then describe the call.  Lazy state is built by the caller before, outside the window.
struct NoDrain { int operator()() const { return B200LDLT_SUCCESS; } };
template <class Enqueue, class Drain = NoDrain>
static int timed_call(Solver* sv, Enqueue&& enqueue, Drain&& drain = Drain()) {
  cudaStream_t st = sv->stream;
  sv->launches = 0;
  CU(cudaEventRecord(sv->ev0, st));
  { const int rc = enqueue(); if (rc != B200LDLT_SUCCESS) return rc; }
  CU(cudaEventRecord(sv->ev1, st));
  { const int rc = drain(); if (rc != B200LDLT_SUCCESS) return rc; }
  CU(cudaStreamSynchronize(st));
  cudaEventElapsedTime(&sv->info.ms_solve_gpu, sv->ev0, sv->ev1);
  sv->info.launches_solve = sv->launches;
  return B200LDLT_SUCCESS;
}

// A timed call on host columns: nin doubles of `in` to the device staging, enqueue(its device address), nout doubles
// back to `out` (which may be `in`), the copies inside the timed window.  Each way the copies run in at most four
// chunks, so that the DMA of one chunk runs under the host copy of the next (the caller's array is pageable: Ipopt
// allocates it per call, IpTSymLinearSolver.cpp:222-241).  The staging grows to the largest call and lasts until the
// next analysis.  nwork: the staging holds at least that many doubles (device scratch of enqueue beyond in and out).
// in_off: `in` is staged at that many doubles from the start (out always at the start).  in2: a second input of nin2
// doubles, staged directly after `in` in the same chunks.
template <class Enqueue>
static int staged_call(Solver* sv, const double* in, size_t nin, double* out, size_t nout, Enqueue&& enqueue,
                       size_t nwork = 0, size_t in_off = 0, const double* in2 = nullptr, size_t nin2 = 0) {
  Analysis& A = *sv->an;
  const size_t nall = nin + nin2, need = std::max(std::max(in_off + nall, nout), nwork);
  if (need > A.d_rhs.n) {
    A.d_rhs.release();
    if (A.h_rhs) cudaFreeHost(A.h_rhs);
    A.h_rhs = nullptr;
    CU(cudaHostAlloc((void**)&A.h_rhs, need * sizeof(double), cudaHostAllocDefault));
    CU(A.d_rhs.alloc(need));   // (so d_rhs.n counts the doubles of both buffers, 0 when either is missing)
  }
  cudaStream_t st = sv->stream;
  double* h = A.h_rhs;
  double* d = A.d_rhs.p;
  auto chunk = [](size_t total) { return std::max<size_t>((total + 3) / 4, 32768); };   // at most 4: ev_chunk
  const size_t ci = chunk(nall), co = chunk(nout);
  auto copy_out = [&]() -> int {
    for (size_t o = 0, k = 0; o < nout; o += co, ++k) {
      CU(cudaEventSynchronize(sv->ev_chunk[k]));
      memcpy(out + o, h + o, std::min(co, nout - o) * sizeof(double));
    }
    return B200LDLT_SUCCESS;
  };
  return timed_call(sv, [&]() -> int {
    for (size_t o = 0; o < nall; o += ci) {
      const size_t m = std::min(ci, nall - o);
      for (size_t e = o; e < o + m;) {   // (a chunk may end in `in` and go on in in2)
        const size_t k = std::min(o + m, e < nin ? nin : nall) - e;
        memcpy(h + in_off + e, e < nin ? in + e : in2 + (e - nin), k * sizeof(double));
        e += k;
      }
      CU(cudaMemcpyAsync(d + in_off + o, h + in_off + o, m * sizeof(double), cudaMemcpyHostToDevice, st));
    }
    { const int rc = enqueue(d); if (rc != B200LDLT_SUCCESS) return rc; }
    for (size_t o = 0, k = 0; o < nout; o += co, ++k) {
      CU(cudaMemcpyAsync(h + o, d + o, std::min(co, nout - o) * sizeof(double), cudaMemcpyDeviceToHost, st));
      CU(cudaEventRecord(sv->ev_chunk[k], st));
    }
    return B200LDLT_SUCCESS;
  }, copy_out);
}

// b200ldlt_solve (job 0) and b200ldlt_solve_partial (job 1..4) on nrhs columns of x, in place (host == true: x in host
// memory) / _device
static int solve_job(Solver* sv, int job, int nrhs, double* x, bool host) {
  if (job < 0 || job > 4) { sv->err = "solve_partial: job must be 0..4"; return B200LDLT_FATAL_ERROR; }
  { const int rc = factors_state(sv, job == 0 ? "solve" : "solve_partial", job == 0); if (rc != B200LDLT_SUCCESS) return rc; }
  if (nrhs <= 0) return no_columns(sv);
  const bool blocked = nrhs > 1 && block_solve_state(sv);
  auto enqueue = [&](double* d) { return enqueue_solve_columns(sv, d, nrhs, blocked, job); };
  const size_t cnt = (size_t)sv->n * nrhs;
  return host ? staged_call(sv, x, cnt, x, cnt, enqueue) : timed_call(sv, [&] { return enqueue(x); });
}

// b200ldlt_lmultiply (host == true: x and y in host memory) / _device
static int lmultiply(Solver* sv, int trans, int nrhs, const double* x, double* y, bool host) {
  if (trans != 0 && trans != 1) { sv->err = "lmultiply: trans must be 0 or 1"; return B200LDLT_FATAL_ERROR; }
  { const int rc = factors_state(sv, "lmultiply"); if (rc != B200LDLT_SUCCESS) return rc; }
  if (nrhs <= 0) return no_columns(sv);
  { const int rc = lmul_state(sv, nrhs); if (rc != B200LDLT_SUCCESS) return rc; }
  const size_t cnt = (size_t)sv->n * nrhs;
  // host: in place in the staging (both kernel pairs allow it)
  if (host) return staged_call(sv, x, cnt, y, cnt, [&](double* d) { return enqueue_lmul_columns(sv, trans, nrhs, d, d); });
  return timed_call(sv, [&] { return enqueue_lmul_columns(sv, trans, nrhs, x, y); });
}

// The index-set check of the pruned calls: "index out of range" when an entry of idx[0..cnt) is outside [0, n), and
// with `distinct` "bindex entry appears twice" when two are equal; nullptr when the set is good.
static const char* bad_index_set(int n, int cnt, const int* idx, bool distinct) {
  for (int i = 0; i < cnt; ++i)
    if (idx[i] < 0 || idx[i] >= n) return "index out of range";
  if (!distinct || cnt < 2) return nullptr;
  std::vector<char> seen(n, 0);
  for (int i = 0; i < cnt; ++i)
    if (seen[idx[i]]++) return "bindex entry appears twice";
  return nullptr;
}

// b200ldlt_sparse_fwd_solve (host == true: b and x in host memory) / _device
static int sparse_fwd(Solver* sv, int nbi, const int* bindex, const double* b, bool host, int* nxi, int* xindex, double* x) {
  const char* bad = (nbi < 0 || nbi > sv->n) ? "nbi must be 0..n"
                  : nbi > 0 && (!bindex || !b || !nxi || !xindex || !x) ? "NULL argument"
                  : bad_index_set(sv->n, nbi, bindex, true);
  if (bad) { sv->err = std::string("sparse_fwd_solve: ") + bad; return B200LDLT_FATAL_ERROR; }
  { const int rc = factors_state(sv, "sparse_fwd_solve"); if (rc != B200LDLT_SUCCESS) return rc; }
  if (nbi == 0) {
    if (nxi) *nxi = 0;
    return no_columns(sv);
  }
  { const int rc = pruned_state(sv, "sparse_fwd_solve"); if (rc != B200LDLT_SUCCESS) return rc; }
  SfsCall C;
  { const int rc = sfs_prepare(sv, nbi, bindex, C); if (rc != B200LDLT_SUCCESS) return rc; }
  // host: x at the start of the staging, b after it
  const int rc = host ? staged_call(sv, b, nbi, x, C.nxi, [&](double* d) { return sfs_enqueue(sv, C, d + C.nxi, d); }, 0, C.nxi)
                      : timed_call(sv, [&] { return sfs_enqueue(sv, C, b, x); });
  if (rc != B200LDLT_SUCCESS) return rc;
  memcpy(xindex, sv->an->pruned->stg.h + C.o_xi, sizeof(int) * (size_t)C.nxi);
  *nxi = C.nxi;
  return B200LDLT_SUCCESS;
}

// b200ldlt_inverse_entries (host == true: vals in host memory) / _device
static int inverse_entries(Solver* sv, int nent, const int* irow, const int* jcol, double* vals, bool host) {
  const char* bad = nent < 0 ? "nent must be >= 0" : nent > 0 && (!irow || !jcol || !vals) ? "NULL argument" : nullptr;
  if (!bad) bad = bad_index_set(sv->n, nent, irow, false);
  if (!bad) bad = bad_index_set(sv->n, nent, jcol, false);
  if (bad) { sv->err = std::string("inverse_entries: ") + bad; return B200LDLT_FATAL_ERROR; }
  { const int rc = factors_state(sv, "inverse_entries"); if (rc != B200LDLT_SUCCESS) return rc; }
  if (nent == 0) return no_columns(sv);
  { const int rc = pruned_state(sv, "inverse_entries"); if (rc != B200LDLT_SUCCESS) return rc; }
  bool several = false;
  for (int t = 0; !several && t < nent; ++t) several = irow[t] != irow[0] || jcol[t] != irow[0];
  const bool blocked = several && block_solve_state(sv);
  InvCall C;
  { const int rc = inv_prepare(sv, nent, irow, jcol, blocked ? sv->an->blk->width : 1, C); if (rc != B200LDLT_SUCCESS) return rc; }
  auto enqueue = [&](double* d) { return inv_enqueue(sv, C, d); };
  return host ? staged_call(sv, nullptr, 0, vals, (size_t)nent, enqueue) : timed_call(sv, [&] { return enqueue(vals); });
}

// b200ldlt_sparse_solve (host == true: b and x in host memory) / _device
static int sparse_solve(Solver* sv, int nrhs, int nbi, const int* bindex, const double* b, int nxs, const int* xsel,
                        double* x, bool host) {
  const int n = sv->n;
  const char* bad = nrhs < 0 ? "nrhs must be >= 0" : (nbi < 0 || nbi > n) ? "nbi must be 0..n" : nxs < 0 ? "nxs must be >= 0"
                  : ((!b && nrhs > 0 && nbi > 0) || (!x && nrhs > 0 && nxs > 0)) ? "NULL argument"
                  : (!bindex && nbi != n) ? "a NULL bindex needs nbi = n" : (!xsel && nxs != n) ? "a NULL xsel needs nxs = n"
                  : nullptr;
  if (!bad && bindex) bad = bad_index_set(n, nbi, bindex, true);
  if (!bad && xsel) bad = bad_index_set(n, nxs, xsel, false);
  if (bad) { sv->err = std::string("sparse_solve: ") + bad; return B200LDLT_FATAL_ERROR; }
  { const int rc = factors_state(sv, "sparse_solve"); if (rc != B200LDLT_SUCCESS) return rc; }
  if (nrhs == 0 || nxs == 0) return no_columns(sv);
  { const int rc = pruned_state(sv, "sparse_solve"); if (rc != B200LDLT_SUCCESS) return rc; }
  const bool blocked = nrhs > 1 && block_solve_state(sv);
  SpsCall C;
  { const int rc = sps_prepare(sv, nbi, bindex, nxs, xsel, C); if (rc != B200LDLT_SUCCESS) return rc; }
  const size_t nin = (size_t)nrhs * nbi, nout = (size_t)nrhs * nxs;
  // host: x at the start of the staging, b after it
  if (host) return staged_call(sv, b, nin, x, nout, [&](double* d) { return sps_enqueue(sv, C, nrhs, blocked, d + nout, d); }, 0, nout);
  return timed_call(sv, [&] { return sps_enqueue(sv, C, nrhs, blocked, b, x); });
}

// b200ldlt_solve_fredholm (host == true: x in host memory) / _device
static int fredholm(Solver* sv, int nrhs, double tol, double* x, int* consistent, bool host) {
  const char* bad = nrhs < 0 ? "nrhs must be >= 0" : !(tol >= 0.0) ? "tol must be >= 0"
                    : nrhs > 0 && (!x || !consistent) ? "NULL argument" : nullptr;
  if (bad) { sv->err = std::string("solve_fredholm: ") + bad; return B200LDLT_FATAL_ERROR; }
  { const int rc = factors_state(sv, "solve_fredholm"); if (rc != B200LDLT_SUCCESS) return rc; }
  if (nrhs == 0) return no_columns(sv);
  Analysis& A = *sv->an;
  const size_t n = sv->n, nb = n * nrhs;
  // no zero pivots: the solve itself, f = 0, every column consistent
  const bool zero_pivots = !A.zpos.empty();
  const bool blocked = (zero_pivots || nrhs > 1) && block_solve_state(sv);
  if (zero_pivots && sv->d_fred_nrm.n < 2 * (size_t)nrhs) CU(sv->d_fred_nrm.alloc(2 * (size_t)nrhs));
  if (zero_pivots && !blocked && A.d_fred_z.n != n) CU(A.d_fred_z.alloc(n));
  std::vector<unsigned long long> nrm(2 * (size_t)nrhs);
  auto enqueue = [&](double* d) -> int {
    if (!zero_pivots) {
      CU(cudaMemsetAsync(d + nb, 0, nb * sizeof(double), sv->stream));
      return enqueue_solve_columns(sv, d, nrhs, blocked);
    }
    { const int rc = enqueue_fredholm(sv, d, nrhs, blocked); if (rc != B200LDLT_SUCCESS) return rc; }
    CU(cudaMemcpyAsync(nrm.data(), sv->d_fred_nrm.p, nrm.size() * sizeof(unsigned long long), cudaMemcpyDeviceToHost, sv->stream));
    return B200LDLT_SUCCESS;
  };
  const int rc = host ? staged_call(sv, x, nb, x, 2 * nb, enqueue) : timed_call(sv, [&] { return enqueue(x); });
  if (rc != B200LDLT_SUCCESS) return rc;
  for (int i = 0; i < nrhs; ++i) {
    double ymax, zmax;
    memcpy(&ymax, &nrm[2 * (size_t)i], sizeof(double));
    memcpy(&zmax, &nrm[2 * (size_t)i + 1], sizeof(double));
    consistent[i] = !zero_pivots || zmax <= tol * ymax ? 1 : 0;
  }
  return B200LDLT_SUCCESS;
}

// ---- Schur mode (b200ldlt_set_schur): S_c, reduce, expand ---------------------------------------------------------------
// nrhs columns of d_b (leading dimension n).  Reduce (d_xs == nullptr): y = b_S - A_SE A_EE^-1 b_E to d_out (leading
// dimension m).  Expand: x to d_out (leading dimension n), x_S = xs (d_xs, leading dimension m), x_E = A_EE^-1 (b_E -
// A_ES xs).  Both start with job 1's forward sweep, which leaves the scaled reduced right-hand side in the Schur positions
// (the root's pivot block is the identity); expand then writes the scaled xs there, applies D^-1 to E and runs job 4's
// backward sweep, which passes the root's values through.  Blocks of up to B200_SOLVE_BLOCK columns (blocked: the result
// of block_solve_state), each column with the arithmetic of a single-column call.  d_out may be d_b.
static int enqueue_sc_columns(Solver* sv, int nrhs, const double* d_b, const double* d_xs, double* d_out, bool blocked) {
  Analysis& A = *sv->an;
  cudaStream_t st = sv->stream;
  const SolvePlan& SP = A.fronts.solve;
  const int n = sv->n, m = (int)sv->sc_vars.size();
  const int rc = for_blocks(nrhs, blocked ? A.blk->width : 1, [&](int c, int w) -> int {
    SweepState& W = w == 1 ? A.sweep : *A.blk;
    const long long ldx = W.M.x, ldb = W.M.bigv;
    const int rc2 = forward(sv, SP, W, d_b + (size_t)c * n, w, false);
    if (rc2 != B200LDLT_SUCCESS) return rc2;
    if (!d_xs) {
      k_sc_reduce<<<dim3(cdiv(m, 256), w), 256, 0, st>>>(m, n - m, A.d_piv_big.p, W.d_x.p, ldx, W.d_bigv.p, ldb,
                                                         A.d_sc_vars.p, A.d_scale.p, d_out + (size_t)c * m);
      ++sv->launches;
      return B200LDLT_SUCCESS;
    }
    k_sc_expand<<<dim3(cdiv(n, 256), w), 256, 0, st>>>(n, m, A.d_ptype.p, A.d_dinv.p, A.d_doff.p, A.d_piv_big.p,
                                                      W.d_x.p, ldx, W.d_bigv.p, ldb, A.d_sc_vars.p, A.d_scale.p,
                                                      d_xs + (size_t)c * m);
    ++sv->launches;
    return backward(sv, SP, W, d_out + (size_t)c * n, w);
  });
  if (rc != B200LDLT_SUCCESS) return rc;
  CU(cudaGetLastError());
  return B200LDLT_SUCCESS;
}

// b200ldlt_schur_complement (host == true: sc in host memory) / _device
static int schur_complement(Solver* sv, double* sc, bool host) {
  if (!sc) { sv->err = "schur_complement: NULL argument"; return B200LDLT_FATAL_ERROR; }
  { const int rc = factors_state(sv, "schur_complement", false, true); if (rc != B200LDLT_SUCCESS) return rc; }
  const Analysis& A = *sv->an;
  const size_t mm = A.d_sc.n;
  auto enqueue = [&](double* d) -> int {
    CU(cudaMemcpyAsync(d, A.d_sc.p, mm * sizeof(double), cudaMemcpyDeviceToDevice, sv->stream));
    return B200LDLT_SUCCESS;
  };
  return host ? staged_call(sv, nullptr, 0, sc, mm, enqueue) : timed_call(sv, [&] { return enqueue(sc); });
}

// b200ldlt_schur_reduce (xs == nullptr) and b200ldlt_schur_expand (host == true: the arrays in host memory) / _device
static int schur_solve(Solver* sv, const char* call, int nrhs, const double* b, const double* xs, double* out, bool host,
                       bool expand) {
  const char* bad = nrhs < 0 ? "nrhs must be >= 0" : nrhs > 0 && (!b || !out || (expand && !xs)) ? "NULL argument" : nullptr;
  if (bad) { sv->err = std::string(call) + ": " + bad; return B200LDLT_FATAL_ERROR; }
  { const int rc = factors_state(sv, call, false, true); if (rc != B200LDLT_SUCCESS) return rc; }
  if (nrhs == 0) return no_columns(sv);
  const size_t n = sv->n, m = sv->sc_vars.size(), nb = n * nrhs, mb = m * nrhs;
  const bool blocked = nrhs > 1 && block_solve_state(sv);
  if (!host) return timed_call(sv, [&] { return enqueue_sc_columns(sv, nrhs, b, expand ? xs : nullptr, out, blocked); });
  if (!expand)   // in place in the staging: y of a block lands below the b of the blocks after it
    return staged_call(sv, b, nb, out, mb, [&](double* d) { return enqueue_sc_columns(sv, nrhs, d, nullptr, d, blocked); });
  return staged_call(sv, b, nb, out, nb, [&](double* d) { return enqueue_sc_columns(sv, nrhs, d, d + nb, d, blocked); },
                     0, 0, xs, mb);
}

// ---- selected inversion (b200ldlt_selected_inverse) ----------------------------------------------------------------
static_assert(SI_MID == DF_MIDMAX && SI_MID == kSolveMidMax, "the fronts above SI_MID read the factorisation's L11^-1");

static int selinv_state(Solver* sv) {
  Analysis& A = *sv->an;
  if (A.selinv) return B200LDLT_SUCCESS;
  const Symbolic& S = A.S;
  const int n = S.n, nsn = S.nsn;
  cudaStream_t st = sv->stream;
  std::unique_ptr<SelInvPlan> P(new SelInvPlan());
  std::vector<long long> eoff(nsn, -1);
  long long etot = 0;
  for (int s = 0; s < nsn; ++s)
    if (S.f(s) > SI_SMALL && S.f(s) <= SI_MID) { eoff[s] = etot; etot += (long long)S.k(s) * S.k(s); }
  CU(P->d_E.alloc(std::max<long long>(etot, 1)));
  std::vector<int> fronts;
  std::vector<SiItem> items;
  std::vector<SiGather> gather;
  P->lev.assign(S.nlevels, SelInvPlan::Level());
  for (int l = 0; l < S.nlevels; ++l) {
    SelInvPlan::Level& L = P->lev[l];
    const int q0 = S.level_ptr[l], q1 = S.level_ptr[l + 1];
    L.g_off = (int)gather.size();
    for (int q = q0; q < q1; ++q) {
      const int s = S.level_sn[q], r = S.r(s);
      for (int b = 0; b < r; ++b)
        for (int a0 = b; a0 < r; a0 += 32) gather.push_back(SiGather{s, b, a0});
    }
    L.g_cnt = (int)gather.size() - L.g_off;
    L.s_off = (int)fronts.size();
    for (int q = q0; q < q1; ++q) {
      const int s = S.level_sn[q];
      if (S.f(s) > SI_SMALL) continue;
      fronts.push_back(s);
      L.smem = std::max(L.smem, ((size_t)S.f(s) * S.f(s) + (size_t)S.k(s) * S.k(s)) * sizeof(double));
    }
    L.s_cnt = (int)fronts.size() - L.s_off;
    L.m_off = (int)fronts.size();
    for (int q = q0; q < q1; ++q) if (S.f(S.level_sn[q]) > SI_SMALL && S.f(S.level_sn[q]) <= SI_MID) fronts.push_back(S.level_sn[q]);
    L.m_cnt = (int)fronts.size() - L.m_off;
    for (int pass = 0; pass < 3; ++pass) {
      L.t_off[pass] = (int)items.size();
      for (int q = q0; q < q1; ++q) {
        const int s = S.level_sn[q], k = S.k(s), r = S.r(s);
        if (S.f(s) <= SI_SMALL) continue;
        const bool big = S.f(s) > SI_MID;
        const int ld_e = big ? (k + DF_BLK - 1) / DF_BLK * DF_BLK : k;
        const double* E = big ? A.d_linv.p + A.linv_off[s] : P->d_E.p + eoff[s];
        const int nkb = (k + 63) / 64, nrb = (r + 63) / 64;
        if (pass < 2) {
          for (int ib = 0; ib < nrb; ++ib)
            for (int jb = 0; jb < nkb; ++jb) items.push_back(SiItem{s, ib, jb, ld_e, E});
        } else {
          for (int ib = 0; ib < nkb; ++ib)
            for (int jb = 0; jb <= ib; ++jb) items.push_back(SiItem{s, ib, jb, ld_e, E});
        }
      }
      L.t_cnt[pass] = (int)items.size() - L.t_off[pass];
    }
  }
  std::vector<int> iperm(n), sn_of(n);
  for (int i = 0; i < n; ++i) iperm[S.perm[i]] = i;
  for (int s = 0; s < nsn; ++s)
    for (int p = S.sn_start[s]; p < S.sn_start[s + 1]; ++p) sn_of[p] = s;
  CU(P->d_fronts.upload(fronts, st));
  CU(P->d_items.upload(items, st));
  CU(P->d_gather.upload(gather, st));
  CU(P->d_eoff.upload(eoff, st));
  CU(P->d_iperm.upload(iperm, st));
  CU(P->d_sn_of.upload(sn_of, st));
  CU(P->d_t2u.upload(S.t2u, st));
  CU(P->d_lpinv.alloc(n));
  CU(P->d_Z.alloc(S.L_off[nsn]));
  CU(cudaMemsetAsync(P->d_Z.p, 0, P->d_Z.n * sizeof(double), st));
  CU(P->d_diag.alloc(n));
  CU(P->d_vals.alloc(sv->nnz));
  // a constant limit, as for the factor kernels: the attribute is per process, so a per-handle value would change it
  // under the other handles
  CU(cudaFuncSetAttribute(k_si_small, cudaFuncAttributeMaxDynamicSharedMemorySize, SI_SMALL_SMEM));
  CU(cudaStreamSynchronize(st));
  if (sv->opt.verbose)
    fprintf(stderr, "[b200ldlt] selected inversion: %zu tile items, Z %.1f MB, L11^-1 (orders %d..%d) %.1f MB\n",
            items.size(), 8e-6 * (double)S.L_off[nsn], SI_SMALL + 1, SI_MID, 8e-6 * (double)etot);
  A.selinv = std::move(P);
  return B200LDLT_SUCCESS;
}

// top level first: per level gather, small fronts, L11^-1 of the middle fronts, the three tile passes; then the output
static int enqueue_selinv(Solver* sv, double* d_diag, double* d_vals) {
  const Analysis& A = *sv->an;
  const SelInvPlan& P = *A.selinv;
  const Symbolic& S = A.S;
  cudaStream_t st = sv->stream;
  const int n = S.n;
  int& L = sv->launches;
  k_si_prep<<<cdiv(n, 256), 256, 0, st>>>(n, P.d_sn_of.p, A.d_sn_start.p, A.d_lperm.p, P.d_lpinv.p); ++L;
  for (int l = S.nlevels - 1; l >= 0; --l) {
    const SelInvPlan::Level& V = P.lev[l];
    if (V.g_cnt) { k_si_gather<<<cdiv(V.g_cnt, 8), 256, 0, st>>>(A.DS, P.d_Z.p, A.d_CB.p, P.d_lpinv.p, P.d_gather.p + V.g_off, V.g_cnt); ++L; }
    if (V.s_cnt) { k_si_small<<<V.s_cnt, 128, V.smem, st>>>(A.DS, A.DN, P.d_Z.p, P.d_fronts.p + V.s_off); ++L; }
    if (V.m_cnt) { k_si_linv<<<V.m_cnt, 256, 0, st>>>(A.DS, A.DN, P.d_fronts.p + V.m_off, P.d_eoff.p, P.d_E.p); ++L; }
    if (V.t_cnt[0]) { k_si_tile<0><<<V.t_cnt[0], 256, 0, st>>>(A.DS, A.DN, P.d_Z.p, P.d_items.p + V.t_off[0]); ++L; }
    if (V.t_cnt[1]) { k_si_tile<1><<<V.t_cnt[1], 256, 0, st>>>(A.DS, A.DN, P.d_Z.p, P.d_items.p + V.t_off[1]); ++L; }
    if (V.t_cnt[2]) { k_si_tile<2><<<V.t_cnt[2], 256, 0, st>>>(A.DS, A.DN, P.d_Z.p, P.d_items.p + V.t_off[2]); ++L; }
  }
  k_si_out<<<cdiv(std::max<long long>(n, sv->nnz), 256), 256, 0, st>>>(
      n, sv->nnz, P.d_iperm.p, P.d_sn_of.p, A.d_sn_start.p, A.d_rows_ptr.p, A.d_L_off.p, P.d_lpinv.p, P.d_Z.p,
      A.d_scale.p, A.d_irn.p, A.d_jcn.p, P.d_t2u.p, A.d_u_dst64.p, d_diag, d_vals);
  ++L;
  CU(cudaGetLastError());
  return B200LDLT_SUCCESS;
}

// b200ldlt_selected_inverse (host == true: diag and vals in host memory) / _device
static int selected_inverse(Solver* sv, double* diag, double* vals, bool host) {
  if (!diag && !vals) { sv->err = "selected_inverse: diag and vals are both NULL"; return B200LDLT_FATAL_ERROR; }
  { const int rc = factors_state(sv, "selected_inverse"); if (rc != B200LDLT_SUCCESS) return rc; }
  { const int rc = selinv_state(sv); if (rc != B200LDLT_SUCCESS) return rc; }
  SelInvPlan& P = *sv->an->selinv;
  double* dd = diag ? (host ? P.d_diag.p : diag) : nullptr;
  double* dv = vals ? (host ? P.d_vals.p : vals) : nullptr;
  return timed_call(sv, [&]() -> int {
    { const int rc = enqueue_selinv(sv, dd, dv); if (rc != B200LDLT_SUCCESS) return rc; }
    if (host && diag) CU(cudaMemcpyAsync(diag, dd, (size_t)sv->n * sizeof(double), cudaMemcpyDeviceToHost, sv->stream));
    if (host && vals) CU(cudaMemcpyAsync(vals, dv, (size_t)sv->nnz * sizeof(double), cudaMemcpyDeviceToHost, sv->stream));
    return B200LDLT_SUCCESS;
  });
}

// ---- error analysis and condition estimation (b200ldlt_error_analysis, b200ldlt_condest) -------------------------------
// The call's state (EaPlan): |A| by rows from S.u_row / S.u_col at the first call after an analysis -- both triangles of
// the unique entries by a counting sort on the column, then a stable one on the row, so each row's columns ascend --
// and the buffers for nrhs right-hand sides and estimator blocks of `width` columns (0: no estimator), grown as needed.
static int ea_state(Solver* sv, int nrhs, int width) {
  Analysis& A = *sv->an;
  cudaStream_t st = sv->stream;
  const int n = sv->n;
  if (!A.ea) {
    const Symbolic& S = A.S;
    std::unique_ptr<EaPlan> P(new EaPlan());
    std::vector<int> er, ec, eu;
    er.reserve(2 * S.nnz_u); ec.reserve(2 * S.nnz_u); eu.reserve(2 * S.nnz_u);
    for (int64_t u = 0; u < S.nnz_u; ++u) {
      er.push_back(S.u_row[u]); ec.push_back(S.u_col[u]); eu.push_back((int)u);
      if (S.u_row[u] != S.u_col[u]) { er.push_back(S.u_col[u]); ec.push_back(S.u_row[u]); eu.push_back((int)u); }
    }
    const size_t m = er.size();
    std::vector<int> cptr(n + 1, 0), rptr(n + 1, 0);
    for (size_t e = 0; e < m; ++e) { cptr[ec[e] + 1]++; rptr[er[e] + 1]++; }
    for (int i = 0; i < n; ++i) { cptr[i + 1] += cptr[i]; rptr[i + 1] += rptr[i]; }
    std::vector<int> byc(m), col(m), uid(m);
    std::vector<int> pos(cptr.begin(), cptr.end() - 1);
    for (size_t e = 0; e < m; ++e) byc[pos[ec[e]]++] = (int)e;
    pos.assign(rptr.begin(), rptr.end() - 1);
    for (const int e : byc) { const int k = pos[er[e]]++; col[k] = ec[e]; uid[k] = eu[e]; }
    CU(P->d_ptr.upload(rptr, st));
    CU(P->d_col.upload(col, st));
    CU(P->d_uid.upload(uid, st));
    CU(P->d_uval.alloc(std::max<int64_t>(S.nnz_u, 1)));
    CU(P->d_amax.alloc(n));
    CU(P->d_res.alloc(MS_NB_MAX));
    CU(P->d_part.alloc((size_t)MS_NB_MAX * ea_parts(n)));
    CU(P->d_cnt.alloc(MS_NB_MAX));
    CU(cudaMemsetAsync(P->d_cnt.p, 0, MS_NB_MAX * sizeof(unsigned), st));
    CU(cudaStreamSynchronize(st));
    A.ea = std::move(P);
  }
  EaPlan& P = *A.ea;
  if (P.d_nrm.n < (size_t)EA_NRM * nrhs + 1) CU(P.d_nrm.alloc((size_t)EA_NRM * nrhs + 1));
  if (P.d_rs.n < (size_t)2 * n * nrhs) CU(P.d_rs.alloc((size_t)2 * n * nrhs));
  if (P.d_v.n < (size_t)n * width) { CU(P.d_v.alloc((size_t)n * width)); CU(P.d_xi.alloc((size_t)n * width)); }
  return B200LDLT_SUCCESS;
}

// One run of Higham's 1-norm estimator, exactly as LAPACK dlacn2 runs it, for ||B||_1 with B v = w o (M v) and
// B^T v = M (w o v) (w == nullptr: B = M).  jump is dlacn2's ISAVE(1) for the product in flight (0: finished).
struct EaEst {
  int xi = 0;                     // its column of the sign vectors
  const double* w = nullptr;
  int jump = 1, iter = 0, j = 0, nprod = 0;
  double est = 0.0;
};

// dlacn2's decision after the product of T's step, from the reductions R of that product
static void ea_decide(EaEst& T, const EaRes& R, int n) {
  ++T.nprod;
  const int jmax = R.jmax < n ? R.jmax : 0;   // (a product without a number in it: IDAMAX's 1)
  switch (T.jump) {
    case 1:                               // B x, x = e/n
      T.est = R.l1;
      T.jump = n == 1 ? 0 : 2;
      break;
    case 2:                               // B^T xi
      T.j = jmax; T.iter = 2; T.jump = 3;
      break;
    case 3: {                             // B e_j: stop on a repeated sign vector or no increase
      const double old = T.est;
      T.est = R.l1;
      T.jump = (R.changes == 0 || T.est <= old) ? 5 : 4;
      break;
    }
    case 4:                               // B^T xi: continue while z[jlast] != max |z| and iter < 5
      T.j = jmax;
      if (R.zjl != R.zmax && T.iter < 5) { ++T.iter; T.jump = 3; } else T.jump = 5;
      break;
    default: {                            // B x, x the alternating vector
      const double t = 2.0 * (R.l1 / (3.0 * (double)n));
      if (t > T.est) T.est = t;
      T.jump = 0;
    }
  }
}

// The estimators E[0..ne) in lockstep (ne <= W.width): per step, the inputs of the unfinished ones (k_ea_prep), ONE job-0
// solve of that many columns through W, their reductions (k_ea_post), one D2H of them and dlacn2's decisions on the host.
// Launches per step: 2 + job 0's.  Each column runs the arithmetic of a single-column solve, so an estimator's results do
// not depend on the others of its block.
static int run_estimators(Solver* sv, SweepState& W, EaEst* E, int ne) {
  static const int kMode[6] = {0, 0, 2, 1, 2, 3};   // the input of each jump: e/n, xi, e_j, xi, alternating
  EaPlan& P = *sv->an->ea;
  cudaStream_t st = sv->stream;
  const int n = sv->n;
  for (;;) {
    EaStep step;
    EaEst* act[MS_NB_MAX];
    int na = 0;
    for (int e = 0; e < ne; ++e) {
      EaEst& T = E[e];
      if (!T.jump) continue;
      const bool k2 = T.jump == 2 || T.jump == 4;
      step.s[na] = EaSlot{k2 ? T.w : nullptr, k2 ? nullptr : T.w, T.xi, kMode[T.jump], T.j, T.j, k2 ? 2 : 1};
      act[na++] = &T;
    }
    if (na == 0) return B200LDLT_SUCCESS;
    k_ea_prep<<<dim3(cdiv(n, EA_THREADS), na), EA_THREADS, 0, st>>>(n, step, P.d_xi.p, P.d_v.p);
    ++sv->launches;
    { const int rc = enqueue_solve(sv, W, 0, P.d_v.p, P.d_v.p, na); if (rc != B200LDLT_SUCCESS) return rc; }
    k_ea_post<<<dim3(ea_parts(n), na), EA_THREADS, 0, st>>>(n, step, P.d_v.p, P.d_xi.p, P.d_part.p, P.d_cnt.p, P.d_res.p);
    ++sv->launches;
    CU(cudaGetLastError());
    EaRes R[MS_NB_MAX];
    CU(cudaMemcpyAsync(R, P.d_res.p, na * sizeof(EaRes), cudaMemcpyDeviceToHost, st));
    CU(cudaStreamSynchronize(st));
    for (int a = 0; a < na; ++a) ea_decide(*act[a], R[a], n);
  }
}

// k_sum_dups into the call's unique values, then the row pass for nrhs columns of d_b / d_x (nrhs = 0: only ||A|| and
// the row maxima) into P.d_nrm, which is cleared first
static int enqueue_ea_rows(Solver* sv, int nrhs, const double* d_b, const double* d_x) {
  const Analysis& A = *sv->an;
  EaPlan& P = *A.ea;
  cudaStream_t st = sv->stream;
  const int n = sv->n;
  const long long nu = A.S.nnz_u;
  CU(cudaMemsetAsync(P.d_nrm.p, 0, ((size_t)EA_NRM * nrhs + 1) * sizeof(unsigned long long), st));
  k_sum_dups<<<cdiv(nu, 256), 256, 0, st>>>(nu, A.d_useg_ptr.p, A.d_useg_src.p, sv->d_vals.p, P.d_uval.p);
  const unsigned g = std::min<unsigned>(cdiv(n, EA_WARPS), EA_ROW_CTAS);
  k_ea_rows<false><<<dim3(g, std::max(nrhs, 1)), EA_THREADS, 0, st>>>(n, nrhs, P.d_ptr.p, P.d_col.p, P.d_uid.p, P.d_uval.p,
                                                                      d_b, d_x, P.d_rs.p, P.d_amax.p, P.d_nrm.p, RfCols{},
                                                                      nullptr);
  sv->launches += 2;
  CU(cudaGetLastError());
  return B200LDLT_SUCCESS;
}

static inline double ea_val(unsigned long long b) { double v; memcpy(&v, &b, sizeof(v)); return v; }

// b200ldlt_error_analysis (host == true: b and x in host memory) / _device
static int error_analysis(Solver* sv, int nrhs, const double* b, const double* x, int cond, b200ldlt_errors* out,
                          bool host) {
  const char* bad = nrhs < 0 ? "nrhs must be >= 0" : cond != 0 && cond != 1 ? "cond must be 0 or 1"
                    : nrhs > 0 && (!b || !x || !out) ? "NULL argument" : nullptr;
  if (bad) { sv->err = std::string("error_analysis: ") + bad; return B200LDLT_FATAL_ERROR; }
  { const int rc = factors_state(sv, "error_analysis"); if (rc != B200LDLT_SUCCESS) return rc; }
  if (nrhs == 0) return no_columns(sv);
  Analysis& A = *sv->an;
  const int n = sv->n;
  const size_t nb = (size_t)n * nrhs;
  // kept singular factors: M is no inverse of A, no estimator runs
  const bool estimate = cond == 1 && A.zpos.empty();
  const bool blocked = estimate && block_solve_state(sv);
  SweepState& W = blocked ? *A.blk : A.sweep;
  { const int rc = ea_state(sv, nrhs, estimate ? W.width : 0); if (rc != B200LDLT_SUCCESS) return rc; }
  EaPlan& P = *A.ea;
  cudaStream_t st = sv->stream;
  std::vector<unsigned long long> nrm((size_t)EA_NRM * nrhs + 1);
  auto at = [&](int c, int k) { return ea_val(nrm[(size_t)EA_NRM * c + k]); };
  std::vector<double> est(2 * (size_t)nrhs, 0.0);
  std::vector<int> nprod(nrhs, 0);
  auto enqueue = [&](const double* d_b, const double* d_x) -> int {
    { const int rc = enqueue_ea_rows(sv, nrhs, d_b, d_x); if (rc != B200LDLT_SUCCESS) return rc; }
    k_ea_class<false><<<dim3(cdiv(n, EA_THREADS), nrhs), EA_THREADS, 0, st>>>(n, d_b, P.d_amax.p, P.d_rs.p, P.d_nrm.p,
                                                                              RfCols{}, nullptr);
    ++sv->launches;
    CU(cudaGetLastError());
    CU(cudaMemcpyAsync(nrm.data(), P.d_nrm.p, nrm.size() * sizeof(unsigned long long), cudaMemcpyDeviceToHost, st));
    if (!estimate) return B200LDLT_SUCCESS;
    CU(cudaStreamSynchronize(st));
    // the estimators of cond1 (weights w1, on I1) and cond2 (w2, on I2) of each column with x != 0 and its set non-empty:
    // blocked, those of up to width / 2 columns in lockstep, else one by one through the single-column state
    return for_blocks(nrhs, blocked ? W.width / 2 : 1, [&](int c0, int w) -> int {
      EaEst E[MS_NB_MAX];
      int slot[MS_NB_MAX], ne = 0;
      for (int c = c0; c < c0 + w; ++c) {
        if (at(c, EA_X) == 0.0) continue;
        const long long n2 = (long long)nrm[(size_t)EA_NRM * c + EA_NI2];
        for (int k = 0; k < 2; ++k) {
          if ((k == 0 ? n - n2 : n2) == 0) continue;
          E[ne].xi = blocked ? ne : 0;
          E[ne].w = P.d_rs.p + (size_t)(2 * c + k) * n;
          slot[ne++] = 2 * c + k;
        }
      }
      if (blocked) {
        const int rc = run_estimators(sv, W, E, ne);
        if (rc != B200LDLT_SUCCESS) return rc;
      } else {
        for (int e = 0; e < ne; ++e) { const int rc = run_estimators(sv, W, E + e, 1); if (rc != B200LDLT_SUCCESS) return rc; }
      }
      for (int e = 0; e < ne; ++e) { est[slot[e]] = E[e].est; nprod[slot[e] / 2] += E[e].nprod; }
      return B200LDLT_SUCCESS;
    });
  };
  const int rc = host ? staged_call(sv, b, nb, nullptr, 0, [&](double* d) { return enqueue(d, d + nb); }, 0, 0, x, nb)
                      : timed_call(sv, [&] { return enqueue(b, x); });
  if (rc != B200LDLT_SUCCESS) return rc;
  const double inf = INFINITY, anorm = ea_val(nrm[(size_t)EA_NRM * nrhs]);
  for (int c = 0; c < nrhs; ++c) {
    b200ldlt_errors& o = out[c];
    o.anorm = anorm;
    o.xnorm = at(c, EA_X);
    o.rnorm = at(c, EA_R);
    o.omega1 = at(c, EA_W1);
    o.omega2 = at(c, EA_W2);
    o.n_i2 = (int)nrm[(size_t)EA_NRM * c + EA_NI2];
    o.nprod = nprod[c];
    if (cond == 0) {
      o.cond1 = o.cond2 = o.ferr = -1.0;
    } else if (!A.zpos.empty()) {
      o.cond1 = o.cond2 = o.ferr = inf;
    } else if (o.xnorm == 0.0) {
      o.cond1 = o.cond2 = o.ferr = at(c, EA_B) == 0.0 ? 0.0 : inf;
    } else {
      o.cond1 = est[2 * (size_t)c] / o.xnorm;
      o.cond2 = est[2 * (size_t)c + 1] / o.xnorm;
      o.ferr = o.omega1 * o.cond1 + o.omega2 * o.cond2;
    }
  }
  return B200LDLT_SUCCESS;
}

// ---- iterative refinement (b200ldlt_solve_refined) -------------------------------------------------------------------
// One column's state: the omegas of its last accepted iterate, its result fields and the residuals evaluated
struct RfCol {
  double first = 0.0, om1 = 0.0, om2 = 0.0;
  int steps = 0, status = -1, nres = 0;
};

// The stopping rule of include/b200ldlt.h after the omegas of iterate k: 0 = go on to x_{k+1} (C now describes x_k),
// 1 = x_k is the result, 2 = x_{k-1} is the result (C still describes it)
static int rf_rule(RfCol& C, double om1, double om2, int k, int max_steps, double tol) {
  const double om = om1 + om2, prev = C.om1 + C.om2;
  C.nres = k + 1;
  if (k == 0) C.first = om;
  auto take = [&](int status) { C.om1 = om1; C.om2 = om2; C.steps = k; C.status = status; return status < 0 ? 0 : 1; };
  auto back = [&](int status) { C.steps = k - 1; C.status = status; return 2; };
  if (!std::isfinite(om)) return k == 0 ? take(3) : back(3);
  if (om <= tol) return take(0);
  if (k >= 1 && om > prev / 2) return om < prev ? take(1) : back(1);
  if (k == max_steps) return take(2);
  return take(-1);
}

// b200ldlt_solve_refined (host == true: b and x in host memory) / _device
static int solve_refined(Solver* sv, int nrhs, const double* b, double* x, int max_steps, double tol,
                         b200ldlt_refined* out, bool host) {
  const char* bad = nrhs < 0 ? "nrhs must be >= 0" : max_steps < 0 ? "max_steps must be >= 0"
                    : !(tol >= 0.0) ? "tol must be >= 0" : nrhs > 0 && (!b || !x || !out) ? "NULL argument"
                    : nrhs > 0 && b == x ? "x must not be b" : nullptr;
  if (bad) { sv->err = std::string("solve_refined: ") + bad; return B200LDLT_FATAL_ERROR; }
  { const int rc = factors_state(sv, "solve_refined"); if (rc != B200LDLT_SUCCESS) return rc; }
  if (nrhs == 0) return no_columns(sv);
  Analysis& A = *sv->an;
  const int n = sv->n;
  const size_t nb = (size_t)n * nrhs;
  const bool blocked = nrhs > 1 && block_solve_state(sv);
  SweepState& W = blocked ? *A.blk : A.sweep;
  const int width = blocked ? W.width : 1;
  { const int rc = ea_state(sv, width, 0); if (rc != B200LDLT_SUCCESS) return rc; }
  EaPlan& P = *A.ea;
  if (P.d_rf_d.n < (size_t)n * width) { CU(P.d_rf_d.alloc((size_t)n * width)); CU(P.d_rf_old.alloc((size_t)n * width)); }
  cudaStream_t st = sv->stream;
  std::vector<RfCol> R(nrhs);
  // x_held: d_x already holds b (the host staging)
  auto enqueue = [&](const double* d_b, double* d_x, bool x_held) -> int {
    const long long nu = A.S.nnz_u;
    k_sum_dups<<<cdiv(nu, 256), 256, 0, st>>>(nu, A.d_useg_ptr.p, A.d_useg_src.p, sv->d_vals.p, P.d_uval.p);
    ++sv->launches;
    const unsigned g = std::min<unsigned>(cdiv(n, EA_WARPS), EA_ROW_CTAS);
    return for_blocks(nrhs, width, [&](int c0, int w) -> int {
      const double* bb = d_b + (size_t)c0 * n;
      double* xb = d_x + (size_t)c0 * n;
      if (!x_held) CU(cudaMemcpyAsync(xb, bb, (size_t)n * w * sizeof(double), cudaMemcpyDeviceToDevice, st));
      { const int rc = enqueue_solve(sv, W, 0, xb, xb, w); if (rc != B200LDLT_SUCCESS) return rc; }
      RfCols act;
      int na = w;
      for (int s = 0; s < w; ++s) act.c[s] = s;
      std::vector<unsigned long long> nrm((size_t)EA_NRM * w + 1);
      for (int k = 0;; ++k) {
        // r (double-double) of the unfinished columns into the slots, s and the omegas; one D2H of the maxima
        CU(cudaMemsetAsync(P.d_nrm.p, 0, ((size_t)EA_NRM * na + 1) * sizeof(unsigned long long), st));
        k_ea_rows<true><<<dim3(g, na), EA_THREADS, 0, st>>>(n, na, P.d_ptr.p, P.d_col.p, P.d_uid.p, P.d_uval.p, bb, xb,
                                                            P.d_rs.p, P.d_amax.p, P.d_nrm.p, act, P.d_rf_d.p);
        k_ea_class<true><<<dim3(cdiv(n, EA_THREADS), na), EA_THREADS, 0, st>>>(n, bb, P.d_amax.p, P.d_rs.p, P.d_nrm.p, act,
                                                                               P.d_rf_d.p);
        sv->launches += 2;
        CU(cudaGetLastError());
        CU(cudaMemcpyAsync(nrm.data(), P.d_nrm.p, (size_t)EA_NRM * na * sizeof(unsigned long long), cudaMemcpyDeviceToHost, st));
        CU(cudaStreamSynchronize(st));
        // the rule per column; a finished column that returns x_{k-1} gets it back, the others' r close up
        RfCols next;
        int nn = 0;
        for (int s = 0; s < na; ++s) {
          const int c = act.c[s];
          const int v = rf_rule(R[c0 + c], ea_val(nrm[(size_t)EA_NRM * s + EA_W1]), ea_val(nrm[(size_t)EA_NRM * s + EA_W2]), k,
                                max_steps, tol);
          if (v == 2)
            CU(cudaMemcpyAsync(xb + (size_t)c * n, P.d_rf_old.p + (size_t)c * n, (size_t)n * sizeof(double),
                               cudaMemcpyDeviceToDevice, st));
          if (v != 0) continue;
          if (nn != s)
            CU(cudaMemcpyAsync(P.d_rf_d.p + (size_t)nn * n, P.d_rf_d.p + (size_t)s * n, (size_t)n * sizeof(double),
                               cudaMemcpyDeviceToDevice, st));
          next.c[nn++] = c;
        }
        if (nn == 0) return B200LDLT_SUCCESS;
        // d = job 0 on the slots, then x_{k+1} = x_k (+) d with x_k kept for a rollback
        { const int rc = enqueue_solve(sv, W, 0, P.d_rf_d.p, P.d_rf_d.p, nn); if (rc != B200LDLT_SUCCESS) return rc; }
        k_rf_update<<<dim3(cdiv(n, EA_THREADS), nn), EA_THREADS, 0, st>>>(n, next, P.d_rf_d.p, xb, P.d_rf_old.p);
        ++sv->launches;
        CU(cudaGetLastError());
        act = next;
        na = nn;
      }
    });
  };
  int rc;
  if (host) {
    // the staging holds x (b on entry, the refined x on exit) and then a copy of b
    rc = staged_call(sv, b, nb, x, nb, [&](double* d) -> int {
      CU(cudaMemcpyAsync(d + nb, d, nb * sizeof(double), cudaMemcpyDeviceToDevice, st));
      return enqueue(d + nb, d, true);
    }, 2 * nb);
  } else {
    rc = timed_call(sv, [&] { return enqueue(b, x, false); });
  }
  if (rc != B200LDLT_SUCCESS) return rc;
  for (int c = 0; c < nrhs; ++c)
    out[c] = b200ldlt_refined{R[c].first, R[c].om1, R[c].om2, R[c].steps, R[c].status, R[c].nres};
  return B200LDLT_SUCCESS;
}

// ---- FGMRES preconditioned by the factors (b200ldlt_solve_gmres) -----------------------------------------------------
// One column's cycle on the host: beta, g, the Givens rotations and the rotated Hessenberg columns (rr[j * GM_RESTART_MAX
// + i] = row i of column j), the steps kept (m) and whether it still steps.  The arithmetic is the header's, one
// rounded double operation per written operation (the x86-64 host build has no FMA to contract into).
struct GmCol {
  double beta = 0.0;
  double cs[GM_RESTART_MAX], sn[GM_RESTART_MAX], g[GM_RESTART_MAX + 1];
  std::vector<double> rr = std::vector<double>((size_t)GM_RESTART_MAX * GM_RESTART_MAX);
  int m = 0, iters = 0;
  bool on = false;
};

// Arnoldi step j of G with its Hessenberg column h[0 .. j + 1]: the rotations, the stopping decision and G.m
static void gm_step(GmCol& G, double* h, int j, int restart, double inner_tol) {
  ++G.iters;
  for (int i = 0; i < j; ++i) {
    const double t = G.cs[i] * h[i] + G.sn[i] * h[i + 1];
    h[i + 1] = G.cs[i] * h[i + 1] - G.sn[i] * h[i];
    h[i] = t;
  }
  const double a = h[j], b = h[j + 1];
  const double rho = std::sqrt(a * a + b * b);
  bool finite = std::isfinite(rho) && rho != 0.0;
  for (int i = 0; i <= j + 1; ++i) finite = finite && std::isfinite(h[i]);
  if (!finite) { G.on = false; return; }   // the step is dropped: G.m stays j
  G.cs[j] = a / rho;
  G.sn[j] = b / rho;
  double* r = G.rr.data() + (size_t)j * GM_RESTART_MAX;
  for (int i = 0; i < j; ++i) r[i] = h[i];
  r[j] = rho;
  G.g[j + 1] = -(G.sn[j] * G.g[j]);
  G.g[j] = G.cs[j] * G.g[j];
  G.m = j + 1;
  G.on = !(b == 0.0 || std::fabs(G.g[j + 1]) <= inner_tol * G.beta || G.m == restart);
}

// y = R^-1 g over G's m kept steps, back substitution with the row's terms in ascending column order
static void gm_solve(const GmCol& G, double* y) {
  for (int i = G.m - 1; i >= 0; --i) {
    double t = G.g[i];
    for (int l = i + 1; l < G.m; ++l) t = t - G.rr[(size_t)l * GM_RESTART_MAX + i] * y[l];
    y[i] = t / G.rr[(size_t)i * GM_RESTART_MAX + i];
  }
}

// b200ldlt_solve_gmres (host == true: b, x and vals in host memory) / _device
static int solve_gmres(Solver* sv, int nrhs, const double* b, double* x, const double* vals, int restart, int max_cycles,
                       double tol, double inner_tol, b200ldlt_gmres* out, bool host) {
  const char* bad = nrhs < 0 ? "nrhs must be >= 0" : restart < 1 || restart > GM_RESTART_MAX ? "restart must be 1..64"
                    : max_cycles < 0 ? "max_cycles must be >= 0" : !(tol >= 0.0) ? "tol must be >= 0"
                    : !(inner_tol >= 0.0) ? "inner_tol must be >= 0" : nrhs > 0 && (!b || !x || !out) ? "NULL argument"
                    : nrhs > 0 && b == x ? "x must not be b" : nullptr;
  if (bad) { sv->err = std::string("solve_gmres: ") + bad; return B200LDLT_FATAL_ERROR; }
  { const int rc = factors_state(sv, "solve_gmres"); if (rc != B200LDLT_SUCCESS) return rc; }
  if (nrhs == 0) return no_columns(sv);
  Analysis& A = *sv->an;
  const int n = sv->n;
  const size_t nb = (size_t)n * nrhs, nv = (size_t)sv->nnz;
  const bool blocked = nrhs > 1 && block_solve_state(sv);
  SweepState& W = blocked ? *A.blk : A.sweep;
  const int width = blocked ? W.width : 1;
  { const int rc = ea_state(sv, width, 0); if (rc != B200LDLT_SUCCESS) return rc; }
  EaPlan& P = *A.ea;
  cudaStream_t st = sv->stream;
  const int parts = ea_parts(n);
  if (P.d_rf_d.n < (size_t)n * width) { CU(P.d_rf_d.alloc((size_t)n * width)); CU(P.d_rf_old.alloc((size_t)n * width)); }
  if (!P.d_gm_h.n) {
    CU(P.d_gm_h.alloc((size_t)MS_NB_MAX * GM_H));
    CU(P.d_gm_y.alloc((size_t)MS_NB_MAX * GM_RESTART_MAX));
    CU(P.d_gm_part.alloc((size_t)MS_NB_MAX * GM_Q * parts));
    CU(P.d_gm_cnt.alloc((size_t)MS_NB_MAX * GM_Q));
    CU(cudaMemsetAsync(P.d_gm_cnt.p, 0, (size_t)MS_NB_MAX * GM_Q * sizeof(unsigned), st));
  }
  const size_t kv = (size_t)(2 * restart + 1) * n;   // V (restart + 1 vectors) and Z (restart) of one column
  if (P.d_gm_kv.n < kv * width && P.d_gm_kv.alloc(kv * width) != cudaSuccess) {
    cudaGetLastError();
    sv->err = "solve_gmres: cannot allocate the Krylov vectors (" + std::to_string(8.0 * kv * width / 1e6) + " MB)";
    return B200LDLT_FATAL_ERROR;
  }
  double* const gkv = P.d_gm_kv.p;   // the Krylov vectors of column c at gkv + c gld, its Hessenberg column at ghb + c GM_H
  double* const ghb = P.d_gm_h.p;
  const long long gld = (long long)kv;
  std::vector<RfCol> R(nrhs);
  std::vector<int> iters(nrhs, 0);
  std::vector<GmCol> G(width);
  std::vector<double> hh((size_t)width * GM_H), yy((size_t)MS_NB_MAX * GM_RESTART_MAX);
  std::vector<unsigned long long> nrm((size_t)EA_NRM * width + 1);
  // x_held: d_x already holds b (the host staging); d_op: the caller's values of A_op, or the factored ones
  auto enqueue = [&](const double* d_b, double* d_x, const double* d_op, bool x_held) -> int {
    const long long nu = A.S.nnz_u;
    k_sum_dups<<<cdiv(nu, 256), 256, 0, st>>>(nu, A.d_useg_ptr.p, A.d_useg_src.p, d_op, P.d_uval.p);
    ++sv->launches;
    const unsigned g = std::min<unsigned>(cdiv(n, EA_WARPS), EA_ROW_CTAS);
    return for_blocks(nrhs, width, [&](int c0, int w) -> int {
      const double* bb = d_b + (size_t)c0 * n;
      double* xb = d_x + (size_t)c0 * n;
      if (!x_held) CU(cudaMemcpyAsync(xb, bb, (size_t)n * w * sizeof(double), cudaMemcpyDeviceToDevice, st));
      { const int rc = enqueue_solve(sv, W, 0, xb, xb, w); if (rc != B200LDLT_SUCCESS) return rc; }
      RfCols act;
      int na = w;
      for (int s = 0; s < w; ++s) act.c[s] = s;
      for (int k = 0;; ++k) {
        // r (double-double) of the unfinished columns into the slots, s, the omegas and beta^2 = ||r||^2; one D2H each
        CU(cudaMemsetAsync(P.d_nrm.p, 0, ((size_t)EA_NRM * na + 1) * sizeof(unsigned long long), st));
        k_ea_rows<true><<<dim3(g, na), EA_THREADS, 0, st>>>(n, na, P.d_ptr.p, P.d_col.p, P.d_uid.p, P.d_uval.p, bb, xb,
                                                            P.d_rs.p, P.d_amax.p, P.d_nrm.p, act, P.d_rf_d.p);
        k_ea_class<true><<<dim3(cdiv(n, EA_THREADS), na), EA_THREADS, 0, st>>>(n, bb, P.d_amax.p, P.d_rs.p, P.d_nrm.p, act,
                                                                               P.d_rf_d.p);
        GmSlots sl;   // the residuals in the solve slots
        for (int s = 0; s < na; ++s) { sl.v[s] = s; sl.h[s] = act.c[s]; }
        k_gm_update<true><<<dim3(parts, na), EA_THREADS, 0, st>>>(n, -1, 0, sl, P.d_rf_d.p, n, ghb, P.d_gm_part.p, P.d_gm_cnt.p);
        sv->launches += 3;
        CU(cudaGetLastError());
        CU(cudaMemcpyAsync(nrm.data(), P.d_nrm.p, (size_t)EA_NRM * na * sizeof(unsigned long long), cudaMemcpyDeviceToHost, st));
        CU(cudaMemcpyAsync(hh.data(), P.d_gm_h.p, (size_t)GM_H * w * sizeof(double), cudaMemcpyDeviceToHost, st));
        CU(cudaStreamSynchronize(st));
        // the rule per column; a finished column that returns x_{k-1} gets it back, the others' r close up
        RfCols next;
        int nn = 0;
        for (int s = 0; s < na; ++s) {
          const int c = act.c[s];
          const int v = rf_rule(R[c0 + c], ea_val(nrm[(size_t)EA_NRM * s + EA_W1]), ea_val(nrm[(size_t)EA_NRM * s + EA_W2]), k,
                                max_cycles, tol);
          if (v == 2)
            CU(cudaMemcpyAsync(xb + (size_t)c * n, P.d_rf_old.p + (size_t)c * n, (size_t)n * sizeof(double),
                               cudaMemcpyDeviceToDevice, st));
          if (v != 0) continue;
          if (nn != s)
            CU(cudaMemcpyAsync(P.d_rf_d.p + (size_t)nn * n, P.d_rf_d.p + (size_t)s * n, (size_t)n * sizeof(double),
                               cudaMemcpyDeviceToDevice, st));
          next.c[nn++] = c;
        }
        if (nn == 0) return B200LDLT_SUCCESS;
        // one cycle: v_0 = r / beta into the slots and V, then the Arnoldi steps of the columns still stepping in lockstep
        int slot[MS_NB_MAX];
        for (int s = 0; s < nn; ++s) {
          const int c = next.c[s];
          sl.v[s] = sl.h[s] = c;
          GmCol& C = G[c];
          C.beta = std::sqrt(hh[(size_t)GM_H * c + GM_Q - 1]);
          C.g[0] = C.beta;
          C.m = 0;
          C.iters = 0;
          C.on = std::isfinite(C.beta) && C.beta != 0.0;
          slot[c] = s;
        }
        k_gm_scale<<<dim3(cdiv(n, EA_THREADS), nn), EA_THREADS, 0, st>>>(n, -1, 0, sl, gkv, gld, ghb, P.d_rf_d.p);
        ++sv->launches;
        CU(cudaGetLastError());
        for (int j = 0;; ++j) {
          GmSlots sa;
          int on[MS_NB_MAX], ns = 0;
          for (int s = 0; s < nn; ++s) {
            const int c = next.c[s];
            if (!G[c].on) continue;
            if (slot[c] != ns)
              CU(cudaMemcpyAsync(P.d_rf_d.p + (size_t)ns * n, P.d_rf_d.p + (size_t)slot[c] * n, (size_t)n * sizeof(double),
                                 cudaMemcpyDeviceToDevice, st));
            slot[c] = ns;
            sa.v[ns] = sa.h[ns] = c;
            on[ns++] = c;
          }
          if (ns == 0) break;
          // z_j = job 0 on v_j, w = A_op z_j, CGS2 against v_0 .. v_j, ||w||, v_{j+1} = w / ||w||
          { const int rc = enqueue_solve(sv, W, 0, P.d_rf_d.p, P.d_rf_d.p, ns); if (rc != B200LDLT_SUCCESS) return rc; }
          k_gm_apply<<<dim3(g, ns), EA_THREADS, 0, st>>>(n, restart, j, P.d_ptr.p, P.d_col.p, P.d_uid.p, P.d_uval.p,
                                                         P.d_rf_d.p, sa, gkv, gld, ghb);
          for (int pass = 0; pass < 2; ++pass) {
            k_gm_dot<<<dim3(parts, ns, j + 1), EA_THREADS, 0, st>>>(n, j, pass * GM_Q, sa, gkv, gld, ghb, P.d_gm_part.p, P.d_gm_cnt.p);
            if (pass == 0) k_gm_update<false><<<dim3(parts, ns), EA_THREADS, 0, st>>>(n, j, 0, sa, gkv, gld, ghb, P.d_gm_part.p, P.d_gm_cnt.p);
            else k_gm_update<true><<<dim3(parts, ns), EA_THREADS, 0, st>>>(n, j, GM_Q, sa, gkv, gld, ghb, P.d_gm_part.p, P.d_gm_cnt.p);
          }
          k_gm_scale<<<dim3(cdiv(n, EA_THREADS), ns), EA_THREADS, 0, st>>>(n, j, GM_Q, sa, gkv, gld, ghb, P.d_rf_d.p);
          sv->launches += 6;
          CU(cudaGetLastError());
          CU(cudaMemcpyAsync(hh.data(), P.d_gm_h.p, (size_t)GM_H * w * sizeof(double), cudaMemcpyDeviceToHost, st));
          CU(cudaStreamSynchronize(st));
          for (int s = 0; s < ns; ++s) {
            const double* hc = hh.data() + (size_t)GM_H * on[s];
            double h[GM_RESTART_MAX + 1];
            for (int i = 0; i <= j; ++i) h[i] = hc[i] + hc[GM_Q + i];
            h[j + 1] = std::sqrt(hc[GM_Q + GM_Q - 1]);
            gm_step(G[on[s]], h, j, restart, inner_tol);
          }
        }
        // x_{k+1} = x_k (+) Z y, x_k kept for a rollback
        GmFinal f;
        for (int s = 0; s < nn; ++s) {
          const int c = next.c[s];
          f.c[s] = c;
          f.m[s] = G[c].m;
          iters[c0 + c] += G[c].iters;
          gm_solve(G[c], yy.data() + (size_t)s * GM_RESTART_MAX);
        }
        CU(cudaMemcpyAsync(P.d_gm_y.p, yy.data(), (size_t)nn * GM_RESTART_MAX * sizeof(double), cudaMemcpyHostToDevice, st));
        k_gm_final<<<dim3(cdiv(n, EA_THREADS), nn), EA_THREADS, 0, st>>>(n, restart, sl, gkv, gld, ghb, f, P.d_gm_y.p, xb, P.d_rf_old.p);
        ++sv->launches;
        CU(cudaGetLastError());
        act = next;
        na = nn;
      }
    });
  };
  int rc;
  if (host) {
    // the staging holds x (b on entry, the solution on exit), the caller's values if any, then a copy of b
    const size_t nin2 = vals ? nv : 0;
    rc = staged_call(sv, b, nb, x, nb, [&](double* d) -> int {
      CU(cudaMemcpyAsync(d + nb + nin2, d, nb * sizeof(double), cudaMemcpyDeviceToDevice, st));
      return enqueue(d + nb + nin2, d, vals ? d + nb : sv->d_vals.p, true);
    }, 2 * nb + nin2, 0, vals, nin2);
  } else {
    rc = timed_call(sv, [&] { return enqueue(b, x, vals ? vals : sv->d_vals.p, false); });
  }
  if (rc != B200LDLT_SUCCESS) return rc;
  for (int c = 0; c < nrhs; ++c)
    out[c] = b200ldlt_gmres{R[c].first, R[c].om1, R[c].om2, R[c].steps, iters[c], R[c].status, R[c].nres};
  return B200LDLT_SUCCESS;
}

// b200ldlt_condest: ||A||_1 from the row pass, est ||M||_1 by one estimator through the single-column state
static int condest(Solver* sv, double* kappa1, double* anorm1, double* ainv1, int* nprod) {
  if (!kappa1) { sv->err = "condest: NULL kappa1"; return B200LDLT_FATAL_ERROR; }
  { const int rc = factors_state(sv, "condest"); if (rc != B200LDLT_SUCCESS) return rc; }
  Analysis& A = *sv->an;
  const bool estimate = A.zpos.empty();
  { const int rc = ea_state(sv, 0, estimate ? 1 : 0); if (rc != B200LDLT_SUCCESS) return rc; }
  EaEst E;
  unsigned long long an = 0;
  const int rc = timed_call(sv, [&]() -> int {
    { const int rc2 = enqueue_ea_rows(sv, 0, nullptr, nullptr); if (rc2 != B200LDLT_SUCCESS) return rc2; }
    if (estimate) { const int rc2 = run_estimators(sv, A.sweep, &E, 1); if (rc2 != B200LDLT_SUCCESS) return rc2; }
    CU(cudaMemcpyAsync(&an, A.ea->d_nrm.p, sizeof(an), cudaMemcpyDeviceToHost, sv->stream));
    return B200LDLT_SUCCESS;
  });
  if (rc != B200LDLT_SUCCESS) return rc;
  const double anorm = ea_val(an), ainv = estimate ? E.est : INFINITY;
  *kappa1 = estimate ? anorm * ainv : INFINITY;
  if (anorm1) *anorm1 = anorm;
  if (ainv1) *ainv1 = ainv;
  if (nprod) *nprod = E.nprod;
  return B200LDLT_SUCCESS;
}
}  // namespace b200

extern "C" {

int b200ldlt_solve_device(b200ldlt_handle h, int nrhs, double* d_rhs) {
  Solver* sv = (Solver*)h;
  if (!sv) return B200LDLT_FATAL_ERROR;
  return solve_job(sv, 0, nrhs, d_rhs, false);
}

int b200ldlt_solve(b200ldlt_handle h, int nrhs, double* rhs) {
  Solver* sv = (Solver*)h;
  if (!sv) return B200LDLT_FATAL_ERROR;
  return solve_job(sv, 0, nrhs, rhs, true);
}

int b200ldlt_solve_partial(b200ldlt_handle h, int job, int nrhs, double* rhs) {
  Solver* sv = (Solver*)h;
  if (!sv) return B200LDLT_FATAL_ERROR;
  return solve_job(sv, job, nrhs, rhs, true);
}

int b200ldlt_solve_partial_device(b200ldlt_handle h, int job, int nrhs, double* d_rhs) {
  Solver* sv = (Solver*)h;
  if (!sv) return B200LDLT_FATAL_ERROR;
  return solve_job(sv, job, nrhs, d_rhs, false);
}

int b200ldlt_enquire_indef(b200ldlt_handle h, int* pivot_var, int* pivot_type, double* dinv2) {
  Solver* sv = (Solver*)h;
  if (!sv) return B200LDLT_FATAL_ERROR;
  { const int rc = factors_state(sv, "enquire_indef", true); if (rc != B200LDLT_SUCCESS) return rc; }
  const Analysis& A = *sv->an;
  cudaStream_t st = sv->stream;
  const int n = sv->n;
  std::vector<int> lperm(n), ptype(n);
  std::vector<double> dinv(n), doff(n);
  CU(cudaMemcpyAsync(lperm.data(), A.d_lperm.p, n * sizeof(int), cudaMemcpyDeviceToHost, st));
  CU(cudaMemcpyAsync(ptype.data(), A.d_ptype.p, n * sizeof(int), cudaMemcpyDeviceToHost, st));
  CU(cudaMemcpyAsync(dinv.data(), A.d_dinv.p, n * sizeof(double), cudaMemcpyDeviceToHost, st));
  CU(cudaMemcpyAsync(doff.data(), A.d_doff.p, n * sizeof(double), cudaMemcpyDeviceToHost, st));
  CU(cudaStreamSynchronize(st));
  const Symbolic& S = A.S;
  for (int s = 0; s < S.nsn; ++s)
    for (int p = S.sn_start[s]; p < S.sn_start[s + 1]; ++p) {
      // pivot t of front s holds the front's local column lperm[p]: permuted column sn_start[s] + lperm[p]
      if (pivot_var) pivot_var[p] = S.perm[S.sn_start[s] + lperm[p]];
      if (pivot_type) pivot_type[p] = ptype[p];
      if (dinv2) { dinv2[2 * (size_t)p] = dinv[p]; dinv2[2 * (size_t)p + 1] = ptype[p] == 2 ? doff[p] : 0.0; }
    }
  return B200LDLT_SUCCESS;
}

int b200ldlt_lmultiply_device(b200ldlt_handle h, int trans, int nrhs, const double* d_x, double* d_y) {
  Solver* sv = (Solver*)h;
  if (!sv) return B200LDLT_FATAL_ERROR;
  return lmultiply(sv, trans, nrhs, d_x, d_y, false);
}

int b200ldlt_lmultiply(b200ldlt_handle h, int trans, int nrhs, const double* x, double* y) {
  Solver* sv = (Solver*)h;
  if (!sv) return B200LDLT_FATAL_ERROR;
  return lmultiply(sv, trans, nrhs, x, y, true);
}

int b200ldlt_sparse_fwd_solve(b200ldlt_handle h, int nbi, const int* bindex, const double* b, int* nxi, int* xindex, double* x) {
  Solver* sv = (Solver*)h;
  if (!sv) return B200LDLT_FATAL_ERROR;
  return sparse_fwd(sv, nbi, bindex, b, true, nxi, xindex, x);
}

int b200ldlt_sparse_fwd_solve_device(b200ldlt_handle h, int nbi, const int* bindex, const double* d_b, int* nxi, int* xindex,
                                     double* d_x) {
  Solver* sv = (Solver*)h;
  if (!sv) return B200LDLT_FATAL_ERROR;
  return sparse_fwd(sv, nbi, bindex, d_b, false, nxi, xindex, d_x);
}

int b200ldlt_sparse_solve(b200ldlt_handle h, int nrhs, int nbi, const int* bindex, const double* b, int nxs, const int* xsel,
                          double* x) {
  Solver* sv = (Solver*)h;
  if (!sv) return B200LDLT_FATAL_ERROR;
  return sparse_solve(sv, nrhs, nbi, bindex, b, nxs, xsel, x, true);
}

int b200ldlt_sparse_solve_device(b200ldlt_handle h, int nrhs, int nbi, const int* bindex, const double* d_b, int nxs,
                                 const int* xsel, double* d_x) {
  Solver* sv = (Solver*)h;
  if (!sv) return B200LDLT_FATAL_ERROR;
  return sparse_solve(sv, nrhs, nbi, bindex, d_b, nxs, xsel, d_x, false);
}

int b200ldlt_inverse_entries(b200ldlt_handle h, int nent, const int* irow, const int* jcol, double* vals) {
  Solver* sv = (Solver*)h;
  if (!sv) return B200LDLT_FATAL_ERROR;
  return inverse_entries(sv, nent, irow, jcol, vals, true);
}

int b200ldlt_inverse_entries_device(b200ldlt_handle h, int nent, const int* irow, const int* jcol, double* d_vals) {
  Solver* sv = (Solver*)h;
  if (!sv) return B200LDLT_FATAL_ERROR;
  return inverse_entries(sv, nent, irow, jcol, d_vals, false);
}

int b200ldlt_alter_d(b200ldlt_handle h, const double* dinv2) {
  Solver* sv = (Solver*)h;
  if (!sv) return B200LDLT_FATAL_ERROR;
  if (!dinv2) { sv->err = "alter_d: no entries"; return B200LDLT_FATAL_ERROR; }
  { const int rc = factors_state(sv, "alter_d"); if (rc != B200LDLT_SUCCESS) return rc; }
  const Analysis& A = *sv->an;
  cudaStream_t st = sv->stream;
  const int n = sv->n;
  if (sv->d_alter.n != 2 * (size_t)n) CU(sv->d_alter.alloc(2 * (size_t)n));
  if (!sv->d_alter_bad.p) CU(sv->d_alter_bad.alloc(1));
  int bad = 0;
  CU(cudaMemcpyAsync(sv->d_alter.p, dinv2, 2 * (size_t)n * sizeof(double), cudaMemcpyHostToDevice, st));
  CU(cudaMemsetAsync(sv->d_alter_bad.p, 0, sizeof(int), st));
  k_alter_check<<<cdiv(n, 256), 256, 0, st>>>(n, A.d_ptype.p, sv->d_alter.p, sv->d_alter_bad.p);
  k_alter<<<cdiv(n, 256), 256, 0, st>>>(n, A.d_ptype.p, sv->d_alter.p, sv->d_alter_bad.p, A.d_dinv.p, A.d_doff.p);
  CU(cudaGetLastError());
  CU(cudaMemcpyAsync(&bad, sv->d_alter_bad.p, sizeof(int), cudaMemcpyDeviceToHost, st));
  CU(cudaStreamSynchronize(st));
  if (bad) {
    sv->err = "alter_d: refused (an entry is not finite, or an off-diagonal entry is non-zero where no 2x2 pivot opens); D is unchanged";
    return B200LDLT_FATAL_ERROR;
  }
  return B200LDLT_SUCCESS;
}

int b200ldlt_set_singular_action(b200ldlt_handle h, int keep) {
  Solver* sv = (Solver*)h;
  if (!sv) return B200LDLT_FATAL_ERROR;
  if (keep != 0 && keep != 1) { sv->err = "set_singular_action: keep must be 0 or 1"; return B200LDLT_FATAL_ERROR; }
  sv->keep_singular = keep == 1;
  return B200LDLT_SUCCESS;
}

int b200ldlt_enquire_zero_pivots(b200ldlt_handle h, int* nzero, int* pos) {
  Solver* sv = (Solver*)h;
  if (!sv) return B200LDLT_FATAL_ERROR;
  if (!nzero) { sv->err = "enquire_zero_pivots: NULL nzero"; return B200LDLT_FATAL_ERROR; }
  { const int rc = factors_state(sv, "enquire_zero_pivots", true); if (rc != B200LDLT_SUCCESS) return rc; }
  const Analysis& A = *sv->an;
  *nzero = (int)A.zpos.size();
  if (pos) std::copy(A.zpos.begin(), A.zpos.end(), pos);
  return B200LDLT_SUCCESS;
}

int b200ldlt_solve_fredholm(b200ldlt_handle h, int nrhs, double tol, double* x, int* consistent) {
  Solver* sv = (Solver*)h;
  if (!sv) return B200LDLT_FATAL_ERROR;
  return fredholm(sv, nrhs, tol, x, consistent, true);
}

int b200ldlt_solve_fredholm_device(b200ldlt_handle h, int nrhs, double tol, double* d_x, int* consistent) {
  Solver* sv = (Solver*)h;
  if (!sv) return B200LDLT_FATAL_ERROR;
  return fredholm(sv, nrhs, tol, d_x, consistent, false);
}

int b200ldlt_selected_inverse(b200ldlt_handle h, double* diag, double* vals) {
  Solver* sv = (Solver*)h;
  if (!sv) return B200LDLT_FATAL_ERROR;
  return selected_inverse(sv, diag, vals, true);
}

int b200ldlt_selected_inverse_device(b200ldlt_handle h, double* d_diag, double* d_vals) {
  Solver* sv = (Solver*)h;
  if (!sv) return B200LDLT_FATAL_ERROR;
  return selected_inverse(sv, d_diag, d_vals, false);
}

int b200ldlt_error_analysis(b200ldlt_handle h, int nrhs, const double* b, const double* x, int cond, b200ldlt_errors* out) {
  Solver* sv = (Solver*)h;
  if (!sv) return B200LDLT_FATAL_ERROR;
  return error_analysis(sv, nrhs, b, x, cond, out, true);
}

int b200ldlt_error_analysis_device(b200ldlt_handle h, int nrhs, const double* d_b, const double* d_x, int cond,
                                   b200ldlt_errors* out) {
  Solver* sv = (Solver*)h;
  if (!sv) return B200LDLT_FATAL_ERROR;
  return error_analysis(sv, nrhs, d_b, d_x, cond, out, false);
}

int b200ldlt_solve_refined(b200ldlt_handle h, int nrhs, const double* b, double* x, int max_steps, double tol,
                           b200ldlt_refined* out) {
  Solver* sv = (Solver*)h;
  if (!sv) return B200LDLT_FATAL_ERROR;
  return solve_refined(sv, nrhs, b, x, max_steps, tol, out, true);
}

int b200ldlt_solve_refined_device(b200ldlt_handle h, int nrhs, const double* d_b, double* d_x, int max_steps,
                                  double tol, b200ldlt_refined* out) {
  Solver* sv = (Solver*)h;
  if (!sv) return B200LDLT_FATAL_ERROR;
  return solve_refined(sv, nrhs, d_b, d_x, max_steps, tol, out, false);
}

int b200ldlt_solve_gmres(b200ldlt_handle h, int nrhs, const double* b, double* x, const double* vals, int restart,
                         int max_cycles, double tol, double inner_tol, b200ldlt_gmres* out) {
  Solver* sv = (Solver*)h;
  if (!sv) return B200LDLT_FATAL_ERROR;
  return solve_gmres(sv, nrhs, b, x, vals, restart, max_cycles, tol, inner_tol, out, true);
}

int b200ldlt_solve_gmres_device(b200ldlt_handle h, int nrhs, const double* d_b, double* d_x, const double* d_vals,
                                int restart, int max_cycles, double tol, double inner_tol, b200ldlt_gmres* out) {
  Solver* sv = (Solver*)h;
  if (!sv) return B200LDLT_FATAL_ERROR;
  return solve_gmres(sv, nrhs, d_b, d_x, d_vals, restart, max_cycles, tol, inner_tol, out, false);
}

int b200ldlt_condest(b200ldlt_handle h, double* kappa1, double* anorm1, double* ainv1, int* nprod) {
  Solver* sv = (Solver*)h;
  if (!sv) return B200LDLT_FATAL_ERROR;
  return condest(sv, kappa1, anorm1, ainv1, nprod);
}

int b200ldlt_set_schur(b200ldlt_handle h, int m, const int* vars) {
  Solver* sv = (Solver*)h;
  if (!sv) return B200LDLT_FATAL_ERROR;
  const char* bad = sv->n <= 0 ? "analyse first" : m < 0 ? "m must be >= 0" : m >= sv->n ? "m must be < n"
                    : m > 0 && !vars ? "NULL vars" : sv->an && sv->an->shard.active ? "not available on a sharded handle" : nullptr;
  if (!bad) {
    std::vector<char> seen(sv->n, 0);
    for (int i = 0; i < m && !bad; ++i) {
      if (vars[i] < 0 || vars[i] >= sv->n) bad = "variable out of range";
      else if (seen[vars[i]]) bad = "variable repeated";
      else seen[vars[i]] = 1;
    }
  }
  if (bad) { sv->err = std::string("set_schur: ") + bad; return B200LDLT_FATAL_ERROR; }
  sv->sc_vars.assign(vars, vars + m);
  // the factors no longer match the mode; the next factor call re-analyses (the ordering places S last)
  if (sv->an) {
    sv->an->factored = false;
    sv->reanalyse = true;
  }
  return B200LDLT_SUCCESS;
}

int b200ldlt_schur_complement(b200ldlt_handle h, double* sc) {
  Solver* sv = (Solver*)h;
  if (!sv) return B200LDLT_FATAL_ERROR;
  return schur_complement(sv, sc, true);
}

int b200ldlt_schur_complement_device(b200ldlt_handle h, double* d_sc) {
  Solver* sv = (Solver*)h;
  if (!sv) return B200LDLT_FATAL_ERROR;
  return schur_complement(sv, d_sc, false);
}

int b200ldlt_schur_reduce(b200ldlt_handle h, int nrhs, const double* b, double* y) {
  Solver* sv = (Solver*)h;
  if (!sv) return B200LDLT_FATAL_ERROR;
  return schur_solve(sv, "schur_reduce", nrhs, b, nullptr, y, true, false);
}

int b200ldlt_schur_reduce_device(b200ldlt_handle h, int nrhs, const double* d_b, double* d_y) {
  Solver* sv = (Solver*)h;
  if (!sv) return B200LDLT_FATAL_ERROR;
  return schur_solve(sv, "schur_reduce", nrhs, d_b, nullptr, d_y, false, false);
}

int b200ldlt_schur_expand(b200ldlt_handle h, int nrhs, const double* b, const double* xs, double* x) {
  Solver* sv = (Solver*)h;
  if (!sv) return B200LDLT_FATAL_ERROR;
  return schur_solve(sv, "schur_expand", nrhs, b, xs, x, true, true);
}

int b200ldlt_schur_expand_device(b200ldlt_handle h, int nrhs, const double* d_b, const double* d_xs, double* d_x) {
  Solver* sv = (Solver*)h;
  if (!sv) return B200LDLT_FATAL_ERROR;
  return schur_solve(sv, "schur_expand", nrhs, d_b, d_xs, d_x, false, true);
}

/* ---- multi-GPU elimination-tree sharding (SURVEY.md section 8e) -------------------------------------------
 * One process per GPU, each with its own handle and the SAME matrix.  After the (replicated, deterministic)
 * analysis, rank g factorises the subtrees it owns; the contribution blocks of the cut are moved to rank 0 by the
 * caller (NCCL send/recv through torch.distributed on the device pointers exported below), which then factorises
 * the top part.  The solve mirrors it.  See ipopt_b200/sharded.py for the orchestration. */
int b200ldlt_shard_setup(b200ldlt_handle h, int rank, int world) {
  Solver* sv = (Solver*)h;
  if (!sv || !sv->an || world < 1 || rank < 0 || rank >= world) { if (sv) sv->err = "shard_setup: analyse first / bad rank"; return B200LDLT_FATAL_ERROR; }
  if (!sv->sc_vars.empty()) { sv->err = "shard_setup: Schur mode"; return B200LDLT_FATAL_ERROR; }
  CU(cudaSetDevice(sv->dev));
  return shard_setup(sv, rank, world);
}

int64_t b200ldlt_shard_array(b200ldlt_handle h, const char* name, int64_t* out, int64_t cap) {
  Solver* sv = (Solver*)h;
  if (!sv || !sv->an || !sv->an->shard.active || !name) return -1;
  const Analysis::Shard& H = sv->an->shard;
  std::string nm(name);
  const std::vector<int>* v = nullptr;
  if (nm == "owner") v = &H.owner;
  else if (nm == "cut_roots") v = &H.cut_roots;
  else if (nm == "top_fronts") v = &H.top_fronts;
  if (!v) return -1;
  if (out) for (int64_t i = 0; i < (int64_t)v->size() && i < cap; ++i) out[i] = (*v)[i];
  return (int64_t)v->size();
}

void* b200ldlt_device_ptr(b200ldlt_handle h, const char* name) {
  Solver* sv = (Solver*)h;
  if (!sv || !name) return nullptr;
  std::string nm(name);
  if (nm == "vals") return sv->d_vals.p;        // the handle's: assemble_augsys_device fills it before the (lazy) analysis
  if (!sv->an) return nullptr;
  const Analysis& A = *sv->an;
  if (nm == "CB") return A.d_CB.p;
  if (nm == "cbv") return A.sweep.d_cbv.p;
  if (nm == "x") return A.sweep.d_x.p;
  if (nm == "counters") return A.d_counters.p;
  if (nm == "scale") return A.d_scale.p;
  return nullptr;
}

/* phase 0: (optional H2D of the pinned values array,) scaling + the subtrees owned by this rank;
 * phase 1: the top part (only rank 0 has work).  Enqueues on the handle's stream and returns. */
int b200ldlt_shard_factor(b200ldlt_handle h, int phase, int from_host) {
  Solver* sv = (Solver*)h;
  if (!sv || !sv->an || !sv->an->shard.active || phase < 0 || phase > 1) { if (sv) sv->err = "shard_factor: shard_setup first"; return B200LDLT_FATAL_ERROR; }
  CU(cudaSetDevice(sv->dev));
  cudaStream_t st = sv->stream;
  if (phase == 0) {
    CU(cudaEventRecord(sv->ev0, st));
    if (from_host) CU(cudaMemcpyAsync(sv->d_vals.p, sv->h_vals, sv->nnz * sizeof(double), cudaMemcpyHostToDevice, st));
    sv->have_dev_vals = true;
  }
  return enqueue_factor(sv, sv->an->shard.part[phase], phase == 0);
}

/* counters_total: CNT_N ints already summed over the ranks (all-reduce of device_ptr("counters")) */
int b200ldlt_shard_factor_finish(b200ldlt_handle h, const int* counters_total, int check_inertia, int expected_neg, int* num_neg) {
  Solver* sv = (Solver*)h;
  if (!sv || !sv->an || !sv->an->shard.active || !counters_total) return B200LDLT_FATAL_ERROR;
  CU(cudaSetDevice(sv->dev));
  CU(cudaEventRecord(sv->ev1, sv->stream));
  CU(cudaStreamSynchronize(sv->stream));
  return settle_factor(sv, counters_total, check_inertia, expected_neg, num_neg);
}

/* phase 0: permute+scale rhs, forward sweep over my subtrees;  phase 1 (rank 0): forward + backward over the top;
 * phase 2: backward sweep over my subtrees;  phase 3: un-permute/un-scale into d_rhs.  d_rhs: dim doubles on the device. */
int b200ldlt_shard_solve(b200ldlt_handle h, int phase, double* d_rhs) {
  Solver* sv = (Solver*)h;
  if (!sv || !sv->an || !sv->an->shard.active || !sv->an->factored) { if (sv) sv->err = "shard_solve: factor first"; return B200LDLT_FATAL_ERROR; }
  Analysis& A = *sv->an;
  CU(cudaSetDevice(sv->dev));
  cudaStream_t st = sv->stream;
  Analysis::Shard& H = A.shard;
  const int n = sv->n;
  int rc = B200LDLT_SUCCESS;
  // (phases 1 and 2 run under phase 0's epoch: k_mark_flags stamps the cut roots and the top fronts with it)
  if (phase == 0) {
    sv->launches = 0;
    rc = forward(sv, H.part[0].solve, A.sweep, d_rhs, 1);
  } else if (phase == 1) {
    if (H.d_mark_cut.n) k_mark_flags<<<cdiv((long long)H.d_mark_cut.n, 256), 256, 0, st>>>(A.sweep.d_done_f.p, H.d_mark_cut.p, (int)H.d_mark_cut.n, A.solve_epoch);
    rc = launch_sweep(sv, H.part[1].solve, A.sweep, 1, true);
    if (rc == B200LDLT_SUCCESS) rc = launch_sweep(sv, H.part[1].solve, A.sweep, 1, false);
  } else if (phase == 2) {
    if (H.rank != 0 && H.d_mark_top.n) k_mark_flags<<<cdiv((long long)H.d_mark_top.n, 256), 256, 0, st>>>(A.sweep.d_done_b.p, H.d_mark_top.p, (int)H.d_mark_top.n, A.solve_epoch);
    rc = launch_sweep(sv, H.part[0].solve, A.sweep, 1, false);
  } else if (phase == 3) {
    k_sol_out<<<cdiv(n, 256), 256, 0, st>>>(n, A.d_perm.p, A.d_scale.p, A.sweep.d_x.p, n, d_rhs);
  } else return B200LDLT_FATAL_ERROR;
  CU(cudaGetLastError());
  return rc;
}

/* ---- device-side callers (SURVEY.md 8f-1) ------------------------------------------------------------------------ */
namespace b200 {
struct AugSeg { const double* src; long long off; long long n; double scale, add; };   // out[off+i] = scale*src[i] + add (src NULL: add)
struct AugSegs { AugSeg s[8]; };
__global__ void __launch_bounds__(256) k_assemble_augsys(AugSegs A, double* __restrict__ out) {
  const AugSeg g = A.s[blockIdx.y];
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < g.n; i += (long long)gridDim.x * blockDim.x) {
    double v;
    if (!g.src) v = g.add;
    else {
      v = g.src[i];
      if (g.scale != 1.0) v = __dmul_rn(g.scale, v);   // IpBlasScal of the SumSymMatrix term (FillValues)
      if (g.add != 0.0) v = __dadd_rn(v, g.add);       // Vector::AddScalar(delta)
    }
    out[g.off + i] = v;
  }
}
}  // namespace b200

int b200ldlt_assemble_augsys_device(b200ldlt_handle h, const b200ldlt_augsys* a) {
  Solver* sv = (Solver*)h;
  if (!sv || !a) return B200LDLT_FATAL_ERROR;
  if (sv->n <= 0 || a->n_d != a->n_s) { sv->err = "assemble_augsys: analyse first / n_d must equal n_s"; return B200LDLT_FATAL_ERROR; }
  const long long total = (long long)a->nnz_w + a->n_x + a->n_s + a->nnz_jc + a->n_c + a->nnz_jd + a->n_s + a->n_d;
  if (total != sv->nnz || a->n_x + a->n_s + a->n_c + a->n_d != sv->n) { sv->err = "assemble_augsys: block sizes do not match the analysed structure"; return B200LDLT_FATAL_ERROR; }
  CU(cudaSetDevice(sv->dev));
  if (!sv->d_vals.p) CU(sv->d_vals.alloc(sv->nnz));
  AugSegs A;
  long long off = 0;
  auto seg = [&](int q, const double* src, long long n, double scale, double add) { A.s[q] = AugSeg{src, off, n, scale, add}; off += n; };
  seg(0, a->W, a->nnz_w, a->W ? a->W_factor : 1.0, 0.0);
  seg(1, a->D_x, a->n_x, 1.0, a->delta_x);
  seg(2, a->D_s, a->n_s, 1.0, a->delta_s);
  seg(3, a->J_c, a->nnz_jc, 1.0, 0.0);
  seg(4, a->D_c, a->n_c, 1.0, -a->delta_c);
  seg(5, a->J_d, a->nnz_jd, 1.0, 0.0);
  seg(6, nullptr, a->n_s, 1.0, -1.0);
  seg(7, a->D_d, a->n_d, 1.0, -a->delta_d);
  if (!a->J_c && a->nnz_jc > 0) { sv->err = "assemble_augsys: J_c missing"; return B200LDLT_FATAL_ERROR; }
  if (!a->J_d && a->nnz_jd > 0) { sv->err = "assemble_augsys: J_d missing"; return B200LDLT_FATAL_ERROR; }
  long long nmax = 1;
  for (int q = 0; q < 8; ++q) nmax = std::max(nmax, A.s[q].n);
  k_assemble_augsys<<<dim3((unsigned)std::min<long long>((nmax + 255) / 256, 1184), 8), 256, 0, sv->stream>>>(A, sv->d_vals.p);
  CU(cudaGetLastError());
  sv->have_dev_vals = true;
  return B200LDLT_SUCCESS;
}

int b200ldlt_solve_refine_device(b200ldlt_handle h, double* d_rhs, int min_steps, int max_steps, double tol,
                                 int* steps_done, double* residual_ratio) {
  Solver* sv = (Solver*)h;
  if (steps_done) *steps_done = 0;
  if (!sv || !sv->an || !sv->an->factored || !sv->have_dev_vals || !d_rhs) { if (sv) sv->err = "solve_refine: factor first (values on the device)"; return B200LDLT_FATAL_ERROR; }
  { const int rc = factors_state(sv, "solve_refine_device", true); if (rc != B200LDLT_SUCCESS) return rc; }
  Analysis& A = *sv->an;
  const int n = sv->n;
  if (!sv->vec) {
    sv->vec = b200vec_create(sv->dev, (void*)sv->stream);
    if (!sv->vec) { sv->err = "solve_refine: b200vec_create failed"; return B200LDLT_FATAL_ERROR; }
  }
  if (!sv->amat) {
    sv->amat = b200vec_tmat_create(sv->vec, n, n, sv->nnz, sv->irn.data(), sv->jcn.data(), 1);
    if (!sv->amat) { sv->err = "solve_refine: could not build the triplet operator"; return B200LDLT_FATAL_ERROR; }
  }
  if ((int)sv->d_ref_b.n < n || (int)sv->d_ref_r.n < n) { CU(sv->d_ref_b.alloc(n)); CU(sv->d_ref_r.alloc(n)); }
  cudaStream_t st = sv->stream;
  CU(cudaMemcpyAsync(sv->d_ref_b.p, d_rhs, (size_t)n * sizeof(double), cudaMemcpyDeviceToDevice, st));
  sv->launches = 0;
  int rc = enqueue_solve(sv, A.sweep, 0, d_rhs, d_rhs, 1);
  if (rc != B200LDLT_SUCCESS) return rc;
  b200vec vb{sv->d_ref_b.p, n, 0, 0.0}, vx{d_rhs, n, 0, 0.0}, vr{sv->d_ref_r.p, n, 0, 0.0};
  double nb = 0.0, ratio = 0.0;
  if (b200vec_amax(sv->vec, &vb, &nb)) { sv->err = b200vec_last_error(sv->vec); return B200LDLT_FATAL_ERROR; }
  int step = 0;
  for (;;) {
    // r = b - A x
    vr.homogeneous = 0;
    if (b200vec_copy(sv->vec, &vb, &vr) || b200vec_tmat_mult(sv->amat, sv->d_vals.p, -1.0, &vx, 1.0, &vr)) { sv->err = b200vec_last_error(sv->vec); return B200LDLT_FATAL_ERROR; }
    double nr = 0.0, nx = 0.0;
    if (b200vec_amax(sv->vec, &vr, &nr) || b200vec_amax(sv->vec, &vx, &nx)) { sv->err = b200vec_last_error(sv->vec); return B200LDLT_FATAL_ERROR; }
    ratio = (nb + nx == 0.0) ? nr : nr / (std::min(nx, 1e6 * nb) + nb);
    if (step >= max_steps || (step >= min_steps && ratio <= tol)) break;
    rc = enqueue_solve(sv, A.sweep, 0, sv->d_ref_r.p, sv->d_ref_r.p, 1);     // d = A^-1 r
    if (rc != B200LDLT_SUCCESS) return rc;
    if (b200vec_axpy(sv->vec, 1.0, &vr, &vx)) { sv->err = b200vec_last_error(sv->vec); return B200LDLT_FATAL_ERROR; }
    ++step;
  }
  CU(cudaStreamSynchronize(st));
  if (steps_done) *steps_done = step;
  if (residual_ratio) *residual_ratio = ratio;
  return B200LDLT_SUCCESS;
}

int b200ldlt_num_neg(b200ldlt_handle h) { return h ? ((Solver*)h)->num_neg : -1; }

int b200ldlt_increase_quality(b200ldlt_handle h) {
  Solver* sv = (Solver*)h;
  if (!sv) return 0;
  // The last factorisation lifted pivots (num_forced) or saw growth beyond 1/u: a larger threshold would only reject
  // more pivots inside the same supernodes.  The pairing / ordering were frozen on the values of the FIRST matrix; redo
  // the analysis on the current values instead (once per matrix: the second request raises the threshold as usual).
  if ((sv->info.num_forced > 0 || sv->info.num_growth > 0) && sv->an && !sv->an->shard.active && !sv->reanalysed_since_raise) {
    sv->reanalyse = true;
    sv->reanalysed_since_raise = true;
    return 1;
  }
  if (sv->pivtol >= sv->opt.pivtolmax) return 0;
  sv->pivtol = std::min(sv->opt.pivtolmax, std::pow(sv->pivtol, 0.75));
  sv->reanalysed_since_raise = false;
  return 1;
}

int b200ldlt_set_pivtol(b200ldlt_handle h, double pivtol, double pivtolmax) {
  Solver* sv = (Solver*)h;
  if (!sv || !(pivtol > 0.0) || !(pivtolmax >= pivtol)) return B200LDLT_FATAL_ERROR;
  sv->opt.pivtol = pivtol; sv->opt.pivtolmax = pivtolmax;
  sv->pivtol = pivtol;
  return B200LDLT_SUCCESS;
}

int b200ldlt_get_info(b200ldlt_handle h, b200ldlt_info* info) {
  if (!h || !info) return B200LDLT_FATAL_ERROR;
  *info = ((Solver*)h)->info;
  return B200LDLT_SUCCESS;
}

int64_t b200ldlt_symbolic_array(b200ldlt_handle h, const char* name, int64_t* out, int64_t cap) {
  Solver* sv = (Solver*)h;
  if (!sv || !name) return -1;
  if (!sv->an) {
    if (sv->n <= 0) return -1;
    if (run_analysis(sv, nullptr) != B200LDLT_SUCCESS) return -1;
  }
  const Analysis& A = *sv->an;
  const Symbolic& S = A.S;
  std::string nm(name);
#define RET(vec)                                                        \
  do {                                                                  \
    int64_t len = (int64_t)(vec).size();                                \
    if (out) for (int64_t i = 0; i < len && i < cap; ++i) out[i] = (int64_t)(vec)[i]; \
    return len;                                                         \
  } while (0)
  if (nm == "perm") RET(S.perm);
  if (nm == "sn_start") RET(S.sn_start);
  if (nm == "sn_parent") RET(S.sn_parent);
  if (nm == "rows_ptr") RET(S.rows_ptr);
  if (nm == "rows") RET(S.rows);
  if (nm == "rel") RET(S.rel);
  if (nm == "L_off") RET(S.L_off);
  if (nm == "cb_off") RET(S.cb_off);
  if (nm == "u_dst64") RET(S.u_dst64);
  if (nm == "uent_ptr") RET(S.uent_ptr);
  if (nm == "t2u") RET(S.t2u);
  if (nm == "sn_level") RET(S.sn_level);
  if (nm == "level_ptr") RET(S.level_ptr);
  if (nm == "level_sn") RET(S.level_sn);
  if (nm == "sparse_run_set") { static const std::vector<int> none; RET(A.pruned ? A.pruned->last_sfs : none); }
  if (nm == "inverse_run_set") { static const std::vector<int> none; RET(A.pruned ? A.pruned->last_inv : none); }
  if (nm == "sparse_solve_fwd_run_set") { static const std::vector<int> none; RET(A.pruned ? A.pruned->last_fwd : none); }
  if (nm == "sparse_solve_bwd_run_set") { static const std::vector<int> none; RET(A.pruned ? A.pruned->last_bwd : none); }
#undef RET
  return -1;
}

int b200ldlt_residual(b200ldlt_handle h, const double* x, const double* b, double* r_inf, double* x_inf, double* b_inf) {
  Solver* sv = (Solver*)h;
  if (!sv || !sv->have_dev_vals) { if (sv) sv->err = "residual: no matrix on the device"; return B200LDLT_FATAL_ERROR; }
  if (!sv->an) { sv->err = "residual: no analysis (factorise first)"; return B200LDLT_FATAL_ERROR; }
  const Analysis& A = *sv->an;
  CU(cudaSetDevice(sv->dev));
  cudaStream_t st = sv->stream;
  const int n = sv->n;
  DevBuf<double> dx, db;
  DevBuf<unsigned long long> dm;
  CU(dx.alloc(n)); CU(db.alloc(n)); CU(dm.alloc(3));
  CU(cudaMemcpyAsync(dx.p, x, n * sizeof(double), cudaMemcpyHostToDevice, st));
  CU(cudaMemcpyAsync(db.p, b, n * sizeof(double), cudaMemcpyHostToDevice, st));
  CU(cudaMemsetAsync(dm.p, 0, 3 * sizeof(unsigned long long), st));
  k_residual_init<<<cdiv(n, 256), 256, 0, st>>>(n, db.p, A.d_res.p);
  k_residual_acc<<<cdiv(sv->nnz, 256), 256, 0, st>>>(sv->nnz, A.d_irn.p, A.d_jcn.p, sv->d_vals.p, dx.p, A.d_res.p);
  k_absmax<<<cdiv(n, 256), 256, 0, st>>>(n, A.d_res.p, dm.p);
  k_absmax<<<cdiv(n, 256), 256, 0, st>>>(n, dx.p, dm.p + 1);
  k_absmax<<<cdiv(n, 256), 256, 0, st>>>(n, db.p, dm.p + 2);
  unsigned long long hm[3];
  CU(cudaMemcpyAsync(hm, dm.p, sizeof(hm), cudaMemcpyDeviceToHost, st));
  CU(cudaStreamSynchronize(st));
  double v[3];
  memcpy(v, hm, sizeof(v));
  if (r_inf) *r_inf = v[0];
  if (x_inf) *x_inf = v[1];
  if (b_inf) *b_inf = v[2];
  return B200LDLT_SUCCESS;
}

}  // extern "C"
