// Host orchestration + extern "C" shim of the GPU LDL^T backend (see include/b200ldlt.h), H100 / sm_90a.
// One translation unit: the kernels are included so nvcc sees launch sites and definitions together.
#include "../../include/b200ldlt.h"
#include "../../include/b200vec.h"

#include <cuda_runtime.h>

#include <algorithm>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <string>
#include <memory>
#include <vector>

#include "factor_kernels.cu"
#include "solve_kernels.cu"
#include "solve_dataflow.cu"
#include "schur_tc.cu"
#include "symbolic.hpp"

namespace b200 {

template <class T>
struct DevBuf {
  T* p = nullptr;
  size_t n = 0;
  ~DevBuf() { release(); }
  void release() { if (p) cudaFree(p); p = nullptr; n = 0; }
  cudaError_t alloc(size_t count) {
    release();
    n = count;
    if (count == 0) return cudaSuccess;
    return cudaMalloc((void**)&p, count * sizeof(T));
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
  DevBuf<SolveTask> d_tf, d_tb;
  DevBuf<int> d_bundle, d_sub_meta, d_ccnt, d_subrow;
  DevBuf<SubDesc> d_subs;
  DevBuf<int2> d_subpair;
  DevBuf<int> d_sub_Loff;
  std::vector<std::unique_ptr<DevBuf<int>>> d_direct;   // per bottom level: the fronts k_solve_direct owns
  std::vector<int> direct_cnt;
  DevBuf<double> d_part;
  DevSolve V;
  int nsub = 0, npair = 0, ntf = 0, ntb = 0;
  long long sub_bytes = 0;
};

struct LevelPlan {
  // big fronts of the level: [big_off, big_off+big_cnt) in front_list
  int big_off = 0, big_cnt = 0, big_kmax = 0, big_fmax = 0, big_rmax = 0, big_chmax = 0;
  long long big_entmax = 0, big_zero_max = 0;
  struct Bucket { int off, cnt, fmax, kmax, threads; size_t smem; int kind = 0; };   // kind 2: k_front_warp2 (order 33..64, <= 32 pivots)
  std::vector<Bucket> small;
  int all_off = 0, all_cnt = 0, fmax = 0;  // whole level (solve)
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

// environment switches for profiling / A-B runs, read ONCE at b200ldlt_create (never on the enqueue path)
struct DebugSwitches {
  bool factor_sections = false;   // B200_FACTOR_SECTIONS=1 (with use_graph=0): timed section marks
  bool one_stream = false;        // B200_ONE_STREAM=1: big-front pipeline on a single stream
  bool solve_timeline = false;    // B200_SOLVE_TIMELINE=1: per-task %globaltimer log of the top solve kernel
  bool cb_at_end = false;         // B200_CB_AT_END=1: Schur complements as one GEMM per level (k_big_schur84) instead of per-panel updates
  int solve_direct = 2;           // B200_SOLVE_DIRECT=D: the D lowest tree levels are solved by k_solve_direct (0 = all inside the subtrees)
  bool solve_nopair = false;      // B200_SOLVE_NOPAIR=1: one subtree per CTA in the solve sweeps (no side-by-side pairs)
  bool no_warp2 = false;          // B200_NO_WARP2=1: fronts of order 33..64 by the shared-memory kernel (one CTA each) instead of k_front_warp2
  bool no_pdl = false;            // B200_NO_PDL=1: chain kernels launched without programmatic dependent launch
  bool factor_timeline = false;   // B200_FACTOR_TIMELINE=1: %globaltimer records of the factorisation kernels (b200ldlt_dump_factor_timeline)
  std::vector<int> buckets;       // B200_BUCKETS=a,b,c: soft split points of the shared-memory front classes
  void read() {
    factor_sections = getenv("B200_FACTOR_SECTIONS") != nullptr;
    one_stream = getenv("B200_ONE_STREAM") != nullptr;
    solve_timeline = getenv("B200_SOLVE_TIMELINE") != nullptr;
    factor_timeline = getenv("B200_FACTOR_TIMELINE") != nullptr;
    cb_at_end = getenv("B200_CB_AT_END") != nullptr;
    solve_nopair = getenv("B200_SOLVE_NOPAIR") != nullptr;
    if (const char* e = getenv("B200_SOLVE_DIRECT")) solve_direct = atoi(e);
    no_pdl = getenv("B200_NO_PDL") != nullptr;
    no_warp2 = getenv("B200_NO_WARP2") != nullptr;
    if (const char* e = getenv("B200_BUCKETS")) {
      for (const char* p = e; *p;) { buckets.push_back(atoi(p)); while (*p && *p != ',') ++p; if (*p) ++p; }
    } else {
      buckets = {48, 96};   // the classes of a level run side by side, so a finer split costs no serial launches
                            // (H100 SXM, 700 W, factorisation at N=400 / 800: {96} and {32,64,96} within 0.4 %)
    }
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
  cudaEvent_t ev_chunk[4] = {nullptr, nullptr, nullptr, nullptr};   // D2H chunks of the host solve path

  int n = 0, nnz = 0;
  std::vector<int> irn, jcn;
  double* h_vals = nullptr;      // pinned
  double* h_rhs = nullptr;       // pinned staging (n * rhs_cap)
  int rhs_cap = 0;
  int* h_counters = nullptr;     // pinned
  bool analysed = false, factored = false, have_dev_vals = false;
  b200vec_ctx vec = nullptr;       // vector kernels on the handle's stream (device-side refinement)
  b200vec_tmat amat = nullptr;     // the matrix as a symmetric triplet operator (residuals)
  DevBuf<double> d_ref_b, d_ref_r;
  int tc_min_r = 0;                // fronts with r >= this use the tensor-core Schur path (0 = off)
  bool reanalyse = false;          // set by increase_quality after forced pivots: next factor re-runs the analysis on its values
  int n_reanalysed = 0;
  long long n_factor = 0;
  bool reanalysed_since_raise = false;
  Symbolic S;
  std::vector<LevelPlan> plan;
  SchurLists schur;
  DevBuf<int8_t> d_tc_dig;           // digit scratch of the tensor-core Schur path (largest level)
  DevBuf<int> d_tc_exp;
  b200ldlt_info info;
  int num_neg = 0;
  double pivtol = 1e-8;

  // device
  DevBuf<int> d_sn_start, d_sn_parent, d_rows, d_rel, d_child_ptr, d_child_idx, d_front_list, d_perm;
  DevBuf<int> d_useg_src, d_u_row, d_u_col, d_irn, d_jcn;
  DevBuf<long long> d_rows_ptr, d_uent_ptr, d_u_dst64, d_L_off, d_cb_off, d_useg_ptr;
  DevBuf<unsigned> d_u_dst;
  DevBuf<double> d_vals, d_uval, d_L, d_W, d_CB, d_dinv, d_doff, d_scale, d_x, d_cbv, d_rhs, d_res, d_colmax;
  DevBuf<int> d_ptype, d_lperm, d_bperm, d_counters, d_einv;
  DevBuf<long long> d_einv_off;
  DevBuf<unsigned long long> d_rmax;
  DevSym DS;
  DevNum DN;
  int launches = 0;
  // solve (solve_dataflow.cu): shared flag / scratch arrays + one plan per front set
  DevBuf<int> d_done_f, d_done_b, d_bflag_f, d_bflag_b, d_bcnt, d_bcnt_b, d_boff;
  DevBuf<long long> d_bigv_off;
  DevBuf<double> d_bigv, d_bigy;
  DevBuf<unsigned long long> d_ticket, d_tlog, d_flog;
  DevBuf<double> d_linv;
  DevBuf<double> d_linv_part;       // partial tiles of the chunked k_linv_gemm items (one launch at a time uses it)
  DevBuf<int> d_linv_cnt;           // their arrival counters (self-resetting)
  DevBuf<long long> d_linv_off, d_gmap_off;
  DevBuf<FrontDesc> d_fdesc;
  DevBuf<int> d_gmap;
  LinvPlan linv_plan;               // explicit inverses of the big fronts' pivot blocks (all fronts)
  std::vector<std::unique_ptr<LinvPlan>> linv_level;   // the same work, split by tree level (issued behind each level's chain)
  std::vector<SolveTask> h_tasks;   // fwd then bwd (debug timeline)
  SolvePlan splan;                  // all fronts
  std::vector<char> solve_direct_front;   // per supernode: solved by k_solve_direct (see build_solve_tables)
  int solve_epoch = 0, df_grid = 0;
  unsigned long long ticket_f = 0, ticket_b = 0;
  int num_sms = 132;
  struct Shard {
    bool active = false;
    int rank = 0, world = 1, nsub = 0;
    std::vector<int> owner, cut_roots, top_fronts;
    std::vector<LevelPlan> plan[2];          // [0] my subtrees, [1] top part
    SchurLists schur[2];
    DevBuf<int> d_fl[2], d_mark_cut, d_mark_top;
    SolvePlan splan[2];
    LinvPlan linv_plan[2];
  } shard;
  cudaGraph_t fgraph = nullptr;
  cudaGraphExec_t fgraph_exec = nullptr;
  double fgraph_u = -1.0;
  int fgraph_launches = 0;

  ~Solver() {
    if (amat) b200vec_tmat_destroy(amat);
    if (vec) b200vec_destroy(vec);
    if (h_vals) cudaFreeHost(h_vals);
    if (h_rhs) cudaFreeHost(h_rhs);
    if (h_counters) cudaFreeHost(h_counters);
    if (ev0) cudaEventDestroy(ev0);
    if (ev1) cudaEventDestroy(ev1);
    for (cudaEvent_t e : ev_chunk) if (e) cudaEventDestroy(e);
    if (fgraph_exec) cudaGraphExecDestroy(fgraph_exec);
    if (fgraph) cudaGraphDestroy(fgraph);
    for (cudaEvent_t e : ev_pool) cudaEventDestroy(e);
    if (stream2) cudaStreamDestroy(stream2);
    if (stream3) cudaStreamDestroy(stream3);
    for (auto& q : side) if (q) cudaStreamDestroy(q);
    if (own_stream && stream) cudaStreamDestroy(stream);
  }
  // debug (B200_FACTOR_SECTIONS=1 with use_graph=0): timed section marks of the last factorisation
  std::vector<std::pair<std::string, cudaEvent_t>> sect;
  void mark(const char* label, int level) {
    if (!dbg.factor_sections || opt.use_graph != 0) return;
    cudaEvent_t e; cudaEventCreate(&e); cudaEventRecord(e, stream);
    sect.emplace_back(std::string(label) + " L" + std::to_string(level), e);
  }
  void dump_sections() {
    if (sect.empty()) return;
    for (size_t i = 1; i < sect.size(); ++i) {
      float ms = 0; cudaEventElapsedTime(&ms, sect[i - 1].second, sect[i].second);
      fprintf(stderr, "[sections] %-18s %8.1f us\n", sect[i].first.c_str(), ms * 1e3);
    }
    for (auto& pr : sect) cudaEventDestroy(pr.second);
    sect.clear();
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
                              std::vector<LevelPlan>& plan, const std::vector<int>& soft, SchurLists& SL, int tc_min_r,
                              bool use_warp2) {
  SL.f.clear(); SL.t.clear(); SL.dfl.clear(); SL.dig_bytes = 0; SL.exp_ints = 0;
  fl.clear();
  fl.reserve(S.nsn);
  plan.assign(S.nlevels, LevelPlan());
  for (int l = 0; l < S.nlevels; ++l) {
    LevelPlan& P = plan[l];
    P.all_off = (int)fl.size();
    P.big_off = (int)fl.size();
    for (int q = S.level_ptr[l]; q < S.level_ptr[l + 1]; ++q) {
      int s = S.level_sn[q];
      if (!take[s]) continue;
      P.fmax = std::max(P.fmax, S.f(s));
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
    // holds enough fronts to fill the GPU.
    // (soft: splits at 48 and 96 by default, DebugSwitches::buckets)
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
        for (int v : soft) if (v < f) cur_lo = std::max(cur_lo, v);
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
    P.all_cnt = (int)fl.size() - P.all_off;
  }
}

static const int kSolveMidMax = 256;   // fronts above this order are "big" in the solve (block tasks + explicit L11 inverse)

static int build_linv_plan(Solver* sv, const Symbolic& S, const std::vector<char>& take, LinvPlan& LP, cudaStream_t st) {
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
  if ((size_t)LP.part_tiles > sv->d_linv_cnt.n) {     // (analysis time: never inside a captured graph)
    CU(cudaStreamSynchronize(st));
    CU(sv->d_linv_part.alloc((size_t)LP.part_tiles * 4096));
    CU(sv->d_linv_cnt.alloc((size_t)LP.part_tiles));
    CU(cudaMemset(sv->d_linv_cnt.p, 0, sv->d_linv_cnt.n * sizeof(int)));
  }
  return B200LDLT_SUCCESS;
}

static int enqueue_linv(Solver* sv, const LinvPlan& LP, cudaStream_t st);

// Triangular-solve plan of the fronts in take[] (see solve_dataflow.cu).
//  * Subtrees: maximal subtrees whose fronts are all taken, of order <= DF_MIDMAX, and whose whole working set (SubLayout)
//    fits the dynamic shared memory of k_solve_sub -> one CTA each, largest first.  Supernodes are numbered in postorder,
//    so a subtree is the contiguous range [root - size + 1, root] and so are its panels, columns, row lists, child lists.
//  * Everything else -> topologically sorted task lists for k_solve_top (forward: levels ascending; backward: descending).
static int build_solve_plan(Solver* sv, const Symbolic& S, const std::vector<char>& take, SolvePlan& SP, cudaStream_t st) {
  const int nsn = S.nsn;
  std::vector<int> size(nsn, 1), ntaken(nsn, 0), subF(nsn, 0);
  for (int s = 0; s < nsn; ++s) {   // children precede parents
    ntaken[s] += take[s] ? 1 : 0; subF[s] = std::max(subF[s], S.f(s));
    const int p = S.sn_parent[s];
    if (p >= 0) { size[p] += size[s]; ntaken[p] += ntaken[s]; subF[p] = std::max(subF[p], subF[s]); }
  }
  const std::vector<char>& direct = sv->solve_direct_front;
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
  SP.d_direct.clear(); SP.direct_cnt.clear();
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
  }
  CU(SP.d_sub_Loff.upload(subLoff, st));
  if (sv->opt.verbose)
    fprintf(stderr, "[b200ldlt] solve plan: %lld fronts (%.1f MB of L) on %d bottom levels by the direct kernel\n", ndirect,
            direct_nnz * 8 / 1e6, (int)SP.direct_cnt.size());
  SP.nsub = nsub; SP.ntf = (int)tf.size(); SP.ntb = (int)tb.size();
  if (sv->opt.verbose)
    fprintf(stderr, "[b200ldlt] solve plan: %d subtrees in %d work items (%.1f MB of L, largest %.0f KB), top: %d fwd / %d bwd tasks, %lld partial slots\n",
            nsub, SP.npair, SP.sub_bytes / 1e6, nsub ? (ownL[roots[0] + 1] - ownL[roots[0] - size[roots[0]] + 1]) * 8 / 1e3 : 0.0, SP.ntf, SP.ntb, npart);
  if (sv->dbg.solve_timeline) { sv->h_tasks = tf; sv->h_tasks.insert(sv->h_tasks.end(), tb.begin(), tb.end()); }
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
  DevSolve& V = SP.V;
  V.tasks = SP.d_tf.p; V.tasks_bwd = SP.d_tb.p; V.ntasks_fwd = SP.ntf; V.ntasks_bwd = SP.ntb;
  V.bundle = SP.d_bundle.p;
  V.done_f = sv->d_done_f.p; V.done_b = sv->d_done_b.p;
  V.bflag_f = sv->d_bflag_f.p; V.bflag_b = sv->d_bflag_b.p; V.bcnt = sv->d_bcnt.p; V.bcnt_b = sv->d_bcnt_b.p;
  V.boff = sv->d_boff.p; V.bigv_off = sv->d_bigv_off.p; V.bigv = sv->d_bigv.p; V.bigy = sv->d_bigy.p;
  V.part = SP.d_part.p; V.ccnt = SP.d_ccnt.p;
  V.ticket = sv->d_ticket.p;
  V.linv = sv->d_linv.p; V.linv_off = sv->d_linv_off.p;
  V.fdesc = sv->d_fdesc.p; V.gmap = sv->d_gmap.p; V.gmap_off = sv->d_gmap_off.p;
  V.subs = SP.d_subs.p; V.sub_meta = SP.d_sub_meta.p; V.subrow = SP.d_subrow.p; V.nsub = nsub;
  V.subpair = SP.d_subpair.p; V.npair = SP.npair; V.sub_Loff = SP.d_sub_Loff.p;
  V.upper_max = sv->opt.smem_front_max;
  V.tlog = nullptr;
  return B200LDLT_SUCCESS;
}

// per-front records shared by every solve plan: descriptors, gather maps of the big fronts, backward row addresses
static int build_solve_tables(Solver* sv, const Symbolic& S, cudaStream_t st) {
  const int nsn = S.nsn;
  // fronts owned by k_solve_direct: on the lowest levels, order <= 64, all children of the same kind (children precede parents)
  sv->solve_direct_front.assign(nsn, 0);
  for (int s = 0; s < nsn; ++s) {
    if (S.sn_level[s] >= sv->dbg.solve_direct || S.f(s) > 64) continue;
    bool all = true;
    for (int q = S.child_ptr[s]; q < S.child_ptr[s + 1]; ++q) all = all && sv->solve_direct_front[S.child_idx[q]];
    sv->solve_direct_front[s] = all ? 1 : 0;
  }
  std::vector<FrontDesc> fd(nsn);
  for (int s = 0; s < nsn; ++s) {
    FrontDesc& d = fd[s];
    d.c0 = S.sn_start[s]; d.k = (unsigned short)S.k(s); d.r = (unsigned short)S.r(s);
    d.ch0 = S.child_ptr[s];
    const int nch = S.child_ptr[s + 1] - S.child_ptr[s];
    if (nch > 65535) { sv->err = "front with more than 65535 children"; return B200LDLT_FATAL_ERROR; }
    d.nch = (unsigned short)nch; d.direct = (unsigned short)sv->solve_direct_front[s];
    d.L_off = S.L_off[s]; d.ro = S.rows_ptr[s];
  }
  CU(sv->d_fdesc.upload(fd, st));
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
    CU(sv->d_gmap_off.upload(goff, st));
    CU(sv->d_gmap.upload(gm, st));
  }
  return B200LDLT_SUCCESS;
}

static int upload_schur_lists(Solver* sv, SchurLists& SL, cudaStream_t st) {
  std::vector<TcFront> f = SL.f; std::vector<TcTile> t = SL.t; std::vector<int> d = SL.dfl;
  if (f.empty()) f.push_back(TcFront{0, 0, 0, 0, 0});
  if (t.empty()) t.push_back(TcTile{0, 0, 0});
  if (d.empty()) d.push_back(0);
  CU(SL.d_f.upload(f, st)); CU(SL.d_t.upload(t, st)); CU(SL.d_dfl.upload(d, st));
  if ((long long)sv->d_tc_dig.n < SL.dig_bytes) CU(sv->d_tc_dig.alloc(SL.dig_bytes));
  if ((long long)sv->d_tc_exp.n < SL.exp_ints) CU(sv->d_tc_exp.alloc(SL.exp_ints));
  return B200LDLT_SUCCESS;
}

static int run_analysis(Solver* sv, const double* vals) {
  // a (re-)analysis invalidates the factors and every buffer sized by the old plan
  sv->factored = false;
  sv->reanalyse = false;
  if (sv->h_rhs) { cudaFreeHost(sv->h_rhs); sv->h_rhs = nullptr; }
  sv->rhs_cap = 0;
  if (sv->fgraph_exec) { cudaGraphExecDestroy(sv->fgraph_exec); sv->fgraph_exec = nullptr; }
  if (sv->fgraph) { cudaGraphDestroy(sv->fgraph); sv->fgraph = nullptr; }
  AnalyseOptions ao;
  ao.ordering = sv->opt.ordering;
  ao.pair_saddle = sv->opt.pair_saddle;
  ao.leaf_k = sv->opt.leaf_k;
  ao.relax_frac = sv->opt.relax_frac;
  std::string e;
  int rc = analyse(sv->n, sv->nnz, sv->irn.data(), sv->jcn.data(), vals, ao, sv->S, e);
  if (rc != 0) { sv->err = e; return B200LDLT_FATAL_ERROR; }
  Symbolic& S = sv->S;
  cudaStream_t st = sv->stream;
  CU(sv->d_sn_start.upload(S.sn_start, st));
  CU(sv->d_sn_parent.upload(S.sn_parent, st));
  CU(sv->d_rows_ptr.upload(S.rows_ptr, st));
  CU(sv->d_rows.upload(S.rows, st));
  CU(sv->d_rel.upload(S.rel, st));
  CU(sv->d_child_ptr.upload(S.child_ptr, st));
  CU(sv->d_child_idx.upload(S.child_idx, st));
  CU(sv->d_uent_ptr.upload(S.uent_ptr, st));
  CU(sv->d_u_dst.upload(S.u_dst, st));
  CU(sv->d_u_dst64.upload(S.u_dst64, st));
  CU(sv->d_L_off.upload(S.L_off, st));
  CU(sv->d_cb_off.upload(S.cb_off, st));
  CU(sv->d_useg_ptr.upload(S.useg_ptr, st));
  CU(sv->d_useg_src.upload(S.useg_src, st));
  CU(sv->d_u_row.upload(S.u_row, st));
  CU(sv->d_u_col.upload(S.u_col, st));
  CU(sv->d_perm.upload(S.perm, st));
  CU(sv->d_irn.upload(sv->irn, st));
  CU(sv->d_jcn.upload(sv->jcn, st));
  const int n = S.n;
  CU(sv->d_vals.alloc(sv->nnz));
  CU(sv->d_uval.alloc(S.nnz_u));
  CU(sv->d_L.alloc(S.L_off[S.nsn]));
  CU(sv->d_W.alloc(S.L_off[S.nsn]));
  CU(sv->d_CB.alloc(std::max<int64_t>(S.cb_off[S.nsn], 1)));
  CU(sv->d_dinv.alloc(n)); CU(sv->d_doff.alloc(n)); CU(sv->d_scale.alloc(n));
  CU(sv->d_x.alloc(n)); CU(sv->d_rhs.alloc(n)); CU(sv->d_res.alloc(n));
  CU(sv->d_cbv.alloc(std::max<size_t>(S.rows.size(), 1)));
  CU(sv->d_ptype.alloc(n)); CU(sv->d_lperm.alloc(n)); CU(sv->d_bperm.alloc(n));
  CU(sv->d_counters.alloc(CNT_N));
  CU(sv->d_colmax.alloc(n));
  CU(sv->d_rmax.alloc(n));
  CU(cudaMemsetAsync(sv->d_rmax.p, 0, n * sizeof(unsigned long long), st));
  CU(cudaMemsetAsync(sv->d_L.p, 0, sv->d_L.n * sizeof(double), st));

  DevSym& D = sv->DS;
  D.n = n; D.nsn = S.nsn;
  D.sn_start = sv->d_sn_start.p; D.sn_parent = sv->d_sn_parent.p;
  D.rows_ptr = sv->d_rows_ptr.p; D.rows = sv->d_rows.p; D.rel = sv->d_rel.p;
  D.child_ptr = sv->d_child_ptr.p; D.child_idx = sv->d_child_idx.p;
  D.uent_ptr = sv->d_uent_ptr.p; D.u_dst = sv->d_u_dst.p; D.u_dst64 = sv->d_u_dst64.p;
  D.L_off = sv->d_L_off.p; D.cb_off = sv->d_cb_off.p;
  DevNum& N = sv->DN;
  N.L = sv->d_L.p; N.W = sv->d_W.p; N.CB = sv->d_CB.p; N.uval = sv->d_uval.p;
  N.dinv = sv->d_dinv.p; N.doff = sv->d_doff.p; N.ptype = sv->d_ptype.p;
  N.lperm = sv->d_lperm.p; N.bperm = sv->d_bperm.p; N.counters = sv->d_counters.p; N.colmax = sv->d_colmax.p;
  N.flog = nullptr;
  if (sv->dbg.factor_timeline) {
    const unsigned long long cap = 1ull << 16;
    CU(sv->d_flog.alloc(2 + cap * FLOG_WORDS));
    const unsigned long long hdr[2] = {0ull, cap};
    CU(cudaMemcpy(sv->d_flog.p, hdr, sizeof(hdr), cudaMemcpyHostToDevice));
    N.flog = sv->d_flog.p;
  }

  // inverse row maps of the children of the (factorisation-)big fronts, for the one-launch extend-add
  {
    std::vector<long long> eoff(S.nsn, -1);
    long long tot = 0;
    for (int c = 0; c < S.nsn; ++c) {
      const int p = S.sn_parent[c];
      if (p >= 0 && S.f(p) > sv->opt.smem_front_max) { eoff[c] = tot; tot += S.f(p); }
    }
    std::vector<int> einv((size_t)std::max<long long>(tot, 1), -1);
    for (int c = 0; c < S.nsn; ++c) if (eoff[c] >= 0) {
      const long long ro = S.rows_ptr[c];
      const int rc = S.r(c);
      for (int j = 0; j < rc; ++j) einv[(size_t)(eoff[c] + S.rel[ro + j])] = j;
    }
    CU(sv->d_einv_off.upload(eoff, st));
    CU(sv->d_einv.upload(einv, st));
    D.einv_off = sv->d_einv_off.p; D.einv = sv->d_einv.p;
  }

  // ---- launch plan: per level, big fronts first then small ones by descending order --------
  std::vector<int> fl;
  {
    std::vector<char> take(S.nsn, 1);
    build_level_plans(S, sv->opt.smem_front_max, take, fl, sv->plan, sv->dbg.buckets, sv->schur, sv->tc_min_r, !sv->dbg.no_warp2);
  }
  CU(sv->d_front_list.upload(fl, st));
  { int rc2 = upload_schur_lists(sv, sv->schur, st); if (rc2 != B200LDLT_SUCCESS) return rc2; }
  CU(cudaFuncSetAttribute(k_tc_schur, cudaFuncAttributeMaxDynamicSharedMemorySize, TC_SMEM_BYTES));
  CU(cudaFuncSetAttribute(k_big_panel, cudaFuncAttributeMaxDynamicSharedMemorySize, CHAIN_SMEM));
  CU(cudaFuncSetAttribute(k_front_warp2, cudaFuncAttributeMaxDynamicSharedMemorySize, 4 * S2_SMEM_PER_WARP));
  CU(cudaFuncSetAttribute(k_front_smem<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, 220 * 1024));
  CU(cudaFuncSetAttribute(k_front_smem<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, 64 * 1024));
  CU(cudaFuncSetAttribute(k_fwd_front, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
  CU(cudaFuncSetAttribute(k_bwd_front, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
  CU(cudaStreamSynchronize(st));


  // ---- triangular solves: flags, scratch, explicit-inverse work lists, plan ------------------------------
  {
    std::vector<int> boff(S.nsn, 0);
    sv->shard.active = false;
    std::vector<long long> bigv_off(S.nsn, 0);
    long long bv = 0; int bo = 0;
    for (int s = 0; s < S.nsn; ++s) if (S.f(s) > DF_MIDMAX) {
      boff[s] = bo; bo += (S.f(s) + DF_BLK - 1) / DF_BLK;
      bigv_off[s] = bv; bv += S.f(s) + (S.f(s) & 1);
    }
    // explicit inverses of the big fronts' pivot blocks (k_linv_*): K64 x K64 doubles per big front
    {
      std::vector<long long> linv_off(S.nsn, -1);
      long long tot = 0;
      for (int s = 0; s < S.nsn; ++s) if (S.f(s) > DF_MIDMAX) {
        linv_off[s] = tot;
        const long long K64 = (long long)((S.k(s) + DF_BLK - 1) / DF_BLK) * DF_BLK;
        tot += K64 * K64;
      }
      CU(sv->d_linv_off.upload(linv_off, st));
      CU(sv->d_linv.alloc(std::max<long long>(tot, 1)));
      CU(cudaMemsetAsync(sv->d_linv.p, 0, sv->d_linv.n * sizeof(double), st));
      std::vector<char> take(S.nsn, 1);
      int rc2 = build_linv_plan(sv, S, take, sv->linv_plan, st);
      if (rc2 != B200LDLT_SUCCESS) return rc2;
      sv->linv_level.clear();
      for (int l = 0; l < S.nlevels; ++l) {
        std::vector<char> tl(S.nsn, 0);
        bool any = false;
        for (int q = 0; q < S.nsn; ++q) if (S.sn_level[q] == l && S.f(q) > kSolveMidMax) { tl[q] = 1; any = true; }
        sv->linv_level.emplace_back(new LinvPlan());
        if (any) { rc2 = build_linv_plan(sv, S, tl, *sv->linv_level.back(), st); if (rc2 != B200LDLT_SUCCESS) return rc2; }
      }
    }
    CU(sv->d_boff.upload(boff, st));
    CU(sv->d_bigv_off.upload(bigv_off, st));
    CU(sv->d_done_f.alloc(S.nsn)); CU(sv->d_done_b.alloc(S.nsn));
    CU(sv->d_bcnt.alloc(S.nsn)); CU(sv->d_bcnt_b.alloc(S.nsn));
    CU(sv->d_bflag_f.alloc(std::max(bo, 1))); CU(sv->d_bflag_b.alloc(std::max(bo, 1)));
    CU(sv->d_bigv.alloc(std::max<long long>(bv, 1))); CU(sv->d_bigy.alloc(std::max<long long>(bv, 1)));
    CU(sv->d_ticket.alloc(2));
    CU(cudaMemsetAsync(sv->d_done_f.p, 0, S.nsn * sizeof(int), st));
    CU(cudaMemsetAsync(sv->d_done_b.p, 0, S.nsn * sizeof(int), st));
    CU(cudaMemsetAsync(sv->d_bcnt.p, 0, S.nsn * sizeof(int), st));
    CU(cudaMemsetAsync(sv->d_bcnt_b.p, 0, S.nsn * sizeof(int), st));
    CU(cudaMemsetAsync(sv->d_bflag_f.p, 0, std::max(bo, 1) * sizeof(int), st));
    CU(cudaMemsetAsync(sv->d_bflag_b.p, 0, std::max(bo, 1) * sizeof(int), st));
    CU(cudaMemsetAsync(sv->d_ticket.p, 0, 2 * sizeof(unsigned long long), st));
    sv->solve_epoch = 0; sv->ticket_f = sv->ticket_b = 0;
    {
      int rc2 = build_solve_tables(sv, S, st);
      if (rc2 != B200LDLT_SUCCESS) return rc2;
      std::vector<char> take(S.nsn, 1);
      rc2 = build_solve_plan(sv, S, take, sv->splan, st);
      if (rc2 != B200LDLT_SUCCESS) return rc2;
    }
    CU(cudaFuncSetAttribute(k_solve<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, DF_DYN_SMEM));
    CU(cudaFuncSetAttribute(k_solve<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, DF_DYN_SMEM));
    if (sv->dbg.solve_timeline) {
      CU(sv->d_tlog.alloc(2 * (size_t)(sv->splan.ntf + sv->splan.ntb) + 8 * (size_t)sv->splan.nsub + 8));
      sv->splan.V.tlog = sv->d_tlog.p;
    }
    int occ = 1;
    CU(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, k_solve<true>, DF_THREADS, DF_DYN_SMEM));
    int occ_b = 1;
    CU(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ_b, k_solve<false>, DF_THREADS, DF_DYN_SMEM));
    CU(cudaDeviceGetAttribute(&sv->num_sms, cudaDevAttrMultiProcessorCount, sv->dev));
    sv->df_grid = std::max(1, std::min(occ, occ_b)) * sv->num_sms;
    if (sv->opt.verbose)
      fprintf(stderr, "[b200ldlt] solve: %d big-front blocks, top grid %d x %d thr (%d/%d CTAs per SM)\n",
              bo, sv->df_grid, DF_THREADS, occ, occ_b);
    CU(cudaStreamSynchronize(st));
  }

  b200ldlt_info& I = sv->info;
  I.n = n; I.nnz_in = S.nnz_in; I.nnz_unique = S.nnz_u;
  I.nsupernodes = S.nsn; I.nlevels = S.nlevels; I.max_front = S.max_front; I.max_pivots = S.max_k;
  I.n_saddle = S.n_saddle; I.n_pairs = S.n_pairs;
  I.nnz_L = S.nnzL; I.nnz_L_true = S.nnzL_true;
  I.L_bytes = (int64_t)sv->d_L.n * 8; I.cb_bytes = (int64_t)sv->d_CB.n * 8;
  I.flops_panel = S.flops_panel; I.flops_schur = S.flops_schur;
  I.t_order_s = S.t_order; I.t_symbolic_s = S.t_symbolic;
  if (sv->opt.verbose)
    fprintf(stderr,
            "[b200ldlt] analyse: n=%d nnz=%lld uniq=%lld saddle=%d pairs=%d nsn=%d levels=%d maxfront=%d maxk=%d "
            "nnzL=%lld (true %lld) flops panel=%.3g schur=%.3g cb=%.1f MB  order %.2fs symbolic %.2fs\n",
            n, (long long)S.nnz_in, (long long)S.nnz_u, S.n_saddle, S.n_pairs, S.nsn, S.nlevels, S.max_front,
            S.max_k, (long long)S.nnzL, (long long)S.nnzL_true, S.flops_panel, S.flops_schur,
            S.cb_total * 8.0 / 1e6, S.t_order, S.t_symbolic);
  sv->analysed = true;
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

// enqueue the whole numeric factorisation of the values in d_vals
static int enqueue_factor(Solver* sv, const std::vector<LevelPlan>* plan_p = nullptr, const int* fl_p = nullptr,
                          bool prologue = true, const LinvPlan* linv_p = nullptr, const SchurLists* sl_p = nullptr) {
  const SchurLists& SL = sl_p ? *sl_p : sv->schur;
  Symbolic& S = sv->S;
  cudaStream_t st = sv->stream;
  DevSym& D = sv->DS;
  DevNum& N = sv->DN;
  N.u = sv->pivtol;
  N.tiny = sv->opt.tiny;
  const int n = S.n;
  const long long nu = S.nnz_u;
  const int* fl = fl_p ? fl_p : sv->d_front_list.p;
  const std::vector<LevelPlan>& plan = plan_p ? *plan_p : sv->plan;
  int& L = sv->launches;
  if (prologue) {
  L = 0;
  sv->ev_next = 0;
  CU(cudaMemsetAsync(sv->d_counters.p, 0, CNT_N * sizeof(int), st));
  CU(cudaMemsetAsync(sv->d_colmax.p, 0, (size_t)n * sizeof(double), st));
  if (sv->DN.flog) CU(cudaMemsetAsync(sv->DN.flog, 0, sizeof(unsigned long long), st));
  k_sum_dups<<<cdiv(nu, 256), 256, 0, st>>>(nu, sv->d_useg_ptr.p, sv->d_useg_src.p, sv->d_vals.p, sv->d_uval.p); ++L;
  k_fill<<<cdiv(n, 256), 256, 0, st>>>(n, sv->d_scale.p, 1.0); ++L;
  for (int sw = 0; sw < sv->opt.scaling; ++sw) {
    k_rowmax<<<cdiv(nu, 256), 256, 0, st>>>(nu, sv->d_u_row.p, sv->d_u_col.p, sv->d_uval.p, sv->d_scale.p, sv->d_rmax.p); ++L;
    k_scale_update<<<cdiv(n, 256), 256, 0, st>>>(n, sv->d_scale.p, sv->d_rmax.p); ++L;
  }
  if (sv->opt.scaling > 0) {
    k_apply_scale<<<cdiv(nu, 256), 256, 0, st>>>(nu, sv->d_u_row.p, sv->d_u_col.p, sv->d_scale.p, sv->d_uval.p); ++L;
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
  sv->mark("prologue", -1);
  for (int l = 0; l < S.nlevels; ++l) {
    const LevelPlan& P = plan[l];
    if (P.big_cnt) {
      const int* bl = fl + P.big_off;
      if (ev_zero_lvl[l]) CU(cudaStreamWaitEvent(st, ev_zero_lvl[l], 0));
      if (P.big_chmax > 0) {
        k_big_extend_all<<<dim3(cdiv(P.big_fmax, 8), P.big_cnt), 256, 0, st>>>(D, N, bl); ++L;
      }
    }
    if (P.big_cnt) sv->mark("big-assemble", l);
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
          k_front_smem<false><<<bk.cnt, bk.threads, bk.smem, sq>>>(D, N, fl + bk.off, bk.cnt, 0); ++L;
        }
      }
      used_side = used;
      // (the side streams are joined at the END of the level: this level's big fronts do not depend on its small fronts,
      //  so the panel chain below runs next to them)
    }
    sv->mark("small-fronts", l);
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
      sv->mark("big-chain", l);
      if (!linv_p && !sv->dbg.one_stream && l < (int)sv->linv_level.size() && sv->linv_level[l]->ndiag > 0) {
        // explicit L11 inverses of this level's fronts: behind the chain on their own stream, concurrent with the Schur
        // complements and the levels above (they only read the finished pivot blocks; k_linv_gemm<1> uses the top k x k
        // part of W as scratch, which nothing reads after the chain)
        cudaEvent_t e = sv->next_event();
        CU(cudaEventRecord(e, st));
        CU(cudaStreamWaitEvent(sv->stream3, e, 0));
        int rc = enqueue_linv(sv, *sv->linv_level[l], sv->stream3);
        if (rc != B200LDLT_SUCCESS) return rc;
        linv_forked = true;
      }
      // Schur complements CB -= L21 (L21 D)^T: tensor cores (Ozaki int8 digits, schur_tc.cu) for the large fronts,
      // register-blocked DFMA tiles for the rest
      if (P.tc_t_cnt > 0) {
        const TcFront* tf = SL.d_f.p + P.tc_f_off;
        k_tc_slice<<<dim3(cdiv(P.tc_rmax, 8), P.tc_f_cnt), 256, 0, st>>>(D, N, tf, 0, sv->d_tc_dig.p, sv->d_tc_exp.p); ++L;
        k_tc_slice<<<dim3(cdiv(P.tc_rmax, 8), P.tc_f_cnt), 256, 0, st>>>(D, N, tf, 1, sv->d_tc_dig.p, sv->d_tc_exp.p); ++L;
        k_tc_schur<<<P.tc_t_cnt, TC_THREADS, TC_SMEM_BYTES, st>>>(D, N, tf, SL.d_t.p + P.tc_t_off, sv->d_tc_dig.p, sv->d_tc_exp.p); ++L;
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
  sv->mark("big-schur(last)", S.nlevels);
  if (linv_forked) {
    cudaEvent_t e = sv->next_event();
    CU(cudaEventRecord(e, sv->stream3));
    CU(cudaStreamWaitEvent(st, e, 0));
  } else {
    int rc = enqueue_linv(sv, linv_p ? *linv_p : sv->linv_plan, st);
    if (rc != B200LDLT_SUCCESS) return rc;
  }
  sv->mark("linv", S.nlevels);
  CU(cudaGetLastError());
  return B200LDLT_SUCCESS;
}

// explicit inverses of the pivot blocks of the big fronts in LP (after their numeric factorisation): level 0 for all
// 64x64 diagonal blocks in one launch, then two tile-GEMM launches per doubling level (all fronts and pairs batched)
static int enqueue_linv(Solver* sv, const LinvPlan& LP, cudaStream_t st) {
  if (LP.ndiag <= 0) return B200LDLT_SUCCESS;
  int& L = sv->launches;
  k_linv_diag<<<LP.ndiag, 64, 0, st>>>(sv->DS, sv->DN, LP.d_diag.p, sv->d_linv_off.p, sv->d_linv.p); ++L;
  for (size_t l = 0; l < LP.ng.size(); ++l) {
    if (LP.ng[l] <= 0) continue;
    k_linv_gemm<1><<<LP.ng[l], 128, 0, st>>>(sv->DS, sv->DN, LP.d_g[l]->p, sv->d_linv_off.p, sv->d_linv.p, sv->d_linv_part.p, sv->d_linv_cnt.p); ++L;
    k_linv_gemm<2><<<LP.ng2[l], 128, 0, st>>>(sv->DS, sv->DN, LP.d_g2[l]->p, sv->d_linv_off.p, sv->d_linv.p, sv->d_linv_part.p, sv->d_linv_cnt.p); ++L;
  }
  CU(cudaGetLastError());
  return B200LDLT_SUCCESS;
}

static int finish_factor(Solver* sv, int check_inertia, int expected_neg, int* num_neg) {
  cudaStream_t st = sv->stream;
  CU(cudaEventRecord(sv->ev1, st));
  CU(cudaMemcpyAsync(sv->h_counters, sv->d_counters.p, CNT_N * sizeof(int), cudaMemcpyDeviceToHost, st));
  CU(cudaStreamSynchronize(st));
  float ms = 0;
  cudaEventElapsedTime(&ms, sv->ev0, sv->ev1);
  sv->dump_sections();
  b200ldlt_info& I = sv->info;
  I.ms_factor_gpu = ms;
  I.launches_factor = sv->launches;
  ++sv->n_factor;
  I.num_neg = sv->h_counters[CNT_NEG];
  I.num_forced = sv->h_counters[CNT_FORCED];
  I.num_tiny = sv->h_counters[CNT_TINY];
  I.num_growth = sv->h_counters[CNT_GROWTH];
  I.num_2x2 = sv->h_counters[CNT_2X2];
  sv->num_neg = I.num_neg;
  if (num_neg) *num_neg = I.num_neg;
  // Factors of a matrix with a noise pivot (SINGULAR) are not offered to the solves.  With num_forced > 0 the factors
  // (and the inertia reported) are those of a matrix perturbed by <= 1e-8 |column| in the lifted pivots; the count is
  // surfaced in b200ldlt_info and drives increase_quality (re-analysis with the current values).
  sv->factored = (I.num_tiny == 0);
  if (sv->opt.verbose > 1)
    fprintf(stderr, "[b200ldlt] factor: %.3f ms, %d launches, neg=%d 2x2=%d forced=%d tiny=%d growth=%d (u=%g)\n", ms,
            sv->launches, I.num_neg, I.num_2x2, I.num_forced, I.num_tiny, I.num_growth, sv->pivtol);
  if (I.num_tiny > 0) return B200LDLT_SINGULAR;
  if (check_inertia && I.num_neg != expected_neg) return B200LDLT_WRONG_INERTIA;
  return B200LDLT_SUCCESS;
}

static int do_factor(Solver* sv, const double* d_vals_ext_in, bool from_host, int check_inertia, int expected_neg,
                     int* num_neg) {
  const double* d_vals_ext = d_vals_ext_in;
  if (num_neg) *num_neg = -1;
  if (sv->n <= 0) { sv->err = "factor before analyse"; return B200LDLT_FATAL_ERROR; }
  CU(cudaSetDevice(sv->dev));
  if (!sv->analysed || sv->reanalyse) {
    if (sv->analysed) ++sv->n_reanalysed;
    std::vector<double> hv;
    const double* vals = sv->h_vals;
    if (!from_host && d_vals_ext) {
      hv.resize(sv->nnz);
      CU(cudaMemcpy(hv.data(), d_vals_ext, sv->nnz * sizeof(double), cudaMemcpyDeviceToHost));
      vals = hv.data();
    }
    int rc = run_analysis(sv, vals);
    if (rc != B200LDLT_SUCCESS) return rc;
    if (!from_host && d_vals_ext) {
      // the analysis re-allocated the device value array (d_vals_ext may have been that very array): restore it
      CU(cudaMemcpy(sv->d_vals.p, hv.data(), sv->nnz * sizeof(double), cudaMemcpyHostToDevice));
      d_vals_ext = sv->d_vals.p;
    }
  }
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
    if (!sv->fgraph_exec || sv->fgraph_u != sv->pivtol) {
      if (sv->fgraph_exec) { cudaGraphExecDestroy(sv->fgraph_exec); sv->fgraph_exec = nullptr; }
      if (sv->fgraph) { cudaGraphDestroy(sv->fgraph); sv->fgraph = nullptr; }
      CU(cudaStreamBeginCapture(st, cudaStreamCaptureModeThreadLocal));
      rc = enqueue_factor(sv);
      cudaError_t ce = cudaStreamEndCapture(st, &sv->fgraph);
      if (rc != B200LDLT_SUCCESS) return rc;
      CU(ce);
      CU(cudaGraphInstantiate(&sv->fgraph_exec, sv->fgraph, 0));
      sv->fgraph_u = sv->pivtol;
      sv->fgraph_launches = sv->launches;
    }
    sv->launches = sv->fgraph_launches;
    CU(cudaGraphLaunch(sv->fgraph_exec, st));
  } else {
    rc = enqueue_factor(sv);
    if (rc != B200LDLT_SUCCESS) return rc;
  }
  return finish_factor(sv, check_inertia, expected_neg, num_neg);
}

__global__ void k_mark_flags(int* flags, const int* __restrict__ list, int n, int value) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) flags[list[i]] = value;
}

// one sweep over the fronts of a plan: ONE persistent kernel (forward: subtrees then top tasks; backward: the reverse)
static int launch_sweep(Solver* sv, const SolvePlan& SP, bool fwd) {
  cudaStream_t st = sv->stream;
  const DevSolve& V = SP.V;
  const long long nt = (long long)(fwd ? SP.ntf : SP.ntb) + SP.npair;
  const int grid = (int)std::min<long long>(sv->df_grid, nt);
  const int nd = (int)SP.direct_cnt.size();
  auto direct = [&](int l) {
    if (SP.direct_cnt[l] <= 0) return;
    const unsigned g = cdiv(SP.direct_cnt[l], DF_THREADS / 32);
    if (fwd) k_solve_direct<true><<<g, DF_THREADS, 0, st>>>(sv->DS, sv->DN, V, SP.d_direct[l]->p, SP.direct_cnt[l], sv->solve_epoch, sv->d_x.p, sv->d_cbv.p);
    else k_solve_direct<false><<<g, DF_THREADS, 0, st>>>(sv->DS, sv->DN, V, SP.d_direct[l]->p, SP.direct_cnt[l], sv->solve_epoch, sv->d_x.p, sv->d_cbv.p);
    ++sv->launches;
  };
  if (fwd) {
    for (int l = 0; l < nd; ++l) direct(l);      // bottom levels first, one launch per level
    if (nt > 0) {
      k_solve<true><<<grid, DF_THREADS, DF_DYN_SMEM, st>>>(sv->DS, sv->DN, V, sv->solve_epoch, sv->ticket_f, sv->d_x.p, sv->d_cbv.p);
      sv->ticket_f += (unsigned long long)nt + grid;
      ++sv->launches;
    }
  } else {
    if (nt > 0) {
      k_solve<false><<<grid, DF_THREADS, DF_DYN_SMEM, st>>>(sv->DS, sv->DN, V, sv->solve_epoch, sv->ticket_b, sv->d_x.p, sv->d_cbv.p);
      sv->ticket_b += (unsigned long long)nt + grid;
      ++sv->launches;
    }
    for (int l = nd - 1; l >= 0; --l) direct(l);
  }
  CU(cudaGetLastError());
  return B200LDLT_SUCCESS;
}

static int enqueue_solve(Solver* sv, const double* d_b, double* d_out) {
  Symbolic& S = sv->S;
  cudaStream_t st = sv->stream;
  const int n = S.n;
  int& L = sv->launches;
  k_rhs_in<<<cdiv(n, 256), 256, 0, st>>>(n, sv->d_perm.p, sv->d_scale.p, d_b, sv->d_x.p); ++L;
  if (sv->opt.use_graph != 2) {   // default: subtree + task-queue sweeps (use_graph == 2 selects the level-per-launch kernels)
    sv->solve_epoch++;
    int rc = launch_sweep(sv, sv->splan, true);
    if (rc == B200LDLT_SUCCESS) rc = launch_sweep(sv, sv->splan, false);
    if (rc != B200LDLT_SUCCESS) return rc;
    k_sol_out<<<cdiv(n, 256), 256, 0, st>>>(n, sv->d_perm.p, sv->d_scale.p, sv->d_x.p, d_out); ++L;
    CU(cudaGetLastError());
    return B200LDLT_SUCCESS;
  }
  const int* fl = sv->d_front_list.p;
  for (int l = 0; l < S.nlevels; ++l) {
    const LevelPlan& P = sv->plan[l];
    int threads = P.fmax <= 64 ? 64 : (P.fmax <= 256 ? 256 : 1024);
    k_fwd_front<<<P.all_cnt, threads, 2 * (size_t)P.fmax * sizeof(double), st>>>(sv->DS, sv->DN, fl + P.all_off, sv->d_x.p, sv->d_cbv.p); ++L;
  }
  for (int l = S.nlevels - 1; l >= 0; --l) {
    const LevelPlan& P = sv->plan[l];
    int threads = P.fmax <= 64 ? 64 : (P.fmax <= 256 ? 256 : 1024);
    k_bwd_front<<<P.all_cnt, threads, (size_t)P.fmax * sizeof(double), st>>>(sv->DS, sv->DN, fl + P.all_off, sv->d_x.p); ++L;
  }
  k_sol_out<<<cdiv(n, 256), 256, 0, st>>>(n, sv->d_perm.p, sv->d_scale.p, sv->d_x.p, d_out); ++L;
  CU(cudaGetLastError());
  return B200LDLT_SUCCESS;
}

static int shard_setup(Solver* sv, int rank, int world) {
  Symbolic& S = sv->S;
  cudaStream_t st = sv->stream;
  Solver::Shard& H = sv->shard;
  H.rank = rank; H.world = world;
  H.nsub = shard_plan(S, world, H.owner);
  H.cut_roots.clear(); H.top_fronts.clear();
  std::vector<char> take[2];
  take[0].assign(S.nsn, 0); take[1].assign(S.nsn, 0);
  std::vector<int> mark_cut;
  for (int s = 0; s < S.nsn; ++s) {
    if (H.owner[s] < 0) { take[1][s] = (rank == 0); H.top_fronts.push_back(s); }
    else {
      take[0][s] = (H.owner[s] == rank);
      const int p = S.sn_parent[s];
      if (p >= 0 && H.owner[p] < 0) { H.cut_roots.push_back(s); if (H.owner[s] != 0) mark_cut.push_back(s); }
    }
  }
  for (int ph = 0; ph < 2; ++ph) {
    std::vector<int> fl;
    build_level_plans(S, sv->opt.smem_front_max, take[ph], fl, H.plan[ph], sv->dbg.buckets, H.schur[ph], sv->tc_min_r, !sv->dbg.no_warp2);
    { int rc2 = upload_schur_lists(sv, H.schur[ph], st); if (rc2 != B200LDLT_SUCCESS) return rc2; }
    { int rc2 = build_linv_plan(sv, S, take[ph], H.linv_plan[ph], st); if (rc2 != B200LDLT_SUCCESS) return rc2; }
    { int rc2 = build_solve_plan(sv, S, take[ph], H.splan[ph], st); if (rc2 != B200LDLT_SUCCESS) return rc2; }
    if (fl.empty()) fl.push_back(0);
    CU(H.d_fl[ph].upload(fl, st));
  }
  if (mark_cut.empty()) mark_cut.push_back(0), H.d_mark_cut.n = 0;
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
  o->use_graph = 1;   /* 1 = CUDA-graph replay of the factorisation + dataflow solve; 0 = plain launches; 2 = level-per-launch solve */
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
  sv->analysed = false; sv->factored = false; sv->have_dev_vals = false;
  if (sv->amat) { b200vec_tmat_destroy(sv->amat); sv->amat = nullptr; }
  if (sv->h_rhs) { cudaFreeHost(sv->h_rhs); sv->h_rhs = nullptr; }
  sv->rhs_cap = 0;   // staging buffers are sized by dim: a new structure invalidates them
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

int b200ldlt_solve_device(b200ldlt_handle h, int nrhs, double* d_rhs) {
  Solver* sv = (Solver*)h;
  if (!sv || !sv->factored) { if (sv) sv->err = "solve before factor"; return B200LDLT_FATAL_ERROR; }
  CU(cudaSetDevice(sv->dev));
  cudaStream_t st = sv->stream;
  sv->launches = 0;
  CU(cudaEventRecord(sv->ev0, st));
  for (int c = 0; c < nrhs; ++c) {
    double* col = d_rhs + (size_t)c * sv->n;
    int rc = enqueue_solve(sv, col, col);
    if (rc != B200LDLT_SUCCESS) return rc;
  }
  CU(cudaEventRecord(sv->ev1, st));
  CU(cudaStreamSynchronize(st));
  cudaEventElapsedTime(&sv->info.ms_solve_gpu, sv->ev0, sv->ev1);
  sv->info.launches_solve = sv->launches;
  return B200LDLT_SUCCESS;
}

int b200ldlt_solve(b200ldlt_handle h, int nrhs, double* rhs) {
  Solver* sv = (Solver*)h;
  if (!sv || !sv->factored) { if (sv) sv->err = "solve before factor"; return B200LDLT_FATAL_ERROR; }
  if (nrhs <= 0) return B200LDLT_SUCCESS;
  CU(cudaSetDevice(sv->dev));
  cudaStream_t st = sv->stream;
  const size_t n = sv->n;
  if (nrhs > sv->rhs_cap) {
    if (sv->h_rhs) cudaFreeHost(sv->h_rhs);
    sv->h_rhs = nullptr;
    CU(cudaHostAlloc((void**)&sv->h_rhs, n * nrhs * sizeof(double), cudaHostAllocDefault));
    CU(sv->d_rhs.alloc(n * nrhs));
    sv->rhs_cap = nrhs;
  }
  // Host rhs -> pinned staging -> device in chunks, so that the DMA of one chunk runs under the host copy of the next (the
  // caller's array is pageable: Ipopt allocates it per call, IpTSymLinearSolver.cpp:222-241); same on the way back.
  const size_t total = n * (size_t)nrhs;
  const size_t chunk = std::max<size_t>((total + 3) / 4, 32768);
  sv->launches = 0;
  CU(cudaEventRecord(sv->ev0, st));
  for (size_t o = 0; o < total; o += chunk) {
    const size_t m = std::min(chunk, total - o);
    memcpy(sv->h_rhs + o, rhs + o, m * sizeof(double));
    CU(cudaMemcpyAsync(sv->d_rhs.p + o, sv->h_rhs + o, m * sizeof(double), cudaMemcpyHostToDevice, st));
  }
  for (int c = 0; c < nrhs; ++c) {
    double* col = sv->d_rhs.p + (size_t)c * n;
    int rc = enqueue_solve(sv, col, col);
    if (rc != B200LDLT_SUCCESS) return rc;
  }
  int nchunk = 0;
  for (size_t o = 0; o < total; o += chunk, ++nchunk) {
    const size_t m = std::min(chunk, total - o);
    CU(cudaMemcpyAsync(sv->h_rhs + o, sv->d_rhs.p + o, m * sizeof(double), cudaMemcpyDeviceToHost, st));
    if (nchunk < 4) CU(cudaEventRecord(sv->ev_chunk[nchunk], st));
  }
  CU(cudaEventRecord(sv->ev1, st));
  nchunk = 0;
  for (size_t o = 0; o < total; o += chunk, ++nchunk) {
    const size_t m = std::min(chunk, total - o);
    if (nchunk < 4) CU(cudaEventSynchronize(sv->ev_chunk[nchunk])); else CU(cudaStreamSynchronize(st));
    memcpy(rhs + o, sv->h_rhs + o, m * sizeof(double));
  }
  CU(cudaStreamSynchronize(st));
  cudaEventElapsedTime(&sv->info.ms_solve_gpu, sv->ev0, sv->ev1);
  sv->info.launches_solve = sv->launches;
  return B200LDLT_SUCCESS;
}

/* debug: write the kernel timeline of the last factorisation (needs env B200_FACTOR_TIMELINE=1 at create time):
 * one line per record: kind s jb level k f t0 t1 ...  (kind: 1 chain role, 2 panel rows, 3 bulk update, 4 front (smem),
 * 5 front (warp), 6 Schur, 7 extend-add, 10-12 L11 inverse; times in ns of %globaltimer) */
int b200ldlt_dump_factor_timeline(b200ldlt_handle h, const char* path) {
  Solver* sv = (Solver*)h;
  if (!sv || !sv->DN.flog) return B200LDLT_FATAL_ERROR;
  std::vector<unsigned long long> t(sv->d_flog.n);
  CU(cudaMemcpy(t.data(), sv->d_flog.p, t.size() * sizeof(unsigned long long), cudaMemcpyDeviceToHost));
  FILE* fp = fopen(path, "w");
  if (!fp) return B200LDLT_FATAL_ERROR;
  const unsigned long long nrec = std::min(t[0], t[1]);
  for (unsigned long long i = 0; i < nrec; ++i) {
    const unsigned long long* r = t.data() + 2 + i * FLOG_WORDS;
    const int s = (int)(long long)r[1];
    const int k = sv->S.sn_start[s + 1] - sv->S.sn_start[s];
    const int f = k + (int)(sv->S.rows_ptr[s + 1] - sv->S.rows_ptr[s]);
    fprintf(fp, "%d %d %d %d %d %d", (int)r[0], s, (int)(long long)r[2], sv->S.sn_level[s], k, f);
    for (unsigned long long q = 0; q < r[3] && q < FLOG_WORDS - 4; ++q) fprintf(fp, " %llu", r[4 + q]);
    fprintf(fp, "\n");
  }
  fclose(fp);
  return B200LDLT_SUCCESS;
}

/* debug: write the per-task timeline of the last solve (needs env B200_SOLVE_TIMELINE=1 at analyse time) */
int b200ldlt_dump_solve_timeline(b200ldlt_handle h, const char* path) {
  Solver* sv = (Solver*)h;
  if (!sv || !sv->splan.V.tlog) return B200LDLT_FATAL_ERROR;
  std::vector<unsigned long long> t(sv->d_tlog.n);
  CU(cudaMemcpy(t.data(), sv->d_tlog.p, t.size() * sizeof(unsigned long long), cudaMemcpyDeviceToHost));
  FILE* fp = fopen(path, "w");
  if (!fp) return B200LDLT_FATAL_ERROR;
  for (size_t i = 0; i < sv->h_tasks.size(); ++i) {
    const SolveTask& T = sv->h_tasks[i];
    int s = T.type == ST_SMALL ? -1 : T.s;
    fprintf(fp, "%zu %d %d %d %d %d %llu %llu\n", i, i < (size_t)sv->splan.ntf ? 0 : 1, T.type, T.s, T.blk,
            s >= 0 ? sv->S.sn_level[s] : -1, t[2 * i], t[2 * i + 1]);
  }
  // subtree records: "S pass index start loaded end nfront nlv"
  const size_t base = 2 * (size_t)(sv->splan.ntf + sv->splan.ntb);
  for (int pass = 0; pass < 2; ++pass)
    for (int u = 0; u < sv->splan.nsub; ++u) {
      const unsigned long long* r = t.data() + base + 4 * ((size_t)pass * sv->splan.nsub + u);
      fprintf(fp, "S %d %d %llu %llu %llu %llu %llu\n", pass, u, r[0], r[1], r[2], r[3] >> 32, r[3] & 0xffffffffull);
    }
  fclose(fp);
  return B200LDLT_SUCCESS;
}

/* ---- multi-GPU elimination-tree sharding (SURVEY.md section 8e) -------------------------------------------
 * One process per GPU, each with its own handle and the SAME matrix.  After the (replicated, deterministic)
 * analysis, rank g factorises the subtrees it owns; the contribution blocks of the cut are moved to rank 0 by the
 * caller (NCCL send/recv through torch.distributed on the device pointers exported below), which then factorises
 * the top part.  The solve mirrors it.  See ipopt_b200/sharded.py for the orchestration. */
int b200ldlt_shard_setup(b200ldlt_handle h, int rank, int world) {
  Solver* sv = (Solver*)h;
  if (!sv || !sv->analysed || world < 1 || rank < 0 || rank >= world) { if (sv) sv->err = "shard_setup: analyse first / bad rank"; return B200LDLT_FATAL_ERROR; }
  CU(cudaSetDevice(sv->dev));
  return shard_setup(sv, rank, world);
}

int64_t b200ldlt_shard_array(b200ldlt_handle h, const char* name, int64_t* out, int64_t cap) {
  Solver* sv = (Solver*)h;
  if (!sv || !sv->shard.active || !name) return -1;
  const Solver::Shard& H = sv->shard;
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
  if (nm == "vals") return sv->d_vals.p;        // exists before the (lazy) analysis: assemble_augsys_device fills it
  if (!sv->analysed) return nullptr;
  if (nm == "CB") return sv->d_CB.p;
  if (nm == "cbv") return sv->d_cbv.p;
  if (nm == "x") return sv->d_x.p;
  if (nm == "counters") return sv->d_counters.p;
  return nullptr;
}

/* phase 0: (optional H2D of the pinned values array,) scaling + the subtrees owned by this rank;
 * phase 1: the top part (only rank 0 has work).  Enqueues on the handle's stream and returns. */
int b200ldlt_shard_factor(b200ldlt_handle h, int phase, int from_host) {
  Solver* sv = (Solver*)h;
  if (!sv || !sv->shard.active || phase < 0 || phase > 1) { if (sv) sv->err = "shard_factor: shard_setup first"; return B200LDLT_FATAL_ERROR; }
  CU(cudaSetDevice(sv->dev));
  cudaStream_t st = sv->stream;
  if (phase == 0) {
    CU(cudaEventRecord(sv->ev0, st));
    if (from_host) CU(cudaMemcpyAsync(sv->d_vals.p, sv->h_vals, sv->nnz * sizeof(double), cudaMemcpyHostToDevice, st));
    sv->have_dev_vals = true;
  }
  return enqueue_factor(sv, &sv->shard.plan[phase], sv->shard.d_fl[phase].p, phase == 0, &sv->shard.linv_plan[phase], &sv->shard.schur[phase]);
}

/* counters_total: CNT_N ints already summed over the ranks (all-reduce of device_ptr("counters")) */
int b200ldlt_shard_factor_finish(b200ldlt_handle h, const int* counters_total, int check_inertia, int expected_neg, int* num_neg) {
  Solver* sv = (Solver*)h;
  if (!sv || !sv->shard.active || !counters_total) return B200LDLT_FATAL_ERROR;
  CU(cudaSetDevice(sv->dev));
  CU(cudaEventRecord(sv->ev1, sv->stream));
  CU(cudaStreamSynchronize(sv->stream));
  cudaEventElapsedTime(&sv->info.ms_factor_gpu, sv->ev0, sv->ev1);
  b200ldlt_info& I = sv->info;
  I.launches_factor = sv->launches;
  I.num_neg = counters_total[CNT_NEG]; I.num_forced = counters_total[CNT_FORCED]; I.num_tiny = counters_total[CNT_TINY];
  I.num_growth = counters_total[CNT_GROWTH]; I.num_2x2 = counters_total[CNT_2X2];
  sv->num_neg = I.num_neg;
  if (num_neg) *num_neg = I.num_neg;
  sv->factored = (I.num_tiny == 0);
  if (I.num_tiny > 0) return B200LDLT_SINGULAR;
  if (check_inertia && I.num_neg != expected_neg) return B200LDLT_WRONG_INERTIA;
  return B200LDLT_SUCCESS;
}

/* phase 0: permute+scale rhs, forward sweep over my subtrees;  phase 1 (rank 0): forward + backward over the top;
 * phase 2: backward sweep over my subtrees;  phase 3: un-permute/un-scale into d_rhs.  d_rhs: dim doubles on the device. */
int b200ldlt_shard_solve(b200ldlt_handle h, int phase, double* d_rhs) {
  Solver* sv = (Solver*)h;
  if (!sv || !sv->shard.active || !sv->factored) { if (sv) sv->err = "shard_solve: factor first"; return B200LDLT_FATAL_ERROR; }
  CU(cudaSetDevice(sv->dev));
  cudaStream_t st = sv->stream;
  Solver::Shard& H = sv->shard;
  const int n = sv->n;
  int rc = B200LDLT_SUCCESS;
  if (phase == 0) {
    sv->launches = 0;
    k_rhs_in<<<cdiv(n, 256), 256, 0, st>>>(n, sv->d_perm.p, sv->d_scale.p, d_rhs, sv->d_x.p);
    sv->solve_epoch++;
    rc = launch_sweep(sv, H.splan[0], true);
  } else if (phase == 1) {
    if (H.d_mark_cut.n) k_mark_flags<<<cdiv((long long)H.d_mark_cut.n, 256), 256, 0, st>>>(sv->d_done_f.p, H.d_mark_cut.p, (int)H.d_mark_cut.n, sv->solve_epoch);
    rc = launch_sweep(sv, H.splan[1], true);
    if (rc == B200LDLT_SUCCESS) rc = launch_sweep(sv, H.splan[1], false);
  } else if (phase == 2) {
    if (H.rank != 0 && H.d_mark_top.n) k_mark_flags<<<cdiv((long long)H.d_mark_top.n, 256), 256, 0, st>>>(sv->d_done_b.p, H.d_mark_top.p, (int)H.d_mark_top.n, sv->solve_epoch);
    rc = launch_sweep(sv, H.splan[0], false);
  } else if (phase == 3) {
    k_sol_out<<<cdiv(n, 256), 256, 0, st>>>(n, sv->d_perm.p, sv->d_scale.p, sv->d_x.p, d_rhs);
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
  if (!sv->analysed && !sv->d_vals.p) CU(sv->d_vals.alloc(sv->nnz));   // (the lazy analysis re-allocates and keeps the contents: see do_factor)
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
  if (!sv || !sv->factored || !sv->have_dev_vals || !d_rhs) { if (sv) sv->err = "solve_refine: factor first (values on the device)"; return B200LDLT_FATAL_ERROR; }
  CU(cudaSetDevice(sv->dev));
  const int n = sv->n;
  if (!sv->vec) {
    sv->vec = b200vec_create(sv->dev, (void*)sv->stream);
    if (!sv->vec) { sv->err = "solve_refine: b200vec_create failed"; return B200LDLT_FATAL_ERROR; }
  }
  if (!sv->amat) {
    sv->amat = b200vec_tmat_create(sv->vec, n, n, sv->nnz, sv->irn.data(), sv->jcn.data(), 1);
    if (!sv->amat) { sv->err = "solve_refine: could not build the triplet operator"; return B200LDLT_FATAL_ERROR; }
  }
  if ((int)sv->d_ref_b.n < n) { CU(sv->d_ref_b.alloc(n)); CU(sv->d_ref_r.alloc(n)); }
  cudaStream_t st = sv->stream;
  CU(cudaMemcpyAsync(sv->d_ref_b.p, d_rhs, (size_t)n * sizeof(double), cudaMemcpyDeviceToDevice, st));
  sv->launches = 0;
  int rc = enqueue_solve(sv, d_rhs, d_rhs);
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
    rc = enqueue_solve(sv, sv->d_ref_r.p, sv->d_ref_r.p);     // d = A^-1 r
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
  if ((sv->info.num_forced > 0 || sv->info.num_growth > 0) && sv->analysed && !sv->shard.active && !sv->reanalysed_since_raise) {
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
  if (!sv->analysed) {
    if (sv->n <= 0) return -1;
    if (run_analysis(sv, nullptr) != B200LDLT_SUCCESS) return -1;
  }
  const Symbolic& S = sv->S;
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
#undef RET
  return -1;
}

int b200ldlt_residual(b200ldlt_handle h, const double* x, const double* b, double* r_inf, double* x_inf, double* b_inf) {
  Solver* sv = (Solver*)h;
  if (!sv || !sv->have_dev_vals) { if (sv) sv->err = "residual: no matrix on the device"; return B200LDLT_FATAL_ERROR; }
  CU(cudaSetDevice(sv->dev));
  cudaStream_t st = sv->stream;
  const int n = sv->n;
  DevBuf<double> dx, db;
  DevBuf<unsigned long long> dm;
  CU(dx.alloc(n)); CU(db.alloc(n)); CU(dm.alloc(3));
  CU(cudaMemcpyAsync(dx.p, x, n * sizeof(double), cudaMemcpyHostToDevice, st));
  CU(cudaMemcpyAsync(db.p, b, n * sizeof(double), cudaMemcpyHostToDevice, st));
  CU(cudaMemsetAsync(dm.p, 0, 3 * sizeof(unsigned long long), st));
  k_residual_init<<<cdiv(n, 256), 256, 0, st>>>(n, db.p, sv->d_res.p);
  k_residual_acc<<<cdiv(sv->nnz, 256), 256, 0, st>>>(sv->nnz, sv->d_irn.p, sv->d_jcn.p, sv->d_vals.p, dx.p, sv->d_res.p);
  k_absmax<<<cdiv(n, 256), 256, 0, st>>>(n, sv->d_res.p, dm.p);
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
