// Blocked triangular solve: a block of nb right-hand sides (2 <= nb <= MS_NB_MAX) through ONE forward and ONE backward
// sweep, with the work decomposition of solve_dataflow.cu (k_solve_direct bottom levels, the persistent k_solve with its
// subtree items and top tasks, the explicit L11^-1 of the big fronts).
//
// Every work item of the single-column sweep becomes nb items, one per column, issued next to each other in the ticket
// order: (item 0, col 0), (item 0, col 1), ..., (item 1, col 0), ...  Each column has its own copy of everything the
// single-column sweep writes -- x, update vectors, bigv / bigy, chunk partials and counters, done / block flags -- so an
// item runs the UNCHANGED single-column front routines of solve_dataflow.cu on its column's slices: the arithmetic of every
// column is the arithmetic of a single-column solve, bit for bit.  What the block shares: the launches, and the dependency
// latency of the sweep (direct levels, subtree walks, flag hops between top tasks) -- the nb columns run their chains side
// by side instead of one after the other.  What it does not share: every (item, column) stages its own panels (subtree and
// mid-front bulk copies), loads its own L / Linv tiles and waits on its own flags.  The items of a front are adjacent
// tickets, so the later copies may find the panel in L2.  Staging a front once per block and looping the columns over
// the staged tile is not built.
// Deadlock freedom carries over: an item only waits for items of its own column that are EARLIER in the ticket order
// (their single-column predecessors, nb times further back), and every ticket holder is resident.
#include <cuda_runtime.h>

#include "kernels.cuh"

namespace b200 {

#define MS_NB_MAX 8          // widest block; wider calls are cut into blocks of this many columns

// where column c of the width-nb solve state lives: base pointer (DevSolve / kernel argument) + c * stride
struct MultiStride {
  int nb;
  int nsn;                   // done_f, done_b, bcnt, bcnt_b
  int nbo;                   // bflag_f, bflag_b (big-front blocks)
  int nccnt;                 // chunk counters
  long long x, cbv;          // x (n), update vectors (rows)
  long long bigv;            // bigv, bigy
  long long part;            // chunk partials (64 doubles per slot)
};

__device__ __forceinline__ DevSolve column_view(const DevSolve& V, const MultiStride& M, int c) {
  DevSolve W = V;
  W.done_f += (long long)c * M.nsn; W.done_b += (long long)c * M.nsn;
  W.bcnt += (long long)c * M.nsn; W.bcnt_b += (long long)c * M.nsn;
  W.bflag_f += (long long)c * M.nbo; W.bflag_b += (long long)c * M.nbo;
  W.ccnt += (long long)c * M.nccnt;
  W.bigv += c * M.bigv; W.bigy += c * M.bigv;
  W.part += c * M.part;
  return W;
}

__device__ __forceinline__ void global_io(FrontIO& io, const DevSym& S, const DevNum& N, const DevSolve& V, double* x,
                                          double* cbv) {
  io.Lbase = N.L; io.L0 = 0; io.xs = x; io.col0 = 0; io.uv = cbv; io.ro0 = 0;
  io.dinv = N.dinv; io.doff = N.doff; io.ptype = N.ptype; io.lperm = N.lperm;
  io.rel = S.rel; io.subrow = nullptr; io.rootx = nullptr;
  io.fd = V.fdesc; io.s0 = 0; io.sR = S.nsn - 1; io.chi = S.child_idx; io.ch00 = 0;
  io.gfd = V.fdesc; io.gcbv = cbv; io.grel = S.rel; io.grows = S.rows; io.gx = x;
}

// permute + scale in / out, column blockIdx.y (same per-entry arithmetic as k_rhs_in / k_sol_out)
__global__ void k_rhs_in_multi(int n, const int* __restrict__ perm, const double* __restrict__ scale,
                               const double* __restrict__ b, double* __restrict__ xp, long long ldx) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  const long long c = blockIdx.y;
  if (i < n) { const int o = perm[i]; xp[c * ldx + i] = scale[o] * b[c * n + o]; }
}
__global__ void k_sol_out_multi(int n, const int* __restrict__ perm, const double* __restrict__ scale,
                                const double* __restrict__ xp, long long ldx, double* __restrict__ x) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  const long long c = blockIdx.y;
  if (i < n) { const int o = perm[i]; x[c * n + o] = scale[o] * xp[c * ldx + i]; }
}

// bottom levels: one warp per (front, column); the nb warps of a front are neighbours (panel from L1 / L2 after the first)
template <bool FWD>
__global__ void __launch_bounds__(DF_THREADS, 2) k_solve_direct_multi(DevSym S, DevNum N, DevSolve V, MultiStride M,
                                                                      const int* __restrict__ list, int cnt, int epoch,
                                                                      double* __restrict__ x, double* __restrict__ cbv) {
  __shared__ double wscr[(DF_THREADS / 32) * DF_WSCR];
  const int w = threadIdx.x >> 5;
  const int g = blockIdx.x * (DF_THREADS / 32) + w;
  if (g >= cnt * M.nb) return;
  const int c = g % M.nb;
  const DevSolve Vc = column_view(V, M, c);
  FrontIO io;
  global_io(io, S, N, Vc, x + c * M.x, cbv + c * M.cbv);
  const int s = list[g / M.nb];
  if (FWD) w64_fwd<false>(io, Vc, s, epoch, wscr + w * DF_WSCR);
  else w64_bwd<false>(io, Vc, s, epoch, -1, Vc.upper_max);
}

// the persistent sweep of k_solve (solve_dataflow.cu) over (work item, column) tickets
template <bool FWD>
__global__ void __launch_bounds__(DF_THREADS, 2) k_solve_multi(DevSym S, DevNum N, DevSolve V, MultiStride M, int epoch,
                                                               unsigned long long ticket_base,
                                                               double* __restrict__ x, double* __restrict__ cbv) {
  extern __shared__ __align__(16) unsigned char smraw[];
  __shared__ unsigned long long s_ticket;
  __shared__ unsigned long long s_mbar;
  __shared__ unsigned long long s_mbar1;
  __shared__ int s_flag;
  double* sm = reinterpret_cast<double*>(smraw);
  double* midscr = sm + (DF_THREADS / 32) * DF_WSCR;
  double* stage = midscr + DF_MIDSCR;
  const long long stage_doubles = (DF_DYN_SMEM / 8) - ((DF_THREADS / 32) * DF_WSCR + DF_MIDSCR);
  const SolveTask* tasks = FWD ? V.tasks : V.tasks_bwd;
  const int ntasks = FWD ? V.ntasks_fwd : V.ntasks_bwd;
  const unsigned long long nb = (unsigned long long)M.nb;
  const unsigned long long total = ((unsigned long long)ntasks + V.npair) * nb;
  unsigned mphase = 0, mphase1 = 0;
  const Team cta{(int)threadIdx.x, DF_THREADS, 0};
  if (threadIdx.x == 0) { mbar_init(&s_mbar, 1); mbar_init(&s_mbar1, 1); }
  __syncthreads();
  while (true) {
    if (threadIdx.x == 0) s_ticket = atomicAdd(V.ticket + (FWD ? 0 : 1), 1ull) - ticket_base;
    __syncthreads();
    const unsigned long long tk = s_ticket;
    __syncthreads();
    if (tk >= total) return;
    const unsigned long long item = tk / nb;
    const int c = (int)(tk - item * nb);
    const DevSolve Vc = column_view(V, M, c);
    double* xc = x + c * M.x;
    double* cbvc = cbv + c * M.cbv;
    const bool is_sub = FWD ? (item < (unsigned long long)V.npair) : (item >= (unsigned long long)ntasks);
    if (is_sub) {
      const int2 pr = V.subpair[FWD ? item : item - ntasks];
      const bool second = pr.y >= 0 && threadIdx.x >= DF_THREADS / 2;
      const Team tm = pr.y < 0 ? cta : Team{(int)threadIdx.x - (second ? DF_THREADS / 2 : 0), DF_THREADS / 2, second ? 2 : 1};
      solve_subtree<FWD>(S, N, Vc, second ? pr.y : pr.x, epoch, second ? smraw + V.subs[pr.x].sbytes : smraw,
                         second ? &s_mbar1 : &s_mbar, second ? mphase1 : mphase, xc, cbvc, tm);
      mphase ^= 1;
      if (pr.y >= 0) mphase1 ^= 1;
      __syncthreads();
      continue;
    }
    const SolveTask T = tasks[FWD ? item - V.npair : item];
    if (T.type == ST_SMALL || T.type == ST_MID) {
      FrontIO io;
      global_io(io, S, N, Vc, xc, cbvc);
      if (T.type == ST_SMALL) {
        const int w = threadIdx.x >> 5;
        if (w < T.blk) {
          const int s = V.bundle[T.s + w];
          if (FWD) w64_fwd<false>(io, Vc, s, epoch, sm + w * DF_WSCR);
          else w64_bwd<false>(io, Vc, s, epoch, S.sn_parent[s], V.upper_max);
        }
      } else {
        const FrontDesc fd = load_fd(V.fdesc + T.s);
        const long long pn = ((long long)(fd.k + fd.r) * fd.k + 1) & ~1LL;
        const double* Lp = nullptr;
        unsigned long long* mb = nullptr;
        unsigned ph = 0;
        if (pn <= stage_doubles) {
          if (threadIdx.x == 0) {
            asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
            mbar_expect_tx(&s_mbar, (unsigned)(pn * 8));
            bulk_g2s(stage, N.L + fd.L_off, (unsigned long long)pn * 8, &s_mbar);
          }
          Lp = stage; mb = &s_mbar; ph = mphase;
          mphase ^= 1;
        }
        if (FWD) mid_fwd<false>(io, Vc, T.s, epoch, midscr, Lp, mb, ph, cta);
        else mid_bwd<false>(io, Vc, T.s, epoch, S.sn_parent[T.s], midscr, Lp, mb, ph, V.upper_max, cta);
      }
    } else if (T.type == ST_FP) {
      big_fp(S, N, Vc, T, epoch, sm, &s_flag, xc, cbvc);
    } else if (T.type == ST_FC) {
      big_fc(S, N, Vc, T, epoch, sm, &s_flag, xc, cbvc);
    } else if (T.type == ST_BT) {
      big_bt(S, N, Vc, T, epoch, sm, &s_flag, xc);
    } else {
      big_bx(S, N, Vc, T, epoch, sm, &s_flag, xc);
    }
    __syncthreads();
  }
}

}  // namespace b200
