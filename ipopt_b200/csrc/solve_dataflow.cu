// Supernodal triangular solve (forward L, D^-1, backward L^T).  Per right-hand side and sweep:
//
//   k_solve_direct<FWD> : the lowest tree levels (fronts of order <= 64 whose children are of the same kind).  A level has
//                      no internal dependencies: one launch per level, one warp per front straight from global memory.
//   k_solve<FWD>      : ONE persistent kernel for everything else; CTAs take work items with an atomic ticket.
//     subtree items   : the tree below the big separator fronts is cut into subtrees whose whole working set -- the L
//                      panels of the fronts walked here, right-hand side, D, permutations, row maps, front descriptors --
//                      fits in shared memory.  TMA bulk copies (cp.async.bulk + mbarrier, one per front, compact layout)
//                      bring the panels in, then the subtree is walked level by level out of shared memory -- fronts of
//                      order <= 64 one warp each, larger ones by the team -- with hardware barriers only: no global flags,
//                      no atomics, no dependent global loads on the critical path; update vectors between the fronts of a
//                      subtree never leave shared memory.  A team is the whole CTA, or one half of it when two subtrees
//                      fit the shared memory together (named barriers, one transaction barrier each).  Largest first.
//     top tasks       : everything above the subtrees.  Fronts up to order 256 are one task each (panel staged in shared
//                      memory by a bulk copy when it fits); a front larger than that is cut into (64-row block) x (2-tile
//                      chunk) GEMV tasks on the EXPLICIT inverse of its pivot block (k_linv_*), so a separator front of
//                      order 1000+ keeps ~100 CTAs busy instead of a chain of block steps.  A task waits for its producers
//                      through ld.acquire/st.release flags; it only ever waits for tasks EARLIER in the (topologically
//                      sorted) list and every ticket holder is resident, so the scheme cannot deadlock.  Chunk partials
//                      are combined by the last-arriving CTA in chunk order (fence + counter): bit-reproducible.
// Forward: direct levels, then subtrees before top tasks; backward: top tasks before subtrees, then the direct levels.
// A block of right-hand sides takes the same launches through the MULTI instantiations of both kernels (see MultiStride).
// The partial solves (L, D, L^T on their own) use the forward sweep with APPLY_D = false, the backward sweep as is, and
// the pivot-order copies / D^-1 pass of solve_kernels.cu.
// L is streamed exactly once per sweep (HBM-bound, SURVEY.md 8d: 2*8*nnz(L) bytes per right-hand side); children ->
// parent data flows through per-front update vectors gathered by the parent (no atomics on the data path).
// Replaces the vendor back-solve of the reference (MUMPS job=3,
// reference src/Algorithm/LinearSolvers/IpMumpsSolverInterface.cpp:543-583).
#include <cuda_runtime.h>
#include <math.h>

#include "kernels.cuh"

namespace b200 {

#define DF_THREADS 256
#define DF_BLK 64            // block-row / block-column size of the big-front tasks
#define DF_CH 2              // 64x64 tiles per chunk task (both tiles are in flight before the task waits for its inputs)
#define DF_MIDMAX 256        // fronts above this order are "big" (block tasks + explicit L11 inverse)
#define DF_DYN_SMEM (100 * 1024)   // dynamic shared memory of both solve kernels (2 CTAs per SM)
#define DF_WSCR 64           // doubles of per-warp scratch (small fronts)
#define DF_MIDSCR 512        // doubles of CTA scratch for a mid front (v[f] | w[f], f <= 256)

enum { ST_SMALL = 0, ST_MID = 1, ST_FP = 2, ST_FC = 3, ST_BT = 4, ST_BX = 5 };

// ST_SMALL : s = offset into bundle[], blk = number of fronts (<= 8, one warp each, order <= 64)
// ST_MID   : s = front
// ST_FP/FC/BT/BX : s = front, blk = 64-block, tiles [t0, t1) of the contraction, chunk q of nq,
//                  pbase = first partial slot of (s, kind, blk), cidx = its arrival counter
struct SolveTask { int type, s, blk, t0, t1, q, nq, pbase, cidx, pad; };

// everything a front routine needs to know about a front, in ONE 32-byte record (two 16-byte loads from one sector)
struct __align__(16) FrontDesc {
  int c0;                  // first (permuted) column
  unsigned short k, r;     // pivot columns, contribution rows
  int ch0;                 // first entry in child_idx
  unsigned short nch, direct;   // direct != 0: the front is solved by k_solve_direct (bottom levels), never inside a subtree / task
  long long L_off;         // panel offset in L
  long long ro;            // offset of the row list / update vector (rows_ptr)
};

// one subtree of k_solve_sub: supernodes [s0, sR] (contiguous: postorder), its level schedule at meta[moff ...]:
//   meta[moff] = nlv ; then nlv+1 level offsets into the front list ; then nlv counts of small (order <= 64) fronts ;
//   then the front list itself (nfront ids, by level, small fronts first)
struct SubDesc {
  int s0, sR, moff, nlv;             // (meta: nlv+1 level offsets, nlv small counts, then the nown OWNED fronts by level)
  int col0, ncol, nrt, rroot, ch00, nchi, parent, sbytes;   // first column / #columns, #rows of all fronts / of the root, child list, parent of the root, shared-memory bytes (SubLayout, rounded up to 128)
  long long nL, ro0;                                     // doubles of the compact panel copy, first row-list offset
  int nown, pad;                                         // fronts walked here (the others in [s0, sR] are direct fronts)
};

struct DevSolve {
  const SolveTask* tasks;      // forward list (top part)
  const SolveTask* tasks_bwd;  // backward list
  int ntasks_fwd, ntasks_bwd;
  const int* bundle;           // front ids of the small bundles
  int* done_f;                 // nsn : epoch when the forward work of a front is complete
  int* done_b;                 // nsn : same for backward
  int* bflag_f;                // per (big front, pivot block): y block published
  int* bflag_b;                // per (big front, pivot block): t block published
  int* bcnt;                   // nsn : finished contribution-row blocks (monotonic)
  int* bcnt_b;                 // nsn : finished backward x blocks (monotonic)
  const int* boff;             // nsn : offset of a big front's blocks in bflag_*
  const long long* bigv_off;   // nsn : offset into bigv / bigy (f doubles per big front)
  double* bigv;                // big fronts: z = D^-1 y (forward), then t (backward), pivoted order
  double* bigy;                // big fronts: y (forward), pivoted order
  double* part;                // chunk partials, 64 doubles per slot
  int* ccnt;                   // chunk arrival counters (monotonic, modulo nq)
  unsigned long long* ticket;  // [0] fwd, [1] bwd (monotonic)
  const double* linv;          // explicit inverses of the big fronts' pivot blocks L11 (K64 x K64 each, see k_linv_*)
  const long long* linv_off;   // nsn : offset of a big front's inverse in linv, -1 = none
  const FrontDesc* fdesc;      // nsn
  const int* gmap;             // big fronts: gather map, gmap[gmap_off[s] + q*f + j] = index into cbv of the entry child q
  const long long* gmap_off;   //   adds to (pre-pivot) local row j of the parent, or -1
  const SubDesc* subs;         // subtrees of k_solve_sub
  const int* sub_meta;
  const int* subrow;           // aligned with rows: backward address of a contribution row inside its subtree:
                               //   >= 0 : column (local index into the subtree's x slice) ; < 0 : -(1 + index into the root's rows)
  int nsub;
  const int* sub_Loff;         // nsn : offset (doubles) of a front's panel inside its subtree's compact shared-memory copy
  const int2* subpair;         // work items of the subtree phase: (u0, u1) two subtrees walked side by side by the two halves
  int npair;                   //   of a CTA (their layouts fit the dynamic shared memory together), or (u0, -1) one subtree by the whole CTA
  int upper_max;               // fronts up to this order carry L11^T in the upper triangle of their pivot block
};

__device__ __forceinline__ int ld_acquire(const int* p) {
  int v;
  asm volatile("ld.acquire.gpu.global.s32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void st_release(int* p, int v) {
  asm volatile("st.release.gpu.global.s32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ void wait_eq(const int* p, int epoch) {
  while (ld_acquire(p) != epoch) __nanosleep(20);
}

// A team = the threads that work on one front / subtree together: the whole CTA (hardware barrier 0, identical to
// __syncthreads) or one half of it (barriers 1 / 2) when two subtrees share a CTA.
struct Team { int tid, nt, bar; };
__device__ __forceinline__ void team_sync(const Team& tm) {
  asm volatile("bar.sync %0, %1;" ::"r"(tm.bar), "r"(tm.nt) : "memory");
}

// ---- TMA 1-D bulk copy global -> shared with mbarrier completion (sm_90+; PTX cp.async.bulk) ---------------------
__device__ __forceinline__ unsigned smem_u32(const void* p) { return (unsigned)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(unsigned long long* bar, unsigned count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_expect_tx(unsigned long long* bar, unsigned bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(unsigned long long* bar, unsigned parity) {
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "WAIT_%=:\n"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
      "@p bra DONE_%=;\n"
      "bra WAIT_%=;\n"
      "DONE_%=:\n"
      "}\n" ::"r"(smem_u32(bar)), "r"(parity) : "memory");
}
// bytes: multiple of 16, both addresses 16-byte aligned; a single request may not exceed the mbarrier tx range -> split
__device__ __forceinline__ void bulk_g2s(void* dst, const void* src, unsigned long long bytes, unsigned long long* bar) {
  const unsigned long long CH = 64 * 1024;
  for (unsigned long long o = 0; o < bytes; o += CH) {
    const unsigned n = (unsigned)((bytes - o < CH) ? (bytes - o) : CH);
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                     smem_u32((const char*)dst + o)),
                 "l"((const char*)src + o), "r"(n), "r"(smem_u32(bar))
                 : "memory");
  }
}

// ------------------------------------------------------------------------------------------------
// Where a front routine finds its data.  SUB = true : shared-memory slices of one subtree (supernodes [s0, sR]); children
// outside that range (only with a sharded tree) are read from global memory.  SUB = false : the global arrays.
// ------------------------------------------------------------------------------------------------
struct FrontIO {
  const double* Lbase; long long L0;     // panel of front s at Lbase + (fd.L_off - L0)
  double* xs; int col0;                  // right-hand side / solution entry of column c at xs[c - col0]
  double* uv; long long ro0;             // update vector of front s at uv + (fd.ro - ro0)
  const double* dinv; const double* doff; const int* ptype; const int* lperm;   // [c - col0]
  const int* rel;                        // [ro - ro0 + j]
  const int* subrow; const double* rootx;   // SUB, backward: addresses of the contribution rows (see DevSolve::subrow)
  const FrontDesc* fd; int s0, sR;       // descriptors: fd[s - s0]
  const int* chi; int ch00;              // child lists: chi[ch - ch00]
  // global arrays (children outside a subtree; rows of ancestors)
  const FrontDesc* gfd; const double* gcbv; const int* grel; const int* grows; const double* gx;
};

template <bool SUB>
__device__ __forceinline__ double ldv(const double* p) { return SUB ? *p : __ldcg(p); }

__device__ __forceinline__ FrontDesc load_fd(const FrontDesc* p) {
  const int4 a = reinterpret_cast<const int4*>(p)[0], b = reinterpret_cast<const int4*>(p)[1];
  FrontDesc d;
  d.c0 = a.x; d.k = (unsigned short)(a.y & 0xffff); d.r = (unsigned short)((unsigned)a.y >> 16);
  d.ch0 = a.z; d.nch = (unsigned short)(a.w & 0xffff); d.direct = (unsigned short)((unsigned)a.w >> 16);
  d.L_off = ((long long)(unsigned)b.x) | ((long long)b.y << 32);
  d.ro = ((long long)(unsigned)b.z) | ((long long)b.w << 32);
  return d;
}

// ------------------------------------------------------------------------------------------------
// fronts of order <= 64: one warp per front, two rows per lane (lane, lane+32)
// scratch per warp: w[64]
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ void w64_load8(const double* __restrict__ P, int f, int k, int i0, int i1, int tb,
                                          double (&l0)[8], double (&l1)[8]) {
#pragma unroll
  for (int q = 0; q < 8; ++q) {
    const int t = tb + q;
    l0[q] = (t < k && i0 > t && i0 < f) ? P[i0 + (size_t)t * f] : 0.0;
    l1[q] = (t < k && i1 > t && i1 < f) ? P[i1 + (size_t)t * f] : 0.0;
  }
}
__device__ __forceinline__ void w64_fstep8(int k, int tb, const double (&l0)[8], const double (&l1)[8], double& v0,
                                           double& v1) {
#pragma unroll
  for (int q = 0; q < 8; ++q) {
    const int t = tb + q;
    if (t < k) {   // warp-uniform
      const double yt = (t < 32) ? __shfl_sync(0xffffffffu, v0, t) : __shfl_sync(0xffffffffu, v1, t - 32);
      v0 = fma(-l0[q], yt, v0);
      v1 = fma(-l1[q], yt, v1);
    }
  }
}

// D^-1 of the pivot rows: dinv_entry (solve_kernels.cu).  APPLY_D = false (partial solve, L only): the pivot rows keep v = the L-solve value instead of D^-1 v
template <bool SUB, bool APPLY_D = true>
__device__ void w64_fwd(const FrontIO& io, const DevSolve& V, int s, int epoch, double* w) {
  const int lane = threadIdx.x & 31;
  const FrontDesc fd = load_fd(io.fd + (s - io.s0));
  const int k = fd.k, r = fd.r, f = k + r, nch = fd.nch;
  const int cl = fd.c0 - io.col0;
  const long long rol = fd.ro - io.ro0;
  const int i0 = lane, i1 = lane + 32;
  const double* __restrict__ P = io.Lbase + (fd.L_off - io.L0);
  double a0[8], a1[8], b0[8], b1[8];
  w64_load8(P, f, k, i0, i1, 0, a0, a1);            // (global: in flight while the children are gathered)
  w[i0] = (i0 < k) ? io.xs[cl + i0] : 0.0;
  w[i1] = (i1 < k) ? io.xs[cl + i1] : 0.0;
  const int lp0 = (i0 < k) ? io.lperm[cl + i0] : i0, lp1 = (i1 < k) ? io.lperm[cl + i1] : i1;
  __syncwarp();
  for (int q0 = 0; q0 < nch; q0 += 32) {
    // child metadata lane-parallel, then the children one after the other (their targets may overlap); the
    // (index, value) pairs of child q+1 are in flight while child q is added
    const int m = min(32, nch - q0);
    int rq = 0, inq = 1;
    long long oq = 0;
    if (lane < m) {
      const int c = io.chi[fd.ch0 - io.ch00 + q0 + lane];
      inq = (!SUB) || (c >= io.s0 && c <= io.sR);
      const FrontDesc cd = load_fd(inq ? io.fd + (c - io.s0) : io.gfd + c);
      if (SUB && cd.direct) inq = 0;      // solved by the direct kernel before this sweep: its update vector is in global memory
      oq = cd.ro; rq = cd.r;
      if (!SUB) wait_eq(V.done_f + c, epoch);
    }
    __syncwarp();
    int nidx0 = 0, nidx1 = 0;
    double nval0 = 0.0, nval1 = 0.0;
    bool nok0 = false, nok1 = false;
    auto fetch = [&](int q) {
      const long long o = __shfl_sync(0xffffffffu, oq, q);
      const int rc = __shfl_sync(0xffffffffu, rq, q);
      const int in = __shfl_sync(0xffffffffu, inq, q);
      const int* __restrict__ rl = (SUB && in) ? io.rel + (o - io.ro0) : io.grel + o;
      const double* __restrict__ src = (SUB && in) ? io.uv + (o - io.ro0) : io.gcbv + o;
      nok0 = lane < rc; nok1 = lane + 32 < rc;
      if (SUB && in) {
        if (nok0) { nidx0 = rl[lane]; nval0 = src[lane]; }
        if (nok1) { nidx1 = rl[lane + 32]; nval1 = src[lane + 32]; }
      } else {
        if (nok0) { nidx0 = rl[lane]; nval0 = __ldcg(src + lane); }
        if (nok1) { nidx1 = rl[lane + 32]; nval1 = __ldcg(src + lane + 32); }
      }
    };
    fetch(0);
    for (int q = 0; q < m; ++q) {
      const int idx0 = nidx0, idx1 = nidx1;
      const double val0 = nval0, val1 = nval1;
      const bool ok0 = nok0, ok1 = nok1;
      if (q + 1 < m) fetch(q + 1);
      if (ok0) w[idx0] += val0;   // rel is strictly increasing inside a child: no two lanes hit the same entry
      if (ok1) w[idx1] += val1;
      __syncwarp();
    }
  }
  double v0 = (i0 < f) ? w[lp0] : 0.0, v1 = (i1 < f) ? w[lp1] : 0.0;
  for (int tb = 0; tb < k; tb += 16) {
    if (tb + 8 < k) w64_load8(P, f, k, i0, i1, tb + 8, b0, b1);
    w64_fstep8(k, tb, a0, a1, v0, v1);
    if (tb + 16 < k) w64_load8(P, f, k, i0, i1, tb + 16, a0, a1);
    if (tb + 8 < k) w64_fstep8(k, tb + 8, b0, b1, v0, v1);
  }
  // D^-1: partner values through shared memory (w is free now)
  __syncwarp();
  w[i0] = v0; w[i1] = v1;
  __syncwarp();
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int i = lane + 32 * h;
    const double v = h ? v1 : v0;
    if (i < k) {
      double y = v;
      if (APPLY_D) {
        const int ty = io.ptype[cl + i];
        if (ty == 1) y = dinv_entry(1, v, 0.0, io.dinv[cl + i], 0.0);
        else if (ty == 2) y = dinv_entry(2, v, w[i + 1], io.dinv[cl + i], io.doff[cl + i]);
        else y = dinv_entry(3, v, w[i - 1], io.dinv[cl + i], io.doff[cl + i - 1]);
      }
      io.xs[cl + i] = y;
    } else if (i < f) io.uv[rol + i - k] = v;
  }
  __syncwarp();
  if (!SUB && lane == 0) st_release(V.done_f + s, epoch);
}

// sum over the 32 lanes of p[t], t = 0..31: lane t receives the total of column t (31 shuffles instead of 32 x 5)
__device__ __forceinline__ double warp_transpose_reduce(double (&p)[32]) {
  const int lane = threadIdx.x & 31;
#pragma unroll
  for (int j = 0; j < 16; ++j) {
    const bool hi = lane & 16;
    const double send = hi ? p[j] : p[j + 16], keep = hi ? p[j + 16] : p[j];
    p[j] = keep + __shfl_xor_sync(0xffffffffu, send, 16);
  }
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    const bool hi = lane & 8;
    const double send = hi ? p[j] : p[j + 8], keep = hi ? p[j + 8] : p[j];
    p[j] = keep + __shfl_xor_sync(0xffffffffu, send, 8);
  }
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const bool hi = lane & 4;
    const double send = hi ? p[j] : p[j + 4], keep = hi ? p[j + 4] : p[j];
    p[j] = keep + __shfl_xor_sync(0xffffffffu, send, 4);
  }
#pragma unroll
  for (int j = 0; j < 2; ++j) {
    const bool hi = lane & 2;
    const double send = hi ? p[j] : p[j + 2], keep = hi ? p[j + 2] : p[j];
    p[j] = keep + __shfl_xor_sync(0xffffffffu, send, 2);
  }
  {
    const bool hi = lane & 1;
    const double send = hi ? p[0] : p[1], keep = hi ? p[1] : p[0];
    p[0] = keep + __shfl_xor_sync(0xffffffffu, send, 1);
  }
  return p[0];
}

// value of contribution row j of the front (backward): the solution entry of that (ancestor) column
template <bool SUB>
__device__ __forceinline__ double cb_row_x(const FrontIO& io, long long rol, long long ro, int j) {
  if (SUB) {
    const int a = io.subrow[rol + j];
    return a >= 0 ? io.xs[a] : io.rootx[-a - 1];
  }
  return __ldcg(io.gx + io.grows[ro + j]);
}

template <bool SUB>
__device__ void w64_bwd(const FrontIO& io, const DevSolve& V, int s, int epoch, int parent, int upper_max) {
  const int lane = threadIdx.x & 31;
  const FrontDesc fd = load_fd(io.fd + (s - io.s0));
  const int k = fd.k, r = fd.r, f = k + r;
  const int cl = fd.c0 - io.col0;
  const long long rol = fd.ro - io.ro0;
  const int i0 = lane, i1 = lane + 32;
  const double* __restrict__ P = io.Lbase + (fd.L_off - io.L0);
  if (!SUB) {
    if (parent >= 0 && lane == 0) wait_eq(V.done_b + parent, epoch);
    __syncwarp();
  }
  double v0 = 0.0, v1 = 0.0;  // entries i0 / i1 of [D^-1 y ; x(rows)]
  if (i0 < k) v0 = io.xs[cl + i0]; else if (i0 < f) v0 = cb_row_x<SUB>(io, rol, fd.ro, i0 - k);
  if (i1 < k) v1 = io.xs[cl + i1]; else if (i1 < f) v1 = cb_row_x<SUB>(io, rol, fd.ro, i1 - k);
  const int lp0 = (i0 < k) ? io.lperm[cl + i0] : 0, lp1 = (i1 < k) ? io.lperm[cl + i1] : 0;
  if (k <= 32) {
    // (1) rectangular part  u_t = sum_{i >= k} L[i,t] v_i : no chain -- column loads with lane = row, per-lane
    //     products for all 32 columns, one transposing warp reduction (lane t gets u_t)
    const bool cb0 = i0 >= k && i0 < f, cb1 = i1 < f;
    const double m0 = cb0 ? v0 : 0.0, m1 = cb1 ? v1 : 0.0;
    double p[32];
#pragma unroll
    for (int tb = 0; tb < 32; tb += 8) {
      double l0[8], l1[8];
#pragma unroll
      for (int q = 0; q < 8; ++q) {
        const int t = tb + q;
        l0[q] = (t < k && cb0) ? P[i0 + (size_t)t * f] : 0.0;
        l1[q] = (t < k && cb1) ? P[i1 + (size_t)t * f] : 0.0;
      }
#pragma unroll
      for (int q = 0; q < 8; ++q) p[tb + q] = fma(l0[q], m0, l1[q] * m1);
    }
    const double u = warp_transpose_reduce(p);
    // (2) triangle, lane t owns column t:  z_t -= L[ii][t] x_ii for ii = k-1 .. t+1.  Row ii of L11 is read from the
    //     UPPER triangle of the pivot block, where the factorisation stored L11^T: P[t + ii*f], t < ii -- contiguous
    //     across the lanes (the lower triangle would be a stride-f gather).
    double z = (lane < k) ? v0 - u : 0.0;
    for (int tb = ((k - 1) >> 3) << 3; tb >= 0; tb -= 8) {
      double lr[8];
#pragma unroll
      for (int q = 0; q < 8; ++q) {
        const int ii = tb + q;
        lr[q] = (ii < k && lane < ii) ? (f <= upper_max ? P[lane + (size_t)ii * f] : P[ii + (size_t)lane * f]) : 0.0;
      }
#pragma unroll
      for (int q = 7; q >= 0; --q) {
        const int ii = tb + q;
        if (ii < k && ii >= 1) {   // warp-uniform
          const double xi = __shfl_sync(0xffffffffu, z, ii);
          z = fma(-lr[q], xi, z);
        }
      }
    }
    if (lane < k) io.xs[cl + lp0] = z;
  } else {
    // columns from the last to the first: v_t -= sum_{i>t} L[i,t] v_i  (column read with lane = row, warp-sum)
    for (int tb = k - 1; tb >= 0; tb -= 8) {
      double l0[8], l1[8];
#pragma unroll
      for (int q = 0; q < 8; ++q) {
        const int t = tb - q;
        l0[q] = (t >= 0 && i0 > t && i0 < f) ? P[i0 + (size_t)t * f] : 0.0;
        l1[q] = (t >= 0 && i1 > t && i1 < f) ? P[i1 + (size_t)t * f] : 0.0;
      }
#pragma unroll
      for (int q = 0; q < 8; ++q) {
        const int t = tb - q;
        if (t >= 0) {
          double part = fma(l0[q], v0, l1[q] * v1);
#pragma unroll
          for (int o = 16; o > 0; o >>= 1) part += __shfl_xor_sync(0xffffffffu, part, o);
          if (t < 32) { if (lane == t) v0 -= part; } else { if (lane == t - 32) v1 -= part; }
        }
      }
    }
    // (all lanes must have read their z entries before the permuted write-back: the reads happened at the top)
    if (i0 < k) io.xs[cl + lp0] = v0;
    if (i1 < k) io.xs[cl + lp1] = v1;
  }
  __syncwarp();
  if (!SUB && lane == 0) st_release(V.done_b + s, epoch);
}

// ------------------------------------------------------------------------------------------------
// mid fronts (65 .. 256): one CTA, blocked by 32; scratch: v[f] | w[f]
// ------------------------------------------------------------------------------------------------
template <bool SUB, bool APPLY_D = true>
__device__ void mid_fwd(const FrontIO& io, const DevSolve& V, int s, int epoch, double* scr, const double* Lp_override,
                        unsigned long long* mbar, unsigned mphase, const Team tm) {
  const FrontDesc fd = load_fd(io.fd + (s - io.s0));
  const int k = fd.k, r = fd.r, f = k + r, nch = fd.nch;
  const int cl = fd.c0 - io.col0;
  const long long rol = fd.ro - io.ro0;
  double* v = scr;
  double* w = scr + f;
  const int tid = tm.tid, nt = tm.nt, lane = tid & 31, warp = tid >> 5;
  if (!SUB) for (int q = tid; q < nch; q += nt) wait_eq(V.done_f + io.chi[fd.ch0 - io.ch00 + q], epoch);
  for (int i = tid; i < f; i += nt) w[i] = (i < k) ? io.xs[cl + i] : 0.0;
  team_sync(tm);
  for (int q = 0; q < nch; ++q) {
    const int c = io.chi[fd.ch0 - io.ch00 + q];
    const bool inr = (!SUB) || (c >= io.s0 && c <= io.sR);
    const FrontDesc cd = load_fd(inr ? io.fd + (c - io.s0) : io.gfd + c);
    const bool in = inr && !cd.direct;
    const int rc = cd.r;
    if (SUB && in) {
      const int* __restrict__ rl = io.rel + (cd.ro - io.ro0);
      const double* __restrict__ src = io.uv + (cd.ro - io.ro0);
      for (int t = tid; t < rc; t += nt) w[rl[t]] += src[t];
    } else {
      const int* __restrict__ rl = io.grel + cd.ro;
      const double* __restrict__ src = io.gcbv + cd.ro;
      for (int t = tid; t < rc; t += nt) w[rl[t]] += __ldcg(src + t);
    }
    team_sync(tm);
  }
  const int* __restrict__ lp = io.lperm + cl;
  for (int i = tid; i < f; i += nt) v[i] = (i < k) ? w[lp[i]] : w[i];
  team_sync(tm);
  const double* __restrict__ P = Lp_override ? Lp_override : io.Lbase + (fd.L_off - io.L0);
  if (mbar) mbar_wait(mbar, mphase);   // the staged panel (bulk copy issued by the caller) has landed
  for (int t0 = 0; t0 < k; t0 += 32) {
    const int nb = min(32, k - t0);
    if (warp == 0) {
      // the triangle of this 32-block: lane = row; the block column is read 8 entries ahead of the shuffle chain
      double yi = (lane < nb) ? v[t0 + lane] : 0.0;
      for (int qb = 0; qb < nb; qb += 8) {
        double l[8];
#pragma unroll
        for (int q = 0; q < 8; ++q) l[q] = (qb + q < nb && lane > qb + q && lane < nb) ? P[(t0 + lane) + (size_t)(t0 + qb + q) * f] : 0.0;
#pragma unroll
        for (int q = 0; q < 8; ++q) {
          if (qb + q < nb) {
            const double yq = __shfl_sync(0xffffffffu, yi, qb + q);
            yi = fma(-l[q], yq, yi);
          }
        }
      }
      if (lane < nb) v[t0 + lane] = yi;
    }
    team_sync(tm);
    for (int i = t0 + nb + tid; i < f; i += nt) {
      double acc = 0.0;
#pragma unroll 8
      for (int q = 0; q < nb; ++q) acc = fma(P[i + (size_t)(t0 + q) * f], v[t0 + q], acc);
      v[i] -= acc;
    }
    team_sync(tm);
  }
  for (int t = tid; t < k; t += nt) {
    double y = v[t];
    if (APPLY_D) {
      const int ty = io.ptype[cl + t];
      if (ty == 1) y = dinv_entry(1, v[t], 0.0, io.dinv[cl + t], 0.0);
      else if (ty == 2) y = dinv_entry(2, v[t], v[t + 1], io.dinv[cl + t], io.doff[cl + t]);
      else y = dinv_entry(3, v[t], v[t - 1], io.dinv[cl + t], io.doff[cl + t - 1]);
    }
    io.xs[cl + t] = y;
  }
  double* __restrict__ out = io.uv + rol;
  for (int i = tid; i < r; i += nt) out[i] = v[k + i];
  team_sync(tm);
  if (!SUB && tid == 0) st_release(V.done_f + s, epoch);
}

template <bool SUB>
__device__ void mid_bwd(const FrontIO& io, const DevSolve& V, int s, int epoch, int parent, double* scr,
                        const double* Lp_override, unsigned long long* mbar, unsigned mphase, int upper_max, const Team tm) {
  const FrontDesc fd = load_fd(io.fd + (s - io.s0));
  const int k = fd.k, r = fd.r, f = k + r;
  const int cl = fd.c0 - io.col0;
  const long long rol = fd.ro - io.ro0;
  double* v = scr;
  const int tid = tm.tid, nt = tm.nt, lane = tid & 31, warp = tid >> 5, nwarp = nt >> 5;
  if (!SUB) {
    if (parent >= 0 && tid == 0) wait_eq(V.done_b + parent, epoch);
    team_sync(tm);
  }
  for (int i = tid; i < f; i += nt) v[i] = (i < k) ? io.xs[cl + i] : cb_row_x<SUB>(io, rol, fd.ro, i - k);
  team_sync(tm);
  const double* __restrict__ P = Lp_override ? Lp_override : io.Lbase + (fd.L_off - io.L0);
  if (mbar) mbar_wait(mbar, mphase);
  const int nblk = (k + 31) / 32;
  for (int b = nblk - 1; b >= 0; --b) {
    const int t0 = b * 32, nb = min(32, k - t0);
    for (int q = warp; q < nb; q += nwarp) {
      const double* col = P + (size_t)(t0 + q) * f;
      double acc = 0.0;
      for (int i = t0 + nb + lane; i < f; i += 32) acc = fma(col[i], v[i], acc);
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
      if (lane == 0) v[t0 + q] -= acc;
    }
    team_sync(tm);
    if (warp == 0) {
      // triangle of this block: lane t owns column t; row q of the block comes from L11^T in the upper triangle when the
      // factorisation stored it (fronts up to order 128), else from the lower triangle (stride-f gather)
      double zi = (lane < nb) ? v[t0 + lane] : 0.0;
      const bool upper = f <= upper_max;
      for (int qb = ((nb - 1) >> 3) << 3; qb >= 0; qb -= 8) {
        double l[8];
#pragma unroll
        for (int q = 0; q < 8; ++q) {
          const int qq = qb + q;
          l[q] = (qq < nb && lane < qq) ? (upper ? P[(t0 + lane) + (size_t)(t0 + qq) * f] : P[(t0 + qq) + (size_t)(t0 + lane) * f]) : 0.0;
        }
#pragma unroll
        for (int q = 7; q >= 0; --q) {
          const int qq = qb + q;
          if (qq < nb && qq >= 1) {   // warp-uniform
            const double zq = __shfl_sync(0xffffffffu, zi, qq);
            zi = fma(-l[q], zq, zi);
          }
        }
      }
      if (lane < nb) v[t0 + lane] = zi;
    }
    team_sync(tm);
  }
  const int* __restrict__ lp = io.lperm + cl;
  for (int t = tid; t < k; t += nt) io.xs[cl + lp[t]] = v[t];
  team_sync(tm);
  if (!SUB && tid == 0) st_release(V.done_b + s, epoch);
}

// ------------------------------------------------------------------------------------------------
// Big fronts (order > 256).  With the EXPLICIT inverse of the unit-lower-triangular pivot block L11 (k_linv_* below,
// once per factorisation) the in-front recurrences become block GEMVs with no chain:
//   forward   FP: y_b   = sum_{c<=b} Linv[b,c] w_c          (w = assembled, pivot-permuted right-hand side)
//             FC: u_j   = w_j - L21[j,:] y                   (update vector handed to the parent)
//   backward  BT: t_b   = z_b - L21[:,b]^T x(rows)           (z = D^-1 y)
//             BX: x_b   = sum_{c>=b} Linv[c,b]^T t_c
// Each (64-block, chunk of <= DF_CH tiles) is one task; ALL tiles of a chunk are in flight before the task waits for its
// inputs, and the w entries it needs are gathered on the fly from the children's update vectors through a precomputed
// gather map (V.gmap: parent row -> entry of each child's update vector) -- no separate gather task, no staging buffer.
// The right-hand side of a big front stays in x[c0..c0+k) until BX overwrites it with the solution: the forward result
// z lives in V.bigv (so FP tasks of other blocks can still read the right-hand side).
// smem: stage[128] | part[256] | ys[64] | red[128] | colacc[64]
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ double big_gather_row(const DevSolve& V, int s, int j, int k, int f, int c0, int nch,
                                                 const double* __restrict__ x, const double* __restrict__ cbv) {
  const int* __restrict__ gm = V.gmap + V.gmap_off[s] + j;
  double v = (j < k) ? x[c0 + j] : 0.0;
  for (int q = 0; q < nch; ++q) {   // fixed child order: deterministic
    const int e = gm[(size_t)q * f];
    if (e >= 0) v += __ldcg(cbv + e);
  }
  return v;
}

// Combine the chunk partials of one (front, kind, block): every CTA stores its 64 partial sums, the LAST one to arrive
// adds them in chunk order (independent of the arrival order).  `out` (shared, 64 doubles) holds this CTA's partial on
// entry and the total on exit.  Returns true (in all threads) for the CTA that must finalise the block.
__device__ __forceinline__ bool chunk_combine(const DevSolve& V, const SolveTask& T, double* out, int* s_flag) {
  if (T.nq == 1) return true;
  const int tid = threadIdx.x;
  if (tid < 64) __stcg(V.part + ((long long)T.pbase + T.q) * 64 + tid, out[tid]);
  __syncthreads();
  if (tid == 0) {
    __threadfence();                                    // release: this CTA's partial before the counter
    const int old = atomicAdd(V.ccnt + T.cidx, 1);
    const int last = ((old + 1) % T.nq) == 0;
    if (last) __threadfence();                          // acquire: the other CTAs' partials after the counter
    *s_flag = last;
  }
  __syncthreads();
  if (!*s_flag) return false;
  if (tid < 64) {
    const double* base = V.part + (long long)T.pbase * 64 + tid;
    double a = 0.0;
    for (int q = 0; q < T.nq; ++q) a += __ldcg(base + (long long)q * 64);
    out[tid] = a;
  }
  __syncthreads();
  return true;
}

// sum the per-thread partials pacc[q] (column t = ty + 4q, row lane tx) over the 64 row lanes -> colacc[64] (smem)
__device__ __forceinline__ void reduce_cols(double (&pacc)[16], double* red, double* colacc) {
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
#pragma unroll
  for (int q = 0; q < 16; ++q) {
    double a = pacc[q];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) a += __shfl_xor_sync(0xffffffffu, a, o);
    if (lane == 0) red[warp * 16 + q] = a;
  }
  __syncthreads();
  if (tid < 64) {
    // column t = tid: ty = t & 3, q = t >> 2 ; warps 2*ty and 2*ty+1 hold the two halves
    const int tyc = tid & 3, q = tid >> 2;
    colacc[tid] = red[(2 * tyc) * 16 + q] + red[(2 * tyc + 1) * 16 + q];
  }
  __syncthreads();
}

// FP: pivot rows [64 blk, +64) of front s, tiles [t0, t1) of Linv's block row.  APPLY_D = false: bigv gets y, not D^-1 y.
template <bool APPLY_D>
__device__ void big_fp(const DevSym& S, const DevNum& N, const DevSolve& V, const SolveTask& T, int epoch, double* sm,
                       int* s_flag, const double* __restrict__ x, const double* __restrict__ cbv) {
  const int s = T.s, rb = T.blk;
  const FrontDesc fd = load_fd(V.fdesc + s);
  const int c0 = fd.c0, k = fd.k;
  const int nkb = (k + DF_BLK - 1) / DF_BLK;
  const long long K64 = (long long)nkb * DF_BLK;
  const int tid = threadIdx.x, tx = tid & 63, ty = tid >> 6;
  double* stage = sm;
  double* part = sm + 128;
  double* ys = part + 256;
  const int r0 = rb * DF_BLK, nrow = min(DF_BLK, k - r0);
  const double* __restrict__ Li = V.linv + V.linv_off[s] + (r0 + tx);
  // both tiles in flight before the children are seen (Linv does not depend on the right-hand side)
  const int f = k + fd.r;
  const bool two = T.t1 - T.t0 > 1;
  double la[16], lb[16];
#pragma unroll
  for (int q = 0; q < 16; ++q) la[q] = Li[((long long)T.t0 * DF_BLK + ty + 4 * q) * K64];
#pragma unroll
  for (int q = 0; q < 16; ++q) lb[q] = two ? Li[((long long)(T.t0 + 1) * DF_BLK + ty + 4 * q) * K64] : 0.0;
  const int ch0 = fd.ch0, nch = fd.nch;
  // gather addresses of this thread's stage entry (they do not depend on the right-hand side): pivot permutation ->
  // per-child index into cbv; up to 4 children in registers, more through the map again
  const int ncols = (T.t1 - T.t0) * DF_BLK;     // <= 128 <= DF_THREADS: one stage entry per thread
  const int gi = T.t0 * DF_BLK + tid;
  int gsrc[4] = {-1, -1, -1, -1};
  int jrow = -1;
  if (tid < ncols && gi < k) {
    jrow = N.lperm[c0 + gi];
    const int* __restrict__ gm = V.gmap + V.gmap_off[s] + jrow;
#pragma unroll
    for (int q = 0; q < 4; ++q) if (q < nch) gsrc[q] = gm[(size_t)q * f];
  }
  // D of this block (finalisation) -- prefetched as well
  int ty2 = 1;
  double dv = 0.0, dof = 0.0, dofm = 0.0;
  if (tid < nrow) {
    const int i = r0 + tid;
    ty2 = N.ptype[c0 + i]; dv = N.dinv[c0 + i]; dof = N.doff[c0 + i];
    if (i > 0) dofm = N.doff[c0 + i - 1];
  }
  for (int q = tid; q < nch; q += DF_THREADS) wait_eq(V.done_f + S.child_idx[ch0 + q], epoch);
  __syncthreads();
  if (tid < ncols) {
    double v = 0.0;
    if (jrow >= 0) {
      v = x[c0 + jrow];
#pragma unroll
      for (int q = 0; q < 4; ++q) if (gsrc[q] >= 0) v += __ldcg(cbv + gsrc[q]);
      if (nch > 4) {
        const int* __restrict__ gm = V.gmap + V.gmap_off[s] + jrow;
        for (int q = 4; q < nch; ++q) { const int e = gm[(size_t)q * f]; if (e >= 0) v += __ldcg(cbv + e); }
      }
    }
    stage[tid] = v;
  }
  __syncthreads();
  double acc = 0.0;
  {
    const double* wc = stage + ty;
#pragma unroll
    for (int q = 0; q < 16; ++q) acc = fma(la[q], wc[4 * q], acc);
    if (two) {
      const double* wd = stage + DF_BLK + ty;
#pragma unroll
      for (int q = 0; q < 16; ++q) acc = fma(lb[q], wd[4 * q], acc);
    }
  }
  part[ty * 64 + tx] = acc;
  __syncthreads();
  if (tid < 64) ys[tid] = part[tid] + part[64 + tid] + part[128 + tid] + part[192 + tid];
  __syncthreads();
  if (!chunk_combine(V, T, ys, s_flag)) return;
  if (tid < nrow) {
    const int i = r0 + tid;
    const long long o = V.bigv_off[s];
    V.bigy[o + i] = ys[tid];              // y block for the contribution rows (pivoted order)
    double z = ys[tid];                    // 2x2 partners never straddle a 32-column panel, so they sit in this block
    if (APPLY_D) {
      if (ty2 == 1) z = dinv_entry(1, ys[tid], 0.0, dv, 0.0);
      else if (ty2 == 2) z = dinv_entry(2, ys[tid], ys[tid + 1], dv, dof);
      else z = dinv_entry(3, ys[tid], ys[tid - 1], dv, dofm);
    }
    V.bigv[o + i] = z;
  }
  __syncthreads();
  if (tid == 0) st_release(V.bflag_f + V.boff[s] + rb, epoch);
}

// FC: contribution rows [k + 64 blk, +64), tiles [t0, t1) of L21's block row
__device__ void big_fc(const DevSym& S, const DevNum& N, const DevSolve& V, const SolveTask& T, int epoch, double* sm,
                       int* s_flag, const double* __restrict__ x, double* __restrict__ cbv) {
  const int s = T.s, j = T.blk;
  const FrontDesc fd = load_fd(V.fdesc + s);
  const int c0 = fd.c0, k = fd.k;
  const int f = k + fd.r;
  const int tid = threadIdx.x, tx = tid & 63, ty = tid >> 6;
  double* stage = sm;
  double* part = sm + 128;
  double* ys = part + 256;
  const int rbase = k + j * DF_BLK, nr = min(DF_BLK, f - rbase);
  const double* __restrict__ P = N.L + fd.L_off + (rbase + tx);
  const bool two = T.t1 - T.t0 > 1;
  double la[16], lb[16];
  {
    const int tc0 = T.t0 * DF_BLK, ncn = min(DF_BLK, k - tc0);
    const double* nx = P + (size_t)tc0 * f;
#pragma unroll
    for (int q = 0; q < 16; ++q) { const int t = ty + 4 * q; la[q] = (tx < nr && t < ncn) ? nx[(size_t)t * f] : 0.0; }
    const int tc1 = tc0 + DF_BLK, ncm = two ? min(DF_BLK, k - tc1) : 0;
    const double* ny = P + (size_t)tc1 * f;
#pragma unroll
    for (int q = 0; q < 16; ++q) { const int t = ty + 4 * q; lb[q] = (tx < nr && t < ncm) ? ny[(size_t)t * f] : 0.0; }
  }
  // addresses of this row's assembled right-hand side entry (needed by the finalising CTA): prefetched
  int gsrc[4] = {-1, -1, -1, -1};
  if (tid < nr) {
    const int* __restrict__ gm = V.gmap + V.gmap_off[s] + (rbase + tid);
#pragma unroll
    for (int q = 0; q < 4; ++q) if (q < fd.nch) gsrc[q] = gm[(size_t)q * f];
  }
  for (int c = T.t0 + tid; c < T.t1; c += DF_THREADS) wait_eq(V.bflag_f + V.boff[s] + c, epoch);
  __syncthreads();
  {
    const double* __restrict__ yb = V.bigy + V.bigv_off[s];
    const int ncols = (T.t1 - T.t0) * DF_BLK;
    for (int i = tid; i < ncols; i += DF_THREADS) {
      const int gi = T.t0 * DF_BLK + i;
      stage[i] = (gi < k) ? __ldcg(yb + gi) : 0.0;
    }
  }
  __syncthreads();
  double acc = 0.0;
  {
    const double* yc = stage + ty;
#pragma unroll
    for (int q = 0; q < 16; ++q) acc = fma(la[q], yc[4 * q], acc);
    if (two) {
      const double* yd = stage + DF_BLK + ty;
#pragma unroll
      for (int q = 0; q < 16; ++q) acc = fma(lb[q], yd[4 * q], acc);
    }
  }
  part[ty * 64 + tx] = acc;
  __syncthreads();
  if (tid < 64) ys[tid] = part[tid] + part[64 + tid] + part[128 + tid] + part[192 + tid];
  __syncthreads();
  if (!chunk_combine(V, T, ys, s_flag)) return;
  if (tid < nr) {
    // the children are complete (every FP task of this front waited for them before publishing the flags seen above)
    double wv = 0.0;
#pragma unroll
    for (int q = 0; q < 4; ++q) if (gsrc[q] >= 0) wv += __ldcg(cbv + gsrc[q]);
    if (fd.nch > 4) {
      const int* __restrict__ gm = V.gmap + V.gmap_off[s] + (rbase + tid);
      for (int q = 4; q < fd.nch; ++q) { const int e = gm[(size_t)q * f]; if (e >= 0) wv += __ldcg(cbv + e); }
    }
    cbv[fd.ro + (rbase - k) + tid] = wv - ys[tid];
  }
  __syncthreads();
  if (tid == 0) {
    const int ncb = (f - k + DF_BLK - 1) / DF_BLK;
    __threadfence();                                 // this block's update vector before the counter
    const int old = atomicAdd(V.bcnt + s, 1);
    if ((old + 1) % ncb == 0) { __threadfence(); st_release(V.done_f + s, epoch); }
  }
}

// BT: column block blk, contribution-row tiles [t0, t1):  t_b = z_b - L21[:, b]^T x(rows)
__device__ void big_bt(const DevSym& S, const DevNum& N, const DevSolve& V, const SolveTask& T, int epoch, double* sm,
                       int* s_flag, const double* __restrict__ x) {
  const int s = T.s, b = T.blk;
  const FrontDesc fd = load_fd(V.fdesc + s);
  const int k = fd.k;
  const long long ro = fd.ro;
  const int r = fd.r, f = k + r;
  const int tid = threadIdx.x, tx = tid & 63, ty = tid >> 6;
  double* stage = sm;
  double* red = sm + 448;
  double* colacc = red + 128;
  const int tc0 = b * DF_BLK, ncol = min(DF_BLK, k - tc0);
  const double* __restrict__ P = N.L + fd.L_off + (size_t)tc0 * f;
  double pacc[16];
#pragma unroll
  for (int q = 0; q < 16; ++q) pacc[q] = 0.0;
  const bool one = T.t1 - T.t0 > 0, two = T.t1 - T.t0 > 1;
  double la[16], lb[16];
  {
    const int rb2 = k + T.t0 * DF_BLK, nr2 = one ? min(DF_BLK, f - rb2) : 0;
    const double* base = P + (rb2 + tx);
#pragma unroll
    for (int q = 0; q < 16; ++q) { const int t = ty + 4 * q; la[q] = (tx < nr2 && t < ncol) ? base[(size_t)t * f] : 0.0; }
    const int rb3 = rb2 + DF_BLK, nr3 = two ? min(DF_BLK, f - rb3) : 0;
    const double* base3 = P + (rb3 + tx);
#pragma unroll
    for (int q = 0; q < 16; ++q) { const int t = ty + 4 * q; lb[q] = (tx < nr3 && t < ncol) ? base3[(size_t)t * f] : 0.0; }
  }
  const int nrows = (T.t1 - T.t0) * DF_BLK;     // <= 128: one stage entry per thread
  const int rix = T.t0 * DF_BLK + tid;
  const int grow = (tid < nrows && rix < r) ? S.rows[ro + rix] : -1;   // row id prefetched before the wait
  {
    const int par = S.sn_parent[s];
    if (par >= 0 && tid == 0) wait_eq(V.done_b + par, epoch);
  }
  __syncthreads();
  if (tid < nrows) stage[tid] = (grow >= 0) ? __ldcg(x + grow) : 0.0;
  __syncthreads();
  {
    const double xa = one ? stage[tx] : 0.0, xb = two ? stage[DF_BLK + tx] : 0.0;
#pragma unroll
    for (int q = 0; q < 16; ++q) pacc[q] = fma(la[q], xa, lb[q] * xb);
  }
  reduce_cols(pacc, red, colacc);
  if (!chunk_combine(V, T, colacc, s_flag)) return;
  if (tid < ncol) {
    double* tv = V.bigv + V.bigv_off[s] + tc0 + tid;
    *tv = *tv - colacc[tid];            // z (written by FP in the forward sweep) -> t, in place
  }
  __syncthreads();
  if (tid == 0) st_release(V.bflag_b + V.boff[s] + b, epoch);
}

// BX: column block blk, tiles [t0, t1) of Linv's block column (t0 >= blk):  x_b = sum_c Linv[c,b]^T t_c
__device__ void big_bx(const DevSym& S, const DevNum& N, const DevSolve& V, const SolveTask& T, int epoch, double* sm,
                       int* s_flag, double* __restrict__ x) {
  const int s = T.s, b = T.blk;
  const FrontDesc fd = load_fd(V.fdesc + s);
  const int c0 = fd.c0, k = fd.k;
  const int nkb = (k + DF_BLK - 1) / DF_BLK;
  const long long K64 = (long long)nkb * DF_BLK;
  const int tid = threadIdx.x, tx = tid & 63, ty = tid >> 6;
  double* stage = sm;
  double* red = sm + 448;
  double* colacc = red + 128;
  const int tc0 = b * DF_BLK, ncol = min(DF_BLK, k - tc0);
  const double* __restrict__ Li = V.linv + V.linv_off[s] + (long long)tc0 * K64 + tx;
  const double* __restrict__ tv = V.bigv + V.bigv_off[s];
  double pacc[16];
#pragma unroll
  for (int q = 0; q < 16; ++q) pacc[q] = 0.0;
  const bool two = T.t1 - T.t0 > 1;
  double la[16], lb[16];
#pragma unroll
  for (int q = 0; q < 16; ++q) la[q] = Li[(long long)T.t0 * DF_BLK + (long long)(ty + 4 * q) * K64];
#pragma unroll
  for (int q = 0; q < 16; ++q) lb[q] = two ? Li[(long long)(T.t0 + 1) * DF_BLK + (long long)(ty + 4 * q) * K64] : 0.0;
  const int lpo = (tid < ncol) ? N.lperm[c0 + tc0 + tid] : 0;   // (prefetched: needed by the finalising CTA)
  for (int c = T.t0 + tid; c < T.t1; c += DF_THREADS) wait_eq(V.bflag_b + V.boff[s] + c, epoch);
  __syncthreads();
  {
    const int nrows = (T.t1 - T.t0) * DF_BLK;
    for (int i = tid; i < nrows; i += DF_THREADS) {
      const int gi = T.t0 * DF_BLK + i;
      stage[i] = (gi < k) ? __ldcg(tv + gi) : 0.0;
    }
  }
  __syncthreads();
  {
    const double ta = stage[tx], tb2 = two ? stage[DF_BLK + tx] : 0.0;
#pragma unroll
    for (int q = 0; q < 16; ++q) pacc[q] = fma(la[q], ta, lb[q] * tb2);
  }
  reduce_cols(pacc, red, colacc);
  if (!chunk_combine(V, T, colacc, s_flag)) return;
  if (tid < ncol) x[c0 + lpo] = colacc[tid];   // final value (the permutation is panel-local)
  __syncthreads();
  if (tid == 0) {
    __threadfence();                                 // this block's solution entries before the counter
    const int old = atomicAdd(V.bcnt_b + s, 1);
    if ((old + 1) % nkb == 0) { __threadfence(); st_release(V.done_b + s, epoch); }
  }
}

// ------------------------------------------------------------------------------------------------
// Explicit inverse of the pivot block L11 of the big fronts, once per factorisation, by recursive doubling:
//   level 0 : the 64x64 diagonal blocks (k_linv_diag: one thread per column, the column in registers);
//   level l : [A 0; B C]^-1 = [A^-1 0; -C^-1 B A^-1  C^-1] for all pairs of neighbouring blocks of 64*2^(l-1)
//             columns, as two batched 64x64-tile GEMM passes (k_linv_gemm<1>: T = B A^-1 into the W scratch of the
//             factorisation, k_linv_gemm<2>: -C^-1 T into Linv).  Work items are enumerated on the host at analysis.
// ------------------------------------------------------------------------------------------------
// front, tile row / column (64-blocks), k-range of tiles [m0, m1).  Long k-ranges are cut into nch chunks (this item is
// chunk ci): the chunks write their partial tiles to scratch slot `slot` and the last one to arrive adds them up in chunk
// order (deterministic) -- the launch then ends with a chunk, not with its longest dot product.  slot = first scratch tile
// of the item (= index of its arrival counter).
struct LinvItem { int s, ib, jb, m0, m1, nch, ci, slot; };
#define LINV_KCHUNK 2     // tiles (of 64) per chunk

#define LI_LD 66
__global__ void __launch_bounds__(64) k_linv_diag(DevSym S, DevNum N, const int* __restrict__ pairs,
                                                  const long long* __restrict__ linv_off, double* __restrict__ linv) {
  __shared__ __align__(16) double Ls[64 * LI_LD];
  const int s = pairs[2 * blockIdx.x], b = pairs[2 * blockIdx.x + 1];
  const int k = S.sn_start[s + 1] - S.sn_start[s];
  const int f = k + (int)(S.rows_ptr[s + 1] - S.rows_ptr[s]);
  const long long K64 = (long long)((k + 63) / 64) * 64;
  const int r0 = b * 64, nd = min(64, k - r0);
  const double* __restrict__ P = N.L + S.L_off[s];
  const int tid = threadIdx.x;
  for (int t = tid; t < 64 * 64; t += 64) {
    const int i = t & 63, q = t >> 6;
    Ls[i + q * LI_LD] = (i < nd && q < nd && i > q) ? P[(r0 + i) + (size_t)(r0 + q) * f] : 0.0;
  }
  __syncthreads();
  // thread j: column j of X = L_dd^-1 by forward substitution on e_j, right-looking (independent FMAs per step)
  double xc[64];
#pragma unroll
  for (int i = 0; i < 64; ++i) xc[i] = (i == tid) ? 1.0 : 0.0;
#pragma unroll
  for (int t = 0; t < 63; ++t) {
    const double xt = xc[t];
    const double* __restrict__ col = Ls + t * LI_LD;
    if (((t + 1) & 1) != 0) xc[t + 1] = fma(-xt, col[t + 1], xc[t + 1]);
#pragma unroll
    for (int q = (t + 2) & ~1; q < 64; q += 2) {
      const double2 l2 = *reinterpret_cast<const double2*>(col + q);
      xc[q] = fma(-xt, l2.x, xc[q]);
      xc[q + 1] = fma(-xt, l2.y, xc[q + 1]);
    }
  }
  __syncthreads();
#pragma unroll
  for (int i = 0; i < 64; ++i) Ls[i + tid * LI_LD] = (i < nd && tid < nd) ? xc[i] : 0.0;
  __syncthreads();
  double* __restrict__ E = linv + linv_off[s] + r0 + (long long)r0 * K64;
  for (int t = tid; t < 64 * 64; t += 64) {
    const int i = t & 63, q = t >> 6;
    E[i + (long long)q * K64] = Ls[i + q * LI_LD];
  }
}

// 64x64 tile per CTA of 128 threads, 8x4 register blocking (rows tx+8q, columns ty+16p), k-slabs of 16 prefetched
// into registers while the current slab is consumed.
template <int PHASE>
__global__ void __launch_bounds__(128) k_linv_gemm(DevSym S, DevNum N, const LinvItem* __restrict__ items,
                                                   const long long* __restrict__ linv_off, double* __restrict__ linv,
                                                   double* __restrict__ part, int* __restrict__ part_cnt) {
  __shared__ double As[16][65];
  __shared__ double Bs[16][65];
  __shared__ int s_last;
  const LinvItem it = items[blockIdx.x];
  const int s = it.s;
  const int k = S.sn_start[s + 1] - S.sn_start[s];
  const long long f = k + (S.rows_ptr[s + 1] - S.rows_ptr[s]);
  const long long K64 = (long long)((k + 63) / 64) * 64;
  double* __restrict__ Li = linv + linv_off[s];
  const double* __restrict__ Lp = N.L + S.L_off[s];
  double* __restrict__ Wp = N.W + S.L_off[s];
  const int tid = threadIdx.x, tx = tid & 7, ty = tid >> 3;
  const int i0 = it.ib * 64, j0 = it.jb * 64;
  // loaders: A element (row i0 + (tid & 63), col kk0 + (tid >> 6) + 2q); B element (row kk0 + (tid & 15), col j0 + (tid >> 4) + 8q)
  double av[8], bv[8];
  auto load = [&](int kk0) {
#pragma unroll
    for (int q = 0; q < 8; ++q) {
      const long long arow = i0 + (tid & 63), acol = kk0 + (tid >> 6) + 2 * q;
      const long long brow = kk0 + (tid & 15), bcol = j0 + (tid >> 4) + 8 * q;
      if (PHASE == 1) {
        av[q] = (arow < k && acol < k) ? Lp[arow + acol * f] : 0.0;
        bv[q] = Li[brow + bcol * K64];
      } else {
        av[q] = Li[arow + acol * K64];
        bv[q] = (brow < k && bcol < k) ? Wp[brow + bcol * f] : 0.0;
      }
    }
  };
  double acc[8][4];
#pragma unroll
  for (int a = 0; a < 8; ++a)
#pragma unroll
    for (int c = 0; c < 4; ++c) acc[a][c] = 0.0;
  const int kbeg = it.m0 * 64, kend = it.m1 * 64;
  load(kbeg);
  for (int kk0 = kbeg; kk0 < kend; kk0 += 16) {
#pragma unroll
    for (int q = 0; q < 8; ++q) {
      As[(tid >> 6) + 2 * q][tid & 63] = av[q];
      Bs[tid & 15][(tid >> 4) + 8 * q] = bv[q];
    }
    __syncthreads();
    if (kk0 + 16 < kend) load(kk0 + 16);
#pragma unroll
    for (int kk = 0; kk < 16; ++kk) {
      double a[8], c[4];
#pragma unroll
      for (int q = 0; q < 8; ++q) a[q] = As[kk][tx + 8 * q];
#pragma unroll
      for (int p = 0; p < 4; ++p) c[p] = Bs[kk][ty + 16 * p];
#pragma unroll
      for (int q = 0; q < 8; ++q)
#pragma unroll
        for (int p = 0; p < 4; ++p) acc[q][p] = fma(a[q], c[p], acc[q][p]);
    }
    __syncthreads();
  }
  if (it.nch > 1) {
    // partial tile -> scratch; the last chunk to arrive sums all of them in chunk order
    double* __restrict__ mine = part + ((size_t)it.slot + it.ci) * 4096;
#pragma unroll
    for (int q = 0; q < 8; ++q)
#pragma unroll
      for (int p = 0; p < 4; ++p) mine[(tx + 8 * q) + 64 * (ty + 16 * p)] = acc[q][p];
    __threadfence();
    __syncthreads();
    if (tid == 0) s_last = (atomicAdd(part_cnt + it.slot, 1) == it.nch - 1) ? 1 : 0;
    __syncthreads();
    if (!s_last) return;
    __threadfence();
    if (tid == 0) part_cnt[it.slot] = 0;          // ready for the next factorisation
    const double* __restrict__ base = part + (size_t)it.slot * 4096;
#pragma unroll
    for (int q = 0; q < 8; ++q)
#pragma unroll
      for (int p = 0; p < 4; ++p) {
        double v = 0.0;
        for (int c = 0; c < it.nch; ++c) v += __ldcg(base + (size_t)c * 4096 + (tx + 8 * q) + 64 * (ty + 16 * p));
        acc[q][p] = v;
      }
  }
#pragma unroll
  for (int q = 0; q < 8; ++q)
#pragma unroll
    for (int p = 0; p < 4; ++p) {
      const long long row = i0 + tx + 8 * q, col = j0 + ty + 16 * p;
      if (PHASE == 1) { if (row < k && col < k) Wp[row + col * f] = acc[q][p]; }
      else Li[row + col * K64] = -acc[q][p];
    }
}

// ------------------------------------------------------------------------------------------------
// Shared-memory layout of one subtree (k_solve_sub).  The same arithmetic runs on the host when the subtrees are cut
// (the byte count must fit DF_DYN_SMEM) and on the device when the slices are carved.
//   doubles : Ls[nL] | xs[ncol] | uv[nrt] | rootx[rroot] | dinv[ncol] | doff[ncol] | wscr[8*DF_WSCR] | midscr[DF_MIDSCR]
//   ints    : lperm[ncol] | ptype[ncol] | rel-or-subrow[nrt] | chi[nchi] | meta[nmeta]
//   FrontDesc fd[nfront] ; mbarrier (8 bytes)
// ------------------------------------------------------------------------------------------------
struct SubLayout {
  long long nL; int ncol, nrt, rroot, nchi, nmeta, nfront;
  __host__ __device__ long long n_doubles() const {
    return nL + 3LL * ncol + nrt + rroot + (DF_THREADS / 32) * DF_WSCR + DF_MIDSCR;
  }
  __host__ __device__ long long n_ints() const { return 2LL * ncol + nrt + nchi + nmeta; }
  __host__ __device__ long long ints_off() const { return ((n_doubles() * 8 + 15) / 16) * 16; }   // bytes
  __host__ __device__ long long fd_off() const { return ints_off() + ((n_ints() * 4 + 15) / 16) * 16; }
  __host__ __device__ long long bytes() const { return fd_off() + (long long)nfront * (long long)sizeof(FrontDesc) + 16; }
};

// one subtree, by the whole CTA (see the file header).  `mbar` / `mphase`: the CTA's transaction barrier and its phase.
template <bool FWD, bool APPLY_D>
__device__ void solve_subtree(const DevSym& S, const DevNum& N, const DevSolve& V, int u, int epoch, unsigned char* smraw,
                              unsigned long long* mbar, unsigned mphase, double* __restrict__ x, double* __restrict__ cbv,
                              const Team tm) {
  const int tid = tm.tid, warp = tid >> 5, NT = tm.nt;
  const SubDesc sd = V.subs[u];
  const int s0 = sd.s0, sR = sd.sR, nfront = sR - s0 + 1, nlv = sd.nlv;
  const int col0 = sd.col0, ncol = sd.ncol, nrt = sd.nrt, rroot = sd.rroot, ch00 = sd.ch00, nchi = sd.nchi;
  const long long nL = sd.nL, ro0 = sd.ro0, roR = sd.ro0 + (sd.nrt - sd.rroot);
  const int nmeta = 2 * nlv + 1 + sd.nown;
  // carve
  double* Ls = reinterpret_cast<double*>(smraw);
  double* xs = Ls + nL;
  double* uv = xs + ncol;
  double* rootx = uv + nrt;
  double* dinv = rootx + rroot;
  double* doff = dinv + ncol;
  double* wscr = doff + ncol;
  double* midscr = wscr + (DF_THREADS / 32) * DF_WSCR;
  SubLayout lay;
  lay.nL = nL; lay.ncol = ncol; lay.nrt = nrt; lay.rroot = rroot; lay.nchi = nchi; lay.nmeta = nmeta; lay.nfront = nfront;
  int* lperm = reinterpret_cast<int*>(smraw + lay.ints_off());
  int* ptype = lperm + ncol;
  int* relsub = ptype + ncol;
  int* chi = relsub + nrt;
  int* meta = chi + nchi;
  FrontDesc* fds = reinterpret_cast<FrontDesc*>(smraw + lay.fd_off());

  // The panels of the subtree's fronts (those the direct kernel does not own) -> compact shared-memory copy, one bulk copy
  // per front, issued by as many threads as there are fronts; thread 0 announces the total byte count.
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");   // earlier generic accesses of this shared memory before the async writes
  if (tid == 0) mbar_expect_tx(mbar, (unsigned)(nL * 8));
  {
    const int nown = sd.nown;
    const int* __restrict__ gfl = V.sub_meta + sd.moff + 2 * nlv + 1;
    for (int i = tid; i < nown; i += NT) {
      const int s = gfl[i];
      const FrontDesc gd = load_fd(V.fdesc + s);
      const long long pn = ((long long)(gd.k + gd.r) * gd.k + 1) & ~1LL;
      bulk_g2s(Ls + V.sub_Loff[s], N.L + gd.L_off, (unsigned long long)pn * 8, mbar);
    }
  }
  // everything else: plain coalesced loads, all in flight together with the bulk copy
  for (int i = tid; i < ncol; i += NT) {
    xs[i] = x[col0 + i];
    dinv[i] = N.dinv[col0 + i];
    doff[i] = N.doff[col0 + i];
    lperm[i] = N.lperm[col0 + i];
    ptype[i] = N.ptype[col0 + i];
  }
  for (int i = tid; i < nrt; i += NT) relsub[i] = FWD ? S.rel[ro0 + i] : V.subrow[ro0 + i];
  for (int i = tid; i < nchi; i += NT) chi[i] = S.child_idx[ch00 + i];
  for (int i = tid; i < nmeta; i += NT) meta[i] = V.sub_meta[sd.moff + i];
  {
    const int4* src = reinterpret_cast<const int4*>(V.fdesc + s0);
    int4* dst = reinterpret_cast<int4*>(fds);
    for (int i = tid; i < 2 * nfront; i += NT) {
      int4 v = src[i];
      if (i & 1) {                       // second half of descriptor i/2: (L_off, ro) -> L_off = offset in the compact copy
        const long long lo = (long long)V.sub_Loff[s0 + (i >> 1)];
        v.x = (int)(unsigned)(lo & 0xffffffffll); v.y = (int)(lo >> 32);
      }
      dst[i] = v;
    }
  }
  if (!FWD) {
    // the root's contribution rows are columns of ancestors: final once the parent front is done
    const int grow = (tid < rroot) ? S.rows[roR + tid] : 0;   // (first chunk's row ids in flight before the wait)
    if (sd.parent >= 0 && tid == 0) wait_eq(V.done_b + sd.parent, epoch);
    team_sync(tm);
    if (tid < rroot) rootx[tid] = __ldcg(x + grow);
    for (int i = tid + NT; i < rroot; i += NT) rootx[i] = __ldcg(x + S.rows[roR + i]);
  }
  FrontIO io;
  io.Lbase = Ls; io.L0 = 0; io.xs = xs; io.col0 = col0; io.uv = uv; io.ro0 = ro0;
  io.dinv = dinv; io.doff = doff; io.ptype = ptype; io.lperm = lperm;
  io.rel = relsub; io.subrow = relsub; io.rootx = rootx;
  io.fd = fds; io.s0 = s0; io.sR = sR; io.chi = chi; io.ch00 = ch00;
  io.gfd = V.fdesc; io.gcbv = cbv; io.grel = S.rel; io.grows = S.rows; io.gx = x;
  team_sync(tm);
  mbar_wait(mbar, mphase);
  const int* lvl = meta;              // nlv + 1 offsets into the front list
  const int* nsm = meta + nlv + 1;    // nlv
  const int* fl = meta + 2 * nlv + 1; // nfront ids
  for (int li = 0; li < nlv; ++li) {
    const int e = FWD ? li : nlv - 1 - li;
    const int b = lvl[e], en = lvl[e + 1], ns = nsm[e];
    for (int q = b + warp; q < b + ns; q += NT / 32) {
      const int s = fl[q];
      if (FWD) w64_fwd<true, APPLY_D>(io, V, s, epoch, wscr + warp * DF_WSCR);
      else w64_bwd<true>(io, V, s, epoch, -1, V.upper_max);
    }
    for (int q = b + ns; q < en; ++q) {   // (mid fronts use their own scratch: no barrier needed before them)
      const int s = fl[q];
      if (FWD) mid_fwd<true, APPLY_D>(io, V, s, epoch, midscr, nullptr, nullptr, 0, tm);
      else mid_bwd<true>(io, V, s, epoch, -1, midscr, nullptr, nullptr, 0, V.upper_max, tm);
    }
    team_sync(tm);
  }
  // results back to global memory: the x slice (forward: z = D^-1 y in pivot order; backward: the solution), the
  // root's update vector (forward), and the done flags (the root's with release semantics: the parent waits for it)
  for (int i = tid; i < ncol; i += NT) x[col0 + i] = xs[i];
  if (FWD) {
    for (int i = tid; i < rroot; i += NT) cbv[roR + i] = uv[(roR - ro0) + i];
    for (int i = tid; i < sd.nown; i += NT) { const int s = fl[i]; if (s != sR) V.done_f[s] = epoch; }
  } else {
    for (int i = tid; i < sd.nown; i += NT) V.done_b[fl[i]] = epoch;
  }
  team_sync(tm);
  if (FWD && tid == 0) st_release(V.done_f + sR, epoch);
}

// ------------------------------------------------------------------------------------------------
// A block of nb right-hand sides (2 <= nb <= MS_NB_MAX) goes through the same launches: the MULTI instantiations of
// k_solve / k_solve_direct turn every work item into nb items, one per column, issued next to each other in the ticket
// order: (item 0, col 0), (item 0, col 1), ..., (item 1, col 0), ...  Each column has its own copy of everything a sweep
// writes -- x, update vectors, bigv / bigy, chunk partials and counters, done / block flags -- so an item runs the same
// front routines on its column's slices: the arithmetic of every column is the arithmetic of a single-column solve, bit for
// bit.  The block shares the launches and the dependency latency of the sweep (direct levels, subtree walks, flag hops
// between top tasks).  It does not share panel traffic: every (item, column) stages its own panels, loads its own L / Linv
// tiles and waits on its own flags (the items of a front are adjacent tickets, so the later copies may find the panel in
// L2).  Deadlock freedom carries over: an item only waits for items of its own column that are EARLIER in the ticket order
// (their single-column predecessors, nb times further back), and every ticket holder is resident.
// ------------------------------------------------------------------------------------------------
#define MS_NB_MAX 8          // widest block; wider calls are cut into blocks of this many columns

// where column c of the sweep state lives: base pointer (DevSolve / kernel argument) + c * stride
struct MultiStride {
  int nb;                    // columns
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

// the front routines on global memory (outside a subtree): x and update vectors of one column
__device__ __forceinline__ void global_io(FrontIO& io, const DevSym& S, const DevNum& N, const DevSolve& V, double* x,
                                          double* cbv) {
  io.Lbase = N.L; io.L0 = 0; io.xs = x; io.col0 = 0; io.uv = cbv; io.ro0 = 0;
  io.dinv = N.dinv; io.doff = N.doff; io.ptype = N.ptype; io.lperm = N.lperm;
  io.rel = S.rel; io.subrow = nullptr; io.rootx = nullptr;
  io.fd = V.fdesc; io.s0 = 0; io.sR = S.nsn - 1; io.chi = S.child_idx; io.ch00 = 0;
  io.gfd = V.fdesc; io.gcbv = cbv; io.grel = S.rel; io.grows = S.rows; io.gx = x;
}

// ------------------------------------------------------------------------------------------------
// ONE persistent kernel per sweep.  Work items are taken with an atomic ticket: forward = subtrees (largest first), then
// the top tasks by level; backward = top tasks (levels descending), then the subtrees.  MULTI: (item, column) tickets over
// M.nb columns.  Otherwise the ticket is the item and the column a compile-time 0 (no per-ticket division, the column view
// is the identity).  APPLY_D = false (forward only): the L solve alone -- the pivot rows keep the values the fused sweep
// has before D^-1, in x (bigv for the big fronts).
// ------------------------------------------------------------------------------------------------
template <bool FWD, bool MULTI, bool APPLY_D = true>
__global__ void __launch_bounds__(DF_THREADS, 2) k_solve(DevSym S, DevNum N, DevSolve V, MultiStride M, int epoch,
                                                         unsigned long long ticket_base,
                                                         double* __restrict__ x, double* __restrict__ cbv) {
  extern __shared__ __align__(16) unsigned char smraw[];
  __shared__ unsigned long long s_ticket;
  __shared__ unsigned long long s_mbar;
  __shared__ unsigned long long s_mbar1;    // second subtree of a pair
  __shared__ int s_flag;
  double* sm = reinterpret_cast<double*>(smraw);                // [0, 8*DF_WSCR + DF_MIDSCR) scratch, then the panel stage
  double* midscr = sm + (DF_THREADS / 32) * DF_WSCR;
  double* stage = midscr + DF_MIDSCR;
  const long long stage_doubles = (DF_DYN_SMEM / 8) - ((DF_THREADS / 32) * DF_WSCR + DF_MIDSCR);
  const SolveTask* tasks = FWD ? V.tasks : V.tasks_bwd;
  const int ntasks = FWD ? V.ntasks_fwd : V.ntasks_bwd;
  const unsigned long long nb = MULTI ? (unsigned long long)M.nb : 1ull;
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
    const unsigned long long item = MULTI ? tk / nb : tk;
    const int c = MULTI ? (int)(tk - item * nb) : 0;
    const DevSolve Vc = column_view(V, M, c);
    double* xc = x + c * M.x;
    double* cbvc = cbv + c * M.cbv;
    const bool is_sub = FWD ? (item < (unsigned long long)V.npair) : (item >= (unsigned long long)ntasks);
    if (is_sub) {
      const int2 pr = V.subpair[FWD ? item : item - ntasks];
      // (u0, -1): one subtree by the whole CTA.  (u0, u1): two subtrees side by side -- threads 0..127 walk u0 in the lower
      // part of the shared memory, threads 128..255 walk u1 above it (own transaction barrier, own hardware barrier).
      const bool second = pr.y >= 0 && threadIdx.x >= DF_THREADS / 2;
      const Team tm = pr.y < 0 ? cta : Team{(int)threadIdx.x - (second ? DF_THREADS / 2 : 0), DF_THREADS / 2, second ? 2 : 1};
      solve_subtree<FWD, APPLY_D>(S, N, Vc, second ? pr.y : pr.x, epoch, second ? smraw + V.subs[pr.x].sbytes : smraw,
                         second ? &s_mbar1 : &s_mbar, second ? mphase1 : mphase, xc, cbvc, tm);
      mphase ^= 1;
      if (pr.y >= 0) mphase1 ^= 1;
      __syncthreads();
      continue;
    }
    const unsigned long long ti = FWD ? item - V.npair : item;
    const SolveTask T = tasks[ti];
    FrontIO io;
    global_io(io, S, N, Vc, xc, cbvc);
    if (T.type == ST_SMALL) {
      const int w = threadIdx.x >> 5;
      if (w < T.blk) {
        const int s = V.bundle[T.s + w];
        if (FWD) w64_fwd<false, APPLY_D>(io, Vc, s, epoch, sm + w * DF_WSCR);
        else w64_bwd<false>(io, Vc, s, epoch, S.sn_parent[s], V.upper_max);
      }
    } else if (T.type == ST_MID) {
      // stage the whole panel in shared memory with one bulk copy when it fits (it does not depend on the right-hand
      // side, so it is in flight while the routine waits for / gathers its inputs)
      const FrontDesc fd = load_fd(V.fdesc + T.s);
      const long long pn = ((long long)(fd.k + fd.r) * fd.k + 1) & ~1LL;
      const double* Lp = nullptr;
      unsigned long long* mb = nullptr;
      unsigned ph = 0;
      if (pn <= stage_doubles) {
        if (threadIdx.x == 0) {
          asm volatile("fence.proxy.async.shared::cta;" ::: "memory");   // earlier generic reads of the stage before the async write
          mbar_expect_tx(&s_mbar, (unsigned)(pn * 8));
          bulk_g2s(stage, N.L + fd.L_off, (unsigned long long)pn * 8, &s_mbar);
        }
        Lp = stage; mb = &s_mbar; ph = mphase;
        mphase ^= 1;
      }
      if (FWD) mid_fwd<false, APPLY_D>(io, Vc, T.s, epoch, midscr, Lp, mb, ph, cta);
      else mid_bwd<false>(io, Vc, T.s, epoch, S.sn_parent[T.s], midscr, Lp, mb, ph, V.upper_max, cta);
    } else if (T.type == ST_FP) {
      big_fp<APPLY_D>(S, N, Vc, T, epoch, sm, &s_flag, xc, cbvc);
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

// ------------------------------------------------------------------------------------------------
// The bottom levels of the tree (fronts of order <= 64 whose descendants are of the same kind: 70 % of all fronts, a third
// of nnz(L) at level 0 alone) need no task machinery at all: a level has no internal dependencies, so ONE launch per level
// gives every front its own warp straight from global memory (column loads issued ahead of the shuffle chain) with every
// warp slot of the GPU busy -- instead of walking them inside the shared-memory subtrees, where they are serialised behind
// each other on a handful of warps.  Forward: these launches precede k_solve<fwd>; backward: they follow k_solve<bwd>.
// Their parents find the update vectors in global memory (FrontDesc::direct).  MULTI: one warp per (front, column), the
// M.nb warps of a front side by side (the panel comes from L1 / L2 after the first).  APPLY_D: as in k_solve.
// ------------------------------------------------------------------------------------------------
template <bool FWD, bool MULTI, bool APPLY_D = true>
__global__ void __launch_bounds__(DF_THREADS, 2) k_solve_direct(DevSym S, DevNum N, DevSolve V, MultiStride M,
                                                                const int* __restrict__ list, int cnt, int epoch,
                                                                double* __restrict__ x, double* __restrict__ cbv) {
  __shared__ double wscr[(DF_THREADS / 32) * DF_WSCR];
  const int w = threadIdx.x >> 5;
  const int g = blockIdx.x * (DF_THREADS / 32) + w;
  const int nb = MULTI ? M.nb : 1;
  if (g >= cnt * nb) return;
  const int c = MULTI ? g % nb : 0;
  const DevSolve Vc = column_view(V, M, c);
  FrontIO io;
  global_io(io, S, N, Vc, x + c * M.x, cbv + c * M.cbv);
  const int s = list[MULTI ? g / nb : g];
  if (FWD) w64_fwd<false, APPLY_D>(io, Vc, s, epoch, wscr + w * DF_WSCR);
  else w64_bwd<false>(io, Vc, s, epoch, -1, Vc.upper_max);
}

}  // namespace b200
