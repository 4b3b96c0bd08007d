// Multiplication by the factors (b200ldlt_lmultiply), sm_90a.  With  S A S = P L D L^T P^T  (include/b200ldlt.h):
//
//   trans = 0 :  y = S^-1 P L x      x in pivot order, y in original order   (k_lmul_n, then k_lmul_gather)
//   trans = 1 :  y = L^T P^T S^-1 x  x in original order, y in pivot order   (k_lmul_in, then k_lmul_t)
//
// L is read as the factorisation left it: the f x k panel of each front (column-major, rows in pivot order inside the
// pivot block, the contribution rows after it), entries strictly below the diagonal; the unit diagonal is implied.  That
// holds for every front class: the big fronts (order > 256) keep the unit lower L11 in their panel after the
// factorisation -- the explicit inverse Linv the solve uses is a separate array, built FROM the panel (k_linv_diag /
// k_linv_gemm read its strictly lower part, and the product B A^-1 of k_linv_gemm<1> goes to the W scratch, not to the
// panel).  2x2 pivots need no special case: the panel entry between the two pivots of a pair is the one the forward
// sweep subtracts, so these kernels multiply by exactly the L whose inverse job 1 applies.
//
// Unlike the sweeps, a multiply has no recurrence: every front works at once, and L is streamed once per block of
// columns.  No atomics on the data path, and every sum runs in a fixed order, so the results are bit-reproducible and
// each column of a block has the bits of a single-column call (the per-column arithmetic does not depend on NCOL).
#include <cuda_runtime.h>

namespace b200 {

#define LM_CH 128   // L x: pivot columns per item (a front's columns are cut into chunks of this many)
#define LM_CW 4     // L^T x: pivot columns per warp

// L x: one warp = rows [t0 + 32 g, +32) of the panel of front s, times its columns [t0, min(t0 + LM_CH, k)).  The
// partial sums of a chunk go to its slots (one per panel row from t0 on: slot + i - t0 for panel row i), which
// k_lmul_gather adds up.
struct LmulItem { int s, t0, g, pad; long long slot; };

// slot values of the chunks: y_i = sum_{t in chunk, t < i} L[i,t] x[c0 + t]  (+ x[c0 + i] for the chunk's own pivot rows)
template <int NCOL>
__global__ void __launch_bounds__(256) k_lmul_n(const FrontDesc* __restrict__ fdesc, const double* __restrict__ L,
                                                const LmulItem* __restrict__ items, int nitems,
                                                const double* __restrict__ x, int n, double* __restrict__ slot,
                                                long long ldslot) {
  const int wid = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (wid >= nitems) return;
  const LmulItem it = items[wid];
  const FrontDesc fd = load_fd(fdesc + it.s);
  const int k = fd.k, f = k + fd.r;
  const int t0 = it.t0, t1 = min(t0 + LM_CH, k);
  const int i = t0 + 32 * it.g + lane;
  if (i >= f) return;
  const double* __restrict__ P = L + fd.L_off + i;
  const double* __restrict__ xs = x + fd.c0;
  const int te = min(t1, i);                 // strictly below the diagonal
  double acc[NCOL];
#pragma unroll
  for (int c = 0; c < NCOL; ++c) acc[c] = 0.0;
#pragma unroll 8
  for (int t = t0; t < te; ++t) {
    const double l = P[(size_t)t * f];
#pragma unroll
    for (int c = 0; c < NCOL; ++c) acc[c] = fma(l, xs[(size_t)c * n + t], acc[c]);
  }
  if (i < t1) {                              // the unit diagonal
#pragma unroll
    for (int c = 0; c < NCOL; ++c) acc[c] = acc[c] + xs[(size_t)c * n + i];
  }
  double* __restrict__ o = slot + it.slot + (i - t0);
#pragma unroll
  for (int c = 0; c < NCOL; ++c) o[(size_t)c * ldslot] = acc[c];
}

// y = S^-1 P (the slots summed per row of L): pivot position p of front s is panel row p - c0 of s (its own chunks:
// own[own_ptr[p] ..], in chunk order) and permuted column q = c0 + lperm[p], which is a contribution row of the
// descendants listed at desc[desc_ptr[q] ..] (fronts ascending, then chunks).  Column blockIdx.y.
__global__ void k_lmul_gather(int n, const int* __restrict__ pcol0, const int* __restrict__ lperm,
                              const int* __restrict__ own_ptr, const int* __restrict__ own,
                              const int* __restrict__ desc_ptr, const int* __restrict__ desc,
                              const int* __restrict__ perm, const double* __restrict__ scale,
                              const double* __restrict__ slot, long long ldslot, double* __restrict__ y) {
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= n) return;
  const long long c = blockIdx.y;
  const double* __restrict__ sl = slot + c * ldslot;
  const int q = pcol0[p] + lperm[p];
  double z = 0.0;
  for (int e = own_ptr[p]; e < own_ptr[p + 1]; ++e) z += sl[own[e]];
  for (int e = desc_ptr[q]; e < desc_ptr[q + 1]; ++e) z += sl[desc[e]];
  const int o = perm[q];
  y[c * n + o] = z / scale[o];               // (a power of two: exact)
}

// w = P^T S^-1 x, indexed by permuted column q (the sweeps' x layout).  Column blockIdx.y.
__global__ void k_lmul_in(int n, const int* __restrict__ perm, const double* __restrict__ scale,
                          const double* __restrict__ x, double* __restrict__ w) {
  const int q = blockIdx.x * blockDim.x + threadIdx.x;
  if (q >= n) return;
  const long long c = blockIdx.y;
  const int o = perm[q];
  w[c * n + q] = x[c * n + o] / scale[o];
}

// L^T w: one warp = pivot columns [t0, t0 + LM_CW) of front s (items: (s, t0)).  y[c0 + t] = w(row t) +
// sum_{i > t} L[i,t] w(row i), where panel row i < k is permuted column c0 + lperm[c0 + i] and row i >= k is
// rows[ro + i - k].  Lanes stride the rows (coalesced panel columns); each lane sums its rows in order, then a fixed
// butterfly adds the lanes (IEEE addition commutes, so every lane holds the same bits).
template <int NCOL>
__global__ void __launch_bounds__(256) k_lmul_t(const FrontDesc* __restrict__ fdesc, const double* __restrict__ L,
                                                const int2* __restrict__ items, int nitems, const int* __restrict__ lperm,
                                                const int* __restrict__ rows, const double* __restrict__ w, int n,
                                                double* __restrict__ y) {
  const int wid = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (wid >= nitems) return;
  const int2 it = items[wid];
  const FrontDesc fd = load_fd(fdesc + it.x);
  const int k = fd.k, f = k + fd.r, c0 = fd.c0, t0 = it.y;
  const int nc = min(LM_CW, k - t0);
  const double* __restrict__ P = L + fd.L_off + (size_t)t0 * f;
  double acc[LM_CW][NCOL];
#pragma unroll
  for (int j = 0; j < LM_CW; ++j)
#pragma unroll
    for (int c = 0; c < NCOL; ++c) acc[j][c] = 0.0;
#pragma unroll 2
  for (int i = t0 + 1 + lane; i < f; i += 32) {
    const int q = i < k ? c0 + lperm[c0 + i] : rows[fd.ro + i - k];
    double wv[NCOL];
#pragma unroll
    for (int c = 0; c < NCOL; ++c) wv[c] = w[(size_t)c * n + q];
#pragma unroll
    for (int j = 0; j < LM_CW; ++j) {
      if (j < nc && i > t0 + j) {
        const double l = P[i + (size_t)j * f];
#pragma unroll
        for (int c = 0; c < NCOL; ++c) acc[j][c] = fma(l, wv[c], acc[j][c]);
      }
    }
  }
#pragma unroll
  for (int j = 0; j < LM_CW; ++j)
#pragma unroll
    for (int c = 0; c < NCOL; ++c) {
      double v = acc[j][c];
#pragma unroll
      for (int off = 16; off > 0; off >>= 1) v += __shfl_xor_sync(0xffffffffu, v, off);
      acc[j][c] = v;
    }
#pragma unroll
  for (int j = 0; j < LM_CW; ++j) {
    if (lane == j && j < nc) {
      const int t = t0 + j;
      const int q = c0 + lperm[c0 + t];
#pragma unroll
      for (int c = 0; c < NCOL; ++c) y[(size_t)c * n + c0 + t] = w[(size_t)c * n + q] + acc[j][c];
    }
  }
}

// ---- alteration of D (b200ldlt_alter_d) ----------------------------------------------------------------------------
// d2[2p] / d2[2p+1]: the new diagonal / off-diagonal entry of D^-1 at pivot position p (the layout of
// b200ldlt_enquire_indef).  Pass 1 validates (every entry finite; the off-diagonal zero unless ptype[p] == 2) and
// raises *bad; pass 2 writes dinv / doff only when *bad is still 0, so a refused call changes nothing.  The doff entries
// of 1x1 pivots and of the second pivot of a pair are left alone (the solve does not read them).
__global__ void k_alter_check(int n, const int* __restrict__ ptype, const double* __restrict__ d2, int* __restrict__ bad) {
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= n) return;
  const double a = d2[2 * (size_t)p], b = d2[2 * (size_t)p + 1];
  if (!isfinite(a) || !isfinite(b) || (b != 0.0 && ptype[p] != 2)) *bad = 1;   // (same value from every writer)
}
__global__ void k_alter(int n, const int* __restrict__ ptype, const double* __restrict__ d2, const int* __restrict__ bad,
                        double* __restrict__ dinv, double* __restrict__ doff) {
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= n || *bad) return;
  dinv[p] = d2[2 * (size_t)p];
  if (ptype[p] == 2) doff[p] = d2[2 * (size_t)p + 1];
}

}  // namespace b200
