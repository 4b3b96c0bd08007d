// Schur mode (b200ldlt_set_schur), sm_90a: the Schur variables S are the last m pivot positions, one root front of order m
// with no rows below it.  The factorisation eliminates every other front and assembles that root without factoring it,
// so its panel holds the scaled Schur complement (lower triangle).  These kernels copy it out unscaled, replace the root's
// factor state by an identity pivot block (so the solve sweeps pass the root's values through unchanged), and move the
// root's values in and out of the sweep state for the reduce / expand calls.
#include <cuda_runtime.h>

#include "kernels.cuh"

namespace b200 {

// sc[i + j m] = P[max(i,j) + min(i,j) m] / (s_i s_j), s_i = scale[vars[i]]: one thread per output entry (coalesced on
// the output side), both triangles from the lower one, so the result is bit-symmetric; the scale factors are powers of
// two, so the unscaling is exact.
__global__ void k_sc_out(int m, const double* __restrict__ P, const int* __restrict__ vars, const double* __restrict__ scale,
                         double* __restrict__ sc) {
  const long long t = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (t >= (long long)m * m) return;
  const int i = (int)(t % m), j = (int)(t / m);
  const int a = max(i, j), b = min(i, j);
  sc[t] = P[a + (long long)b * m] / scale[vars[i]] / scale[vars[j]];
}

// The root's factor state as an identity pivot block: the m x m panel (ld m) unit lower with zeros everywhere else,
// lperm / bperm identity, 1x1 pivots with D^-1 = 1, and (linv != nullptr: order > 256) the explicit L11^-1 block of
// K64 x K64 doubles = I on the first m columns, zero in the padding.  c0 = n - m, the root's first pivot position.
__global__ void k_sc_identity(int m, int c0, long long k64, double* __restrict__ P, int* __restrict__ lperm,
                              int* __restrict__ bperm, int* __restrict__ ptype, double* __restrict__ dinv,
                              double* __restrict__ doff, double* __restrict__ linv) {
  const long long t = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  const long long mm = (long long)m * m;
  if (t < mm) P[t] = (t % m == t / m) ? 1.0 : 0.0;
  if (t < m) {
    lperm[c0 + t] = (int)t; bperm[c0 + t] = (int)t; ptype[c0 + t] = 1;
    dinv[c0 + t] = 1.0; doff[c0 + t] = 0.0;
  }
  if (linv && t < k64 * k64) {
    const long long i = t % k64, j = t / k64;
    linv[t] = (i == j && i < m) ? 1.0 : 0.0;
  }
}

// reduce, after a forward sweep without D (sweep values as k_piv_out reads them): y[c m + i] = v(c0 + i) / s_i, column
// blockIdx.y
__global__ void k_sc_reduce(int m, int c0, const long long* __restrict__ piv_big, const double* __restrict__ xp, long long ldx,
                            const double* __restrict__ big, long long ldbig, const int* __restrict__ vars,
                            const double* __restrict__ scale, double* __restrict__ y) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  const long long c = blockIdx.y;
  if (i >= m) return;
  const int p = c0 + i;
  const long long q = piv_big[p];
  const double v = q >= 0 ? big[c * ldbig + q] : xp[c * ldx + p];
  y[c * m + i] = v / scale[vars[i]];
}

// expand, between a forward sweep without D and the backward sweep, in place on the sweep values of column blockIdx.y:
// the pivots of E (p < c0) become D^-1 v, rounded as k_dinv / k_fred round it (so the backward sweep computes x_E with
// job 0's arithmetic), and the Schur positions take the caller's solution in the scaled system, xs[c m + i] / s_i (the
// root's D^-1 is 1).  The thread of the first pivot of a 2x2 block reads and writes both of its entries.
__global__ void k_sc_expand(int n, int m, const int* __restrict__ ptype, const double* __restrict__ dinv,
                            const double* __restrict__ doff, const long long* __restrict__ piv_big, double* __restrict__ xp,
                            long long ldx, double* __restrict__ big, long long ldbig, const int* __restrict__ vars,
                            const double* __restrict__ scale, const double* __restrict__ xs) {
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  const long long c = blockIdx.y;
  if (p >= n) return;
  auto get = [&](int r) { const long long q = piv_big[r]; return q >= 0 ? big[c * ldbig + q] : xp[c * ldx + r]; };
  auto put = [&](int r, double v) {
    const long long q = piv_big[r];
    if (q >= 0) big[c * ldbig + q] = v; else xp[c * ldx + r] = v;
  };
  const int c0 = n - m;
  if (p >= c0) {
    const int i = p - c0;
    put(p, xs[c * m + i] / scale[vars[i]]);
    return;
  }
  const int ty = ptype[p];
  if (ty == 1) {
    put(p, dinv_entry(1, get(p), 0.0, dinv[p], 0.0));
  } else if (ty == 2) {
    const double v0 = get(p), v1 = get(p + 1);
    put(p, dinv_entry(2, v0, v1, dinv[p], doff[p]));
    put(p + 1, dinv_entry(3, v1, v0, dinv[p + 1], doff[p]));
  }
}

}  // namespace b200
