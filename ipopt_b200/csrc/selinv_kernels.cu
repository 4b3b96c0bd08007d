// Selected inversion (b200ldlt_selected_inverse), sm_90a: Z = L^-T D^-1 L^-1 (pivot order) on the pattern of L, computed
// top-down over the elimination tree, one tree level at a time.  For a front s with pivot columns J (k of them, pivot
// order) and rows R below (r of them, the order of its row list), L11 / L21 the parts of its panel and E = L11^-1:
//   G    = Z_RR                                    (k_si_gather: from the parent's Z panel and the parent's G)
//   B    = L21 E                                   (r x k)
//   Z_RJ = -G B                                    (the rows below the pivot block of s's Z panel)
//   Z_JJ = E^T D_J^-1 E - B^T Z_RJ                  (lower triangle, the pivot block of s's Z panel)
// Every entry of Z is written by exactly one thread as one dot product in a fixed order (no atomics, no split sums), so
// the result is bit-reproducible.  The Z panels have the layout of the L panels (L_off, f x k column-major, ld f); G
// lives in the front's contribution-block slot (CB, cb_off, r x r, lower triangle), B of the fronts above SI_SMALL in
// the rows below the pivot block of the front's W slot.
#include <cuda_runtime.h>

#include "kernels.cuh"

namespace b200 {

#define SI_SMALL 96   // fronts of order <= this: one CTA per front in shared memory (k_si_small)
#define SI_SMALL_SMEM (2 * SI_SMALL * SI_SMALL * 8)   // its largest need, (f^2 + k^2) doubles
#define SI_MID 256    // fronts of order (SI_SMALL, SI_MID] get their L11^-1 from k_si_linv (above: the factorisation's)

// one 64 x 64 output tile of a front of order > SI_SMALL; E = L11^-1 of the front (column-major, leading dimension ld_e)
struct SiItem { int s, ib, jb, ld_e; const double* E; };

// lpinv[sn_start[s] + lperm[p]] = p - sn_start[s]: pre-pivot local column -> pivot index inside the front
__global__ void k_si_prep(int n, const int* __restrict__ sn_of, const int* __restrict__ sn_start, const int* __restrict__ lperm,
                          int* __restrict__ lpinv) {
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p < n) { const int c0 = sn_start[sn_of[p]]; lpinv[c0 + lperm[p]] = p - c0; }
}

// G of the fronts with r > 0, lower triangle, one 32-row segment of a column per warp: item (s, b, a0) covers the
// entries (a, b) with a0 <= a < min(a0 + 32, r), a >= b.  Row list indices map through rel into the parent front (pre-pivot
// local index); those below k_p are pivot columns of the parent (through lpinv), the others its rows.
struct SiGather { int s, b, a0; };
__global__ void __launch_bounds__(256) k_si_gather(DevSym S, const double* __restrict__ Z, double* __restrict__ CB,
                                                   const int* __restrict__ lpinv, const SiGather* __restrict__ items,
                                                   int nitems) {
  const int w = blockIdx.x * 8 + (threadIdx.x >> 5);
  if (w >= nitems) return;
  const SiGather it = items[w];
  const int s = it.s, b = it.b, a = it.a0 + (threadIdx.x & 31);
  const int r = (int)(S.rows_ptr[s + 1] - S.rows_ptr[s]);
  if (a >= r) return;
  const int p = S.sn_parent[s];
  const int c0p = S.sn_start[p], kp = S.sn_start[p + 1] - c0p;
  const long long rp = S.rows_ptr[p + 1] - S.rows_ptr[p], fp = kp + rp;
  const int* __restrict__ rel = S.rel + S.rows_ptr[s];
  const double* __restrict__ Zp = Z + S.L_off[p];
  const int ra = rel[a], rb = rel[b];   // rel increases along the row list: ra >= rb
  double v;
  if (rb >= kp) v = CB[S.cb_off[p] + (ra - kp) + (rb - kp) * rp];
  else if (ra >= kp) v = Zp[ra + lpinv[c0p + rb] * fp];
  else {
    const int ta = lpinv[c0p + ra], tb = lpinv[c0p + rb];
    v = Zp[max(ta, tb) + min(ta, tb) * fp];
  }
  CB[S.cb_off[s] + a + (long long)b * r] = v;
}

// (D^-1 X)[m, j] for column j of X (leading dimension ld) inside front c0: the rounding of dinv_entry
__device__ __forceinline__ double si_dx(const DevNum& N, int c0, int m, const double* __restrict__ x) {
  const int ty = N.ptype[c0 + m];
  if (ty == 1) return dinv_entry(1, x[m], 0.0, N.dinv[c0 + m], 0.0);
  if (ty == 2) return dinv_entry(2, x[m], x[m + 1], N.dinv[c0 + m], N.doff[c0 + m]);
  return dinv_entry(3, x[m], x[m - 1], N.dinv[c0 + m], N.doff[c0 + m - 1]);
}

// fronts of order <= SI_SMALL, one CTA each, everything in shared memory (f^2 + k^2 doubles)
__global__ void __launch_bounds__(128) k_si_small(DevSym S, DevNum N, double* __restrict__ Z, const int* __restrict__ fronts) {
  extern __shared__ double sm[];
  const int s = fronts[blockIdx.x];
  const int c0 = S.sn_start[s], k = S.sn_start[s + 1] - c0;
  const int r = (int)(S.rows_ptr[s + 1] - S.rows_ptr[s]), f = k + r;
  const int tid = threadIdx.x, nt = blockDim.x;
  const double* __restrict__ P = N.L + S.L_off[s];
  const double* __restrict__ G = N.CB + S.cb_off[s];
  double* __restrict__ Zs = Z + S.L_off[s];
  double* Lp = sm;              // f x k (ld f): L11 and L21; rows k.. become Z_RJ
  double* E = Lp + f * k;       // k x k (ld k): L11^-1
  double* Gs = E + k * k;       // r x r: G, both triangles
  double* Bs = Gs + r * r;      // r x k (ld r): B
  for (int e = tid; e < f * k; e += nt) Lp[e] = P[e];
  for (int e = tid; e < r * r; e += nt) {
    const int a = e % r, b = e / r;
    Gs[e] = a >= b ? G[a + b * r] : G[b + a * r];
  }
  __syncthreads();
  // column j of L11^-1 by forward substitution on e_j
  for (int j = tid; j < k; j += nt) {
    double* __restrict__ x = E + j * k;
    for (int i = 0; i < j; ++i) x[i] = 0.0;
    x[j] = 1.0;
    for (int i = j + 1; i < k; ++i) {
      double acc = 0.0;
      for (int m = j; m < i; ++m) acc = fma(Lp[i + m * f], x[m], acc);
      x[i] = -acc;
    }
  }
  __syncthreads();
  for (int e = tid; e < r * k; e += nt) {
    const int i = e % r, j = e / r;
    double acc = 0.0;
    for (int m = j; m < k; ++m) acc = fma(Lp[k + i + m * f], E[m + j * k], acc);
    Bs[i + j * r] = acc;
  }
  __syncthreads();
  for (int e = tid; e < r * k; e += nt) {
    const int i = e % r, j = e / r;
    double acc = 0.0;
    for (int m = 0; m < r; ++m) acc = fma(Gs[i + m * r], Bs[m + j * r], acc);
    Lp[k + i + j * f] = -acc;
    Zs[k + i + j * f] = -acc;
  }
  __syncthreads();
  for (int e = tid; e < k * k; e += nt) {
    const int i = e % k, j = e / k;
    if (i < j) continue;
    double acc = 0.0;
    for (int m = i; m < k; ++m) acc = fma(E[m + i * k], si_dx(N, c0, m, E + j * k), acc);
    for (int m = 0; m < r; ++m) acc = fma(-Bs[m + i * r], Lp[k + m + j * f], acc);
    Zs[i + j * f] = acc;
  }
}

// L11^-1 of the fronts of order (SI_SMALL, SI_MID], one CTA each, one column per thread (forward substitution on e_j)
// into E + eoff[s] (leading dimension k)
__global__ void __launch_bounds__(256) k_si_linv(DevSym S, DevNum N, const int* __restrict__ fronts,
                                                 const long long* __restrict__ eoff, double* __restrict__ E) {
  const int s = fronts[blockIdx.x];
  const int k = S.sn_start[s + 1] - S.sn_start[s];
  const long long f = k + (S.rows_ptr[s + 1] - S.rows_ptr[s]);
  const double* __restrict__ P = N.L + S.L_off[s];
  for (int j = threadIdx.x; j < k; j += blockDim.x) {
    double* __restrict__ x = E + eoff[s] + (long long)j * k;
    for (int i = 0; i < j; ++i) x[i] = 0.0;
    x[j] = 1.0;
    for (int i = j + 1; i < k; ++i) {
      double acc = 0.0;
      for (int m = j; m < i; ++m) acc = fma(P[i + m * f], x[m], acc);
      x[i] = -acc;
    }
  }
}

// 64 x 64 tiles of the fronts of order > SI_SMALL, 256 threads, 4 x 4 outputs per thread, k-slabs of 16 through shared
// memory; the sum of each output runs over m in ascending order.
//   PASS 0: B    = L21 E            -> W rows k..
//   PASS 1: Z_RJ = -G B             -> Z rows k..
//   PASS 2: Z_JJ = E^T D^-1 E - B^T Z_RJ  (tiles ib >= jb, entries i >= j)
template <int PASS>
__global__ void __launch_bounds__(256) k_si_tile(DevSym S, DevNum N, double* __restrict__ Z, const SiItem* __restrict__ items) {
  __shared__ double As[16][65];
  __shared__ double Bs[16][65];
  const SiItem it = items[blockIdx.x];
  const int s = it.s;
  const int c0 = S.sn_start[s], k = S.sn_start[s + 1] - c0;
  const int r = (int)(S.rows_ptr[s + 1] - S.rows_ptr[s]);
  const long long f = k + r, ld_e = it.ld_e;
  const double* __restrict__ P = N.L + S.L_off[s];
  const double* __restrict__ G = N.CB + S.cb_off[s];
  const double* __restrict__ E = it.E;
  double* __restrict__ Bm = N.W + S.L_off[s] + k;   // B (r x k, ld f)
  double* __restrict__ Zs = Z + S.L_off[s];
  const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
  const int i0 = it.ib * 64, j0 = it.jb * 64;
  const int nr = PASS == 2 ? k : r;   // rows of the output
  double acc[4][4];
#pragma unroll
  for (int a = 0; a < 4; ++a)
#pragma unroll
    for (int c = 0; c < 4; ++c) acc[a][c] = 0.0;
  // stage h (PASS 2 has two: the D^-1 term over m < k, then the B^T Z_RJ term over m < r)
  for (int h = 0; h < (PASS == 2 ? 2 : 1); ++h) {
    int mbeg, mend;
    if (PASS == 0) { mbeg = j0; mend = k; }                  // E[m, j] = 0 for m < j
    else if (PASS == 1) { mbeg = 0; mend = r; }
    else if (h == 0) { mbeg = i0; mend = k; }                // E[m, i] = 0 for m < i
    else { mbeg = 0; mend = r; }
    auto getA = [&](int i, int m) -> double {   // A(i, m), i < nr
      if (i >= nr || m >= mend) return 0.0;
      if (PASS == 0) return P[k + i + m * f];
      if (PASS == 1) return i >= m ? G[i + (long long)m * r] : G[m + (long long)i * r];
      if (h == 0) return E[m + i * ld_e];
      return -Bm[m + i * f];
    };
    auto getB = [&](int m, int j) -> double {   // B(m, j), j < k
      if (j >= k || m >= mend) return 0.0;
      if (PASS == 0) return E[m + j * ld_e];
      if (PASS == 1) return Bm[m + j * f];
      if (h == 0) return si_dx(N, c0, m, E + j * ld_e);
      return Zs[k + m + j * f];
    };
    for (int m0 = mbeg; m0 < mend; m0 += 16) {
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        const int e = tid + 256 * q;            // 1024 elements of each 64 x 16 / 16 x 64 slab
        As[e >> 6][e & 63] = getA(i0 + (e & 63), m0 + (e >> 6));
        Bs[e >> 6][e & 63] = getB(m0 + (e >> 6), j0 + (e & 63));
      }
      __syncthreads();
#pragma unroll
      for (int mm = 0; mm < 16; ++mm) {
        double a[4], b[4];
#pragma unroll
        for (int q = 0; q < 4; ++q) { a[q] = As[mm][tx + 16 * q]; b[q] = Bs[mm][ty + 16 * q]; }
#pragma unroll
        for (int q = 0; q < 4; ++q)
#pragma unroll
          for (int p = 0; p < 4; ++p) acc[q][p] = fma(a[q], b[p], acc[q][p]);
      }
      __syncthreads();
    }
  }
#pragma unroll
  for (int q = 0; q < 4; ++q)
#pragma unroll
    for (int p = 0; p < 4; ++p) {
      const int i = i0 + tx + 16 * q, j = j0 + ty + 16 * p;
      if (i >= nr || j >= k) continue;
      if (PASS == 0) Bm[i + j * f] = acc[q][p];
      else if (PASS == 1) Zs[k + i + j * f] = -acc[q][p];
      else if (i >= j) Zs[i + j * f] = acc[q][p];
    }
}

// the outputs, original order, scaled by S_i S_j (the smaller original index first; powers of two, so exact):
// threads [0, n) diag[i] = M_ii (diag != nullptr); threads [0, nnz) vals[e] = M at triplet e (vals != nullptr), through
// t2u -> u_dst64 = (pre-pivot local row, column) of the front holding the smaller permuted index
__global__ void k_si_out(int n, long long nnz, const int* __restrict__ iperm, const int* __restrict__ sn_of,
                         const int* __restrict__ sn_start, const long long* __restrict__ rows_ptr,
                         const long long* __restrict__ L_off, const int* __restrict__ lpinv, const double* __restrict__ Z,
                         const double* __restrict__ scale, const int* __restrict__ irn, const int* __restrict__ jcn,
                         const int* __restrict__ t2u, const long long* __restrict__ u_dst64, double* __restrict__ diag,
                         double* __restrict__ vals) {
  const long long e = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (diag && e < n) {
    const int i = (int)e, q = iperm[i], s = sn_of[q];
    const long long f = (sn_start[s + 1] - sn_start[s]) + (rows_ptr[s + 1] - rows_ptr[s]);
    const int t = lpinv[q];
    diag[i] = Z[L_off[s] + t + t * f] * scale[i] * scale[i];
  }
  if (vals && e < nnz) {
    const int i = irn[e] - 1, j = jcn[e] - 1;
    const int a = min(i, j), b = max(i, j);
    const int s = sn_of[min(iperm[i], iperm[j])], c0 = sn_start[s], k = sn_start[s + 1] - c0;
    const long long f = k + (rows_ptr[s + 1] - rows_ptr[s]);
    const long long d = u_dst64[t2u[e]];
    const int lr = (int)(d % f), lc = (int)(d / f);
    const int tc = lpinv[c0 + lc];
    double v;
    if (lr < k) {
      const int tr = lpinv[c0 + lr];
      v = Z[L_off[s] + max(tr, tc) + min(tr, tc) * f];
    } else {
      v = Z[L_off[s] + lr + tc * f];
    }
    vals[e] = v * scale[a] * scale[b];
  }
}

}  // namespace b200
