// Error analysis and condition estimation (b200ldlt_error_analysis, b200ldlt_condest), sm_90a.
//
// k_ea_rows / k_ea_class: one pass over |A| by rows for all right-hand-side columns (r = b - A x, s = |A||x|, the row
// maxima and sums of |A|), then the row classes I1 / I2 of Arioli, Demmel and Duff, the componentwise backward errors and
// the weights w1, w2.  k_ea_prep / k_ea_post: one step of Higham's 1-norm estimator (LAPACK dlacn2) for a block of
// estimator columns around one solve: prep builds each column's next input, post reduces each column's product to the
// few numbers the host needs for dlacn2's decisions.
//
// k_ea_rows<true> / k_ea_class<true> / k_rf_update: one step of iterative refinement (b200ldlt_solve_refined) for the
// unfinished columns of a block -- the residual in double-double straight into the solve's slots, s and the backward
// errors as above, and after the solve of the slots x += d with x saved for a rollback.
//
// Every result is bit-reproducible: maxima are atomicMax on the bit patterns of non-negative doubles (exact, whatever the
// order), |I2| an integer count, and every sum has a fixed order -- a row's entries by a fixed lane split and shuffle tree,
// a vector's 1-norm by a fixed grid (a function of n only), a fixed tree in each CTA and the CTAs' partials in order.
#include <cuda_runtime.h>

#include "kernels.cuh"

namespace b200 {

#define EA_THREADS 256
#define EA_WARPS (EA_THREADS / 32)
#define EA_PARTS_MAX 264     // CTAs per estimator column of k_ea_post (2 per SM)
#define EA_ROW_CTAS 1056     // CTAs per right-hand side of k_ea_rows (grid-stride over the rows)

// per right-hand side c, nrm[EA_NRM c + k]: bit patterns of non-negative doubles, max-reduced (EA_X .. EA_W2), and the
// count |I2| (EA_NI2); nrm[EA_NRM nrhs] = ||A||_inf
enum { EA_X = 0, EA_R, EA_B, EA_W1, EA_W2, EA_NI2, EA_NRM };

// one estimator column of a step: its input (mode 0: e/n, 1: e_j, 2: the stored sign vector, 3: the alternating vector)
// times pre (nullptr: 1), and its product M v times post (nullptr: 1); kase 1 (a product with B) stores the signs of
// the product in xi and counts their changes, kase 2 (with B^T) finds max |z|, its first index and z[jlast]
struct EaSlot {
  const double* pre;
  const double* post;
  int xi, mode, j, jlast, kase;
};
struct EaStep { EaSlot s[MS_NB_MAX]; };

struct EaPart { double l1, zmax; int jmax, changes; };
struct EaRes { double l1, zmax, zjl; int jmax, changes; };

static inline int ea_parts(int n) { return (int)std::min<long long>(((long long)n + EA_THREADS - 1) / EA_THREADS, EA_PARTS_MAX); }

// |v| with NaN as +inf, so that a NaN shows in the maxima (fmax would drop it)
__device__ __forceinline__ double ea_abs(double v) { const double a = fabs(v); return a == a ? a : INFINITY; }
__device__ __forceinline__ unsigned long long ea_bits(double a) { return (unsigned long long)__double_as_longlong(a); }

// max over the CTA (v >= 0) of each of NV values, then one atomicMax per value (skipped for 0: the buffers start at 0)
template <int NV>
__device__ __forceinline__ void ea_cta_max(double (&v)[NV], unsigned long long* const (&dst)[NV]) {
  __shared__ double red[NV][EA_WARPS];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
  for (int k = 0; k < NV; ++k) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v[k] = fmax(v[k], __shfl_xor_sync(0xffffffffu, v[k], o));
    if (lane == 0) red[k][warp] = v[k];
  }
  __syncthreads();
  if (threadIdx.x == 0) {
#pragma unroll
    for (int k = 0; k < NV; ++k) {
      double m = 0.0;
      for (int w = 0; w < EA_WARPS; ++w) m = fmax(m, red[k][w]);
      const unsigned long long b = ea_bits(m);
      if (b) atomicMax(dst[k], b);
    }
  }
}

// The columns of a refinement step: slot s (blockIdx.y) holds column c[s] of b and x (counted from the block's first)
struct RfCols { int c[MS_NB_MAX]; };

// (s, t) with s + t = a + b exactly (Knuth's TwoSum, six rounded operations, no contraction)
__device__ __forceinline__ void rf_two_sum(double a, double b, double& s, double& t) {
  s = __dadd_rn(a, b);
  const double bb = __dsub_rn(s, a);
  t = __dadd_rn(__dsub_rn(a, __dsub_rn(s, bb)), __dsub_rn(b, bb));
}

// One warp per row i of |A| (grid-stride), column c = blockIdx.y of b / x (b == nullptr: only the A part).  The row's
// entries (both triangles of the unique entries, columns ascending) are split over the lanes by position, each lane sums
// its own in order, and a shuffle tree combines the lanes: a fixed order.
//   r_i = b_i - sum_j a_ij x_j,  s_i = sum_j |a_ij| |x_j|  -> rs[2 c n + i], rs[(2 c + 1) n + i]
//   max |x_i|, max |r_i|, max |b_i|  -> nrm (EA_X, EA_R, EA_B of column c)
// and, for c = 0: amax[i] = max_j |a_ij| and max_i sum_j |a_ij| -> nrm[EA_NRM nrhs].
// DD (refinement): slot c = blockIdx.y reads column cols.c[c] of b / x, and r is accumulated in double-double in the
// order include/b200ldlt.h states and written to rout[c n + i] (s, the norms and the A part as above, by slot).
template <bool DD>
__global__ void __launch_bounds__(EA_THREADS) k_ea_rows(int n, int nrhs, const int* __restrict__ ptr,
                                                        const int* __restrict__ col, const int* __restrict__ uid,
                                                        const double* __restrict__ uval, const double* __restrict__ b,
                                                        const double* __restrict__ x, double* __restrict__ rs,
                                                        double* __restrict__ amax, unsigned long long* __restrict__ nrm,
                                                        RfCols cols, double* __restrict__ rout) {
  const int lane = threadIdx.x & 31;
  const int c = blockIdx.y;
  const size_t cc = DD ? (size_t)cols.c[c] : (size_t)c;
  const bool rhs = b != nullptr, mat = c == 0;
  const double* xc = rhs ? x + cc * n : nullptr;
  const double* bc = rhs ? b + cc * n : nullptr;
  double mx[4] = {0.0, 0.0, 0.0, 0.0};   // |x|, |r|, |b|, row sum of |A|
  const int nwarps = gridDim.x * EA_WARPS;
  for (int i = blockIdx.x * EA_WARPS + (threadIdx.x >> 5); i < n; i += nwarps) {
    double ax = 0.0, sx = 0.0, am = 0.0, as = 0.0;
    double hi = 0.0, lo = 0.0;   // DD: this lane's (h, l)
    if (DD && lane == 0) hi = bc[i];
    for (int e = ptr[i] + lane; e < ptr[i + 1]; e += 32) {
      const double a = uval[uid[e]];
      if (rhs) {
        const double xj = xc[col[e]];
        if (DD) {
          const double na = -a, p = __dmul_rn(na, xj), q = __fma_rn(na, xj, -p);
          double t;
          rf_two_sum(hi, p, hi, t);
          lo = __dadd_rn(lo, __dadd_rn(t, q));
        } else {
          ax += a * xj;
        }
        sx += fabs(a) * fabs(xj);
      }
      if (mat) { am = fmax(am, fabs(a)); as += fabs(a); }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      if (DD) {
        const double h2 = __shfl_xor_sync(0xffffffffu, hi, o), l2 = __shfl_xor_sync(0xffffffffu, lo, o);
        double t;
        rf_two_sum(hi, h2, hi, t);
        lo = __dadd_rn(__dadd_rn(lo, l2), t);
      } else {
        ax += __shfl_xor_sync(0xffffffffu, ax, o);
      }
      sx += __shfl_xor_sync(0xffffffffu, sx, o);
      am = fmax(am, __shfl_xor_sync(0xffffffffu, am, o));
      as += __shfl_xor_sync(0xffffffffu, as, o);
    }
    if (lane == 0) {
      if (rhs) {
        const double r = DD ? __dadd_rn(hi, lo) : bc[i] - ax;
        if (DD) rout[(size_t)c * n + i] = r;
        else rs[(size_t)2 * c * n + i] = r;
        rs[(size_t)(2 * c + 1) * n + i] = sx;
        mx[0] = fmax(mx[0], ea_abs(xc[i]));
        mx[1] = fmax(mx[1], ea_abs(r));
        mx[2] = fmax(mx[2], ea_abs(bc[i]));
      }
      if (mat) { amax[i] = am; mx[3] = fmax(mx[3], ea_abs(as)); }
    }
  }
  unsigned long long* base = nrm + (size_t)EA_NRM * c;
  unsigned long long* const dst[4] = {base + EA_X, base + EA_R, base + EA_B, nrm + (size_t)EA_NRM * nrhs};
  ea_cta_max<4>(mx, dst);
}

// Row classes and backward errors of column c = blockIdx.y, after k_ea_rows (rs holds r and s, overwritten by w1, w2):
//   tau_i = ctau (a_i ||x|| + |b_i|), ctau = 1000 n 2^-52;  i in I2 iff s_i + |b_i| <= tau_i, else I1;
//   omega1 = max_I1 |r_i| / (s_i + |b_i|),  omega2 = max_I2 |r_i| / (s_i + a_i ||x||)  (a term with r_i = 0 is 0);
//   w1 = s_i + |b_i| on I1, w2 = s_i + a_i ||x|| on I2, 0 elsewhere;  |I2| counted.
// RF (refinement): slot c reads column cols.c[c] of b and its r from rin[c n + i]; rs keeps s, no weights are written.
template <bool RF>
__global__ void __launch_bounds__(EA_THREADS) k_ea_class(int n, const double* __restrict__ b, const double* __restrict__ amax,
                                                         double* __restrict__ rs, unsigned long long* __restrict__ nrm,
                                                         RfCols cols, const double* __restrict__ rin) {
  const int i = blockIdx.x * EA_THREADS + threadIdx.x;
  const int c = blockIdx.y;
  const size_t cc = RF ? (size_t)cols.c[c] : (size_t)c;
  unsigned long long* base = nrm + (size_t)EA_NRM * c;
  const double xn = __longlong_as_double((long long)base[EA_X]);
  const double ctau = 1000.0 * (double)n * 0x1p-52;
  double om[2] = {0.0, 0.0};
  int in2 = 0;
  if (i < n) {
    double* r_w1 = rs + (size_t)2 * c * n;
    double* s_w2 = rs + (size_t)(2 * c + 1) * n;
    const double r = RF ? rin[(size_t)c * n + i] : r_w1[i];
    const double s = s_w2[i], ab = fabs(b[cc * n + i]), ax = amax[i] * xn;
    const double tau = ctau * (ax + ab);
    double w1 = 0.0, w2 = 0.0;
    if (s + ab <= tau) {
      in2 = 1;
      w2 = s + ax;
      if (r != 0.0) om[1] = ea_abs(r / w2);
    } else {
      w1 = s + ab;
      if (r != 0.0) om[0] = ea_abs(r / w1);
    }
    if (!RF) {
      r_w1[i] = w1;
      s_w2[i] = w2;
    }
  }
  const unsigned cnt = __syncthreads_count(in2);
  unsigned long long* const dst[2] = {base + EA_W1, base + EA_W2};
  ea_cta_max<2>(om, dst);
  if (threadIdx.x == 0 && cnt) atomicAdd(base + EA_NI2, (unsigned long long)cnt);
}

// The update of a refinement step: slot s = blockIdx.y holds the correction d of column c = cols.c[s] (counted from the
// block's first); xold[c n + i] = x[c n + i], then x[c n + i] = x[c n + i] (+) d[s n + i], one rounded add.
__global__ void __launch_bounds__(EA_THREADS) k_rf_update(int n, RfCols cols, const double* __restrict__ d,
                                                          double* __restrict__ x, double* __restrict__ xold) {
  const int i = blockIdx.x * EA_THREADS + threadIdx.x;
  if (i >= n) return;
  const size_t c = (size_t)cols.c[blockIdx.y];
  const double v = x[c * n + i];
  xold[c * n + i] = v;
  x[c * n + i] = __dadd_rn(v, d[(size_t)blockIdx.y * n + i]);
}

// The input of estimator column s = blockIdx.y of a step: v[s n + i] = (its mode's vector)_i * pre_i
__global__ void __launch_bounds__(EA_THREADS) k_ea_prep(int n, EaStep st, const signed char* __restrict__ xi,
                                                        double* __restrict__ v) {
  const int i = blockIdx.x * EA_THREADS + threadIdx.x;
  if (i >= n) return;
  const EaSlot& S = st.s[blockIdx.y];
  double a;
  switch (S.mode) {
    case 0: a = 1.0 / (double)n; break;
    case 1: a = i == S.j ? 1.0 : 0.0; break;
    case 2: a = (double)xi[(size_t)S.xi * n + i]; break;
    default: a = ((i & 1) ? -1.0 : 1.0) * (1.0 + (double)i / (double)(n - 1)); break;
  }
  if (S.pre) a *= S.pre[i];
  v[(size_t)blockIdx.y * n + i] = a;
}

// The reductions of estimator column s = blockIdx.y after its product, y_i = v[s n + i] * post_i, over ea_parts(n) CTAs
// (grid-stride, each thread in index order): ||y||_1, and for kase 1 the number of i with sign(y_i) != xi_i, after which
// xi_i = sign(y_i) (+1 for y_i >= 0, -0 included); for kase 2 max |y_i| and its first index.  Each CTA reduces by a fixed
// tree into part[s P + blockIdx.x]; the last CTA of the column to finish adds the P partials in order, reads y[jlast] and
// writes res[s] (and resets the column's arrival counter for the next step).
__global__ void __launch_bounds__(EA_THREADS) k_ea_post(int n, EaStep st, const double* __restrict__ v,
                                                        signed char* __restrict__ xi, EaPart* __restrict__ part,
                                                        unsigned* __restrict__ cnt, EaRes* __restrict__ res) {
  const int s = blockIdx.y, P = gridDim.x;
  const EaSlot& S = st.s[s];
  const double* vs = v + (size_t)s * n;
  signed char* xs = xi + (size_t)S.xi * n;
  double l1 = 0.0, zmax = -1.0;
  int jmax = INT_MAX, changes = 0;
  for (int i = blockIdx.x * EA_THREADS + threadIdx.x; i < n; i += P * EA_THREADS) {
    const double y = S.post ? vs[i] * S.post[i] : vs[i];
    const double a = fabs(y);
    l1 += a;
    if (S.kase == 1) {
      const signed char g = y >= 0.0 ? 1 : -1;
      changes += g != xs[i];
      xs[i] = g;
    } else if (a > zmax) {
      zmax = a; jmax = i;
    }
  }
  // (value, index) pairs: the larger value, on a tie the smaller index -- associative and commutative, so exact
  auto better = [](double a, int ia, double b, int ib) { return a > b || (a == b && ia < ib); };
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    l1 += __shfl_xor_sync(0xffffffffu, l1, o);
    changes += __shfl_xor_sync(0xffffffffu, changes, o);
    const double z2 = __shfl_xor_sync(0xffffffffu, zmax, o);
    const int j2 = __shfl_xor_sync(0xffffffffu, jmax, o);
    if (better(z2, j2, zmax, jmax)) { zmax = z2; jmax = j2; }
  }
  __shared__ EaPart red[EA_WARPS];
  __shared__ bool last;
  if (lane == 0) red[warp] = EaPart{l1, zmax, jmax, changes};
  __syncthreads();
  if (threadIdx.x == 0) {
    EaPart t = red[0];
    for (int w = 1; w < EA_WARPS; ++w) {
      t.l1 += red[w].l1;
      t.changes += red[w].changes;
      if (better(red[w].zmax, red[w].jmax, t.zmax, t.jmax)) { t.zmax = red[w].zmax; t.jmax = red[w].jmax; }
    }
    part[(size_t)s * P + blockIdx.x] = t;
    __threadfence();
    last = atomicAdd(cnt + s, 1u) == (unsigned)P - 1;
  }
  __syncthreads();
  if (!last || threadIdx.x != 0) return;
  __threadfence();
  const EaPart* ps = part + (size_t)s * P;
  EaRes R{0.0, -1.0, 0.0, INT_MAX, 0};
  for (int q = 0; q < P; ++q) {
    const double pl = __ldcg(&ps[q].l1), pz = __ldcg(&ps[q].zmax);
    const int pj = __ldcg(&ps[q].jmax), pc = __ldcg(&ps[q].changes);
    R.l1 += pl;
    R.changes += pc;
    if (better(pz, pj, R.zmax, R.jmax)) { R.zmax = pz; R.jmax = pj; }
  }
  const int jl = S.jlast;
  R.zjl = S.post ? vs[jl] * S.post[jl] : vs[jl];
  res[s] = R;
  cnt[s] = 0u;
}

}  // namespace b200
