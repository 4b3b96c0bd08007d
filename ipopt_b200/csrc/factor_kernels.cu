// Numeric factorisation kernels of the supernodal multifrontal LDL^T (sm_90a).
//
// What the reference delegates to the vendor library's numeric phase (MUMPS job=2,
// reference src/Algorithm/LinearSolvers/IpMumpsSolverInterface.cpp:448-541): per front
// assemble original entries + children contribution blocks (extend-add), eliminate the
// fully-summed block with 1x1/2x2 Bunch-Kaufman pivots (threshold-tested against the whole
// front column), form the Schur complement, hand the contribution block to the parent.
//
// Two execution classes:
//   * fronts of order <= smem_front_max: ONE CTA does gather + extend-add + pivoted
//     factorisation + Schur update entirely in shared memory and writes L / CB once;
//   * larger fronts: global-memory blocked right-looking algorithm (32-wide panels) made of
//     batched kernels (diag-block factor, panel TRSM, trailing update, Schur GEMM).
#include <cuda_runtime.h>
#include <math.h>

#include "kernels.cuh"

namespace b200 {

#define BK_ALPHA 0.6403882032022076  // (1+sqrt(17))/8
#define NB 32                        // panel width of the big-front path

// --------------------------------------------------------------------------------------------
// small utility kernels
// --------------------------------------------------------------------------------------------
__global__ void k_sum_dups(long long nu, const long long* __restrict__ useg_ptr,
                           const int* __restrict__ useg_src, const double* __restrict__ vals,
                           double* __restrict__ uval) {
  long long u = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (u >= nu) return;
  double acc = 0.0;
  for (long long q = useg_ptr[u]; q < useg_ptr[u + 1]; ++q) acc += vals[useg_src[q]];
  uval[u] = acc;
}

// rmax[i] = max_j |a_ij| s_i s_j  (bit pattern of non-negative doubles orders like integers)
__global__ void k_rowmax(long long nu, const int* __restrict__ u_row, const int* __restrict__ u_col,
                         const double* __restrict__ uval, const double* __restrict__ scale,
                         unsigned long long* __restrict__ rmax) {
  long long u = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (u >= nu) return;
  int i = u_row[u], j = u_col[u];
  double a = fabs(uval[u]) * scale[i] * scale[j];
  if (!(a > 0.0)) return;  // also skips NaN
  unsigned long long b = (unsigned long long)__double_as_longlong(a);
  atomicMax(rmax + i, b);
  if (i != j) atomicMax(rmax + j, b);
}

__global__ void k_scale_update(int n, double* __restrict__ scale, unsigned long long* __restrict__ rmax) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  double m = __longlong_as_double((long long)rmax[i]);
  rmax[i] = 0ull;
  if (m > 0.0 && isfinite(m)) {
    // power-of-two factor closest to 1/sqrt(m): scaling stays exact in floating point
    int e;
    frexp(m, &e);  // m = f * 2^e, f in [0.5,1)
    scale[i] *= ldexp(1.0, -((e) / 2));
  }
}

__global__ void k_apply_scale(long long nu, const int* __restrict__ u_row, const int* __restrict__ u_col,
                              const double* __restrict__ scale, double* __restrict__ uval) {
  long long u = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (u >= nu) return;
  uval[u] *= scale[u_row[u]] * scale[u_col[u]];
}

__global__ void k_fill(int n, double* x, double v) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) x[i] = v;
}

// --------------------------------------------------------------------------------------------
// pivoted LDL^T of a dense symmetric front held in shared memory (full square storage).
//   F   : f x f, leading dimension ld, LOWER triangle valid on entry (the strictly upper part is never read)
//   k   : number of fully-summed (pivot) columns, candidates are rows/cols [0,k)
//   lp  : k ints, out: pivot position t holds original local column lp[t]
//   pt  : k ints, out: pivot type (1, 2, 3)
//   cv1, cv2 : f doubles scratch;  sh : >= 4 ints scratch
//   dinv/doff : global arrays already offset to this front's first pivot
// On exit columns [0,k) of F hold L (strictly lower part; F[t+1,t] of a 2x2 pivot holds the
// off-diagonal of D and must be written out as 0) and F[k:, k:] holds the Schur complement.
// All threads of the CTA must call this; blockDim.x is a multiple of 32.
// --------------------------------------------------------------------------------------------
__device__ __forceinline__ void warp_argmax(double& v, int& idx) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    double ov = __shfl_xor_sync(0xffffffffu, v, o);
    int oi = __shfl_xor_sync(0xffffffffu, idx, o);
    if (ov > v || (ov == v && oi >= 0 && (idx < 0 || oi < idx))) { v = ov; idx = oi; }
  }
}
__device__ __forceinline__ double warp_max(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmax(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

// warp-wide max of floats in ONE reduction instruction: REDUX.MAX on an order-preserving integer image of the float
// (non-negative floats keep their bits, negative ones -- the -1 "no candidate" sentinels -- get their magnitude bits
// flipped), NaN ignored unless every lane holds one, as redux.sync.max.f32 does.  The pivot SEARCH runs on float-rounded
// magnitudes (the tests are inequalities with slack >= 1e-8, the selected entries are then re-read exactly).
__device__ __forceinline__ float wredux_max(float v) {
  const int b = __float_as_int(v);
  const int m = __reduce_max_sync(0xffffffffu, (v != v) ? INT_MIN : (b ^ ((b >> 31) & 0x7fffffff)));
  return (m == INT_MIN) ? __int_as_float(0x7fffffff) : __int_as_float(m ^ ((m >> 31) & 0x7fffffff));
}

// The pivoted front factorisation runs either on a whole CTA (WARP=false, __syncthreads) or on a single
// warp (WARP=true, __syncwarp; several fronts per CTA).
template <bool WARP>
__device__ __forceinline__ void gsync() { if (WARP) __syncwarp(); else __syncthreads(); }

template <bool WARP>
__device__ void swap_sym(double* F, int ld, int f, int p, int q) {
  // symmetric interchange of rows/cols p < q of a matrix whose LOWER triangle is stored (the strictly upper part
  // of F is never read); one pass, index t handled by one thread; caller syncs before.
  const int tid = WARP ? (threadIdx.x & 31) : threadIdx.x, nt = WARP ? 32 : blockDim.x;
  if (p > q) { const int x = p; p = q; q = x; }
  for (int t = tid; t < f; t += nt) {
    double* u; double* v;
    if (t < p) { u = F + p + t * ld; v = F + q + t * ld; }             // row segments left of p
    else if (t == p) { u = F + p + p * ld; v = F + q + q * ld; }       // the two diagonal entries
    else if (t < q) { u = F + t + p * ld; v = F + q + t * ld; }        // column p below p  <->  row q between p and q
    else if (t == q) continue;                                         // F[q][p] stays
    else { u = F + t + p * ld; v = F + t + q * ld; }                   // column segments below q
    const double a = *u, b = *v;
    *u = b; *v = a;
  }
  gsync<WARP>();
}

template <bool WARP>
__device__ void factor_front_smem(double* F, int ld, int f, int k, int* lp, int* pt, double* cv1,
                                  double* cv2, volatile int* sh, double u, double tiny,
                                  double* dinv, double* doff, int* ptype_g, int* counters) {
  const int tid = WARP ? (threadIdx.x & 31) : threadIdx.x, nt = WARP ? 32 : blockDim.x;
  const int lane = tid & 31, warp = tid >> 5, nwarp = nt >> 5;
  for (int t = tid; t < k; t += nt) lp[t] = t;
  if (tid == 0) { sh[2] = 0; sh[6] = 0; }
  int par = 0;   // decisions alternate between sh[0..2] and sh[4..6]: no barrier needed before the next one is written
  int c_neg = 0, c_forced = 0, c_tiny = 0, c_2x2 = 0;  // only meaningful on thread 0
  int j = 0, kend = k, progress = 0;
  bool forced = false;
  gsync<WARP>();
  while (j < k) {
    if (j == kend) {  // no candidate left in this pass
      if (progress > 0) { kend = k; progress = 0; }
      else { forced = true; kend = k; }
    }
    // ---------------- pivot decision by warp 0 ----------------
    if (warp == 0) {
      int type = 0, r = -1;
      if (forced) {
        // every remaining candidate failed the threshold test: force 1x1 pivots.  If the whole remaining
        // column is rounding noise (scaled matrix, entries O(1)) the matrix is numerically singular.
        double cm = 0.0;
        for (int i = j + lane; i < f; i += 32) cm = fmax(cm, fabs(F[i + j * ld]));
        cm = (double)wredux_max(__double2float_ru(cm));
        type = 1; r = j;
        if (lane == 0) sh[4 * par + 2] = !(cm > 1e-12);
      } else {
        double lam = 0.0, gam = 0.0;
        int ridx = -1;
        for (int i = j + 1 + lane; i < f; i += 32) {
          double v = fabs(F[i + j * ld]);
          if (i < kend) { if (v > lam) { lam = v; ridx = i; } }
          else gam = fmax(gam, v);
        }
        {
          // one-instruction float reductions; the winning lane's exact (lam, ridx) pair is then broadcast
          const float lamf = (ridx >= 0) ? __double2float_ru(lam) : -1.0f;
          const float lmax = wredux_max(lamf);
          gam = (double)wredux_max(__double2float_ru(gam));
          const unsigned bal = __ballot_sync(0xffffffffu, ridx >= 0 && lamf == lmax);
          if (bal) {
            const int src = __ffs(bal) - 1;
            lam = __shfl_sync(0xffffffffu, lam, src);
            ridx = __shfl_sync(0xffffffffu, ridx, src);
          } else { lam = 0.0; ridx = -1; }
        }
        double ajj = fabs(F[j + j * ld]);
        bool ok1 = (ajj > tiny) && (ajj >= u * fmax(lam, gam));
        if (lam == 0.0 || ridx < 0) { if (ok1) { type = 1; r = j; } }
        else if (ok1 && ajj >= BK_ALPHA * lam) { type = 1; r = j; }
        else {
          r = ridx;
          double sig = 0.0, gamr = 0.0, cj = 0.0, cr = 0.0;
          for (int m = j + lane; m < f; m += 32) {
            if (m == r) continue;
            double v = (m < r) ? fabs(F[r + m * ld]) : fabs(F[m + r * ld]);
            if (m < kend) sig = fmax(sig, v); else gamr = fmax(gamr, v);
            if (m != j) { cr = fmax(cr, v); cj = fmax(cj, fabs(F[m + j * ld])); }
          }
          sig = (double)wredux_max(__double2float_ru(sig)); gamr = (double)wredux_max(__double2float_ru(gamr));
          cj = (double)wredux_max(__double2float_ru(cj)); cr = (double)wredux_max(__double2float_ru(cr));
          double arr = fabs(F[r + r * ld]);
          if (ok1 && ajj * sig >= BK_ALPHA * lam * lam) { type = 1; r = j; }
          else if (arr > tiny && arr >= BK_ALPHA * sig && arr >= u * fmax(sig, gamr)) { type = 2; }
          else {
            double a = F[j + j * ld], b = F[r + j * ld], c = F[r + r * ld];
            double det = a * c - b * b, adet = fabs(det);
            if (lam > tiny && adet > 0.0 && isfinite(adet) &&
                (fabs(c) * cj + fabs(b) * cr) * u <= adet && (fabs(a) * cr + fabs(b) * cj) * u <= adet)
              type = 3;
          }
        }
      }
      if (lane == 0) { sh[4 * par] = type; sh[4 * par + 1] = r; }
    }
    gsync<WARP>();
    const int type = sh[4 * par], r = sh[4 * par + 1], noise = sh[4 * par + 2];
    par ^= 1;
    if (type == 0) {  // reject for now: park column j at the end of the candidate range
      if (j != kend - 1) {
        swap_sym<WARP>(F, ld, f, j, kend - 1);
        if (tid == 0) { int t = lp[j]; lp[j] = lp[kend - 1]; lp[kend - 1] = t; }
      }
      --kend;
      continue;
    }
    if (type == 2 && r != j) {
      swap_sym<WARP>(F, ld, f, j, r);
      if (tid == 0) { int t = lp[j]; lp[j] = lp[r]; lp[r] = t; }
    }
    if (type == 3 && r != j + 1) {
      swap_sym<WARP>(F, ld, f, j + 1, r);
      if (tid == 0) { int t = lp[j + 1]; lp[j + 1] = lp[r]; lp[r] = t; }
    }
    if (type != 3) {
      // ---------------- 1x1 pivot at j ----------------
      double d = F[j + j * ld];
      if (forced) {
        if (noise || !(fabs(d) > tiny)) {  // zero (or NaN) pivot: static perturbation, reported as SINGULAR
          d = (d < 0.0) ? -1.5e-8 : 1.5e-8;
          if (tid == 0) ++c_tiny;
        } else {
          // static pivoting: lift the pivot to the threshold (see warp_ldlt32); cv2[j] holds max|column j|
          double offmax = 0.0;
          for (int i = j + 1; i < f; ++i) offmax = fmax(offmax, fabs(F[i + j * ld]));
          d = copysign(fmax(fabs(d), 1e-8 * offmax), d);
          if (tid == 0) ++c_forced;
        }
      }
      const double dv = d;
      const double rdv = 1.0 / dv;
      // Deferred scaling: column j keeps the UNSCALED values c = l * d (only the final write-out applies D^-1, kept in
      // cv1 = dinv / cv2 = doff), so the update below reads column j that nobody writes -- no barrier before it and no
      // separate scaling pass.
      if (tid == 0) {
        pt[j] = 1; dinv[j] = rdv; doff[j] = 0.0; ptype_g[j] = 1;
        cv1[j] = rdv; cv2[j] = 0.0;
        if (dv < 0.0) ++c_neg;
      }
      // trailing update, 4 columns per trip so the shared-memory loads overlap (latency-bound otherwise)
      const double* __restrict__ cj = F + j * ld;
      for (int i = j + 1 + lane; i < f; i += 32) {
        const double li = cj[i] * rdv;
        const int mend = min(i, k - 1);                 // pivot columns only: the contribution block is updated once, at the end
        int m = j + 1 + warp;
        for (; m + 3 * nwarp <= mend; m += 4 * nwarp) {   // lower triangle only: columns m <= i
          const double c0 = cj[m], c1 = cj[m + nwarp], c2 = cj[m + 2 * nwarp], c3 = cj[m + 3 * nwarp];
          double* q0 = F + i + m * ld;
          double* q1 = q0 + nwarp * ld;
          double* q2 = q1 + nwarp * ld;
          double* q3 = q2 + nwarp * ld;
          const double f0 = *q0, f1 = *q1, f2 = *q2, f3 = *q3;
          *q0 = fma(-li, c0, f0); *q1 = fma(-li, c1, f1); *q2 = fma(-li, c2, f2); *q3 = fma(-li, c3, f3);
        }
        for (; m <= mend; m += nwarp) F[i + m * ld] = fma(-li, cj[m], F[i + m * ld]);
      }
      gsync<WARP>();
      j += 1;
    } else {
      // ---------------- 2x2 pivot at (j, j+1) ----------------
      const double a = F[j + j * ld], b = F[j + 1 + j * ld], c = F[j + 1 + (j + 1) * ld];
      const double det = a * c - b * b;
      const double idet = 1.0 / det;
      const double da = c * idet, db = a * idet, dof = -b * idet;   // D^-1 of the 2x2 block
      if (tid == 0) {
        pt[j] = 2; pt[j + 1] = 3; ptype_g[j] = 2; ptype_g[j + 1] = 3;
        dinv[j] = da; dinv[j + 1] = db; doff[j] = dof; doff[j + 1] = 0.0;
        cv1[j] = da; cv1[j + 1] = db; cv2[j] = dof; cv2[j + 1] = 0.0;
        ++c_2x2;
        if (det < 0.0) c_neg += 1; else if (a < 0.0) c_neg += 2;
      }
      // columns j, j+1 stay unscaled (see the 1x1 case): l = [c1 c2] D^-1 is formed on the fly
      const double* __restrict__ cj = F + j * ld;
      const double* __restrict__ cj1 = F + (j + 1) * ld;
      for (int i = j + 2 + lane; i < f; i += 32) {
        const double r1 = cj[i], r2 = cj1[i];
        const double l1 = fma(r1, da, r2 * dof), l2 = fma(r1, dof, r2 * db);
        const int mend = min(i, k - 1);
        int m = j + 2 + warp;
        for (; m + 3 * nwarp <= mend; m += 4 * nwarp) {
          const double a0 = cj[m], a1 = cj[m + nwarp], a2 = cj[m + 2 * nwarp], a3 = cj[m + 3 * nwarp];
          const double b0 = cj1[m], b1 = cj1[m + nwarp], b2 = cj1[m + 2 * nwarp], b3 = cj1[m + 3 * nwarp];
          double* q0 = F + i + m * ld;
          double* q1 = q0 + nwarp * ld;
          double* q2 = q1 + nwarp * ld;
          double* q3 = q2 + nwarp * ld;
          const double f0 = *q0, f1 = *q1, f2 = *q2, f3 = *q3;
          *q0 = fma(-l2, b0, fma(-l1, a0, f0)); *q1 = fma(-l2, b1, fma(-l1, a1, f1));
          *q2 = fma(-l2, b2, fma(-l1, a2, f2)); *q3 = fma(-l2, b3, fma(-l1, a3, f3));
        }
        for (; m <= mend; m += nwarp) F[i + m * ld] = fma(-l2, cj1[m], fma(-l1, cj[m], F[i + m * ld]));
      }
      gsync<WARP>();
      j += 2;
    }
    ++progress;
  }
  // ---------------- deferred Schur complement of the contribution block ----------------
  // CB[i][m] -= sum_t L[i][t] W[m][t] (i >= m >= k), W = L D = the unscaled pivot columns.  Entry (i, m) belongs to one thread
  // (lane <- row, warp <- column), so there is no barrier inside; the L entries of a row are formed once per chunk of 8
  // pivots and reused for all its columns.  (During the pivot loop only the k pivot columns were updated: the pivot search
  // and the interchanges never look at the contribution block.)
  if (f > k) {
    for (int i = k + lane; i < f; i += 32) {
      for (int t0 = 0; t0 < k; t0 += 8) {
        double l[8];
#pragma unroll
        for (int q = 0; q < 8; ++q) {
          const int t = t0 + q;
          double v = 0.0;
          if (t < k) {
            const int ty = pt[t];
            if (ty == 1) v = F[i + t * ld] * cv1[t];
            else if (ty == 2) v = fma(F[i + t * ld], cv1[t], F[i + (t + 1) * ld] * cv2[t]);
            else v = fma(F[i + (t - 1) * ld], cv2[t - 1], F[i + t * ld] * cv1[t]);
          }
          l[q] = v;
        }
        for (int m = k + warp; m <= i; m += nwarp) {
          double acc = F[i + m * ld];
#pragma unroll
          for (int q = 0; q < 8; ++q)
            if (t0 + q < k) acc = fma(-l[q], F[m + (t0 + q) * ld], acc);
          F[i + m * ld] = acc;
        }
      }
    }
  }
  if (tid == 0) {
    if (c_neg) atomicAdd(counters + CNT_NEG, c_neg);
    if (c_forced) atomicAdd(counters + CNT_FORCED, c_forced);
    if (c_tiny) atomicAdd(counters + CNT_TINY, c_tiny);
    if (c_2x2) atomicAdd(counters + CNT_2X2, c_2x2);
  }
  gsync<WARP>();
}

// --------------------------------------------------------------------------------------------
// Register-resident pivoted LDL^T of a symmetric front of order f <= 32 by ONE warp.
//   lane i owns ROW i (original local index) of the full symmetric matrix: a[c] = F[i][column at position c];
//   column positions are kept compacted ("cid[c]" = original index of the column at position c, uniform
//   across lanes) so every register index is a compile-time constant: the pivot column is always a[0], a 2x2
//   partner is first swapped to a[1], and after an elimination all columns shift left.
//   Rows never move: the pivot row is reached with warp shuffles (F[g][c] = F[c][g] = lane cid[c]'s a[0]).
// Same pivot rule as factor_front_smem (Bunch-Kaufman inside the candidates [0,k), threshold u against the
// whole column, failed columns retried after the others, forced + flagged at the very end).
// Output: Lraw[i*33 + t] = L entry of original row i in pivot column t; order[t] = original index of pivot t;
//         pt/dinv_s/doff_s per pivot; on exit a[c], c < f-k, holds the Schur complement column k+c for row i.
// --------------------------------------------------------------------------------------------
__device__ __forceinline__ void wred_max_idx(double& v, int& idx) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    double ov = __shfl_xor_sync(0xffffffffu, v, o);
    int oi = __shfl_xor_sync(0xffffffffu, idx, o);
    if (ov > v || (ov == v && oi < idx)) { v = ov; idx = oi; }
  }
}

// TWO = true: fronts of order 33..64 with k <= 32.  The warp also carries rows 32..f-1 (lane -> row 32 + lane) of the
// first 32 columns in b[]: they are never pivot candidates (all candidates are among rows 0..k-1 < 32), but they take part
// in every threshold test, receive every update (so b[c], c < 32-k, ends as the Schur complement column k+c of row
// 32+lane) and their L entries go to Lraw[(32+lane)*33 + t].  The block rows >= 32 x columns >= 32 of the Schur
// complement is formed afterwards from L and D (dpiv/dpb: the pivots themselves, see k_front_warp2).
template <bool TWO>
__device__ void warp_ldlt32(double (&a)[32], double (&b)[32], const int f, const int k, const double u, const double tiny,
                            double* __restrict__ Lraw, int* __restrict__ order, int* __restrict__ pt,
                            double* __restrict__ dinv_s, double* __restrict__ doff_s,
                            double* __restrict__ colbuf /* 64 doubles of shared memory, 16-byte aligned */,
                            const double gext /* lane c: max |entry| of column c in rows OUTSIDE the block (0 if none) */,
                            int* counters, double* __restrict__ dpiv = nullptr, double* __restrict__ dpb = nullptr) {
  const int lane = threadIdx.x & 31;
  // mypos = current POSITION of the column whose original index is this lane (columns stay compacted)
  int mypos = lane;
  colbuf[lane] = 0.0; colbuf[32 + lane] = 0.0;
  __syncwarp();
  const bool me2 = TWO && (lane + 32 < f);          // this lane carries a second row
  unsigned alive = (f >= 32) ? 0xffffffffu : ((1u << f) - 1u);
  unsigned cand = (k >= 32) ? 0xffffffffu : ((1u << k) - 1u);
  int nc = k, npass = k, t = 0, progress = 0;
  bool forced = false;
  int c_neg = 0, c_forced = 0, c_tiny = 0, c_2x2 = 0;
  int my_order = 0, my_pt = 1;
  double my_dinv = 0.0, my_doff = 0.0;
  while (nc > 0) {
    if (npass == 0) {
      if (progress > 0) { npass = nc; progress = 0; }
      else { forced = true; npass = nc; }
    }
    const bool me_alive = (alive >> lane) & 1u;
    const bool me_cand = (cand >> lane) & 1u;
    int g0 = __ffs(__ballot_sync(0xffffffffu, me_alive && mypos == 0)) - 1;
    // ---- pivot search on column 0 ----
    const double v0 = fabs(a[0]);
    const float v0f = __double2float_ru(v0);
    const float lam_in = (me_cand && lane != g0) ? v0f : -1.0f;
    const float lamf = wredux_max(lam_in);
    float gam_in = (me_alive && !me_cand) ? v0f : 0.0f;
    float w0f = 0.0f;
    if (TWO) { w0f = me2 ? __double2float_ru(fabs(b[0])) : 0.0f; gam_in = fmaxf(gam_in, w0f); }
    const float gamf = wredux_max(gam_in);
    int r = __ffs(__ballot_sync(0xffffffffu, lam_in == lamf)) - 1;   // lowest lane holding the maximum
    double lam = 0.0;
    if (lamf < 0.0f) r = -1;
    else lam = __shfl_sync(0xffffffffu, v0, r);                       // exact magnitude of the selected entry
    const double gam = fmax((double)gamf, __shfl_sync(0xffffffffu, gext, g0));
    const double ajj = fabs(__shfl_sync(0xffffffffu, a[0], g0));
    const bool ok1 = (ajj > tiny) && (ajj >= u * fmax(lam, gam));
    int type = 0;
    bool noise = false;
    const double colmax_f = fmax(lam, gam);
    if (forced) { type = 1; noise = !(fmax(ajj, colmax_f) > 1e-12); }
    else if (lam == 0.0 || r < 0) { if (ok1) type = 1; }
    else if (ok1 && ajj >= BK_ALPHA * lam) type = 1;
    else {
      // bring column r to position 1
      const int p = __shfl_sync(0xffffffffu, mypos, r);
      if (p > 1) {
        double ta = a[1];
#pragma unroll
        for (int c = 2; c < 32; ++c)
          if (c == p) { double x = a[c]; a[c] = ta; ta = x; }
        a[1] = ta;
        if (TWO) {
          double tb = b[1];
#pragma unroll
          for (int c = 2; c < 32; ++c)
            if (c == p) { double x = b[c]; b[c] = tb; tb = x; }
          b[1] = tb;
        }
        if (mypos == 1) mypos = p; else if (mypos == p) mypos = 1;
      }
      const double v1 = fabs(a[1]);
      const float v1f = __double2float_ru(v1);
      const bool other = me_alive && lane != g0 && lane != r;
      const float w1f = (TWO && me2) ? __double2float_ru(fabs(b[1])) : 0.0f;   // the second rows are always "other" rows
      double sig = (double)wredux_max((me_cand && lane != r) ? v1f : 0.0f);
      double gamr = (double)wredux_max(fmaxf((me_alive && !me_cand) ? v1f : 0.0f, w1f));
      double cj = (double)wredux_max(fmaxf(other ? v0f : 0.0f, w0f)), cr = (double)wredux_max(fmaxf(other ? v1f : 0.0f, w1f));
      {
        const double ge_r = __shfl_sync(0xffffffffu, gext, r), ge_j = __shfl_sync(0xffffffffu, gext, g0);
        gamr = fmax(gamr, ge_r); cr = fmax(cr, ge_r); cj = fmax(cj, ge_j);
      }
      const double crr = __shfl_sync(0xffffffffu, a[1], r);
      const double arr = fabs(crr);
      if (ok1 && ajj * sig >= BK_ALPHA * lam * lam) type = 1;
      else if (arr > tiny && arr >= BK_ALPHA * sig && arr >= u * fmax(sig, gamr)) {
        // 1x1 on r: swap positions 0 and 1
        double x = a[0]; a[0] = a[1]; a[1] = x;
        if (TWO) { double y = b[0]; b[0] = b[1]; b[1] = y; }
        if (mypos == 0) mypos = 1; else if (mypos == 1) mypos = 0;
        g0 = r;
        type = 1;
      } else {
        const double pa = __shfl_sync(0xffffffffu, a[0], g0), pb = __shfl_sync(0xffffffffu, a[0], r);
        const double det = pa * crr - pb * pb, adet = fabs(det);
        if (lam > tiny && adet > 0.0 && isfinite(adet) &&
            (fabs(crr) * cj + fabs(pb) * cr) * u <= adet && (fabs(pa) * cr + fabs(pb) * cj) * u <= adet)
          type = 3;
      }
    }
    if (type == 0) {
      // park column 0 behind the remaining candidates (position nc-1) and try the next one
      const double ta = a[0];
#pragma unroll
      for (int c = 0; c < 31; ++c) {
        if (c < nc - 1) a[c] = a[c + 1];
        else if (c == nc - 1) a[c] = ta;
      }
      if (nc == 32) a[31] = ta;
      if (TWO) {
        const double tb = b[0];
#pragma unroll
        for (int c = 0; c < 31; ++c) {
          if (c < nc - 1) b[c] = b[c + 1];
          else if (c == nc - 1) b[c] = tb;
        }
        if (nc == 32) b[31] = tb;
      }
      if (mypos == 0) mypos = nc - 1; else if (mypos < nc) mypos -= 1;
      --npass;
      continue;
    }
    if (type == 1) {
      double dd = __shfl_sync(0xffffffffu, a[0], g0);
      if (forced) {
        if (noise || !(fabs(dd) > tiny)) { dd = (dd < 0.0) ? -1.5e-8 : 1.5e-8; ++c_tiny; }
        else {
          // static pivoting: a pivot that fails the threshold test everywhere in its supernode is lifted to the
          // threshold (|l_ij| stays <= 1e8; the factors are those of a matrix perturbed by <= 1e-8 |column|,
          // which the caller's iterative refinement absorbs).  Counted and reported in num_forced.
          dd = copysign(fmax(fabs(dd), 1e-8 * colmax_f), dd);
          ++c_forced;
        }
      }
      const double c0v = a[0];
      const double rinv = 1.0 / dd;
      const double l = (me_alive && lane != g0) ? c0v * rinv : 0.0;
      const double lb = (TWO && me2) ? b[0] * rinv : 0.0;
      // pivot row by position: F[g0][col at position c] = F[that col's row][g0] = that lane's a[0]
      if (me_alive) colbuf[mypos] = c0v;
      __syncwarp();
      const double2* cb2 = reinterpret_cast<const double2*>(colbuf);
#pragma unroll
      for (int c2 = 0; c2 < 16; ++c2) {
        const double2 pp = cb2[c2];
        if (c2 > 0) a[2 * c2] = fma(-l, pp.x, a[2 * c2]);
        a[2 * c2 + 1] = fma(-l, pp.y, a[2 * c2 + 1]);
        if (TWO) {
          if (c2 > 0) b[2 * c2] = fma(-lb, pp.x, b[2 * c2]);
          b[2 * c2 + 1] = fma(-lb, pp.y, b[2 * c2 + 1]);
        }
      }
      __syncwarp();
      Lraw[lane * 33 + t] = l;
      if (TWO) { Lraw[(32 + lane) * 33 + t] = lb; if (lane == 0) { dpiv[t] = dd; dpb[t] = 0.0; } }
      if (lane == t) { my_order = g0; my_pt = 1; my_dinv = rinv; my_doff = 0.0; }   // lane t keeps pivot t's record
      if (dd < 0.0) ++c_neg;
      alive &= ~(1u << g0); cand &= ~(1u << g0);
#pragma unroll
      for (int c = 0; c < 31; ++c) a[c] = a[c + 1];
      a[31] = 0.0;
      if (TWO) {
#pragma unroll
        for (int c = 0; c < 31; ++c) b[c] = b[c + 1];
        b[31] = 0.0;
      }
      mypos -= 1;
      nc -= 1; npass = max(npass - 1, 0); t += 1;
    } else {
      const double pa = __shfl_sync(0xffffffffu, a[0], g0), pb = __shfl_sync(0xffffffffu, a[0], r);
      const double pc2 = __shfl_sync(0xffffffffu, a[1], r);
      const double det = pa * pc2 - pb * pb;
      const double c1 = a[0], c2v = a[1];
      const bool other = me_alive && lane != g0 && lane != r;
      const double idet = 1.0 / det;
      const double l1 = other ? (pc2 * c1 - pb * c2v) * idet : 0.0;
      const double l2 = other ? (pa * c2v - pb * c1) * idet : 0.0;
      const double e1 = TWO ? b[0] : 0.0, e2 = TWO ? b[1] : 0.0;
      const double m1 = (TWO && me2) ? (pc2 * e1 - pb * e2) * idet : 0.0;
      const double m2 = (TWO && me2) ? (pa * e2 - pb * e1) * idet : 0.0;
      if (me_alive) { colbuf[mypos] = c1; colbuf[32 + mypos] = c2v; }
      __syncwarp();
      const double2* cb1 = reinterpret_cast<const double2*>(colbuf);
      const double2* cb2 = reinterpret_cast<const double2*>(colbuf + 32);
#pragma unroll
      for (int q = 1; q < 16; ++q) {
        const double2 p1 = cb1[q], p2 = cb2[q];
        a[2 * q] = fma(-l2, p2.x, fma(-l1, p1.x, a[2 * q]));
        a[2 * q + 1] = fma(-l2, p2.y, fma(-l1, p1.y, a[2 * q + 1]));
        if (TWO) {
          b[2 * q] = fma(-m2, p2.x, fma(-m1, p1.x, b[2 * q]));
          b[2 * q + 1] = fma(-m2, p2.y, fma(-m1, p1.y, b[2 * q + 1]));
        }
      }
      __syncwarp();
      Lraw[lane * 33 + t] = l1;
      Lraw[lane * 33 + t + 1] = l2;
      if (TWO) {
        Lraw[(32 + lane) * 33 + t] = m1;
        Lraw[(32 + lane) * 33 + t + 1] = m2;
        if (lane == 0) { dpiv[t] = pa; dpb[t] = pb; dpiv[t + 1] = pc2; dpb[t + 1] = 0.0; }
      }
      if (lane == t) { my_order = g0; my_pt = 2; my_dinv = pc2 * idet; my_doff = -pb * idet; }
      if (lane == t + 1) { my_order = r; my_pt = 3; my_dinv = pa * idet; my_doff = 0.0; }
      ++c_2x2;
      if (det < 0.0) c_neg += 1; else if (pa < 0.0) c_neg += 2;
      alive &= ~((1u << g0) | (1u << r)); cand &= ~((1u << g0) | (1u << r));
#pragma unroll
      for (int c = 0; c < 30; ++c) a[c] = a[c + 2];
      a[30] = 0.0; a[31] = 0.0;
      if (TWO) {
#pragma unroll
        for (int c = 0; c < 30; ++c) b[c] = b[c + 2];
        b[30] = 0.0; b[31] = 0.0;
      }
      mypos -= 2;
      nc -= 2; npass = max(npass - 2, 0); t += 2;
    }
    ++progress;
  }
  if (lane < k) { order[lane] = my_order; pt[lane] = my_pt; dinv_s[lane] = my_dinv; doff_s[lane] = my_doff; }
  if (lane == 0) {
    if (c_neg) atomicAdd(counters + CNT_NEG, c_neg);
    if (c_forced) atomicAdd(counters + CNT_FORCED, c_forced);
    if (c_tiny) atomicAdd(counters + CNT_TINY, c_tiny);
    if (c_2x2) atomicAdd(counters + CNT_2X2, c_2x2);
  }
  __syncwarp();
}

// --------------------------------------------------------------------------------------------
// Class S/M: one CTA per front, everything in shared memory.
// smem: F[ld*f] | cv1[f] | cv2[f] | lp[k] | pt[k] | sh[8]
// --------------------------------------------------------------------------------------------
template <bool WARP>
__global__ void k_front_smem(DevSym S, DevNum N, const int* __restrict__ front_list, int nfronts,
                             int smem_per_group /*bytes, WARP mode only*/) {
  extern __shared__ double smem[];
  const int group = WARP ? (blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5)) : blockIdx.x;
  if (group >= nfronts) return;
  const int s = front_list[group];
  const int c0 = S.sn_start[s], k = S.sn_start[s + 1] - c0;
  const int r = (int)(S.rows_ptr[s + 1] - S.rows_ptr[s]);
  const int f = k + r, ld = f | 1;
  double* F = WARP ? (double*)((char*)smem + (size_t)(threadIdx.x >> 5) * smem_per_group) : smem;
  double* cv1 = F + (size_t)ld * f;
  double* cv2 = cv1 + f;
  int* lp = (int*)(cv2 + f);
  int* pt = lp + k;
  int* sh = pt + k;
  const int tid = WARP ? (threadIdx.x & 31) : threadIdx.x, nt = WARP ? 32 : blockDim.x;
  unsigned long long ts[4];
  const bool tlog = N.flog != nullptr && threadIdx.x == 0 && (blockIdx.x == 0 || blockIdx.x == gridDim.x - 1);
  if (tlog) ts[0] = flog_now();

  for (int t = tid; t < ld * f; t += nt) F[t] = 0.0;
  gsync<WARP>();
  // original entries (unique -> no write conflicts)
  for (long long uu = S.uent_ptr[s] + tid; uu < S.uent_ptr[s + 1]; uu += nt) {
    unsigned d = S.u_dst[uu];
    int lr = d & 0xffffu, lc = d >> 16;
    F[lr + lc * ld] = N.uval[uu];   // lower triangle only (lr >= lc)
  }
  gsync<WARP>();
  // extend-add of the children contribution blocks, one child at a time (deterministic)
  for (int q = S.child_ptr[s]; q < S.child_ptr[s + 1]; ++q) {
    const int c = S.child_idx[q];
    const int rc = (int)(S.rows_ptr[c + 1] - S.rows_ptr[c]);
    const double* __restrict__ cb = N.CB + S.cb_off[c];
    const int* __restrict__ rl = S.rel + S.rows_ptr[c];
    for (int jj = tid >> 5; jj < rc; jj += (nt >> 5)) {
      const int lj = rl[jj];
      for (int ii = jj + (tid & 31); ii < rc; ii += 32) {
        const int li = rl[ii];
        F[li + lj * ld] += cb[ii + (size_t)jj * rc];   // rel is increasing: li >= lj
      }
    }
    gsync<WARP>();
  }

  if (tlog) ts[1] = flog_now();
  factor_front_smem<WARP>(F, ld, f, k, lp, pt, cv1, cv2, sh, N.u, N.tiny, N.dinv + c0, N.doff + c0,
                          N.ptype + c0, N.counters);
  if (tlog) ts[2] = flog_now();

  // write L panel (f x k, ld = f), unit diagonal.  The strictly-upper part of the k x k pivot block receives L11^T
  // (entry (i, t), i < t, = L[t][i]): the backward solve of the small fronts reads row t of L11 as the contiguous
  // column segment P[0..t) + t*f instead of a stride-f gather (solve_dataflow.cu, w64_bwd).
  // (the pivot columns of F hold the unscaled values L*D: apply D^-1 = {cv1 = dinv, cv2 = doff} here)
  double* __restrict__ P = N.L + S.L_off[s];
  auto lval = [&](int row, int col) -> double {   // L[row][col], row > col
    const int ty = pt[col];
    if (ty == 1) return F[row + col * ld] * cv1[col];
    if (ty == 2) return (row == col + 1) ? 0.0 : fma(F[row + col * ld], cv1[col], F[row + (col + 1) * ld] * cv2[col]);
    return fma(F[row + (col - 1) * ld], cv2[col - 1], F[row + col * ld] * cv1[col]);
  };
  for (int t = tid >> 5; t < k; t += (nt >> 5)) {
    for (int i = tid & 31; i < f; i += 32) {
      double v;
      if (i < t) v = lval(t, i);
      else if (i == t) v = 1.0;
      else v = lval(i, t);
      P[i + (size_t)t * f] = v;
    }
  }
  for (int t = tid; t < k; t += nt) N.lperm[c0 + t] = lp[t];
  // contribution block (lower part)
  double* __restrict__ cbo = N.CB + S.cb_off[s];
  for (int m = tid >> 5; m < r; m += (nt >> 5))
    for (int i = m + (tid & 31); i < r; i += 32) cbo[i + (size_t)m * r] = F[(k + i) + (k + m) * ld];
  if (tlog) { ts[3] = flog_now(); flog_put(N, 4, s, f, ts, 4); }
}

// --------------------------------------------------------------------------------------------
// Class XS: fronts of order <= 32, ONE WARP per front (4 fronts per CTA), factorisation in registers.
// smem per warp: F/Lraw[33*32] doubles | dinv_s[32] | doff_s[32] | order[32] | pt[32]
// --------------------------------------------------------------------------------------------
#define XS_SMEM_PER_WARP ((33 * 32 + 64 + 64) * 8 + 64 * 4)
__global__ void __launch_bounds__(128) k_front_warp(DevSym S, DevNum N, const int* __restrict__ front_list, int nfronts) {
  extern __shared__ double smem[];
  const int group = blockIdx.x * 4 + (threadIdx.x >> 5);
  if (group >= nfronts) return;
  const int s = front_list[group];
  FlogScope fs(N, 5, s, 0);
  const int c0 = S.sn_start[s], k = S.sn_start[s + 1] - c0;
  const int r = (int)(S.rows_ptr[s + 1] - S.rows_ptr[s]);
  const int f = k + r;
  double* F = (double*)((char*)smem + (size_t)(threadIdx.x >> 5) * XS_SMEM_PER_WARP);
  double* colbuf = F + 33 * 32;       // 64 doubles (offset 8448 B: 16-byte aligned)
  double* dinv_s = colbuf + 64;
  double* doff_s = dinv_s + 32;
  int* order = (int*)(doff_s + 32);
  int* pt = order + 32;
  const int lane = threadIdx.x & 31;
  const int ld = 33;
  for (int t = lane; t < 33 * 32; t += 32) F[t] = 0.0;
  __syncwarp();
  for (long long uu = S.uent_ptr[s] + lane; uu < S.uent_ptr[s + 1]; uu += 32) {
    unsigned d = S.u_dst[uu];
    int lr = d & 0xffffu, lc = d >> 16;
    double v = N.uval[uu];
    F[lr + lc * ld] = v;
    F[lc + lr * ld] = v;
  }
  __syncwarp();
  for (int q = S.child_ptr[s]; q < S.child_ptr[s + 1]; ++q) {
    const int c = S.child_idx[q];
    const int rc = (int)(S.rows_ptr[c + 1] - S.rows_ptr[c]);
    const double* __restrict__ cb = N.CB + S.cb_off[c];
    const int* __restrict__ rl = S.rel + S.rows_ptr[c];
    const int li = (lane < rc) ? rl[lane] : 0;
    for (int jj = 0; jj < rc; ++jj) {
      const int lj = __shfl_sync(0xffffffffu, li, jj);
      if (lane >= jj && lane < rc) {
        const double v = cb[lane + (size_t)jj * rc];
        F[li + lj * ld] += v;
        if (li != lj) F[lj + li * ld] += v;
      }
    }
    __syncwarp();
  }
  double a[32];
#pragma unroll
  for (int c = 0; c < 32; ++c) a[c] = F[lane + c * ld];   // lanes >= f / columns >= f read zeros
  __syncwarp();
  warp_ldlt32<false>(a, a, f, k, N.u, N.tiny, F, order, pt, dinv_s, doff_s, colbuf, 0.0, N.counters);
  // L panel in pivot order
  double* __restrict__ P = N.L + S.L_off[s];
  const int orig = (lane < k) ? order[lane] : lane;
#pragma unroll
  for (int t = 0; t < 32; ++t) {
    if (t < k && lane < f) {
      double v;
      if (lane < t) v = F[order[t] * 33 + lane];   // L11^T in the upper triangle (see k_front_smem)
      else if (lane == t) v = 1.0;
      else v = F[orig * 33 + t];
      P[lane + (size_t)t * f] = v;
    }
  }
  if (lane < k) {
    N.lperm[c0 + lane] = order[lane];
    N.dinv[c0 + lane] = dinv_s[lane];
    N.doff[c0 + lane] = doff_s[lane];
    N.ptype[c0 + lane] = pt[lane];
  }
  // contribution block (lower part): row = lane (>= k), column position c <-> original column k + c
  double* __restrict__ cbo = N.CB + S.cb_off[s];
#pragma unroll
  for (int c = 0; c < 32; ++c)
    if (lane >= k && lane < f && c <= lane - k) cbo[(lane - k) + (size_t)c * r] = a[c];
  fs.done();
}

// --------------------------------------------------------------------------------------------
// Class S2: fronts of order 33..64 with at most 32 pivot columns, ONE WARP per front (4 fronts per CTA), two rows per lane:
// the first 32 columns of the front are factorised in registers (warp_ldlt32<true>: rows 0..31 in a[], rows 32..f-1 in
// b[]); the trailing block rows >= 32 x columns >= 32 of the contribution block is  C22 - L2 D L2^T  formed afterwards
// from the finished panel (lane = row, L rows of the partners broadcast from shared memory).
// smem per warp: P0/Lraw[64*33] doubles (P0 = first 32 columns, column-major ld 66; aliased by Lraw once the columns are
//   in registers) | C22[32*33] | colbuf[64] | dinv_s[32] | doff_s[32] | dpiv[32] | dpb[32] | order[32] | pt[32]
// --------------------------------------------------------------------------------------------
#define S2_LD 66
#define S2_SMEM_PER_WARP ((64 * 33 + 32 * 33 + 64 + 4 * 32) * 8 + 64 * 4)
__global__ void __launch_bounds__(128, 2) k_front_warp2(DevSym S, DevNum N, const int* __restrict__ front_list, int nfronts) {
  extern __shared__ double smem[];
  const int group = blockIdx.x * 4 + (threadIdx.x >> 5);
  if (group >= nfronts) return;
  const int s = front_list[group];
  FlogScope fs(N, 5, s, 1);
  const int c0 = S.sn_start[s], k = S.sn_start[s + 1] - c0;
  const int r = (int)(S.rows_ptr[s + 1] - S.rows_ptr[s]);
  const int f = k + r, f1 = f - 32;            // 32 < f <= 64, k <= 32 (guaranteed by the launch plan)
  double* P0 = (double*)((char*)smem + (size_t)(threadIdx.x >> 5) * S2_SMEM_PER_WARP);
  double* C22 = P0 + 64 * 33;
  double* colbuf = C22 + 32 * 33;        // offset (2112 + 1056) * 8 bytes: 16-byte aligned
  double* dinv_s = colbuf + 64;
  double* doff_s = dinv_s + 32;
  double* dpiv = doff_s + 32;
  double* dpb = dpiv + 32;
  int* order = (int*)(dpb + 32);
  int* pt = order + 32;
  const int lane = threadIdx.x & 31;
  for (int t = lane; t < 64 * 33 + 32 * 33; t += 32) P0[t] = 0.0;
  __syncwarp();
  // entry (li, lj), li >= lj, of the front: columns < 32 live in P0 (the top 32 x 32 block with both triangles), the rest in C22
  auto put = [&](int li, int lj, double v, bool add) {
    if (lj < 32) {
      double* d1 = P0 + li + lj * S2_LD;
      *d1 = add ? *d1 + v : v;
      if (li < 32 && li != lj) { double* d2 = P0 + lj + li * S2_LD; *d2 = add ? *d2 + v : v; }
    } else {
      double* d1 = C22 + (li - 32) + (lj - 32) * 33;
      *d1 = add ? *d1 + v : v;
    }
  };
  for (long long uu = S.uent_ptr[s] + lane; uu < S.uent_ptr[s + 1]; uu += 32) {
    const unsigned d = S.u_dst[uu];
    put((int)(d & 0xffffu), (int)(d >> 16), N.uval[uu], false);     // unique entries: no write conflicts
  }
  __syncwarp();
  const int ch0 = S.child_ptr[s], nch = S.child_ptr[s + 1] - ch0;
  for (int q0 = 0; q0 < nch; q0 += 32) {
   // the descriptors of up to 32 children lane-parallel (three dependent global loads each), then the children in order
   long long m_cb = 0, m_ro = 0;
   int m_rc = 0;
   if (q0 + lane < nch) {
     const int c = S.child_idx[ch0 + q0 + lane];
     m_ro = S.rows_ptr[c]; m_rc = (int)(S.rows_ptr[c + 1] - m_ro); m_cb = S.cb_off[c];
   }
   for (int qq = 0; qq < min(32, nch - q0); ++qq) {
    const int rc = __shfl_sync(0xffffffffu, m_rc, qq);              // <= 63: the child's rows are rows of this front
    const double* __restrict__ cb = N.CB + __shfl_sync(0xffffffffu, m_cb, qq);
    const int* __restrict__ rl = S.rel + __shfl_sync(0xffffffffu, m_ro, qq);
    const int li0 = (lane < rc) ? rl[lane] : 0, li1 = (lane + 32 < rc) ? rl[lane + 32] : 0;
    // rel is strictly increasing inside a child, so the entries (ii, jj) of one child land on pairwise distinct addresses
    // (the mirrored writes of the top block included): no synchronisation inside a child, and the loads of 8 columns are in
    // flight together (the loop is latency-bound otherwise: one dependent global load per column)
    for (int jj0 = 0; jj0 < rc; jj0 += 8) {
      double v0[8], v1[8];
#pragma unroll
      for (int u = 0; u < 8; ++u) {
        const int jj = jj0 + u;
        v0[u] = (jj < rc && lane >= jj && lane < rc) ? cb[lane + (size_t)jj * rc] : 0.0;
        v1[u] = (jj < rc && lane + 32 >= jj && lane + 32 < rc) ? cb[lane + 32 + (size_t)jj * rc] : 0.0;
      }
#pragma unroll
      for (int u = 0; u < 8; ++u) {
        const int jj = jj0 + u;
        if (jj < rc) {     // warp-uniform
          const int lj = (jj < 32) ? __shfl_sync(0xffffffffu, li0, jj) : __shfl_sync(0xffffffffu, li1, jj - 32);
          if (lane >= jj && lane < rc) put(li0, lj, v0[u], true);
          if (lane + 32 >= jj && lane + 32 < rc) put(li1, lj, v1[u], true);
        }
      }
    }
    __syncwarp();
   }
  }
  double a[32], b[32];
#pragma unroll
  for (int c = 0; c < 32; ++c) { a[c] = P0[lane + c * S2_LD]; b[c] = P0[32 + lane + c * S2_LD]; }   // rows >= f read zeros
  __syncwarp();     // every lane has its columns: the region becomes Lraw
  double* Lraw = P0;
  warp_ldlt32<true>(a, b, f, k, N.u, N.tiny, Lraw, order, pt, dinv_s, doff_s, colbuf, 0.0, N.counters, dpiv, dpb);
  // L panel in pivot order (f x k, ld = f); L11^T in the upper triangle of the pivot block (see k_front_smem)
  double* __restrict__ P = N.L + S.L_off[s];
  const int orig = (lane < k) ? order[lane] : lane;
#pragma unroll 4
  for (int t = 0; t < 32; ++t) {
    if (t < k) {
      double v;
      if (lane < t) v = Lraw[order[t] * 33 + lane];
      else if (lane == t) v = 1.0;
      else v = Lraw[orig * 33 + t];
      P[lane + (size_t)t * f] = v;
      if (lane < f1) P[32 + lane + (size_t)t * f] = Lraw[(32 + lane) * 33 + t];
    }
  }
  if (lane < k) {
    N.lperm[c0 + lane] = order[lane];
    N.dinv[c0 + lane] = dinv_s[lane];
    N.doff[c0 + lane] = doff_s[lane];
    N.ptype[c0 + lane] = pt[lane];
  }
  // contribution block (lower part, r x r, ld = r).  Columns k..31 of the front: what is left in a[] / b[].
  double* __restrict__ cbo = N.CB + S.cb_off[s];
#pragma unroll
  for (int c = 0; c < 32; ++c) {
    if (c < 32 - k) {
      if (lane >= k && c <= lane - k) cbo[(lane - k) + (size_t)c * r] = a[c];
      if (lane < f1) cbo[(32 - k + lane) + (size_t)c * r] = b[c];
    }
  }
  // columns >= 32: C22[i][j] - sum_t (L D)[i][t] L[j][t], row i = 32 + lane, partners j <= lane
  {
    double wrow[32];
#pragma unroll
    for (int t = 0; t < 32; ++t) wrow[t] = (t < k && lane < f1) ? Lraw[(32 + lane) * 33 + t] : 0.0;
    // w = l D: 1x1 pivots w_t = l_t d_t; 2x2 pivots (t, t+1): w_t = l_t d_tt + l_t+1 d_o, w_t+1 = l_t d_o + l_t+1 d_t+1,t+1
    double prevl = 0.0;
#pragma unroll
    for (int t = 0; t < 32; ++t) {
      const double lt = wrow[t];
      if (t < k) {
        const int ty = pt[t];
        double w = lt * dpiv[t];
        if (ty == 2) w = fma(wrow[(t + 1) & 31], dpb[t], w);          // (still the L entry: ascending t)
        else if (ty == 3) w = fma(prevl, dpb[(t + 31) & 31], w);
        prevl = lt;
        wrow[t] = w;
      }
    }
    for (int j = 0; j < f1; ++j) {
      const double* __restrict__ lj = Lraw + (32 + j) * 33;
      double acc = 0.0;
#pragma unroll
      for (int t = 0; t < 32; ++t) acc = fma(wrow[t], lj[t], acc);     // (entries t >= k of wrow are zero)
      if (j <= lane && lane < f1) cbo[(32 - k + lane) + (size_t)(32 - k + j) * r] = C22[lane + j * 33] - acc;
    }
  }
  fs.done();
}

// --------------------------------------------------------------------------------------------
// Class L (big fronts), global-memory blocked path.
// --------------------------------------------------------------------------------------------
__global__ void k_big_zero(DevSym S, DevNum N, const int* __restrict__ front_list) {
  const int s = front_list[blockIdx.y];
  const long long k = S.sn_start[s + 1] - S.sn_start[s];
  const long long r = S.rows_ptr[s + 1] - S.rows_ptr[s];
  const long long f = k + r, nl = f * k, nc = r * r;
  double* P = N.L + S.L_off[s];
  double* C = N.CB + S.cb_off[s];
  for (long long t = blockIdx.x * (long long)blockDim.x + threadIdx.x; t < nl + nc;
       t += (long long)gridDim.x * blockDim.x) {
    if (t < nl) P[t] = 0.0; else C[t - nl] = 0.0;
  }
}

__global__ void k_big_assemble(DevSym S, DevNum N, const int* __restrict__ front_list) {
  const int s = front_list[blockIdx.y];
  double* P = N.L + S.L_off[s];
  for (long long uu = S.uent_ptr[s] + blockIdx.x * (long long)blockDim.x + threadIdx.x;
       uu < S.uent_ptr[s + 1]; uu += (long long)gridDim.x * blockDim.x)
    P[S.u_dst64[uu]] = N.uval[uu];
}

// extend-add of ALL children of every big front in the list in one launch: each WARP owns one column of the parent
// front and applies the children one after the other (fixed order => deterministic, no atomics; no two warps touch
// the same parent entry).  The child column that lands in the warp's parent column comes from the inverse row map
// einv built at analysis; per-child metadata is fetched lane-parallel (one child per lane) and broadcast.
__global__ void __launch_bounds__(256) k_big_extend_all(DevSym S, DevNum N, const int* __restrict__ front_list) {
  const int p = front_list[blockIdx.y];
  const int c0p = S.sn_start[p];
  const int kp = S.sn_start[p + 1] - c0p;
  const int rp = (int)(S.rows_ptr[p + 1] - S.rows_ptr[p]);
  const int fp = kp + rp;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int lj = blockIdx.x * 8 + warp;
  if (lj >= fp) return;
  unsigned long long ts[2];
  const bool tlog = N.flog != nullptr && threadIdx.x == 0 && (blockIdx.x == 0 || (blockIdx.x + 1) * 8 >= fp);
  if (tlog) ts[0] = flog_now();
  // destination column indexed by the parent row li >= lj
  double* __restrict__ dst = (lj < kp) ? N.L + S.L_off[p] + (size_t)lj * fp
                                       : N.CB + S.cb_off[p] + (size_t)(lj - kp) * rp - kp;
  const int ch0 = S.child_ptr[p], nch = S.child_ptr[p + 1] - ch0;
  for (int q0 = 0; q0 < nch; q0 += 32) {
    int jj = -1, rc = 0;
    long long ro = 0, co = 0;
    if (q0 + lane < nch) {
      const int c = S.child_idx[ch0 + q0 + lane];
      ro = S.rows_ptr[c];
      rc = (int)(S.rows_ptr[c + 1] - ro);
      co = S.cb_off[c];
      jj = S.einv[S.einv_off[c] + lj];
    }
    unsigned has = __ballot_sync(0xffffffffu, jj >= 0);
    while (has) {
      const int src = __ffs(has) - 1;
      has &= has - 1;
      const int jq = __shfl_sync(0xffffffffu, jj, src), rq = __shfl_sync(0xffffffffu, rc, src);
      const long long roq = __shfl_sync(0xffffffffu, ro, src), coq = __shfl_sync(0xffffffffu, co, src);
      const double* __restrict__ cbcol = N.CB + coq + (size_t)jq * rq;
      const int* __restrict__ rl = S.rel + roq;
      // four independent gather / add / scatter groups in flight (the rows of one child column are distinct)
      int ii = jq + lane;
      for (; ii + 96 < rq; ii += 128) {
        const int r0 = rl[ii], r1 = rl[ii + 32], r2 = rl[ii + 64], r3 = rl[ii + 96];
        const double v0 = cbcol[ii], v1 = cbcol[ii + 32], v2 = cbcol[ii + 64], v3 = cbcol[ii + 96];
        const double d0 = dst[r0], d1 = dst[r1], d2 = dst[r2], d3 = dst[r3];
        dst[r0] = d0 + v0; dst[r1] = d1 + v1; dst[r2] = d2 + v2; dst[r3] = d3 + v3;
      }
      for (; ii < rq; ii += 32) dst[rl[ii]] += cbcol[ii];
      __syncwarp();   // the next child may add to the same parent entries from other lanes
    }
  }
  // the column is final now: max |entry| below its 32x32 diagonal block for the first three panels (the threshold test of
  // the first chain steps; later panels get theirs from k_big_update)
  if (lj < min(3 * NB, kp)) {
    const int below = (lj / NB + 1) * NB;
    double m = 0.0;
    for (int i = below + lane; i < fp; i += 32) m = fmax(m, fabs(dst[i]));
    m = warp_max(m);
    if (lane == 0) N.colmax[c0p + lj] = m;
  }
  if (tlog) { ts[1] = flog_now(); flog_put(N, 7, p, 0, ts, 2); }
}

// column maxima of the first panel below its diagonal block (later panels get theirs from k_big_update)
__global__ void k_big_colmax0(DevSym S, DevNum N, const int* __restrict__ front_list) {
  const int s = front_list[blockIdx.x];
  const int c0 = S.sn_start[s], k = S.sn_start[s + 1] - c0;
  const int f = k + (int)(S.rows_ptr[s + 1] - S.rows_ptr[s]);
  const int nb = min(3 * NB, k);   // panels 0, 1 and 2 (a later panel's values lack the earlier panels' updates: a stale estimate)
  const double* __restrict__ P = N.L + S.L_off[s];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarp = blockDim.x >> 5;
  for (int j = blockIdx.y * nwarp + warp; j < nb; j += gridDim.y * nwarp) {   // one column per warp, 8 CTAs per front
    const int below = (j / NB + 1) * NB;
    double m = 0.0;
    for (int i = below + lane; i < f; i += 32) m = fmax(m, fabs(P[i + (size_t)j * f]));
    m = warp_max(m);
    if (lane == 0) N.colmax[c0 + j] = m;
  }
}

// Reciprocal on the pivot chain: MUFU.RCP64H seed (>= 20 bits) + one cubically convergent correction = 3 dependent FMAs
// instead of the 5 (+ range checks) of the correctly rounded 1.0 / d; the result is within ~1 ulp.  d must be a normal number.
__device__ __forceinline__ double fast_rcp(const double d) {
  double r;
  asm("rcp.approx.ftz.f64 %0, %1;" : "=d"(r) : "d"(d));
  double e = fma(-d, r, 1.0);
  e = fma(e, e, e);
  return fma(r, e, r);
}

// --------------------------------------------------------------------------------------------
// cta_ldlt32s: pivoted LDL^T of a symmetric block of order f <= 32 (all f columns are candidates) by FOUR warps -- the
// diagonal blocks of the big fronts are the serial chain of the factorisation, so what counts is the latency of ONE pivot
// step.  Same pivoting rules as warp_ldlt32 (Bunch-Kaufman 1x1 / 2x2 with the threshold test against the whole front
// column, failed columns retried after the others, forced pivots at the end), organised as follows:
//   * the block lives in shared memory As[c * 33 + i] = A[i][c] (full symmetric storage) NEXT to the owners' registers
//     (warp w: columns 8w..8w+7, lane = row): after every update the owners store their live columns back, so any
//     column -- the candidate AND a 2x2 partner -- is one conflict-free shared-memory read away: ONE barrier per pivot
//     step, no publishing, no register select;
//   * a 1x1 pivot is first tried against the float-rounded-UP column maximum (one redux, no arg-max, no exact re-read):
//     that test is conservative, so whenever it passes the exact test passes too;
//   * candidates are taken in index order from a bit mask (parked columns wait for the next pass) -- all bookkeeping is
//     warp-uniform integer work.
// Output as warp_ldlt32: Lraw[i*33 + t] (must not alias As), order[t], pt[t], dinv_s[t], doff_s[t] (written by warp 0).
// All 128 threads must call this.
// gext_s: 32 doubles of shared memory holding max |entry| of column c in rows OUTSIDE the block.
// --------------------------------------------------------------------------------------------
__device__ void cta_ldlt32s(double (&a)[8], const int f, const double u, const double tiny,
                            double* __restrict__ As, double* __restrict__ Lraw, int* __restrict__ order, int* __restrict__ pt,
                            double* __restrict__ dinv_s, double* __restrict__ doff_s, const double* __restrict__ gext_s,
                            int* counters, unsigned long long* prof = nullptr /* debug: [0] fast steps<<40|cycles, [1] other steps<<40|cycles */) {
  unsigned long long pf_fast = 0, pf_slow = 0; long long pf_t0 = 0; bool pf_pending = false;
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  unsigned cand = (f >= 32) ? 0xffffffffu : ((1u << f) - 1u);
  unsigned parked = 0;
  int t = 0, progress = 0;
  bool forced = false;
  int c_neg = 0, c_forced = 0, c_tiny = 0, c_2x2 = 0;
  int my_order = 0, my_pt = 1;
  double my_dinv = 0.0, my_doff = 0.0;
  const unsigned lbit = 1u << lane;
  // The pivot TESTS run in float arithmetic first, with every rounding on the safe side (a double-precision operation has
  // ~10x the latency of a float one on this part, and a step is a chain of dependent operations): a float test can PROVE an
  // inequality of the exact test true or false; whenever it cannot, the exact double-precision sequence decides.
  const float tiny_up = __double2float_ru(tiny), u_up = __double2float_ru(u);
  const float alpha_up = __double2float_ru(BK_ALPHA), alpha_dn = __double2float_rd(BK_ALPHA);
  // 1x1 pivot: pivot column values pc (lane = row), pivot dd with reciprocal rinv, column g, pr[q] = A[8w+q][g]
  auto apply1 = [&](const double pc, const double dd, const double rinv, const int g, const double (&pr)[8]) {
    const double l = ((cand & lbit) && lane != g) ? pc * rinv : 0.0;
    cand &= ~(1u << g);
#pragma unroll
    for (int q = 0; q < 8; ++q) a[q] = fma(-l, pr[q], a[q]);
#pragma unroll
    for (int q = 0; q < 8; ++q)
      if ((cand >> (8 * w + q)) & 1u) As[(8 * w + q) * 33 + lane] = a[q];
    if (w == 0) {
      Lraw[lane * 33 + t] = l;
      if (lane == t) { my_order = g; my_pt = 1; my_dinv = rinv; my_doff = 0.0; }
    }
    if (dd < 0.0) ++c_neg;
    t += 1;
    ++progress;
  };
  while (cand != 0u) {
    unsigned avail = cand & ~parked;
    if (avail == 0u) {
      if (progress > 0) progress = 0; else forced = true;
      parked = 0u;
      avail = cand;
    }
    const int g0 = __ffs(avail) - 1;
    if (prof) {
      const long long now = clock64();
      if (pf_pending) pf_slow += (1ull << 40) + (unsigned long long)(now - pf_t0);
      pf_t0 = now; pf_pending = true;
    }
    __syncthreads();                                   // the previous step's column stores are visible
    const double* __restrict__ cA = As + g0 * 33;
    // everything a 1x1 pivot on g0 needs is loaded (and its reciprocal started) before the search
    const double a0 = cA[lane];                        // A[lane][g0]
    const double pa0 = cA[g0];
    const double gam = gext_s[g0];
    double pr0[8];
#pragma unroll
    for (int q = 0; q < 8; ++q) pr0[q] = cA[8 * w + q];   // A[8w+q][g0]
    const bool me_cand = (cand & lbit) != 0u;
    const float v0f = __double2float_ru(fabs(a0));
    const float lam_in = (me_cand && lane != g0) ? v0f : -1.0f;
    const float lamf = wredux_max(lam_in);             // >= the exact maximum lam
    const double rinv0 = fast_rcp(pa0);                // (issued behind the reduction: the two latencies overlap)
    const double ajj = fabs(pa0);
    const float ajj_dn = __double2float_rd(ajj), ajj_up = __double2float_ru(ajj);
    const float gam_up = __double2float_ru(gam), lam_up = fmaxf(lamf, 0.0f);
    if (!forced && ajj_dn > tiny_up && ajj_dn >= __fmul_ru(u_up, fmaxf(lam_up, gam_up)) && ajj_dn >= __fmul_ru(alpha_up, lam_up)) {
      apply1(a0, pa0, rinv0, g0, pr0);                 // proven: |pivot| > tiny, >= u * column max, >= alpha * lam
      if (prof) { pf_fast += (1ull << 40) + (unsigned long long)(clock64() - pf_t0); pf_pending = false; }
      continue;
    }
    int r = -1;
    if (lamf >= 0.0f) r = __ffs(__ballot_sync(0xffffffffu, lam_in == lamf)) - 1;
    const float lam_lo = (lamf > 0.0f) ? nextafterf(lamf, 0.0f) : 0.0f;      // lam > lam_lo (lamf is lam rounded up)
    // can the exact 1x1 test (ajj >= alpha * lam) still pass?  proven impossible when ajj_up < alpha_dn * lam_lo
    const bool no_1x1 = !forced && r >= 0 && lam_lo > 0.0f && ajj_up < __fmul_rd(alpha_dn, lam_lo);
    double lam = 0.0;
    bool ok1 = false;
    if (!no_1x1) {
      if (r >= 0) lam = fabs(cA[r]);                   // exact magnitude of the selected entry
      ok1 = (ajj > tiny) && (ajj >= u * fmax(lam, gam));
      const double colmax_f = fmax(lam, gam);
      if (forced) {
        double dd = pa0;
        const bool noise = !(fmax(ajj, colmax_f) > 1e-12);
        if (noise || !(fabs(dd) > tiny)) { dd = (dd < 0.0) ? -1.5e-8 : 1.5e-8; ++c_tiny; }
        else { dd = copysign(fmax(fabs(dd), 1e-8 * colmax_f), dd); ++c_forced; }
        apply1(a0, dd, 1.0 / dd, g0, pr0);
        continue;
      }
      if (lam == 0.0 || r < 0) {
        if (ok1) apply1(a0, pa0, rinv0, g0, pr0);
        else parked |= 1u << g0;
        continue;
      }
      if (ok1 && ajj >= BK_ALPHA * lam) { apply1(a0, pa0, rinv0, g0, pr0); continue; }
    }
    // ---- second column: the arg-max partner r ----
    const double* __restrict__ cB = As + r * 33;
    const double a1 = cB[lane];                        // A[lane][r]
    const double crr = cB[r];
    const double ge_r = gext_s[r];
    const double pb = cA[r];                           // A[r][g0]  (|pb| = lam)
    double pr1[8];
#pragma unroll
    for (int q = 0; q < 8; ++q) pr1[q] = cB[8 * w + q];   // A[8w+q][r]
    const double det = pa0 * crr - pb * pb, adet = fabs(det);
    const double idet = fast_rcp(det);                 // (started before the tests that decide whether it is used)
    const double n1 = crr * a0 - pb * a1, n2 = pa0 * a1 - pb * a0;   // numerators of the two multipliers
    const float v1f = __double2float_ru(fabs(a1));
    const bool other = me_cand && lane != g0 && lane != r;
    const float sigf = wredux_max((me_cand && lane != r) ? v1f : 0.0f);
    const float cjf = fmaxf(wredux_max(other ? v0f : 0.0f), gam_up);
    const float crf = fmaxf(wredux_max(other ? v1f : 0.0f), __double2float_ru(ge_r));
    const double arr = fabs(crr);
    bool take22 = false;
    {
      // float proof of the common outcome: the two 1x1 alternatives of the 2x2 branch fail and the 2x2 threshold test passes
      const float arr_up = __double2float_ru(arr), pb_up = __double2float_ru(fabs(pb)), adet_dn = __double2float_rd(adet);
      const float sig_lo = (sigf > 0.0f) ? nextafterf(sigf, 0.0f) : 0.0f;
      const bool sig_fails = no_1x1 ? (__fmul_ru(ajj_up, sigf) < __fmul_rd(alpha_dn, __fmul_rd(lam_lo, lam_lo))) : false;
      const bool r_fails = arr_up < __fmul_rd(alpha_dn, sig_lo) || arr_up <= 0.0f;
      const float lhs1 = __fmul_ru(__fmaf_ru(arr_up, cjf, __fmul_ru(pb_up, crf)), u_up);
      const float lhs2 = __fmul_ru(__fmaf_ru(ajj_up, crf, __fmul_ru(pb_up, cjf)), u_up);
      take22 = sig_fails && r_fails && lam_lo > tiny_up && adet_dn > 0.0f && isfinite(adet) && lhs1 <= adet_dn && lhs2 <= adet_dn;
    }
    if (!take22) {
      // exact sequence (identical decisions; reached when a float bound was inconclusive)
      if (no_1x1) { lam = fabs(pb); ok1 = (ajj > tiny) && (ajj >= u * fmax(lam, gam)); }
      const double sig = (double)sigf;
      const double cjm = (double)cjf, cr = (double)crf;
      // Of the two columns read in this step one stays alive when the pivot is 1x1 (on g0 or on r) and is then rewritten
      // by its owner: in those two branches every warp must have finished reading before any store.
      if (ok1 && ajj * sig >= BK_ALPHA * lam * lam) { __syncthreads(); apply1(a0, pa0, rinv0, g0, pr0); continue; }
      if (arr > tiny && arr >= BK_ALPHA * sig && arr >= u * fmax(sig, ge_r)) { __syncthreads(); apply1(a1, crr, 1.0 / crr, r, pr1); continue; }   // 1x1 on r
      take22 = lam > tiny && adet > 0.0 && isfinite(adet) &&
               (arr * cjm + fabs(pb) * cr) * u <= adet && (ajj * cr + fabs(pb) * cjm) * u <= adet;
    }
    if (take22) {
      const double l1 = other ? n1 * idet : 0.0;
      const double l2 = other ? n2 * idet : 0.0;
      cand &= ~((1u << g0) | (1u << r));
#pragma unroll
      for (int q = 0; q < 8; ++q) a[q] = fma(-l2, pr1[q], fma(-l1, pr0[q], a[q]));
#pragma unroll
      for (int q = 0; q < 8; ++q)
        if ((cand >> (8 * w + q)) & 1u) As[(8 * w + q) * 33 + lane] = a[q];
      if (w == 0) {
        Lraw[lane * 33 + t] = l1;
        Lraw[lane * 33 + t + 1] = l2;
        if (lane == t) { my_order = g0; my_pt = 2; my_dinv = crr * idet; my_doff = -pb * idet; }
        if (lane == t + 1) { my_order = r; my_pt = 3; my_dinv = pa0 * idet; my_doff = 0.0; }
      }
      ++c_2x2;
      if (det < 0.0) c_neg += 1; else if (pa0 < 0.0) c_neg += 2;
      t += 2;
      ++progress;
      continue;
    }
    parked |= 1u << g0;                                // nothing acceptable now: retry after the other candidates
  }
  if (prof) {
    if (pf_pending) pf_slow += (1ull << 40) + (unsigned long long)(clock64() - pf_t0);
    prof[0] = pf_fast; prof[1] = pf_slow;
  }
  if (w == 0) {
    if (lane < f) { order[lane] = my_order; pt[lane] = my_pt; dinv_s[lane] = my_dinv; doff_s[lane] = my_doff; }
    if (lane == 0) {
      if (c_neg) atomicAdd(counters + CNT_NEG, c_neg);
      if (c_forced) atomicAdd(counters + CNT_FORCED, c_forced);
      if (c_tiny) atomicAdd(counters + CNT_TINY, c_tiny);
      if (c_2x2) atomicAdd(counters + CNT_2X2, c_2x2);
    }
  }
  __syncthreads();
}

// --------------------------------------------------------------------------------------------
// THE CHAIN ROLE of the big-front panel pipeline (CTA 0 of k_big_panel): everything on the critical path of one panel
// step.  Call p (jbp = first column of panel p, or -NB for the first call) produces the pivoted LDL^T of block p+1:
//   A. all operand tiles fetched with asynchronous copies (in flight together, zero-filled where masked);
//   B. (p >= 1) the rank-32 update of panel p-1 applied to the two tiles the chain owns: rows of block p+1 x columns of
//      panel p, and block (p+1, p+1).  Inputs: L / W rows of block p+1 at panel p-1 (rows role of the previous launch) and
//      W rows of block p at panel p-1 (chain role of the previous launch).  The bulk k_big_update(q) skips these tiles.
//   C. (p >= 0) the panel rows of block p+1:  X = A_perm L_bb(p)^-T (= L D),  L = X D^-1 (four warps, shuffles) -> L / W
//      for the bulk update; then this panel's rank-32 update of block (p+1, p+1).
//   D. pivoted LDL^T of block (p+1, p+1) by four warps (cta_ldlt32s).
// It needs the previous k_big_panel and the bulk k_big_update of panel p-2: the bulk stream always has a full chain step
// of slack, so the chain (one launch per 32 pivots) is never gated by the trailing updates.
// dynamic smem: 8 tiles of 32 x 33 doubles
// --------------------------------------------------------------------------------------------
#define CHAIN_TILE (NB * 33)
#define CHAIN_SMEM (8 * CHAIN_TILE * (int)sizeof(double))
// C[i][j] -= sum_t A[i][t] B[j][t] on 32 x 32 row-major tiles (ld 33), 2 x 4 entries per thread (128 threads: rows a, a+16;
// columns b + 8w).  LOWER: only the lower triangle is needed -- the quadrant rows < 16 x columns >= 16 is skipped.
template <bool LOWER>
__device__ __forceinline__ void chain_tile_update(double* __restrict__ C, const double* __restrict__ A, const double* __restrict__ B) {
  const int tid = threadIdx.x, a = tid & 15, b = tid >> 4;
  double acc0[4], acc1[4];
#pragma unroll
  for (int w = 0; w < 4; ++w) { acc0[w] = 0.0; acc1[w] = 0.0; }
#pragma unroll 8
  for (int t = 0; t < NB; ++t) {
    const double l0 = A[a * 33 + t], l1 = A[(a + 16) * 33 + t];
#pragma unroll
    for (int w = 0; w < 4; ++w) {
      const double wv = B[(b + 8 * w) * 33 + t];
      if (!LOWER || w < 2) acc0[w] = fma(l0, wv, acc0[w]);
      acc1[w] = fma(l1, wv, acc1[w]);
    }
  }
#pragma unroll
  for (int w = 0; w < 4; ++w) {
    const int jj = b + 8 * w;
    if (!LOWER || (w < 2 && jj <= a)) C[a * 33 + jj] -= acc0[w];
    if (!LOWER || jj <= a + 16) C[(a + 16) * 33 + jj] -= acc1[w];
  }
}

__device__ __forceinline__ void cp_async8(double* smem_dst, const double* gsrc, bool valid) {
  const unsigned d = (unsigned)__cvta_generic_to_shared(smem_dst);
  const int sz = valid ? 8 : 0;      // src-size 0: the 8 bytes are zero-filled
  asm volatile("cp.async.ca.shared.global [%0], [%1], 8, %2;" ::"r"(d), "l"(gsrc), "r"(sz) : "memory");
}

__device__ void chain_role(const DevSym& S, const DevNum& N, const int s, const int jbp, double* __restrict__ csm) {
  __shared__ double gext_s[NB];
  __shared__ double dinv_s[NB], doff_s[NB];
  __shared__ int order[NB], pt[NB];
  __shared__ double di[NB], dup[NB], dlo[NB];
  __shared__ int bp[NB];
  double* A1 = csm;                    // rows of the new block x columns of panel p
  double* A2 = csm + CHAIN_TILE;       // the new diagonal block (lower part), then the symmetric working copy of cta_ldlt32s
  double* Lr = csm + 2 * CHAIN_TILE;   // L rows of the new block at panel p-1
  double* WrN = csm + 3 * CHAIN_TILE;  // W rows of the new block at panel p-1
  double* WrP = csm + 4 * CHAIN_TILE;  // W rows of block p at panel p-1
  double* Lbb = csm + 5 * CHAIN_TILE;  // L_bb(p), pivot order, strictly lower
  double* Ln = csm + 6 * CHAIN_TILE;   // L rows of the new block at panel p (computed here)
  double* Wn = csm + 7 * CHAIN_TILE;   // W rows of the new block at panel p (computed here)
  const int c0 = S.sn_start[s], k = S.sn_start[s + 1] - c0;
  const int o = jbp + NB;              // first column of the block to factor
  if (o >= k) return;
  const int f = k + (int)(S.rows_ptr[s + 1] - S.rows_ptr[s]);
  const int nbn = min(NB, k - o);
  const bool has_p = jbp >= 0, has_pp = jbp >= NB;
  const int jbq = jbp - NB;
  double* __restrict__ P = N.L + S.L_off[s];
  double* __restrict__ Wp = N.W + S.L_off[s];
  const int tid = threadIdx.x, lane = tid & 31, w = tid >> 5;
  unsigned long long ts[8];
  const bool tlog = N.flog != nullptr && tid == 0;
  if (tlog) ts[0] = flog_now();
  // ---- all global loads in flight at once (asynchronous copies straight into the tiles, zero-filled where masked) ----
#pragma unroll
  for (int e8 = 0; e8 < 8; ++e8) {
    const int e = tid + 128 * e8, ii = e & 31, jj = e >> 5;     // consecutive threads -> consecutive rows (coalesced columns)
    const bool rin = ii < nbn;
    cp_async8(A2 + ii * 33 + jj, P + (o + ii) + (size_t)(o + jj) * f, rin && jj < nbn && ii >= jj);
    if (has_p) {
      cp_async8(A1 + ii * 33 + jj, P + (o + ii) + (size_t)(jbp + jj) * f, rin);
      cp_async8(Lbb + ii * 33 + jj, P + (jbp + ii) + (size_t)(jbp + jj) * f, ii > jj);
    }
    if (has_pp) {
      cp_async8(Lr + ii * 33 + jj, P + (o + ii) + (size_t)(jbq + jj) * f, rin);
      cp_async8(WrN + ii * 33 + jj, Wp + (o + ii) + (size_t)(jbq + jj) * f, rin);
      cp_async8(WrP + ii * 33 + jj, Wp + (jbp + ii) + (size_t)(jbq + jj) * f, true);
    }
  }
  asm volatile("cp.async.commit_group;" ::: "memory");
  if (has_p && tid < NB) {
    const double d = N.dinv[c0 + jbp + tid], od = N.doff[c0 + jbp + tid];
    const int ty = N.ptype[c0 + jbp + tid];
    double om = 0.0; int tym = 1;
    if (tid > 0) { om = N.doff[c0 + jbp + tid - 1]; tym = N.ptype[c0 + jbp + tid - 1]; }
    di[tid] = d;
    dup[tid] = (ty == 2) ? od : 0.0;                      // first column of a 2x2 pivot: + x[t+1] * offdiag
    dlo[tid] = (ty == 3 && tym == 2) ? om : 0.0;           // second column:              + x[t-1] * offdiag
    bp[tid] = N.bperm[c0 + jbp + tid];
  }
  const double gext = (lane < nbn) ? N.colmax[c0 + o + lane] : 0.0;
  asm volatile("cp.async.wait_group 0;" ::: "memory");
  __syncthreads();
  if (tlog) ts[1] = flog_now();
  if (has_pp) {
    // B. panel p-1's update of the two tiles (independent of each other: no barrier in between)
    chain_tile_update<false>(A1, Lr, WrP);
    chain_tile_update<true>(A2, Lr, WrN);
    __syncthreads();
  }
  if (tlog) ts[2] = flog_now();
  if (has_p) {
    // C. rows of the new block at panel p: X = A_perm L_bb^-T (= L D), L = X D^-1.  Warp w solves rows 8w..8w+7; lane q
    // holds entry q of each row and row q of L_bb, the pivot entry x[t] travels by shuffle (31 steps of 8 independent
    // shuffle + FMA pairs).
    double lq[NB];
#pragma unroll
    for (int t = 0; t < NB; ++t) lq[t] = Lbb[lane * 33 + t];     // strictly lower: lq[t] = 0 for t >= lane
    double x[8];
    const int bpl = bp[lane];
#pragma unroll
    for (int i = 0; i < 8; ++i) x[i] = A1[(8 * w + i) * 33 + bpl];
#pragma unroll
    for (int t = 0; t < NB - 1; ++t) {
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        const double xt = __shfl_sync(0xffffffffu, x[i], t);
        x[i] = fma(-xt, lq[t], x[i]);                            // (lq[t] = 0 leaves the finished entries alone)
      }
    }
    const double dq = di[lane], duq = dup[lane], dlq = dlo[lane];
    const double lim = 1.0 / N.u;
    double lmax = 0.0;
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const double xn = __shfl_down_sync(0xffffffffu, x[i], 1), xp = __shfl_up_sync(0xffffffffu, x[i], 1);
      double v = x[i] * dq;
      v = fma(xn, duq, v);             // (dup = 0 in the last column, dlo = 0 in the first: the wrapped lanes do not count)
      v = fma(xp, dlq, v);
      if (8 * w + i < nbn) lmax = fmax(lmax, fabs(v));
      Ln[(8 * w + i) * 33 + lane] = v;
      Wn[(8 * w + i) * 33 + lane] = x[i];
    }
    if (lmax > lim) atomicAdd(N.counters + CNT_GROWTH, 1);
    __syncthreads();
    chain_tile_update<true>(A2, Ln, Wn);      // this panel's update of the new diagonal block
    // the new rows go to L / W for the bulk update (coalesced: consecutive threads -> consecutive rows of a column)
#pragma unroll
    for (int e8 = 0; e8 < 8; ++e8) {
      const int e = tid + 128 * e8, ii = e & 31, jj = e >> 5;
      if (ii < nbn) {
        P[(o + ii) + (size_t)(jbp + jj) * f] = Ln[ii * 33 + jj];
        Wp[(o + ii) + (size_t)(jbp + jj) * f] = Wn[ii * 33 + jj];
      }
    }
    __syncthreads();
  }
  // D. pivoted LDL^T of the new diagonal block
  if (tlog) ts[3] = flog_now();
  double a[8];
#pragma unroll
  for (int q = 0; q < 8; ++q) { const int c = 8 * w + q; a[q] = (c <= lane) ? A2[lane * 33 + c] : A2[c * 33 + lane]; }
  if (w == 0) gext_s[lane] = gext;
  __syncthreads();   // A2 becomes the full symmetric working copy of cta_ldlt32s: A2[c * 33 + i] = A[i][c]
#pragma unroll
  for (int q = 0; q < 8; ++q) A2[(8 * w + q) * 33 + lane] = a[q];
  __shared__ unsigned long long prof_s[2];
  cta_ldlt32s(a, nbn, N.u, N.tiny, A2, Ln, order, pt, dinv_s, doff_s, gext_s, N.counters, tlog ? prof_s : nullptr);
  if (tlog) ts[4] = flog_now();
  const int mine = (lane < nbn) ? order[lane] : 0;
#pragma unroll
  for (int q = 0; q < 8; ++q) {
    const int j = 8 * w + q;
    if (j < nbn && lane < nbn) {
      double v;
      if (lane < j) v = 0.0;
      else if (lane == j) v = 1.0;
      else v = Ln[mine * 33 + j];
      P[(o + lane) + (size_t)(o + j) * f] = v;
    }
  }
  if (w == 0 && lane < nbn) {
    N.bperm[c0 + o + lane] = mine;
    N.lperm[c0 + o + lane] = o + mine;
    N.dinv[c0 + o + lane] = dinv_s[lane];
    N.doff[c0 + o + lane] = doff_s[lane];
    N.ptype[c0 + o + lane] = pt[lane];
  }
  if (tlog) { ts[5] = flog_now(); ts[6] = prof_s[0]; ts[7] = prof_s[1]; flog_put(N, 1, s, jbp, ts, 8); }
}

// --------------------------------------------------------------------------------------------
// ONE launch per panel of the big fronts: k_big_panel(p), jb = first column of panel p.  Three CTA roles:
//   blockIdx.x == 0               the chain role (chain_role above): LDL^T of diagonal block p+1
//   1 .. nrowblk                  the rows below block p+1 (one row per thread), LEFT-LOOKING by one panel:
//                                   a   = A[i, panel p] - L[i, panel p-1] * W[block p, panel p-1]^T     (the update of panel p-1)
//                                   W   = a_perm * L_bb(p)^-T  (= L*D),   L = W * D^-1
//                                 (right-looking triangular solve: x[q] -= x[t] L[q][t] for all q > t, independent FMAs)
//   > nrowblk                     row interchanges of block p applied to the L columns on the left: one WARP per column
//                                 (the 32 rows of a column are one 256-byte segment; the permutation is a warp shuffle)
// All roles depend on the same two things -- the previous k_big_panel and the bulk update of panel p-2 -- and not on each
// other, so the critical path of a front is ONE kernel per 32 pivots; the bulk rank-32 update (k_big_update) of a panel
// has a whole chain step to complete.  k_big_panel(-NB) (chain role only) factors block 0.
// --------------------------------------------------------------------------------------------
#define TRSM_LD 34          // even leading dimension: column t of the block starts 16-byte aligned
#define TRSM_SWAP_COLS 32   // columns per row-swap CTA (4 warps x 8)
__global__ void __launch_bounds__(128) k_big_panel(DevSym S, DevNum N, const int* __restrict__ front_list, int jb,
                                                   int nrowblk) {
  extern __shared__ double csm[];
  const int s = front_list[blockIdx.y];
  // Programmatic dependent launch (the launches of one front's panels follow each other on the chain stream): let the next
  // panel's CTAs become resident now, and wait here until the previous panel kernel has completed and flushed.  Both are
  // no-ops when the kernel was launched without the attribute.
  asm volatile("griddepcontrol.launch_dependents;");
  asm volatile("griddepcontrol.wait;" ::: "memory");
  if (blockIdx.x == 0) { chain_role(S, N, s, jb, csm); return; }
  if (jb < 0) return;
  __shared__ __align__(16) double Lb[NB * TRSM_LD];
  __shared__ __align__(16) double Wb[NB * TRSM_LD];   // Wb[t' * LD + t] = W[jb + bperm[t]][jbq + t']
  __shared__ double di[NB], dup[NB], dlo[NB];
  __shared__ int bp[NB];
  const int bx = (int)blockIdx.x - 1;
  const int c0 = S.sn_start[s], k = S.sn_start[s + 1] - c0;
  if (jb >= k) return;
  const int f = k + (int)(S.rows_ptr[s + 1] - S.rows_ptr[s]);
  const int nb = min(NB, k - jb);
  const int row0 = jb + nb;
  double* P = N.L + S.L_off[s];
  const int tid = threadIdx.x;
  const int nxt = max(0, min(NB, k - row0));   // rows of the next diagonal block: the chain role's
  if (bx >= nrowblk) {
    // ---- left part: rows jb..jb+nb of columns [0, jb) get the block permutation ----
    const int lane = tid & 31, warp = tid >> 5;
    const int cbeg = (bx - nrowblk) * TRSM_SWAP_COLS;
    if (cbeg >= jb) return;
    const int src = (lane < nb) ? N.bperm[c0 + jb + lane] : lane;
    double v[TRSM_SWAP_COLS / 4];
#pragma unroll
    for (int q = 0; q < TRSM_SWAP_COLS / 4; ++q) {
      const int c = cbeg + warp + 4 * q;
      v[q] = (c < jb && lane < nb) ? P[(size_t)c * f + jb + lane] : 0.0;
    }
#pragma unroll
    for (int q = 0; q < TRSM_SWAP_COLS / 4; ++q) {
      const int c = cbeg + warp + 4 * q;
      const double w = __shfl_sync(0xffffffffu, v[q], src);
      if (c < jb && lane < nb) P[(size_t)c * f + jb + lane] = w;
    }
    return;
  }
  if ((long long)bx * blockDim.x >= f - row0 - nxt) return;
  double* Wp = N.W + S.L_off[s];
  const int i = row0 + nxt + bx * blockDim.x + tid;
  const bool active = i < f;
  const bool has_q = jb >= NB;                 // there is a panel p-1 whose update this kernel applies
  const int jbq = jb - NB;
  unsigned long long ts[2];
  const bool tlog = N.flog != nullptr && tid == 0 && (bx == 0 || (long long)(bx + 1) * blockDim.x >= f - row0 - nxt);
  if (tlog) ts[0] = flog_now();
  // issue all global loads up front: the diagonal block, its D, the W rows of this block at panel p-1 (permuted), and this
  // thread's rows (panel p-1: L; panel p: A, columns in pivot order)
  if (tid < NB) {
    double d = 0.0, o = 0.0, om = 0.0;
    int ty = 1, tym = 1, b = tid;
    if (tid < nb) {
      d = N.dinv[c0 + jb + tid]; o = N.doff[c0 + jb + tid]; ty = N.ptype[c0 + jb + tid]; b = N.bperm[c0 + jb + tid];
      if (tid > 0) { om = N.doff[c0 + jb + tid - 1]; tym = N.ptype[c0 + jb + tid - 1]; }
    }
    di[tid] = d;
    dup[tid] = (ty == 2) ? o : 0.0;                  // first column of a 2x2 pivot: + x[t+1] * offdiag
    dlo[tid] = (ty == 3 && tym == 2) ? om : 0.0;      // second column:              + x[t-1] * offdiag
    bp[tid] = b;
  }
  {
    double lb[NB * NB / 128];
#pragma unroll
    for (int q = 0; q < NB * NB / 128; ++q) {
      const int t = tid + 128 * q, ii = t & (NB - 1), jj = t / NB;
      lb[q] = (ii < nb && jj < nb && ii > jj) ? P[(jb + ii) + (size_t)(jb + jj) * f] : 0.0;
    }
#pragma unroll
    for (int q = 0; q < NB * NB / 128; ++q) {
      const int t = tid + 128 * q, ii = t & (NB - 1), jj = t / NB;
      Lb[ii + jj * TRSM_LD] = lb[q];
    }
  }
  __syncthreads();   // bp
  if (has_q) {
    double wb[NB * NB / 128];
#pragma unroll
    for (int q = 0; q < NB * NB / 128; ++q) {
      const int t = tid + 128 * q, ii = t & (NB - 1), jj = t / NB;     // ii = position in the block (pivot order), jj = t'
      wb[q] = (ii < nb) ? Wp[(jb + bp[ii]) + (size_t)(jbq + jj) * f] : 0.0;
    }
#pragma unroll
    for (int q = 0; q < NB * NB / 128; ++q) {
      const int t = tid + 128 * q, ii = t & (NB - 1), jj = t / NB;
      Wb[ii + jj * TRSM_LD] = wb[q];
    }
  }
  double x[NB];
#pragma unroll
  for (int t = 0; t < NB; ++t) x[t] = (active && t < nb) ? P[i + (size_t)(jb + bp[t]) * f] : 0.0;
  __syncthreads();
  if (has_q) {
    // the rank-32 update of panel p-1 on this row (fixed summation order t' = 0..31)
#pragma unroll
    for (int t8 = 0; t8 < NB; t8 += 8) {
      double lq[8];
#pragma unroll
      for (int u = 0; u < 8; ++u) lq[u] = active ? P[i + (size_t)(jbq + t8 + u) * f] : 0.0;
#pragma unroll
      for (int u = 0; u < 8; ++u) {
        const double* __restrict__ wr = Wb + (t8 + u) * TRSM_LD;
#pragma unroll
        for (int t = 0; t < NB; t += 2) {
          const double2 w2 = *reinterpret_cast<const double2*>(wr + t);
          x[t] = fma(-lq[u], w2.x, x[t]);
          x[t + 1] = fma(-lq[u], w2.y, x[t + 1]);
        }
      }
    }
  }
#pragma unroll
  for (int t = 0; t < NB - 1; ++t) {
    const double xt = x[t];
    const double* __restrict__ col = Lb + t * TRSM_LD;
    if (((t + 1) & 1) != 0) x[t + 1] = fma(-xt, col[t + 1], x[t + 1]);
#pragma unroll
    for (int q = (t + 2) & ~1; q < NB; q += 2) {
      const double2 l2 = *reinterpret_cast<const double2*>(col + q);
      x[q] = fma(-xt, l2.x, x[q]);
      x[q + 1] = fma(-xt, l2.y, x[q + 1]);
    }
  }
  const double lim = 1.0 / N.u;
  double lmax = 0.0;
  double l[NB];
#pragma unroll
  for (int t = 0; t < NB; ++t) {
    double v = x[t] * di[t];
    if (t + 1 < NB) v = fma(x[t + 1], dup[t], v);
    if (t > 0) v = fma(x[t - 1], dlo[t], v);
    l[t] = v;
    lmax = fmax(lmax, fabs(v));
  }
  if (active) {
#pragma unroll
    for (int t = 0; t < NB; ++t)
      if (t < nb) { Wp[i + (size_t)(jb + t) * f] = x[t]; P[i + (size_t)(jb + t) * f] = l[t]; }
  }
  if (active && lmax > lim) atomicAdd(N.counters + CNT_GROWTH, 1);
  if (tlog) { ts[1] = flog_now(); flog_put(N, 2, s, jb, ts, 2); }
}

#define TM 64
#define TK 16
// Bulk trailing update of panel jb (= panel p): C -= L_panel * W_panel^T (rank NB) on the pivot columns from panel p+2 on
// (the columns of panel p+1 get this update inside k_big_panel(p+1), left-looking), lower 64x64 tiles.  One k-step (the
// whole rank-32 slab of both operands in shared memory); the C tile is prefetched before the contraction so its latency
// overlaps the FMAs.  Skips diagonal block (p+2, p+2) (the chain role of k_big_panel(p+1) updates it) and records the
// column maxima of panel p+3 below its diagonal block for the threshold test of chain step p+2 (reduced per warp: one
// atomic per column and warp instead of one per entry).
__global__ void __launch_bounds__(256) k_big_update(DevSym S, DevNum N, const int* __restrict__ front_list, int jb) {
  __shared__ double As[NB][TM + 1];
  __shared__ double Bs[NB][TM + 1];
  const int s = front_list[blockIdx.z];
  const int c0 = S.sn_start[s], k = S.sn_start[s + 1] - c0;
  const int o = jb + 2 * NB;                  // first row / column of the region
  if (o >= k) return;
  const int r = (int)(S.rows_ptr[s + 1] - S.rows_ptr[s]);
  const int f = k + r;
  const int M = f - o, Nk = k - o;            // rows below; remaining pivot columns
  const int i0 = blockIdx.x * TM, j0 = blockIdx.y * TM;
  if (i0 >= M || j0 >= Nk || i0 + TM - 1 < j0) return;
  unsigned long long ts[2];
  const bool tlog = N.flog != nullptr && threadIdx.x == 0 && j0 == 0 && (i0 == 0 || i0 + TM >= M);
  if (tlog) ts[0] = flog_now();
  const long long ld = f;
  double* __restrict__ C = N.L + S.L_off[s] + o + (long long)o * ld;
  const double* __restrict__ A = N.L + S.L_off[s] + o + (long long)jb * ld;
  const double* __restrict__ Bm = N.W + S.L_off[s] + o + (long long)jb * ld;
  double* colmax_next = N.colmax + c0 + o;
  const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
  {
    double av[8], bv[8];
#pragma unroll
    for (int q = 0; q < 8; ++q) {
      const int t = tid + 256 * q, ii = t & (TM - 1), kk = t / TM;
      av[q] = (i0 + ii < M) ? A[i0 + ii + (long long)kk * ld] : 0.0;
      bv[q] = (j0 + ii < Nk) ? Bm[j0 + ii + (long long)kk * ld] : 0.0;
    }
#pragma unroll
    for (int q = 0; q < 8; ++q) {
      const int t = tid + 256 * q, ii = t & (TM - 1), kk = t / TM;
      As[kk][ii] = av[q]; Bs[kk][ii] = bv[q];
    }
  }
  double c[4][4];
#pragma unroll
  for (int q = 0; q < 4; ++q)
#pragma unroll
    for (int p = 0; p < 4; ++p) {
      const int gi = i0 + tx + 16 * q, gj = j0 + ty + 16 * p;
      c[q][p] = (gi < M && gj < Nk && gi >= gj) ? C[gi + (long long)gj * ld] : 0.0;
    }
  __syncthreads();
#pragma unroll 8
  for (int kk = 0; kk < NB; ++kk) {
    double a[4], b[4];
#pragma unroll
    for (int q = 0; q < 4; ++q) { a[q] = As[kk][tx + 16 * q]; b[q] = Bs[kk][ty + 16 * q]; }
#pragma unroll
    for (int q = 0; q < 4; ++q)
#pragma unroll
      for (int p = 0; p < 4; ++p) c[q][p] = fma(-a[q], b[p], c[q][p]);
  }
  const int lane = tid & 31;
#pragma unroll
  for (int p = 0; p < 4; ++p) {
    const int gj = j0 + ty + 16 * p;
    float m = 0.0f;
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const int gi = i0 + tx + 16 * q;
      if (gi < M && gj < Nk && gi >= gj) {
        if (gi < min(NB, Nk) && gj < NB) continue; // diagonal block (p+2, p+2): the chain role's
        C[gi + (long long)gj * ld] = c[q][p];
        if (gi >= 2 * NB) m = fmaxf(m, __double2float_ru(fabs(c[q][p])));
      }
    }
    // columns [NB, 2NB) of the region are diagonal block p+3: the chain runs up to two panels ahead of this update, so a
    // block's threshold maxima are the ones recorded two panels earlier
    if (j0 == 0 && p >= 2) {   // (warp-uniform)
      const float m_lo = wredux_max((lane < 16) ? m : 0.0f), m_hi = wredux_max((lane >= 16) ? m : 0.0f);
      if ((lane == 0 || lane == 16) && gj < Nk) {
        const float mm = (lane == 0) ? m_lo : m_hi;
        if (mm > 0.0f)
          atomicMax(reinterpret_cast<unsigned long long*>(colmax_next + gj), (unsigned long long)__double_as_longlong((double)mm));
      }
    }
  }
  if (tlog) { ts[1] = flog_now(); flog_put(N, 3, s, jb, ts, 2); }
}

// Contribution-block share of a panel's update: CB -= L21[:, panel] * W21[:, panel]^T (rank nb) on the lower 64x64 tiles of
// the r x r contribution block.  Issued once per panel behind k_big_panel on its own stream, so the Schur complement of a
// front is finished a few microseconds after its last panel instead of costing a GEMM at the end of the level (the chain
// is latency-bound and leaves the SMs idle).  Panels are applied in stream order => deterministic.
__global__ void __launch_bounds__(256) k_big_update_cb(DevSym S, DevNum N, const int* __restrict__ front_list, int jb) {
  __shared__ double As[NB][TM + 1];
  __shared__ double Bs[NB][TM + 1];
  const int s = front_list[blockIdx.z];
  const int c0 = S.sn_start[s], k = S.sn_start[s + 1] - c0;
  if (jb >= k) return;
  const int r = (int)(S.rows_ptr[s + 1] - S.rows_ptr[s]);
  const int i0 = blockIdx.x * TM, j0 = blockIdx.y * TM;
  if (i0 >= r || j0 >= r || i0 + TM - 1 < j0) return;
  const long long ld = k + r;
  const int nb = min(NB, k - jb);
  double* __restrict__ C = N.CB + S.cb_off[s];
  const double* __restrict__ A = N.L + S.L_off[s] + k + (long long)jb * ld;
  const double* __restrict__ Bm = N.W + S.L_off[s] + k + (long long)jb * ld;
  const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
  unsigned long long ts[2];
  const bool tlog = N.flog != nullptr && tid == 0 && j0 == 0 && (i0 == 0 || i0 + TM >= r);
  if (tlog) ts[0] = flog_now();
  {
    double av[8], bv[8];
#pragma unroll
    for (int q = 0; q < 8; ++q) {
      const int t = tid + 256 * q, ii = t & (TM - 1), kk = t / TM;
      av[q] = (i0 + ii < r && kk < nb) ? A[i0 + ii + (long long)kk * ld] : 0.0;
      bv[q] = (j0 + ii < r && kk < nb) ? Bm[j0 + ii + (long long)kk * ld] : 0.0;
    }
#pragma unroll
    for (int q = 0; q < 8; ++q) {
      const int t = tid + 256 * q, ii = t & (TM - 1), kk = t / TM;
      As[kk][ii] = av[q]; Bs[kk][ii] = bv[q];
    }
  }
  double c[4][4];
#pragma unroll
  for (int q = 0; q < 4; ++q)
#pragma unroll
    for (int p = 0; p < 4; ++p) {
      const int gi = i0 + tx + 16 * q, gj = j0 + ty + 16 * p;
      c[q][p] = (gi < r && gj < r && gi >= gj) ? C[gi + (long long)gj * r] : 0.0;
    }
  __syncthreads();
#pragma unroll 8
  for (int kk = 0; kk < NB; ++kk) {
    double a[4], b[4];
#pragma unroll
    for (int q = 0; q < 4; ++q) { a[q] = As[kk][tx + 16 * q]; b[q] = Bs[kk][ty + 16 * q]; }
#pragma unroll
    for (int q = 0; q < 4; ++q)
#pragma unroll
      for (int p = 0; p < 4; ++p) c[q][p] = fma(-a[q], b[p], c[q][p]);
  }
#pragma unroll
  for (int q = 0; q < 4; ++q)
#pragma unroll
    for (int p = 0; p < 4; ++p) {
      const int gi = i0 + tx + 16 * q, gj = j0 + ty + 16 * p;
      if (gi < r && gj < r && gi >= gj) C[gi + (long long)gj * r] = c[q][p];
    }
  if (tlog) { ts[1] = flog_now(); flog_put(N, 8, s, jb, ts, 2); }
}

// --------------------------------------------------------------------------------------------
// Schur complement with 8x4 register blocking: 64x64 tile per CTA of 128 threads (thread = rows tx+8q, columns
// ty+16p), 12 shared-memory loads per 32 FMAs (the 4x4 version needs 8 per 16 and is shared-memory bound),
// next k-slab prefetched into registers while the current one is consumed.
// --------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(128) k_big_schur84(DevSym S, DevNum N, const int* __restrict__ front_list) {
  __shared__ double As[TK][TM + 1];
  __shared__ double Bs[TK][TM + 1];
  const int s = front_list[blockIdx.z];
  const int k = S.sn_start[s + 1] - S.sn_start[s];
  const int r = (int)(S.rows_ptr[s + 1] - S.rows_ptr[s]);
  const long long f = k + r;
  const int i0 = blockIdx.x * TM, j0 = blockIdx.y * TM;
  if (i0 >= r || j0 >= r || i0 + TM - 1 < j0) return;
  unsigned long long ts[2];
  const bool tlog = N.flog != nullptr && threadIdx.x == 0 && j0 == 0 && (i0 == 0 || i0 + TM >= r);
  if (tlog) ts[0] = flog_now();
  double* __restrict__ C = N.CB + S.cb_off[s];
  const double* __restrict__ A = N.L + S.L_off[s] + k;
  const double* __restrict__ Bm = N.W + S.L_off[s] + k;
  const int tid = threadIdx.x, tx = tid & 7, ty = tid >> 3;
  const int li = tid & 63, lk = tid >> 6;   // loader: element (row li, k-index lk + 2q)
  double acc[8][4];
#pragma unroll
  for (int a = 0; a < 8; ++a)
#pragma unroll
    for (int b = 0; b < 4; ++b) acc[a][b] = 0.0;
  double av[8], bv[8];
  auto load = [&](int k0) {
#pragma unroll
    for (int q = 0; q < 8; ++q) {
      const long long gk = k0 + lk + 2 * q;
      av[q] = (i0 + li < r && gk < k) ? A[i0 + li + gk * f] : 0.0;
      bv[q] = (j0 + li < r && gk < k) ? Bm[j0 + li + gk * f] : 0.0;
    }
  };
  load(0);
  for (int k0 = 0; k0 < k; k0 += TK) {
#pragma unroll
    for (int q = 0; q < 8; ++q) { As[lk + 2 * q][li] = av[q]; Bs[lk + 2 * q][li] = bv[q]; }
    __syncthreads();
    if (k0 + TK < k) load(k0 + TK);
#pragma unroll
    for (int kk = 0; kk < TK; ++kk) {
      double a[8], b[4];
#pragma unroll
      for (int q = 0; q < 8; ++q) a[q] = As[kk][tx + 8 * q];
#pragma unroll
      for (int p2 = 0; p2 < 4; ++p2) b[p2] = Bs[kk][ty + 16 * p2];
#pragma unroll
      for (int q = 0; q < 8; ++q)
#pragma unroll
        for (int p2 = 0; p2 < 4; ++p2) acc[q][p2] = fma(a[q], b[p2], acc[q][p2]);
    }
    __syncthreads();
  }
#pragma unroll
  for (int q = 0; q < 8; ++q)
#pragma unroll
    for (int p2 = 0; p2 < 4; ++p2) {
      const int gi = i0 + tx + 8 * q, gj = j0 + ty + 16 * p2;
      if (gi < r && gj < r && gi >= gj) C[gi + (long long)gj * r] -= acc[q][p2];
    }
  if (tlog) { ts[1] = flog_now(); flog_put(N, 6, s, 0, ts, 2); }
}

}  // namespace b200
