// Supernodal triangular-solve kernels (forward L, block-diagonal D^-1, backward L^T), sm_90a.
//
// Replaces the vendor back-solve the reference calls once per right-hand side
// (MUMPS job=3, reference src/Algorithm/LinearSolvers/IpMumpsSolverInterface.cpp:543-583).
// HBM-bound: every entry of L is streamed once per sweep.  Level-scheduled over the
// supernodal elimination tree; contributions travel child -> parent through per-front
// update vectors (gathered by the parent, so no atomics and bit-reproducible results).
#include <cuda_runtime.h>
#include <math.h>

#include "kernels.cuh"

namespace b200 {

#define SB 32  // block size of the in-front triangular solves

// xp[i] = scale[perm[i]] * b[perm[i]]
__global__ void k_rhs_in(int n, const int* __restrict__ perm, const double* __restrict__ scale,
                         const double* __restrict__ b, double* __restrict__ xp) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) { int o = perm[i]; xp[i] = scale[o] * b[o]; }
}
// x[perm[i]] = scale[perm[i]] * xp[i]
__global__ void k_sol_out(int n, const int* __restrict__ perm, const double* __restrict__ scale,
                          const double* __restrict__ xp, double* __restrict__ x) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) { int o = perm[i]; x[o] = scale[o] * xp[i]; }
}

// Forward sweep for the fronts of one level: one CTA per front.
// smem: v[f] | w[f]
__global__ void k_fwd_front(DevSym S, DevNum N, const int* __restrict__ front_list,
                            double* __restrict__ x, double* __restrict__ cbv) {
  extern __shared__ double sm[];
  const int s = front_list[blockIdx.x];
  const int c0 = S.sn_start[s], k = S.sn_start[s + 1] - c0;
  const int r = (int)(S.rows_ptr[s + 1] - S.rows_ptr[s]);
  const int f = k + r;
  double* v = sm;
  double* w = sm + f;
  const int tid = threadIdx.x, nt = blockDim.x, lane = tid & 31, warp = tid >> 5, nwarp = nt >> 5;
  for (int i = tid; i < f; i += nt) w[i] = (i < k) ? x[c0 + i] : 0.0;
  __syncthreads();
  for (int q = S.child_ptr[s]; q < S.child_ptr[s + 1]; ++q) {
    const int c = S.child_idx[q];
    const long long o = S.rows_ptr[c];
    const int rc = (int)(S.rows_ptr[c + 1] - o);
    for (int t = tid; t < rc; t += nt) w[S.rel[o + t]] += cbv[o + t];
    __syncthreads();
  }
  const int* __restrict__ lp = N.lperm + c0;
  for (int i = tid; i < f; i += nt) v[i] = (i < k) ? w[lp[i]] : w[i];
  __syncthreads();
  const double* __restrict__ P = N.L + S.L_off[s];
  __shared__ double Lb[SB * (SB + 1)];
  for (int t0 = 0; t0 < k; t0 += SB) {
    const int nb = min(SB, k - t0);
    // stage the diagonal block in shared memory (coalesced), then a warp solves it from there
    for (int t = tid; t < nb * nb; t += nt) {
      int i = t % nb, q = t / nb;
      Lb[i + q * (SB + 1)] = P[(t0 + i) + (size_t)(t0 + q) * f];
    }
    __syncthreads();
    if (warp == 0) {
      double yi = (lane < nb) ? v[t0 + lane] : 0.0;
      for (int q = 0; q < nb; ++q) {
        double yq = __shfl_sync(0xffffffffu, yi, q);
        if (lane > q && lane < nb) yi -= Lb[lane + q * (SB + 1)] * yq;
      }
      if (lane < nb) v[t0 + lane] = yi;
    }
    __syncthreads();
    // rows below the block: v[i] -= L[i, t0:t0+nb] * y
    for (int i = t0 + nb + tid; i < f; i += nt) {
      double acc = 0.0;
      for (int q = 0; q < nb; ++q) acc += P[i + (size_t)(t0 + q) * f] * v[t0 + q];
      v[i] -= acc;
    }
    __syncthreads();
  }
  // D^-1 and write-back (pivoted order in the front's own slots)
  for (int t = tid; t < k; t += nt) {
    const int ty = N.ptype[c0 + t];
    double y;
    if (ty == 1) y = v[t] * N.dinv[c0 + t];
    else if (ty == 2) y = v[t] * N.dinv[c0 + t] + v[t + 1] * N.doff[c0 + t];
    else y = v[t - 1] * N.doff[c0 + t - 1] + v[t] * N.dinv[c0 + t];
    x[c0 + t] = y;
  }
  double* __restrict__ out = cbv + S.rows_ptr[s];
  for (int i = tid; i < r; i += nt) out[i] = v[k + i];
}

// Backward sweep for the fronts of one level: one CTA per front.
// smem: v[f]
__global__ void k_bwd_front(DevSym S, DevNum N, const int* __restrict__ front_list,
                            double* __restrict__ x) {
  extern __shared__ double sm[];
  const int s = front_list[blockIdx.x];
  const int c0 = S.sn_start[s], k = S.sn_start[s + 1] - c0;
  const long long ro = S.rows_ptr[s];
  const int r = (int)(S.rows_ptr[s + 1] - ro);
  const int f = k + r;
  double* v = sm;
  const int tid = threadIdx.x, nt = blockDim.x, lane = tid & 31, warp = tid >> 5, nwarp = nt >> 5;
  for (int i = tid; i < f; i += nt) v[i] = (i < k) ? x[c0 + i] : x[S.rows[ro + (i - k)]];
  __syncthreads();
  const double* __restrict__ P = N.L + S.L_off[s];
  __shared__ double Lb[SB * (SB + 1)];
  const int nblk = (k + SB - 1) / SB;
  for (int b = nblk - 1; b >= 0; --b) {
    const int t0 = b * SB, nb = min(SB, k - t0);
    for (int t = tid; t < nb * nb; t += nt) {
      int i = t % nb, q = t / nb;
      Lb[i + q * (SB + 1)] = P[(t0 + i) + (size_t)(t0 + q) * f];
    }
    // v[t] -= sum_{i >= t0+nb} L[i,t] * v[i]   (one warp per column, coalesced down the column)
    for (int q = warp; q < nb; q += nwarp) {
      const double* col = P + (size_t)(t0 + q) * f;
      double acc = 0.0;
      for (int i = t0 + nb + lane; i < f; i += 32) acc += col[i] * v[i];
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
      if (lane == 0) v[t0 + q] -= acc;
    }
    __syncthreads();
    // diagonal block: solve L_bb^T z = v  (lane i owns row t0+i; go from the last row up)
    if (warp == 0) {
      double zi = (lane < nb) ? v[t0 + lane] : 0.0;
      for (int q = nb - 1; q >= 0; --q) {
        double zq = __shfl_sync(0xffffffffu, zi, q);
        if (lane < q) zi -= Lb[q + lane * (SB + 1)] * zq;
      }
      if (lane < nb) v[t0 + lane] = zi;
    }
    __syncthreads();
  }
  const int* __restrict__ lp = N.lperm + c0;
  for (int t = tid; t < k; t += nt) x[c0 + lp[t]] = v[t];
}

// r = b - A x from the original triplets (tests / bench parity helper)
__global__ void k_residual_init(int n, const double* __restrict__ b, double* __restrict__ r) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) r[i] = b[i];
}
__global__ void k_residual_acc(long long nnz, const int* __restrict__ irn, const int* __restrict__ jcn,
                               const double* __restrict__ a, const double* __restrict__ x,
                               double* __restrict__ r) {
  long long e = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (e >= nnz) return;
  int i = irn[e] - 1, j = jcn[e] - 1;
  double v = a[e];
  atomicAdd(r + i, -v * x[j]);
  if (i != j) atomicAdd(r + j, -v * x[i]);
}
__global__ void k_absmax(int n, const double* __restrict__ v, unsigned long long* out) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  double a = (i < n) ? fabs(v[i]) : 0.0;
  if (!(a == a)) a = INFINITY;  // NaN -> inf so it is visible
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) a = fmax(a, __shfl_xor_sync(0xffffffffu, a, o));
  if ((threadIdx.x & 31) == 0 && a > 0.0) atomicMax(out, (unsigned long long)__double_as_longlong(a));
}

}  // namespace b200
