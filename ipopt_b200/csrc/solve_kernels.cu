// Around the triangular solve (solve_dataflow.cu), sm_90a: permutation + scaling of the right-hand sides in and of the
// solutions out, and the residual helpers.
#include <cuda_runtime.h>
#include <math.h>

#include "kernels.cuh"

namespace b200 {

// xp[i] = scale[perm[i]] * b[perm[i]], column blockIdx.y (b: leading dimension n, xp: ldx)
__global__ void k_rhs_in(int n, const int* __restrict__ perm, const double* __restrict__ scale,
                         const double* __restrict__ b, double* __restrict__ xp, long long ldx) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  const long long c = blockIdx.y;
  if (i < n) { const int o = perm[i]; xp[c * ldx + i] = scale[o] * b[c * n + o]; }
}
// x[perm[i]] = scale[perm[i]] * xp[i], column blockIdx.y (x: leading dimension n, xp: ldx)
__global__ void k_sol_out(int n, const int* __restrict__ perm, const double* __restrict__ scale,
                          const double* __restrict__ xp, long long ldx, double* __restrict__ x) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  const long long c = blockIdx.y;
  if (i < n) { const int o = perm[i]; x[c * n + o] = scale[o] * xp[c * ldx + i]; }
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
