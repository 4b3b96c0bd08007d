// FGMRES preconditioned by the factors (b200ldlt_solve_gmres), sm_90a: the Krylov layer of one Arnoldi step for the
// active columns of a block -- the product with the operator A_op, the two passes of classical Gram-Schmidt (multi-dot,
// then update), the norm and the normalisation -- and the final update x += Z y with x saved for a rollback.
//
// Every result is bit-reproducible and every order is the one include/b200ldlt.h states: a row of A_op z by the lane
// split and shuffle tree of k_ea_rows, and every dot product and squared norm over the fixed grid of ea_parts(n) CTAs
// (grid-stride, each thread in index order), a shuffle-xor tree in each warp, the warps in order and the CTAs' partials
// in order.  All arithmetic is explicit __dadd_rn / __dsub_rn / __dmul_rn / __ddiv_rn / __dsqrt_rn: nothing is fused.
#include <cuda_runtime.h>

#include "kernels.cuh"

namespace b200 {

#define GM_RESTART_MAX 64    // largest restart (Arnoldi steps per cycle)
#define GM_Q (GM_RESTART_MAX + 1)   // reductions per column and pass: the dots with v_0 .. v_63, then one norm (GM_Q - 1)
#define GM_H (2 * GM_Q)      // doubles per column of the Hessenberg buffer: the first pass's results, then the second's

// The slots of one launch: slot s = blockIdx.y works on the Krylov vectors at V(s) = kv + v[s] ld (v_q at V(s) + q n,
// q = 0 .. restart, then z_q at V(s) + (restart + 1 + q) n), and its reductions land in H(s) = hb + h[s] GM_H, at
// H(s)[off + q].  (kv, ld and hb are kernel arguments of their own: a struct that mixes pointers with the dynamically
// indexed arrays is copied to a stack frame.)
struct GmSlots { int v[MS_NB_MAX], h[MS_NB_MAX]; };
#define GM_ARGS double* __restrict__ kv, long long ld, double* __restrict__ hb
#define GM_V(sl, s) (kv + (size_t)(sl).v[s] * ld)
#define GM_HS(sl, s) (hb + (size_t)(sl).h[s] * GM_H)

// The sum over the CTAs of gridDim.x of one value per thread: a shuffle-xor tree in each warp, the warps in order, the
// CTA's partial into part[blockIdx.x]; the last CTA to arrive adds the partials in order (from 0.0) into *res and
// resets the arrival counter
__device__ __forceinline__ void gm_sum(double v, double* __restrict__ part, unsigned* __restrict__ cnt,
                                       double* __restrict__ res) {
  __shared__ double red[EA_WARPS];
  __shared__ bool last;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, P = gridDim.x;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = __dadd_rn(v, __shfl_xor_sync(0xffffffffu, v, o));
  if (lane == 0) red[warp] = v;
  __syncthreads();
  if (threadIdx.x == 0) {
    double t = red[0];
    for (int w = 1; w < EA_WARPS; ++w) t = __dadd_rn(t, red[w]);
    part[blockIdx.x] = t;
    __threadfence();
    last = atomicAdd(cnt, 1u) == (unsigned)P - 1;
  }
  __syncthreads();
  if (!last || threadIdx.x != 0) return;
  __threadfence();
  double r = 0.0;
  for (int q = 0; q < P; ++q) r = __dadd_rn(r, __ldcg(&part[q]));
  *res = r;
  *cnt = 0u;
}

// w = A_op z for slot s = blockIdx.y: one warp per row i (grid-stride) over |A|'s row structure (EaPlan) with the unique
// values of A_op; lane l takes the row's entries l, l + 32, ... in order, t = t (+) (a_ij (*) z_j) from 0, then for
// o = 16, 8, 4, 2, 1: t = t (+) t' of lane l xor o; w_i = lane 0's t.  z is solve slot s (z[s n + i]); lane 0 also
// stores z_i as z_j of the slot (v[s] + (restart + 1 + j) n), and w goes to v_{j+1} (v[s] + (j + 1) n).
__global__ void __launch_bounds__(EA_THREADS) k_gm_apply(int n, int restart, int j, const int* __restrict__ ptr,
                                                         const int* __restrict__ col, const int* __restrict__ uid,
                                                         const double* __restrict__ uval, const double* __restrict__ z,
                                                         GmSlots sl, GM_ARGS) {
  const int lane = threadIdx.x & 31;
  const int s = blockIdx.y;
  const double* zs = z + (size_t)s * n;
  double* w = GM_V(sl, s) + (size_t)(j + 1) * n;
  double* zk = GM_V(sl, s) + (size_t)(restart + 1 + j) * n;
  const int nwarps = gridDim.x * EA_WARPS;
  for (int i = blockIdx.x * EA_WARPS + (threadIdx.x >> 5); i < n; i += nwarps) {
    double t = 0.0;
    for (int e = ptr[i] + lane; e < ptr[i + 1]; e += 32) t = __dadd_rn(t, __dmul_rn(uval[uid[e]], zs[col[e]]));
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) t = __dadd_rn(t, __shfl_xor_sync(0xffffffffu, t, o));
    if (lane == 0) {
      w[i] = t;
      zk[i] = zs[i];
    }
  }
}

// The multi-dot of a Gram-Schmidt pass, grid (ea_parts(n), slots, j + 1): h[s][off + q] = v_q . v_{j+1} of slot s =
// blockIdx.y, q = blockIdx.z, each term v_q,i (*) w_i added (+) in the fixed order of gm_sum
__global__ void __launch_bounds__(EA_THREADS) k_gm_dot(int n, int j, int off, GmSlots sl, GM_ARGS, double* __restrict__ part,
                                                       unsigned* __restrict__ cnt) {
  const int s = blockIdx.y, q = blockIdx.z, P = gridDim.x;
  const double* a = GM_V(sl, s) + (size_t)q * n;
  const double* w = GM_V(sl, s) + (size_t)(j + 1) * n;
  double t = 0.0;
  for (int i = blockIdx.x * EA_THREADS + threadIdx.x; i < n; i += P * EA_THREADS) t = __dadd_rn(t, __dmul_rn(a[i], w[i]));
  const size_t k = (size_t)s * GM_Q + q;
  gm_sum(t, part + k * P, cnt + k, GM_HS(sl, s) + off + q);
}

// The update of a Gram-Schmidt pass, grid (ea_parts(n), slots): w = v_{j+1} of slot s, for q = 0 .. j in order
// w_i = w_i (-) (h[s][off + q] (*) v_q,i).  NRM: also ||w||^2 of the updated w (terms w_i (*) w_i, order of gm_sum) into
// h[s][off + GM_Q - 1].  Called with j + 1 = 0 vectors and NRM for the squared norm of v_0 as it stands.
template <bool NRM>
__global__ void __launch_bounds__(EA_THREADS) k_gm_update(int n, int j, int off, GmSlots sl, GM_ARGS, double* __restrict__ part,
                                                          unsigned* __restrict__ cnt) {
  const int s = blockIdx.y, P = gridDim.x;
  const double* hs = GM_HS(sl, s) + off;
  const double* v0 = GM_V(sl, s);
  double* w = GM_V(sl, s) + (size_t)(j + 1) * n;
  double t2 = 0.0;
  for (int i = blockIdx.x * EA_THREADS + threadIdx.x; i < n; i += P * EA_THREADS) {
    double t = w[i];
    for (int q = 0; q <= j; ++q) t = __dsub_rn(t, __dmul_rn(hs[q], v0[(size_t)q * n + i]));
    if (j >= 0) w[i] = t;
    if (NRM) t2 = __dadd_rn(t2, __dmul_rn(t, t));
  }
  if (NRM) {
    const size_t k = (size_t)s * GM_Q + GM_Q - 1;
    gm_sum(t2, part + k * P, cnt + k, GM_HS(sl, s) + off + GM_Q - 1);
  }
}

// The normalisation: v_{j+1} of slot s = blockIdx.y becomes w_i (/) sqrt(nrm2), nrm2 = h[s][off + GM_Q - 1] (sqrt
// correctly rounded), and is copied into solve slot s (out[s n + i]), the input of the next job-0 solve.  w is v_{j+1}
// as it stands, or for j = -1 (v_0 = r / beta) the residual in solve slot s itself.
__global__ void __launch_bounds__(EA_THREADS) k_gm_scale(int n, int j, int off, GmSlots sl, GM_ARGS, double* __restrict__ out) {
  const int i = blockIdx.x * EA_THREADS + threadIdx.x;
  if (i >= n) return;
  const int s = blockIdx.y;
  const double h = __dsqrt_rn(GM_HS(sl, s)[off + GM_Q - 1]);
  double* v = GM_V(sl, s) + (size_t)(j + 1) * n;
  double* o = out + (size_t)s * n;
  const double r = __ddiv_rn(j < 0 ? o[i] : v[i], h);
  v[i] = r;
  o[i] = r;
}

// The correction of one cycle, slot s = blockIdx.y: column c = cols.c[s] of x (counted from the block's first), its
// m = m[s] vectors z_0 .. z_{m-1} at V(s) + (restart + 1 + q) n and y_q = y[s GM_RESTART_MAX + q]:
// d = 0, d = d (+) (y_q (*) z_q,i) for q = 0 .. m - 1 in order; xold_i = x_i, x_i = x_i (+) d.
struct GmFinal { int c[MS_NB_MAX]; int m[MS_NB_MAX]; };
__global__ void __launch_bounds__(EA_THREADS) k_gm_final(int n, int restart, GmSlots sl, GM_ARGS, GmFinal f,
                                                         const double* __restrict__ y, double* __restrict__ x,
                                                         double* __restrict__ xold) {
  const int i = blockIdx.x * EA_THREADS + threadIdx.x;
  if (i >= n) return;
  const int s = blockIdx.y, m = f.m[s];
  const double* z = GM_V(sl, s) + (size_t)(restart + 1) * n + i;
  const double* ys = y + (size_t)s * GM_RESTART_MAX;
  double d = 0.0;
  for (int q = 0; q < m; ++q) d = __dadd_rn(d, __dmul_rn(ys[q], z[(size_t)q * n]));
  const size_t c = (size_t)f.c[s];
  const double v = x[c * n + i];
  xold[c * n + i] = v;
  x[c * n + i] = __dadd_rn(v, d);
}

}  // namespace b200
