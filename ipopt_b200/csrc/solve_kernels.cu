// Around the triangular solve (solve_dataflow.cu), sm_90a: permutation + scaling of the right-hand sides in and of the
// solutions out, the pivot-order copies and the D^-1 pass of the partial solves, and the residual helpers.
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

// Entry p of y = D^-1 v, pivot order.  ty = ptype[p], d = dinv[p]; for a 2x2 pivot vq = v at the partner and o = the
// pair's off-diagonal (doff at its first pivot).  Each row of a pair is "first entry x its coefficient" fused onto the
// rounded product of the second entry: exactly what the fused forward sweeps compiled to before this helper existed
// (sm_90a SASS: DMUL, then DFMA).  The intrinsics pin that rounding, so the fused sweeps (solve_dataflow.cu) and
// k_dinv produce the same bits whatever the compiler would contract.
__device__ __forceinline__ double dinv_entry(int ty, double v, double vq, double d, double o) {
  if (ty == 1) return __dmul_rn(v, d);
  if (ty == 2) return __fma_rn(v, d, __dmul_rn(vq, o));   // first of the pair:  d v + o vq
  return __fma_rn(vq, o, __dmul_rn(v, d));                // second of the pair: o vq + d v
}

// Partial solves: vectors in pivot order (position p = sn_start[s] + t for pivot t of front s).  Between the sweeps the
// value of position p lives in xp[p], or in big[piv_big[p]] when p is a pivot of a big front (piv_big[p] >= 0: those
// keep their forward result in bigv, see solve_dataflow.cu).  Column blockIdx.y; b / out: leading dimension n.
// out = sweep values (after a forward sweep without D)
__global__ void k_piv_out(int n, const long long* __restrict__ piv_big, const double* __restrict__ xp, long long ldx,
                          const double* __restrict__ big, long long ldbig, double* __restrict__ out) {
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  const long long c = blockIdx.y;
  if (p < n) { const long long q = piv_big[p]; out[c * n + p] = q >= 0 ? big[c * ldbig + q] : xp[c * ldx + p]; }
}
// sweep values = b (before a backward sweep)
__global__ void k_piv_in(int n, const long long* __restrict__ piv_big, const double* __restrict__ b,
                         double* __restrict__ xp, long long ldx, double* __restrict__ big, long long ldbig) {
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  const long long c = blockIdx.y;
  if (p < n) {
    const long long q = piv_big[p];
    const double v = b[c * n + p];
    if (q >= 0) big[c * ldbig + q] = v; else xp[c * ldx + p] = v;
  }
}
// out = D^-1 b, pivot order, the partner of a 2x2 pivot read from b (b and out must not overlap).  piv_big == nullptr:
// out[p] (leading dimension n); else the sweep values, as k_piv_in writes them (out = xp, leading dimension ldx).
__global__ void k_dinv(int n, const int* __restrict__ ptype, const double* __restrict__ dinv,
                       const double* __restrict__ doff, const double* __restrict__ b, const long long* __restrict__ piv_big,
                       double* __restrict__ out, long long ldx, double* __restrict__ big, long long ldbig) {
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  const long long c = blockIdx.y;
  if (p >= n) return;
  const double* bc = b + c * n;
  const int ty = ptype[p];
  double y;
  if (ty == 1) y = dinv_entry(1, bc[p], 0.0, dinv[p], 0.0);
  else if (ty == 2) y = dinv_entry(2, bc[p], bc[p + 1], dinv[p], doff[p]);
  else y = dinv_entry(3, bc[p], bc[p - 1], dinv[p], doff[p - 1]);
  if (!piv_big) { out[c * n + p] = y; return; }
  const long long q = piv_big[p];
  if (q >= 0) big[c * ldbig + q] = y; else out[c * ldx + p] = y;
}

// Fredholm alternative (b200ldlt_solve_fredholm), between a forward sweep without D and the backward sweep, on the sweep
// values (see k_piv_out) of column blockIdx.y = c holding y = L^-1 P^T S b.  In place, column c becomes D^+ y -- D^-1 from
// dinv / doff through dinv_entry exactly as k_dinv rounds it, so the backward sweep gives job 0's bits; dinv = 0 at the
// zero pivots makes it D^+ -- and z = y on the zero pivots (zflag[p] != 0, always 1x1 pivots), 0 elsewhere, goes to
// column zcol + c of the sweep values (zout == nullptr) or to zout[c * n + p].  nrm[2c] / nrm[2c+1] (double bits,
// atomicMax; zero-initialised) receive max_p |y_p| and max_Z |y_p|, NaN counted as infinity.  The thread of the first
// pivot of a 2x2 block reads and writes both of its entries, so no thread reads what another writes.
__global__ void k_fred(int n, const int* __restrict__ ptype, const double* __restrict__ dinv, const double* __restrict__ doff,
                       const unsigned char* __restrict__ zflag, const long long* __restrict__ piv_big, double* __restrict__ xp,
                       long long ldx, double* __restrict__ big, long long ldbig, int zcol, double* __restrict__ zout,
                       unsigned long long* __restrict__ nrm) {
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  const long long c = blockIdx.y;
  const int ty = p < n ? ptype[p] : 3;
  double ay = 0.0, az = 0.0;
  // sweep value at position r (v) and where it lives; the outputs y (column c) and z (column zcol + c or zout)
  auto get = [&](int r) { const long long q = piv_big[r]; return q >= 0 ? big[c * ldbig + q] : xp[c * ldx + r]; };
  auto put = [&](int r, double y, double z) {
    const long long q = piv_big[r];
    if (q >= 0) { big[c * ldbig + q] = y; if (!zout) big[(zcol + c) * ldbig + q] = z; }
    else { xp[c * ldx + r] = y; if (!zout) xp[(zcol + c) * ldx + r] = z; }
    if (zout) zout[c * n + r] = z;
  };
  auto mag = [](double v) { return (v == v) ? fabs(v) : INFINITY; };
  if (ty == 1) {
    const double v = get(p);
    ay = mag(v);
    const bool zp = zflag[p] != 0;
    if (zp) az = ay;
    put(p, dinv_entry(1, v, 0.0, dinv[p], 0.0), zp ? v : 0.0);
  } else if (ty == 2) {
    const double v0 = get(p), v1 = get(p + 1);
    ay = fmax(mag(v0), mag(v1));
    put(p, dinv_entry(2, v0, v1, dinv[p], doff[p]), 0.0);
    put(p + 1, dinv_entry(3, v1, v0, dinv[p + 1], doff[p]), 0.0);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    ay = fmax(ay, __shfl_xor_sync(0xffffffffu, ay, o));
    az = fmax(az, __shfl_xor_sync(0xffffffffu, az, o));
  }
  if ((threadIdx.x & 31) == 0) {
    if (ay > 0.0) atomicMax(nrm + 2 * c, (unsigned long long)__double_as_longlong(ay));
    if (az > 0.0) atomicMax(nrm + 2 * c + 1, (unsigned long long)__double_as_longlong(az));
  }
}
// x[perm[i]] = scale[perm[i]] * xp[i] as k_sol_out, for the 2w columns of a Fredholm block: column c < w to x + c n, the
// null-space columns c >= w to x + (fcol + c - w) n
__global__ void k_fred_out(int n, const int* __restrict__ perm, const double* __restrict__ scale, const double* __restrict__ xp,
                           long long ldx, double* __restrict__ x, int w, long long fcol) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  const long long c = blockIdx.y;
  const long long oc = c < w ? c : fcol + c - w;
  if (i < n) { const int o = perm[i]; x[oc * n + o] = scale[o] * xp[c * ldx + i]; }
}

// Entries of A^-1 (b200ldlt_inverse_entries), after the forward stage of a block of unit columns (k_sps_in and the
// pruned sweep).  The y store: column c0 + blockIdx.y of the call keeps its reach at [yoff[c], yoff[c + 1]), ypos the
// pivot positions and y the sweep values there (see k_piv_out), read from column blockIdx.y of the sweep state.  Also
// the output of the sparse forward solve: one column with yoff = {0, nxi}.
__global__ void k_inv_out(int c0, const long long* __restrict__ yoff, const int* __restrict__ ypos,
                          const long long* __restrict__ piv_big, const double* __restrict__ xp, long long ldx,
                          const double* __restrict__ big, long long ldbig, double* __restrict__ y) {
  const long long c = blockIdx.y;
  const long long i = yoff[c0 + c] + blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (i < yoff[c0 + c + 1]) {
    const int p = ypos[i];
    const long long q = piv_big[p];
    y[i] = q >= 0 ? big[c * ldbig + q] : xp[c * ldx + p];
  }
}

// one entry M_ij = y_i^T D^-1 y_j: the common suffix of the two columns in the y store, m elements at a (y_i) and b (y_j)
struct InvEnt {
  long long a, b;
  int m, pad;
};

// One warp per entry.  Lane l sums, in ascending order from +0, the terms that start at suffix offsets o = l (mod 32):
// d (a b) for a 1x1 pivot, (d1 (a1 b1) + d2 (a2 b2)) + o12 ((a1 b2) + (a2 b1)) for a 2x2 pivot at its first position,
// nothing at its second; then s += shfl_xor(s, k) for k = 16, 8, 4, 2, 1.  Every operation is rounded on its own (no
// FMA), and each term and each butterfly step is symmetric in its operands, so (i, j) and (j, i) give the same bits and
// a float64 replay on the host reproduces them.
__global__ void k_inv_dot(int nent, const InvEnt* __restrict__ ent, const double* __restrict__ y, const int* __restrict__ ypos,
                          const int* __restrict__ ptype, const double* __restrict__ dinv, const double* __restrict__ doff,
                          double* __restrict__ vals) {
  const int t = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int l = threadIdx.x & 31;
  if (t >= nent) return;   // (the whole warp)
  const InvEnt E = ent[t];
  const double* ya = y + E.a;
  const double* yb = y + E.b;
  const int* pa = ypos + E.a;
  double s = 0.0;
  for (int o = l; o < E.m; o += 32) {
    const int p = pa[o], ty = ptype[p];
    if (ty == 1) {
      s = __dadd_rn(s, __dmul_rn(dinv[p], __dmul_rn(ya[o], yb[o])));
    } else if (ty == 2) {
      const double a1 = ya[o], a2 = ya[o + 1], b1 = yb[o], b2 = yb[o + 1];
      const double dd = __dadd_rn(__dmul_rn(dinv[p], __dmul_rn(a1, b1)), __dmul_rn(dinv[p + 1], __dmul_rn(a2, b2)));
      const double od = __dmul_rn(doff[p], __dadd_rn(__dmul_rn(a1, b2), __dmul_rn(a2, b1)));
      s = __dadd_rn(s, __dadd_rn(dd, od));
    }
  }
#pragma unroll
  for (int k = 16; k > 0; k >>= 1) s = __dadd_rn(s, __shfl_xor_sync(0xffffffffu, s, k));
  if (l == 0) vals[t] = s;
}

// Sparse solve (b200ldlt_sparse_solve): job 0 of a block of compact right-hand sides with one pattern, swept forward over
// the run set R_f of the pattern and backward over the run set R_b of the selection.  Column blockIdx.y = c of the sweep
// state (x: leading dimension ldx, update vectors ldcbv, flags ldf); column c of b at b + c nbi.
// k_sps_in, the input of all three pruned calls (the sparse forward solve: one column; the entries of A^-1: b an
// identity, whose entries the scaling, a power of two, multiplies exactly): blocks [0, cdiv(ncol, 256)): x = P^T S b at
// the ncol positions of R_f, the scaled entry of b where b has one (bi[j] >= 0: its index into the compact column;
// k_rhs_in's single multiply) and 0 elsewhere.  Blocks after that: frontier front fr[q] (a child of R_f outside R_f), the column's
// slice of its update vector zeroed and its forward flag set to this sweep's epoch, so that its parent neither waits for
// it nor adds anything from it.
__global__ void k_sps_in(int ncol, const int* __restrict__ pos, const int* __restrict__ bi, const int* __restrict__ perm,
                         const double* __restrict__ scale, const double* __restrict__ b, int nbi, double* __restrict__ xp,
                         long long ldx, int nfr, const int* __restrict__ fr, const long long* __restrict__ rows_ptr,
                         double* __restrict__ cbv, long long ldcbv, int* __restrict__ done_f, long long ldf, int epoch) {
  const long long c = blockIdx.y;
  const int nxb = (ncol + 255) / 256;
  if ((int)blockIdx.x < nxb) {
    const int j = blockIdx.x * 256 + threadIdx.x;
    if (j < ncol) {
      const int p = pos[j], q = bi[j];
      xp[c * ldx + p] = q >= 0 ? scale[perm[p]] * b[c * nbi + q] : 0.0;
    }
    return;
  }
  if ((int)blockIdx.x - nxb >= nfr) return;
  const int f = fr[blockIdx.x - nxb];
  const long long r0 = rows_ptr[f], r1 = rows_ptr[f + 1];
  for (long long e = r0 + threadIdx.x; e < r1; e += blockDim.x) cbv[c * ldcbv + e] = 0.0;
  if (threadIdx.x == 0) done_f[c * ldf + f] = epoch;
}
// k_sps_mid, between the forward sweep and the backward sweep, under the backward epoch.  Blocks [0, cdiv(nz, 256)): the
// forward result at the nz positions zpos (the positions the backward sweep reads that the forward sweep did not write)
// set to 0, in x or in bigv through piv_big, wherever k_dinv writes it.  Blocks after that: the backward flag of
// frontier front fb[q] (a parent of R_b outside R_b) set to this sweep's epoch, so that its children do not wait for it.
__global__ void k_sps_mid(int nz, const int* __restrict__ zpos, const long long* __restrict__ piv_big, double* __restrict__ xp,
                          long long ldx, double* __restrict__ big, long long ldbig, int nfb, const int* __restrict__ fb,
                          int* __restrict__ done_b, long long ldf, int epoch) {
  const long long c = blockIdx.y;
  const int nzb = (nz + 255) / 256;
  if ((int)blockIdx.x < nzb) {
    const int j = blockIdx.x * 256 + threadIdx.x;
    if (j < nz) {
      const int p = zpos[j];
      const long long q = piv_big[p];
      if (q >= 0) big[c * ldbig + q] = 0.0; else xp[c * ldx + p] = 0.0;
    }
    return;
  }
  const int q = (blockIdx.x - nzb) * 256 + threadIdx.x;
  if (q < nfb) done_b[c * ldf + fb[q]] = epoch;
}
// k_sps_out: out[c nxs + i] = S P x at the variable of pivot position xpos[i] (k_sol_out's single multiply)
__global__ void k_sps_out(int nxs, const int* __restrict__ xpos, const int* __restrict__ perm, const double* __restrict__ scale,
                          const double* __restrict__ xp, long long ldx, double* __restrict__ out) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  const long long c = blockIdx.y;
  if (i < nxs) { const int p = xpos[i]; out[c * nxs + i] = scale[perm[p]] * xp[c * ldx + p]; }
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
