// EXPERIMENTAL kernels kept for A/B comparisons -- NOT compiled into libb200ldlt.so (see profiles/r1_summary.md for the
// measurements that retired them): the panelised shared-memory front kernel (k_front_mid), the per-child extend-add
// (k_big_extend_add), the 4x4-blocked Schur kernel (tile_syrk / k_big_schur) and the FP64 tensor-pipe DMMA Schur kernel
// (k_big_schur_dmma).  To try one: include this file after factor_kernels.cu and add the launch by hand.
#include "factor_kernels.cu"
namespace b200 {
// --------------------------------------------------------------------------------------------
// Class M: fronts of order 33..128, one CTA, front in shared memory, PANELISED: the 32x32 diagonal block of each
// panel is factorised in registers by warp 0 (warp_ldlt32, ~2.5x faster per pivot than the CTA-wide column loop of
// k_front_smem), the panel rows and the trailing update are CTA-parallel.
// smem: colbuf[64] | F[ld*f] | Lp[f*33] | Wp[f*33] | T[32*33] | dinv_s[32] | doff_s[32] | gmax[32] | order[32] | pt[32]
// --------------------------------------------------------------------------------------------
__host__ __device__ inline size_t mid_smem_bytes(int f) {
  const size_t ld = (size_t)(f | 1);
  return (ld * f + 2 * (size_t)f * 33 + 32 * 33 + 64 + 32 + 32 + 32) * sizeof(double) + 64 * sizeof(int);
}

__global__ void __launch_bounds__(256) k_front_mid(DevSym S, DevNum N, const int* __restrict__ front_list) {
  extern __shared__ double smem[];
  const int s = front_list[blockIdx.x];
  const int c0 = S.sn_start[s], k = S.sn_start[s + 1] - c0;
  const int r = (int)(S.rows_ptr[s + 1] - S.rows_ptr[s]);
  const int f = k + r, ld = f | 1;
  double* colbuf = smem;                 // first: warp_ldlt32 reads it with 16-byte vector loads
  double* F = colbuf + 64;
  double* Lp = F + (size_t)ld * f;
  double* Wp = Lp + (size_t)f * 33;
  double* T = Wp + (size_t)f * 33;
  double* dinv_s = T + 32 * 33;
  double* doff_s = dinv_s + 32;
  double* gmax = doff_s + 32;
  int* order = (int*)(gmax + 32);
  int* pt = order + 32;
  const int tid = threadIdx.x, nt = blockDim.x, lane = tid & 31, warp = tid >> 5, nwarp = nt >> 5;

  for (int t = tid; t < ld * f; t += nt) F[t] = 0.0;
  __syncthreads();
  for (long long uu = S.uent_ptr[s] + tid; uu < S.uent_ptr[s + 1]; uu += nt) {
    unsigned d = S.u_dst[uu];
    int lr = d & 0xffffu, lc = d >> 16;
    double v = N.uval[uu];
    F[lr + lc * ld] = v;
    F[lc + lr * ld] = v;
  }
  __syncthreads();
  for (int q = S.child_ptr[s]; q < S.child_ptr[s + 1]; ++q) {
    const int c = S.child_idx[q];
    const int rc = (int)(S.rows_ptr[c + 1] - S.rows_ptr[c]);
    const double* __restrict__ cb = N.CB + S.cb_off[c];
    const int* __restrict__ rl = S.rel + S.rows_ptr[c];
    for (int jj = warp; jj < rc; jj += nwarp) {
      const int lj = rl[jj];
      for (int ii = jj + lane; ii < rc; ii += 32) {
        const int li = rl[ii];
        const double v = cb[ii + (size_t)jj * rc];
        F[li + lj * ld] += v;
        if (li != lj) F[lj + li * ld] += v;
      }
    }
    __syncthreads();
  }
  double* __restrict__ P = N.L + S.L_off[s];
  for (int jb = 0; jb < k; jb += 32) {
    const int nb = min(32, k - jb), below = jb + nb;
    // 1. column maxima below the diagonal block (threshold test sees the whole front column)
    for (int c = warp; c < nb; c += nwarp) {
      double m = 0.0;
      for (int i = below + lane; i < f; i += 32) m = fmax(m, fabs(F[i + (jb + c) * ld]));
      m = warp_max(m);
      if (lane == 0) gmax[c] = m;
    }
    __syncthreads();
    // 2. pivoted LDL^T of the diagonal block in registers (warp 0)
    if (warp == 0) {
      double a[32];
#pragma unroll
      for (int c = 0; c < 32; ++c) a[c] = (lane < nb && c < nb) ? F[(jb + lane) + (jb + c) * ld] : 0.0;
      const double gext = (lane < nb) ? gmax[lane] : 0.0;
      warp_ldlt32<false>(a, a, nb, nb, N.u, N.tiny, T, order, pt, dinv_s, doff_s, colbuf, gext, N.counters);
      if (lane < nb) {
        N.lperm[c0 + jb + lane] = jb + order[lane];
        N.dinv[c0 + jb + lane] = dinv_s[lane];
        N.doff[c0 + jb + lane] = doff_s[lane];
        N.ptype[c0 + jb + lane] = pt[lane];
      }
    }
    __syncthreads();
    // 3a. the block's row interchanges for the L columns already written (columns [0, jb), rows [jb, jb+nb))
    for (int c = tid; c < jb; c += nt) {
      double* col = P + (size_t)c * f + jb;
      double tmp[32];
#pragma unroll
      for (int t = 0; t < 32; ++t) tmp[t] = (t < nb) ? col[t] : 0.0;
      // permute through this thread's private slice of Wp (free until step 3b)
      double* sl = Wp + (size_t)c * 33;
#pragma unroll
      for (int t = 0; t < 32; ++t) sl[t] = tmp[t];
      for (int t = 0; t < nb; ++t) col[t] = sl[order[t]];
    }
    __syncthreads();
    // 3b. panel rows below the block: x = A_perm L_bb^-T (= L D), l = x D^-1
    for (int i = below + tid; i < f; i += nt) {
      double x[32];
#pragma unroll
      for (int t = 0; t < 32; ++t) x[t] = (t < nb) ? F[i + (jb + order[t]) * ld] : 0.0;
#pragma unroll
      for (int t = 0; t < 32; ++t) {
        if (t < nb) {
          double acc = x[t];
          const double* lrow = T + order[t] * 33;   // row of L_bb in pivot order: Lraw[order[t]][q], q < t
#pragma unroll
          for (int q = 0; q < 32; ++q)
            if (q < t) acc -= x[q] * lrow[q];
          x[t] = acc;
        }
      }
#pragma unroll
      for (int t = 0; t < 32; ++t) {
        if (t < nb) {
          double l;
          const int ty = pt[t];
          if (ty == 1) l = x[t] * dinv_s[t];
          else if (ty == 2) l = x[t] * dinv_s[t] + x[(t + 1 < 32) ? t + 1 : t] * doff_s[t];
          else l = x[(t > 0) ? t - 1 : 0] * doff_s[(t > 0) ? t - 1 : 0] + x[t] * dinv_s[t];
          Lp[i * 33 + t] = l;
          Wp[i * 33 + t] = x[t];
          P[i + (size_t)(jb + t) * f] = l;
        }
      }
    }
    // L_bb (pivot order) and zeros above it
    for (int e = tid; e < nb * (jb + nb); e += nt) {
      const int t = e / (jb + nb), i = e % (jb + nb);
      double v;
      if (i < jb + t) v = 0.0;
      else if (i == jb + t) v = 1.0;
      else v = T[order[i - jb] * 33 + t];
      P[i + (size_t)(jb + t) * f] = v;
    }
    __syncthreads();
    // 4. trailing update (full square so the next diagonal block / column maxima read consistent values)
    const int m = f - below;
    for (int e = tid; e < ((m + 3) / 4) * ((m + 3) / 4); e += nt) {
      const int bi = e % ((m + 3) / 4), bj = e / ((m + 3) / 4);
      const int i0 = below + 4 * bi, j0 = below + 4 * bj;
      double acc[4][4];
#pragma unroll
      for (int a2 = 0; a2 < 4; ++a2)
#pragma unroll
        for (int b2 = 0; b2 < 4; ++b2) acc[a2][b2] = 0.0;
      for (int t = 0; t < nb; ++t) {
        double lv[4], wv[4];
#pragma unroll
        for (int q = 0; q < 4; ++q) {
          lv[q] = (i0 + q < f) ? Lp[(i0 + q) * 33 + t] : 0.0;
          wv[q] = (j0 + q < f) ? Wp[(j0 + q) * 33 + t] : 0.0;
        }
#pragma unroll
        for (int a2 = 0; a2 < 4; ++a2)
#pragma unroll
          for (int b2 = 0; b2 < 4; ++b2) acc[a2][b2] = fma(lv[a2], wv[b2], acc[a2][b2]);
      }
#pragma unroll
      for (int a2 = 0; a2 < 4; ++a2)
#pragma unroll
        for (int b2 = 0; b2 < 4; ++b2)
          if (i0 + a2 < f && j0 + b2 < f) F[(i0 + a2) + (j0 + b2) * ld] -= acc[a2][b2];
    }
    __syncthreads();
  }
  double* __restrict__ cbo = N.CB + S.cb_off[s];
  for (int mcol = warp; mcol < r; mcol += nwarp)
    for (int i = mcol + lane; i < r; i += 32) cbo[i + (size_t)mcol * r] = F[(k + i) + (k + mcol) * ld];
}

// extend-add of the q-th child of every big front in the list (one pass per child rank =>
// no two CTAs touch the same parent entry; deterministic, no atomics)
__global__ void k_big_extend_add(DevSym S, DevNum N, const int* __restrict__ front_list, int q) {
  const int p = front_list[blockIdx.y];
  const int nch = S.child_ptr[p + 1] - S.child_ptr[p];
  if (q >= nch) return;
  const int c = S.child_idx[S.child_ptr[p] + q];
  const int rc = (int)(S.rows_ptr[c + 1] - S.rows_ptr[c]);
  const int kp = S.sn_start[p + 1] - S.sn_start[p];
  const int rp = (int)(S.rows_ptr[p + 1] - S.rows_ptr[p]);
  const int fp = kp + rp;
  const double* __restrict__ cb = N.CB + S.cb_off[c];
  const int* __restrict__ rl = S.rel + S.rows_ptr[c];
  double* P = N.L + S.L_off[p];
  double* C = N.CB + S.cb_off[p];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarp = blockDim.x >> 5;
  for (int jj = blockIdx.x * nwarp + warp; jj < rc; jj += gridDim.x * nwarp) {
    const int lj = rl[jj];
    for (int ii = jj + lane; ii < rc; ii += 32) {
      const int li = rl[ii];
      const double v = cb[ii + (size_t)jj * rc];
      if (lj < kp) P[li + (size_t)lj * fp] += v;
      else C[(li - kp) + (size_t)(lj - kp) * rp] += v;
    }
  }
}

// C[i,j] -= sum_t A[i,t] * B[j,t] on the lower trapezoid i >= j (global coordinates aligned:
// row i of C and column j of C refer to the same front index origin). 64x64 tiles, 256 threads.
__device__ __forceinline__ void tile_syrk(double* __restrict__ C, long long ldc,
                                          const double* __restrict__ A,
                                          const double* __restrict__ Bm, long long ld, int M, int Nn,
                                          int K, int ti, int tj, double* colmax_next = nullptr) {
  __shared__ double As[TK][TM + 1];
  __shared__ double Bs[TK][TM + 1];
  const int i0 = ti * TM, j0 = tj * TM;
  if (i0 + TM - 1 < j0) return;  // tile strictly above the diagonal
  const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
  double acc[4][4];
#pragma unroll
  for (int a = 0; a < 4; ++a)
#pragma unroll
    for (int b = 0; b < 4; ++b) acc[a][b] = 0.0;
  for (int k0 = 0; k0 < K; k0 += TK) {
    for (int t = threadIdx.x; t < TM * TK; t += 256) {
      int ii = t % TM, kk = t / TM;
      int gi = i0 + ii, gj = j0 + ii, gk = k0 + kk;
      As[kk][ii] = (gi < M && gk < K) ? A[gi + (long long)gk * ld] : 0.0;
      Bs[kk][ii] = (gj < Nn && gk < K) ? Bm[gj + (long long)gk * ld] : 0.0;
    }
    __syncthreads();
#pragma unroll
    for (int kk = 0; kk < TK; ++kk) {
      double a[4], b[4];
#pragma unroll
      for (int q = 0; q < 4; ++q) { a[q] = As[kk][tx + 16 * q]; b[q] = Bs[kk][ty + 16 * q]; }
#pragma unroll
      for (int q = 0; q < 4; ++q)
#pragma unroll
        for (int p = 0; p < 4; ++p) acc[q][p] = fma(a[q], b[p], acc[q][p]);
    }
    __syncthreads();
  }
#pragma unroll
  for (int q = 0; q < 4; ++q)
#pragma unroll
    for (int p = 0; p < 4; ++p) {
      int gi = i0 + tx + 16 * q, gj = j0 + ty + 16 * p;
      if (gi < M && gj < Nn && gi >= gj) {
        // colmax_next != nullptr marks the panel update: the 32x32 diagonal block of the NEXT panel is updated by
        // CTA 0 of k_big_trsm instead, so the next k_big_diag does not have to wait for this (bulk) kernel
        if (colmax_next && gi < min(NB, Nn) && gj < NB) continue;   // (a partial last panel has fewer than 32 columns)
        const double nv = C[gi + (long long)gj * ldc] - acc[q][p];
        C[gi + (long long)gj * ldc] = nv;
        // columns [32,64) of the trailing matrix are the panel AFTER next: record their maxima below its diagonal
        // block (the next panel's chain kernel runs concurrently with this update, so it uses the values recorded
        // one panel earlier)
        if (colmax_next && gj >= NB && gj < 2 * NB && gi >= 2 * NB)
          atomicMax(reinterpret_cast<unsigned long long*>(colmax_next + gj), (unsigned long long)__double_as_longlong(fabs(nv)));
      }
    }
}

// --------------------------------------------------------------------------------------------
// FP64 tensor-pipe version of the Schur-complement contraction: C[i,j] -= sum_t A[i,t] * B[j,t], lower tiles only,
// with mma.sync.m8n8k4.f64 (DMMA - the only FP64 path of the tensor pipe; wgmma has no f64 type).
// CTA tile 128x128, K step 16, 8 warps as 4(M) x 2(N), each warp 32x64 = 4 x 8 DMMA tiles (64 accumulators/thread).
// Shared tiles As/Bs[16][132]: row stride 132 doubles (== 4 mod 16) makes the 64-bit fragment loads conflict-free.
// --------------------------------------------------------------------------------------------
#define DM_T 128
#define DM_K 16
#define DM_LD 132
__device__ __forceinline__ void dmma_8x8x4(double& c0, double& c1, const double a, const double b) {
  asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};\n"
               : "+d"(c0), "+d"(c1) : "d"(a), "d"(b));
}

__global__ void __launch_bounds__(256) k_big_schur_dmma(DevSym S, DevNum N, const int* __restrict__ front_list) {
  __shared__ double As[DM_K * DM_LD];
  __shared__ double Bs[DM_K * DM_LD];
  const int s = front_list[blockIdx.z];
  const int k = S.sn_start[s + 1] - S.sn_start[s];
  const int r = (int)(S.rows_ptr[s + 1] - S.rows_ptr[s]);
  const int f = k + r;
  const int ti = blockIdx.x, tj = blockIdx.y;
  if (tj > ti || ti * DM_T >= r) return;                 // lower tiles only
  double* __restrict__ C = N.CB + S.cb_off[s];
  const double* __restrict__ A = N.L + S.L_off[s] + k;    // rows k.. of L   (ld = f)
  const double* __restrict__ B = N.W + S.L_off[s] + k;    // rows k.. of L*D (ld = f)
  const int i0 = ti * DM_T, j0 = tj * DM_T;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int gid = lane >> 2, tig = lane & 3;
  const int wm = (warp & 3) * 32, wn = (warp >> 2) * 64;
  double acc[4][8][2];
#pragma unroll
  for (int a = 0; a < 4; ++a)
#pragma unroll
    for (int b = 0; b < 8; ++b) { acc[a][b][0] = 0.0; acc[a][b][1] = 0.0; }
  // global -> register prefetch: thread loads row (tid & 127), k columns (tid >> 7) + 2q
  const int lrow = tid & 127, lk = tid >> 7;
  double pa[8], pb[8];
  auto prefetch = [&](int k0) {
#pragma unroll
    for (int q = 0; q < 8; ++q) {
      const int kk = k0 + lk + 2 * q;
      pa[q] = (i0 + lrow < r && kk < k) ? A[(size_t)(i0 + lrow) + (size_t)kk * f] : 0.0;
      pb[q] = (j0 + lrow < r && kk < k) ? B[(size_t)(j0 + lrow) + (size_t)kk * f] : 0.0;
    }
  };
  prefetch(0);
  for (int k0 = 0; k0 < k; k0 += DM_K) {
#pragma unroll
    for (int q = 0; q < 8; ++q) {
      As[(lk + 2 * q) * DM_LD + lrow] = pa[q];
      Bs[(lk + 2 * q) * DM_LD + lrow] = pb[q];
    }
    __syncthreads();
    if (k0 + DM_K < k) prefetch(k0 + DM_K);
#pragma unroll
    for (int ks = 0; ks < DM_K; ks += 4) {
      double af[4], bf[8];
#pragma unroll
      for (int a = 0; a < 4; ++a) af[a] = As[(ks + tig) * DM_LD + wm + a * 8 + gid];
#pragma unroll
      for (int b = 0; b < 8; ++b) bf[b] = Bs[(ks + tig) * DM_LD + wn + b * 8 + gid];
#pragma unroll
      for (int a = 0; a < 4; ++a)
#pragma unroll
        for (int b = 0; b < 8; ++b) dmma_8x8x4(acc[a][b][0], acc[a][b][1], af[a], bf[b]);
    }
    __syncthreads();
  }
#pragma unroll
  for (int a = 0; a < 4; ++a)
#pragma unroll
    for (int b = 0; b < 8; ++b)
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const int gi = i0 + wm + a * 8 + gid, gj = j0 + wn + b * 8 + 2 * tig + e;
        if (gi < r && gj < r && gi >= gj) C[(size_t)gi + (size_t)gj * r] -= acc[a][b][e];
      }
}

// Schur complement: CB -= L21 * (L21 D)^T  (the dense contraction of the front)
__global__ void __launch_bounds__(256) k_big_schur(DevSym S, DevNum N, const int* __restrict__ front_list) {
  const int s = front_list[blockIdx.z];
  const int k = S.sn_start[s + 1] - S.sn_start[s];
  const int r = (int)(S.rows_ptr[s + 1] - S.rows_ptr[s]);
  const int f = k + r;
  if ((int)blockIdx.x * TM >= r || (int)blockIdx.y * TM >= r) return;
  double* C = N.CB + S.cb_off[s];
  const double* P = N.L + S.L_off[s];
  const double* Wp = N.W + S.L_off[s];
  tile_syrk(C, r, P + k, Wp + k, f, r, r, k, blockIdx.x, blockIdx.y);
}



// stand-alone diagonal-block kernels (superseded by k_big_chain, which fuses them with the next block's panel rows)
// factor the NB x NB diagonal block at panel offset jb (pivoting restricted to the block).
// ONE WARP per front, block held in registers (warp_ldlt32).
__global__ void __launch_bounds__(32) k_big_diag(DevSym S, DevNum N, const int* __restrict__ front_list, int jb) {
  __shared__ double T[33 * NB];
  __shared__ __align__(16) double colbuf[64];
  __shared__ double dinv_s[NB], doff_s[NB];
  __shared__ int order[NB], pt[NB];
  const int s = front_list[blockIdx.x];
  const int c0 = S.sn_start[s], k = S.sn_start[s + 1] - c0;
  if (jb >= k) return;
  const int f = k + (int)(S.rows_ptr[s + 1] - S.rows_ptr[s]);
  const int nb = min(NB, k - jb);
  double* __restrict__ P = N.L + S.L_off[s];
  const int lane = threadIdx.x;
  // lower part, coalesced per column, through a shared tile
  {
    double tmp[NB];
#pragma unroll
    for (int j = 0; j < NB; ++j) tmp[j] = (j < nb && lane >= j && lane < nb) ? P[(jb + lane) + (size_t)(jb + j) * f] : 0.0;
#pragma unroll
    for (int j = 0; j < NB; ++j) T[lane * 33 + j] = tmp[j];
  }
  __syncwarp();
  double a[32];
#pragma unroll
  for (int c = 0; c < 32; ++c) a[c] = (c <= lane) ? T[lane * 33 + c] : T[c * 33 + lane];
  __syncwarp();
  const double gext = (lane < nb) ? N.colmax[c0 + jb + lane] : 0.0;
  warp_ldlt32<false>(a, a, nb, nb, N.u, N.tiny, T, order, pt, dinv_s, doff_s, colbuf, gext, N.counters);
  // write the block back in pivot order: L[t2][t] = Lraw[order[t2]][t]
  const int mine = (lane < nb) ? order[lane] : 0;
#pragma unroll
  for (int j = 0; j < NB; ++j) {
    if (j < nb && lane < nb) {
      double v;
      if (lane < j) v = 0.0;
      else if (lane == j) v = 1.0;
      else v = T[mine * 33 + j];
      P[(jb + lane) + (size_t)(jb + j) * f] = v;
    }
  }
  if (lane < nb) {
    N.bperm[c0 + jb + lane] = mine;
    N.lperm[c0 + jb + lane] = jb + mine;
    N.dinv[c0 + jb + lane] = dinv_s[lane];
    N.doff[c0 + jb + lane] = doff_s[lane];
    N.ptype[c0 + jb + lane] = pt[lane];
  }
}

// 4-warp version of k_big_diag (same inputs / outputs)
__global__ void __launch_bounds__(128) k_big_diag4(DevSym S, DevNum N, const int* __restrict__ front_list, int jb) {
  __shared__ double T[33 * NB];
  __shared__ double colA[64], colB[64];
  __shared__ double dinv_s[NB], doff_s[NB];
  __shared__ int order[NB], pt[NB];
  const int s = front_list[blockIdx.x];
  const int c0 = S.sn_start[s], k = S.sn_start[s + 1] - c0;
  if (jb >= k) return;
  const int f = k + (int)(S.rows_ptr[s + 1] - S.rows_ptr[s]);
  const int nb = min(NB, k - jb);
  double* __restrict__ P = N.L + S.L_off[s];
  const int tid = threadIdx.x, lane = tid & 31, w = tid >> 5;
  // lower part of the block, coalesced per column, into the shared tile (8 columns per warp)
#pragma unroll
  for (int q = 0; q < 8; ++q) {
    const int j = 8 * w + q;
    T[lane * 33 + j] = (j < nb && lane >= j && lane < nb) ? P[(jb + lane) + (size_t)(jb + j) * f] : 0.0;
  }
  __syncthreads();
  double a[8];
#pragma unroll
  for (int q = 0; q < 8; ++q) { const int c = 8 * w + q; a[q] = (c <= lane) ? T[lane * 33 + c] : T[c * 33 + lane]; }
  const double gext = (lane < nb) ? N.colmax[c0 + jb + lane] : 0.0;
  __syncthreads();   // T is reused as Lraw
  cta_ldlt32(a, nb, N.u, N.tiny, T, order, pt, dinv_s, doff_s, colA, colB, gext, N.counters);
  // write the block back in pivot order: L[t2][t] = Lraw[order[t2]][t]
  const int mine = (lane < nb) ? order[lane] : 0;
#pragma unroll
  for (int q = 0; q < 8; ++q) {
    const int j = 8 * w + q;
    if (j < nb && lane < nb) {
      double v;
      if (lane < j) v = 0.0;
      else if (lane == j) v = 1.0;
      else v = T[mine * 33 + j];
      P[(jb + lane) + (size_t)(jb + j) * f] = v;
    }
  }
  if (w == 0 && lane < nb) {
    N.bperm[c0 + jb + lane] = mine;
    N.lperm[c0 + jb + lane] = jb + mine;
    N.dinv[c0 + jb + lane] = dinv_s[lane];
    N.doff[c0 + jb + lane] = doff_s[lane];
    N.ptype[c0 + jb + lane] = pt[lane];
  }
}


}  // namespace b200
