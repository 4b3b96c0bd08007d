// Device-side data descriptors shared by the numeric kernels (sm_90a).
#pragma once
#include <cstdint>

namespace b200 {

// counters[] layout
// CNT_ZLIST: entries appended to DevNum::zlist (one per pivot counted in CNT_TINY)
enum { CNT_NEG = 0, CNT_FORCED = 1, CNT_TINY = 2, CNT_GROWTH = 3, CNT_2X2 = 4, CNT_ZLIST = 5, CNT_N = 8 };

// An entry of DevNum::zlist: a 1x1 pivot the forced branch replaced by +-1.5e-8 because it was zero.  zl_noise: its whole
// column was rounding noise (a ZERO PIVOT: D_pp = 0 describes the matrix); otherwise |pivot| <= tiny under a column that
// is not noise (a LIFTED ZERO).  zl_neg: the stored pivot is -1.5e-8 (counted in CNT_NEG).
__device__ __forceinline__ int zl_entry(int pos, bool noise, bool neg) { return (pos << 2) | (noise ? 0 : 2) | (neg ? 1 : 0); }
__device__ __forceinline__ void zl_put(int* counters, int* zlist, int pos, bool noise, bool neg) {
  zlist[atomicAdd(counters + CNT_ZLIST, 1)] = zl_entry(pos, noise, neg);
}

struct DevSym {
  int n, nsn;
  const int* sn_start;         // nsn+1
  const int* sn_parent;        // nsn
  const long long* rows_ptr;   // nsn+1
  const int* rows;             // permuted row ids
  const int* rel;              // index in the parent front
  const int* child_ptr;        // nsn+1
  const int* child_idx;
  const long long* uent_ptr;   // nsn+1
  const unsigned* u_dst;       // (lcol<<16)|lrow
  const long long* u_dst64;    // lrow + lcol*f
  const long long* L_off;      // nsn+1
  const long long* cb_off;     // nsn+1
  // children of the big fronts: inverse of rel -- einv[einv_off[c] + j] = index of parent-front row j in child c's
  // row list, or -1 (einv_off[c] = -1 if c's parent is not a big front)
  const long long* einv_off;   // nsn
  const int* einv;
};

struct DevNum {
  double* L;        // supernodal panels, f x k column-major, unit diagonal implied
  double* W;        // L*D for big fronts (same offsets as L), scratch
  double* CB;       // contribution blocks r x r (lower part valid)
  double* uval;     // summed+scaled unique entries
  double* dinv;     // n : D^-1 diagonal
  double* doff;     // n : D^-1 off-diagonal at the first column of a 2x2 pivot
  int* ptype;       // n : 1 = 1x1, 2 = first of 2x2, 3 = second of 2x2
  int* lperm;       // n : pivot position t of supernode s holds pre-pivot local column lperm[start+t]
  int* bperm;       // n : block-local permutation of the last panel step (big fronts)
  double* colmax;   // n : big fronts only: max |entry| of a panel column BELOW its 32x32 diagonal block at panel start
  int* counters;    // CNT_N
  int* zlist;       // n : the forced zero pivots, zl_entry encoded, in arrival order (count: counters[CNT_ZLIST])
  double u;         // pivot threshold
  double tiny;      // zero-pivot threshold (scaled matrix)
};

// the sparse solve (b200ldlt_sparse_solve, solve_kernels.cu): the input of compact right-hand sides (the input of every
// pruned forward sweep), the stage between the two sweeps and the output at the selected variables
__global__ void k_sps_in(int ncol, const int* __restrict__ pos, const int* __restrict__ bi, const int* __restrict__ perm,
                         const double* __restrict__ scale, const double* __restrict__ b, int nbi, double* __restrict__ xp,
                         long long ldx, int nfr, const int* __restrict__ fr, const long long* __restrict__ rows_ptr,
                         double* __restrict__ cbv, long long ldcbv, int* __restrict__ done_f, long long ldf, int epoch);
__global__ void k_sps_mid(int nz, const int* __restrict__ zpos, const long long* __restrict__ piv_big, double* __restrict__ xp,
                          long long ldx, double* __restrict__ big, long long ldbig, int nfb, const int* __restrict__ fb,
                          int* __restrict__ done_b, long long ldf, int epoch);
__global__ void k_sps_out(int nxs, const int* __restrict__ xpos, const int* __restrict__ perm, const double* __restrict__ scale,
                          const double* __restrict__ xp, long long ldx, double* __restrict__ out);

}  // namespace b200
