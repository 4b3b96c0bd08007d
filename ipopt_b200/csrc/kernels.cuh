// Device-side data descriptors shared by the numeric kernels (sm_90a).
#pragma once
#include <cstdint>

namespace b200 {

// counters[] layout
enum { CNT_NEG = 0, CNT_FORCED = 1, CNT_TINY = 2, CNT_GROWTH = 3, CNT_2X2 = 4, CNT_N = 8 };

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
  double u;         // pivot threshold
  double tiny;      // zero-pivot threshold (scaled matrix)
  unsigned long long* flog;   // debug (B200_FACTOR_TIMELINE): [0] = next record, [1] = capacity, then 12 words per record
};

// ---- debug timeline of the factorisation: %globaltimer stamps written by the first / last CTA of a launch ----
#define FLOG_WORDS 12
__device__ __forceinline__ unsigned long long flog_now() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}
__device__ __forceinline__ void flog_put(const DevNum& N, int kind, int s, int jb, const unsigned long long* ts, int nts) {
  const unsigned long long slot = atomicAdd(N.flog, 1ull);
  if (slot >= N.flog[1]) return;
  unsigned long long* r = N.flog + 2 + slot * FLOG_WORDS;
  r[0] = (unsigned long long)kind; r[1] = (unsigned long long)(long long)s; r[2] = (unsigned long long)(long long)jb; r[3] = (unsigned long long)nts;
  for (int i = 0; i < nts && i < FLOG_WORDS - 4; ++i) r[4 + i] = ts[i];
}
// start/end of the first and the last CTA of a grid (kernels that are not on the chain)
struct FlogScope {
  const DevNum& N; int kind, s, jb; unsigned long long t0; bool on;
  __device__ __forceinline__ FlogScope(const DevNum& N_, int kind_, int s_, int jb_) : N(N_), kind(kind_), s(s_), jb(jb_), t0(0), on(false) {
    if (N.flog && threadIdx.x == 0) {
      const unsigned long long nb = (unsigned long long)gridDim.x * gridDim.y * gridDim.z;
      const unsigned long long b = blockIdx.x + (unsigned long long)gridDim.x * (blockIdx.y + (unsigned long long)gridDim.y * blockIdx.z);
      on = (b == 0 || b == nb - 1);
      if (on) t0 = flog_now();
    }
  }
  __device__ __forceinline__ void done() {
    if (on) { unsigned long long ts[2] = {t0, flog_now()}; flog_put(N, kind, s, jb, ts, 2); }
  }
};

}  // namespace b200
