// Schur-complement contraction of the big fronts on the Hopper tensor cores (warpgroup MMA, wgmma), sm_90a.
//
//   CB -= L21 * (L21 D)^T            (the dense GEMM of a front: SURVEY.md 8d "Schur update GEMM")
//
// wgmma has no FP64 type, so the FP64 product is computed EXACTLY-in-integers by an Ozaki split:
//   1. every row of A = L21 and of B = W21 = L21 D is scaled by a power of two so that |entry| <= 1/2, and cut into
//      NS = 8 signed base-128 digits  x = sum_s d_s 2^(-7(s+1)),  |d_s| <= 64  (int8).  All steps are exact in FP64.
//   2. for every digit pair (s, s') with s + s' < NS the int8 GEMM  A_s B_s'^T  runs on the tensor cores
//      (wgmma.mma_async .s32.s8.s8, int32 accumulation in registers: exact -- |sum| <= 64*64*k*(NS) < 2^31 for
//      k < 65536).  Pairs with the same d = s + s' share one accumulator (same weight 2^(-7(d+2))): 8 accumulators.
//   3. epilogue: recombine the 8 accumulators in FP64 (int32 -> double is exact), undo the row scalings (exact) and
//      subtract from the contribution block.
// The dropped pairs (s + s' >= NS) bound the error by ~ (NS+1) k 2^(12-7(NS+2)) = 9k 2^-58 relative to
// rowscale_i * rowscale_j, i.e. below the rounding error k*2^-53*|A||B| of an FP64 GEMM for the k seen here.
//
// Data movement: the digit matrices are written by k_tc_slice directly in the shared-memory operand layout of wgmma
// (K-major, no swizzle: 8-row x 16-byte core matrices), one contiguous unit per (64-row block, 32-column K step) holding
// all 8 digits, so the GEMM kernel stages them with plain 1-D TMA bulk copies (cp.async.bulk + mbarrier) -- no tensor maps.
// Tile and warp roles: one CTA per 64 x 64 lower tile of the contribution block, 288 threads.  Warpgroups 0 and 1
// (warps 0-7) each own 32 columns of the tile: 8 accumulators of m64n32 = 128 int32 registers per thread, which is what
// bounds the tile (the 8 accumulators of a 64 x 64 tile fill half the register file of an SM).  Warp 8 is the TMA producer.
#include <cuda_runtime.h>
#include <stdint.h>

#include "kernels.cuh"

namespace b200 {

#define TC_NS 8            // digits per operand
#define TC_BM 64           // rows of A per tile (= wgmma M)
#define TC_BN 64           // rows of B per tile: two warpgroups x wgmma N = 32
#define TC_WN 32           // columns of the tile per consumer warpgroup (wgmma N)
#define TC_BK 32           // K per wgmma instruction (int8)
#define TC_STAGES 4
#define TC_THREADS 288     // 2 consumer warpgroups + 1 producer warp
#define TC_A_UNIT (TC_NS * 2 * TC_BM * 16)   // bytes of one (64-row block, K step) unit of A digits  = 16 KB
#define TC_B_UNIT (TC_NS * 2 * TC_BN * 16)   // bytes of one (64-row block, K step) unit of B digits  = 16 KB
#define TC_STAGE_BYTES (TC_A_UNIT + TC_B_UNIT)
#define TC_SMEM_BYTES (TC_STAGES * TC_STAGE_BYTES + 1024)

// one big front's digit storage: A (L21) and B (W21) in 64-row blocks, nks = ceil(k / 32) K steps
struct TcFront {
  int s;                 // supernode
  int nks;               // K steps
  long long a_off;       // byte offset of its A units: [row block][K step] x TC_A_UNIT
  long long b_off;       // byte offset of its B units: [row block][K step] x TC_B_UNIT
  long long e_off;       // offset (ints) of its row exponents: ea[r] then eb[r]
};
struct TcTile { int fi, ti, tj; };   // front index in the TcFront list, row block of A, row block of B (lower tiles only)

// ------------------------------------------------------------------------------------------------
// digit extraction.  One warp per row of the front's L21 / W21 (r rows, k columns, ld = f):
// pass 1: row maximum -> exponent e with |x| 2^-e <= 1/2 ; pass 2: digits, written in the wgmma operand layout
//   unit(rowblock, kstep) : [digit s][k chunk j (16 bytes)][row in block][16 bytes]
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) k_tc_slice(DevSym S, DevNum N, const TcFront* __restrict__ fronts, int which /*0: A = L21, 1: B = W21*/,
                                                  int8_t* __restrict__ dig, int* __restrict__ expo) {
  const TcFront F = fronts[blockIdx.y];
  const int s = F.s;
  const int k = S.sn_start[s + 1] - S.sn_start[s];
  const int r = (int)(S.rows_ptr[s + 1] - S.rows_ptr[s]);
  const long long f = k + r;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int BR = which ? TC_BN : TC_BM;
  const long long unit = which ? TC_B_UNIT : TC_A_UNIT;
  const double* __restrict__ X = (which ? N.W : N.L) + S.L_off[s] + k;   // rows k.. of the panel
  int8_t* __restrict__ out = dig + (which ? F.b_off : F.a_off);
  int* __restrict__ ex = expo + F.e_off + (which ? r : 0);
  const int nrb = (r + BR - 1) / BR;
  for (int row = blockIdx.x * 8 + warp; row < nrb * BR; row += gridDim.x * 8) {
    const int rb = row / BR, ri = row % BR;
    // row maximum (rows beyond r are padding: all-zero digits)
    double m = 0.0;
    if (row < r) for (int t = lane; t < k; t += 32) m = fmax(m, fabs(X[row + t * f]));
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) m = fmax(m, __shfl_xor_sync(0xffffffffu, m, o));
    int e = 0;
    if (m > 0.0 && isfinite(m)) { frexp(m, &e); e += 1; }   // m = fr 2^e', fr in [0.5,1)  ->  |x| 2^-(e'+1) < 1/2
    if (lane == 0 && row < r) ex[row] = e;
    const double sc = ldexp(1.0, -e);
    for (int t = lane; t < F.nks * TC_BK; t += 32) {
      double x = (row < r && t < k) ? X[row + t * f] * sc : 0.0;   // exact (power-of-two scaling)
      const int ks = t / TC_BK, tt = t % TC_BK, j = tt >> 4, b = tt & 15;
      int8_t* u = out + ((long long)rb * F.nks + ks) * unit + (long long)j * BR * 16 + (long long)ri * 16 + b;
#pragma unroll
      for (int q = 0; q < TC_NS; ++q) {
        x *= 128.0;
        const double d = rint(x);          // |d| <= 64
        x -= d;                            // exact
        u[(long long)q * 2 * BR * 16] = (int8_t)(int)d;
      }
    }
  }
}

// ---- PTX wrappers -------------------------------------------------------------------------------------------------
__device__ __forceinline__ unsigned tc_smem_u32(const void* p) { return (unsigned)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void tc_mbar_init(unsigned long long* bar, unsigned count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(tc_smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void tc_mbar_expect_tx(unsigned long long* bar, unsigned bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(tc_smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void tc_mbar_arrive(unsigned long long* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(tc_smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void tc_mbar_wait(unsigned long long* bar, unsigned parity) {
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "TCWAIT_%=:\n"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
      "@p bra TCDONE_%=;\n"
      "bra TCWAIT_%=;\n"
      "TCDONE_%=:\n"
      "}\n" ::"r"(tc_smem_u32(bar)), "r"(parity) : "memory");
}
__device__ __forceinline__ void tc_bulk_g2s(void* dst, const void* src, unsigned bytes, unsigned long long* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(tc_smem_u32(dst)),
               "l"(src), "r"(bytes), "r"(tc_smem_u32(bar))
               : "memory");
}
// wgmma shared-memory descriptor, K-major operand without swizzle (canonical layout ((8,m),(16 B,2)):((16 B,SBO),(1,LBO)):
// LBO = byte distance of the two 16-byte K chunks, SBO = byte distance of consecutive 8-row core matrices)
__device__ __forceinline__ unsigned long long tc_smem_desc(unsigned addr_bytes, unsigned lbo_bytes, unsigned sbo_bytes) {
  unsigned long long d = 0;
  d |= (unsigned long long)((addr_bytes >> 4) & 0x3fff);           // start address   bits [0,14)
  d |= (unsigned long long)((lbo_bytes >> 4) & 0x3fff) << 16;      // leading (K) byte offset  bits [16,30)
  d |= (unsigned long long)((sbo_bytes >> 4) & 0x3fff) << 32;      // stride (M/N) byte offset bits [32,46)
  return d;                                                         // base offset 0, layout type 0 (no swizzle)
}
// D(64 x 32, s32) += A(64 x 32, s8, smem) * B(32 x 32, s8, smem)^T
__device__ __forceinline__ void tc_wgmma_i8(int (&c)[16], unsigned long long adesc, unsigned long long bdesc) {
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "setp.ne.b32 p, %18, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n32k32.s32.s8.s8 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, %16, %17, p;\n"
      "}\n"
      : "+r"(c[0]), "+r"(c[1]), "+r"(c[2]), "+r"(c[3]), "+r"(c[4]), "+r"(c[5]), "+r"(c[6]), "+r"(c[7]), "+r"(c[8]), "+r"(c[9]),
        "+r"(c[10]), "+r"(c[11]), "+r"(c[12]), "+r"(c[13]), "+r"(c[14]), "+r"(c[15])
      : "l"(adesc), "l"(bdesc), "r"(1)
      : "memory");
}
__device__ __forceinline__ void tc_wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void tc_wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void tc_wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// keeps the accumulators in registers across the asynchronous MMAs (no spill / copy between issue and wait)
__device__ __forceinline__ void tc_fence_acc(int (&c)[16]) {
#pragma unroll
  for (int j = 0; j < 16; ++j) asm volatile("" : "+r"(c[j])::"memory");
}

// ------------------------------------------------------------------------------------------------
// the GEMM: one CTA per (front, 64 x 64) lower tile of the contribution block
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(TC_THREADS, 1) k_tc_schur(DevSym S, DevNum N, const TcFront* __restrict__ fronts,
                                                             const TcTile* __restrict__ tiles, const int8_t* __restrict__ dig,
                                                             const int* __restrict__ expo) {
  extern __shared__ __align__(1024) unsigned char tc_smem[];
  __shared__ unsigned long long full_bar[TC_STAGES], empty_bar[TC_STAGES];
  const TcTile T = tiles[blockIdx.x];
  const TcFront F = fronts[T.fi];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int nks = F.nks;

  if (threadIdx.x == 0) {
    for (int i = 0; i < TC_STAGES; ++i) { tc_mbar_init(&full_bar[i], 1); tc_mbar_init(&empty_bar[i], 2); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  if (warp == 8) {
    // ===== TMA producer: per K step one 16 KB unit of A digits and one 16 KB unit of B digits =====
    if (lane == 0) {
      const int8_t* a_src = dig + F.a_off + (long long)T.ti * nks * TC_A_UNIT;
      const int8_t* b_src = dig + F.b_off + (long long)T.tj * nks * TC_B_UNIT;
      for (int ks = 0; ks < nks; ++ks) {
        const int st = ks % TC_STAGES;
        const unsigned ph = (ks / TC_STAGES) & 1;
        tc_mbar_wait(&empty_bar[st], ph ^ 1);                       // consumers freed the slot (first pass: immediate)
        unsigned char* sa = tc_smem + (size_t)st * TC_STAGE_BYTES;
        tc_mbar_expect_tx(&full_bar[st], TC_STAGE_BYTES);
        tc_bulk_g2s(sa, a_src + (long long)ks * TC_A_UNIT, TC_A_UNIT, &full_bar[st]);
        tc_bulk_g2s(sa + TC_A_UNIT, b_src + (long long)ks * TC_B_UNIT, TC_B_UNIT, &full_bar[st]);
      }
    }
    return;
  }

  // ===== consumer warpgroup wg (warps 4wg .. 4wg+3): columns 32 wg .. 32 wg + 31 of the tile =====
  const int wg = warp >> 2;
  int acc[TC_NS][16];
#pragma unroll
  for (int d = 0; d < TC_NS; ++d)
#pragma unroll
    for (int j = 0; j < 16; ++j) acc[d][j] = 0;
  for (int ks = 0; ks < nks; ++ks) {
    const int st = ks % TC_STAGES;
    const unsigned ph = (ks / TC_STAGES) & 1;
    tc_mbar_wait(&full_bar[st], ph);
    const unsigned sa = tc_smem_u32(tc_smem + (size_t)st * TC_STAGE_BYTES);
    const unsigned sb = sa + TC_A_UNIT + wg * (TC_WN * 16);
    tc_wgmma_fence();
    // the 36 digit pairs (s, s'), s + s' < 8, into accumulator d = s + s'
#pragma unroll
    for (int d = 0; d < TC_NS; ++d) {
#pragma unroll
      for (int q = 0; q <= d; ++q) {
        // A digit q, B digit d - q ; within a unit: digit stride 2*rows*16 bytes, K-chunk (LBO) rows*16, 8-row group (SBO) 128
        const unsigned long long ad = tc_smem_desc(sa + q * (2 * TC_BM * 16), TC_BM * 16, 128);
        const unsigned long long bd = tc_smem_desc(sb + (d - q) * (2 * TC_BN * 16), TC_BN * 16, 128);
        tc_wgmma_i8(acc[d], ad, bd);
      }
    }
    tc_wgmma_commit();
#pragma unroll
    for (int d = 0; d < TC_NS; ++d) tc_fence_acc(acc[d]);
    // the previous K step's MMAs have read their slot once at most this step's group is in flight
    tc_wgmma_wait<1>();
    if (ks > 0 && (threadIdx.x & 127) == 0) tc_mbar_arrive(&empty_bar[(ks - 1) % TC_STAGES]);
  }
  tc_wgmma_wait<0>();
#pragma unroll
  for (int d = 0; d < TC_NS; ++d) tc_fence_acc(acc[d]);

  // ===== epilogue: accumulator fragment of m64n32 -- register 4i+h of a thread holds row 16 (warp % 4) + lane / 4 + 8 (h / 2),
  // column 8 i + 2 (lane % 4) + (h % 2) of the warpgroup's 64 x 32 block =====
  const int s = F.s;
  const int r = (int)(S.rows_ptr[s + 1] - S.rows_ptr[s]);
  const int* __restrict__ ea = expo + F.e_off;
  const int* __restrict__ eb = ea + r;
  double* __restrict__ C = N.CB + S.cb_off[s];
  const int gi0 = T.ti * TC_BM + 16 * (warp & 3) + (lane >> 2);
  const int gj0 = T.tj * TC_BN + wg * TC_WN + 2 * (lane & 3);
#pragma unroll
  for (int h2 = 0; h2 < 2; ++h2) {
    const int gi = gi0 + 8 * h2;
    if (gi >= r) continue;
    const int ei = ea[gi];
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int reg = 4 * (j >> 1) + 2 * h2 + (j & 1);
      double a = 0.0;
      // smallest weight first
#pragma unroll
      for (int d = TC_NS - 1; d >= 0; --d) a = fma((double)acc[d][reg], ldexp(1.0, -7 * (d + 2)), a);
      const int gj = gj0 + 8 * (j >> 1) + (j & 1);
      if (gj < r && gj <= gi) C[gi + (long long)gj * r] -= ldexp(a, ei + eb[gj]);
    }
  }
}

}  // namespace b200
