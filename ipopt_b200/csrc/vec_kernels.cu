// Device-resident dense-vector, expansion-matrix and triplet-SpMV kernels (C ABI: include/b200vec.h), sm_90a.
//
// Replaces the host loops of the reference's src/LinAlg on the interior-point hot path (SURVEY.md 8a rows V1-V9):
// IpDenseVector.cpp:93-1500, IpBlas.cpp:270-298, IpExpansionMatrix.cpp:27-372, TMatrices/IpGenTMatrix.cpp:46-130,
// TMatrices/IpSymTMatrix.cpp:46-110.  The host side of every entry point reproduces the reference's "homogeneous"
// (scalar) fast paths -- they decide the representation of the result -- and launches ONE fused kernel for the dense
// case.  All kernels are HBM-bound streams: 256-thread CTAs, grid-stride, grid = a multiple of the SM count.
//   * element-wise maps: explicit __dmul_rn/__dadd_rn/__ddiv_rn in the reference's operation order (nvcc would otherwise
//     contract a*b+c into an FMA and differ from the reference's x86 loops in the last bit);
//   * reductions: per-thread accumulation, warp-shuffle tree, shared-memory tree over the warps, per-CTA partials
//     combined by the last-arriving CTA in a fixed order (bit-reproducible); one D2H of 8 bytes per reduction.
#include "../../include/b200vec.h"

#include <cuda_runtime.h>

#include <algorithm>
#include <cfloat>
#include <cmath>
#include <cstdio>
#include <string>
#include <vector>

namespace b200v {

struct Ctx {
  int dev = 0;
  cudaStream_t st = nullptr;
  bool own = false;
  double* d_part = nullptr;     // per-CTA partials
  unsigned* d_cnt = nullptr;    // arrival counter of the reductions
  double* d_out = nullptr;
  double* h_out = nullptr;      // pinned
  int max_blocks = 1056;        // 132 SMs (H100 SXM) x 8 CTAs; set from the device in b200vec_create
  int64_t launches = 0;
  std::string err;
};

struct TMat {
  Ctx* c;
  int nrows, ncols, nnz, symmetric;
  // entries grouped by OUTPUT row in triplet order: for row i the contributions rptr[i]..rptr[i+1]; each refers to
  // triplet e = ent[q] and reads x at xcol[q] (0-based).  (for A^T x: same with the roles of rows and columns swapped)
  int *d_rptr = nullptr, *d_ent = nullptr, *d_xcol = nullptr;
  int *d_tptr = nullptr, *d_tent = nullptr, *d_txcol = nullptr;
};

#define VCU(call)                                                                    \
  do {                                                                               \
    cudaError_t e__ = (call);                                                        \
    if (e__ != cudaSuccess) { c->err = std::string(#call) + ": " + cudaGetErrorString(e__); return 4; } \
  } while (0)

static inline int grid_for(const Ctx* c, long long n) { return (int)std::max<long long>(1, std::min<long long>((n + 255) / 256, c->max_blocks)); }

// ---------------------------------------------------------------------------------------------------------------
// element-wise kernels.  OP codes select the loop body; a and b are the scalars of the call.
// ---------------------------------------------------------------------------------------------------------------
enum {
  U_SCAL, U_ADDS, U_RECIP, U_ABS, U_SQRT, U_SGN, U_FILL, U_DIVS, U_MULS, U_MAXS, U_MINS, U_SELS,
  B_COPY, B_AXPY, B_HAXPY /* y = a + b x */, B_DIV, B_RDIV /* y = a / x */, B_MUL, B_MULH /* y = a x */, B_SEL, B_SELH,
  B_MAX, B_MAXH, B_MIN, B_MINH
};

template <int OP>
__global__ void __launch_bounds__(256) k_unary(int n, double* __restrict__ y, double a) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const double v = (OP == U_FILL) ? 0.0 : y[i];
    double r;
    if (OP == U_SCAL) r = __dmul_rn(a, v);
    else if (OP == U_ADDS) r = __dadd_rn(v, __dmul_rn(1.0, a));   // IpBlasAxpy(1., &scalar, 0, ...): *y += alpha * *x
    else if (OP == U_RECIP) r = __ddiv_rn(1.0, v);
    else if (OP == U_ABS) r = fabs(v);
    else if (OP == U_SQRT) r = __dsqrt_rn(v);
    else if (OP == U_SGN) r = (v > 0.0) ? 1.0 : ((v < 0.0) ? -1.0 : 0.0);
    else if (OP == U_FILL) r = a;
    else if (OP == U_DIVS) r = __ddiv_rn(v, a);
    else if (OP == U_MULS) r = __dmul_rn(v, a);
    else if (OP == U_MAXS) r = (v > a) ? v : a;                    // Ipopt::Max(a,b) = a > b ? a : b  (IpUtils.hpp)
    else if (OP == U_MINS) r = (v < a) ? v : a;
    else /* U_SELS */ r = (v > 0.0) ? a : ((v < 0.0) ? -a : v);
    y[i] = r;
  }
}

template <int OP>
__global__ void __launch_bounds__(256) k_binary(int n, const double* __restrict__ x, double* __restrict__ y, double a, double b) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const double xv = x[i];
    const double yv = (OP == B_COPY || OP == B_HAXPY || OP == B_RDIV || OP == B_MULH || OP == B_MAXH || OP == B_MINH || OP == B_SELH) ? 0.0 : y[i];
    double r;
    if (OP == B_COPY) r = xv;
    else if (OP == B_AXPY) r = fma(a, xv, yv);                     // BLAS daxpy (the reference's OpenBLAS kernels are FMA kernels)
    else if (OP == B_HAXPY) r = __dadd_rn(a, __dmul_rn(b, xv));    // vals[i] = scalar_ + alpha * x[i]
    else if (OP == B_DIV) r = __ddiv_rn(yv, xv);
    else if (OP == B_RDIV) r = __ddiv_rn(a, xv);
    else if (OP == B_MUL) r = __dmul_rn(yv, xv);
    else if (OP == B_MULH) r = __dmul_rn(a, xv);
    else if (OP == B_SEL) r = (yv > 0.0) ? xv : ((yv < 0.0) ? -xv : yv);
    else if (OP == B_MAX) r = (yv > xv) ? yv : xv;
    else if (OP == B_MAXH) r = (a > xv) ? a : xv;
    else if (OP == B_MIN) r = (yv < xv) ? yv : xv;
    else /* B_MINH */ r = (a < xv) ? a : xv;
    y[i] = r;
  }
}

// y = a v1 + b v2 + c y with the reference's special-cased loop bodies (a, b in {0, 1, -1, other}; c in {0, other}):
// the code (ca, cb) picks the expression, so e.g. a == 1 adds v1 without a multiply exactly like the reference.
__device__ __forceinline__ double a2v_term(int code, double coef, double v) {
  return code == 1 ? v : (code == 2 ? -v : __dmul_rn(coef, v));
}
__global__ void __launch_bounds__(256) k_add_two(int n, int ca, double a, const double* __restrict__ v1, int cb, double b,
                                                 const double* __restrict__ v2, int cc, double c, double* __restrict__ y) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    // reference order: ((a v1 [+-] b v2) + c y); with c == -1 the reference writes  "... - values_[i]"
    double r = 0.0;
    bool have = false;
    if (ca != 0) { r = a2v_term(ca, a, v1[i]); have = true; }
    if (cb != 0) {
      const double v = v2[i];
      if (!have) { r = a2v_term(cb, b, v); have = true; }
      else r = (cb == 1) ? __dadd_rn(r, v) : ((cb == 2) ? __dadd_rn(r, -v) : __dadd_rn(r, __dmul_rn(b, v)));
    }
    if (cc != 0) {
      const double yv = y[i];
      const double t = (cc == 1) ? yv : ((cc == 2) ? -yv : __dmul_rn(c, yv));
      r = have ? __dadd_rn(r, t) : t;
    } else if (!have) r = 0.0;
    y[i] = r;
  }
}

// y = a z / s + c y   (modes pick the homogeneous operands; expression order as in the reference)
// zmode/smode: 0 = dense, 1 = scalar ; ymode: 0 = c == 0, 1 = y homogeneous (val = c*scalar precomputed), 2 = dense
__global__ void __launch_bounds__(256) k_add_quot(int n, double a, const double* __restrict__ z, int zmode, double zs,
                                                  const double* __restrict__ s, int smode, double ss, int ymode, double c,
                                                  double val, double* __restrict__ y) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    double q;
    if (zmode == 1 && smode == 1) q = __ddiv_rn(__dmul_rn(a, zs), ss);
    else if (zmode == 1) q = __ddiv_rn(__dmul_rn(a, zs), s[i]);            // a * z_scalar / s[i]
    else if (smode == 1) q = __ddiv_rn(__dmul_rn(z[i], a), ss);            // z[i] * a / s_scalar
    else q = __ddiv_rn(__dmul_rn(a, z[i]), s[i]);                          // a * z[i] / s[i]
    double r;
    if (ymode == 0) r = q;
    else if (ymode == 1) r = __dadd_rn(val, q);
    else r = __dadd_rn(__dmul_rn(c, y[i]), q);
    y[i] = r;
  }
}

// ---------------------------------------------------------------------------------------------------------------
// reductions
// ---------------------------------------------------------------------------------------------------------------
enum { R_DOT, R_DOTS /* sum a*x */, R_SUMSQ, R_ASUM, R_AMAX, R_MAX, R_MIN, R_SUM, R_SUMLOG, R_FTB, R_FTB_HX, R_FTB_HD };

template <int OP>
__device__ __forceinline__ double red_identity() {
  if (OP == R_MAX) return -DBL_MAX;
  if (OP == R_MIN) return DBL_MAX;
  if (OP == R_FTB || OP == R_FTB_HX || OP == R_FTB_HD) return 1.0;
  return 0.0;
}
template <int OP>
__device__ __forceinline__ double red_combine(double u, double v) {
  if (OP == R_AMAX || OP == R_MAX) return fmax(u, v);
  if (OP == R_MIN || OP == R_FTB || OP == R_FTB_HX || OP == R_FTB_HD) return fmin(u, v);
  return u + v;
}
template <int OP>
__device__ __forceinline__ double red_term(const double* __restrict__ x, const double* __restrict__ y, int i, double a, double b) {
  if (OP == R_DOT) return x[i] * y[i];
  if (OP == R_DOTS) return a * x[i];
  if (OP == R_SUMSQ) { const double v = x[i] * a; return v * v; }
  if (OP == R_ASUM || OP == R_AMAX) return fabs(x[i]);
  if (OP == R_MAX || OP == R_MIN || OP == R_SUM) return x[i];
  if (OP == R_SUMLOG) return log(x[i]);
  // FracToBound: alpha = min(alpha, -tau / delta_i * x_i) where delta_i < 0   (a = tau, y = delta, b = homogeneous scalar)
  if (OP == R_FTB) { const double d = y[i]; return d < 0.0 ? __dmul_rn(__ddiv_rn(-a, d), x[i]) : 1.0; }
  if (OP == R_FTB_HX) { const double d = y[i]; return d < 0.0 ? __dmul_rn(__ddiv_rn(-a, d), b) : 1.0; }   // x homogeneous (= b)
  /* R_FTB_HD: delta homogeneous (= b < 0) */ return __dmul_rn(__ddiv_rn(-a, b), x[i]);
}

template <int OP>
__global__ void __launch_bounds__(256) k_reduce(int n, const double* __restrict__ x, const double* __restrict__ y, double a,
                                                double b, double* __restrict__ part, unsigned* __restrict__ cnt,
                                                double* __restrict__ out) {
  __shared__ double sh[8];
  __shared__ bool last;
  double acc = red_identity<OP>();
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x)
    acc = red_combine<OP>(acc, red_term<OP>(x, y, i, a, b));
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) acc = red_combine<OP>(acc, __shfl_xor_sync(0xffffffffu, acc, o));
  if (lane == 0) sh[warp] = acc;
  __syncthreads();
  if (warp == 0) {
    acc = (lane < 8) ? sh[lane] : red_identity<OP>();
#pragma unroll
    for (int o = 4; o > 0; o >>= 1) acc = red_combine<OP>(acc, __shfl_xor_sync(0xffffffffu, acc, o));
    if (lane == 0) {
      part[blockIdx.x] = acc;
      __threadfence();
      const unsigned old = atomicInc(cnt, gridDim.x - 1);   // wraps to 0 after the last CTA: no reset needed
      last = (old == gridDim.x - 1);
    }
  }
  __syncthreads();
  if (!last) return;
  __threadfence();
  // the last CTA combines the partials in a fixed order: thread t takes t, t+256, ...; then the same tree as above
  acc = red_identity<OP>();
  for (int i = threadIdx.x; i < (int)gridDim.x; i += blockDim.x) acc = red_combine<OP>(acc, __ldcg(part + i));
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) acc = red_combine<OP>(acc, __shfl_xor_sync(0xffffffffu, acc, o));
  __syncthreads();
  if (lane == 0) sh[warp] = acc;
  __syncthreads();
  if (warp == 0) {
    acc = (lane < 8) ? sh[lane] : red_identity<OP>();
#pragma unroll
    for (int o = 4; o > 0; o >>= 1) acc = red_combine<OP>(acc, __shfl_xor_sync(0xffffffffu, acc, o));
    if (lane == 0) *out = acc;
  }
}

// ---------------------------------------------------------------------------------------------------------------
// expansion matrix (exp_pos is injective: scatter without conflicts)
// ---------------------------------------------------------------------------------------------------------------
// mode 0: y[p[i]] += alpha x[i] (acode: 1 -> +x, 2 -> -x, 3 -> alpha*x) ; mode 1: y[p[i]] += val (x homogeneous)
__global__ void __launch_bounds__(256) k_exp_mult(int ncols, const int* __restrict__ p, int acode, double alpha,
                                                  const double* __restrict__ x, int xh, double val, double* __restrict__ y) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < ncols; i += gridDim.x * blockDim.x) {
    const int t = p[i];
    const double yv = y[t];
    double r;
    if (xh) r = __dadd_rn(yv, val);
    else if (acode == 1) r = __dadd_rn(yv, x[i]);
    else if (acode == 2) r = __dadd_rn(yv, -x[i]);
    else r = __dadd_rn(yv, __dmul_rn(alpha, x[i]));
    y[t] = r;
  }
}
__global__ void __launch_bounds__(256) k_exp_transmult(int ncols, const int* __restrict__ p, int acode, double alpha,
                                                       const double* __restrict__ x, int xh, double val, double* __restrict__ y) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < ncols; i += gridDim.x * blockDim.x) {
    const double yv = y[i];
    double r;
    if (xh) r = __dadd_rn(yv, val);
    else if (acode == 1) r = __dadd_rn(yv, x[p[i]]);
    else if (acode == 2) r = __dadd_rn(yv, -x[p[i]]);
    else r = __dadd_rn(yv, __dmul_rn(alpha, x[p[i]]));
    y[i] = r;
  }
}
// X[p[i]] += alpha Z[i] / S[i]
__global__ void __launch_bounds__(256) k_exp_msinvz(int ncols, const int* __restrict__ p, int acode, double alpha,
                                                    const double* __restrict__ S, const double* __restrict__ Z, int zh,
                                                    double val, double* __restrict__ X) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < ncols; i += gridDim.x * blockDim.x) {
    const int t = p[i];
    const double xv = X[t], s = S[i];
    double r;
    if (zh) r = __dadd_rn(xv, __ddiv_rn(val, s));
    else if (acode == 1) r = __dadd_rn(xv, __ddiv_rn(Z[i], s));
    else if (acode == 2) r = __dadd_rn(xv, -__ddiv_rn(Z[i], s));
    else r = __dadd_rn(xv, __ddiv_rn(__dmul_rn(alpha, Z[i]), s));   // alpha * Z[i] / S[i]
    X[t] = r;
  }
}
// X[i] = (R[i] + alpha Z[i] D[p[i]]) / S[i]
__global__ void __launch_bounds__(256) k_exp_sinv(int ncols, const int* __restrict__ p, int acode, double alpha,
                                                  const double* __restrict__ S, const double* __restrict__ R, int rh, double rs,
                                                  const double* __restrict__ Z, int zh, double val,
                                                  const double* __restrict__ D, double* __restrict__ X) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < ncols; i += gridDim.x * blockDim.x) {
    const double rv = rh ? rs : R[i];
    double num;
    if (zh) {
      if (rh && val == 0.0) num = rv;
      else num = __dadd_rn(rv, __dmul_rn(val, D[p[i]]));
    } else if (acode == 1) num = __dadd_rn(rv, __dmul_rn(Z[i], D[p[i]]));
    else if (acode == 2) num = __dadd_rn(rv, -__dmul_rn(Z[i], D[p[i]]));
    else num = __dadd_rn(rv, __dmul_rn(__dmul_rn(alpha, Z[i]), D[p[i]]));   // alpha * Z[i] * D[...]
    X[i] = __ddiv_rn(num, S[i]);
  }
}

// ---------------------------------------------------------------------------------------------------------------
// triplet SpMV: one thread per output row, contributions in triplet order (same order as the reference's loop)
// ---------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) k_tmat_mult(int nrows, const int* __restrict__ rptr, const int* __restrict__ ent,
                                                   const int* __restrict__ xcol, const double* __restrict__ vals,
                                                   double alpha, const double* __restrict__ x, int xh, double as,
                                                   double* __restrict__ y) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < nrows; i += gridDim.x * blockDim.x) {
    double acc = y[i];
    for (int q = rptr[i]; q < rptr[i + 1]; ++q) {
      const double v = vals[ent[q]];
      acc = xh ? __dadd_rn(acc, __dmul_rn(as, v)) : __dadd_rn(acc, __dmul_rn(__dmul_rn(alpha, v), x[xcol[q]]));
    }
    y[i] = acc;
  }
}

}  // namespace b200v

using namespace b200v;

// ===============================================================================================================
extern "C" {

b200vec_ctx b200vec_create(int device, void* stream) {
  int ndev = 0;
  cudaError_t e = cudaGetDeviceCount(&ndev);
  if (e != cudaSuccess || ndev == 0) {
    fprintf(stderr, "[b200vec] FATAL: no usable CUDA device (%s); there is no CPU fallback\n",
            e != cudaSuccess ? cudaGetErrorString(e) : "device count is 0");
    return nullptr;
  }
  Ctx* c = new Ctx();
  if (device >= 0) c->dev = device; else cudaGetDevice(&c->dev);
  if (cudaSetDevice(c->dev) != cudaSuccess) { delete c; return nullptr; }
  if (stream) c->st = (cudaStream_t)stream;
  else { cudaStreamCreateWithFlags(&c->st, cudaStreamNonBlocking); c->own = true; }
  int sms = 132;
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, c->dev);
  c->max_blocks = sms * 8;
  cudaMalloc((void**)&c->d_part, c->max_blocks * sizeof(double));
  cudaMalloc((void**)&c->d_cnt, sizeof(unsigned));
  cudaMalloc((void**)&c->d_out, sizeof(double));
  cudaMemset(c->d_cnt, 0, sizeof(unsigned));
  cudaHostAlloc((void**)&c->h_out, sizeof(double), cudaHostAllocDefault);
  return (b200vec_ctx)c;
}

void b200vec_destroy(b200vec_ctx cc) {
  Ctx* c = (Ctx*)cc;
  if (!c) return;
  cudaSetDevice(c->dev);
  cudaStreamSynchronize(c->st);
  cudaFree(c->d_part); cudaFree(c->d_cnt); cudaFree(c->d_out); cudaFreeHost(c->h_out);
  if (c->own) cudaStreamDestroy(c->st);
  delete c;
}

const char* b200vec_last_error(b200vec_ctx cc) { return cc ? ((Ctx*)cc)->err.c_str() : "null context"; }
int64_t b200vec_launches(b200vec_ctx cc) { return cc ? ((Ctx*)cc)->launches : 0; }
int b200vec_sync(b200vec_ctx cc) {
  Ctx* c = (Ctx*)cc;
  if (!c) return 4;
  VCU(cudaSetDevice(c->dev));
  VCU(cudaStreamSynchronize(c->st));
  return 0;
}

}  // extern "C"

namespace b200v {

template <int OP>
static int unary(Ctx* c, b200vec* y, double a) {
  if (y->n <= 0) return 0;
  k_unary<OP><<<grid_for(c, y->n), 256, 0, c->st>>>(y->n, y->d, a);
  ++c->launches;
  VCU(cudaGetLastError());
  return 0;
}
template <int OP>
static int binary(Ctx* c, const double* x, b200vec* y, double a, double b) {
  if (y->n <= 0) return 0;
  k_binary<OP><<<grid_for(c, y->n), 256, 0, c->st>>>(y->n, x, y->d, a, b);
  ++c->launches;
  VCU(cudaGetLastError());
  return 0;
}
template <int OP>
static int reduce(Ctx* c, int n, const double* x, const double* y, double a, double b, double* out) {
  k_reduce<OP><<<grid_for(c, n), 256, 0, c->st>>>(n, x, y, a, b, c->d_part, c->d_cnt, c->d_out);
  ++c->launches;
  VCU(cudaGetLastError());
  VCU(cudaMemcpyAsync(c->h_out, c->d_out, sizeof(double), cudaMemcpyDeviceToHost, c->st));
  VCU(cudaStreamSynchronize(c->st));
  *out = *c->h_out;
  return 0;
}
static inline int coef_code(double v) { return v == 0.0 ? 0 : (v == 1.0 ? 1 : (v == -1.0 ? 2 : 3)); }

}  // namespace b200v

#define CTX Ctx* c = (Ctx*)cc; if (!c) return 4; if (cudaSetDevice(c->dev) != cudaSuccess) return 4

extern "C" {

// ---- V3 ------------------------------------------------------------------------------------------------------
int b200vec_copy(b200vec_ctx cc, const b200vec* x, b200vec* y) {   // CopyImpl :93-113
  CTX;
  if (x->n != y->n) { c->err = "copy: dimension mismatch"; return 4; }
  y->homogeneous = x->homogeneous;
  if (x->homogeneous) { y->scalar = x->scalar; return 0; }
  return binary<B_COPY>(c, x->d, y, 0.0, 0.0);
}
int b200vec_scal(b200vec_ctx cc, double alpha, b200vec* y) {       // ScalImpl :115-128
  CTX;
  if (y->homogeneous) { y->scalar *= alpha; return 0; }
  return unary<U_SCAL>(c, y, alpha);
}
int b200vec_set(b200vec_ctx cc, double alpha, b200vec* y) {        // SetImpl :263-276
  CTX;
  y->homogeneous = 1; y->scalar = alpha;
  return 0;
}
int b200vec_add_scalar(b200vec_ctx cc, double scalar, b200vec* y) {   // AddScalarImpl :618-631
  CTX;
  if (y->homogeneous) { y->scalar += scalar; return 0; }
  return unary<U_ADDS>(c, y, scalar);
}
// ---- V1 ------------------------------------------------------------------------------------------------------
int b200vec_axpy(b200vec_ctx cc, double alpha, const b200vec* x, b200vec* y) {   // AxpyImpl :130-177
  CTX;
  if (x->n != y->n) { c->err = "axpy: dimension mismatch"; return 4; }
  if (y->n == 0) return 0;
  if (y->homogeneous) {
    if (x->homogeneous) { y->scalar += alpha * x->scalar; return 0; }
    y->homogeneous = 0;
    return binary<B_HAXPY>(c, x->d, y, y->scalar, alpha);
  }
  if (x->homogeneous) {
    if (x->scalar != 0.0) return unary<U_ADDS>(c, y, alpha * x->scalar);   // *y += alpha * *x  (IpBlas.cpp:284-289)
    return 0;
  }
  return binary<B_AXPY>(c, x->d, y, alpha, 0.0);
}
// ---- V2 ------------------------------------------------------------------------------------------------------
int b200vec_dot(b200vec_ctx cc, const b200vec* x, const b200vec* y, double* out) {   // DotImpl :179-219 (this = y)
  CTX;
  if (x->n != y->n) { c->err = "dot: dimension mismatch"; return 4; }
  if (y->n == 0) { *out = 0.0; return 0; }
  if (y->homogeneous && x->homogeneous) { *out = y->n * y->scalar * x->scalar; return 0; }
  if (y->homogeneous) return reduce<R_DOTS>(c, x->n, x->d, nullptr, y->scalar, 0.0, out);
  if (x->homogeneous) return reduce<R_DOTS>(c, y->n, y->d, nullptr, x->scalar, 0.0, out);
  return reduce<R_DOT>(c, y->n, x->d, y->d, 0.0, 0.0, out);
}
int b200vec_nrm2(b200vec_ctx cc, const b200vec* x, double* out) {   // Nrm2Impl :221-232
  CTX;
  if (x->homogeneous) { *out = std::sqrt((double)x->n) * std::fabs(x->scalar); return 0; }
  if (x->n == 0) { *out = 0.0; return 0; }
  // plain sum of squares first; only if that over/underflowed, the scaled two-pass form of BLAS dnrm2
  double ss = 0.0;
  int rc = reduce<R_SUMSQ>(c, x->n, x->d, nullptr, 1.0, 0.0, &ss);
  if (rc) return rc;
  if (std::isfinite(ss) && ss > 1e-280) { *out = std::sqrt(ss); return 0; }
  double amax = 0.0;
  rc = reduce<R_AMAX>(c, x->n, x->d, nullptr, 0.0, 0.0, &amax);
  if (rc) return rc;
  if (!(amax > 0.0) || !std::isfinite(amax)) { *out = amax; return 0; }
  rc = reduce<R_SUMSQ>(c, x->n, x->d, nullptr, 1.0 / amax, 0.0, &ss);   // sum (x_i / amax)^2
  *out = amax * std::sqrt(ss);
  return rc;
}
int b200vec_asum(b200vec_ctx cc, const b200vec* x, double* out) {   // AsumImpl :234-245
  CTX;
  if (x->homogeneous) { *out = x->n * std::fabs(x->scalar); return 0; }
  if (x->n == 0) { *out = 0.0; return 0; }
  return reduce<R_ASUM>(c, x->n, x->d, nullptr, 0.0, 0.0, out);
}
int b200vec_amax(b200vec_ctx cc, const b200vec* x, double* out) {   // AmaxImpl :247-261
  CTX;
  if (x->n == 0) { *out = 0.0; return 0; }
  if (x->homogeneous) { *out = std::fabs(x->scalar); return 0; }
  return reduce<R_AMAX>(c, x->n, x->d, nullptr, 0.0, 0.0, out);
}
int b200vec_max(b200vec_ctx cc, const b200vec* x, double* out) {    // MaxImpl :633-655
  CTX;
  if (x->n == 0) { *out = -DBL_MAX; return 0; }
  if (x->homogeneous) { *out = x->scalar; return 0; }
  return reduce<R_MAX>(c, x->n, x->d, nullptr, 0.0, 0.0, out);
}
int b200vec_min(b200vec_ctx cc, const b200vec* x, double* out) {    // MinImpl :657-679
  CTX;
  if (x->n == 0) { *out = DBL_MAX; return 0; }
  if (x->homogeneous) { *out = x->scalar; return 0; }
  return reduce<R_MIN>(c, x->n, x->d, nullptr, 0.0, 0.0, out);
}
int b200vec_sum(b200vec_ctx cc, const b200vec* x, double* out) {    // SumImpl :681-698
  CTX;
  if (x->homogeneous) { *out = x->n * x->scalar; return 0; }
  if (x->n == 0) { *out = 0.0; return 0; }
  return reduce<R_SUM>(c, x->n, x->d, nullptr, 0.0, 0.0, out);
}
int b200vec_sumlogs(b200vec_ctx cc, const b200vec* x, double* out) {   // SumLogsImpl :700-721
  CTX;
  if (x->n == 0) { *out = 0.0; return 0; }
  if (x->homogeneous) { *out = x->n * std::log(x->scalar); return 0; }
  return reduce<R_SUMLOG>(c, x->n, x->d, nullptr, 0.0, 0.0, out);
}
// ---- V4 ------------------------------------------------------------------------------------------------------
int b200vec_ew_divide(b200vec_ctx cc, const b200vec* x, b200vec* y) {   // :278-327
  CTX;
  if (x->n != y->n) { c->err = "ew_divide: dimension mismatch"; return 4; }
  if (y->n == 0) return 0;
  if (y->homogeneous) {
    if (x->homogeneous) { y->scalar /= x->scalar; return 0; }
    y->homogeneous = 0;
    return binary<B_RDIV>(c, x->d, y, y->scalar, 0.0);
  }
  if (x->homogeneous) return unary<U_DIVS>(c, y, x->scalar);
  return binary<B_DIV>(c, x->d, y, 0.0, 0.0);
}
int b200vec_ew_multiply(b200vec_ctx cc, const b200vec* x, b200vec* y) {   // :329-383
  CTX;
  if (x->n != y->n) { c->err = "ew_multiply: dimension mismatch"; return 4; }
  if (y->n == 0) return 0;
  if (y->homogeneous) {
    if (x->homogeneous) { y->scalar *= x->scalar; return 0; }
    y->homogeneous = 0;
    return binary<B_MULH>(c, x->d, y, y->scalar, 0.0);
  }
  if (x->homogeneous) { if (x->scalar != 1.0) return unary<U_MULS>(c, y, x->scalar); return 0; }
  return binary<B_MUL>(c, x->d, y, 0.0, 0.0);
}
int b200vec_ew_select(b200vec_ctx cc, const b200vec* x, b200vec* y) {   // :385-457
  CTX;
  if (x->n != y->n) { c->err = "ew_select: dimension mismatch"; return 4; }
  if (y->n == 0) return 0;
  if (y->homogeneous) {
    if (y->scalar == 0.0) return 0;
    if (x->homogeneous) { y->scalar *= x->scalar; return 0; }
    y->homogeneous = 0;
    return binary<B_MULH>(c, x->d, y, y->scalar, 0.0);   // vals[i] = scalar_ * values_x[i]
  }
  if (x->homogeneous) { if (x->scalar != 1.0) return unary<U_SELS>(c, y, x->scalar); return 0; }
  return binary<B_SEL>(c, x->d, y, 0.0, 0.0);
}
int b200vec_ew_max(b200vec_ctx cc, const b200vec* x, b200vec* y) {   // :459-505
  CTX;
  if (x->n != y->n) { c->err = "ew_max: dimension mismatch"; return 4; }
  if (y->n == 0) return 0;
  if (y->homogeneous) {
    if (x->homogeneous) { y->scalar = (y->scalar > x->scalar) ? y->scalar : x->scalar; return 0; }
    y->homogeneous = 0;
    return binary<B_MAXH>(c, x->d, y, y->scalar, 0.0);
  }
  if (x->homogeneous) return unary<U_MAXS>(c, y, x->scalar);
  return binary<B_MAX>(c, x->d, y, 0.0, 0.0);
}
int b200vec_ew_min(b200vec_ctx cc, const b200vec* x, b200vec* y) {   // :507-553
  CTX;
  if (x->n != y->n) { c->err = "ew_min: dimension mismatch"; return 4; }
  if (y->n == 0) return 0;
  if (y->homogeneous) {
    if (x->homogeneous) { y->scalar = (y->scalar < x->scalar) ? y->scalar : x->scalar; return 0; }
    y->homogeneous = 0;
    return binary<B_MINH>(c, x->d, y, y->scalar, 0.0);
  }
  if (x->homogeneous) return unary<U_MINS>(c, y, x->scalar);
  return binary<B_MIN>(c, x->d, y, 0.0, 0.0);
}
int b200vec_ew_reciprocal(b200vec_ctx cc, b200vec* y) {   // :555-574
  CTX;
  if (y->n == 0) return 0;
  if (y->homogeneous) { y->scalar = 1.0 / y->scalar; return 0; }
  return unary<U_RECIP>(c, y, 0.0);
}
int b200vec_ew_abs(b200vec_ctx cc, b200vec* y) {          // :576-590
  CTX;
  if (y->homogeneous) { y->scalar = std::fabs(y->scalar); return 0; }
  return unary<U_ABS>(c, y, 0.0);
}
int b200vec_ew_sqrt(b200vec_ctx cc, b200vec* y) {         // :592-606
  CTX;
  if (y->homogeneous) { y->scalar = std::sqrt(y->scalar); return 0; }
  return unary<U_SQRT>(c, y, 0.0);
}
int b200vec_ew_sgn(b200vec_ctx cc, b200vec* y) {          // :723-759
  CTX;
  if (y->homogeneous) { y->scalar = y->scalar > 0.0 ? 1.0 : (y->scalar < 0.0 ? -1.0 : 0.0); return 0; }
  return unary<U_SGN>(c, y, 0.0);
}
// ---- V5 ------------------------------------------------------------------------------------------------------
int b200vec_add_two_vectors(b200vec_ctx cc, double a, const b200vec* v1, double b, const b200vec* v2, double cv, b200vec* y) {
  CTX;   // AddTwoVectorsImpl :762-1322
  if (y->n == 0) return 0;
  const bool h1 = (a != 0.0) && v1->homogeneous, h2 = (b != 0.0) && v2->homogeneous;
  const double s1 = h1 ? v1->scalar : 0.0, s2 = h2 ? v2->scalar : 0.0;
  if ((a != 0.0 && v1->n != y->n) || (b != 0.0 && v2->n != y->n)) { c->err = "add_two_vectors: dimension mismatch"; return 4; }
  if ((cv == 0.0 || y->homogeneous) && h1 && h2) {
    double val = 0.0;
    if (cv != 0.0) val = cv * y->scalar;
    y->homogeneous = 1;
    y->scalar = val + a * s1 + b * s2;
    return 0;
  }
  if (cv == 0.0) y->homogeneous = 0;
  if (y->homogeneous || h1 || h2) {
    // Vector::AddTwoVectorsImpl (IpVector.cpp:45-113): composed from Copy / Scal / Axpy / Set
    int rc = 0;
    if (cv == 0.0) {
      if (a == 1.0) { rc = b200vec_copy(cc, v1, y); if (!rc && b != 0.0) rc = b200vec_axpy(cc, b, v2, y); }
      else if (a == 0.0) {
        if (b == 0.0) rc = b200vec_set(cc, 0.0, y);
        else { rc = b200vec_copy(cc, v2, y); if (!rc && b != 1.0) rc = b200vec_scal(cc, b, y); }
      } else {
        if (b == 1.0) { rc = b200vec_copy(cc, v2, y); if (!rc) rc = b200vec_axpy(cc, a, v1, y); }
        else if (b == 0.0) { rc = b200vec_copy(cc, v1, y); if (!rc) rc = b200vec_scal(cc, a, y); }
        else { rc = b200vec_copy(cc, v1, y); if (!rc) rc = b200vec_scal(cc, a, y); if (!rc) rc = b200vec_axpy(cc, b, v2, y); }
      }
    } else {
      if (cv != 1.0) rc = b200vec_scal(cc, cv, y);
      if (!rc && a != 0.0) rc = b200vec_axpy(cc, a, v1, y);
      if (!rc && b != 0.0) rc = b200vec_axpy(cc, b, v2, y);
    }
    return rc;
  }
  // all dense: one fused kernel with the reference's special-cased expressions
  const int ccode = coef_code(cv);   // the reference distinguishes c == 1 (adds y), c == -1 (subtracts y), general c
  k_add_two<<<grid_for(c, y->n), 256, 0, c->st>>>(y->n, coef_code(a), a, a != 0.0 ? v1->d : nullptr, coef_code(b), b,
                                                  b != 0.0 ? v2->d : nullptr, ccode, cv, y->d);
  ++c->launches;
  VCU(cudaGetLastError());
  return 0;
}
// ---- V6 ------------------------------------------------------------------------------------------------------
int b200vec_frac_to_bound(b200vec_ctx cc, const b200vec* x, const b200vec* delta, double tau, double* out) {   // :1324-1389
  CTX;
  if (x->n != delta->n) { c->err = "frac_to_bound: dimension mismatch"; return 4; }
  if (x->n == 0) { *out = 1.0; return 0; }
  if (x->homogeneous) {
    if (delta->homogeneous) {
      double alpha = 1.0;
      if (delta->scalar < 0.0) alpha = std::min(alpha, -tau / delta->scalar * x->scalar);
      *out = alpha;
      return 0;
    }
    return reduce<R_FTB_HX>(c, x->n, nullptr, delta->d, tau, x->scalar, out);
  }
  if (delta->homogeneous) {
    if (!(delta->scalar < 0.0)) { *out = 1.0; return 0; }
    return reduce<R_FTB_HD>(c, x->n, x->d, nullptr, tau, delta->scalar, out);
  }
  return reduce<R_FTB>(c, x->n, x->d, delta->d, tau, 0.0, out);
}
// ---- V7 ------------------------------------------------------------------------------------------------------
int b200vec_add_vector_quotient(b200vec_ctx cc, double a, const b200vec* z, const b200vec* s, double cv, b200vec* y) {   // :1391-1540
  CTX;
  if (z->n != y->n || s->n != y->n) { c->err = "add_vector_quotient: dimension mismatch"; return 4; }
  if (y->n == 0) return 0;
  const bool hz = z->homogeneous, hs = s->homogeneous;
  if ((cv == 0.0 || y->homogeneous) && hz && hs) {
    if (cv == 0.0) y->scalar = a * z->scalar / s->scalar;
    else y->scalar = cv * y->scalar + a * z->scalar / s->scalar;
    y->homogeneous = 1;
    return 0;
  }
  int ymode = 2;
  double val = 0.0;
  if (cv == 0.0) ymode = 0;
  else if (y->homogeneous) { ymode = 1; val = cv * y->scalar; }
  k_add_quot<<<grid_for(c, y->n), 256, 0, c->st>>>(y->n, a, z->d, hz ? 1 : 0, z->scalar, s->d, hs ? 1 : 0, s->scalar, ymode,
                                                   cv, val, y->d);
  ++c->launches;
  VCU(cudaGetLastError());
  y->homogeneous = 0;
  return 0;
}

// ---- V8 ------------------------------------------------------------------------------------------------------
static int exp_prepare_y(b200vec_ctx cc, double beta, b200vec* y) {
  // "if (beta != 0) y.Scal(beta) else y.Set(0)" -- then the result is written into dense storage
  Ctx* c = (Ctx*)cc;
  int rc;
  if (beta != 0.0) rc = b200vec_scal(cc, beta, y); else rc = b200vec_set(cc, 0.0, y);
  if (rc) return rc;
  if (y->homogeneous) {   // dense_y->Values(): materialise the homogeneous value
    y->homogeneous = 0;
    rc = unary<U_FILL>(c, y, y->scalar);
  }
  return rc;
}
int b200vec_exp_mult(b200vec_ctx cc, int nrows, int ncols, const int* exp_pos, double alpha, const b200vec* x, double beta, b200vec* y) {
  CTX;   // MultVectorImpl :27-96
  if (x->n != ncols || y->n != nrows) { c->err = "exp_mult: dimension mismatch"; return 4; }
  int rc = exp_prepare_y(cc, beta, y);
  if (rc || ncols == 0) return rc;
  const double val = x->homogeneous ? alpha * x->scalar : 0.0;
  if (x->homogeneous && val == 0.0) return 0;
  k_exp_mult<<<grid_for(c, ncols), 256, 0, c->st>>>(ncols, exp_pos, alpha == 1.0 ? 1 : (alpha == -1.0 ? 2 : 3), alpha, x->d,
                                                    x->homogeneous, val, y->d);
  ++c->launches;
  VCU(cudaGetLastError());
  return 0;
}
int b200vec_exp_transmult(b200vec_ctx cc, int nrows, int ncols, const int* exp_pos, double alpha, const b200vec* x, double beta, b200vec* y) {
  CTX;   // TransMultVectorImpl :98-167
  if (x->n != nrows || y->n != ncols) { c->err = "exp_transmult: dimension mismatch"; return 4; }
  int rc = exp_prepare_y(cc, beta, y);
  if (rc || ncols == 0) return rc;
  const double val = x->homogeneous ? alpha * x->scalar : 0.0;
  if (x->homogeneous && val == 0.0) return 0;
  k_exp_transmult<<<grid_for(c, ncols), 256, 0, c->st>>>(ncols, exp_pos, alpha == 1.0 ? 1 : (alpha == -1.0 ? 2 : 3), alpha,
                                                         x->d, x->homogeneous, val, y->d);
  ++c->launches;
  VCU(cudaGetLastError());
  return 0;
}
int b200vec_exp_add_msinvz(b200vec_ctx cc, int nrows, int ncols, const int* exp_pos, double alpha, const b200vec* S, const b200vec* Z, b200vec* X) {
  CTX;   // AddMSinvZImpl :170-239
  if (S->n != ncols || Z->n != ncols || X->n != nrows) { c->err = "exp_add_msinvz: dimension mismatch"; return 4; }
  if (S->homogeneous) { c->err = "exp_add_msinvz: homogeneous S takes the generic path of the caller (Matrix::AddMSinvZImpl)"; return 4; }
  if (X->homogeneous) { X->homogeneous = 0; int rc = unary<U_FILL>(c, X, X->scalar); if (rc) return rc; }
  if (ncols == 0) return 0;
  const double val = Z->homogeneous ? alpha * Z->scalar : 0.0;
  if (Z->homogeneous && val == 0.0) return 0;
  k_exp_msinvz<<<grid_for(c, ncols), 256, 0, c->st>>>(ncols, exp_pos, alpha == 1.0 ? 1 : (alpha == -1.0 ? 2 : 3), alpha, S->d,
                                                      Z->d, Z->homogeneous, val, X->d);
  ++c->launches;
  VCU(cudaGetLastError());
  return 0;
}
int b200vec_exp_sinv_blrm_zmtdbr(b200vec_ctx cc, int nrows, int ncols, const int* exp_pos, double alpha, const b200vec* S,
                                 const b200vec* R, const b200vec* Z, const b200vec* D, b200vec* X) {
  CTX;   // SinvBlrmZMTdBrImpl :241-372
  if (S->n != ncols || R->n != ncols || Z->n != ncols || X->n != ncols || D->n != nrows) { c->err = "exp_sinv_blrm_zmtdbr: dimension mismatch"; return 4; }
  if (S->homogeneous || D->homogeneous) { c->err = "exp_sinv_blrm_zmtdbr: homogeneous S or D takes the generic path of the caller"; return 4; }
  X->homogeneous = 0;
  if (ncols == 0) return 0;
  const double val = Z->homogeneous ? alpha * Z->scalar : 0.0;
  k_exp_sinv<<<grid_for(c, ncols), 256, 0, c->st>>>(ncols, exp_pos, alpha == 1.0 ? 1 : (alpha == -1.0 ? 2 : 3), alpha, S->d, R->d,
                                                    R->homogeneous, R->scalar, Z->d, Z->homogeneous, val, D->d, X->d);
  ++c->launches;
  VCU(cudaGetLastError());
  return 0;
}

// ---- V9 ------------------------------------------------------------------------------------------------------
b200vec_tmat b200vec_tmat_create(b200vec_ctx cc, int nrows, int ncols, int nnz, const int* irow, const int* jcol, int symmetric) {
  Ctx* c = (Ctx*)cc;
  if (!c || nrows < 0 || ncols < 0 || nnz < 0) return nullptr;
  if (symmetric && nrows != ncols) return nullptr;
  for (int e = 0; e < nnz; ++e)
    if (irow[e] < 1 || irow[e] > nrows || jcol[e] < 1 || jcol[e] > ncols) return nullptr;
  cudaSetDevice(c->dev);
  TMat* m = new TMat();
  m->c = c; m->nrows = nrows; m->ncols = ncols; m->nnz = nnz; m->symmetric = symmetric;
  // group the contributions by output index keeping the order in which the reference's loop produces them:
  // general: y[irow] += a*v*x[jcol] ; symmetric: y[irn] += a*v*x[jcn], then (off-diagonal) y[jcn] += a*v*x[irn]
  auto build = [&](bool trans, int nout, int** d_ptr, int** d_ent, int** d_xc) {
    std::vector<int> ptr(nout + 1, 0);
    auto visit = [&](auto&& f) {
      for (int e = 0; e < nnz; ++e) {
        const int i = (trans ? jcol[e] : irow[e]) - 1, j = (trans ? irow[e] : jcol[e]) - 1;
        f(i, e, j);
        if (symmetric && i != j) f(j, e, i);
      }
    };
    visit([&](int i, int, int) { ptr[i + 1]++; });
    for (int i = 0; i < nout; ++i) ptr[i + 1] += ptr[i];
    std::vector<int> pos(ptr.begin(), ptr.end() - 1), ent(std::max(ptr[nout], 1)), xc(std::max(ptr[nout], 1));
    visit([&](int i, int e, int j) { ent[pos[i]] = e; xc[pos[i]] = j; pos[i]++; });
    cudaMalloc((void**)d_ptr, ptr.size() * sizeof(int));
    cudaMalloc((void**)d_ent, ent.size() * sizeof(int));
    cudaMalloc((void**)d_xc, xc.size() * sizeof(int));
    cudaMemcpy(*d_ptr, ptr.data(), ptr.size() * sizeof(int), cudaMemcpyHostToDevice);
    cudaMemcpy(*d_ent, ent.data(), ent.size() * sizeof(int), cudaMemcpyHostToDevice);
    cudaMemcpy(*d_xc, xc.data(), xc.size() * sizeof(int), cudaMemcpyHostToDevice);
  };
  build(false, nrows, &m->d_rptr, &m->d_ent, &m->d_xcol);
  if (!symmetric) build(true, ncols, &m->d_tptr, &m->d_tent, &m->d_txcol);
  if (cudaGetLastError() != cudaSuccess) { b200vec_tmat_destroy((b200vec_tmat)m); return nullptr; }
  return (b200vec_tmat)m;
}
void b200vec_tmat_destroy(b200vec_tmat mm) {
  TMat* m = (TMat*)mm;
  if (!m) return;
  cudaFree(m->d_rptr); cudaFree(m->d_ent); cudaFree(m->d_xcol);
  cudaFree(m->d_tptr); cudaFree(m->d_tent); cudaFree(m->d_txcol);
  delete m;
}
static int tmat_apply(TMat* m, bool trans, const double* values, double alpha, const b200vec* x, double beta, b200vec* y) {
  Ctx* c = m->c;
  b200vec_ctx cc = (b200vec_ctx)c;
  if (cudaSetDevice(c->dev) != cudaSuccess) return 4;
  const int nout = trans ? m->ncols : m->nrows, nin = trans ? m->nrows : m->ncols;
  if (x->n != nin || y->n != nout) { c->err = "tmat: dimension mismatch"; return 4; }
  int rc = (beta != 0.0) ? b200vec_scal(cc, beta, y) : b200vec_set(cc, 0.0, y);
  if (rc) return rc;
  if (m->nnz == 0 && !m->symmetric) return 0;   // GenTMatrix returns before touching Values(); SymTMatrix does not
  if (y->homogeneous) { y->homogeneous = 0; rc = unary<U_FILL>(c, y, y->scalar); if (rc) return rc; }
  if (m->nnz == 0 || nout == 0) return 0;
  const bool t = trans && !m->symmetric;
  k_tmat_mult<<<grid_for(c, nout), 256, 0, c->st>>>(nout, t ? m->d_tptr : m->d_rptr, t ? m->d_tent : m->d_ent,
                                                    t ? m->d_txcol : m->d_xcol, values, alpha, x->d, x->homogeneous,
                                                    alpha * x->scalar, y->d);
  ++c->launches;
  VCU(cudaGetLastError());
  return 0;
}
int b200vec_tmat_mult(b200vec_tmat mm, const double* values, double alpha, const b200vec* x, double beta, b200vec* y) {
  if (!mm) return 4;
  return tmat_apply((TMat*)mm, false, values, alpha, x, beta, y);
}
int b200vec_tmat_transmult(b200vec_tmat mm, const double* values, double alpha, const b200vec* x, double beta, b200vec* y) {
  if (!mm) return 4;
  return tmat_apply((TMat*)mm, true, values, alpha, x, beta, y);
}

}  // extern "C"
