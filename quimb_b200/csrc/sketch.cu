// The sketched left-environment step of successive randomized compression
// (tensor_network_1d_compress_src, quimb/tensor/tn1d/compress.py:1653-1840)
// on the MPS / MPO ladder.  For site s with noise Omega[B, o] the new
// environment is
//
//   LE'[B, b, u] = sum LE[B, a, v] A[a, p, b] W[v, u, o, p] Omega[B, o]
//
// and this kernel computes its first half,
//
//   H[B, a, u, p] = sum_v LE[B, a, v] T_B[v, (u, p)],
//   T_B[v, (u, p)] = sum_o W[v, u, o, p] Omega[B, o],
//
// leaving LE' = H A to one ordinary contraction (rows (B, u), K = (a, p)).
// Through the contraction engine the first half is two launches, the second
// a batched GEMM with K = D_w and N = D_w d that the DMMA tiles pad to 32.
//
// One CTA owns one sample B, a tile of NT (u, p) columns and RA rows a.  Per
// chunk of VC values of v it forms its slice of T_B in shared memory (the sum
// over o, in order), stages the LE rows of the chunk, and each thread adds
// the chunk into up to OPT outputs, in v order.  So LE is read once per
// column tile (once for every ladder with D_w d <= 64) and H written once;
// the tile shape is a function of (na, D_w d) alone and every output is a
// sequential sum over v, so the bits depend on the shape only.  Single
// precision is widened on load and accumulated in fp64 (pairs of fp64 for
// complex64), rounded once on the store.
#include <algorithm>
#include <climits>

#include "common.cuh"

namespace qb {

constexpr int SK_THREADS = 256;
constexpr int SK_NT = 64;         // (u, p) columns per tile
constexpr int SK_VC = 8;          // values of v per chunk
constexpr int SK_OPT = 4;         // outputs per thread
constexpr int SK_MAX_RA = 256;    // rows a per tile

struct SketchShape {
  int nt, ra;
  int64_t ctiles, rtiles, blocks;
};

static SketchShape sketch_shape(int64_t nB, int64_t na, int64_t nup) {
  SketchShape s;
  s.nt = (int)std::min<int64_t>(nup, SK_NT);
  s.ra = (int)std::min<int64_t>(std::min(SK_MAX_RA, SK_THREADS * SK_OPT / s.nt), na);
  s.ctiles = (nup + s.nt - 1) / s.nt;
  s.rtiles = (na + s.ra - 1) / s.ra;
  s.blocks = nB * s.ctiles * s.rtiles;
  return s;
}

// widened element types: storage T, accumulator A
__device__ __forceinline__ double sk_load(const double *p) { return *p; }
__device__ __forceinline__ double sk_load(const float *p) { return (double)*p; }
__device__ __forceinline__ double2 sk_load(const double2 *p) { return *p; }
__device__ __forceinline__ double2 sk_load(const float2 *p) {
  const float2 x = *p;
  return make_double2((double)x.x, (double)x.y);
}
__device__ __forceinline__ void sk_store(double *p, double x) { *p = x; }
__device__ __forceinline__ void sk_store(float *p, double x) { *p = (float)x; }
__device__ __forceinline__ void sk_store(double2 *p, double2 x) { *p = x; }
__device__ __forceinline__ void sk_store(float2 *p, double2 x) {
  *p = make_float2((float)x.x, (float)x.y);
}
__device__ __forceinline__ void sk_zero(double &x) { x = 0.0; }
__device__ __forceinline__ void sk_zero(double2 &x) { x = make_double2(0.0, 0.0); }
// acc += x * y, a fixed order of fused operations
__device__ __forceinline__ void sk_fma(double &acc, double x, double y) { acc = fma(x, y, acc); }
__device__ __forceinline__ void sk_fma(double2 &acc, double2 x, double2 y) {
  acc.x = fma(-x.y, y.y, fma(x.x, y.x, acc.x));
  acc.y = fma(x.y, y.x, fma(x.x, y.y, acc.y));
}

template <typename T> struct SkAcc;
template <> struct SkAcc<double> { using type = double; };
template <> struct SkAcc<float> { using type = double; };
template <> struct SkAcc<double2> { using type = double2; };
template <> struct SkAcc<float2> { using type = double2; };

struct SketchArgs {
  int64_t nB, na, nv, nu, no, np;
  int64_t le0, le1, le2;              // LE[B, a, v]
  int64_t w0, w1, w2, w3;             // W[v, u, o, p]
  int64_t om0, om1;                   // Omega[B, o]
  int64_t h0, h1, h2, h3;             // H[B, a, u, p]
  int nt, ra;
  int64_t ctiles, rtiles;
  const void *LE, *W, *Om;
  void *H;
};

template <typename T>
__global__ void __launch_bounds__(SK_THREADS) sketch_env_kernel(SketchArgs g) {
  using A = typename SkAcc<T>::type;
  __shared__ A Ts[SK_VC][SK_NT];
  __shared__ A Ls[SK_MAX_RA][SK_VC];
  const T *LE = static_cast<const T *>(g.LE);
  const T *W = static_cast<const T *>(g.W);
  const T *Om = static_cast<const T *>(g.Om);
  T *H = static_cast<T *>(g.H);
  const int t = threadIdx.x;

  int64_t blk = blockIdx.x;
  const int64_t rt = blk % g.rtiles;
  blk /= g.rtiles;
  const int64_t ct = blk % g.ctiles;
  const int64_t B = blk / g.ctiles;
  const int64_t a0 = rt * g.ra, c0 = ct * g.nt;
  const int rows = (int)min((int64_t)g.ra, g.na - a0);
  const int cols = (int)min((int64_t)g.nt, g.nu * g.np - c0);
  const int nout = rows * cols;

  A acc[SK_OPT];
#pragma unroll
  for (int j = 0; j < SK_OPT; ++j) sk_zero(acc[j]);

  const T *le = LE + B * g.le0 + a0 * g.le1;
  const T *om = Om + B * g.om0;
  for (int64_t v0 = 0; v0 < g.nv; v0 += SK_VC) {
    const int vc = (int)min((int64_t)SK_VC, g.nv - v0);
    // this sample's slice of the W . Omega table
    for (int e = t; e < vc * cols; e += SK_THREADS) {
      const int vv = e / cols, c = e - vv * cols;
      const int64_t col = c0 + c;
      const int64_t u = col / g.np, p = col - u * g.np;
      const T *w = W + (v0 + vv) * g.w0 + u * g.w1 + p * g.w3;
      A s;
      sk_zero(s);
      for (int64_t o = 0; o < g.no; ++o) sk_fma(s, sk_load(w + o * g.w2), sk_load(om + o * g.om1));
      Ts[vv][c] = s;
    }
    // the LE rows of this chunk
    for (int e = t; e < rows * vc; e += SK_THREADS) {
      const int r = e / vc, vv = e - r * vc;
      Ls[r][vv] = sk_load(le + r * g.le1 + (v0 + vv) * g.le2);
    }
    __syncthreads();
#pragma unroll
    for (int j = 0; j < SK_OPT; ++j) {
      const int idx = t + j * SK_THREADS;
      if (idx < nout) {
        const int r = idx / cols, c = idx - r * cols;
        A s = acc[j];
        for (int vv = 0; vv < vc; ++vv) sk_fma(s, Ls[r][vv], Ts[vv][c]);
        acc[j] = s;
      }
    }
    __syncthreads();
  }

#pragma unroll
  for (int j = 0; j < SK_OPT; ++j) {
    const int idx = t + j * SK_THREADS;
    if (idx < nout) {
      const int r = idx / cols, c = idx - r * cols;
      const int64_t col = c0 + c;
      const int64_t u = col / g.np, p = col - u * g.np;
      sk_store(H + B * g.h0 + (a0 + r) * g.h1 + u * g.h2 + p * g.h3, acc[j]);
    }
  }
}

}  // namespace qb

using namespace qb;

extern "C" int qb_sketch_env(int dtype, int64_t nB, int64_t na, int64_t nv, int64_t nu,
                             int64_t no, int64_t np, const void *LE, const int64_t lestride[3],
                             const void *W, const int64_t wstride[4], const void *Om,
                             const int64_t omstride[2], void *H, const int64_t hstride[4],
                             void *stream) {
  if (dtype != QB_F32 && dtype != QB_F64 && dtype != QB_C64 && dtype != QB_C128) {
    set_error("qb_sketch_env: unknown dtype %d", dtype);
    return -1;
  }
  if (nB < 1 || na < 1 || nv < 1 || nu < 1 || no < 1 || np < 1) {
    set_error("qb_sketch_env: extents (B %lld, a %lld, v %lld, u %lld, o %lld, p %lld) must "
              "be >= 1", (long long)nB, (long long)na, (long long)nv, (long long)nu,
              (long long)no, (long long)np);
    return -2;
  }
  const uintptr_t align = (uintptr_t)dtype_size(dtype) - 1;
  auto bad = [&](const void *p) { return !p || (reinterpret_cast<uintptr_t>(p) & align); };
  if (bad(LE) || bad(W) || bad(Om) || bad(H) || !lestride || !wstride || !omstride ||
      !hstride) {
    set_error("qb_sketch_env: LE, W, Omega, H or a stride array is null or misaligned");
    return -3;
  }
  if (nu > INT64_MAX / np) {
    set_error("qb_sketch_env: u p = %lld x %lld overflows", (long long)nu, (long long)np);
    return -4;
  }
  const SketchShape s = sketch_shape(nB, na, nu * np);
  if (nB > INT_MAX || s.ctiles * s.rtiles > INT_MAX / nB) {
    set_error("qb_sketch_env: %lld samples x %lld tiles exceed one grid", (long long)nB,
              (long long)(s.ctiles * s.rtiles));
    return -4;
  }
  SketchArgs g;
  g.nB = nB; g.na = na; g.nv = nv; g.nu = nu; g.no = no; g.np = np;
  g.le0 = lestride[0]; g.le1 = lestride[1]; g.le2 = lestride[2];
  g.w0 = wstride[0]; g.w1 = wstride[1]; g.w2 = wstride[2]; g.w3 = wstride[3];
  g.om0 = omstride[0]; g.om1 = omstride[1];
  g.h0 = hstride[0]; g.h1 = hstride[1]; g.h2 = hstride[2]; g.h3 = hstride[3];
  g.nt = s.nt; g.ra = s.ra; g.ctiles = s.ctiles; g.rtiles = s.rtiles;
  g.LE = LE; g.W = W; g.Om = Om; g.H = H;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const unsigned grid = (unsigned)s.blocks;
  switch (dtype) {
    case QB_F64: sketch_env_kernel<double><<<grid, SK_THREADS, 0, st>>>(g); break;
    case QB_C128: sketch_env_kernel<double2><<<grid, SK_THREADS, 0, st>>>(g); break;
    case QB_F32: sketch_env_kernel<float><<<grid, SK_THREADS, 0, st>>>(g); break;
    default: sketch_env_kernel<float2><<<grid, SK_THREADS, 0, st>>>(g); break;
  }
  QB_LAUNCH_CHECK();
  return 0;
}
