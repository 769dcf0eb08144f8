// Batched MPS sampling, the per-site selection pass (MatrixProductState.sample
// / sample_configuration, quimb/tensor/tn1d/core.py:3871-3990).
//
// The host driver (quimb_b200/tebd.py:mps_sample) carries one left vector
// per sample: at site i the DMMA engine forms W = V . A_i (C x d x r), and
// this kernel turns each sample's slice W[c] into its outcome.  One warp per
// sample, grid-stride over samples:
//   pi[s] = sum_j |W[c, s, j]|^2      lane-strided over j, then a butterfly
//   p = pi / sum(pi), cdf = cumsum(p) / cdf[-1]   (numpy's order, one lane)
//   x = #{s : cdf[s] <= u}            (searchsorted side='right')
//   omega *= p[x];  V[c] = W[c, x] / sqrt(pi[x])   (unit-norm row)
// The arithmetic of a row depends on (d, r) only -- never on C, the grid or
// the row's neighbours -- so a row gives the same bits alone or in a batch.
#include <algorithm>

#include "common.cuh"

namespace qb {

constexpr int SAMPLE_MAX_D = 256;   // pi of one warp's sample lives in smem
constexpr int SAMPLE_WARPS = 8;

__device__ __forceinline__ double abs2(double v) { return __dmul_rn(v, v); }
__device__ __forceinline__ double abs2(double2 v) {
  return __dadd_rn(__dmul_rn(v.x, v.x), __dmul_rn(v.y, v.y));
}
__device__ __forceinline__ double div_rn(double v, double s) { return __ddiv_rn(v, s); }
__device__ __forceinline__ double2 div_rn(double2 v, double s) {
  return make_double2(__ddiv_rn(v.x, s), __ddiv_rn(v.y, s));
}
template <typename T> __device__ __forceinline__ T zero_of();
template <> __device__ __forceinline__ double zero_of<double>() { return 0.0; }
template <> __device__ __forceinline__ double2 zero_of<double2>() {
  return make_double2(0.0, 0.0);
}

// numpy's pairwise summation of a contiguous float64 vector (np.sum:
// 0 + pairwise(a, n); blocks of 8 partial sums up to 128 elements, halves on
// multiples of 8 above).  DEPTH bounds the recursion (n <= 256 needs 2).
template <int DEPTH>
__device__ __noinline__ double np_pairwise_sum(const double *a, int n) {
  if (DEPTH == 0 || n <= 128) {
    if (n < 8) {
      double res = 0.0;
      for (int i = 0; i < n; ++i) res = __dadd_rn(res, a[i]);
      return res;
    }
    double r[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) r[j] = a[j];
    int i = 8;
    for (; i < n - (n % 8); i += 8)
#pragma unroll
      for (int j = 0; j < 8; ++j) r[j] = __dadd_rn(r[j], a[i + j]);
    double res = __dadd_rn(__dadd_rn(__dadd_rn(r[0], r[1]), __dadd_rn(r[2], r[3])),
                           __dadd_rn(__dadd_rn(r[4], r[5]), __dadd_rn(r[6], r[7])));
    for (; i < n; ++i) res = __dadd_rn(res, a[i]);
    return res;
  }
  int n2 = n / 2;
  n2 -= n2 % 8;
  return __dadd_rn(np_pairwise_sum<(DEPTH > 0 ? DEPTH - 1 : 0)>(a, n2),
                   np_pairwise_sum<(DEPTH > 0 ? DEPTH - 1 : 0)>(a + n2, n - n2));
}

template <typename T>
__global__ void __launch_bounds__(SAMPLE_WARPS * 32)
    sample_select_kernel(int64_t C, int d, int64_t r, const T *__restrict__ W,
                         const double *__restrict__ u, int64_t ldu,
                         int64_t *__restrict__ config, int64_t ldc,
                         double *__restrict__ omega, T *__restrict__ V) {
  __shared__ double sh_pi[SAMPLE_WARPS][SAMPLE_MAX_D];
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  double *pi = sh_pi[wid];
  for (int64_t c = (int64_t)blockIdx.x * SAMPLE_WARPS + wid; c < C;
       c += (int64_t)gridDim.x * SAMPLE_WARPS) {
    const T *Wc = W + c * d * r;
    for (int s = 0; s < d; ++s) {
      const T *row = Wc + (int64_t)s * r;
      double acc = 0.0;
#pragma unroll 4
      for (int64_t j = lane; j < r; j += 32) acc = __dadd_rn(acc, abs2(row[j]));
#pragma unroll
      for (int o = 16; o > 0; o >>= 1)
        acc = __dadd_rn(acc, __shfl_xor_sync(0xffffffffu, acc, o));
      if (lane == 0) pi[s] = acc;
    }
    __syncwarp();
    int64_t x = -1;
    double scale = 0.0;
    if (lane == 0) {
      const double uc = u[c * ldu];
      const double tot = np_pairwise_sum<3>(pi, d);
      // a zero or non-finite total makes numpy's p NaN (rng.choice raises);
      // u outside [0, 1) is never drawn by a Generator
      if (tot > 0.0 && isfinite(tot) && uc >= 0.0 && uc < 1.0) {
        double last = 0.0;
        for (int s = 0; s < d; ++s) last = __dadd_rn(last, __ddiv_rn(pi[s], tot));
        double cum = 0.0;
        x = 0;
        for (int s = 0; s < d; ++s) {
          cum = __dadd_rn(cum, __ddiv_rn(pi[s], tot));
          if (__ddiv_rn(cum, last) <= uc) x = s + 1;
        }
        // cdf[d-1] == 1 > u, so x < d, and p[x] > 0 (a zero-probability
        // outcome repeats its predecessor's cdf value, which is <= u)
        omega[c] = __dmul_rn(omega[c], __ddiv_rn(pi[x], tot));
        scale = __dsqrt_rn(pi[x]);
        config[c * ldc] = x;
      } else {
        omega[c] = __longlong_as_double(0x7ff8000000000000LL);
        config[c * ldc] = -1;
      }
    }
    x = __shfl_sync(0xffffffffu, x, 0);
    scale = __shfl_sync(0xffffffffu, scale, 0);
    T *Vc = V + c * r;
    if (x >= 0) {
      const T *row = Wc + x * r;
      for (int64_t j = lane; j < r; j += 32) Vc[j] = div_rn(row[j], scale);
    } else {
      for (int64_t j = lane; j < r; j += 32) Vc[j] = zero_of<T>();
    }
    __syncwarp();   // pi is rewritten by this warp's next sample
  }
}

}  // namespace qb

using namespace qb;

extern "C" int qb_sample_select(int dtype, int64_t C, int64_t d, int64_t r, const void *W,
                                const double *u, int64_t ldu, int64_t *config, int64_t ldc,
                                double *omega, void *V, void *stream) {
  if (dtype != QB_F64 && dtype != QB_C128) {
    set_error("qb_sample_select: dtype must be QB_F64 or QB_C128 (got %d)", dtype);
    return -1;
  }
  if (C < 0) { set_error("qb_sample_select: C < 0"); return -2; }
  if (d < 1 || d > SAMPLE_MAX_D) {
    set_error("qb_sample_select: physical dimension d = %lld outside [1, %d]",
              (long long)d, SAMPLE_MAX_D);
    return -3;
  }
  if (r < 1) { set_error("qb_sample_select: r < 1"); return -4; }
  if (C == 0) return 0;
  const uintptr_t align = dtype == QB_C128 ? 15 : 7;
  if (!W || (reinterpret_cast<uintptr_t>(W) & align)) {
    set_error("qb_sample_select: W is null or misaligned");
    return -5;
  }
  if (!u) { set_error("qb_sample_select: u is null"); return -6; }
  if (ldu < 1) { set_error("qb_sample_select: ldu < 1"); return -7; }
  if (!config) { set_error("qb_sample_select: config is null"); return -8; }
  if (ldc < 1) { set_error("qb_sample_select: ldc < 1"); return -9; }
  if (!omega) { set_error("qb_sample_select: omega is null"); return -10; }
  if (!V || (reinterpret_cast<uintptr_t>(V) & align)) {
    set_error("qb_sample_select: V is null or misaligned");
    return -11;
  }
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const int64_t blocks =
      std::min<int64_t>((C + SAMPLE_WARPS - 1) / SAMPLE_WARPS, (int64_t)sm_count() * 8);
  if (dtype == QB_F64)
    sample_select_kernel<double><<<(unsigned)blocks, SAMPLE_WARPS * 32, 0, st>>>(
        C, (int)d, r, static_cast<const double *>(W), u, ldu, config, ldc, omega,
        static_cast<double *>(V));
  else
    sample_select_kernel<double2><<<(unsigned)blocks, SAMPLE_WARPS * 32, 0, st>>>(
        C, (int)d, r, static_cast<const double2 *>(W), u, ldu, config, ldc, omega,
        static_cast<double2 *>(V));
  QB_LAUNCH_CHECK();
  return 0;
}
