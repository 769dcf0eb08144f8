// HBM-bound helpers of the hot path: strided permute-copy (quimb's
// fuse = transpose+reshape, array_ops.py:148-180), Lanczos vector algebra
// (axpby / dot / scale -- the dsaupd inner loop behind
// quimb/linalg/scipy_linalg.py:113-128) and diagonal scaling
// (rdmul / ldmul, decomp.py:580-615).  All are single-pass, coalesced and
// sized in multiples of the SM count.
#include <algorithm>
#include <vector>

#include "common.cuh"

namespace qb {

// ------------------------------------------------------------- permute ----
constexpr int PMAX = 16;
struct PermParams {
  const void *src;
  void *dst;
  int32_t n;  // number of "rest" modes (excluding the two tile modes)
  int32_t ext[PMAX];
  int64_t ss[PMAX], ds[PMAX];
  // tile modes: d = fastest in dst, s = fastest in src (may coincide)
  int64_t ext_d, ext_s;
  int64_t d_ss, d_ds;  // strides of mode d in src / dst
  int64_t s_ss, s_ds;  // strides of mode s in src / dst
  int64_t rest;        // product of rest extents
  int32_t same;        // d == s: plain row copy
  int32_t conj;
};

// Conjugation flips the sign bit of the imaginary part (IEEE negate), so the
// copy stays bitwise: an arithmetic -x compiles to an add, which replaces a
// NaN's payload with the canonical NaN.
template <typename T>
__device__ __forceinline__ T conj_if(T v, int) { return v; }
template <>
__device__ __forceinline__ double2 conj_if(double2 v, int c) {
  if (c) v.y = __longlong_as_double(__double_as_longlong(v.y) ^ (long long)(1ULL << 63));
  return v;
}
template <>
__device__ __forceinline__ float2 conj_if(float2 v, int c) {
  if (c) v.y = __int_as_float(__float_as_int(v.y) ^ (int)0x80000000u);
  return v;
}

template <typename T>
__global__ void __launch_bounds__(256)
    permute_tiled_kernel(const __grid_constant__ PermParams p) {
  __shared__ T tile[32][33];
  const T *src = static_cast<const T *>(p.src);
  T *dst = static_cast<T *>(p.dst);
  const int64_t tiles_d = (p.ext_d + 31) / 32, tiles_s = (p.ext_s + 31) / 32;
  const int64_t per_rest = tiles_d * tiles_s;
  const int64_t total = per_rest * p.rest;
  for (int64_t w = blockIdx.x; w < total; w += gridDim.x) {
    int64_t r = w / per_rest, tt = w - r * per_rest;
    int64_t td = tt / tiles_s, ts = tt - td * tiles_s;
    int64_t so = 0, dof = 0;
    for (int i = 0; i < p.n; ++i) {
      int64_t e = p.ext[i], q = r / e, d = r - q * e;
      so += d * p.ss[i];
      dof += d * p.ds[i];
      r = q;
    }
    const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
    {
      int64_t s = ts * 32 + tx;
#pragma unroll
      for (int j = 0; j < 32; j += 8) {
        int64_t d = td * 32 + ty + j;
        if (s < p.ext_s && d < p.ext_d)
          tile[ty + j][tx] = src[so + s * p.s_ss + d * p.d_ss];
      }
    }
    __syncthreads();
    {
      int64_t d = td * 32 + tx;
#pragma unroll
      for (int j = 0; j < 32; j += 8) {
        int64_t s = ts * 32 + ty + j;
        if (s < p.ext_s && d < p.ext_d)
          dst[dof + d * p.d_ds + s * p.s_ds] = conj_if(tile[tx][ty + j], p.conj);
      }
    }
    __syncthreads();
  }
}

template <typename T>
__global__ void __launch_bounds__(256)
    permute_rows_kernel(const __grid_constant__ PermParams p) {
  // fastest mode is shared by src and dst: copy rows of ext_d elements
  const T *src = static_cast<const T *>(p.src);
  T *dst = static_cast<T *>(p.dst);
  const int64_t chunks = (p.ext_d + 255) / 256;
  const int64_t total = chunks * p.rest;
  for (int64_t w = blockIdx.x; w < total; w += gridDim.x) {
    int64_t r = w / chunks, c = w - r * chunks;
    int64_t so = 0, dof = 0;
    for (int i = 0; i < p.n; ++i) {
      int64_t e = p.ext[i], q = r / e, d = r - q * e;
      so += d * p.ss[i];
      dof += d * p.ds[i];
      r = q;
    }
    int64_t x = c * 256 + threadIdx.x;
    if (x < p.ext_d)
      dst[dof + x * p.d_ds] = conj_if(src[so + x * p.d_ss], p.conj);
  }
}

struct PM {
  int64_t ext, ss, ds;
};

template <typename T>
static int launch_permute_t(const PermParams &p, cudaStream_t st) {
  int blocks;
  if (p.same) {
    int64_t total = ((p.ext_d + 255) / 256) * p.rest;
    blocks = (int)std::min<int64_t>(total, (int64_t)sm_count() * 16);
    if (blocks < 1) blocks = 1;
    permute_rows_kernel<T><<<blocks, 256, 0, st>>>(p);
  } else {
    int64_t total = ((p.ext_d + 31) / 32) * ((p.ext_s + 31) / 32) * p.rest;
    blocks = (int)std::min<int64_t>(total, (int64_t)sm_count() * 16);
    if (blocks < 1) blocks = 1;
    permute_tiled_kernel<T><<<blocks, 256, 0, st>>>(p);
  }
  QB_LAUNCH_CHECK();
  return 0;
}

// ------------------------------------------------------------ fill zero ---
__global__ void fill_zero_kernel(void *ptr, int64_t nbytes16, int64_t tail_off,
                                 int tail) {
  uint4 z = make_uint4(0, 0, 0, 0);
  uint4 *q = static_cast<uint4 *>(ptr);
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < nbytes16;
       i += (int64_t)gridDim.x * blockDim.x)
    q[i] = z;
  if (blockIdx.x == 0 && threadIdx.x < tail)
    static_cast<unsigned char *>(ptr)[tail_off + threadIdx.x] = 0;
}

// -------------------------------------------------------- vector algebra --
template <typename R>
__global__ void __launch_bounds__(256)
    axpby_real_kernel(int64_t n, R a, const R *__restrict__ x, R b,
                      R *__restrict__ y) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n;
       i += (int64_t)gridDim.x * blockDim.x) {
    R yv = (b == R(0)) ? R(0) : b * y[i];
    y[i] = a * x[i] + yv;
  }
}
template <typename R, typename R2>
__global__ void __launch_bounds__(256)
    axpby_cplx_kernel(int64_t n, R ar, R ai, const R2 *__restrict__ x, R br,
                      R bi, R2 *__restrict__ y) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n;
       i += (int64_t)gridDim.x * blockDim.x) {
    R2 xv = x[i], yv = y[i], o;
    o.x = ar * xv.x - ai * xv.y;
    o.y = ar * xv.y + ai * xv.x;
    if (br != R(0) || bi != R(0)) {
      o.x += br * yv.x - bi * yv.y;
      o.y += br * yv.y + bi * yv.x;
    }
    y[i] = o;
  }
}

template <typename R>
__global__ void __launch_bounds__(256)
    scale_kernel(int64_t nreal, R ar, R ai, const R *__restrict__ div, int cplx,
                 R *__restrict__ x) {
  // complex data viewed as 2*n reals when the factor is real
  R f = ar, g = ai;
  if (div) {
    // divide by a device scalar (real part only is used: norms are real)
    // an exactly zero divisor (norm of an exactly zero vector: Krylov
    // breakdown) leaves a zero vector, not NaNs
    R d = div[0];
    f = (d == R(0)) ? R(0) : ar / d;
    g = (d == R(0)) ? R(0) : ai / d;
  }
  if (!cplx || g == R(0)) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < nreal;
         i += (int64_t)gridDim.x * blockDim.x)
      x[i] *= f;
  } else {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
         i < nreal / 2; i += (int64_t)gridDim.x * blockDim.x) {
      R re = x[2 * i], im = x[2 * i + 1];
      x[2 * i] = f * re - g * im;
      x[2 * i + 1] = f * im + g * re;
    }
  }
}

template <typename R>
__global__ void __launch_bounds__(256)
    scale_into_kernel(int64_t nreal, R a, const R *__restrict__ div, const R *__restrict__ x,
                      R *__restrict__ y) {
  R f = a;
  if (div) {
    const R d = div[0];
    f = (d == R(0)) ? R(0) : a / d;
  }
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < nreal;
       i += (int64_t)gridDim.x * blockDim.x)
    y[i] = x[i] * f;
}

// two-stage deterministic dot: stage 1 one partial per block (fixed grid),
// stage 2 a single block sums the partials in a fixed order
constexpr int DOT_BLOCKS = 592;  // 4 per SM
template <typename R, int CPLX>
__global__ void __launch_bounds__(256)
    dot_stage1_kernel(int64_t n, const R *__restrict__ x,
                      const R *__restrict__ y, double *__restrict__ part) {
  double sr = 0.0, si = 0.0;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n;
       i += (int64_t)gridDim.x * blockDim.x) {
    if (CPLX) {
      double xr = x[2 * i], xi = x[2 * i + 1], yr = y[2 * i], yi = y[2 * i + 1];
      sr += xr * yr + xi * yi;  // conj(x) * y
      si += xr * yi - xi * yr;
    } else {
      sr += (double)x[i] * (double)y[i];
    }
  }
  __shared__ double shr[8], shi[8];
  sr = warp_sum(sr);
  if (CPLX) si = warp_sum(si);
  if ((threadIdx.x & 31) == 0) { shr[threadIdx.x >> 5] = sr; shi[threadIdx.x >> 5] = si; }
  __syncthreads();
  if (threadIdx.x == 0) {
    double a = 0, b = 0;
    for (int w = 0; w < 8; ++w) { a += shr[w]; b += shi[w]; }
    part[2 * blockIdx.x] = a;
    part[2 * blockIdx.x + 1] = b;
  }
}
template <typename R, int CPLX>
__global__ void __launch_bounds__(256)
    dot_stage2_kernel(int nparts, const double *__restrict__ part,
                      R *__restrict__ out) {
  __shared__ double shr[256], shi[256];
  double a = 0, b = 0;
  for (int i = threadIdx.x; i < nparts; i += 256) { a += part[2 * i]; b += part[2 * i + 1]; }
  shr[threadIdx.x] = a; shi[threadIdx.x] = b;
  __syncthreads();
  for (int s = 128; s > 0; s >>= 1) {
    if (threadIdx.x < s) { shr[threadIdx.x] += shr[threadIdx.x + s]; shi[threadIdx.x] += shi[threadIdx.x + s]; }
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    out[0] = (R)shr[0];
    if (CPLX) out[1] = (R)shi[0];
  }
}

template <typename R>
__global__ void __launch_bounds__(256)
    scale_diag_kernel(int64_t rows, int64_t cols, int epr, R *__restrict__ x,
                      const R *__restrict__ d, int side, int sq) {
  // epr: reals per element (1 real, 2 complex); x is rows x cols row-major
  const int64_t total = rows * cols;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total;
       i += (int64_t)gridDim.x * blockDim.x) {
    int64_t r = i / cols, c = i - r * cols;
    R f = d[side ? c : r];
    if (sq) f = sqrt(f);
    if (epr == 1) x[i] *= f;
    else { x[2 * i] *= f; x[2 * i + 1] *= f; }
  }
}

struct FillDesc {
  int rank;
  int64_t shape[QB_MAX_RANK];
  int64_t stride[QB_MAX_RANK];  // in reals
};
// strided zero fill (one thread per element; epr reals per element)
__global__ void __launch_bounds__(256)
    fill_zero_strided_kernel(double *__restrict__ base, const FillDesc d,
                             int64_t total, int epr, int real_bytes) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total;
       i += (int64_t)gridDim.x * blockDim.x) {
    int64_t rem = i, off = 0;
    for (int k = d.rank - 1; k >= 0; --k) {
      const int64_t q = rem / d.shape[k];
      off += (rem - q * d.shape[k]) * d.stride[k];
      rem = q;
    }
    if (real_bytes == 8) {
      double *p = base + off;
      for (int e = 0; e < epr; ++e) p[e] = 0.0;
    } else {
      float *p = reinterpret_cast<float *>(base) + off;
      for (int e = 0; e < epr; ++e) p[e] = 0.0f;
    }
  }
}

int launch_fill_zero(const qb_tensor_t *C, cudaStream_t st) {
  // contiguous, 16-byte aligned outputs take the vector fill; anything else
  // (a strided `out=` view, an 8-byte aligned slice) is zeroed element-wise
  // through its strides
  int64_t n = 1;
  for (int i = 0; i < C->rank; ++i) n *= C->shape[i];
  int64_t bytes = n * dtype_size(C->dtype);
  if (bytes == 0) return 0;
  bool contiguous = true;
  {
    int64_t expect = 1;
    for (int i = C->rank - 1; i >= 0; --i) {
      if (C->shape[i] != 1 && C->stride[i] != expect) contiguous = false;
      expect *= C->shape[i];
    }
  }
  if (!contiguous || (reinterpret_cast<uintptr_t>(C->ptr) & 15)) {
    const bool cplx = (C->dtype == QB_C128 || C->dtype == QB_C64);
    const int epr = cplx ? 2 : 1;
    const int real_bytes = (int)dtype_size(C->dtype) / epr;
    FillDesc d;
    d.rank = C->rank;
    for (int i = 0; i < C->rank; ++i) {
      d.shape[i] = C->shape[i];
      d.stride[i] = C->stride[i] * epr;
    }
    int blocks = (int)std::min<int64_t>((n + 255) / 256, (int64_t)sm_count() * 8);
    fill_zero_strided_kernel<<<blocks, 256, 0, st>>>(static_cast<double *>(C->ptr), d, n,
                                                     epr, real_bytes);
    QB_LAUNCH_CHECK();
    return 0;
  }
  int64_t n16 = bytes / 16;
  int tail = (int)(bytes - n16 * 16);
  int blocks = (int)std::min<int64_t>((n16 + 255) / 256 + 1, (int64_t)sm_count() * 8);
  fill_zero_kernel<<<blocks, 256, 0, st>>>(C->ptr, n16, n16 * 16, tail);
  QB_LAUNCH_CHECK();
  return 0;
}

}  // namespace qb

using namespace qb;

extern "C" {

int qb_permute(const qb_tensor_t *src, qb_tensor_t *dst, int conj,
               void *stream) {
  if (!src) return -1;
  if (!dst) return -2;
  if (src->rank != dst->rank || src->dtype != dst->dtype) {
    set_error("qb_permute: rank/dtype mismatch");
    return -2;
  }
  std::vector<PM> ms;
  int64_t total = 1;
  for (int i = 0; i < src->rank; ++i) {
    if (src->shape[i] != dst->shape[i]) {
      set_error("qb_permute: shape mismatch on axis %d", i);
      return -2;
    }
    total *= src->shape[i];
    if (src->shape[i] > 1) ms.push_back({src->shape[i], src->stride[i], dst->stride[i]});
  }
  if (total == 0) return 0;
  // order by destination stride, then merge jointly contiguous neighbours
  std::stable_sort(ms.begin(), ms.end(),
                   [](const PM &a, const PM &b) { return a.ds < b.ds; });
  std::vector<PM> mg;
  for (auto &x : ms) {
    if (!mg.empty()) {
      PM &l = mg.back();
      if (x.ss == l.ss * l.ext && x.ds == l.ds * l.ext) { l.ext *= x.ext; continue; }
    }
    mg.push_back(x);
  }
  PermParams p;
  memset(&p, 0, sizeof(p));
  p.src = src->ptr; p.dst = dst->ptr; p.conj = conj && dtype_is_complex(src->dtype);
  if (mg.empty()) mg.push_back({1, 1, 1});
  // d = first (smallest dst stride); s = mode with smallest src stride
  size_t di = 0, si = 0;
  for (size_t i = 1; i < mg.size(); ++i)
    if (mg[i].ss < mg[si].ss) si = i;
  p.ext_d = mg[di].ext; p.d_ss = mg[di].ss; p.d_ds = mg[di].ds;
  p.same = (si == di) || mg[si].ss >= mg[di].ss;
  if (p.same) si = di;
  p.ext_s = p.same ? 1 : mg[si].ext;
  p.s_ss = p.same ? 0 : mg[si].ss;
  p.s_ds = p.same ? 0 : mg[si].ds;
  p.rest = 1;
  for (size_t i = 0; i < mg.size(); ++i) {
    if (i == di || i == si) continue;
    if (p.n >= PMAX) {
      set_error("qb_permute: more than %d non-mergeable modes", PMAX);
      return -100;
    }
    if (mg[i].ext > 0x7fffffffLL) { set_error("qb_permute: extent too large"); return -100; }
    p.ext[p.n] = (int32_t)mg[i].ext; p.ss[p.n] = mg[i].ss; p.ds[p.n] = mg[i].ds;
    p.rest *= mg[i].ext;
    ++p.n;
  }
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  switch (src->dtype) {
    case QB_F32: return launch_permute_t<float>(p, st);
    case QB_F64: return launch_permute_t<double>(p, st);
    case QB_C64: return launch_permute_t<float2>(p, st);
    case QB_C128: return launch_permute_t<double2>(p, st);
  }
  set_error("qb_permute: bad dtype %d", src->dtype);
  return -1;
}

static int ew_blocks(int64_t n) {
  int64_t b = (n + 255) / 256;
  int64_t cap = (int64_t)sm_count() * 8;
  if (b > cap) b = cap;
  if (b < 1) b = 1;
  return (int)b;
}

int qb_axpby(int dtype, int64_t n, const double alpha[2], const void *x,
             const double beta[2], void *y, void *stream) {
  if (n <= 0) return 0;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  switch (dtype) {
    case QB_F64:
      axpby_real_kernel<double><<<ew_blocks(n), 256, 0, st>>>(
          n, alpha[0], (const double *)x, beta[0], (double *)y);
      break;
    case QB_F32:
      axpby_real_kernel<float><<<ew_blocks(n), 256, 0, st>>>(
          n, (float)alpha[0], (const float *)x, (float)beta[0], (float *)y);
      break;
    case QB_C128:
      axpby_cplx_kernel<double, double2><<<ew_blocks(n), 256, 0, st>>>(
          n, alpha[0], alpha[1], (const double2 *)x, beta[0], beta[1], (double2 *)y);
      break;
    case QB_C64:
      axpby_cplx_kernel<float, float2><<<ew_blocks(n), 256, 0, st>>>(
          n, (float)alpha[0], (float)alpha[1], (const float2 *)x, (float)beta[0],
          (float)beta[1], (float2 *)y);
      break;
    default: set_error("qb_axpby: bad dtype"); return -1;
  }
  QB_LAUNCH_CHECK();
  return 0;
}

int qb_scale(int dtype, int64_t n, const double alpha[2],
             const void *dev_div_scalar, void *x, void *stream) {
  if (n <= 0) return 0;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const int cplx = dtype_is_complex(dtype);
  const int64_t nreal = cplx ? 2 * n : n;
  if (dtype == QB_F64 || dtype == QB_C128)
    scale_kernel<double><<<ew_blocks(nreal), 256, 0, st>>>(
        nreal, alpha[0], alpha[1], (const double *)dev_div_scalar, cplx, (double *)x);
  else if (dtype == QB_F32 || dtype == QB_C64)
    scale_kernel<float><<<ew_blocks(nreal), 256, 0, st>>>(
        nreal, (float)alpha[0], (float)alpha[1], (const float *)dev_div_scalar, cplx, (float *)x);
  else { set_error("qb_scale: bad dtype"); return -1; }
  QB_LAUNCH_CHECK();
  return 0;
}

// y = x * alpha / (*div)  (real factor; complex data as 2 n reals): the
// normalised copy of a Krylov residual in one pass instead of copy + scale
int qb_scale_into(int dtype, int64_t n, double alpha, const void *dev_div_scalar,
                  const void *x, void *y, void *stream) {
  if (n <= 0) return 0;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const int64_t nreal = dtype_is_complex(dtype) ? 2 * n : n;
  if (dtype == QB_F64 || dtype == QB_C128)
    scale_into_kernel<double><<<ew_blocks(nreal), 256, 0, st>>>(
        nreal, alpha, (const double *)dev_div_scalar, (const double *)x, (double *)y);
  else if (dtype == QB_F32 || dtype == QB_C64)
    scale_into_kernel<float><<<ew_blocks(nreal), 256, 0, st>>>(
        nreal, (float)alpha, (const float *)dev_div_scalar, (const float *)x, (float *)y);
  else { set_error("qb_scale_into: bad dtype"); return -1; }
  QB_LAUNCH_CHECK();
  return 0;
}

int64_t qb_dot_workspace(int64_t n) { (void)n; return (int64_t)DOT_BLOCKS * 2 * 8; }

int qb_dot(int dtype, int64_t n, const void *x, const void *y, void *out,
           void *workspace, void *stream) {
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (!workspace) { set_error("qb_dot: workspace required"); return -6; }
  double *part = static_cast<double *>(workspace);
  switch (dtype) {
    case QB_F64:
      dot_stage1_kernel<double, 0><<<DOT_BLOCKS, 256, 0, st>>>(n, (const double *)x, (const double *)y, part);
      QB_LAUNCH_CHECK();
      dot_stage2_kernel<double, 0><<<1, 256, 0, st>>>(DOT_BLOCKS, part, (double *)out);
      break;
    case QB_F32:
      dot_stage1_kernel<float, 0><<<DOT_BLOCKS, 256, 0, st>>>(n, (const float *)x, (const float *)y, part);
      QB_LAUNCH_CHECK();
      dot_stage2_kernel<float, 0><<<1, 256, 0, st>>>(DOT_BLOCKS, part, (float *)out);
      break;
    case QB_C128:
      dot_stage1_kernel<double, 1><<<DOT_BLOCKS, 256, 0, st>>>(n, (const double *)x, (const double *)y, part);
      QB_LAUNCH_CHECK();
      dot_stage2_kernel<double, 1><<<1, 256, 0, st>>>(DOT_BLOCKS, part, (double *)out);
      break;
    case QB_C64:
      dot_stage1_kernel<float, 1><<<DOT_BLOCKS, 256, 0, st>>>(n, (const float *)x, (const float *)y, part);
      QB_LAUNCH_CHECK();
      dot_stage2_kernel<float, 1><<<1, 256, 0, st>>>(DOT_BLOCKS, part, (float *)out);
      break;
    default: set_error("qb_dot: bad dtype"); return -1;
  }
  QB_LAUNCH_CHECK();
  return 0;
}

int qb_scale_diag(int dtype, int64_t rows, int64_t cols, void *x,
                  const void *d, int side, int sqrt_d, void *stream) {
  if (rows * cols <= 0) return 0;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const int epr = dtype_is_complex(dtype) ? 2 : 1;
  if (dtype == QB_F64 || dtype == QB_C128)
    scale_diag_kernel<double><<<ew_blocks(rows * cols), 256, 0, st>>>(
        rows, cols, epr, (double *)x, (const double *)d, side, sqrt_d);
  else if (dtype == QB_F32 || dtype == QB_C64)
    scale_diag_kernel<float><<<ew_blocks(rows * cols), 256, 0, st>>>(
        rows, cols, epr, (float *)x, (const float *)d, side, sqrt_d);
  else { set_error("qb_scale_diag: bad dtype"); return -1; }
  QB_LAUNCH_CHECK();
  return 0;
}

}  // extern "C"

// ------------------------------------------------- Lanczos block algebra ----
// h[j] = <V[j], w>  for j < m  (V is m x n row-major, real fp64), one pass
// over V and w; deterministic two-stage reduction.
namespace qb {
constexpr int MD_MAX = 16;
constexpr int MD_BLOCKS = 592;

__global__ void __launch_bounds__(256)
    multi_dot_stage1(int m, int64_t n, const double *__restrict__ V, int64_t ldv,
                     const double *__restrict__ w, double *__restrict__ part) {
  double acc[MD_MAX];
#pragma unroll
  for (int j = 0; j < MD_MAX; ++j) acc[j] = 0.0;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n;
       i += (int64_t)gridDim.x * blockDim.x) {
    const double wi = w[i];
#pragma unroll
    for (int j = 0; j < MD_MAX; ++j)
      if (j < m) acc[j] += V[(int64_t)j * ldv + i] * wi;
  }
  __shared__ double sh[8][MD_MAX];
#pragma unroll
  for (int j = 0; j < MD_MAX; ++j) {
    double v = (j < m) ? warp_sum(acc[j]) : 0.0;
    if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5][j] = v;
  }
  __syncthreads();
  if (threadIdx.x < m) {
    double s = 0.0;
    for (int wv = 0; wv < 8; ++wv) s += sh[wv][threadIdx.x];
    part[(int64_t)blockIdx.x * MD_MAX + threadIdx.x] = s;
  }
}
__global__ void __launch_bounds__(256)
    multi_dot_stage2(int m, int nparts, const double *__restrict__ part,
                     double *__restrict__ out) {
  __shared__ double sh[256];
  for (int j = 0; j < m; ++j) {
    double a = 0.0;
    for (int i = threadIdx.x; i < nparts; i += 256) a += part[(int64_t)i * MD_MAX + j];
    sh[threadIdx.x] = a;
    __syncthreads();
    for (int s = 128; s > 0; s >>= 1) {
      if (threadIdx.x < s) sh[threadIdx.x] += sh[threadIdx.x + s];
      __syncthreads();
    }
    if (threadIdx.x == 0) out[j] = sh[0];
    __syncthreads();
  }
}
// w[i] += alpha * sum_j h[j] * V[j][i]   (h on the device)
__global__ void __launch_bounds__(256)
    multi_axpy_kernel(int m, int64_t n, const double *__restrict__ V, int64_t ldv,
                      const double *__restrict__ h, double alpha, double *__restrict__ w) {
  double hj[MD_MAX];
#pragma unroll
  for (int j = 0; j < MD_MAX; ++j) hj[j] = (j < m) ? alpha * h[j] : 0.0;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n;
       i += (int64_t)gridDim.x * blockDim.x) {
    double s = w[i];
#pragma unroll
    for (int j = 0; j < MD_MAX; ++j)
      if (j < m) s += hj[j] * V[(int64_t)j * ldv + i];
    w[i] = s;
  }
}
}  // namespace qb

extern "C" {

int64_t qb_multi_dot_workspace(void) { return (int64_t)qb::MD_BLOCKS * qb::MD_MAX * 8; }

int qb_multi_dot(int dtype, int m, int64_t n, const void *V, int64_t ldv,
                 const void *w, void *out, void *workspace, void *stream) {
  using namespace qb;
  if (dtype != QB_F64) { set_error("qb_multi_dot: f64 only"); return -1; }
  if (m < 1 || m > MD_MAX) { set_error("qb_multi_dot: 1 <= m <= %d", MD_MAX); return -2; }
  if (!workspace) { set_error("qb_multi_dot: workspace required"); return -8; }
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  multi_dot_stage1<<<MD_BLOCKS, 256, 0, st>>>(m, n, (const double *)V, ldv,
                                              (const double *)w, (double *)workspace);
  QB_LAUNCH_CHECK();
  multi_dot_stage2<<<1, 256, 0, st>>>(m, MD_BLOCKS, (const double *)workspace, (double *)out);
  QB_LAUNCH_CHECK();
  return 0;
}

int qb_multi_axpy(int dtype, int m, int64_t n, const void *V, int64_t ldv,
                  const void *h, double alpha, void *w, void *stream) {
  using namespace qb;
  if (dtype != QB_F64) { set_error("qb_multi_axpy: f64 only"); return -1; }
  if (m < 1 || m > MD_MAX) { set_error("qb_multi_axpy: 1 <= m <= %d", MD_MAX); return -2; }
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  int64_t b = (n + 255) / 256;
  if (b > (int64_t)sm_count() * 8) b = (int64_t)sm_count() * 8;
  multi_axpy_kernel<<<(unsigned)b, 256, 0, st>>>(m, n, (const double *)V, ldv,
                                                 (const double *)h, alpha, (double *)w);
  QB_LAUNCH_CHECK();
  return 0;
}

}  // extern "C"
