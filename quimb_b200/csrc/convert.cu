// Precision conversion passes (HBM bound).  f32 / c64 tensors are contracted
// by widening them to f64 / c128 (exact), running the fp64 engines and
// rounding the result once -- every intermediate product/sum is carried in
// fp64, so results are at least as accurate as the reference's fp32 path.
// Shapes above its tile minimum take the native int8 engine (ozaki_tc.cu).
#include "common.cuh"

namespace qb {

template <typename S, typename D>
__global__ void __launch_bounds__(256)
    convert_contig_kernel(const S *__restrict__ src, D *__restrict__ dst, int64_t n) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n;
       i += (int64_t)gridDim.x * blockDim.x)
    dst[i] = (D)src[i];
}

}  // namespace qb

using namespace qb;

extern "C" int qb_convert(int src_dtype, int dst_dtype, int64_t n, const void *src,
                          void *dst, void *stream) {
  // contiguous conversion between f32<->f64 and c64<->c128 (complex data is
  // converted as 2n reals)
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (n <= 0) return 0;
  int64_t nr = n;
  bool widen;
  if (src_dtype == QB_F32 && dst_dtype == QB_F64) widen = true;
  else if (src_dtype == QB_F64 && dst_dtype == QB_F32) widen = false;
  else if (src_dtype == QB_C64 && dst_dtype == QB_C128) { widen = true; nr = 2 * n; }
  else if (src_dtype == QB_C128 && dst_dtype == QB_C64) { widen = false; nr = 2 * n; }
  else {
    set_error("qb_convert: unsupported conversion %d -> %d", src_dtype, dst_dtype);
    return -1;
  }
  int64_t b = (nr + 255) / 256;
  if (b > (int64_t)sm_count() * 8) b = (int64_t)sm_count() * 8;
  if (widen)
    convert_contig_kernel<float, double><<<(unsigned)b, 256, 0, st>>>(
        (const float *)src, (double *)dst, nr);
  else
    convert_contig_kernel<double, float><<<(unsigned)b, 256, 0, st>>>(
        (const double *)src, (float *)dst, nr);
  QB_LAUNCH_CHECK();
  return 0;
}

// ---- complex <-> real-embedding helpers -------------------------------------
// Complex QR / SVD run on the real kernels through the interleaved embedding
//   E[2i+a, 2j+b] = [[re, -im], [im, re]][a][b]  of z[i, j]:
// the stabilised real QR of E is the embedding of the stabilised complex QR
// (uniqueness for positive diagonal), and every real singular vector of E is
// the image of a complex singular vector of z.
namespace qb {

__global__ void __launch_bounds__(256)
    embed_complex_kernel(const double2 *__restrict__ z, int64_t m, int64_t n,
                         double *__restrict__ E) {
  const int64_t total = m * n;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total;
       i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t r = i / n, c = i - r * n;
    const double2 v = z[i];
    double *row0 = E + (2 * r) * (2 * n) + 2 * c;
    double *row1 = row0 + 2 * n;
    *reinterpret_cast<double2 *>(row0) = make_double2(v.x, -v.y);
    *reinterpret_cast<double2 *>(row1) = make_double2(v.y, v.x);
  }
}

// out[i, c] = E[2i, c*cs] + 1j * E[2i+1, c*cs],  i < m, c < ncols
__global__ void __launch_bounds__(256)
    extract_complex_kernel(const double *__restrict__ E, int64_t ld, int64_t m,
                           int64_t ncols, int64_t cs, double2 *__restrict__ out) {
  const int64_t total = m * ncols;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total;
       i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t r = i / ncols, c = i - r * ncols;
    out[i] = make_double2(E[(2 * r) * ld + c * cs], E[(2 * r + 1) * ld + c * cs]);
  }
}

}  // namespace qb

extern "C" int qb_embed_complex(int64_t m, int64_t n, const void *z, void *E,
                                void *stream) {
  using namespace qb;
  if (m * n <= 0) return 0;
  int64_t b = (m * n + 255) / 256;
  if (b > (int64_t)sm_count() * 8) b = (int64_t)sm_count() * 8;
  embed_complex_kernel<<<(unsigned)b, 256, 0, static_cast<cudaStream_t>(stream)>>>(
      (const double2 *)z, m, n, (double *)E);
  QB_LAUNCH_CHECK();
  return 0;
}

extern "C" int qb_extract_complex(int64_t m, int64_t ncols, int64_t col_step,
                                  const void *E, int64_t ld, void *out, void *stream) {
  using namespace qb;
  if (m * ncols <= 0) return 0;
  int64_t b = (m * ncols + 255) / 256;
  if (b > (int64_t)sm_count() * 8) b = (int64_t)sm_count() * 8;
  extract_complex_kernel<<<(unsigned)b, 256, 0, static_cast<cudaStream_t>(stream)>>>(
      (const double *)E, ld, m, ncols, col_step, (double2 *)out);
  QB_LAUNCH_CHECK();
  return 0;
}
