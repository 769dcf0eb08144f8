// The per-term evaluation of PEPS.compute_local_expectation
// (quimb/tensor/tn2d/core.py:4335-4348): for every term t of a call,
//
//   out[2 t]     = sum_{m, a} G_t[a, b(m)] * rho_p[m, n(m, a)]   = Tr[G_t rho_p]
//   out[2 t + 1] = sum_m rho_p[m, m]                              = Tr[rho_p]
//
// rho_p is the reduced density matrix of the term's plaquette p (ket index
// m, bra index n, each the C-ordered multi-index of the plaquette's sites),
// b(m) is the term's part of m and n(m, a) is m with that part replaced by a:
// the sites outside the term are traced, so a bond on its own 1x2 plaquette,
// a site on a 1x2 plaquette and a diagonal pair on a 2x2 plaquette are one
// code path.  The reference instead contracts the whole gated plaquette
// network once per term.
//
// One warp per term.  The D dg products (dg = the term's dimension) are summed
// lane-strided in index order, then by a fixed butterfly; the trace likewise.
// The order depends only on the descriptor, so the bits depend only on the
// inputs, never on the grid, the stream or the launch history, and a NaN or
// Inf reaches only the terms whose rho or G holds it.
#include "common.cuh"

namespace qb {

constexpr int PLAQ_THREADS = 256;
constexpr int PLAQ_WARPS = PLAQ_THREADS / 32;

__device__ __forceinline__ double pq_zero(double) { return 0.0; }
__device__ __forceinline__ double2 pq_zero(double2) { return make_double2(0.0, 0.0); }
// acc += g * r
__device__ __forceinline__ void pq_fma(double &acc, double g, double r) { acc = fma(g, r, acc); }
__device__ __forceinline__ void pq_fma(double2 &acc, double2 g, double2 r) {
  acc.x = fma(g.x, r.x, fma(-g.y, r.y, acc.x));
  acc.y = fma(g.x, r.y, fma(g.y, r.x, acc.y));
}
__device__ __forceinline__ double pq_add(double a, double b) { return a + b; }
__device__ __forceinline__ double2 pq_add(double2 a, double2 b) {
  return make_double2(a.x + b.x, a.y + b.y);
}
__device__ __forceinline__ double pq_shfl(double v, int o) {
  return __shfl_xor_sync(0xffffffffu, v, o);
}
__device__ __forceinline__ double2 pq_shfl(double2 v, int o) {
  return make_double2(__shfl_xor_sync(0xffffffffu, v.x, o),
                      __shfl_xor_sync(0xffffffffu, v.y, o));
}

template <typename T>
__global__ void __launch_bounds__(PLAQ_THREADS)
    plaquette_expec_kernel(int64_t n_terms, const int64_t *__restrict__ desc,
                           const T *__restrict__ rho, const T *__restrict__ G,
                           T *__restrict__ out) {
  const int lane = threadIdx.x & 31;
  const int64_t t = (int64_t)blockIdx.x * PLAQ_WARPS + (threadIdx.x >> 5);
  if (t >= n_terms) return;   // whole warps exit together
  const int64_t *d = desc + t * QB_PLAQ_DESC_WORDS;
  const T *r = rho + d[0];
  const T *g = G + d[1];
  const int ns = (int)d[2], nt = (int)d[3];
  const int p0 = (int)d[4], p1 = nt == 2 ? (int)d[5] : -1;
  // C-order strides of the plaquette sites, and the term's two (the second
  // a unit-dimension dummy for one-site terms)
  int D = 1, s0 = 1, s1 = 1, d0 = 1, d1 = 1;
  for (int s = ns - 1; s >= 0; --s) {
    const int ds = (int)d[6 + s];
    if (s == p0) { s0 = D; d0 = ds; }
    if (s == p1) { s1 = D; d1 = ds; }
    D *= ds;
  }
  const int dg = d0 * d1;
  T acc = pq_zero(T()), tr = pq_zero(T());
  for (int e = lane; e < D * dg; e += 32) {
    const int m = e / dg, a = e - (e / dg) * dg;
    const int b0 = (m / s0) % d0, b1 = (m / s1) % d1;
    const int a0 = a / d1, a1 = a - (a / d1) * d1;
    const int n = m + (a0 - b0) * s0 + (a1 - b1) * s1;
    pq_fma(acc, __ldg(g + a * dg + b0 * d1 + b1), __ldg(r + m * D + n));
  }
  for (int m = lane; m < D; m += 32) tr = pq_add(tr, __ldg(r + m * D + m));
#pragma unroll
  for (int w = 16; w > 0; w >>= 1) {
    acc = pq_add(acc, pq_shfl(acc, w));
    tr = pq_add(tr, pq_shfl(tr, w));
  }
  if (lane == 0) {
    out[2 * t] = acc;
    out[2 * t + 1] = tr;
  }
}

// every descriptor checked on the host before anything is copied or launched
static int plaquette_check(const int64_t *desc, int64_t n_terms, int64_t rho_elems,
                           int64_t g_elems) {
  for (int64_t t = 0; t < n_terms; ++t) {
    const int64_t *d = desc + t * QB_PLAQ_DESC_WORDS;
    const int64_t ns = d[2], nt = d[3];
    bool ok = ns >= 1 && ns <= QB_PLAQ_MAX_SITES && (nt == 1 || nt == 2);
    int64_t D = 1, dg = 1;
    for (int s = 0; ok && s < ns; ++s) {
      ok = d[6 + s] >= 1 && d[6 + s] <= QB_PLAQ_MAX_DIM;
      D *= ok ? d[6 + s] : 1;
    }
    ok = ok && D <= QB_PLAQ_MAX_DIM && d[4] >= 0 && d[4] < ns;
    ok = ok && (nt == 1 || (d[5] > d[4] && d[5] < ns));
    if (ok) dg = d[6 + d[4]] * (nt == 2 ? d[6 + d[5]] : 1);
    ok = ok && d[0] >= 0 && d[0] <= rho_elems - D * D && d[1] >= 0 && d[1] <= g_elems - dg * dg;
    if (!ok) {
      set_error("qb_plaquette_expec: descriptor of term %lld is invalid (sites %lld, "
                "term sites %lld, rho offset %lld of %lld, G offset %lld of %lld)",
                (long long)t, (long long)ns, (long long)nt, (long long)d[0],
                (long long)rho_elems, (long long)d[1], (long long)g_elems);
      return -3;
    }
  }
  return 0;
}

}  // namespace qb

using namespace qb;

extern "C" int qb_plaquette_expec(int dtype, int64_t n_terms, const int64_t *desc,
                                  void *desc_dev, const void *rho, int64_t rho_elems,
                                  const void *G, int64_t g_elems, void *out, void *stream) {
  if (dtype != QB_F64 && dtype != QB_C128) {
    set_error("qb_plaquette_expec: dtype must be QB_F64 or QB_C128 (got %d)", dtype);
    return -1;
  }
  if (n_terms < 0) {
    set_error("qb_plaquette_expec: n_terms = %lld < 0", (long long)n_terms);
    return -2;
  }
  if (n_terms == 0) return 0;
  const uintptr_t align = dtype == QB_C128 ? 15 : 7;
  auto bad = [&](const void *p, uintptr_t a) {
    return !p || (reinterpret_cast<uintptr_t>(p) & a);
  };
  if (bad(desc, 7) || bad(desc_dev, 7) || bad(rho, align) || bad(G, align) || bad(out, align)) {
    set_error("qb_plaquette_expec: a descriptor, rho, G or out pointer is null or misaligned");
    return -4;
  }
  if (int rc = plaquette_check(desc, n_terms, rho_elems, g_elems)) return rc;
  const int64_t blocks = (n_terms + PLAQ_WARPS - 1) / PLAQ_WARPS;
  if (blocks > 0x7fffffff) {
    set_error("qb_plaquette_expec: %lld terms need more than 2^31 - 1 blocks",
              (long long)n_terms);
    return -2;
  }
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  QB_CUDA_CHECK(cudaMemcpyAsync(desc_dev, desc, (size_t)n_terms * QB_PLAQ_DESC_WORDS * 8,
                                cudaMemcpyHostToDevice, st));
  const int64_t *dd = static_cast<const int64_t *>(desc_dev);
  if (dtype == QB_F64)
    plaquette_expec_kernel<double><<<(unsigned)blocks, PLAQ_THREADS, 0, st>>>(
        n_terms, dd, static_cast<const double *>(rho), static_cast<const double *>(G),
        static_cast<double *>(out));
  else
    plaquette_expec_kernel<double2><<<(unsigned)blocks, PLAQ_THREADS, 0, st>>>(
        n_terms, dd, static_cast<const double2 *>(rho), static_cast<const double2 *>(G),
        static_cast<double2 *>(out));
  QB_LAUNCH_CHECK();
  return 0;
}
