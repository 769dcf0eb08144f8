// The last step of every reduced density matrix of an MPS
// (MatrixProductState.partial_trace_to_dense_canonical / local expectations,
// quimb/tensor/tn1d/core.py:2827-3087):
//
//   out[m, n] = sum_{a < n1, b < n2} U[a, m, b] * conj(V[a, n, b])
//
// with M, N <= 64 and a summed extent K = n1 * n2 that reaches 2^20 at
// chi = 1024.  On the contraction engine this is an M = N = D GEMM padded to
// a 32 x 32 tile plus a split-K reduction; here U and V are read once.
//
// Pass 1: G blocks, each owning a contiguous run of K-tiles of TK columns.
// A tile is staged in shared memory (Us[M][TK], Vs[N][TK]; k = a * n2 + b, b
// fastest, so a contiguous b axis is read coalesced).  Thread t owns the
// outputs t, t + 256, ... (M N >= 256) or, for smaller M N, output t % (M N)
// on k-lane t / (M N); lanes are summed in lane order at the end of the block.
// Pass 2 (only when G > 1): one warp per output sums the G partials
// lane-strided, then a fixed butterfly.  TK and G are functions of
// (n1, M, N, n2) alone, so the bits never depend on the device, the stream,
// the launch history or whether U aliases V.
#include <algorithm>

#include "common.cuh"

namespace qb {

constexpr int RDM_THREADS = 256;
constexpr int RDM_MAX_MN = 64;
constexpr int RDM_MAX_OPT = RDM_MAX_MN * RDM_MAX_MN / RDM_THREADS;   // outputs / thread
constexpr int64_t RDM_SMEM_BYTES = 32 * 1024;                         // at 16 B / element
constexpr int64_t RDM_MAX_TK = 1024;
constexpr int64_t RDM_MAX_BLOCKS = 1024;

struct RdmShape {
  int64_t tk, tiles, blocks;
};

static RdmShape rdm_shape(int64_t n1, int64_t M, int64_t N, int64_t n2) {
  RdmShape s;
  int64_t tk = RDM_SMEM_BYTES / ((M + N) * 16);
  int64_t p = 1;
  while (p * 2 <= std::min(tk, RDM_MAX_TK)) p *= 2;
  s.tk = p;
  s.tiles = (n1 * n2 + s.tk - 1) / s.tk;
  s.blocks = std::min(s.tiles, RDM_MAX_BLOCKS);
  return s;
}

__device__ __forceinline__ double ld_elem(const double *p) { return __ldg(p); }
__device__ __forceinline__ double2 ld_elem(const double2 *p) { return __ldg(p); }
__device__ __forceinline__ double zero_elem(double) { return 0.0; }
__device__ __forceinline__ double2 zero_elem(double2) { return make_double2(0.0, 0.0); }
// acc += u * conj(v)
__device__ __forceinline__ void fma_conj(double &acc, double u, double v) {
  acc = fma(u, v, acc);
}
__device__ __forceinline__ void fma_conj(double2 &acc, double2 u, double2 v) {
  acc.x = fma(u.x, v.x, fma(u.y, v.y, acc.x));
  acc.y = fma(u.y, v.x, fma(-u.x, v.y, acc.y));
}
__device__ __forceinline__ double add_elem(double a, double b) { return a + b; }
__device__ __forceinline__ double2 add_elem(double2 a, double2 b) {
  return make_double2(a.x + b.x, a.y + b.y);
}
__device__ __forceinline__ double shfl_xor(double v, int o) {
  return __shfl_xor_sync(0xffffffffu, v, o);
}
__device__ __forceinline__ double2 shfl_xor(double2 v, int o) {
  return make_double2(__shfl_xor_sync(0xffffffffu, v.x, o),
                      __shfl_xor_sync(0xffffffffu, v.y, o));
}

struct RdmArgs {
  int64_t n1, n2, K, tk, tiles;
  int M, N;
  int64_t us0, us1, us2, vs0, vs1, vs2;
  const void *U, *V;
  void *dst;   // out (one block) or the partials, blocks x M N
};

template <typename T, bool ALIAS>
__global__ void __launch_bounds__(RDM_THREADS, 2) rdm_partial_kernel(RdmArgs g) {
  extern __shared__ __align__(16) unsigned char rdm_smem[];
  __shared__ T red[RDM_THREADS];
  T *Us = reinterpret_cast<T *>(rdm_smem);
  T *Vs = ALIAS ? Us : Us + (int64_t)g.M * g.tk;
  const T *U = static_cast<const T *>(g.U);
  const T *V = static_cast<const T *>(g.V);
  const int t = threadIdx.x;
  const int tk = (int)g.tk;
  const int P = g.M * g.N;
  const int lanes = P >= RDM_THREADS ? 1 : RDM_THREADS / P;
  const int lane = P >= RDM_THREADS ? 0 : t / P;
  const int nout = P >= RDM_THREADS ? (P - t + RDM_THREADS - 1) / RDM_THREADS
                                    : (lane < lanes ? 1 : 0);
  T acc[RDM_MAX_OPT];
#pragma unroll
  for (int j = 0; j < RDM_MAX_OPT; ++j) acc[j] = zero_elem(T());

  const int64_t t0 = (int64_t)blockIdx.x * g.tiles / gridDim.x;
  const int64_t t1 = ((int64_t)blockIdx.x + 1) * g.tiles / gridDim.x;
  // loader: cw columns per pass, thread t on column t % cw and rows
  // t / cw, t / cw + 256 / cw, ...; one (a, b) division per column
  const int cw = min(tk, RDM_THREADS);
  const int r0 = t / cw, rstep = RDM_THREADS / cw;
  for (int64_t tile = t0; tile < t1; ++tile) {
    const int64_t k0 = tile * g.tk;
    const int len = (int)(g.K - k0 < g.tk ? g.K - k0 : g.tk);
    for (int kk = t % cw; kk < len; kk += cw) {
      const int64_t k = k0 + kk;
      const int64_t a = k / g.n2, b = k - a * g.n2;
      const T *ub = U + a * g.us0 + b * g.us2;
      for (int m = r0; m < g.M; m += rstep) Us[m * tk + kk] = ld_elem(ub + m * g.us1);
      if (!ALIAS) {
        const T *vb = V + a * g.vs0 + b * g.vs2;
        for (int n = r0; n < g.N; n += rstep) Vs[n * tk + kk] = ld_elem(vb + n * g.vs1);
      }
    }
    __syncthreads();
#pragma unroll
    for (int j = 0; j < RDM_MAX_OPT; ++j) {
      if (j < nout) {
        const int o = P >= RDM_THREADS ? t + j * RDM_THREADS : t % P;
        const T *ur = Us + (o / g.N) * tk;
        const T *vr = Vs + (o % g.N) * tk;
        T s = acc[j];
        for (int kk = lane; kk < len; kk += lanes) fma_conj(s, ur[kk], vr[kk]);
        acc[j] = s;
      }
    }
    __syncthreads();
  }

  T *dst = static_cast<T *>(g.dst) + (int64_t)blockIdx.x * P;
  if (P >= RDM_THREADS) {
#pragma unroll
    for (int j = 0; j < RDM_MAX_OPT; ++j)
      if (j < nout) dst[t + j * RDM_THREADS] = acc[j];
  } else {
    if (lane < lanes) red[t] = acc[0];
    __syncthreads();
    if (t < P) {
      T s = red[t];
      for (int l = 1; l < lanes; ++l) s = add_elem(s, red[l * P + t]);
      dst[t] = s;
    }
  }
}

template <typename T>
__global__ void __launch_bounds__(RDM_THREADS)
    rdm_final_kernel(const T *__restrict__ part, int64_t blocks, int P, T *__restrict__ out) {
  const int lane = threadIdx.x & 31;
  const int o = blockIdx.x * (RDM_THREADS / 32) + (threadIdx.x >> 5);
  if (o >= P) return;   // whole warps exit together
  T s = zero_elem(T());
  for (int64_t b = lane; b < blocks; b += 32) s = add_elem(s, part[b * P + o]);
#pragma unroll
  for (int w = 16; w > 0; w >>= 1) s = add_elem(s, shfl_xor(s, w));
  if (lane == 0) out[o] = s;
}

template <typename T>
static int rdm_launch(const RdmArgs &g0, bool alias, int64_t blocks, void *out, void *ws,
                       cudaStream_t st) {
  RdmArgs g = g0;
  g.dst = blocks > 1 ? ws : out;
  const size_t smem = (size_t)((alias ? g.M : g.M + g.N) * g.tk) * sizeof(T);
  if (alias)
    rdm_partial_kernel<T, true><<<(unsigned)blocks, RDM_THREADS, smem, st>>>(g);
  else
    rdm_partial_kernel<T, false><<<(unsigned)blocks, RDM_THREADS, smem, st>>>(g);
  QB_LAUNCH_CHECK();
  if (blocks > 1) {
    const int P = g.M * g.N;
    const unsigned fb = (unsigned)((P + RDM_THREADS / 32 - 1) / (RDM_THREADS / 32));
    rdm_final_kernel<T><<<fb, RDM_THREADS, 0, st>>>(static_cast<const T *>(ws), blocks, P,
                                                     static_cast<T *>(out));
    QB_LAUNCH_CHECK();
  }
  return 0;
}

static int rdm_check_shape(const char *who, int64_t n1, int64_t M, int64_t N, int64_t n2) {
  if (M < 1 || M > RDM_MAX_MN || N < 1 || N > RDM_MAX_MN) {
    set_error("%s: M = %lld, N = %lld outside [1, %d]", who, (long long)M, (long long)N,
              RDM_MAX_MN);
    return -2;
  }
  if (n1 < 1 || n2 < 1) {
    set_error("%s: n1 = %lld, n2 = %lld must be >= 1", who, (long long)n1, (long long)n2);
    return -3;
  }
  return 0;
}

}  // namespace qb

using namespace qb;

extern "C" int64_t qb_rdm_workspace(int64_t n1, int64_t M, int64_t N, int64_t n2) {
  if (int rc = rdm_check_shape("qb_rdm_workspace", n1, M, N, n2)) return rc;
  const RdmShape s = rdm_shape(n1, M, N, n2);
  return s.blocks > 1 ? s.blocks * M * N * 16 : 0;
}

extern "C" int qb_rdm_reduce(int dtype, int64_t n1, int64_t M, int64_t N, int64_t n2,
                             const void *U, const int64_t ustride[3], const void *V,
                             const int64_t vstride[3], void *out, void *workspace,
                             int64_t ws_bytes, void *stream) {
  if (dtype != QB_F64 && dtype != QB_C128) {
    set_error("qb_rdm_reduce: dtype must be QB_F64 or QB_C128 (got %d)", dtype);
    return -1;
  }
  if (int rc = rdm_check_shape("qb_rdm_reduce", n1, M, N, n2)) return rc;
  const uintptr_t align = dtype == QB_C128 ? 15 : 7;
  auto bad = [&](const void *p) { return !p || (reinterpret_cast<uintptr_t>(p) & align); };
  if (bad(U) || bad(V) || bad(out) || !ustride || !vstride) {
    set_error("qb_rdm_reduce: U, V, out or a stride array is null or misaligned");
    return -4;
  }
  const RdmShape s = rdm_shape(n1, M, N, n2);
  const int64_t need = s.blocks > 1 ? s.blocks * M * N * 16 : 0;
  if (need > 0 && (bad(workspace) || ws_bytes < need)) {
    set_error("qb_rdm_reduce: workspace of %lld bytes given, %lld needed",
              (long long)ws_bytes, (long long)need);
    return -6;
  }
  RdmArgs g;
  g.n1 = n1; g.n2 = n2; g.K = n1 * n2; g.tk = s.tk; g.tiles = s.tiles;
  g.M = (int)M; g.N = (int)N;
  g.us0 = ustride[0]; g.us1 = ustride[1]; g.us2 = ustride[2];
  g.vs0 = vstride[0]; g.vs1 = vstride[1]; g.vs2 = vstride[2];
  g.U = U; g.V = V; g.dst = nullptr;
  const bool alias = U == V && M == N && g.us0 == g.vs0 && g.us1 == g.vs1 && g.us2 == g.vs2;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  return dtype == QB_F64 ? rdm_launch<double>(g, alias, s.blocks, out, workspace, st)
                         : rdm_launch<double2>(g, alias, s.blocks, out, workspace, st);
}
