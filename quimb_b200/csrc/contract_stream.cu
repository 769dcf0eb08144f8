// Streaming engine for "apply a small operator to a big tensor" contractions:
//   C[m, n] = alpha * sum_k op(A)[m, k] * op(B)[k, n] + beta * C[m, n]
// with N, K <= 32 (real) or N, K <= 16 (complex) (gate application in
// circuit trees, MPO legs, physical indices: the steps cotengra's pairwise loop issues for
// quimb/tensor/circuit/exact.py amplitudes, tensor_core.py:3786-3808).  Such a
// step moves (M*K + M*N) elements for 2*M*N*K flops -- arithmetic intensity
// of a few flop/byte, i.e. HBM-bound, and a 128 x 32 DMMA tile would spend
// most of its MMA slots and shared-memory traffic on padding.  Here every
// thread owns output rows: it gathers the K inputs of a row straight from
// global memory through the planner's mode strides (no transpose, no staging),
// multiplies by the operator held in shared memory and writes the N outputs.
//
// The row arithmetic, the table fill and the batch addressing are
// __host__ __device__ functions shared by the kernel and by a host executor
// (qb_debug_contract_stream_host: TEST entry on host pointers, used by the
// CPU tier to check the index bookkeeping against numpy; the product never
// calls it).
//
// Status: selected only on explicit request (QB_ENGINE_STREAM, or
// QB_ENGINE=stream in the environment): it has not been timed against the
// DMMA path on the H100.
#include <cuda_runtime.h>

#include "internal.h"


namespace qb {

#define QB_HD __host__ __device__ __forceinline__

// mixed-radix decode of a linear group index into two element offsets
// (mode 0 varies fastest), host + device
QB_HD void sdecode2(int64_t idx, const ModeGroup &g, int64_t &o0, int64_t &o1) {
  int64_t a = 0, b = 0;
  for (int i = 0; i < g.n; ++i) {
    const int64_t e = g.ext[i];
    const int64_t q = idx / e;
    const int64_t d = idx - q * e;
    a += d * g.s0[i];
    b += d * g.s1[i];
    idx = q;
  }
  o0 = a;
  o1 = b;
}

// base pointers of batch entry zb (in doubles)
template <bool CPLX>
QB_HD void stream_batch_base(const ContractParams &p, int64_t zb, const double *&A,
                             const double *&B, double *&C) {
  constexpr int ES = CPLX ? 2 : 1;
  A = static_cast<const double *>(p.A);
  B = static_cast<const double *>(p.B);
  C = static_cast<double *>(p.C);
  if (p.dA) {
    A = static_cast<const double *>(p.dA[zb]);
    B = static_cast<const double *>(p.dB[zb]);
    C = static_cast<double *>(p.dC[zb]);
  } else if (p.b.n) {
    int64_t oa, ob, oc = 0;
    sdecode2(zb, p.b, oa, ob);
    int64_t r = zb;
    for (int i = 0; i < p.b.n; ++i) {
      const int64_t e = p.b.ext[i];
      const int64_t q = r / e;
      oc += (r - q * e) * p.bsC[i];
      r = q;
    }
    A += oa * ES;
    B += ob * ES;
    C += oc * ES;
  }
}

// operator table Bs[k][n] (conjugation applied), A offsets of the K inputs of a
// row and C offsets of its N outputs; entries tid, tid + nthr, ...
template <bool CPLX>
QB_HD void stream_fill_tables(const ContractParams &p, const double *B, int tid, int nthr,
                              double *Bs, int64_t *kOffA, int64_t *nOffC) {
  constexpr int ES = CPLX ? 2 : 1;
  const int K = (int)p.K, N = (int)p.N;
  for (int i = tid; i < K * N; i += nthr) {
    const int k = i / N, n = i - k * N;
    int64_t oa, obk, obn, oc;
    sdecode2(k, p.k, oa, obk);
    sdecode2(n, p.n, obn, oc);
    const double *src = B + (obk + obn) * ES;
    Bs[i * ES] = src[0];
    if (CPLX) Bs[i * ES + 1] = p.conjB ? -src[1] : src[1];
  }
  for (int i = tid; i < K; i += nthr) {
    int64_t oa, ob;
    sdecode2(i, p.k, oa, ob);
    kOffA[i] = oa * ES;
  }
  for (int i = tid; i < N; i += nthr) {
    int64_t ob, oc;
    sdecode2(i, p.n, ob, oc);
    nOffC[i] = oc * ES;
  }
}

// one output row
template <bool CPLX, int KMAX, int NMAX>
QB_HD void stream_row(const ContractParams &p, const double *A, double *C, int64_t m,
                      const double *Bs, const int64_t *kOffA, const int64_t *nOffC) {
  constexpr int ES = CPLX ? 2 : 1;
  const int K = (int)p.K, N = (int)p.N;
  int64_t oa, oc;
  sdecode2(m, p.m, oa, oc);
  oa *= ES;
  oc *= ES;
  double ar[KMAX], ai[KMAX];
#pragma unroll
  for (int k = 0; k < KMAX; ++k) {
    ar[k] = 0.0;
    ai[k] = 0.0;
    if (k < K) {
      const double *src = A + oa + kOffA[k];
      ar[k] = src[0];
      if (CPLX) ai[k] = p.conjA ? -src[1] : src[1];
    }
  }
  const double alpha = p.alpha, beta = p.beta;
  // small operators: fully unrolled; 16 outputs: a rolled loop keeps the
  // register count (and with it the occupancy of this HBM-bound kernel) in check
#pragma unroll(NMAX <= 4 ? NMAX : 1)
  for (int n = 0; n < NMAX; ++n) {
    if (n < N) {
      double cr = 0.0, ci = 0.0;
#pragma unroll
      for (int k = 0; k < KMAX; ++k) {
        if (k < K) {
          const double br = Bs[(k * N + n) * ES];
          if (CPLX) {
            const double bi = Bs[(k * N + n) * ES + 1];
            cr += ar[k] * br - ai[k] * bi;
            ci += ar[k] * bi + ai[k] * br;
          } else {
            cr += ar[k] * br;
          }
        }
      }
      double *dst = C + oc + nOffC[n];
      if (beta != 0.0) {
        dst[0] = alpha * cr + beta * dst[0];
        if (CPLX) dst[1] = alpha * ci + beta * dst[1];
      } else {
        dst[0] = alpha * cr;
        if (CPLX) dst[1] = alpha * ci;
      }
    }
  }
}

constexpr int kStreamThreads = 256;

template <bool CPLX, int KMAX, int NMAX>
__global__ void __launch_bounds__(kStreamThreads)
contract_stream_kernel(const __grid_constant__ ContractParams p) {
  constexpr int ES = CPLX ? 2 : 1;
  __shared__ double Bs[KMAX * NMAX * ES];
  __shared__ int64_t kOffA[KMAX];
  __shared__ int64_t nOffC[NMAX];
  const int tid = threadIdx.x;
  for (int64_t zb = blockIdx.y; zb < p.nbatch; zb += gridDim.y) {
    const double *A, *B;
    double *C;
    stream_batch_base<CPLX>(p, zb, A, B, C);
    __syncthreads();  // the previous batch entry is done with the tables
    stream_fill_tables<CPLX>(p, B, tid, kStreamThreads, Bs, kOffA, nOffC);
    __syncthreads();
    for (int64_t m = (int64_t)blockIdx.x * kStreamThreads + tid; m < p.M;
         m += (int64_t)gridDim.x * kStreamThreads)
      stream_row<CPLX, KMAX, NMAX>(p, A, C, m, Bs, kOffA, nOffC);
  }
}

bool stream_eligible(const PairPlan &plan) {
  const ContractParams &p = plan.p;
  // real operators up to 32 x 32 (the (w d d) = 20-wide MPO step of the DMRG
  // two-site matvec), complex ones up to 16 x 16 (register budget)
  const int lim = plan.dtype == QB_F64 ? 32 : 16;
  return (plan.dtype == QB_F64 || plan.dtype == QB_C128) && p.N >= 1 && p.K >= 1 &&
         p.N <= lim && p.K <= lim && p.M >= 1;
}

template <bool CPLX, int KMAX, int NMAX>
static int launch_stream_t(const ContractParams &p, cudaStream_t st) {
  const int sms = sm_count();
  const int64_t want = (p.M + kStreamThreads - 1) / kStreamThreads;
  const int64_t cap = (int64_t)sms * 8;  // 8 resident CTAs of 256 threads per SM
  dim3 grid((unsigned)std::max<int64_t>(1, std::min<int64_t>(want, cap)),
            (unsigned)std::max<int64_t>(1, std::min<int64_t>(p.nbatch, 65535)));
  contract_stream_kernel<CPLX, KMAX, NMAX><<<grid, kStreamThreads, 0, st>>>(p);
  QB_LAUNCH_CHECK();
  return 0;
}

StreamVariant stream_variant(const ContractParams &p) {
  if (p.N <= 4 && p.K <= 4) return {4, 4};
  if (p.N <= 4 && p.K <= 16) return {16, 4};
  if (p.K <= 4 && p.N <= 16) return {4, 16};
  if (p.N <= 16 && p.K <= 16) return {16, 16};
  return {32, 32};
}

template <bool CPLX>
static int launch_stream_c(const PairPlan &plan, cudaStream_t st) {
  ContractParams p = plan.p;
  p.splitk = 1;
  p.partial = nullptr;
  const StreamVariant v = stream_variant(p);
  if (v.kmax == 4 && v.nmax == 4) return launch_stream_t<CPLX, 4, 4>(p, st);
  if (v.kmax == 16 && v.nmax == 4) return launch_stream_t<CPLX, 16, 4>(p, st);
  if (v.kmax == 4 && v.nmax == 16) return launch_stream_t<CPLX, 4, 16>(p, st);
  if (v.kmax == 16 && v.nmax == 16) return launch_stream_t<CPLX, 16, 16>(p, st);
  if constexpr (!CPLX) return launch_stream_t<false, 32, 32>(p, st);
  return -9;
}

int launch_contract_stream(const PairPlan &plan, cudaStream_t st) {
  if (!stream_eligible(plan)) {
    set_error("streaming engine: needs N, K <= 32 (real) / 16 (complex) (got N = %lld, K = %lld)",
              (long long)plan.p.N, (long long)plan.p.K);
    return -9;
  }
  if (plan.dtype == QB_F64) return launch_stream_c<false>(plan, st);
  return launch_stream_c<true>(plan, st);
}

// ---- host executor of the same row functions (TEST entry) -----------------
template <bool CPLX>
static void stream_host_t(const ContractParams &p) {
  constexpr int ES = CPLX ? 2 : 1;
  double Bs[32 * 32 * ES];
  int64_t kOffA[32], nOffC[32];
  const StreamVariant v = stream_variant(p);
  for (int64_t zb = 0; zb < p.nbatch; ++zb) {
    const double *A, *B;
    double *C;
    stream_batch_base<CPLX>(p, zb, A, B, C);
    stream_fill_tables<CPLX>(p, B, 0, 1, Bs, kOffA, nOffC);
    for (int64_t m = 0; m < p.M; ++m) {
      if (v.kmax == 4 && v.nmax == 4) stream_row<CPLX, 4, 4>(p, A, C, m, Bs, kOffA, nOffC);
      else if (v.kmax == 16 && v.nmax == 4) stream_row<CPLX, 16, 4>(p, A, C, m, Bs, kOffA, nOffC);
      else if (v.kmax == 4 && v.nmax == 16) stream_row<CPLX, 4, 16>(p, A, C, m, Bs, kOffA, nOffC);
      else if (v.kmax == 16 && v.nmax == 16) stream_row<CPLX, 16, 16>(p, A, C, m, Bs, kOffA, nOffC);
      else stream_row<CPLX, 32, 32>(p, A, C, m, Bs, kOffA, nOffC);
    }
  }
}

int contract_stream_host(const PairPlan &plan) {
  if (!stream_eligible(plan)) return -9;
  ContractParams p = plan.p;
  if (p.dA) return -9;
  if (plan.dtype == QB_F64) stream_host_t<false>(p);
  else if (plan.dtype == QB_C128) stream_host_t<true>(p);
  else return -9;
  return 0;
}

}  // namespace qb
