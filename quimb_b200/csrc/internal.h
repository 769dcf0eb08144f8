// Library-internal helpers shared between translation units.
#pragma once
#include <math.h>
#include <string.h>

#include "common.cuh"
#include "plan.h"

namespace qb {

int launch_contract_f64(const PairPlan &plan, cudaStream_t st);
int launch_contract_c128(const PairPlan &plan, cudaStream_t st);
// a stream-K route runs the pair schedule (2-CTA clusters, one per tile) rather
// than the segment loop; qb_contract_pair_schedule reports it
bool streamk_pair(const PairPlan &plan);
int launch_fill_zero(const qb_tensor_t *C, cudaStream_t st);

// int8 tensor-core (wgmma) error-free-split engine (ozaki_tc.cu)
bool ozaki_eligible(const PairPlan &plan);
int64_t ozaki_workspace_bytes(const PairPlan &plan);
int launch_contract_ozaki(const PairPlan &plan, void *workspace, cudaStream_t st);

// streaming engine for small-operator steps (contract_stream.cu)
bool stream_eligible(const PairPlan &plan);
// compiled (KMAX, NMAX) register-array bounds the launch and the host executor
// pick for an eligible plan; qb_contract_pair_route reports the same pair
struct StreamVariant {
  int kmax, nmax;
};
StreamVariant stream_variant(const ContractParams &p);
int launch_contract_stream(const PairPlan &plan, cudaStream_t st);
int contract_stream_host(const PairPlan &plan);  // TEST: same row code on host pointers

// C(MxN) = alpha * A(MxK) * B(KxN) + beta * C on strided fp64 matrices
// (element strides; any of them may describe a transposed view).
int gemm_f64(const double *A, int64_t a_rs, int64_t a_cs, const double *B,
             int64_t b_rs, int64_t b_cs, double *C, int64_t c_rs, int64_t c_cs,
             int64_t M, int64_t N, int64_t K, double alpha, double beta,
             cudaStream_t st, double *splitk_ws = nullptr,
             int64_t splitk_ws_elems = 0, int max_splitk = 1);

// QB_TRACE=1 tuning buffer (api.cu): 2^20 uint64 stamps, null when tracing is off
unsigned long long *trace_buffer();

// Exponent range of the decompositions (linalg.cu, svd_jacobi.cu).  The
// Householder panels and the Jacobi Gram sum squares of entries over up to
// 2^14 rows, and the Jacobi rotation squares Gram entries again (fast path
// guarded at 1e+-280 ~ 2^+-930).  With max|x| in [2^-200, 2^200] the Gram of
// the leading columns stays within 2^+-414 and its square within 2^+-830, so
// the input is factored as given.  Outside that window (and finite) the input
// is scaled by 2^-e, e = ilogb(max|x|), like LAPACK's dlascl, and the outputs
// are scaled back.  maxbits = the bits of max|x| (a NaN sorts above +inf).
constexpr int kDecompSafeExp = 200;
__host__ __device__ inline bool decomp_finite(unsigned long long maxbits) {
  return maxbits < 0x7FF0000000000000ull;
}
__host__ __device__ inline int decomp_scale_exp(unsigned long long maxbits) {
  if (!decomp_finite(maxbits) || maxbits == 0) return 0;
  double mx;
  memcpy(&mx, &maxbits, sizeof(mx));
  const int e = ilogb(mx);
  return (e < -kDecompSafeExp || e > kDecompSafeExp) ? e : 0;
}

// Householder QR entry shared by qb_qr_stab and the SVD's preconditioner
// (linalg.cu).  keep_scaled: R is left in the units of the scaled input;
// the bits of max|X| are then at qr_maxbits(ws) (device memory).
int qr_f64(int64_t m, int64_t n, const double *X, double *Q, double *R,
           int stabilized, double *ws, cudaStream_t st, bool keep_scaled = false);
int64_t qr_workspace_doubles(int64_t m, int64_t n);
inline unsigned long long *qr_maxbits(double *ws) {
  return reinterpret_cast<unsigned long long *>(ws);
}

// What the Householder QR of an m x n matrix launches (qb_qr_route)
struct QrRoute {
  int nb;           // inner (register-resident) panel width
  int nbo;          // outer (aggregated) panel width
  int64_t nout;     // outer panels
  int64_t npan;     // inner panels
  int panel_mask;   // bit i: panel instantiation i of qr_panel_kind launched
  int wy_t;         // 1: wy_t_kernel forms aggregated T factors
};
bool qr_route(int64_t m, int64_t n, QrRoute &r);

}  // namespace qb
