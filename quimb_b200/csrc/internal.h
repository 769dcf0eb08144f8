// Library-internal helpers shared between translation units.
#pragma once
#include "common.cuh"
#include "plan.h"

namespace qb {

int launch_contract_f64(const PairPlan &plan, cudaStream_t st);
int launch_contract_c128(const PairPlan &plan, cudaStream_t st);
int launch_fill_zero(const qb_tensor_t *C, cudaStream_t st);

// int8 tensor-core (wgmma) error-free-split engine (ozaki_tc.cu)
bool ozaki_eligible(const PairPlan &plan);
int64_t ozaki_workspace_bytes(const PairPlan &plan);
int launch_contract_ozaki(const PairPlan &plan, void *workspace, cudaStream_t st);

// streaming engine for small-operator steps (contract_stream.cu)
bool stream_eligible(const PairPlan &plan);
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

}  // namespace qb
