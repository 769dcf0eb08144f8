// Shared helpers for the quimb_b200 CUDA sources (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>

#include <atomic>
#include <string>

#include "../../include/quimb_b200.h"

namespace qb {

// ---------------------------------------------------------------- errors ---
void set_error(const char *fmt, ...);
extern std::atomic<int64_t> g_launch_count;

#define QB_CUDA_CHECK(expr)                                                 \
  do {                                                                      \
    cudaError_t _e = (expr);                                                \
    if (_e != cudaSuccess) {                                                \
      qb::set_error("%s failed at %s:%d: %s", #expr, __FILE__, __LINE__,    \
                    cudaGetErrorString(_e));                                \
      return 1000 + (int)_e;                                                \
    }                                                                       \
  } while (0)

#define QB_LAUNCH_CHECK()                                                   \
  do {                                                                      \
    qb::g_launch_count.fetch_add(1, std::memory_order_relaxed);             \
    cudaError_t _e = cudaGetLastError();                                    \
    if (_e != cudaSuccess) {                                                \
      qb::set_error("kernel launch failed at %s:%d: %s", __FILE__,          \
                    __LINE__, cudaGetErrorString(_e));                      \
      return 1000 + (int)_e;                                                \
    }                                                                       \
  } while (0)

static inline int dtype_size(int dt) {
  switch (dt) {
    case QB_F32: return 4;
    case QB_F64: return 8;
    case QB_C64: return 8;
    case QB_C128: return 16;
  }
  return 0;
}
static inline bool dtype_is_complex(int dt) {
  return dt == QB_C64 || dt == QB_C128;
}

int sm_count();

// ----------------------------------------------------------- device bits ---
#ifdef __CUDACC__

__device__ __forceinline__ uint32_t smem_u32(const void *p) {
  return (uint32_t)__cvta_generic_to_shared(p);
}

// 8-byte async copy global->shared; src_bytes == 0 zero-fills the destination
__device__ __forceinline__ void cp_async8(uint32_t dst, const void *src,
                                          int src_bytes) {
  asm volatile("cp.async.ca.shared.global [%0], [%1], 8, %2;\n" ::"r"(dst),
               "l"(src), "r"(src_bytes)
               : "memory");
}
__device__ __forceinline__ void cp_async16(uint32_t dst, const void *src,
                                           int src_bytes) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;\n" ::"r"(dst),
               "l"(src), "r"(src_bytes)
               : "memory");
}
__device__ __forceinline__ void cp_async_commit() {
  asm volatile("cp.async.commit_group;\n" ::: "memory");
}
template <int N>
__device__ __forceinline__ void cp_async_wait() {
  asm volatile("cp.async.wait_group %0;\n" ::"n"(N) : "memory");
}

// D(16x8) += A(16x8, row) * B(8x8, col) in fp64 on the tensor cores
// (one DMMA on sm_90a).  Fragment ownership (g = lane/4,
// t = lane%4):  a0:(g,t) a1:(g+8,t) a2:(g,t+4) a3:(g+8,t+4);
// b0:(k=t,n=g) b1:(k=t+4,n=g);  c0:(g,2t) c1:(g,2t+1) c2:(g+8,2t) c3:(g+8,2t+1)
__device__ __forceinline__ void dmma_16x8x8(double (&c)[4], const double (&a)[4],
                                            const double (&b)[2]) {
  asm volatile(
      "mma.sync.aligned.m16n8k8.row.col.f64.f64.f64.f64 "
      "{%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};\n"
      : "+d"(c[0]), "+d"(c[1]), "+d"(c[2]), "+d"(c[3])
      : "d"(a[0]), "d"(a[1]), "d"(a[2]), "d"(a[3]), "d"(b[0]), "d"(b[1]));
}

__device__ __forceinline__ double warp_sum(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

#endif  // __CUDACC__

}  // namespace qb
