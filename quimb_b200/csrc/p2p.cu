// Peer-memory exchange kernels for the bond-sharded two-site eigensolve
// (SURVEY 8e; quimb_b200/dist.py:BondShard).  One process per GPU; every rank
// owns one "symmetric" allocation made here with cudaMalloc and exported to
// its peers through CUDA IPC, so that kernels can store straight into a
// peer's HBM over NVLink / NVSwitch:
//
//   allgather_push_kernel   every rank streams its row slab of a vector into
//                           the gather buffer of ALL ranks (its own included)
//                           and raises one flag word per peer; the last CTA
//                           then waits for the peers' flags, so kernel
//                           completion == the full vector is resident locally.
//                           ONE launch replaces ncclAllGather + its stream
//                           synchronisation.
//   allreduce_small_kernel  <= 64 doubles (the inner products of a
//                           Gram-Schmidt pass): every rank stores its partial
//                           into slot [rank] of every peer, flags, waits for
//                           all slots and sums them in rank order -- the
//                           result is bit-identical on all ranks.  ONE CTA.
//
// Flags are monotone 64-bit epochs (never reset), data buffers alternate on
// the parity of the epoch; a rank can run at most one epoch ahead of its
// slowest peer because completing epoch e needs every peer's flag of epoch e,
// which a peer only raises after everything it enqueued before (the consumers
// of epoch e-1 on its stream) has been issued in stream order.
//
// Spins are bounded (about 4 s of %globaltimer): a peer that died makes the
// kernel give up, set the error word and return instead of hanging the GPU.
#include <cuda_runtime.h>

#include "common.cuh"

namespace qb {

constexpr int P2P_MAX_RANKS = 16;

struct P2PPeers {
  void *buf[P2P_MAX_RANKS];               // base of every rank's symmetric block
  int world, rank;
};

// layout of a symmetric block (bytes):
//   [0, 4096)        gather flags   uint64[P2P_MAX_RANKS] (+ padding)
//   [4096, 8192)     reduce flags   uint64[P2P_MAX_RANKS]
//   [8192, 8192+2*16*64*8)  reduce slots  double[2][P2P_MAX_RANKS][64]
//   [65536, ...)     gather data    2 x gather_bytes
constexpr size_t P2P_GFLAG_OFF = 0, P2P_RFLAG_OFF = 4096, P2P_RSLOT_OFF = 8192,
                 P2P_DATA_OFF = 65536;
constexpr int P2P_RMAX = 64;

__device__ __forceinline__ unsigned long long p2p_now() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}
__device__ __forceinline__ void st_release_sys(unsigned long long *p, unsigned long long v) {
  asm volatile("st.release.sys.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}
__device__ __forceinline__ unsigned long long ld_acquire_sys(const unsigned long long *p) {
  unsigned long long v;
  asm volatile("ld.acquire.sys.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
  return v;
}

// returns false on timeout
__device__ __forceinline__ bool p2p_wait_flag(const unsigned long long *flag,
                                              unsigned long long epoch) {
  const unsigned long long t0 = p2p_now();
  while (ld_acquire_sys(flag) < epoch) {
    if (p2p_now() - t0 > 4000000000ull) return false;
    __nanosleep(64);
  }
  return true;
}

// x: this rank's slab (n16 16-byte words), stored at byte offset dst_off of
// every rank's gather buffer of parity (epoch & 1).
__global__ void __launch_bounds__(512)
    allgather_push_kernel(const P2PPeers P, const uint4 *__restrict__ x, int64_t n16,
                          size_t dst_off, size_t gather_bytes,
                          unsigned long long epoch, unsigned int *counter, int *err) {
  const size_t base = P2P_DATA_OFF + (size_t)(epoch & 1) * gather_bytes + dst_off;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n16; i += stride) {
    const uint4 v = x[i];
#pragma unroll 1
    for (int q = 0; q < P.world; ++q) {
      // start with the next rank so the ranks do not all hit the same peer
      const int p = (P.rank + q) % P.world;
      uint4 *dst = reinterpret_cast<uint4 *>(static_cast<char *>(P.buf[p]) + base) + i;
      *dst = v;
    }
  }
  __threadfence_system();
  __syncthreads();
  __shared__ bool last;
  if (threadIdx.x == 0) last = (atomicAdd(counter, 1u) == gridDim.x - 1);
  __syncthreads();
  if (!last) return;
  // all CTAs of this rank have stored (and fenced) their part
  if (threadIdx.x == 0) *counter = 0;
  if (threadIdx.x < P.world) {
    __threadfence_system();
    unsigned long long *f = reinterpret_cast<unsigned long long *>(
        static_cast<char *>(P.buf[threadIdx.x]) + P2P_GFLAG_OFF) + P.rank;
    st_release_sys(f, epoch);
    const unsigned long long *mine = reinterpret_cast<const unsigned long long *>(
        static_cast<const char *>(P.buf[P.rank]) + P2P_GFLAG_OFF) + threadIdx.x;
    if (!p2p_wait_flag(mine, epoch)) atomicExch(err, 1);
  }
}

// in-place sum over ranks of m <= 64 doubles
__global__ void __launch_bounds__(64)
    allreduce_small_kernel(const P2PPeers P, double *__restrict__ x, int m,
                           unsigned long long epoch, int *err) {
  const int t = threadIdx.x;
  const size_t slot = P2P_RSLOT_OFF + (size_t)(epoch & 1) * P2P_MAX_RANKS * P2P_RMAX * 8;
  if (t < m) {
    const double v = x[t];
    for (int q = 0; q < P.world; ++q) {
      const int p = (P.rank + q) % P.world;
      double *dst = reinterpret_cast<double *>(static_cast<char *>(P.buf[p]) + slot) +
                    P.rank * P2P_RMAX + t;
      *dst = v;
    }
  }
  __threadfence_system();
  __syncthreads();
  if (t < P.world) {
    unsigned long long *f = reinterpret_cast<unsigned long long *>(
        static_cast<char *>(P.buf[t]) + P2P_RFLAG_OFF) + P.rank;
    st_release_sys(f, epoch);
    const unsigned long long *mine = reinterpret_cast<const unsigned long long *>(
        static_cast<const char *>(P.buf[P.rank]) + P2P_RFLAG_OFF) + t;
    if (!p2p_wait_flag(mine, epoch)) atomicExch(err, 1);
  }
  __syncthreads();
  if (t < m) {
    const double *s = reinterpret_cast<const double *>(
        static_cast<const char *>(P.buf[P.rank]) + slot) + t;
    // start from rank 0's value, not from +0.0: one rank is the identity and
    // a sum of -0.0 partials stays -0.0 (IEEE addition of the partials)
    double acc = __ldcg(s);
    for (int r = 1; r < P.world; ++r) acc += __ldcg(s + r * P2P_RMAX);  // L2, fixed order
    x[t] = acc;
  }
}

static int fill_peers(P2PPeers &P, void *const *bufs, int world, int rank) {
  if (world < 1 || world > P2P_MAX_RANKS || rank < 0 || rank >= world) {
    set_error("qb_p2p: world %d / rank %d out of range (max %d ranks)", world, rank,
              P2P_MAX_RANKS);
    return -1;
  }
  for (int i = 0; i < world; ++i) {
    if (!bufs[i]) { set_error("qb_p2p: null peer buffer %d", i); return -2; }
    P.buf[i] = bufs[i];
  }
  P.world = world; P.rank = rank;
  return 0;
}

}  // namespace qb

using namespace qb;

extern "C" {

int64_t qb_p2p_block_bytes(int64_t gather_bytes) {
  if (gather_bytes < 0) return -1;
  const int64_t g = (gather_bytes + 255) / 256 * 256;
  return (int64_t)P2P_DATA_OFF + 2 * g + 256;
}

int64_t qb_p2p_data_offset(int64_t gather_bytes, int parity) {
  const int64_t g = (gather_bytes + 255) / 256 * 256;
  return (int64_t)P2P_DATA_OFF + (parity & 1) * g;
}

int qb_p2p_alloc(int64_t bytes, void **ptr) {
  if (!ptr || bytes <= 0) return -1;
  QB_CUDA_CHECK(cudaMalloc(ptr, (size_t)bytes));
  QB_CUDA_CHECK(cudaMemset(*ptr, 0, (size_t)bytes));
  QB_CUDA_CHECK(cudaDeviceSynchronize());
  return 0;
}

int qb_p2p_free(void *ptr) {
  if (ptr) QB_CUDA_CHECK(cudaFree(ptr));
  return 0;
}

int qb_p2p_export(void *ptr, unsigned char *handle64) {
  if (!ptr || !handle64) return -1;
  static_assert(sizeof(cudaIpcMemHandle_t) == 64, "IPC handle size");
  cudaIpcMemHandle_t h;
  QB_CUDA_CHECK(cudaIpcGetMemHandle(&h, ptr));
  memcpy(handle64, &h, 64);
  return 0;
}

int qb_p2p_import(const unsigned char *handle64, void **peer_ptr) {
  if (!handle64 || !peer_ptr) return -1;
  cudaIpcMemHandle_t h;
  memcpy(&h, handle64, 64);
  QB_CUDA_CHECK(cudaIpcOpenMemHandle(peer_ptr, h, cudaIpcMemLazyEnablePeerAccess));
  return 0;
}

int qb_p2p_unimport(void *peer_ptr) {
  if (peer_ptr) QB_CUDA_CHECK(cudaIpcCloseMemHandle(peer_ptr));
  return 0;
}

// Checks shared by both entry points: -3 null scratch, -4 epoch 0 (the flags
// start at 0, so a wait for epoch 0 would pass before any peer has stored).
static int check_epoch_scratch(const char *fn, uint64_t epoch, const void *scratch) {
  if (!scratch) {
    set_error("%s: scratch is null (8 bytes of zeroed device memory)", fn);
    return -3;
  }
  if (epoch == 0) {
    set_error("%s: epoch must be >= 1 (flags start at 0)", fn);
    return -4;
  }
  return 0;
}

// Push `bytes` (multiple of 16, 16-byte aligned source) from x into every
// rank's gather buffer at byte offset dst_off; returns when the kernel is
// enqueued.  After the kernel the full gathered vector of this epoch sits at
// qb_p2p_data_offset(gather_bytes, epoch & 1) of the LOCAL block.
// `scratch` = 8 bytes of zero-initialised device memory (CTA counter + error
// word) owned by the caller.  An empty slab (bytes == 0) still launches one
// CTA: it raises this rank's flags and waits for the peers' like any other.
int qb_p2p_allgather(void *const *peer_bufs, int world, int rank, const void *x,
                     int64_t bytes, int64_t dst_off, int64_t gather_bytes,
                     uint64_t epoch, void *scratch, void *stream) {
  P2PPeers P;
  int rc = fill_peers(P, peer_bufs, world, rank);
  if (rc) return rc;
  rc = check_epoch_scratch("qb_p2p_allgather", epoch, scratch);
  if (rc) return rc;
  if (bytes < 0 || dst_off < 0) {
    set_error("qb_p2p_allgather: negative slab size %lld or offset %lld", (long long)bytes,
              (long long)dst_off);
    return -5;
  }
  if (bytes % 16 || dst_off % 16 || (reinterpret_cast<uintptr_t>(x) & 15)) {
    set_error("qb_p2p_allgather: slab must be 16-byte aligned and a multiple of 16 bytes");
    return -5;
  }
  if (bytes > 0 && !x) {
    set_error("qb_p2p_allgather: slab of %lld bytes at a null pointer", (long long)bytes);
    return -5;
  }
  const int64_t g = gather_bytes < 0 ? -1 : (gather_bytes + 255) / 256 * 256;
  if (g < 0 || bytes > g || dst_off > g - bytes) {
    set_error("qb_p2p_allgather: slab exceeds the gather buffer");
    return -6;
  }
  const int64_t n16 = bytes / 16;
  int blocks = (int)std::max<int64_t>(1, std::min<int64_t>((n16 + 511) / 512, sm_count()));
  unsigned int *counter = static_cast<unsigned int *>(scratch);
  int *err = reinterpret_cast<int *>(counter + 1);
  allgather_push_kernel<<<blocks, 512, 0, static_cast<cudaStream_t>(stream)>>>(
      P, static_cast<const uint4 *>(x), n16, (size_t)dst_off, (size_t)g,
      (unsigned long long)epoch, counter, err);
  QB_LAUNCH_CHECK();
  return 0;
}

int qb_p2p_allreduce_small(void *const *peer_bufs, int world, int rank, void *x, int m,
                           uint64_t epoch, void *scratch, void *stream) {
  P2PPeers P;
  int rc = fill_peers(P, peer_bufs, world, rank);
  if (rc) return rc;
  rc = check_epoch_scratch("qb_p2p_allreduce_small", epoch, scratch);
  if (rc) return rc;
  if (m < 0 || m > P2P_RMAX) {
    set_error("qb_p2p_allreduce_small: m = %d outside [0, %d]", m, P2P_RMAX);
    return -5;
  }
  if (m > 0 && (!x || (reinterpret_cast<uintptr_t>(x) & 7))) {
    set_error("qb_p2p_allreduce_small: x must be a non-null, 8-byte aligned double array");
    return -5;
  }
  // m == 0 still launches and raises the epoch's flags: a skipped epoch would
  // let the next one reuse the slot parity a slow peer may still be reading
  int *err = reinterpret_cast<int *>(static_cast<unsigned int *>(scratch) + 1);
  allreduce_small_kernel<<<1, 64, 0, static_cast<cudaStream_t>(stream)>>>(
      P, static_cast<double *>(x), m, (unsigned long long)epoch, err);
  QB_LAUNCH_CHECK();
  return 0;
}

}  // extern "C"
