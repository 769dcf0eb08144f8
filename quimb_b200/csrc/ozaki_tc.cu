// fp64 pairwise contraction on the int8 tensor cores (Hopper wgmma).
//
// The tensor cores' fp64 rate is far below their int8 rate, so large real-fp64
// contractions can run as an ERROR-FREE integer decomposition (Ozaki scheme):
//
//   A[m,k] = 2^eA[m] * sum_p qA_p[m,k] 2^-(6+7p),   qA_p in [-64, 64] (int8)
//   B[k,n] = 2^eB[n] * sum_q qB_q[k,n] 2^-(6+7q)
//   C[m,n] = 2^(eA[m]+eB[n]-12) * sum_d 2^-7d * sum_{p+q=d} sum_k qA_p qB_q
//
// Every int8 x int8 product and every int32 accumulation is exact (|sum| <
// 2^31 for (d+1) K 2^12 < 2^31, i.e. K < 65536), so the only error is the
// truncation of the operands to 6+7(S-1) bits below each row/column maximum
// and the dropped cross terms p+q >= S:  S = 8 gives ~2^-53 relative to
// rowmax(A) colmax(B) K, i.e. fp64-level results (tests: 1e-12 vs DMMA).
//
// Pipeline (3 kernels):
//   1. ozaki_rowmax_kernel   per-row (A) / per-column (B) max |x|   (HBM bound)
//   2. ozaki_split_kernel    strided fp64 -> S packed int8 K-major slice
//                            planes [S][rows][K]; the INDEX PERMUTATION of the
//                            contraction is folded into this gather, so the
//                            GEMM kernel sees canonical operands  (HBM bound)
//   3. ozaki_gemm_kernel     128 x BN output tile per CTA, 3 warpgroups:
//        warpgroup 0  TMA producer (one thread, registers handed to the
//                consumers with setmaxnreg): cp.async.bulk.tensor
//                (SWIZZLE_128B) of the S B-slice tiles of a k-block (double
//                buffered) and of the A slice tiles through a 4-slot ring,
//                mbarrier full/empty;
//        warpgroups 1-2  64 rows each: wgmma.mma_async m64nBNk32 s8.s8.s32,
//                for p: for q <= S-1-p: acc[p+q] += A_p B_q; the S
//                anti-diagonal accumulators live in registers (S x BN/2 per
//                thread); then the epilogue combines them in fp64 with exact
//                power-of-two weights, applies the row / column scales and
//                alpha/beta and scatters to the strided C (output
//                permutation folded into the store).
//
// The same engine serves all four dtypes natively.
//   * float32 / complex64 (PEPS boundary contraction): S = 4 slices (6 + 7*3
//     = 27 bits below the row maximum, finer than the 24-bit significand),
//     10 slice products, 128 x 64 output tiles; the split kernel reads the
//     strided single-precision operand directly and the epilogue rounds once
//     to float -- no widening passes through HBM.  float64: S = 8, 36 slice
//     products, 128 x 32 tiles.
//   * complex64 / complex128: the real GEMM of the embedding
//       A_e[m, 2k+c] = (re, im)(A[m,k]),   B_e[2k+c, 2n+d] = [[re, im], [-im, re]]
//     (C_e[m, 2n+d] is the interleaved storage of complex C); the embedding is
//     produced inside the split kernel's gather (conjugation = a sign there),
//     so complex operands cost no extra pass either.
//
// Range and special values.  The exponents eA, eB stay integers: the split
// kernel scales with ldexp(x, 6 - e) and the epilogue applies
// ldexp(v * alpha, eA + eB - 12), so rows with a subnormal maximum and
// products of huge rows with tiny columns neither overflow nor flush in an
// intermediate.  A NaN counts as infinite in the row maximum, so a row or
// column that holds a NaN or an infinity has a non-finite maximum: it gets
// zero slices and the exponent kOzNonFinite, and the epilogue computes the
// output elements of such rows and columns as plain fp64 dot products over
// the original operands.  Their class (NaN, +inf, -inf) is then the one IEEE
// arithmetic gives; finite inputs never take that branch.
#include <cuda.h>
#include <math.h>

#include <algorithm>

#include "internal.h"

namespace qb {

constexpr int OZ_BM = 128;     // tile rows (2 consumer warpgroups x 64)
constexpr int OZ_BK = 128;     // bytes (= int8 elements) of K per slice tile
constexpr int OZ_MAXS = 8;     // max slices, double: 8 x 32 columns of accumulators
constexpr int OZ_MAXS_SINGLE = 4;  // max slices, single: 4 x 64 columns
constexpr int OZ_BN_DOUBLE = 32;   // tile columns
constexpr int OZ_BN_SINGLE = 64;
constexpr int OZ_ASLOTS = 4;   // A ring depth
constexpr int OZ_A_TILE = OZ_BM * OZ_BK;  // 16 KB

// ------------------------------------------------------------------ PTX ----
__device__ __forceinline__ void mbar_init(uint64_t *bar, int count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t *bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)),
               "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t *bar, uint32_t parity) {
  asm volatile(
      "{\n"
      ".reg .pred P1;\n"
      "LAB_WAIT:\n"
      "mbarrier.try_wait.parity.shared::cta.b64 P1, [%0], %1;\n"
      "@P1 bra DONE;\n"
      "bra LAB_WAIT;\n"
      "DONE:\n"
      "}\n" ::"r"(smem_u32(bar)),
      "r"(parity)
      : "memory");
}
__device__ __forceinline__ void tma_load_3d(void *dst, const CUtensorMap *map,
                                            uint64_t *bar, int c0, int c1, int c2) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes "
      "[%0], [%1, {%3, %4, %5}], [%2];" ::"r"(smem_u32(dst)),
      "l"(map), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2)
      : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t *bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void wgmma_fence() {
  asm volatile("wgmma.fence.sync.aligned;" ::: "memory");
}
__device__ __forceinline__ void wgmma_commit() {
  asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory");
}
template <int N>
__device__ __forceinline__ void wgmma_wait() {
  asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory");
}

// D(64 x BN, s32, registers) += A(64 x 32, s8, smem) * B(32 x BN, s8, smem),
// both operands K-major.  Thread t of the warpgroup holds, for every 8-column
// chunk j, d[4j + 2h + e] = D[16 (t/32) + (t%32)/4 + 8h][8j + 2 (t%4) + e].
template <int BN>
__device__ __forceinline__ void wgmma_s8(int32_t (&d)[BN / 2], uint64_t adesc, uint64_t bdesc);

template <>
__device__ __forceinline__ void wgmma_s8<32>(int32_t (&d)[16], uint64_t adesc, uint64_t bdesc) {
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "setp.ne.b32 p, %18, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n32k32.s32.s8.s8 "
      "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15}, %16, %17, p;\n"
      "}\n"
      : "+r"(d[0]), "+r"(d[1]), "+r"(d[2]), "+r"(d[3]), "+r"(d[4]), "+r"(d[5]), "+r"(d[6]),
        "+r"(d[7]), "+r"(d[8]), "+r"(d[9]), "+r"(d[10]), "+r"(d[11]), "+r"(d[12]),
        "+r"(d[13]), "+r"(d[14]), "+r"(d[15])
      : "l"(adesc), "l"(bdesc), "r"(1)
      : "memory");
}

template <>
__device__ __forceinline__ void wgmma_s8<64>(int32_t (&d)[32], uint64_t adesc, uint64_t bdesc) {
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "setp.ne.b32 p, %34, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n64k32.s32.s8.s8 "
      "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,"
      "%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31}, %32, %33, p;\n"
      "}\n"
      : "+r"(d[0]), "+r"(d[1]), "+r"(d[2]), "+r"(d[3]), "+r"(d[4]), "+r"(d[5]), "+r"(d[6]),
        "+r"(d[7]), "+r"(d[8]), "+r"(d[9]), "+r"(d[10]), "+r"(d[11]), "+r"(d[12]),
        "+r"(d[13]), "+r"(d[14]), "+r"(d[15]), "+r"(d[16]), "+r"(d[17]), "+r"(d[18]),
        "+r"(d[19]), "+r"(d[20]), "+r"(d[21]), "+r"(d[22]), "+r"(d[23]), "+r"(d[24]),
        "+r"(d[25]), "+r"(d[26]), "+r"(d[27]), "+r"(d[28]), "+r"(d[29]), "+r"(d[30]),
        "+r"(d[31])
      : "l"(adesc), "l"(bdesc), "r"(1)
      : "memory");
}

// K-major, SWIZZLE_128B shared-memory matrix descriptor (sm_90 wgmma format):
// start>>4 [0,14), LBO [16,30) = 1 (unused for swizzled K-major), SBO [32,46)
// = 1024>>4 (8 rows of 128 B), base offset [49,52) = 0 (1024-aligned tiles),
// layout type [62,64) = 1 (SWIZZLE_128B).  A K step of 32 bytes inside the
// 128-byte swizzle row advances the start address by 2.
__device__ __forceinline__ uint64_t wgmma_desc_sw128(uint32_t smem_addr) {
  return (uint64_t)((smem_addr >> 4) & 0x3FFF) | (1ull << 16) | (64ull << 32) | (1ull << 62);
}

// --------------------------------------------------- operand preparation ----
struct SplitParams {
  const void *src;
  int32_t single;      // 1: float / complex64 source, 0: double / complex128
  int32_t role;        // 0 real; 1 complex, A-role (K doubled); 2 complex, B-role
                       // (rows and K doubled: [[re, im], [-im, re]])
  int32_t conj;        // complex operand enters conjugated
  ModeGroup rows;      // s0 = stride of the row (free) modes in src (elements)
  ModeGroup ks;        // s0 = stride of the contracted modes in src
  int64_t R, K;        // extents of the (embedded) real operand
  int64_t Rpad, Kpad;  // padded extents of the slice planes
  int32_t S;
  int32_t k_contig;    // 1: consecutive k contiguous in memory, 0: rows
  unsigned long long *rowmax;  // [Rpad] max |x| as raw double bits
  int32_t *expo;               // [Rpad] e: the row's slices carry x * 2^(6-e)
  int8_t *slices;              // [S][Rpad][Kpad]
};

// exponent of a row / column holding a NaN or an infinity: its slices are
// zero and the GEMM epilogue computes its outputs directly in fp64
constexpr int kOzNonFinite = 0x7fffffff;

// element (r_e, k_e) of the real operand the GEMM sees: `off` = element offset
// of the underlying (possibly complex) entry, d = r_e & 1, c = k_e & 1
__device__ __forceinline__ double oz_elem(const void *src, int single, int role, int conj,
                                          int64_t off, int d, int c) {
  if (role == 0)
    return single ? (double)static_cast<const float *>(src)[off]
                  : static_cast<const double *>(src)[off];
  double re, im;
  if (single) {
    const float2 z = static_cast<const float2 *>(src)[off];
    re = z.x; im = z.y;
  } else {
    const double2 z = static_cast<const double2 *>(src)[off];
    re = z.x; im = z.y;
  }
  if (conj) im = -im;
  if (role == 1) return c ? im : re;
  // B-role: B_e[2k+c, 2n+d]
  if (c == d) return re;
  return c ? -im : im;
}
__device__ __forceinline__ double oz_load(const SplitParams &P, int64_t off, int d, int c) {
  return oz_elem(P.src, P.single, P.role, P.conj, off, d, c);
}
// |x| for the row maximum; a NaN counts as infinite, so the maximum of a row
// is finite exactly when every entry is (fmax alone would skip the NaN)
__device__ __forceinline__ double oz_mag(double x) {
  const double a = fabs(x);
  return a == a ? a : (double)INFINITY;
}

__global__ void __launch_bounds__(256)
    ozaki_rowmax_kernel(const __grid_constant__ SplitParams P) {
  __shared__ int64_t roff[64];
  __shared__ int64_t koff[256];
  __shared__ double red[8][65];
  const int tid = threadIdx.x;
  const int64_t r0 = (int64_t)blockIdx.x * 64, k0 = (int64_t)blockIdx.y * 256;
  const int rsh = P.role == 2 ? 1 : 0, ksh = P.role != 0 ? 1 : 0;
  if (tid < 64) {
    int64_t r = r0 + tid, o = -1, d;
    if (r < P.R) decode2(r >> rsh, P.rows, o, d);
    roff[tid] = o;
  }
  {
    int64_t k = k0 + tid, o = -1, d;
    if (k < P.K) decode2(k >> ksh, P.ks, o, d);
    koff[tid] = o;
  }
  __syncthreads();
  if (P.k_contig) {
    const int tx = tid & 31, ty = tid >> 5;
    for (int i = 0; i < 8; ++i) {
      const int r = ty + 8 * i;
      const int64_t ro = roff[r];
      double m = 0.0;
      if (ro >= 0) {
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          const int64_t ko = koff[tx + 32 * j];
          if (ko >= 0) m = fmax(m, oz_mag(oz_load(P, ro + ko, (int)((r0 + r) & 1), (tx + 32 * j) & 1)));
        }
      }
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) m = fmax(m, __shfl_xor_sync(0xffffffffu, m, o));
      if (tx == 0 && ro >= 0 && m > 0.0)
        atomicMax(&P.rowmax[r0 + r], (unsigned long long)__double_as_longlong(m));
    }
  } else {
    const int tx = tid & 31, ty = tid >> 5;
    double m0 = 0.0, m1 = 0.0;
    const int64_t ro0 = roff[tx], ro1 = roff[tx + 32];
    for (int j = 0; j < 32; ++j) {
      const int64_t ko = koff[ty + 8 * j];
      if (ko >= 0) {
        const int c = (ty + 8 * j) & 1;   // k0 is even
        if (ro0 >= 0) m0 = fmax(m0, oz_mag(oz_load(P, ro0 + ko, tx & 1, c)));
        if (ro1 >= 0) m1 = fmax(m1, oz_mag(oz_load(P, ro1 + ko, tx & 1, c)));
      }
    }
    red[ty][tx] = m0; red[ty][tx + 32] = m1;
    __syncthreads();
    if (tid < 64) {
      double m = 0.0;
      for (int w = 0; w < 8; ++w) m = fmax(m, red[w][tid]);
      if (roff[tid] >= 0 && m > 0.0)
        atomicMax(&P.rowmax[r0 + tid], (unsigned long long)__double_as_longlong(m));
    }
  }
}

// tile: 32 rows x 128 k of the operand -> S x (32 x 128) int8
__global__ void __launch_bounds__(256)
    ozaki_split_kernel(const __grid_constant__ SplitParams P) {
  __shared__ double tile[32][8 * 17];  // [row][k/16][16 + 1 pad]
  __shared__ int64_t roff[32];
  __shared__ int64_t koff[128];
  __shared__ int sh_s[32];
  const int tid = threadIdx.x;
  const int64_t r0 = (int64_t)blockIdx.x * 32, k0 = (int64_t)blockIdx.y * 128;
  const int rsh = P.role == 2 ? 1 : 0, ksh = P.role != 0 ? 1 : 0;
  if (tid < 32) {
    const int64_t r = r0 + tid;
    int64_t o = -1, d;
    int e = 0;
    if (r < P.R) {
      const double mx = __longlong_as_double((long long)P.rowmax[r]);
      if (!isfinite(mx)) {
        e = kOzNonFinite;  // zero slices (o stays -1)
      } else {
        decode2(r >> rsh, P.rows, o, d);
        if (mx > 0.0) e = ilogb(mx) + 1;  // mx * 2^-e in [0.5, 1)
      }
    }
    if (blockIdx.y == 0) P.expo[r] = e;
    // x * 2^(6-e) in (-64, 64), applied by ldexp: 2^(6-e) itself is not a
    // double for rows whose maximum is below 2^-1017
    roff[tid] = o; sh_s[tid] = 6 - e;
  }
  if (tid < 128) {
    const int64_t k = k0 + tid;
    int64_t o = -1, d;
    if (k < P.K) decode2(k >> ksh, P.ks, o, d);
    koff[tid] = o;
  }
  __syncthreads();
  // gather the tile, coalesced along the contiguous direction
  for (int idx = tid; idx < 32 * 128; idx += 256) {
    int r, k;
    if (P.k_contig) { k = idx & 127; r = idx >> 7; } else { r = idx & 31; k = idx >> 5; }
    const int64_t ro = roff[r], ko = koff[k];
    double x = 0.0;
    if (ro >= 0 && ko >= 0) x = ldexp(oz_load(P, ro + ko, r & 1, k & 1), sh_s[r]);  // r0, k0 even
    tile[r][(k >> 4) * 17 + (k & 15)] = x;
  }
  __syncthreads();
  // each thread: one row, 16 consecutive k -> S packed 16-byte vectors
  const int seg = tid & 7, row = tid >> 3;
  double t[16];
#pragma unroll
  for (int i = 0; i < 16; ++i) t[i] = tile[row][seg * 17 + i];
  const int64_t gr = r0 + row, gk = k0 + seg * 16;
  const int64_t plane = P.Rpad * P.Kpad;
  for (int s = 0; s < P.S; ++s) {
    uint32_t w[4] = {0, 0, 0, 0};
#pragma unroll
    for (int i = 0; i < 16; ++i) {
      const double q = rint(t[i]);
      t[i] = (t[i] - q) * 128.0;
      w[i >> 2] |= ((uint32_t)(uint8_t)(int8_t)(int)q) << (8 * (i & 3));
    }
    *reinterpret_cast<uint4 *>(P.slices + (int64_t)s * plane + gr * P.Kpad + gk) =
        make_uint4(w[0], w[1], w[2], w[3]);
  }
}

// ------------------------------------------------------------- the GEMM ----
struct OzGemmParams {
  ContractParams c;   // for the C scatter (mode groups m, n with s1 = stride in C)
  int32_t S;
  int32_t nkb;        // k-blocks of 128
  int32_t cplx;       // C is complex (interleaved): column 2n+d of the real GEMM
  int64_t Me, Ne, Ke;     // extents of the real GEMM
  const int32_t *expA;    // [Mpad] row exponents (kOzNonFinite: computed directly)
  const int32_t *expB;    // [Npad] column exponents
};

// fp64 dot product of GEMM row m and column ne straight from the strided
// operands (c.A, c.B through the m / n / k mode groups).  Only the outputs of
// rows and columns that hold a NaN or an infinity take it, so they come out in
// the class IEEE arithmetic gives (NaN, +inf or -inf).
__device__ __noinline__ double oz_direct_dot(const OzGemmParams &P, int single, int64_t m,
                                             int64_t ne) {
  const ContractParams &c = P.c;
  const int cplx = P.cplx;
  int64_t oa, ob, t;
  decode2(m, c.m, oa, t);
  decode2(ne >> cplx, c.n, ob, t);
  double s = 0.0;
  for (int64_t k = 0; k < P.Ke; ++k) {
    int64_t ka, kb;
    decode2(k >> cplx, c.k, ka, kb);
    s += oz_elem(c.A, single, cplx ? 1 : 0, c.conjA, oa + ka, 0, (int)(k & 1)) *
         oz_elem(c.B, single, cplx ? 2 : 0, c.conjB, ob + kb, (int)(ne & 1), (int)(k & 1));
  }
  return s;
}

// BN output columns per CTA, NSL accumulators (the most slices the
// instantiation takes): NSL x BN/2 = 128 accumulator registers per consumer
// thread -- 32 columns with 8 slices (double), 64 with 4 (single).
template <int BN, int NSL>
struct OzSmem {
  static constexpr int B_TILE = BN * OZ_BK;               // 4 / 8 KB
  static constexpr size_t TILES = (size_t)OZ_ASLOTS * OZ_A_TILE + 2 * (size_t)NSL * B_TILE;
  static constexpr size_t BYTES = TILES + 1024 /*align*/ + 8192 /*tables, barriers*/;
};

constexpr int OZ_THREADS = 384;    // producer warpgroup + 2 consumer warpgroups
constexpr int OZ_CONSUMER_WARPS = 8;

template <int BN, int NSL, typename OutT>
__global__ void __launch_bounds__(OZ_THREADS, 1)
    ozaki_gemm_kernel(const __grid_constant__ CUtensorMap mapA,
                      const __grid_constant__ CUtensorMap mapB,
                      const __grid_constant__ OzGemmParams P) {
  constexpr int B_TILE = OzSmem<BN, NSL>::B_TILE;
  extern __shared__ unsigned char oz_smem_raw[];
  unsigned char *base = reinterpret_cast<unsigned char *>(
      ((uintptr_t)oz_smem_raw + 1023) & ~(uintptr_t)1023);
  unsigned char *sA = base;                                   // 4 x 16 KB
  unsigned char *sB = base + (size_t)OZ_ASLOTS * OZ_A_TILE;   // 2 x NSL x B_TILE
  unsigned char *aux = base + OzSmem<BN, NSL>::TILES;
  uint64_t *fullA = reinterpret_cast<uint64_t *>(aux);        // [4]
  uint64_t *emptyA = fullA + OZ_ASLOTS;                       // [4]
  uint64_t *fullB = emptyA + OZ_ASLOTS;                       // [2]
  uint64_t *emptyB = fullB + 2;                               // [2]
  int64_t *offCm = reinterpret_cast<int64_t *>(aux + 256);    // [128]
  int64_t *offCn = offCm + OZ_BM;                             // [BN]
  int32_t *expM = reinterpret_cast<int32_t *>(offCn + BN);    // [128]
  int32_t *expN = expM + OZ_BM;                               // [BN]

  const int tid = threadIdx.x, lane = tid & 31;
  const int S = P.S, nkb = P.nkb;
  const int tm = blockIdx.x, tn = blockIdx.y;

  if (tid == 0) {
    for (int i = 0; i < OZ_ASLOTS; ++i) {
      mbar_init(&fullA[i], 1);
      mbar_init(&emptyA[i], OZ_CONSUMER_WARPS);
    }
    for (int i = 0; i < 2; ++i) {
      mbar_init(&fullB[i], 1);
      mbar_init(&emptyB[i], OZ_CONSUMER_WARPS);
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  // epilogue tables (consumer threads); offsets in units of OutT
  if (tid >= 128) {
    const int e = tid - 128;
    const int csh = P.cplx ? 1 : 0;
    if (e < OZ_BM) {
      const int64_t m = (int64_t)tm * OZ_BM + e;
      int64_t oa, oc = -1;
      if (m < P.Me) { decode2(m, P.c.m, oa, oc); oc <<= csh; }
      offCm[e] = oc;
      expM[e] = P.expA[(int64_t)tm * OZ_BM + e];
    } else if (e - OZ_BM < BN) {
      const int c = e - OZ_BM;
      const int64_t ne = (int64_t)tn * BN + c;
      int64_t ob, oc = -1;
      if (ne < P.Ne) { decode2(ne >> csh, P.c.n, ob, oc); oc = (oc << csh) + (csh ? (ne & 1) : 0); }
      offCn[c] = oc;
      expN[c] = P.expB[(int64_t)tn * BN + c];
    }
  }
  __syncthreads();

  if (tid < 128) {
    // ======================= TMA producer warpgroup ========================
    asm volatile("setmaxnreg.dec.sync.aligned.u32 40;");
    if (tid == 0) {
      int ia = 0;
      for (int kb = 0; kb < nkb; ++kb) {
        const int sb = kb & 1;
        mbar_wait(&emptyB[sb], ((kb >> 1) & 1) ^ 1);
        mbar_expect_tx(&fullB[sb], (uint32_t)S * B_TILE);
        for (int q = 0; q < S; ++q)
          tma_load_3d(sB + ((size_t)sb * NSL + q) * B_TILE, &mapB, &fullB[sb],
                      kb * OZ_BK, tn * BN, q);
        for (int p = 0; p < S; ++p, ++ia) {
          const int sa = ia % OZ_ASLOTS;
          mbar_wait(&emptyA[sa], ((ia / OZ_ASLOTS) & 1) ^ 1);
          mbar_expect_tx(&fullA[sa], OZ_A_TILE);
          tma_load_3d(sA + (size_t)sa * OZ_A_TILE, &mapA, &fullA[sa], kb * OZ_BK,
                      tm * OZ_BM, p);
        }
      }
    }
    return;
  }
  // ===================== consumer warpgroups (wgmma) ======================
  asm volatile("setmaxnreg.inc.sync.aligned.u32 232;");
  const int ct = tid - 128;
  const int half = ct >> 7;          // rows [64 half, 64 half + 64) of the tile
  const int wq = (ct >> 5) & 3;      // warp within the warpgroup
  int32_t acc[NSL][BN / 2];
#pragma unroll
  for (int d = 0; d < NSL; ++d)
#pragma unroll
    for (int i = 0; i < BN / 2; ++i) acc[d][i] = 0;

  // for p: for q <= S-1-p: acc[p+q] += A_p B_q, one commit group per A slice;
  // a slot is released once the group after it has been issued and the
  // group using it has retired (wgmma.wait_group 1)
  int ia = 0, pend_a = -1, pend_b = -1;
  for (int kb = 0; kb < nkb; ++kb) {
    const int sb = kb & 1;
    mbar_wait(&fullB[sb], (kb >> 1) & 1);
#pragma unroll
    for (int p = 0; p < NSL; ++p) {
      if (p < S) {
        const int sa = ia % OZ_ASLOTS;
        mbar_wait(&fullA[sa], (ia / OZ_ASLOTS) & 1);
        const uint64_t adesc = wgmma_desc_sw128(
            smem_u32(sA + (size_t)sa * OZ_A_TILE + (size_t)half * 64 * OZ_BK));
        wgmma_fence();
#pragma unroll
        for (int q = 0; q < NSL; ++q) {
          if (p + q < S) {
            const uint64_t bdesc =
                wgmma_desc_sw128(smem_u32(sB + ((size_t)sb * NSL + q) * B_TILE));
#pragma unroll
            for (int k4 = 0; k4 < OZ_BK / 32; ++k4)
              wgmma_s8<BN>(acc[p + q], adesc + (uint64_t)(k4 * 2), bdesc + (uint64_t)(k4 * 2));
          }
        }
        wgmma_commit();
        wgmma_wait<1>();
        if (lane == 0) {
          if (pend_a >= 0) mbar_arrive(&emptyA[pend_a]);
          if (pend_b >= 0) mbar_arrive(&emptyB[pend_b]);
        }
        pend_a = sa;
        pend_b = (p == S - 1) ? sb : -1;
        ++ia;
      }
    }
  }
  wgmma_wait<0>();

  // ============================== epilogue ================================
  // combine the S accumulators in fp64 with exact power-of-two weights,
  // apply alpha and the row / column scales 2^(eA + eB - 12) in one ldexp (no
  // intermediate can overflow or underflow), add beta C, scatter to the
  // strided C
  OutT *C = static_cast<OutT *>(P.c.C);
  const double alpha = P.c.alpha, beta = P.c.beta;
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int row = half * 64 + wq * 16 + (lane >> 2) + 8 * h;
    const int64_t om = offCm[row];
    if (om < 0) continue;
    const int eM = expM[row];
#pragma unroll
    for (int j = 0; j < BN / 8; ++j) {
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const int i = 4 * j + 2 * h + e;
        const int col = 8 * j + 2 * (lane & 3) + e;
        double v = 0.0, w = ldexp(1.0, -7 * (S - 1));
#pragma unroll
        for (int d = NSL - 1; d >= 0; --d) {
          if (d < S) {
            v += w * (double)acc[d][i];
            w *= 128.0;
          }
        }
        const int64_t on = offCn[col];
        if (on >= 0) {
          const int eN = expN[col];
          double val;
          if (eM == kOzNonFinite || eN == kOzNonFinite)
            val = alpha * oz_direct_dot(P, sizeof(OutT) == 4, (int64_t)tm * OZ_BM + row,
                                        (int64_t)tn * BN + col);
          else
            val = ldexp(v * alpha, eM + eN - 12);
          if (beta != 0.0) val += beta * (double)C[om + on];
          C[om + on] = (OutT)val;
        }
      }
    }
  }
}

// ------------------------------------------------------------------ host ----
typedef CUresult (*PFN_encodeTiled)(CUtensorMap *, CUtensorMapDataType, cuuint32_t, void *,
                                    const cuuint64_t *, const cuuint64_t *,
                                    const cuuint32_t *, const cuuint32_t *,
                                    CUtensorMapInterleave, CUtensorMapSwizzle,
                                    CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static PFN_encodeTiled get_encode() {
  static PFN_encodeTiled fn = nullptr;
  if (!fn) {
    void *p = nullptr;
    cudaDriverEntryPointQueryResult qres;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres) ==
            cudaSuccess &&
        qres == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<PFN_encodeTiled>(p);
  }
  return fn;
}

static int make_slice_map(CUtensorMap *map, const int8_t *ptr, int64_t Kpad, int64_t Rpad,
                          int S, int box_rows) {
  PFN_encodeTiled enc = get_encode();
  if (!enc) {
    set_error("cuTensorMapEncodeTiled is unavailable");
    return 2000;
  }
  cuuint64_t dims[3] = {(cuuint64_t)Kpad, (cuuint64_t)Rpad, (cuuint64_t)S};
  cuuint64_t strides[2] = {(cuuint64_t)Kpad, (cuuint64_t)(Kpad * Rpad)};
  cuuint32_t box[3] = {(cuuint32_t)OZ_BK, (cuuint32_t)box_rows, 1};
  cuuint32_t estr[3] = {1, 1, 1};
  CUresult r = enc(map, CU_TENSOR_MAP_DATA_TYPE_UINT8, 3, (void *)ptr, dims, strides, box,
                   estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                   CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_error("cuTensorMapEncodeTiled failed with %d", (int)r);
    return 2000 + (int)r;
  }
  return 0;
}

struct OzGeom {
  int S, BN, cplx, single;
  int64_t Me, Ne, Ke;            // extents of the real GEMM
  int64_t Mpad, Npad, Kpad;
  int64_t off_rmA, off_rmB, off_scA, off_scB, off_slA, off_slB, total;  // bytes
};

// int8 slices per operand: all the accumulator columns the GEMM kernel holds
// (8 for fp64 / complex128, 4 for fp32 / complex64)
static int oz_slices(bool single) { return single ? OZ_MAXS_SINGLE : OZ_MAXS; }

static void oz_geometry(const PairPlan &plan, OzGeom &g) {
  const ContractParams &p = plan.p;
  auto up = [](int64_t x, int64_t a) { return (x + a - 1) / a * a; };
  g.single = (plan.dtype == QB_F32 || plan.dtype == QB_C64) ? 1 : 0;
  g.cplx = dtype_is_complex(plan.dtype) ? 1 : 0;
  g.S = oz_slices(g.single);
  g.BN = g.single ? OZ_BN_SINGLE : OZ_BN_DOUBLE;
  g.Me = p.M;
  g.Ne = g.cplx ? 2 * p.N : p.N;
  g.Ke = g.cplx ? 2 * p.K : p.K;
  g.Mpad = up(g.Me, OZ_BM);
  g.Npad = up(g.Ne, OZ_BM);  // multiple of 128 so the split kernel tiles evenly
  g.Kpad = up(g.Ke, OZ_BK);
  int64_t off = 0;
  g.off_rmA = off; off += up(g.Mpad * 8, 1024);
  g.off_rmB = off; off += up(g.Npad * 8, 1024);
  g.off_scA = off; off += up(g.Mpad * 8, 1024);
  g.off_scB = off; off += up(g.Npad * 8, 1024);
  g.off_slA = off; off += up((int64_t)g.S * g.Mpad * g.Kpad, 1024);
  g.off_slB = off; off += up((int64_t)g.S * g.Npad * g.Kpad, 1024);
  g.total = off;
}

bool ozaki_eligible(const PairPlan &plan) {
  const ContractParams &p = plan.p;
  const int64_t f = dtype_is_complex(plan.dtype) ? 2 : 1;
  return p.nbatch == 1 && !p.dA && p.M >= 128 && f * p.N >= 64 && f * p.K >= 128 &&
         f * p.K < 65536 && !plan.empty_out && !plan.zero_fill;
}

int64_t ozaki_workspace_bytes(const PairPlan &plan) {
  OzGeom g;
  oz_geometry(plan, g);
  return g.total;
}

template <int BN, int NSL, typename OutT>
static int oz_launch_gemm(const CUtensorMap &mapA, const CUtensorMap &mapB,
                          const OzGemmParams &gp, dim3 grid, cudaStream_t st) {
  auto kern = ozaki_gemm_kernel<BN, NSL, OutT>;
  static bool attr_set = false;
  if (!attr_set) {
    QB_CUDA_CHECK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                       (int)OzSmem<BN, NSL>::BYTES));
    attr_set = true;
  }
  kern<<<grid, OZ_THREADS, OzSmem<BN, NSL>::BYTES, st>>>(mapA, mapB, gp);
  QB_LAUNCH_CHECK();
  return 0;
}

int launch_contract_ozaki(const PairPlan &plan, void *workspace, cudaStream_t st) {
  const ContractParams &p = plan.p;
  OzGeom g;
  oz_geometry(plan, g);
  unsigned char *ws = static_cast<unsigned char *>(workspace);
  if (((uintptr_t)ws & 255) != 0) {
    set_error("ozaki workspace must be 256-byte aligned");
    return -10;
  }
  QB_CUDA_CHECK(cudaMemsetAsync(ws, 0, g.off_scA, st));  // row/col maxima = 0
  auto prep = [&](const void *src, int role, int conj, const ModeGroup &rows,
                  const ModeGroup &ks, bool k_second, int64_t R, int64_t Rpad,
                  int64_t off_rm, int64_t off_sc, int64_t off_sl) -> int {
    SplitParams sp;
    memset(&sp, 0, sizeof(sp));
    sp.src = src;
    sp.single = g.single;
    sp.role = role;
    sp.conj = conj;
    sp.rows.n = rows.n; sp.ks.n = ks.n;
    for (int i = 0; i < rows.n; ++i) {
      sp.rows.ext[i] = rows.ext[i];
      sp.rows.s0[i] = rows.s0[i];
    }
    for (int i = 0; i < ks.n; ++i) {
      sp.ks.ext[i] = ks.ext[i];
      sp.ks.s0[i] = k_second ? ks.s1[i] : ks.s0[i];
    }
    sp.R = R; sp.K = g.Ke; sp.Rpad = Rpad; sp.Kpad = g.Kpad; sp.S = g.S;
    const int64_t ksm = ks.n ? sp.ks.s0[0] : 1, rsm = rows.n ? sp.rows.s0[0] : (int64_t)1 << 60;
    sp.k_contig = (ksm <= rsm) ? 1 : 0;
    sp.rowmax = reinterpret_cast<unsigned long long *>(ws + off_rm);
    sp.expo = reinterpret_cast<int32_t *>(ws + off_sc);
    sp.slices = reinterpret_cast<int8_t *>(ws + off_sl);
    dim3 g1((unsigned)((R + 63) / 64), (unsigned)((g.Ke + 255) / 256));
    ozaki_rowmax_kernel<<<g1, 256, 0, st>>>(sp);
    QB_LAUNCH_CHECK();
    dim3 g2((unsigned)(Rpad / 32), (unsigned)(g.Kpad / 128));
    ozaki_split_kernel<<<g2, 256, 0, st>>>(sp);
    QB_LAUNCH_CHECK();
    return 0;
  };
  int rc;
  // A: rows = m modes (stride in A = s0), k modes (stride in A = s0)
  if ((rc = prep(p.A, g.cplx ? 1 : 0, p.conjA, p.m, p.k, false, g.Me, g.Mpad,
                 g.off_rmA, g.off_scA, g.off_slA)))
    return rc;
  // B: rows = n modes (stride in B = s0), k modes (stride in B = s1)
  if ((rc = prep(p.B, g.cplx ? 2 : 0, p.conjB, p.n, p.k, true, g.Ne, g.Npad,
                 g.off_rmB, g.off_scB, g.off_slB)))
    return rc;

  CUtensorMap mapA, mapB;
  if ((rc = make_slice_map(&mapA, reinterpret_cast<int8_t *>(ws + g.off_slA), g.Kpad, g.Mpad,
                           g.S, OZ_BM)))
    return rc;
  if ((rc = make_slice_map(&mapB, reinterpret_cast<int8_t *>(ws + g.off_slB), g.Kpad, g.Npad,
                           g.S, g.BN)))
    return rc;
  OzGemmParams gp;
  gp.c = p;
  gp.S = g.S;
  gp.nkb = (int)(g.Kpad / OZ_BK);
  gp.cplx = g.cplx;
  gp.Me = g.Me; gp.Ne = g.Ne; gp.Ke = g.Ke;
  gp.expA = reinterpret_cast<const int32_t *>(ws + g.off_scA);
  gp.expB = reinterpret_cast<const int32_t *>(ws + g.off_scB);
  dim3 grid((unsigned)(g.Mpad / OZ_BM), (unsigned)((g.Ne + g.BN - 1) / g.BN));
  if (g.single) return oz_launch_gemm<OZ_BN_SINGLE, OZ_MAXS_SINGLE, float>(mapA, mapB, gp, grid, st);
  return oz_launch_gemm<OZ_BN_DOUBLE, OZ_MAXS, double>(mapA, mapB, gp, grid, st);
}

}  // namespace qb
