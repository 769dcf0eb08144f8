// Pairwise tensor contraction on the fp64 tensor cores (DMMA) of sm_90a.
//
//   C[m, n, batch] = sum_k op(A)[m, k, batch] * op(B)[k, n, batch]
//
// where m, n, k and batch are *groups of tensor modes* with arbitrary
// strides (see plan.h).  No operand is ever transposed or copied in global
// memory: a CTA turns its tile's logical indices into element offsets through
// small per-tile tables held in shared memory, and the cp.async tile loads
// gather straight from the strided tensors, so the index permutation that
// numpy.tensordot performs as a separate transpose-copy
// (quimb -> cotengra -> autoray do("tensordot")) is folded into the load.
// Where the planner proves an operand's tile rows and k-blocks affine
// (plan.h, affine_feed), the large real tile gathers it from one per-thread
// address advanced by constant steps instead, and spends the registers the
// tables held on prefetching the next k-step's fragments.
//
// Pipeline: STAGES-deep cp.async ring (16-byte copies whenever the planner
// proved pairs of elements contiguous, 8-byte otherwise), one __syncthreads
// per k-block, warp tiles of m16n8k8 DMMA, accumulators in registers,
// direct (optionally 16-byte) strided stores.  Split-K writes partial tiles
// to a workspace that a second kernel reduces deterministically.
//
// complex128 runs through the same kernel as a real GEMM of twice the N and
// K extents:  A is read as reals with (re,im) as the fastest contracted
// mode, C is written as reals with (re,im) as the fastest n mode, and the
// B tile (kept as complex in shared memory, half the bytes) is expanded on
// the fly in the fragment read:
//     Bhat[(k,a),(n,c)] = sign(a,c) * B[k,n].component(a xor c)
// sign = -1 for (a=1,c=0); conjugation of either operand only changes the
// per-thread sign rule, so it is free.
#include "common.cuh"
#include "plan.h"

namespace qb {

template <int BM, int BN, int BK, int WARPS_M, int WARPS_N, int STAGES>
struct KernelCfg {
  static constexpr int NT = WARPS_M * WARPS_N * 32;
  static constexpr int WM = BM / WARPS_M;
  static constexpr int WN = BN / WARPS_N;
  static constexpr int MT = WM / 16;
  static constexpr int NT8 = WN / 8;
  // tile storage: either [row][k] with pitch BK+4 or [k][row] with pitch
  // rows+4; both are bank-conflict free for the DMMA fragment reads
  // (pitch == 4 mod 16 doubles).  The complex B tile is [k/2][n/2] complex
  // with pitch BN/2+2 complex, which needs fewer doubles than either.
  static constexpr int A_ELEMS =
      (BM * (BK + 4) > BK * (BM + 4)) ? BM * (BK + 4) : BK * (BM + 4);
  static constexpr int B_ELEMS =
      (BN * (BK + 4) > BK * (BN + 4)) ? BN * (BK + 4) : BK * (BN + 4);
  static constexpr int BC_PITCH = BN / 2 + 2;  // complex elements
  // A tile in k-pair layout (contract_tile, LA == 2): [k/2][row][2], the
  // pairs of k of one row adjacent, pitch 2*BM+8 per pair of k (== 8 mod
  // 16 doubles: fragment reads conflict free per half-warp, see load_af)
  static constexpr int AP_PITCH = 2 * BM + 8;
  static_assert(BK / 2 * AP_PITCH <= A_ELEMS, "k-pair A tile fits the stage");
  static constexpr size_t SMEM =
      (size_t)STAGES * (A_ELEMS + B_ELEMS) * 8       // tiles
      + (size_t)(2 * BM + 2 * BN) * 8                // m/n offset tables
      + (size_t)(2 * 2 * BK) * 8;                    // k offset tables (x2)
};

// gather one ROWS x BK tile of 8-byte elements into shared memory
template <int ROWS, int BK, int NT, int KM = -1>
__device__ __forceinline__ void load_tile(
    double *__restrict__ sm, const double *__restrict__ gbase,
    const int64_t *__restrict__ row_off, const int64_t *__restrict__ k_off,
    int vec, int thr, int tid) {
  // vec: 0 scalar, 1 pairs along rows, 2 pairs along k.  thr: 1 walk k.
  // smem layout: vec==1 or (vec==0 && thr==0) -> [k][row]; else [row][k]
  // KM >= 0: the layout is a compile-time constant (specialised kernels)
  const bool kmajor = KM >= 0 ? (KM == 1) : ((vec == 2) || (vec == 0 && thr == 1));
  // the 8-warp 128x128 tile issues up to 16 copies per thread; unrolled in
  // full, ptxas keeps the index arithmetic of all of them live across the
  // k-loop and spills
  constexpr int UNROLL = NT >= 256 ? 4 : 16;
  const int s_row = kmajor ? (BK + 4) : 1;
  const int s_k = kmajor ? 1 : (ROWS + 4);
  if (vec == 0) {
    constexpr int TOTAL = ROWS * BK;
#pragma unroll UNROLL
    for (int c0 = 0; c0 < TOTAL; c0 += NT) {
      int c = c0 + tid;
      if (TOTAL % NT != 0 && c >= TOTAL) break;
      int r, k;
      if (thr) { k = c % BK; r = c / BK; } else { r = c % ROWS; k = c / ROWS; }
      int64_t ro = row_off[r], ko = k_off[k];
      bool ok = (ro >= 0) && (ko >= 0);
      const double *src = ok ? (gbase + ro + ko) : gbase;
      cp_async8(smem_u32(sm + r * s_row + k * s_k), src, ok ? 8 : 0);
    }
  } else if (vec == 2) {
    constexpr int TOTAL = ROWS * BK / 2;
    constexpr int KC = BK / 2;
#pragma unroll UNROLL
    for (int c0 = 0; c0 < TOTAL; c0 += NT) {
      int c = c0 + tid;
      if (TOTAL % NT != 0 && c >= TOTAL) break;
      int r, kc;
      if (thr) { kc = c % KC; r = c / KC; } else { r = c % ROWS; kc = c / ROWS; }
      int k = kc * 2;
      int64_t ro = row_off[r], ko = k_off[k];
      bool ok = (ro >= 0) && (ko >= 0);
      const double *src = ok ? (gbase + ro + ko) : gbase;
      cp_async16(smem_u32(sm + r * s_row + k * s_k), src, ok ? 16 : 0);
    }
  } else {
    constexpr int TOTAL = ROWS * BK / 2;
    constexpr int RC = ROWS / 2;
#pragma unroll UNROLL
    for (int c0 = 0; c0 < TOTAL; c0 += NT) {
      int c = c0 + tid;
      if (TOTAL % NT != 0 && c >= TOTAL) break;
      int rc, k;
      if (thr) { k = c % BK; rc = c / BK; } else { rc = c % RC; k = c / RC; }
      int r = rc * 2;
      int64_t ro = row_off[r], ko = k_off[k];
      bool ok = (ro >= 0) && (ko >= 0);
      const double *src = ok ? (gbase + ro + ko) : gbase;
      cp_async16(smem_u32(sm + r * s_row + k * s_k), src, ok ? 16 : 0);
    }
  }
}

// gather the complex B tile: (BK/2) x (BN/2) complex elements, layout
// [k][n] with pitch PITCH complex; offsets are in doubles (already x2)
template <int NC, int KC, int PITCH, int NT>
__device__ __forceinline__ void load_tile_cplx(
    double *__restrict__ sm, const double *__restrict__ gbase,
    const int64_t *__restrict__ n_off, const int64_t *__restrict__ k_off,
    int thr, int tid) {
  constexpr int TOTAL = NC * KC;
  constexpr int UNROLL = NT >= 256 ? 4 : 16;  // as in load_tile
#pragma unroll UNROLL
  for (int c0 = 0; c0 < TOTAL; c0 += NT) {
    int c = c0 + tid;
    if (TOTAL % NT != 0 && c >= TOTAL) break;
    int n, k;
    if (thr) { k = c % KC; n = c / KC; } else { n = c % NC; k = c / NC; }
    int64_t no = n_off[n], ko = k_off[k];
    bool ok = (no >= 0) && (ko >= 0);
    const double *src = ok ? (gbase + no + ko) : gbase;
    cp_async16(smem_u32(sm + (k * PITCH + n) * 2), src, ok ? 16 : 0);
  }
}

// Affine gather of one real operand tile (plan.h, affine_feed): copy i of
// this thread reads src + i * step and lands at sm + i * sm_step bytes into
// the stage; the next k-block starts kstep further on.  The addresses are
// those the offset tables give, without the tables or predicates.
struct AffineFeed {
  const double *src;
  int64_t step, kstep;
  uint32_t sm, sm_step;
  bool wide;  // 16-byte copies (vec != 0)
};

// LAYOUT: 0 [k][row], 1 [row][k], 2 k pairs ([k/2][row][2], pitch PP)
template <int ROWS, int BK, int NT, int LAYOUT, int PP = 0>
__device__ __forceinline__ AffineFeed affine_setup(const double *base, int64_t rstep,
                                                   int64_t kstep, int vec, int thr,
                                                   int tid) {
  // units: pairs of rows (vec 1) or of k (vec 2), single elements otherwise.
  // NT is a multiple of both tile extents in units, so a thread keeps its
  // inner coordinate and advances its outer one by NT / inner per copy
  static_assert(NT % ROWS == 0 && NT % BK == 0 && (ROWS * BK / 2) % NT == 0,
                "affine feed needs an affine thread walk");
  const int ur = vec == 1 ? 2 : 1, uk = vec == 2 ? 2 : 1;
  const int inner = thr ? BK / uk : ROWS / ur;
  const int a = tid % inner, b = tid / inner, db = NT / inner;
  const int ru = thr ? b : a, ku = thr ? a : b;
  static_assert(LAYOUT != 2 || PP % 2 == 0, "k-pair layout: even pitch");
  // (the k-pair layout takes 16-byte pairs of k, whose first k is even)
  constexpr int s_row = LAYOUT == 1 ? BK + 4 : LAYOUT == 2 ? 2 : 1;
  constexpr int s_k = LAYOUT == 1 ? 1 : LAYOUT == 2 ? PP / 2 : ROWS + 4;
  AffineFeed f;
  f.src = base + ru * rstep + ku * kstep;
  f.sm = (uint32_t)(ru * ur * s_row + ku * uk * s_k) * 8;
  f.step = thr ? db * rstep : db * kstep;
  f.sm_step = (uint32_t)(thr ? db * ur * s_row : db * uk * s_k) * 8;
  f.kstep = (BK / uk) * kstep;
  f.wide = vec != 0;
  return f;
}

template <int ROWS, int BK, int NT>
__device__ __forceinline__ void load_affine(uint32_t stage, const AffineFeed &f, int kb) {
  // a running address, not unrolled: unrolled, ptxas keeps every copy's
  // offset live across the k-loop (they do not depend on kb) and spills
  const double *src = f.src + kb * f.kstep;
  uint32_t dst = stage + f.sm;
  if (f.wide) {
#pragma unroll 1
    for (int i = 0; i < ROWS * BK / 2 / NT; ++i, src += f.step, dst += f.sm_step)
      cp_async16(dst, src, 16);
  } else {
#pragma unroll 1
    for (int i = 0; i < ROWS * BK / NT; ++i, src += f.step, dst += f.sm_step)
      cp_async8(dst, src, 8);
  }
}

__device__ __forceinline__ double flip_sign(double v, unsigned mask_hi) {
  // mask_hi is 0 or 0x80000000
  return __hiloint2double(__double2hiint(v) ^ (int)mask_hi, __double2loint(v));
}

__device__ __forceinline__ unsigned long long global_ns() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}
// tuning: stamp phase `ph` of segment `seg` of this CTA (8 phases x 4 segments)
#define QB_TRACE(ph)                                                        \
  do {                                                                      \
    if (p.trace && threadIdx.x == 0 && sk.seg < 4)                          \
      p.trace[((size_t)sk.bid * 4 + sk.seg) * 8 + (ph)] = global_ns();      \
  } while (0)

// thread-block cluster primitives (the stream-K pair schedule)
__device__ __forceinline__ int cluster_ctarank() {
  uint32_t r;
  asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
  return (int)r;
}
// every thread of both CTAs arrives; writes before it are visible after it
__device__ __forceinline__ void cluster_sync() {
  asm volatile("barrier.cluster.arrive.release.aligned;\n\t"
               "barrier.cluster.wait.acquire.aligned;" ::: "memory");
}
// the address of the same shared-memory byte in CTA `rank` of the cluster
__device__ __forceinline__ uint32_t cluster_map(uint32_t addr, int rank) {
  uint32_t r;
  asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(r) : "r"(addr), "r"(rank));
  return r;
}
__device__ __forceinline__ double ld_cluster(uint32_t addr) {
  double v;
  asm volatile("ld.shared::cluster.f64 %0, [%1];" : "=d"(v) : "r"(addr));
  return v;
}

// stream-K bookkeeping of one tile segment
struct SkSeg {
  int mode;        // 0: classic tile, 1: tail (write partial), 2: head (sum peers)
  int bid;         // this CTA (partial slot)
  int peer0, peer1;  // head: CTAs [peer0, peer1) hold the rest of the tile
  double *part;    // [grid][BM*BN] partial accumulators
  int *flags;      // [grid]
  int seg;         // ordinal of this segment within the CTA (trace only)
};

// FEED: bit 0 / bit 1 = A / B gathered by the affine feed (real operands with
// a compile-time layout only); 0 = offset tables for both.
// PAIR: [kbeg, kend) is one k-half of the tile and the other CTA of this
// 2-CTA cluster runs the other half (streamk_pair_grid); the two halves are
// summed through distributed shared memory and each CTA stores half the rows
template <int BM, int BN, int BK, int WARPS_M, int WARPS_N, int STAGES,
          bool CPLX, int LA = -1, int LB = -1, int FEED = 0, bool PAIR = false>
__device__ __forceinline__ void contract_tile(const ContractParams &p, int pid,
                                              int64_t zb, int ks, int64_t kbeg,
                                              int64_t kend, const SkSeg sk) {
  using Cfg = KernelCfg<BM, BN, BK, WARPS_M, WARPS_N, STAGES>;
  constexpr int NT = Cfg::NT;
  constexpr bool AFA = (FEED & 1) != 0, AFB = (FEED & 2) != 0;
  static_assert(FEED == 0 || (!CPLX && LA >= 0 && LB >= 0), "affine feed: real, fixed layout");
  static_assert(LA != 2 || FEED == 3, "k-pair A tile: both operands affine");
  static_assert(LB != 2, "k-pair layout: A tile only");
  constexpr int MT = Cfg::MT, NT8 = Cfg::NT8;
  constexpr int NCB = BN / 2, KCB = BK / 2;  // complex B tile extents

  extern __shared__ __align__(16) unsigned char smem_raw[];
  double *sA = reinterpret_cast<double *>(smem_raw);
  double *sB = sA + (size_t)STAGES * Cfg::A_ELEMS;
  int64_t *offAm = reinterpret_cast<int64_t *>(sB + (size_t)STAGES * Cfg::B_ELEMS);
  int64_t *offCm = offAm + BM;
  int64_t *offBn = offCm + BM;
  int64_t *offCn = offBn + BN;
  int64_t *ktabA = offCn + BN;      // [2][BK]
  int64_t *ktabB = ktabA + 2 * BK;  // [2][BK]

  QB_TRACE(0);
  // let the next kernel of the stream become resident as SMs free up ...
  asm volatile("griddepcontrol.launch_dependents;");
  // ... and do not touch global memory before the previous one has finished
  // (pointer-array batches read their arrays right away)
  if (p.dA) asm volatile("griddepcontrol.wait;" ::: "memory");
  const int tid = threadIdx.x;
  const int warp = tid >> 5, lane = tid & 31;
  const int g = lane >> 2, t = lane & 3;
  const int wm0 = (warp / WARPS_N) * Cfg::WM;
  const int wn0 = (warp % WARPS_N) * Cfg::WN;

  // effective real extents
  const int64_t Nh = CPLX ? 2 * p.N : p.N;
  const int64_t Kh = CPLX ? 2 * p.K : p.K;

  // ---- which tile / batch / k-split am I -------------------------------
  int tm, tn;
  {
    // grouped rasterisation: walk 8 m-tiles down before moving along n so
    // that concurrently resident CTAs share B panels in L2
    const int G = 8;
    int width = G * p.tiles_n;
    int group = pid / width;
    int first_m = group * G;
    int gsz = min(p.tiles_m - first_m, G);
    int rem = pid - group * width;
    tm = first_m + rem % gsz;
    tn = rem / gsz;
  }
  const int64_t m0 = (int64_t)tm * BM, n0 = (int64_t)tn * BN;

  const double *A = static_cast<const double *>(p.A);
  const double *B = static_cast<const double *>(p.B);
  double *C = static_cast<double *>(p.C);
  constexpr int ES = CPLX ? 2 : 1;  // doubles per element
  if (p.dA) {
    A = static_cast<const double *>(p.dA[zb]);
    B = static_cast<const double *>(p.dB[zb]);
    C = static_cast<double *>(p.dC[zb]);
  } else if (p.b.n) {
    int64_t oa, ob, oc = 0;
    decode2(zb, p.b, oa, ob);
    {  // C batch offset
      int64_t r = zb;
      for (int i = 0; i < p.b.n; ++i) {
        int64_t e = p.b.ext[i];
        int64_t q = r / e;
        oc += (r - q * e) * p.bsC[i];
        r = q;
      }
    }
    A += oa * ES; B += ob * ES; C += oc * ES;
  }

  // ---- per-tile offset tables (in doubles) -----------------------------
  for (int i = tid; i < BM; i += NT) {
    int64_t m = m0 + i, oa = -1, oc = -1;
    if (m < p.M) { decode2(m, p.m, oa, oc); oa *= ES; oc *= ES; }
    offAm[i] = oa; offCm[i] = oc;
  }
  for (int i = tid; i < BN; i += NT) {
    int64_t nh = n0 + i, ob = -1, oc = -1;
    if (nh < Nh) {
      if (CPLX) {
        decode2(nh >> 1, p.n, ob, oc);
        ob *= 2; oc = oc * 2 + (nh & 1);
      } else {
        decode2(nh, p.n, ob, oc);
      }
    }
    // complex: offBn is indexed by the complex column i/2 (even i writes it)
    if (CPLX) { if ((i & 1) == 0) offBn[i >> 1] = ob; }
    else offBn[i] = ob;
    offCn[i] = oc;
  }
  const int nkb = (int)((kend - kbeg + BK - 1) / BK);

  auto fill_ktab = [&](int kb) {
    // offsets of k-block kb into parity slot kb&1 (threads < BK)
    if (!(AFA && AFB) && tid < BK) {
      int64_t kh = kbeg + (int64_t)kb * BK + tid, oa = -1, ob = -1;
      if (kb < nkb && kh < kend) {
        if (CPLX) {
          decode2(kh >> 1, p.k, oa, ob);
          oa = oa * 2 + (kh & 1); ob *= 2;
        } else {
          decode2(kh, p.k, oa, ob);
        }
      }
      ktabA[(kb & 1) * BK + tid] = oa;
      if (CPLX) { if ((tid & 1) == 0) ktabB[(kb & 1) * BK + (tid >> 1)] = ob; }
      else ktabB[(kb & 1) * BK + tid] = ob;
    }
  };
  AffineFeed fA, fB;  // set once the row tables are visible
  auto issue = [&](int kb) {
    if (kb < nkb) {
      const int st = kb % STAGES;
      if constexpr (AFA)
        load_affine<BM, BK, NT>(smem_u32(sA + (size_t)st * Cfg::A_ELEMS), fA, kb);
      else
        load_tile<BM, BK, NT, LA>(sA + (size_t)st * Cfg::A_ELEMS, A, offAm,
                                  ktabA + (kb & 1) * BK, CPLX ? 2 : p.vecA, p.thrA, tid);
      if constexpr (AFB)
        load_affine<BN, BK, NT>(smem_u32(sB + (size_t)st * Cfg::B_ELEMS), fB, kb);
      else if (CPLX)
        load_tile_cplx<NCB, KCB, Cfg::BC_PITCH, NT>(
            sB + (size_t)st * Cfg::B_ELEMS, B, offBn, ktabB + (kb & 1) * BK,
            p.thrB, tid);
      else
        load_tile<BN, BK, NT, LB>(sB + (size_t)st * Cfg::B_ELEMS, B, offBn,
                                  ktabB + (kb & 1) * BK, p.vecB, p.thrB, tid);
    }
    cp_async_commit();
  };

  // prologue: tables for block 0, then STAGES-1 loads in flight
  fill_ktab(0);
  if (!p.dA) asm volatile("griddepcontrol.wait;" ::: "memory");
  __syncthreads();
  QB_TRACE(1);
  // affine operands: row 0 of the tile is in range (the planner proved
  // whole tiles), its table entry is the tile's base
  if constexpr (AFA)
    fA = affine_setup<BM, BK, NT, LA, Cfg::AP_PITCH>(A + offAm[0] + kbeg / (p.vecA == 2 ? 2 : 1) * p.kstepA,
                                           p.rstepA, p.kstepA, p.vecA, p.thrA, tid);
  if constexpr (AFB)
    fB = affine_setup<BN, BK, NT, LB>(B + offBn[0] + kbeg / (p.vecB == 2 ? 2 : 1) * p.kstepB,
                                           p.rstepB, p.kstepB, p.vecB, p.thrB, tid);
#pragma unroll 1
  for (int s = 0; s < STAGES - 1; ++s) {
    issue(s);
    fill_ktab(s + 1);
    __syncthreads();
  }

  QB_TRACE(2);
  double acc[MT][NT8][4];
#pragma unroll
  for (int i = 0; i < MT; ++i)
#pragma unroll
    for (int j = 0; j < NT8; ++j)
#pragma unroll
      for (int v = 0; v < 4; ++v) acc[i][j][v] = 0.0;

  const int vecA = CPLX ? 2 : p.vecA;
  const bool a_kmajor = LA >= 0 ? (LA == 1) : ((vecA == 2) || (vecA == 0 && p.thrA == 1));
  const bool b_kmajor = LB >= 0 ? (LB == 1) : ((p.vecB == 2) || (p.vecB == 0 && p.thrB == 1));
  const int sAm = a_kmajor ? (BK + 4) : 1, sAk = a_kmajor ? 1 : (BM + 4);
  const int sBn = b_kmajor ? (BK + 4) : 1, sBk = b_kmajor ? 1 : (BN + 4);
  // complex B expansion: per-thread component and sign (a = t&1, c = g&1)
  const int ca = t & 1, cc = g & 1, comp = ca ^ cc;
  unsigned sgn_mask = 0;
  if (CPLX) {
    int neg = (ca == 1 && cc == 0) ? 1 : 0;
    if (p.conjB && comp == 1) neg ^= 1;
    if (p.conjA && ca == 1) neg ^= 1;
    sgn_mask = neg ? 0x80000000u : 0u;
  }

  const bool early = ((warp >> 2) & 1) == 0 || (NT <= 128);
  // fragments of k-step kk: A row block i, B column block j
  auto load_af = [&](const double *tA, int kk, int i, double (&a)[4]) {
    const int r = wm0 + i * 16 + g;
    if constexpr (LA == 2) {
      // (r, k) at (k/2)*P + 2r + (k&1); kk is a multiple of 8, so k = kk+t
      // is in pair kk/2 + t/2.  Per half-warp (g < 4 or g >= 4) lanes of
      // t < 2 cover 8 consecutive doubles and lanes of t >= 2 the 8 that
      // P == 8 mod 16 shifts them to: 16 distinct banks of 8 bytes
      constexpr int P = Cfg::AP_PITCH;
      const double *q = tA + 2 * r + (t >> 1) * P + (t & 1) + (kk / 2) * P;
      a[0] = q[0];
      a[1] = q[16];
      a[2] = q[2 * P];
      a[3] = q[2 * P + 16];
      return;
    }
    a[0] = tA[r * sAm + (kk + t) * sAk];
    a[1] = tA[(r + 8) * sAm + (kk + t) * sAk];
    a[2] = tA[r * sAm + (kk + t + 4) * sAk];
    a[3] = tA[(r + 8) * sAm + (kk + t + 4) * sAk];
  };
  auto load_bf = [&](const double *tB, int kk, int j, double (&b)[2]) {
    const int c = wn0 + j * 8 + g;
    if (CPLX) {
      const int kc0 = (kk + t) >> 1, kc1 = (kk + t + 4) >> 1, nc = c >> 1;
      b[0] = flip_sign(tB[(kc0 * Cfg::BC_PITCH + nc) * 2 + comp], sgn_mask);
      b[1] = flip_sign(tB[(kc1 * Cfg::BC_PITCH + nc) * 2 + comp], sgn_mask);
    } else {
      b[0] = tB[c * sBn + (kk + t) * sBk];
      b[1] = tB[c * sBn + (kk + t + 4) * sBk];
    }
  };
#pragma unroll 1
  for (int kb = 0; kb < nkb; ++kb) {
    cp_async_wait<STAGES - 2>();
    __syncthreads();  // stage kb landed; stage kb-1 free; next ktab visible
    if (kb == 0) QB_TRACE(3);
    // the two warps that share a scheduler (warp, warp+4) issue their
    // gathers at different points of the k-block so that one of them always
    // has DMMAs ready while the other does address arithmetic
    if (early) issue(kb + STAGES - 1);
    fill_ktab(kb + STAGES);
    const double *tA = sA + (size_t)(kb % STAGES) * Cfg::A_ELEMS;
    const double *tB = sB + (size_t)(kb % STAGES) * Cfg::B_ELEMS;
    if constexpr (FEED == 0) {
      double af[MT][4], bf[NT8][2];
#pragma unroll
      for (int kk = 0; kk < BK; kk += 8) {
        if (kk == 8 && !early) issue(kb + STAGES - 1);
#pragma unroll
        for (int i = 0; i < MT; ++i) load_af(tA, kk, i, af[i]);
#pragma unroll
        for (int j = 0; j < NT8; ++j) load_bf(tB, kk, j, bf[j]);
#pragma unroll
        for (int i = 0; i < MT; ++i)
#pragma unroll
          for (int j = 0; j < NT8; ++j) dmma_16x8x8(acc[i][j], af[i], bf[j]);
      }
    } else {
      // fragment prefetch on the registers the tables no longer need: the B
      // fragments of k-step kk+8 load while k-step kk's DMMAs issue, and
      // A row block i of kk+8 as soon as its last DMMA of kk has issued.
      // Same DMMAs, same order.
      double af[MT][4], bf[2][NT8][2];
#pragma unroll
      for (int i = 0; i < MT; ++i) load_af(tA, 0, i, af[i]);
#pragma unroll
      for (int j = 0; j < NT8; ++j) load_bf(tB, 0, j, bf[0][j]);
#pragma unroll
      for (int kk = 0; kk < BK; kk += 8) {
        const int cur = (kk / 8) & 1;
        const bool more = kk + 8 < BK;
        if (kk == 8 && !early) issue(kb + STAGES - 1);
        if (more) {
#pragma unroll
          for (int j = 0; j < NT8; ++j) load_bf(tB, kk + 8, j, bf[cur ^ 1][j]);
        }
#pragma unroll
        for (int i = 0; i < MT; ++i) {
#pragma unroll
          for (int j = 0; j < NT8; ++j) dmma_16x8x8(acc[i][j], af[i], bf[cur][j]);
          if (more) load_af(tA, kk + 8, i, af[i]);
        }
      }
    }
  }
  cp_async_wait<0>();
  QB_TRACE(4);

  // ---- stream-K: tail segments park their accumulators, heads collect ----
  if (sk.mode == 1) {
    double *dst = sk.part + (size_t)sk.bid * (BM * BN);
#pragma unroll
    for (int i = 0; i < MT; ++i)
#pragma unroll
      for (int j = 0; j < NT8; ++j)
#pragma unroll
        for (int v = 0; v < 4; ++v)
          __stcg(&dst[((i * NT8 + j) * 4 + v) * NT + tid], acc[i][j][v]);
    __threadfence();
    __syncthreads();
    if (tid == 0) atomicExch(&sk.flags[sk.bid], 1);
    QB_TRACE(6);
    return;
  }
  if (sk.mode == 2) {
    for (int c = sk.peer0; c < sk.peer1; ++c) {
      if (tid == 0) {
        while (atomicAdd(&sk.flags[c], 0) == 0) __nanosleep(100);
        atomicExch(&sk.flags[c], 0);  // left clean for the next launch
      }
      __syncthreads();
      __threadfence();
      const double *src = sk.part + (size_t)c * (BM * BN);
#pragma unroll
      for (int i = 0; i < MT; ++i)
#pragma unroll
        for (int j = 0; j < NT8; ++j)
#pragma unroll
          for (int v = 0; v < 4; ++v)
            acc[i][j][v] += __ldcg(&src[((i * NT8 + j) * 4 + v) * NT + tid]);
    }
  }

  // ---- stream-K pair: rank r stores warp row r of the tile; the other warp
  // row parks its accumulators in this CTA's (now idle) ring for the peer ----
  bool own = true;
  if constexpr (PAIR) {
    constexpr int HALF = NT / WARPS_M;  // threads of one warp row
    static_assert(WARPS_M == 2, "one warp row per CTA of the pair");
    static_assert((size_t)MT * NT8 * 4 * HALF <= (size_t)STAGES * Cfg::A_ELEMS,
                  "parked half fits the A ring");
    const int rank = cluster_ctarank();
    own = warp / WARPS_N == rank;
    const int slot = tid % HALF;
    __syncthreads();  // no warp reads the ring any more
    if (!own) {
#pragma unroll
      for (int i = 0; i < MT; ++i)
#pragma unroll
        for (int j = 0; j < NT8; ++j)
#pragma unroll
          for (int v = 0; v < 4; ++v) sA[((i * NT8 + j) * 4 + v) * HALF + slot] = acc[i][j][v];
    }
    cluster_sync();  // both parked halves visible cluster-wide
    if (own) {
      // the peer's warps of this warp row ran the other k-half of these rows;
      // a + b == b + a, so both CTAs' sums are the same whichever half is local
      const uint32_t peer = cluster_map(smem_u32(sA + slot), rank ^ 1);
#pragma unroll
      for (int i = 0; i < MT; ++i)
#pragma unroll
        for (int j = 0; j < NT8; ++j)
#pragma unroll
          for (int v = 0; v < 4; ++v)
            acc[i][j][v] += ld_cluster(peer + ((i * NT8 + j) * 4 + v) * HALF * 8);
    }
    cluster_sync();  // the peer has read this CTA's shared memory: it may exit
  }

  QB_TRACE(5);
  // ---- epilogue ----------------------------------------------------------
  if (!PAIR && p.splitk > 1) {
    // canonical [split][batch][M][Nh] partial buffer
    double *P = p.partial + ((int64_t)ks * p.nbatch + zb) * p.M * Nh;
#pragma unroll
    for (int i = 0; i < MT; ++i)
#pragma unroll
      for (int j = 0; j < NT8; ++j)
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          int64_t m = m0 + wm0 + i * 16 + g + h * 8;
          int64_t n = n0 + wn0 + j * 8 + 2 * t;
          if (m < p.M) {
            if (n < Nh) P[m * Nh + n] = acc[i][j][2 * h];
            if (n + 1 < Nh) P[m * Nh + n + 1] = acc[i][j][2 * h + 1];
          }
        }
    return;
  }
  const bool vecC = CPLX ? true : (p.vecC != 0);
  const double alpha = p.alpha, beta = p.beta;
#pragma unroll
  for (int i = 0; i < MT; ++i)
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int r = wm0 + i * 16 + g + h * 8;
      const int64_t om = own ? offCm[r] : -1;
      if (om < 0) continue;
#pragma unroll
      for (int j = 0; j < NT8; ++j) {
        const int c = wn0 + j * 8 + 2 * t;
        const int64_t on0 = offCn[c], on1 = offCn[c + 1];
        double v0 = alpha * acc[i][j][2 * h], v1 = alpha * acc[i][j][2 * h + 1];
        if (vecC) {
          // (c, c+1) are contiguous and 16B aligned (planner / complex pair)
          if (on0 >= 0) {
            double2 *dst = reinterpret_cast<double2 *>(C + om + on0);
            if (beta != 0.0) {
              double2 old = *dst;
              v0 += beta * old.x; v1 += beta * old.y;
            }
            *dst = make_double2(v0, v1);
          }
        } else {
          if (on0 >= 0) {
            if (beta != 0.0) v0 += beta * C[om + on0];
            C[om + on0] = v0;
          }
          if (on1 >= 0) {
            if (beta != 0.0) v1 += beta * C[om + on1];
            C[om + on1] = v1;
          }
        }
      }
    }
  // pair: thread 0 of rank 1 stores nothing; stamp once the owners have
  if constexpr (PAIR) {
    if (p.trace) __syncthreads();
  }
  QB_TRACE(6);
}

template <int BM, int BN, int BK, int WARPS_M, int WARPS_N, int STAGES,
          bool CPLX, int LA, int LB, int FEED>
__device__ __forceinline__ void classic_grid(const ContractParams &p) {
  const int64_t Kh = CPLX ? 2 * p.K : p.K;
  const int ks = blockIdx.z;
  const int64_t kbeg = (int64_t)ks * p.k_per_split;  // in real-k units
  const int64_t kend = min(Kh, kbeg + p.k_per_split);
  SkSeg sk{0, (int)(blockIdx.x + gridDim.x * (blockIdx.y + gridDim.y * blockIdx.z)), 0, 0, nullptr, nullptr, 0};
  contract_tile<BM, BN, BK, WARPS_M, WARPS_N, STAGES, CPLX, LA, LB, FEED>(
      p, blockIdx.x, blockIdx.y, ks, kbeg, kend, sk);
}

template <int BM, int BN, int BK, int WARPS_M, int WARPS_N, int STAGES,
          bool CPLX, int LA = -1, int LB = -1>
__global__ void __launch_bounds__(WARPS_M *WARPS_N * 32, 1)
    contract_f64_kernel(const __grid_constant__ ContractParams p) {
  classic_grid<BM, BN, BK, WARPS_M, WARPS_N, STAGES, CPLX, LA, LB, 0>(p);
}

// the large real tile with at least one operand on the affine feed
template <int BM, int BN, int BK, int WARPS_M, int WARPS_N, int STAGES, int LA,
          int LB, int FEED>
__global__ void __launch_bounds__(WARPS_M *WARPS_N * 32, 1)
    contract_f64_affine_kernel(const __grid_constant__ ContractParams p) {
  classic_grid<BM, BN, BK, WARPS_M, WARPS_N, STAGES, false, LA, LB, FEED>(p);
}

// The large real tile with both operands affine and the A tile in k-pair
// layout (LA == 2): for an A operand whose 16-byte pairs lie along k while
// its threads walk rows (plan.h, a_kpair), e.g. an MPS site tensor read as
// [b', (a', p)].  In [row][k] layout each 32-byte sector of a warp's
// contiguous read lands in two rows 288 bytes apart; in k-pair layout a
// sector is 32 contiguous bytes of the tile.  Same tile contents, same DMMAs
template <int BM, int BN, int BK, int WARPS_M, int WARPS_N, int STAGES, int LB>
__global__ void __launch_bounds__(WARPS_M *WARPS_N * 32, 1)
    contract_f64_kpair_kernel(const __grid_constant__ ContractParams p) {
  classic_grid<BM, BN, BK, WARPS_M, WARPS_N, STAGES, false, 2, LB, 3>(p);
}

// Stream-K: one persistent CTA per SM; the (tile, k-block) iteration space is
// cut into gridDim.x equal contiguous ranges, so every SM gets the same number
// of k-blocks whatever the tile count (no wave quantisation).  A range that
// starts inside a tile is a TAIL: its accumulators go to a per-CTA slot of the
// workspace; the CTA whose range holds the first k-block of that tile (the
// HEAD, processed last in its range, i.e. long after the tails were written)
// adds them in a fixed order and runs the normal epilogue.
template <int BM, int BN, int BK, int WARPS_M, int WARPS_N, int STAGES,
          bool CPLX, int LA, int LB, int FEED>
__device__ __forceinline__ void streamk_grid(const ContractParams &p) {
  const int64_t Kh = CPLX ? 2 * p.K : p.K;
  const int64_t nkbT = (Kh + BK - 1) / BK;
  const int64_t tiles = (int64_t)p.tiles_m * p.tiles_n;
  const int G = gridDim.x, bid = blockIdx.x;
  // equal shares of COST: every tile carries sk_head extra k-blocks (fix-up
  // + epilogue) that are charged to whoever runs its first k-block
  const int64_t H = p.sk_head, span = nkbT + H, total_cost = tiles * span;
  auto start = [&](int c) -> int64_t {
    const int64_t x = total_cost * c / G, t = x / span;
    return t * nkbT + max(x - t * span - H, (int64_t)0);
  };
  const int64_t u0 = start(bid), u1 = start(bid + 1);
  double *part = p.partial;
  int *flags = p.flags;
  int seg = 0;
  for (int64_t u = u0; u < u1;) {
    const int64_t tile = u / nkbT, kb0 = u - tile * nkbT;
    const int64_t kb1 = min(nkbT, kb0 + (u1 - u));
    SkSeg sk{0, bid, 0, 0, part, flags, seg++};
    if (kb0 > 0) sk.mode = 1;
    else if (kb1 < nkbT) {
      // peers: CTAs after this one whose range starts inside this tile
      sk.mode = 2;
      sk.peer0 = bid + 1;
      int c = bid + 1;
      while (c < G && start(c) < (tile + 1) * nkbT) ++c;
      sk.peer1 = c;
    }
    contract_tile<BM, BN, BK, WARPS_M, WARPS_N, STAGES, CPLX, LA, LB, FEED>(
        p, (int)tile, 0, 0, kb0 * BK, min(Kh, kb1 * BK), sk);
    u += kb1 - kb0;
    __syncthreads();  // shared memory is reused by the next segment
  }
}

template <int BM, int BN, int BK, int WARPS_M, int WARPS_N, int STAGES,
          bool CPLX, int LA = -1, int LB = -1>
__global__ void __launch_bounds__(WARPS_M *WARPS_N * 32, 1)
    contract_f64_streamk_kernel(const __grid_constant__ ContractParams p) {
  streamk_grid<BM, BN, BK, WARPS_M, WARPS_N, STAGES, CPLX, LA, LB, 0>(p);
}

template <int BM, int BN, int BK, int WARPS_M, int WARPS_N, int STAGES, int LA,
          int LB, int FEED>
__global__ void __launch_bounds__(WARPS_M *WARPS_N * 32, 1)
    contract_f64_affine_streamk_kernel(const __grid_constant__ ContractParams p) {
  streamk_grid<BM, BN, BK, WARPS_M, WARPS_N, STAGES, false, LA, LB, FEED>(p);
}

template <int BM, int BN, int BK, int WARPS_M, int WARPS_N, int STAGES, int LB>
__global__ void __launch_bounds__(WARPS_M *WARPS_N * 32, 1)
    contract_f64_kpair_streamk_kernel(const __grid_constant__ ContractParams p) {
  streamk_grid<BM, BN, BK, WARPS_M, WARPS_N, STAGES, false, 2, LB, 3>(p);
}

// Stream-K pair schedule, for a stream-K grid with at most half as many tiles
// as CTAs: the equal-cost cut is then "every tile in two halves".  The grid
// runs as clusters of 2 CTAs; cluster c takes tile c (the same grouped
// rasterisation), rank 0 its first nkbT/2 k-blocks and rank 1 the rest, and
// the two halves are summed in distributed shared memory (contract_tile,
// PAIR): no workspace, no flags, and no wait outside the cluster.
template <int BM, int BN, int BK, int WARPS_M, int WARPS_N, int STAGES,
          bool CPLX, int LA, int LB, int FEED>
__device__ __forceinline__ void streamk_pair_grid(const ContractParams &p) {
  const int tile = blockIdx.x / 2;
  // surplus clusters: both CTAs leave here, before either reaches a barrier
  if (tile >= p.tiles_m * p.tiles_n) return;
  const int64_t Kh = CPLX ? 2 * p.K : p.K;
  const int64_t kmid = (Kh + BK - 1) / BK / 2 * BK;
  const int rank = cluster_ctarank();
  SkSeg sk{0, (int)blockIdx.x, 0, 0, nullptr, nullptr, 0};
  contract_tile<BM, BN, BK, WARPS_M, WARPS_N, STAGES, CPLX, LA, LB, FEED, true>(
      p, tile, 0, 0, rank ? kmid : 0, rank ? Kh : kmid, sk);
}

template <int BM, int BN, int BK, int WARPS_M, int WARPS_N, int STAGES,
          bool CPLX, int LA = -1, int LB = -1>
__global__ void __launch_bounds__(WARPS_M *WARPS_N * 32, 1)
    contract_f64_pair_kernel(const __grid_constant__ ContractParams p) {
  streamk_pair_grid<BM, BN, BK, WARPS_M, WARPS_N, STAGES, CPLX, LA, LB, 0>(p);
}

template <int BM, int BN, int BK, int WARPS_M, int WARPS_N, int STAGES, int LA,
          int LB, int FEED>
__global__ void __launch_bounds__(WARPS_M *WARPS_N * 32, 1)
    contract_f64_affine_pair_kernel(const __grid_constant__ ContractParams p) {
  streamk_pair_grid<BM, BN, BK, WARPS_M, WARPS_N, STAGES, false, LA, LB, FEED>(p);
}

template <int BM, int BN, int BK, int WARPS_M, int WARPS_N, int STAGES, int LB>
__global__ void __launch_bounds__(WARPS_M *WARPS_N * 32, 1)
    contract_f64_kpair_pair_kernel(const __grid_constant__ ContractParams p) {
  streamk_pair_grid<BM, BN, BK, WARPS_M, WARPS_N, STAGES, false, 2, LB, 3>(p);
}

// deterministic split-K reduction + strided scatter into C
template <bool CPLX>
__global__ void splitk_reduce_f64_kernel(const __grid_constant__ ContractParams p) {
  const int64_t Nh = CPLX ? 2 * p.N : p.N;
  const int64_t MN = p.M * Nh;
  const int64_t total = MN * p.nbatch;
  constexpr int ES = CPLX ? 2 : 1;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total;
       i += (int64_t)gridDim.x * blockDim.x) {
    int64_t zb = i / MN, r = i - zb * MN;
    int64_t m = r / Nh, nh = r - m * Nh;
    double s = 0.0;
    for (int ks = 0; ks < p.splitk; ++ks)
      s += p.partial[((int64_t)ks * p.nbatch + zb) * MN + r];
    int64_t oa, om, on, ob, oc = 0;
    decode2(m, p.m, oa, om);
    decode2(CPLX ? (nh >> 1) : nh, p.n, ob, on);
    double *C = static_cast<double *>(p.C);
    if (p.dC) C = static_cast<double *>(p.dC[zb]);
    else {
      int64_t q = zb;
      for (int j = 0; j < p.b.n; ++j) {
        int64_t e = p.b.ext[j];
        int64_t qq = q / e;
        oc += (q - qq * e) * p.bsC[j];
        q = qq;
      }
    }
    double *dst = &C[(oc + om + on) * ES + (CPLX ? (nh & 1) : 0)];
    s *= p.alpha;
    if (p.beta != 0.0) s += p.beta * *dst;
    *dst = s;
  }
}

// Launch with programmatic stream serialisation: the CTAs of this kernel may
// become resident while the previous kernel in the stream drains (they build
// their offset tables, then block in griddepcontrol.wait until it has
// completed and flushed), which hides the launch latency between the
// back-to-back contractions of a tree / an MPS sweep.  Launches recorded into
// a stream capture go without the attribute.  cluster > 1: CTAs are launched
// in thread-block clusters of that many along x.
template <typename Kern>
static int launch_pdl(Kern kern, dim3 grid, int threads, size_t smem, cudaStream_t st,
                      const ContractParams &p, int cluster = 1) {
  cudaLaunchConfig_t cfg;
  memset(&cfg, 0, sizeof(cfg));
  cfg.gridDim = grid; cfg.blockDim = dim3(threads); cfg.dynamicSmemBytes = smem;
  cfg.stream = st;
  cudaLaunchAttribute attr[2];
  unsigned n = 0;
  if (cluster > 1) {
    attr[n].id = cudaLaunchAttributeClusterDimension;
    attr[n].val.clusterDim.x = cluster;
    attr[n].val.clusterDim.y = 1;
    attr[n].val.clusterDim.z = 1;
    ++n;
  }
  cudaStreamCaptureStatus cap = cudaStreamCaptureStatusNone;
  cudaStreamIsCapturing(st, &cap);
  if (cap == cudaStreamCaptureStatusNone) {
    attr[n].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[n].val.programmaticStreamSerializationAllowed = 1;
    ++n;
  }
  cfg.attrs = n ? attr : nullptr; cfg.numAttrs = n;
  QB_CUDA_CHECK(cudaLaunchKernelEx(&cfg, kern, p));
  QB_LAUNCH_CHECK();
  return 0;
}

// FEED != 0: the large real tile with affine operands (contract_tile)
template <int BM, int BN, int BK, int WARPS_M, int WARPS_N, int STAGES,
          bool CPLX, int LA = -1, int LB = -1, int FEED = 0>
static int launch_cfg(const ContractParams &p, cudaStream_t st) {
  using Cfg = KernelCfg<BM, BN, BK, WARPS_M, WARPS_N, STAGES>;
  auto kern = [] {
    if constexpr (FEED == 0)
      return contract_f64_kernel<BM, BN, BK, WARPS_M, WARPS_N, STAGES, CPLX, LA, LB>;
    else if constexpr (LA == 2)
      return contract_f64_kpair_kernel<BM, BN, BK, WARPS_M, WARPS_N, STAGES, LB>;
    else
      return contract_f64_affine_kernel<BM, BN, BK, WARPS_M, WARPS_N, STAGES, LA, LB, FEED>;
  }();
  static bool attr_set = false;
  if (!attr_set) {
    QB_CUDA_CHECK(cudaFuncSetAttribute(
        kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)Cfg::SMEM));
    attr_set = true;
  }
  if (p.nbatch > 65535 || p.splitk > 65535) {
    set_error("batch count %lld exceeds the launch limit", (long long)p.nbatch);
    return -100;
  }
  dim3 grid((unsigned)((int64_t)p.tiles_m * p.tiles_n), (unsigned)p.nbatch,
            (unsigned)p.splitk);
  return launch_pdl(kern, grid, Cfg::NT, Cfg::SMEM, st, p);
}

// The cfg-0 (large) tile: 128 x 128, BK 32, 3 stages, 8 warps.  Its real
// kernels are specialised on the shared-memory layout of the operands
// (a_kmajor / b_kmajor, plan.h), which the route carries, and on which
// operands the planner proved affine (feedA / feedB).  The complex kernel
// takes its layout at run time and always gathers through the tables.
using LargeCfg = KernelCfg<128, 128, 32, 2, 4, 3>;

// 2-CTA clusters of the large tile that the current device holds at once,
// asked once per device; -1 without a device.  Every pair kernel has the same
// block, the same shared memory and one CTA per SM, so one kernel answers for
// all of them.
static int pair_active_clusters() {
  constexpr int kMaxDevices = 64;
  static std::atomic<int> known[kMaxDevices];  // clusters + 1; 0 = not asked yet
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || dev >= kMaxDevices) {
    cudaGetLastError();
    return -1;
  }
  int n = known[dev].load();
  if (n) return n - 1;
  auto kern = contract_f64_pair_kernel<128, 128, 32, 2, 4, 3, true>;
  cudaLaunchConfig_t cfg;
  memset(&cfg, 0, sizeof(cfg));
  cfg.gridDim = dim3(2); cfg.blockDim = dim3(LargeCfg::NT);
  cfg.dynamicSmemBytes = LargeCfg::SMEM;
  cudaLaunchAttribute attr;
  attr.id = cudaLaunchAttributeClusterDimension;
  attr.val.clusterDim.x = 2; attr.val.clusterDim.y = 1; attr.val.clusterDim.z = 1;
  cfg.attrs = &attr; cfg.numAttrs = 1;
  n = 0;
  if (cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize,
                           (int)LargeCfg::SMEM) != cudaSuccess ||
      cudaOccupancyMaxActiveClusters(&n, kern, &cfg) != cudaSuccess) {
    cudaGetLastError();  // no pair schedule on this device
    n = 0;
  }
  known[dev].store(n + 1);
  return n;
}

bool streamk_pair(const PairPlan &plan) {
  const int G = plan.streamk;
  const int64_t tiles = (int64_t)plan.p.tiles_m * plan.p.tiles_n;
  if (G <= 0 || G % 2 != 0 || tiles * 2 > G || plan.p.nbatch != 1) return false;
  int clusters = pair_active_clusters();
  if (clusters < 0) clusters = G / 2;
  // all tiles in one wave of clusters
  return clusters >= tiles;
}

// G CTAs as G/2 clusters; the flag words stay untouched (and zero)
template <bool CPLX, int LA, int LB, int FEED>
static int launch_pair_l(const PairPlan &plan, cudaStream_t st) {
  auto kern = [] {
    if constexpr (FEED == 0)
      return contract_f64_pair_kernel<128, 128, 32, 2, 4, 3, CPLX, LA, LB>;
    else if constexpr (LA == 2)
      return contract_f64_kpair_pair_kernel<128, 128, 32, 2, 4, 3, LB>;
    else
      return contract_f64_affine_pair_kernel<128, 128, 32, 2, 4, 3, LA, LB, FEED>;
  }();
  static bool attr_set = false;
  if (!attr_set) {
    QB_CUDA_CHECK(cudaFuncSetAttribute(
        kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)LargeCfg::SMEM));
    attr_set = true;
  }
  return launch_pdl(kern, dim3(plan.streamk), LargeCfg::NT, LargeCfg::SMEM, st, plan.p, 2);
}

template <bool CPLX, int LA, int LB, int FEED>
static int launch_streamk_l(const PairPlan &plan, cudaStream_t st) {
  if (streamk_pair(plan)) return launch_pair_l<CPLX, LA, LB, FEED>(plan, st);
  using Cfg = LargeCfg;
  auto kern = [] {
    if constexpr (FEED == 0)
      return contract_f64_streamk_kernel<128, 128, 32, 2, 4, 3, CPLX, LA, LB>;
    else if constexpr (LA == 2)
      return contract_f64_kpair_streamk_kernel<128, 128, 32, 2, 4, 3, LB>;
    else
      return contract_f64_affine_streamk_kernel<128, 128, 32, 2, 4, 3, LA, LB, FEED>;
  }();
  static bool attr_set = false;
  if (!attr_set) {
    QB_CUDA_CHECK(cudaFuncSetAttribute(
        kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)Cfg::SMEM));
    attr_set = true;
  }
  const int G = plan.streamk;
  if (!plan.flags_clean)
    QB_CUDA_CHECK(cudaMemsetAsync(plan.p.flags, 0, sizeof(int) * G, st));
  return launch_pdl(kern, dim3(G), Cfg::NT, Cfg::SMEM, st, plan.p);
}

template <int LA, int LB>
static int launch_streamk_feed(const PairPlan &plan, cudaStream_t st) {
  if (LA == 1 && a_kpair(plan.p)) return launch_streamk_l<false, 2, LB, 3>(plan, st);
  switch (plan.p.feedA | plan.p.feedB << 1) {
    case 0: return launch_streamk_l<false, LA, LB, 0>(plan, st);
    case 1: return launch_streamk_l<false, LA, LB, 1>(plan, st);
    case 2: return launch_streamk_l<false, LA, LB, 2>(plan, st);
    default: return launch_streamk_l<false, LA, LB, 3>(plan, st);
  }
}

template <bool CPLX>
static int launch_streamk(const PairPlan &plan, const Route &r, cudaStream_t st) {
  if constexpr (CPLX) {
    return launch_streamk_l<true, -1, -1, 0>(plan, st);
  } else {
    switch (r.layout) {
      case 0: return launch_streamk_feed<0, 0>(plan, st);
      case 1: return launch_streamk_feed<0, 1>(plan, st);
      case 2: return launch_streamk_feed<1, 0>(plan, st);
      default: return launch_streamk_feed<1, 1>(plan, st);
    }
  }
}

template <int LA, int LB>
static int launch_cfg0_feed(const ContractParams &p, cudaStream_t st) {
  if (LA == 1 && a_kpair(p)) return launch_cfg<128, 128, 32, 2, 4, 3, false, 2, LB, 3>(p, st);
  switch (p.feedA | p.feedB << 1) {
    case 0: return launch_cfg<128, 128, 32, 2, 4, 3, false, LA, LB, 0>(p, st);
    case 1: return launch_cfg<128, 128, 32, 2, 4, 3, false, LA, LB, 1>(p, st);
    case 2: return launch_cfg<128, 128, 32, 2, 4, 3, false, LA, LB, 2>(p, st);
    default: return launch_cfg<128, 128, 32, 2, 4, 3, false, LA, LB, 3>(p, st);
  }
}

template <bool CPLX>
static int launch_cfg0(const ContractParams &p, const Route &r, cudaStream_t st) {
  if constexpr (CPLX) {
    return launch_cfg<128, 128, 32, 2, 4, 3, true>(p, st);
  } else {
    switch (r.layout) {
      case 0: return launch_cfg0_feed<0, 0>(p, st);
      case 1: return launch_cfg0_feed<0, 1>(p, st);
      case 2: return launch_cfg0_feed<1, 0>(p, st);
      default: return launch_cfg0_feed<1, 1>(p, st);
    }
  }
}

template <bool CPLX>
static int launch_contract_t(const PairPlan &plan, cudaStream_t st) {
  const ContractParams &p = plan.p;
  const Route r = dmma_route(plan, p.partial != nullptr);
  if (r.kind == ROUTE_DMMA_STREAMK) return launch_streamk<CPLX>(plan, r, st);
  int rc;
  switch (r.cfg) {
    case 0: rc = launch_cfg0<CPLX>(p, r, st); break;
    case 1: rc = launch_cfg<64, 64, 16, 2, 2, 4, CPLX>(p, st); break;
    case 2: rc = launch_cfg<128, 32, 16, 4, 1, 4, CPLX>(p, st); break;
    case 3: rc = launch_cfg<32, 128, 16, 1, 4, 4, CPLX>(p, st); break;
    default: rc = launch_cfg<32, 32, 16, 2, 1, 4, CPLX>(p, st); break;
  }
  if (rc) return rc;
  if (r.splitk > 1) {
    int64_t total = p.M * p.N * p.nbatch * (CPLX ? 2 : 1);
    int blocks = (int)std::min<int64_t>((total + 255) / 256, (int64_t)sm_count() * 8);
    splitk_reduce_f64_kernel<CPLX><<<blocks, 256, 0, st>>>(p);
    QB_LAUNCH_CHECK();
  }
  return 0;
}

int launch_contract_f64(const PairPlan &plan, cudaStream_t st) {
  return launch_contract_t<false>(plan, st);
}
int launch_contract_c128(const PairPlan &plan, cudaStream_t st) {
  return launch_contract_t<true>(plan, st);
}

}  // namespace qb
