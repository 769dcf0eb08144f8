// Host-side planner: turns a labelled pairwise contraction of two strided
// tensors into a (batched) GEMM *view* -- groups of modes with strides in
// A, B and C -- without moving any data.  This is the integer "index
// bookkeeping" half of quimb's tensordot/einsum path (cotengra's pairwise
// step; see quimb/tensor/tensor_core.py:3786-3808 for the tensordot call
// site): which axes are free / contracted / batch, and in which order the
// output axes come out, is decided by the caller's labelsC and is
// reproduced bit-exactly because C is addressed through its own strides.
#pragma once
#include <stdint.h>
#include <stdlib.h>

#include <algorithm>
#include <vector>

#include "common.cuh"

namespace qb {

constexpr int MAXM = 12;  // modes per group after merging

struct ModeGroup {
  int32_t n;
  int32_t ext[MAXM];
  int64_t s0[MAXM];
  int64_t s1[MAXM];
};

// Parameters of one contraction launch.  Passed by value (__grid_constant__).
struct ContractParams {
  const void *A;
  const void *B;
  void *C;
  // for pointer-array batched launches (may be null)
  const void *const *dA;
  const void *const *dB;
  void *const *dC;
  int64_t M, N, K, nbatch;
  ModeGroup m;        // s0 = stride in A, s1 = stride in C
  ModeGroup n;        // s0 = stride in B, s1 = stride in C
  ModeGroup k;        // s0 = stride in A, s1 = stride in B
  ModeGroup b;        // s0 = stride in A, s1 = stride in B
  int64_t bsC[MAXM];  // batch stride in C
  int32_t vecA, vecB, vecC;  // 0: scalar, 1: pairs along M (N for B), 2: pairs along K
  int32_t thrA, thrB;        // 0: consecutive threads walk M (N), 1: walk K
  int32_t conjA, conjB;
  int32_t splitk;            // >1: partial sums to workspace
  int64_t k_per_split;       // multiple of BK
  double *partial;           // [splitk][nbatch][M][N]
  int32_t tiles_m, tiles_n;
  // C = alpha * A.B + beta * C   (real scalars; beta != 0 reads C)
  double alpha, beta;
  // stream-K: per-CTA "partial parked" flags (self-resetting: zero between
  // launches) and the cost, in k-blocks, charged to the CTA that owns a tile's
  // fix-up + epilogue when the iteration space is cut into equal shares
  int *flags;
  int32_t sk_head;
  // affine operand feed of the large real tile (affine_feed below): feedX = 1
  // when every row of a tile and every k-block of operand X sits at
  // tile_base + row_unit * rstepX + k_unit * kstepX (units: the operand's
  // 16-byte pairs along rows / k, single elements otherwise)
  int32_t feedA, feedB;
  int64_t rstepA, kstepA, rstepB, kstepB;
  // tuning (QB_TRACE=1): per-CTA globaltimer stamps of the kernel phases
  unsigned long long *trace;
};

struct PairPlan {
  ContractParams p;
  int dtype;
  int cfg;           // tile configuration id
  int streamk;       // >0: persistent stream-K launch with this many CTAs
  bool flags_clean;  // caller keeps the flag words zero between launches
  bool empty_out;    // output has zero elements
  bool zero_fill;    // contracted extent is zero -> C = 0
  int64_t out_elems;
};

struct RawMode {
  int32_t label;
  int64_t ext;
  int64_t sA, sB, sC;
  bool inA, inB, inC;
};

inline int find_mode(std::vector<RawMode> &v, int32_t label) {
  for (size_t i = 0; i < v.size(); ++i)
    if (v[i].label == label) return (int)i;
  return -1;
}

struct GM {
  int64_t ext, a, b, c;
};

inline void merge_group(std::vector<GM> &g) {
  // merge neighbours that are jointly contiguous in every tensor
  std::vector<GM> out;
  for (auto &x : g) {
    if (!out.empty()) {
      GM &l = out.back();
      if (x.a == l.a * l.ext && x.b == l.b * l.ext && x.c == l.c * l.ext) {
        l.ext *= x.ext;
        continue;
      }
    }
    out.push_back(x);
  }
  g.swap(out);
}

// tile configurations (must match the instantiations in contract_dmma.cu)
struct TileCfg {
  int bm, bn, bk, threads;
};
static const TileCfg kTileCfgs[] = {
    {128, 128, 32, 256},  // 0: large (3 stages)
    {64, 64, 16, 128},    // 1: medium
    {128, 32, 16, 128},   // 2: tall (small N)
    {32, 128, 16, 128},   // 3: wide (small M)
    {32, 32, 16, 64},     // 4: small
};
constexpr int kNumTileCfgs = 5;

// fp64 tensor-core rate of one SM per microsecond: H100 SXM, 128 DMMA FMA per
// clock at the 1.98 GHz boost clock (data sheet: 67 TFLOP/s over 132 SMs)
constexpr double kDmmaFmaPerSmUs = 128.0 * 1980.0;

inline int64_t cdiv(int64_t a, int64_t b) { return (a + b - 1) / b; }

// Affine feed of one operand of the large real tile (rows_tile x bk blocks).
// It holds when
//  - the leading modes of the operand's row group form one run that is
//    jointly strided in this operand (stride[i] = stride[i-1] * ext[i-1])
//    over a multiple of rows_tile rows: every tile's rows then sit at
//    tile_base + r * stride[0];
//  - its whole k group, counted in the operand's vector units (pairs of k when
//    vec == 2), is one such run and K is a multiple of bk: a k-block's
//    offsets are block_base + k_unit * kstep, and block_base advances by a
//    constant per k-block.
// The tile's thread walk (NT a multiple of both tile extents in units) keeps
// every copy of a thread on base + i * step; contract_dmma.cu asserts that.
// Steps are in doubles, per unit: rows in pairs when vec == 1.
inline bool affine_feed(const ModeGroup &rows, const ModeGroup &k, bool k_second, int vec,
                        int rows_tile, int bk, int64_t &rstep, int64_t &kstep) {
  if (rows.n == 0 || k.n == 0) return false;
  int64_t run = rows.ext[0];
  for (int i = 1; i < rows.n && rows.s0[i] == rows.s0[i - 1] * rows.ext[i - 1]; ++i)
    run *= rows.ext[i];
  if (run % rows_tile) return false;
  auto ks = [&](int i) { return k_second ? k.s1[i] : k.s0[i]; };
  int64_t K = 1;
  for (int i = 0; i < k.n; ++i) K *= k.ext[i];
  if (K % bk) return false;
  // the first k mode in units: extent / uk at stride uk (vec == 2 proved
  // unit stride and an even extent); a mode of one pair drops out
  const int uk = vec == 2 ? 2 : 1;
  int first = 0;
  int64_t e = k.ext[0] / uk, s = ks(0) * uk;
  if (e == 1) { first = 1; e = k.ext[1]; s = ks(1); }  // k.n > 1: K >= bk > 2
  kstep = s;
  for (int i = first + 1; i < k.n; ++i) {
    if (ks(i) != s * e) return false;
    s = ks(i); e = k.ext[i];
  }
  rstep = rows.s0[0] * (vec == 1 ? 2 : 1);
  return true;
}

// returns 0 or a negative argument-error code; fills plan
inline int plan_pair(const qb_tensor_t *A, const int32_t *la,
                     const qb_tensor_t *B, const int32_t *lb,
                     const qb_tensor_t *C, const int32_t *lc, int conjA,
                     int conjB, PairPlan &plan, int max_splitk = 64) {
  if (!A) return -1;
  if (!B) return -3;
  if (!C) return -5;
  if (A->rank < 0 || A->rank > QB_MAX_RANK) return -1;
  if (B->rank < 0 || B->rank > QB_MAX_RANK) return -3;
  if (C->rank < 0 || C->rank > QB_MAX_RANK) return -5;
  if (A->dtype != B->dtype || A->dtype != C->dtype) {
    set_error("dtype mismatch A=%d B=%d C=%d", A->dtype, B->dtype, C->dtype);
    return -1;
  }
  std::vector<RawMode> modes;
  auto add = [&](const qb_tensor_t *T, const int32_t *lab, int which) -> int {
    for (int i = 0; i < T->rank; ++i) {
      int j = find_mode(modes, lab[i]);
      if (j < 0) {
        RawMode r{lab[i], T->shape[i], 0, 0, 0, false, false, false};
        modes.push_back(r);
        j = (int)modes.size() - 1;
      }
      RawMode &r = modes[j];
      if (r.ext != T->shape[i]) {
        set_error("extent mismatch for label %d: %lld vs %lld", lab[i],
                  (long long)r.ext, (long long)T->shape[i]);
        return -(2 * which + 2);
      }
      // a label repeated inside one tensor addresses its diagonal:
      // strides simply add up
      if (which == 0) { r.sA += T->stride[i]; r.inA = true; }
      if (which == 1) { r.sB += T->stride[i]; r.inB = true; }
      if (which == 2) {
        if (r.inC) {
          set_error("label %d repeated in the output", lab[i]);
          return -6;
        }
        r.sC += T->stride[i]; r.inC = true;
      }
    }
    return 0;
  };
  int rc;
  if ((rc = add(A, la, 0))) return rc;
  if ((rc = add(B, lb, 1))) return rc;
  if ((rc = add(C, lc, 2))) return rc;

  std::vector<GM> gm, gn, gk, gb;
  bool zero_k = false, zero_out = false;
  for (auto &r : modes) {
    if (r.inC && !r.inA && !r.inB) {
      set_error("output label %d appears in neither input", r.label);
      return -6;
    }
    if (r.ext == 0) {
      if (r.inC) zero_out = true; else zero_k = true;
      continue;
    }
    if (r.ext == 1) continue;  // contributes nothing to addressing
    GM g{r.ext, r.sA, r.sB, r.sC};
    if (r.inC) {
      if (r.inA && r.inB) gb.push_back(g);
      else if (r.inA) gm.push_back(g);
      else gn.push_back(g);
    } else {
      gk.push_back(g);  // contracted, or summed-out of one operand (stride 0)
    }
  }
  // order inside a group is free: choose it for memory contiguity
  auto by_a = [](const GM &x, const GM &y) {
    if (x.a != y.a) return x.a < y.a;
    return x.c < y.c;
  };
  auto by_b = [](const GM &x, const GM &y) {
    if (x.b != y.b) return x.b < y.b;
    return x.c < y.c;
  };
  auto by_c = [](const GM &x, const GM &y) { return x.c < y.c; };
  std::stable_sort(gm.begin(), gm.end(), by_a);
  std::stable_sort(gn.begin(), gn.end(), by_b);
  {
    // K: honour the operand whose unit-stride mode is contracted
    bool a_unit_in_k = false, b_unit_in_k = false;
    for (auto &g : gk) {
      if (g.a == 1) a_unit_in_k = true;
      if (g.b == 1) b_unit_in_k = true;
    }
    if (b_unit_in_k && !a_unit_in_k) std::stable_sort(gk.begin(), gk.end(), by_b);
    else std::stable_sort(gk.begin(), gk.end(), by_a);
  }
  std::stable_sort(gb.begin(), gb.end(), by_c);
  merge_group(gm);
  merge_group(gn);
  merge_group(gk);
  merge_group(gb);
  if ((int)gm.size() > MAXM || (int)gn.size() > MAXM || (int)gk.size() > MAXM ||
      (int)gb.size() > MAXM) {
    set_error("too many non-mergeable modes in one group (max %d): permute "
              "the operand first", MAXM);
    return -100;
  }
  for (auto &g : gm) if (g.ext > 0x7fffffffLL) { set_error("mode extent too large"); return -100; }
  for (auto &g : gn) if (g.ext > 0x7fffffffLL) { set_error("mode extent too large"); return -100; }
  for (auto &g : gk) if (g.ext > 0x7fffffffLL) { set_error("mode extent too large"); return -100; }
  for (auto &g : gb) if (g.ext > 0x7fffffffLL) { set_error("mode extent too large"); return -100; }

  ContractParams &p = plan.p;
  memset(&p, 0, sizeof(p));
  p.A = A->ptr; p.B = B->ptr; p.C = C->ptr;
  p.M = p.N = p.K = p.nbatch = 1;
  p.m.n = (int)gm.size(); p.n.n = (int)gn.size();
  p.k.n = (int)gk.size(); p.b.n = (int)gb.size();
  for (int i = 0; i < p.m.n; ++i) { p.m.ext[i] = (int32_t)gm[i].ext; p.m.s0[i] = gm[i].a; p.m.s1[i] = gm[i].c; p.M *= gm[i].ext; }
  for (int i = 0; i < p.n.n; ++i) { p.n.ext[i] = (int32_t)gn[i].ext; p.n.s0[i] = gn[i].b; p.n.s1[i] = gn[i].c; p.N *= gn[i].ext; }
  for (int i = 0; i < p.k.n; ++i) { p.k.ext[i] = (int32_t)gk[i].ext; p.k.s0[i] = gk[i].a; p.k.s1[i] = gk[i].b; p.K *= gk[i].ext; }
  for (int i = 0; i < p.b.n; ++i) { p.b.ext[i] = (int32_t)gb[i].ext; p.b.s0[i] = gb[i].a; p.b.s1[i] = gb[i].b; p.bsC[i] = gb[i].c; p.nbatch *= gb[i].ext; }
  p.conjA = conjA; p.conjB = conjB;
  p.alpha = 1.0; p.beta = 0.0;
  plan.dtype = A->dtype;
  plan.empty_out = zero_out;
  plan.zero_fill = zero_k && !zero_out;
  plan.out_elems = 1;
  for (int i = 0; i < C->rank; ++i) plan.out_elems *= C->shape[i];

  // ---- vectorisation: 16-byte chunks = 2 fp64 (or one complex128) --------
  const int esz = dtype_size(A->dtype);
  const int vlen = 16 / esz;  // elements per 16 bytes (f64: 2, c128: 1)
  auto all_even = [&](const ModeGroup &g, bool second, int skip) {
    for (int i = 0; i < g.n; ++i) {
      if (i == skip) continue;
      int64_t s = second ? g.s1[i] : g.s0[i];
      if (s % vlen) return false;
    }
    return true;
  };
  auto aligned16 = [](const void *q) { return ((uintptr_t)q & 15) == 0; };
  p.vecA = p.vecB = p.vecC = 0;
  if (vlen == 2) {
    bool bevenA = true, bevenB = true, bevenC = true;
    for (int i = 0; i < p.b.n; ++i) {
      if (p.b.s0[i] % 2) bevenA = false;
      if (p.b.s1[i] % 2) bevenB = false;
      if (p.bsC[i] % 2) bevenC = false;
    }
    if (aligned16(p.A) && bevenA) {
      if (p.k.n && p.k.s0[0] == 1 && p.k.ext[0] % 2 == 0 &&
          all_even(p.k, false, 0) && all_even(p.m, false, -1))
        p.vecA = 2;
      else if (p.m.n && p.m.s0[0] == 1 && p.m.ext[0] % 2 == 0 &&
               all_even(p.m, false, 0) && all_even(p.k, false, -1))
        p.vecA = 1;
    }
    if (aligned16(p.B) && bevenB) {
      if (p.k.n && p.k.s1[0] == 1 && p.k.ext[0] % 2 == 0 &&
          all_even(p.k, true, 0) && all_even(p.n, false, -1))
        p.vecB = 2;
      else if (p.n.n && p.n.s0[0] == 1 && p.n.ext[0] % 2 == 0 &&
               all_even(p.n, false, 0) && all_even(p.k, true, -1))
        p.vecB = 1;
    }
    if (aligned16(p.C) && bevenC && p.n.n && p.n.s1[0] == 1 &&
        p.n.ext[0] % 2 == 0 && all_even(p.n, true, 0) &&
        all_even(p.m, true, -1))
      p.vecC = 1;
  }
  // thread walk direction: follow the smaller remaining stride
  auto walk = [&](int vec, const ModeGroup &free_g, const ModeGroup &kg,
                  bool k_second) -> int {
    const int64_t INF = (int64_t)1 << 62;
    auto ks = [&](int i) { return k_second ? kg.s1[i] : kg.s0[i]; };
    int64_t um = free_g.n ? free_g.s0[0] : INF;
    int64_t uk = kg.n ? ks(0) : INF;
    if (vec == 2 && kg.ext[0] == 2) uk = kg.n > 1 ? ks(1) : INF;
    if (vec == 1 && free_g.ext[0] == 2) um = free_g.n > 1 ? free_g.s0[1] : INF;
    if (um == 0) um = INF;  // broadcast dims give no locality
    if (uk == 0) uk = INF;
    return uk <= um ? 1 : 0;
  };
  p.thrA = walk(p.vecA, p.m, p.k, false);
  p.thrB = walk(p.vecB, p.n, p.k, true);

  // ---- tile configuration -----------------------------------------------
  int cfg;
  // complex runs as a real GEMM with doubled N and K (see contract_dmma.cu)
  const bool cplx = dtype_is_complex(A->dtype);
  const int64_t M = p.M, N = cplx ? 2 * p.N : p.N, Kh = cplx ? 2 * p.K : p.K;
  // cost model: time ~ waves * (padded tile work) / (per-CTA rate), plus the
  // split-K partial write + reduce traffic.  occ = resident CTAs per SM,
  // eff = assumed fraction of the DMMA peak at full occupancy.
  static const int kOcc[kNumTileCfgs] = {1, 2, 2, 2, 5};
  static const double kEff[kNumTileCfgs] = {0.73, 0.60, 0.50, 0.50, 0.30};
  const int nsm = sm_count();
  const double kFmaPerUs = nsm * kDmmaFmaPerSmUs;  // chip FMA rate / us
  const double kBytesPerUs = 3.35e6;  // HBM3 bandwidth of the H100 SXM data sheet
  double best_t = 1e300;
  int best_cfg = 1, best_split = 1;
  int64_t best_kper = 0;
  for (int c = 0; c < kNumTileCfgs; ++c) {
    const TileCfg &tc = kTileCfgs[c];
    const int64_t tiles = cdiv(M, tc.bm) * cdiv(N, tc.bn) * p.nbatch;
    const int64_t kblocks = std::max<int64_t>(cdiv(Kh, tc.bk), 1);
    const int64_t slots = (int64_t)nsm * kOcc[c];
    for (int64_t sk = 1; sk <= max_splitk; sk *= 2) {
      if (sk > 1 && (kblocks / sk < 4)) break;
      const int64_t kb_per = cdiv(kblocks, sk);
      const int64_t nsplit = cdiv(kblocks, kb_per);
      const int64_t units = tiles * nsplit;
      const double waves = (double)cdiv(units, slots);
      // CTAs only share an SM when there are enough of them; a lone CTA
      // is capped by how many of the 4 sub-partitions its warps cover
      const double share = (double)std::min<int64_t>(kOcc[c], cdiv(units, nsm));
      const double warpcap = std::min(1.0, (tc.threads / 32) / 4.0) * 0.8;
      const double cta_rate =
          kDmmaFmaPerSmUs * std::min(kEff[c] / share, warpcap);
      double t = waves * ((double)tc.bm * tc.bn * kb_per * tc.bk) / cta_rate;
      t += 3.0;  // launch latency
      if (nsplit > 1)
        t += 3.0 + (double)(nsplit + 1) * p.nbatch * M * N * 8.0 / kBytesPerUs;
      if (t < best_t) {
        best_t = t; best_cfg = c; best_split = (int)nsplit;
        best_kper = kb_per * tc.bk;
      }
    }
  }
  cfg = best_cfg;
  plan.cfg = cfg;
  const TileCfg &tc = kTileCfgs[cfg];
  p.tiles_m = (int32_t)cdiv(M, tc.bm);
  p.tiles_n = (int32_t)cdiv(N, tc.bn);
  p.splitk = best_split;
  p.k_per_split = best_kper;
  if (cfg == 0 && !cplx) {
    p.feedA = affine_feed(p.m, p.k, false, p.vecA, tc.bm, tc.bk, p.rstepA, p.kstepA);
    p.feedB = affine_feed(p.n, p.k, true, p.vecB, tc.bn, tc.bk, p.rstepB, p.kstepB);
  }
  // stream-K (large tile only): when the tile count leaves SMs idle in the
  // last wave, cut the (tile, k-block) space into one equal range per SM
  plan.streamk = 0;
  plan.flags_clean = false;
  {
    // one persistent CTA per SM: owners spin on their peers' flags, so every
    // CTA of the grid must be resident at once
    const int G = nsm;
    const int64_t tiles = (int64_t)p.tiles_m * p.tiles_n;
    const int64_t kblocks = cdiv(Kh, tc.bk);
    const double eff = (double)(tiles * p.splitk) / (double)(cdiv(tiles * p.splitk, G) * G);
    if (cfg == 0 && p.nbatch == 1 && tiles >= 32 && tiles * kblocks >= 8LL * G &&
        (eff < 0.93 || p.splitk > 1)) {
      plan.streamk = G;
      p.splitk = 1;
      p.k_per_split = kblocks * tc.bk;
      // fix-up (wait + collect the peers' partial tiles) + epilogue of a
      // shared tile cost its owner about head_us = this many k-blocks; it gets
      // that much less of the main loop.  9 us is an estimate that has not
      // been measured on the H100
      constexpr double head_us = 9.0;
      const double kb_us = (double)tc.bm * tc.bn * tc.bk / (0.9 * kDmmaFmaPerSmUs);
      int64_t H = (int64_t)(head_us / kb_us + 0.5);
      const int64_t share = tiles * (kblocks + H) / G;
      if (H >= share / 2) H = 0;
      p.sk_head = (int32_t)H;
    }
  }
  return 0;
}

// layout of the operand tiles in shared memory ([row][k] = "k-major"); for
// real operands the large-tile kernels are specialised on it so that every
// fragment address is base + immediate
inline int a_kmajor(const ContractParams &p) {
  return (p.vecA == 2) || (p.vecA == 0 && p.thrA == 1);
}
inline int b_kmajor(const ContractParams &p) {
  return (p.vecB == 2) || (p.vecB == 0 && p.thrB == 1);
}
// the large real tile keeps A in k-pair layout ([k/2][row][2], contract_dmma.cu)
// when both operands take the affine feed and A's 16-byte pairs of k are
// gathered by threads that walk rows: each 32-byte sector a warp reads then
// lands in 32 contiguous bytes of the tile rather than in two rows
inline bool a_kpair(const ContractParams &p) {
  return p.feedA && p.feedB && p.vecA == 2 && p.thrA == 0;
}

// Which kernel a contraction runs.  select_route (api.cu) decides the engine;
// dmma_route fills in the DMMA details.  The launchers read the same fields,
// so qb_contract_pair_route reports exactly what qb_contract_pair runs.
enum RouteKind {
  ROUTE_EMPTY = 0,         // output has no elements: nothing runs
  ROUTE_ZERO_FILL = 1,     // contracted extent 0: C = 0 (beta = 0)
  ROUTE_WIDEN = 2,         // single precision below the int8 engine's minimum
  ROUTE_INT8 = 3,          // int8 error-free-split engine (ozaki_tc.cu)
  ROUTE_STREAM = 4,        // streaming engine (contract_stream.cu)
  ROUTE_DMMA = 5,          // DMMA tile kernel, classic grid (+ split-K reduce)
  ROUTE_DMMA_STREAMK = 6,  // DMMA large tile, persistent stream-K grid
};
struct Route {
  int kind;
  int cfg;        // DMMA tile configuration, -1 otherwise
  int splitk;     // split-K factor (1: none)
  int streamk;    // stream-K grid (CTAs), 0 otherwise
  int sk_head;    // stream-K cost of a tile's fix-up, in k-blocks
  int bk;         // DMMA k-block depth
  int layout;     // cfg 0, real: a_kmajor * 2 + b_kmajor; -1 otherwise
  int launches;   // kernels launched (beta = 0)
  int stream_k;   // streaming engine: compiled (KMAX, NMAX) variant, 0 otherwise
  int stream_n;
};

// DMMA part of a route.  A stream-K grid needs the workspace scratch that the
// planner sized for it (internal GEMMs without scratch run classic launches).
inline Route dmma_route(const PairPlan &plan, bool have_scratch) {
  Route r{ROUTE_DMMA, plan.cfg, plan.p.splitk, 0, 0, kTileCfgs[plan.cfg].bk, -1, 1};
  const bool cplx = dtype_is_complex(plan.dtype);
  if (plan.streamk > 0 && have_scratch) {
    r.kind = ROUTE_DMMA_STREAMK;
    r.splitk = 1;
    r.streamk = plan.streamk;
    r.sk_head = plan.p.sk_head;
  } else if (r.splitk > 1) {
    r.launches = 2;  // + splitk_reduce_f64_kernel
  }
  if (plan.cfg == 0 && !cplx)
    r.layout = a_kmajor(plan.p) * 2 + b_kmajor(plan.p);
  return r;
}

// scratch for partial sums (stream-K parked tiles / split-K partial outputs)
inline int64_t plan_scratch_bytes(const PairPlan &plan) {
  if (plan.streamk > 0)
    return (int64_t)plan.streamk * (128 * 128 * 8);
  if (plan.p.splitk <= 1) return 0;
  return (int64_t)plan.p.splitk * plan.p.nbatch * plan.p.M * plan.p.N * 8 *
         (dtype_is_complex(plan.dtype) ? 2 : 1);
}
// caller-visible workspace: a 1 KiB header (stream-K flag words, kept zero
// between launches) followed by the scratch
constexpr int64_t kWsHeaderBytes = 1024;
inline int64_t plan_workspace_bytes(const PairPlan &plan) {
  const int64_t s = plan_scratch_bytes(plan);
  return s > 0 ? s + kWsHeaderBytes : 0;
}

#ifdef __CUDACC__
// mixed-radix decode of a linear group index into two element offsets
__device__ __forceinline__ void decode2(int64_t idx, const ModeGroup &g,
                                        int64_t &o0, int64_t &o1) {
  int64_t a = 0, b = 0;
  if (idx <= 0xffffffffLL) {
    uint32_t r = (uint32_t)idx;
#pragma unroll 1
    for (int i = 0; i < g.n; ++i) {
      uint32_t e = (uint32_t)g.ext[i];
      uint32_t q = r / e;
      uint32_t d = r - q * e;
      a += (int64_t)d * g.s0[i];
      b += (int64_t)d * g.s1[i];
      r = q;
    }
  } else {
#pragma unroll 1
    for (int i = 0; i < g.n; ++i) {
      int64_t e = g.ext[i];
      int64_t q = idx / e;
      int64_t d = idx - q * e;
      a += d * g.s0[i];
      b += d * g.s1[i];
      idx = q;
    }
  }
  o0 = a;
  o1 = b;
}

#endif  // __CUDACC__

}  // namespace qb
