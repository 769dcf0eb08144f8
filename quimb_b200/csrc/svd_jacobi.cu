// qb_svd / qb_svd_trunc <- svd_truncated (quimb/tensor/decomp.py:829-1118):
// thin SVD by one-sided block Jacobi on the R factor of a QR preconditioner,
// with the reference's truncation rule (:901-937), renormalisation (:940-965),
// trimming (:968-1029) and absorption of the singular values (:693-721) fused
// into the epilogue, so that a truncated split is ONE library call that
// writes exactly the kept factors.
//
// Round structure:
//
//   * a sweep is cut into INDEPENDENT sub-tournaments (2 or 4 groups of column
//     blocks: round robin inside every group, then bipartite rounds between
//     groups, themselves split into independent halves), each running on its
//     own CUDA stream.  Launches of different streams are co-resident on an SM
//     (2-4 CTAs per SM), so the latency-bound 32 x 32 eigen-solve of one pair
//     overlaps the DMMA-bound Gram / apply phases of others -- the phases of
//     one launch all coincide, which is what left the tensor pipe 33 % busy;
//   * a column-block pair is owned by a CLUSTER of 2 CTAs (rows dealt in
//     64-row chunks, 4 cp.async stages);
//   * the partial Gram is computed with each warp owning one 16 x 8 output
//     tile over all rows of the chunk: no cross-warp reduction, only the
//     fixed-order cluster reduction through distributed shared memory;
//   * rotations from two rsqrt (cos 2t = |a| r, u = (1 + cos 2t) / 2,
//     c = u rsqrt(u), s = sin 2t rsqrt(u) / 2) instead of sqrt + divide +
//     rsqrt: half the dependent latency of a Jacobi step, same rounding-level
//     orthogonality;
#include <cooperative_groups.h>
#include <math.h>
#include <stdlib.h>

#include <algorithm>
#include <vector>

#include "internal.h"

namespace qb {

namespace jac2 {

constexpr int JB = 16;          // columns per block
constexpr int JP = 2 * JB;      // columns per pair
constexpr int JPITCH = JP + 4;  // smem pitch (== 4 mod 16 doubles)

struct Params {
  double *W;       // rows_w x ld  working matrix (columns get orthogonalised)
  double *V;       // rows_v x ld  accumulated right rotations
  int64_t ld;
  int rows_w, rows_v;
  const int2 *pairs;  // column-block pairs of this launch (one per cluster)
  double tol;
  const double *negl;  // Gram diagonals <= *negl: numerically zero columns
  int *flag;                     // set to 1 when any pair still needed rotating
  unsigned long long *offmax;    // max scaled off-diagonal met (double bits)
  int inner_max;
  unsigned long long *trace;
  int trace_slot;
};

__device__ __forceinline__ unsigned long long now_ns() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}
#define J2_TRACE(ph)                                                       \
  do {                                                                     \
    if (P.trace && blockIdx.x == 0 && threadIdx.x == 0)                    \
      P.trace[(size_t)P.trace_slot * 8 + (ph)] = now_ns();              \
  } while (0)

// Which pairs rotate, and which flag a sweep as unconverged.  Both tests are
// relative to the column norms, so a pair is flagged only if it is rotated:
//  * a column whose squared norm is at most negl (eps |W|_F, squared) is
//    numerically zero (rank deficiency).  Rotating it against others only
//    re-creates rounding noise at the scale of the large column, which never
//    converges; it takes no part, and its singular value is returned as 0;
//  * otherwise the measure is |g_pq| / sqrt(g_pp g_qq), formed without
//    underflow when g_pp g_qq underflows (columns far below the largest);
//  * a pair rotates when |g_pq| > 1e-300 or its measure exceeds 2^-60 (far
//    below the convergence tolerance), so small columns that are far from
//    orthogonal still rotate.
constexpr double kJacSkip = 1e-300;
constexpr double kJacRelSkip = 0x1p-60;

__device__ __forceinline__ double pair_off(double v, double gpp, double gqq, double negl) {
  v = fabs(v);
  if (!(v > 0.0) || gpp <= negl || gqq <= negl) return 0.0;
  const double d = gpp * gqq;
  if (d > 0.0) return v * rsqrt(d);
  return v / (sqrt(gpp) * sqrt(gqq));
}

__device__ __forceinline__ bool pair_rotates(double apq, double app, double aqq, double negl) {
  if (app <= negl || aqq <= negl) return false;
  const double v = fabs(apq);
  return v > kJacSkip || (v > 0.0 && v > kJacRelSkip * (sqrt(app) * sqrt(aqq)));
}

__device__ __forceinline__ void rr_pair(int k, int round, int nblk, int &p, int &q) {
  const int m = nblk - 1;
  int a, b;
  if (k == 0) { a = m; b = round; }
  else { a = (round + k) % m; b = (round - k + m) % m; }
  p = min(a, b); q = max(a, b);
}

template <int CH>
__device__ __forceinline__ void load_chunk(double (*Xs)[JPITCH], const double *M,
                                           int64_t ld, int rows, int row0,
                                           int cp, int cq, int tid) {
#pragma unroll
  for (int i = 0; i < CH / 16; ++i) {
    const int idx = tid + 256 * i;       // CH * 16 double2 per chunk
    const int r = idx >> 4, c2 = (idx & 15) * 2;
    const int gc = (c2 < JB) ? (cp + c2) : (cq + c2 - JB);
    const int gr = row0 + r;
    const bool ok = gr < rows;
    const double *src = ok ? (M + (int64_t)gr * ld + gc) : M;
    cp_async16(smem_u32(&Xs[r][c2]), src, ok ? 16 : 0);
  }
}

// Position layout of the 32 x 32 eigen-solve (Brent-Luk style): the 32
// column "players" of a pair sit in 16 A-slots and 16 B-slots; slot pair k is
// rotated at every step and the players then move one slot round the circle
// (A_0 fixed), so thread (k1, k2) always owns the 2 x 2 block (rows A_k1, B_k1)
// x (columns A_k2, B_k2).  GA[rowpos][k] = G[row][A_k], GB[rowpos][k] =
// G[row][B_k] with rowpos = k (A-slots), 16 + k (B-slots): every access of a
// half-warp is to 16 consecutive doubles, the diagonal reads GA[k][k] hit
// distinct banks with the even pitch 18, and the 15-double gap between the two
// arrays keeps the "moved" writes (one lane of a half-warp lands in the other
// array) off the banks of the rest.
constexpr int GPITCH = 18;
struct PosG {
  double A[JP][GPITCH];
  double pad[15];
  double B[JP][GPITCH];
};

template <int CH, int STG>
struct Smem {
  double Xs[STG][CH][JPITCH];
  double Gs[JP][JP + 1];       // player-order scratch: reduced Gram, sort
  PosG Gp[2];                  // position-order Gram, ping-pong
  double Gpart[JP][JP];
  double Jm[JP][JPITCH];
  double redmax[8];
  double dg[JP];
  int rank_s[JP];
  int ctl[4];                  // [0] = 1: rotate (written by cluster rank 0)
};

// player sitting in slot (isB, k) at the start of a sweep (circle method, step 0)
__device__ __forceinline__ int slot_player(int isB, int k) {
  if (!isB) return k == 0 ? JP - 1 : k;
  return k == 0 ? 0 : JP - 1 - k;
}
// slot a player moves to after a step: A_0 stays, A_1 -> B_0, A_k -> A_{k-1},
// B_k -> B_{k+1}, B_15 -> A_15
__device__ __forceinline__ void slot_next(int isB, int k, int &nB, int &nk) {
  if (!isB) {
    if (k == 0) { nB = 0; nk = 0; }
    else if (k == 1) { nB = 1; nk = 0; }
    else { nB = 0; nk = k - 1; }
  } else {
    if (k == JB - 1) { nB = 0; nk = JB - 1; }
    else { nB = 1; nk = k + 1; }
  }
}

// One round of one sub-tournament: cluster c of the launch owns pair
// P.pairs[c]; see the file header.  CH rows per streamed chunk, STG cp.async
// stages; the cluster size comes from the launch attribute.
template <int CH, int STG, int MINB>
__global__ void __launch_bounds__(256, MINB) jacobi_round_kernel(const Params P) {
  namespace cg = cooperative_groups;
  cg::cluster_group cluster = cg::this_cluster();
  const int rank = (int)cluster.block_rank();
  const int CS = (int)cluster.num_blocks();
  extern __shared__ __align__(16) unsigned char jac2_smem[];
  Smem<CH, STG> &S = *reinterpret_cast<Smem<CH, STG> *>(jac2_smem);

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int g = lane >> 2, t = lane & 3;
  const int2 pr = P.pairs[blockIdx.x / CS];
  const int cp = pr.x * JB, cq = pr.y * JB;

  J2_TRACE(0);
  // ---------------- phase 1: partial Gram over this CTA's row chunks --------
  // warp (ta, tj) owns the 16 x 8 tile rows ta*16.., cols tj*8.. of the Gram
  {
    const int ta = warp >> 2, tj = warp & 3;
    double acc[4] = {0.0, 0.0, 0.0, 0.0};
    const int nch_all = (P.rows_w + CH - 1) / CH;
    const int nmine = (nch_all - rank + CS - 1) / CS;  // chunks rank, rank+CS, ...
    auto issue = [&](int i) {
      if (i < nmine)
        load_chunk<CH>(S.Xs[i % STG], P.W, P.ld, P.rows_w, (rank + i * CS) * CH, cp, cq, tid);
      cp_async_commit();
    };
    for (int s = 0; s < STG - 1; ++s) issue(s);
    for (int i = 0; i < nmine; ++i) {
      cp_async_wait<STG - 2>();
      __syncthreads();
      issue(i + STG - 1);
      const double(*X)[JPITCH] = S.Xs[i % STG];
#pragma unroll
      for (int kb = 0; kb < CH; kb += 8) {
        double af[4], bf[2];
        af[0] = X[kb + t][ta * 16 + g];
        af[1] = X[kb + t][ta * 16 + g + 8];
        af[2] = X[kb + t + 4][ta * 16 + g];
        af[3] = X[kb + t + 4][ta * 16 + g + 8];
        bf[0] = X[kb + t][tj * 8 + g];
        bf[1] = X[kb + t + 4][tj * 8 + g];
        dmma_16x8x8(acc, af, bf);
      }
    }
    cp_async_wait<0>();
#pragma unroll
    for (int h = 0; h < 2; ++h)
      *reinterpret_cast<double2 *>(&S.Gpart[ta * 16 + g + h * 8][tj * 8 + 2 * t]) =
          make_double2(acc[2 * h], acc[2 * h + 1]);
  }
  J2_TRACE(1);
  cluster.sync();
  // ---------------- phase 2 (cluster rank 0 only): J^T G J = diag -----------
  // The other CTAs of the cluster wait in the hardware cluster barrier (their
  // warps are descheduled), so co-resident CTAs of other streams get the SM.
  if (rank == 0) {
    double(*G)[JP + 1] = S.Gs;
    const double negl = *P.negl;
    // full Gram = sum over the cluster in rank order, then symmetrised
    for (int idx = tid; idx < JP * JP; idx += 256) {
      double sum = 0.0;
      for (int q = 0; q < CS; ++q) sum += cluster.map_shared_rank(&S.Gpart[0][0], q)[idx];
      S.Jm[idx / JP][idx % JP] = sum;       // Jm as scratch for the raw sum
    }
    __syncthreads();
    for (int idx = tid; idx < JP * JP; idx += 256) {
      const int r = idx / JP, c = idx % JP;
      G[r][c] = 0.5 * (S.Jm[r][c] + S.Jm[c][r]);
    }
    __syncthreads();
    double mx = 0.0;
    for (int idx = tid; idx < JP * JP; idx += 256) {
      const int r = idx / JP, c = idx % JP;
      if (r < c) mx = fmax(mx, pair_off(G[r][c], G[r][r], G[c][c], negl));
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) mx = fmax(mx, __shfl_xor_sync(0xffffffffu, mx, o));
    if (lane == 0) S.redmax[warp] = mx;
    __syncthreads();
    double off0 = 0.0;
    for (int w = 0; w < 8; ++w) off0 = fmax(off0, S.redmax[w]);
    J2_TRACE(2);
    const bool rotate = off0 > P.tol;
    if (tid == 0) {
      S.ctl[0] = rotate ? 1 : 0;
      atomicMax(P.offmax, (unsigned long long)__double_as_longlong(off0));
      if (rotate) atomicOr(P.flag, 1);
    }
    if (rotate) {
      // thread (k1, k2): rows (A_k1, B_k1) x columns (A_k2, B_k2)
      const int k1 = tid >> 4, k2 = tid & 15;
      const int rA = slot_player(0, k1), rB = slot_player(1, k1);
      const int cA = slot_player(0, k2), cB = slot_player(1, k2);
      double gAA = G[rA][cA], gAB = G[rA][cB], gBA = G[rB][cA], gBB = G[rB][cB];
      // J = I in player space; this thread's two rows r = k1, k1 + 16
      double jA[2], jB[2];
#pragma unroll
      for (int it = 0; it < 2; ++it) {
        const int r = k1 + 16 * it;
        jA[it] = (r == cA) ? 1.0 : 0.0;
        jB[it] = (r == cB) ? 1.0 : 0.0;
      }
      // where this thread's four entries go after a step (fixed for all steps)
      int nrA_B, nrA_k, nrB_B, nrB_k, ncA_B, ncA_k, ncB_B, ncB_k;
      slot_next(0, k1, nrA_B, nrA_k); slot_next(1, k1, nrB_B, nrB_k);
      slot_next(0, k2, ncA_B, ncA_k); slot_next(1, k2, ncB_B, ncB_k);
      const int rowA = nrA_k + 16 * nrA_B, rowB = nrB_k + 16 * nrB_B;
      // seed the position buffers so that the first step reads its diagonal
      int cur = 0;
      S.Gp[0].A[k1][k2] = gAA; S.Gp[0].B[k1][k2] = gAB;
      S.Gp[0].A[16 + k1][k2] = gBA; S.Gp[0].B[16 + k1][k2] = gBB;
      __syncthreads();
      for (int sweep = 0; sweep < P.inner_max; ++sweep) {
        if (sweep > 0) {
          // scaled off-diagonal mass of the current iterate (position layout)
          if (k1 == k2) { S.dg[k1] = gAA; S.dg[16 + k1] = gBB; }
          __syncthreads();
          const double dA1 = S.dg[k1], dB1 = S.dg[16 + k1], dA2 = S.dg[k2], dB2 = S.dg[16 + k2];
          double m = fmax(pair_off(gAB, dA1, dB2, negl), pair_off(gBA, dB1, dA2, negl));
          if (k1 != k2)
            m = fmax(m, fmax(pair_off(gAA, dA1, dA2, negl), pair_off(gBB, dB1, dB2, negl)));
#pragma unroll
          for (int o = 16; o > 0; o >>= 1) m = fmax(m, __shfl_xor_sync(0xffffffffu, m, o));
          if (lane == 0) S.redmax[warp] = m;
          __syncthreads();
          double off = 0.0;
          for (int w = 0; w < 8; ++w) off = fmax(off, S.redmax[w]);
          __syncthreads();
          if (off <= 1e-15 || off <= 1e-4 * off0) break;
        }
        for (int step = 0; step < JP - 1; ++step) {
          const PosG &Gc = S.Gp[cur];
          PosG &Gw = S.Gp[cur ^ 1];
          // the 16 rotations of the step, computed by lanes 0-15 of every warp
          // from the diagonal blocks (same instruction sequence everywhere)
          double c = 1.0, sn = 0.0;
          if (lane < 16) {
            const double app = Gc.A[lane][lane], aqq = Gc.B[16 + lane][lane];
            const double apq = Gc.B[lane][lane];
            if (pair_rotates(apq, app, aqq, negl)) {
              // tan 2t = b / a with a = aqq - app, b = 2 apq, |t| <= pi / 4
              const double a = __dsub_rn(aqq, app), b = __dmul_rn(2.0, apq);
              const double n2 = __fma_rn(a, a, __dmul_rn(b, b));
              if (n2 > 1e-280 && n2 < 1e280) {
                const double r = rsqrt(n2);
                const double c2t = __dmul_rn(fabs(a), r);                   // cos 2t >= 0
                const bool neg = (a < 0.0) != (b < 0.0);                    // sign of a b
                const double s2t = __dmul_rn(neg ? -fabs(b) : fabs(b), r);  // sin 2t
                const double u = __fma_rn(0.5, c2t, 0.5);                   // cos^2 t
                const double ru = rsqrt(u);
                c = __dmul_rn(u, ru);
                sn = __dmul_rn(__dmul_rn(0.5, s2t), ru);
              } else {
                // badly scaled pair: the textbook formula on the ratio
                const double tt = copysign(fabs(b), __dmul_rn(a, b)) / (fabs(a) + hypot(a, b));
                c = rsqrt(__fma_rn(tt, tt, 1.0));
                sn = __dmul_rn(c, tt);
              }
            }
          }
          const double c2 = __shfl_sync(0xffffffffu, c, k2), s2 = __shfl_sync(0xffffffffu, sn, k2);
          const double c1 = __shfl_sync(0xffffffffu, c, k1), s1 = __shfl_sync(0xffffffffu, sn, k1);
          // columns (A_k2, B_k2) then rows (A_k1, B_k1)
          const double a0 = c2 * gAA - s2 * gAB, a1 = s2 * gAA + c2 * gAB;
          const double b0 = c2 * gBA - s2 * gBB, b1 = s2 * gBA + c2 * gBB;
          double n00 = c1 * a0 - s1 * b0, n01 = c1 * a1 - s1 * b1;
          double n10 = s1 * a0 + c1 * b0, n11 = s1 * a1 + c1 * b1;
          if (k1 == k2) { n01 = 0.0; n10 = 0.0; }  // the annihilated pair
          // move: every entry to the slots its row / column players take next
          (ncA_B ? Gw.B : Gw.A)[rowA][ncA_k] = n00;
          (ncB_B ? Gw.B : Gw.A)[rowA][ncB_k] = n01;
          (ncA_B ? Gw.B : Gw.A)[rowB][ncA_k] = n10;
          (ncB_B ? Gw.B : Gw.A)[rowB][ncB_k] = n11;
          // J <- J R on columns (A_k2, B_k2), then the columns move with their
          // players: shuffles inside the 16-lane group
#pragma unroll
          for (int it = 0; it < 2; ++it) {
            const double ja = c2 * jA[it] - s2 * jB[it];
            const double jb = s2 * jA[it] + c2 * jB[it];
            const double ja_dn = __shfl_down_sync(0xffffffffu, ja, 1, 16);  // A[k2 + 1]
            const double jb_up = __shfl_up_sync(0xffffffffu, jb, 1, 16);    // B[k2 - 1]
            jA[it] = (k2 == 0) ? ja : (k2 == JB - 1 ? jb : ja_dn);
            jB[it] = (k2 == 0) ? ja_dn : jb_up;
          }
          __syncthreads();
          cur ^= 1;
          const PosG &Gr = S.Gp[cur];
          gAA = Gr.A[k1][k2]; gAB = Gr.B[k1][k2];
          gBA = Gr.A[16 + k1][k2]; gBB = Gr.B[16 + k1][k2];
        }
        // 31 steps = one full turn of the circle: the players are back in
        // their starting slots
      }
      J2_TRACE(3);
      // J (player order) and the new column norms; sort: larger norms first
      __syncthreads();
#pragma unroll
      for (int it = 0; it < 2; ++it) {
        G[k1 + 16 * it][cA] = jA[it];
        G[k1 + 16 * it][cB] = jB[it];
      }
      if (k1 == k2) { S.dg[cA] = gAA; S.dg[cB] = gBB; }
      __syncthreads();
      if (tid < JP) {
        const double d = S.dg[tid];
        int rk = 0;
        for (int j = 0; j < JP; ++j) {
          const double dj = S.dg[j];
          rk += (dj > d) || (dj == d && j < tid);
        }
        S.rank_s[tid] = rk;
      }
      __syncthreads();
      for (int idx = tid; idx < JP * JP; idx += 256) {
        const int r = idx / JP, cc = idx % JP;
        S.Jm[r][S.rank_s[cc]] = G[r][cc];
      }
    }
    __syncthreads();
  }
  cluster.sync();   // J (or the decision not to rotate) is published by rank 0
  const int *ctl0 = cluster.map_shared_rank(&S.ctl[0], 0);
  if (ctl0[0] == 0) {
    cluster.sync();  // rank 0 stays until everybody has read its flag
    return;
  }

  J2_TRACE(4);
  // ---------------- phase 3: apply J to this CTA's rows of W and V ----------
  {
    constexpr int RT = CH / 16;       // 16-row tiles per chunk
    constexpr int CG = 8 / RT;        // column groups (warps per row tile)
    constexpr int NT = 4 / CG;        // 8-column tiles per warp
    const int nchw = (P.rows_w + CH - 1) / CH, nchv = (P.rows_v + CH - 1) / CH;
    const int ntot = nchw + nchv;
    const int nmine = (ntot - rank + CS - 1) / CS;
    auto chunk_src = [&](int i, double *&M, int &rows, int &row0) {
      const int ch = rank + i * CS;
      if (ch < nchw) { M = P.W; rows = P.rows_w; row0 = ch * CH; }
      else { M = P.V; rows = P.rows_v; row0 = (ch - nchw) * CH; }
    };
    auto issue = [&](int i) {
      if (i < nmine) {
        double *M; int rows, row0;
        chunk_src(i, M, rows, row0);
        load_chunk<CH>(S.Xs[i % STG], M, P.ld, rows, row0, cp, cq, tid);
      }
      cp_async_commit();
    };
    for (int s = 0; s < STG - 1; ++s) issue(s);
    const int mt = warp % RT, nh = warp / RT;
    // this warp's slice of J (read from rank 0's shared memory through the
    // cluster window) stays in registers for the whole phase
    const double *Jr = cluster.map_shared_rank(&S.Jm[0][0], 0);
    double bj[JP / 8][NT][2];
#pragma unroll
    for (int kk = 0; kk < JP / 8; ++kk)
#pragma unroll
      for (int j = 0; j < NT; ++j) {
        bj[kk][j][0] = Jr[(kk * 8 + t) * JPITCH + nh * (8 * NT) + j * 8 + g];
        bj[kk][j][1] = Jr[(kk * 8 + t + 4) * JPITCH + nh * (8 * NT) + j * 8 + g];
      }
    for (int i = 0; i < nmine; ++i) {
      cp_async_wait<STG - 2>();
      __syncthreads();
      issue(i + STG - 1);
      double *M; int rows, row0;
      chunk_src(i, M, rows, row0);
      const double(*X)[JPITCH] = S.Xs[i % STG];
      double c2[NT][4];
#pragma unroll
      for (int j = 0; j < NT; ++j)
#pragma unroll
        for (int v = 0; v < 4; ++v) c2[j][v] = 0.0;
#pragma unroll
      for (int kk = 0; kk < JP / 8; ++kk) {
        double af[4];
        af[0] = X[mt * 16 + g][kk * 8 + t];
        af[1] = X[mt * 16 + g + 8][kk * 8 + t];
        af[2] = X[mt * 16 + g][kk * 8 + t + 4];
        af[3] = X[mt * 16 + g + 8][kk * 8 + t + 4];
#pragma unroll
        for (int j = 0; j < NT; ++j) dmma_16x8x8(c2[j], af, bj[kk][j]);
      }
#pragma unroll
      for (int j = 0; j < NT; ++j)
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int r = row0 + mt * 16 + g + h * 8;
          const int c = nh * (8 * NT) + j * 8 + 2 * t;  // column within the pair
          if (r < rows) {
            const int gc = (c < JB) ? (cp + c) : (cq + c - JB);
            *reinterpret_cast<double2 *>(M + (int64_t)r * P.ld + gc) =
                make_double2(c2[j][2 * h], c2[j][2 * h + 1]);
          }
        }
    }
    cp_async_wait<0>();
  }
  J2_TRACE(5);
  cluster.sync();  // nobody exits while peers may read its shared memory
  J2_TRACE(6);
}

// ---------------------------------------------------------------- schedule ---
// A sweep as a list of phases; inside a phase `ngroups` independent launch
// sequences (one per stream), each a list of rounds, each round a list of
// column-block pairs (disjoint blocks).
struct Phase {
  // rounds[g][r] = (offset into the pair array, number of pairs)
  std::vector<std::vector<std::pair<int, int>>> rounds;
};

static void rr_rounds(const std::vector<int> &blk, std::vector<std::vector<int2>> &out) {
  // circle-method round robin over the blocks in `blk` (odd count: one bye)
  std::vector<int> b = blk;
  if (b.size() % 2) b.push_back(-1);
  const int nb = (int)b.size(), m = nb - 1;
  for (int round = 0; round < m; ++round) {
    std::vector<int2> prs;
    for (int k = 0; k < nb / 2; ++k) {
      int x, y;
      if (k == 0) { x = m; y = round; }
      else { x = (round + k) % m; y = (round - k + m) % m; }
      int p = b[x], q = b[y];
      if (p < 0 || q < 0) continue;
      prs.push_back(make_int2(std::min(p, q), std::max(p, q)));
    }
    if (!prs.empty()) out.push_back(prs);
  }
}

static void bip_rounds(const std::vector<int> &A, const std::vector<int> &B,
                       std::vector<std::vector<int2>> &out) {
  // all pairs A x B, |A| <= |B|: round r pairs A[i] with B[(i + r) % |B|]
  const std::vector<int> &a = A.size() <= B.size() ? A : B;
  const std::vector<int> &b = A.size() <= B.size() ? B : A;
  const int nb = (int)b.size();
  for (int r = 0; r < nb; ++r) {
    std::vector<int2> prs;
    for (int i = 0; i < (int)a.size(); ++i) {
      const int p = a[i], q = b[(i + r) % nb];
      prs.push_back(make_int2(std::min(p, q), std::max(p, q)));
    }
    if (!prs.empty()) out.push_back(prs);
  }
}

struct Schedule {
  std::vector<int2> pairs;                 // flat
  std::vector<Phase> phases;
  int ngroups = 1;
};

static std::vector<int> slice(const std::vector<int> &v, int lo, int hi) {
  return std::vector<int>(v.begin() + lo, v.begin() + hi);
}

static void build_schedule(int nblk, int ngroups, Schedule &S) {
  S.pairs.clear(); S.phases.clear(); S.ngroups = ngroups;
  std::vector<int> all(nblk);
  for (int i = 0; i < nblk; ++i) all[i] = i;
  auto add_phase = [&](const std::vector<std::vector<std::vector<int2>>> &groups) {
    Phase ph;
    for (const auto &gr : groups) {
      std::vector<std::pair<int, int>> rr;
      for (const auto &round : gr) {
        rr.emplace_back((int)S.pairs.size(), (int)round.size());
        S.pairs.insert(S.pairs.end(), round.begin(), round.end());
      }
      ph.rounds.push_back(rr);
    }
    S.phases.push_back(ph);
  };
  if (ngroups <= 1 || nblk < 4 * ngroups) {
    S.ngroups = 1;
    std::vector<std::vector<int2>> r;
    rr_rounds(all, r);
    add_phase({r});
    return;
  }
  // the blocks in `ngroups` contiguous sets, each set in two halves
  const int G = ngroups;
  std::vector<std::vector<int>> set(G);
  for (int s = 0; s < G; ++s) set[s] = slice(all, nblk * s / G, nblk * (s + 1) / G);
  auto halves = [](const std::vector<int> &v, std::vector<int> &a, std::vector<int> &b) {
    const int h = (int)v.size() / 2;
    a = slice(v, 0, h); b = slice(v, h, (int)v.size());
  };
  // phase A: round robin inside every set
  {
    std::vector<std::vector<std::vector<int2>>> groups(G);
    for (int s = 0; s < G; ++s) rr_rounds(set[s], groups[s]);
    add_phase(groups);
  }
  // phases B..: the sets meet pairwise (round robin over the sets); a meeting
  // of two sets is all pairs A x B, run as two independent halves at a time:
  // (Aa x Ba, Ab x Bb) then (Aa x Bb, Ab x Ba) -> G groups per phase again
  std::vector<int> sid(G);
  for (int s = 0; s < G; ++s) sid[s] = s;
  std::vector<std::vector<int2>> meet;
  rr_rounds(sid, meet);
  for (const auto &mr : meet) {
    for (int cross = 0; cross < 2; ++cross) {
      std::vector<std::vector<std::vector<int2>>> groups;
      for (const int2 &ab : mr) {
        std::vector<int> Aa, Ab, Ba, Bb;
        halves(set[ab.x], Aa, Ab);
        halves(set[ab.y], Ba, Bb);
        std::vector<std::vector<int2>> g0, g1;
        if (cross == 0) { bip_rounds(Aa, Ba, g0); bip_rounds(Ab, Bb, g1); }
        else { bip_rounds(Aa, Bb, g0); bip_rounds(Ab, Ba, g1); }
        groups.push_back(g0);
        groups.push_back(g1);
      }
      add_phase(groups);
    }
  }
}

// ------------------------------------------------------------ small kernels ---
__global__ void __launch_bounds__(256)
    colnorm_kernel(const double *__restrict__ W, int64_t ld, int rows, int ncols,
                   double *__restrict__ out) {
  __shared__ double sh[8][33];
  const int c = blockIdx.x * 32 + (threadIdx.x & 31);
  const int ry = threadIdx.x >> 5;
  double s = 0.0;
  if (c < ncols)
    for (int r = ry; r < rows; r += 8) {
      const double v = W[(int64_t)r * ld + c];
      s += v * v;
    }
  sh[ry][threadIdx.x & 31] = s;
  __syncthreads();
  if (ry == 0 && c < ncols) {
    double tot = 0.0;
    for (int k = 0; k < 8; ++k) tot += sh[k][threadIdx.x & 31];
    out[c] = sqrt(tot);
  }
}

// *negl = (eps |W|_F)^2 from the column norms s (fixed summation order):
// columns whose squared norm is at most this are numerically zero
__global__ void __launch_bounds__(256)
    negligible_kernel(const double *__restrict__ s, int n, double *__restrict__ negl) {
  __shared__ double sh[256];
  double acc = 0.0;
  for (int i = threadIdx.x; i < n; i += 256) acc += s[i] * s[i];
  sh[threadIdx.x] = acc;
  __syncthreads();
  for (int o = 128; o > 0; o >>= 1) {
    if (threadIdx.x < o) sh[threadIdx.x] += sh[threadIdx.x + o];
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    const double t = 2.220446049250313e-16;
    *negl = t * t * sh[0];
  }
}

// UR[:, k] = Z[:, perm[k]] * ls[k]   (rows_w x nk, row-major, ld nk), and
// VH[k, :] = (W[:, perm[k]] / s[perm[k]]) * rs[k]   (nk x rows_w): the kept
// columns only, with the absorbed powers of the singular values folded in.
__global__ void __launch_bounds__(256)
    gather_scaled_kernel(const double *__restrict__ W, const double *__restrict__ Z,
                         int64_t ld, int n, int nk, const int *__restrict__ perm,
                         const double *__restrict__ s, const double *__restrict__ lscale,
                         const double *__restrict__ rscale, double *__restrict__ UR,
                         double *__restrict__ VH) {
  const int64_t tot_u = UR ? (int64_t)n * nk : 0, tot_v = VH ? (int64_t)nk * n : 0;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < tot_u + tot_v;
       i += (int64_t)gridDim.x * blockDim.x) {
    if (i < tot_u) {
      const int64_t r = i / nk;
      const int k = (int)(i - r * nk);
      UR[i] = Z[r * ld + perm[k]] * lscale[k];
    } else {
      const int64_t j = i - tot_u;
      const int k = (int)(j / n);
      const int64_t r = j - (int64_t)k * n;
      const int c = perm[k];
      const double sv = s[c];
      VH[j] = (sv > 0.0) ? (W[r * ld + c] / sv) * rscale[k] : 0.0;
    }
  }
}

__global__ void pad_copy_kernel(const double *__restrict__ src, int64_t rows,
                                int64_t cols, int64_t ld_src, double *__restrict__ dst,
                                int64_t ld_dst, int64_t rows_dst, int mode) {
  // mode 1: identity; mode 2: dst = [src^T | 0]; mode 3: dst = [src | 0]
  const int64_t tot = rows_dst * ld_dst;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < tot;
       i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t r = i / ld_dst, c = i - r * ld_dst;
    double v = 0.0;
    if (mode == 1) v = (r == c) ? 1.0 : 0.0;
    else if (r < rows && c < cols) v = (mode == 3) ? src[r * ld_src + c] : src[c * ld_src + r];
    dst[i] = v;
  }
}

// ------------------------------------------------------------------ driver ---
struct Geom {
  int64_t npad, qr_off, q1_off, r_off, w_off, v_off, s_off, ur_off, perm_off,
      flag_off, pairs_off, scale_off, total;
};

static bool geometry(int64_t m, int64_t n, Geom &g) {
  const int64_t q = qr_workspace_doubles(m, n);
  if (q < 0) return false;
  g.npad = ((n + JP - 1) / JP) * JP;
  auto al = [](int64_t x) { return (x + 31) / 32 * 32; };
  int64_t off = 0;
  g.qr_off = off; off += al(q);
  g.q1_off = off; off += al(m * n);
  g.r_off = off; off += al(n * n);
  g.w_off = off; off += al(n * g.npad);
  g.v_off = off; off += al(g.npad * g.npad);
  g.s_off = off; off += al(g.npad);
  g.ur_off = off; off += al(n * n);
  g.perm_off = off; off += al((g.npad + 1) / 2 + 1);
  g.flag_off = off; off += 32;
  const int64_t nblk = g.npad / JB;
  g.pairs_off = off; off += al(nblk * (nblk - 1) / 2 + 8);   // int2 == one double each
  g.scale_off = off; off += al(2 * n);
  g.total = off;
  return true;
}

// launch geometry of a round: CTAs per cluster, rows per streamed chunk and
// cp.async stages (jacobi_round_kernel<kJacCh, kJacStg, 1>)
constexpr int kJacCs = 2, kJacCh = 64, kJacStg = 4;

// independent sub-tournaments (streams) of a sweep over nblk column blocks
static int pick_groups(int nblk) {
  int groups = nblk < 16 ? 1 : (nblk < 64 ? 2 : 4);
  while (groups > 1 && (nblk < 4 * groups || nblk % (2 * groups))) groups /= 2;
  return groups;
}

static int launch_round(const Params &P, int npairs, cudaStream_t st) {
  auto kern = jacobi_round_kernel<kJacCh, kJacStg, 1>;
  const size_t smem = sizeof(Smem<kJacCh, kJacStg>);
  static bool attr_set = false;
  if (!attr_set) {
    QB_CUDA_CHECK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                       (int)smem));
    attr_set = true;
  }
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3((unsigned)(npairs * kJacCs), 1, 1);
  cfg.blockDim = dim3(256, 1, 1);
  cfg.dynamicSmemBytes = smem;
  cfg.stream = st;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeClusterDimension;
  attr[0].val.clusterDim.x = (unsigned)kJacCs;
  attr[0].val.clusterDim.y = 1;
  attr[0].val.clusterDim.z = 1;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  QB_CUDA_CHECK(cudaLaunchKernelEx(&cfg, kern, P));
  g_launch_count.fetch_add(1, std::memory_order_relaxed);
  return 0;
}

struct SideStreams {
  cudaStream_t cap = nullptr;      // origin stream of the sweep-graph capture
  cudaStream_t s[4] = {nullptr, nullptr, nullptr, nullptr};
  cudaEvent_t fork = nullptr, join[4] = {nullptr, nullptr, nullptr, nullptr};
  bool ok = false;
};
static SideStreams &side_streams() {
  static thread_local SideStreams S;
  if (!S.ok) {
    for (int i = 0; i < 4; ++i) {
      cudaStreamCreateWithFlags(&S.s[i], cudaStreamNonBlocking);
      cudaEventCreateWithFlags(&S.join[i], cudaEventDisableTiming);
    }
    cudaEventCreateWithFlags(&S.fork, cudaEventDisableTiming);
    cudaStreamCreateWithFlags(&S.cap, cudaStreamNonBlocking);
    S.ok = true;
  }
  return S;
}

// Sweeps 1 .. kGraphSweeps - 1 of a multi-group schedule replay a cached CUDA
// graph (QB_JAC_GRAPH=0: direct launches); later sweeps run direct launches
// with fuller inner solves (inner_max = 4).
constexpr int kGraphSweeps = 25;
static bool sweep_graph_eligible(int ngroups) {
  static const bool use_graph = [] {
    const char *e = getenv("QB_JAC_GRAPH");
    return !(e && atoi(e) == 0);
  }();
  return use_graph && !trace_buffer() && ngroups > 1;
}

// Jacobi iteration on W (n x npad, ld npad) accumulating rotations in Z
// (npad x npad).  Returns the number of sweeps (negative: error code).
static int jacobi_iterate(double *W, double *Z, int64_t n, int64_t npad, int2 *d_pairs,
                          int *flag, const double *negl, int *sweeps_out, cudaStream_t st) {
  const int nblk = (int)(npad / JB);
  Schedule sched;
  build_schedule(nblk, pick_groups(nblk), sched);
  QB_CUDA_CHECK(cudaMemcpyAsync(d_pairs, sched.pairs.data(), sizeof(int2) * sched.pairs.size(),
                                cudaMemcpyHostToDevice, st));
  Params P;
  P.W = W; P.V = Z; P.ld = npad; P.rows_w = (int)n; P.rows_v = Z ? (int)npad : 0;
  P.tol = 1e-15 * sqrt((double)n) * 8.0;
  P.negl = negl;
  P.flag = flag;
  P.offmax = reinterpret_cast<unsigned long long *>(flag + 2);
  P.trace = trace_buffer() ? trace_buffer() + 16 * 8192 : nullptr;
  SideStreams &SS = side_streams();
  const bool multi = sched.ngroups > 1;
  int sweeps = 0;
  const int max_sweeps = 60;
  int slot = 0;
  bool done = false;
  // one sweep = every phase forked over the group streams and joined again;
  // `origin` is the stream the forks hang off (the caller's, or the capture
  // stream when the sweep is recorded into a CUDA graph)
  auto enqueue_sweep = [&](cudaStream_t origin) -> int {
    for (const Phase &ph : sched.phases) {
      if (multi) QB_CUDA_CHECK(cudaEventRecord(SS.fork, origin));
      for (size_t g = 0; g < ph.rounds.size(); ++g) {
        cudaStream_t gs = multi ? SS.s[g % 4] : origin;
        if (multi) QB_CUDA_CHECK(cudaStreamWaitEvent(gs, SS.fork, 0));
        for (const auto &rd : ph.rounds[g]) {
          P.pairs = d_pairs + rd.first;
          P.trace_slot = (slot++) & 1023;
          int rc = launch_round(P, rd.second, gs);
          if (rc) return rc;
        }
        if (multi) {
          QB_CUDA_CHECK(cudaEventRecord(SS.join[g % 4], gs));
          QB_CUDA_CHECK(cudaStreamWaitEvent(origin, SS.join[g % 4], 0));
        }
      }
    }
    return 0;
  };
  // Sweeps after the first replay a CUDA graph of the sweep (the launch
  // sequence of a sweep is fixed: ~500 cluster launches on 4 streams cost more
  // host time than the device needs to run them).  The executable graph is
  // cached per (buffers, size; the schedule is a function of npad): a DMRG
  // sweep factors the same shape in the same workspace at every site.
  struct SweepGraph {
    cudaGraphExec_t exec = nullptr;
    const void *W = nullptr, *Z = nullptr, *pairs = nullptr;
    int64_t n = 0, npad = 0;
  };
  static thread_local SweepGraph SG;
  const bool graph_ok = sweep_graph_eligible(sched.ngroups);
  auto graph_matches = [&]() {
    return SG.exec && SG.W == W && SG.Z == Z && SG.pairs == d_pairs && SG.n == n &&
           SG.npad == npad;
  };
  for (; sweeps < max_sweeps && !done; ++sweeps) {
    // one inner sweep per visit is fastest; fall back to fuller inner solves
    // if the outer iteration is unusually slow
    P.inner_max = (sweeps < kGraphSweeps) ? 1 : 4;
    QB_CUDA_CHECK(cudaMemsetAsync(flag, 0, 16, st));
    bool launched = false;
    if (graph_ok && sweeps >= 1 && sweeps < kGraphSweeps) {
      if (!graph_matches()) {
        if (SG.exec) { cudaGraphExecDestroy(SG.exec); SG.exec = nullptr; }
        cudaGraph_t gr = nullptr;
        bool ok = cudaStreamBeginCapture(SS.cap, cudaStreamCaptureModeThreadLocal) == cudaSuccess;
        if (ok) {
          const int rc = enqueue_sweep(SS.cap);
          ok = (cudaStreamEndCapture(SS.cap, &gr) == cudaSuccess) && rc == 0 && gr;
        }
        if (ok) ok = cudaGraphInstantiate(&SG.exec, gr, 0) == cudaSuccess;
        if (gr) cudaGraphDestroy(gr);
        if (ok) {
          SG.W = W; SG.Z = Z; SG.pairs = d_pairs; SG.n = n; SG.npad = npad;
        } else {
          cudaGetLastError();     // clear; fall back to direct launches
          SG.exec = nullptr;
        }
      }
      if (SG.exec) {
        QB_CUDA_CHECK(cudaGraphLaunch(SG.exec, st));
        g_launch_count.fetch_add(1, std::memory_order_relaxed);
        launched = true;
      }
    }
    if (!launched) {
      int rc = enqueue_sweep(st);
      if (rc) return -rc;
    }
    struct { int flag; int pad; unsigned long long off; } h = {0, 0, 0};
    QB_CUDA_CHECK(cudaMemcpyAsync(&h, flag, 16, cudaMemcpyDeviceToHost, st));
    QB_CUDA_CHECK(cudaStreamSynchronize(st));
    // converged when a whole sweep rotated nothing.  (Stopping one sweep
    // earlier because the largest scaled off-diagonal was tiny is NOT safe:
    // for close singular values the rotation ANGLES stay large however small
    // the off-diagonal is, and they re-mix third columns at first order --
    // measured: 1e-11 .. 2e-10 loss of orthogonality on degenerate spectra.)
    if (!h.flag) done = true;
  }
  if (sweeps_out) *sweeps_out = sweeps;
  if (!done) {
    set_error("qb_svd: Jacobi did not converge in %d sweeps", max_sweeps);
    return -2;
  }
  return sweeps;
}

}  // namespace jac2

// quimb's absorb codes -> powers of s on the two factors and which to form
struct AbsorbPlan { double lpow, rpow; bool want_l, want_r, want_s; };
static bool absorb_plan(int absorb, AbsorbPlan &a) {
  switch (absorb) {
    case QB_ABSORB_FULL:    a = {0.0, 0.0, true, true, true}; return true;
    case QB_ABSORB_S:       a = {0.0, 0.0, false, false, true}; return true;
    case QB_ABSORB_LEFT:    a = {1.0, 0.0, true, true, false}; return true;
    case QB_ABSORB_LFACTOR: a = {1.0, 0.0, true, false, false}; return true;
    case QB_ABSORB_RORTHOG: a = {0.0, 0.0, false, true, false}; return true;
    case QB_ABSORB_BOTH:    a = {0.5, 0.5, true, true, false}; return true;
    case QB_ABSORB_LSQRT:   a = {0.5, 0.0, true, false, false}; return true;
    case QB_ABSORB_RSQRT:   a = {0.0, 0.5, false, true, false}; return true;
    case QB_ABSORB_RIGHT:   a = {0.0, 1.0, true, true, false}; return true;
    case QB_ABSORB_LORTHOG: a = {0.0, 0.0, true, false, false}; return true;
    case QB_ABSORB_RFACTOR: a = {0.0, 1.0, false, true, false}; return true;
  }
  return false;
}

// Epilogue algorithm of an absorb mode (see svd_trunc_tall)
enum { EPI_ACCUMULATE = 0, EPI_LEFT = 1, EPI_RIGHT = 2, EPI_VALUES = 3 };
static int epilogue_kind(int absorb) {
  static const bool no_accum_ok = [] {
    const char *e = getenv("QB_SVD_ACCUMULATE");
    return !(e && atoi(e) == 1);
  }();
  if (!no_accum_ok) return EPI_ACCUMULATE;
  if (absorb == QB_ABSORB_LEFT || absorb == QB_ABSORB_LFACTOR || absorb == QB_ABSORB_RORTHOG)
    return EPI_LEFT;
  if (absorb == QB_ABSORB_RIGHT || absorb == QB_ABSORB_LORTHOG || absorb == QB_ABSORB_RFACTOR)
    return EPI_RIGHT;
  if (absorb == QB_ABSORB_S) return EPI_VALUES;
  return EPI_ACCUMULATE;
}

// SVD of row-major X (m x n), m >= n, with the truncation / absorb epilogue.
// U: m x nk (ld nk), S: nk, VH: nk x n, written compactly for the kept rank.
static int svd_trunc_tall(int64_t m, int64_t n, const double *X, double cutoff,
                          int cutoff_mode, int64_t max_bond, int absorb, int renorm,
                          double *U, double *S, double *VH, int64_t *n_keep_out,
                          double *err_out, int64_t *n_null_out, double *ws,
                          int *sweeps_out, cudaStream_t st) {
  using namespace jac2;
  Geom g;
  if (!geometry(m, n, g)) {
    set_error("qb_svd: unsupported shape %lld x %lld", (long long)m, (long long)n);
    return -2;
  }
  AbsorbPlan ap;
  if (!absorb_plan(absorb, ap)) {
    set_error("qb_svd_trunc: invalid absorb code %d", absorb);
    return -8;
  }
  double *Q1 = ws + g.q1_off, *R = ws + g.r_off, *W = ws + g.w_off;
  double *Z = ws + g.v_off, *sv = ws + g.s_off, *UR = ws + g.ur_off;
  int *perm = reinterpret_cast<int *>(ws + g.perm_off);
  int *flag = reinterpret_cast<int *>(ws + g.flag_off);
  int2 *d_pairs = reinterpret_cast<int2 *>(ws + g.pairs_off);
  double *d_scale = ws + g.scale_off;
  const int blocks = sm_count() * 4;
  // Modes whose RIGHT factor is the isometry (left / lfactor / rorthog) and the
  // values-only mode need no accumulated rotations: with W = R^T the rotated
  // columns are W Z = Y S, so V = Y is read off the normalised columns and
  // U (f S) = f X Y is one GEMM on the original matrix -- the apply phase
  // touches half the rows, Z is never formed and neither is Q1.  (The mirror
  // family -- right / lorthog / rfactor -- reaches this path through the
  // transpose in the host layer for square input.)  Modes that return BOTH
  // isometries (None, both, lsqrt, rsqrt) keep the accumulation: dividing the
  // other factor by tiny singular values would lose its orthogonality.
  // (Mirror family, U the isometry: rotate the columns of R itself,
  // R Z' = U_R S, so U = Q1 U_R from the normalised columns and
  // (f S) V^T = f U_R^T R by one GEMM.)
  const int epi = epilogue_kind(absorb);
  const bool right_family = epi == EPI_RIGHT;
  const bool vals_only = epi == EPI_VALUES;
  const bool accumulate = epi == EPI_ACCUMULATE;
  const bool need_u = ap.want_l && U;
  // R in the units of 2^-e X (decomp_scale_exp): the Jacobi iteration, the
  // rotated columns and their norms stay scaled, the singular values the keep
  // rule and the absorbed powers see are scaled back
  int rc = qr_f64(m, n, X, (need_u && (accumulate || right_family)) ? Q1 : nullptr, R,
                  /*stabilized=*/0, ws + g.qr_off, st, /*keep_scaled=*/true);
  if (rc) return rc;
  unsigned long long maxbits = 0;
  QB_CUDA_CHECK(cudaMemcpyAsync(&maxbits, qr_maxbits(ws + g.qr_off), sizeof(maxbits),
                                cudaMemcpyDeviceToHost, st));
  QB_CUDA_CHECK(cudaStreamSynchronize(st));
  if (!decomp_finite(maxbits)) {
    set_error("qb_svd: the input contains NaN or Inf");
    return -9;
  }
  const int e = decomp_scale_exp(maxbits);
  const int64_t npad = g.npad;
  // W = R^T, or R itself for the accumulation-free right family
  pad_copy_kernel<<<blocks, 256, 0, st>>>(R, n, n, n, W, npad, n,
                                          (right_family && !accumulate) ? 3 : 2);
  QB_LAUNCH_CHECK();
  if (accumulate) {
    pad_copy_kernel<<<blocks, 256, 0, st>>>(nullptr, 0, 0, 0, Z, npad, npad, 1);
    QB_LAUNCH_CHECK();
  } else {
    Z = nullptr;
  }
  double *negl = reinterpret_cast<double *>(flag) + 4;
  colnorm_kernel<<<(unsigned)(npad / 32), 256, 0, st>>>(W, npad, (int)n, (int)npad, sv);
  QB_LAUNCH_CHECK();
  negligible_kernel<<<1, 256, 0, st>>>(sv, (int)n, negl);
  QB_LAUNCH_CHECK();
  int sw = jacobi_iterate(W, Z, n, npad, d_pairs, flag, negl, sweeps_out, st);
  if (sw < 0) return -sw;
  colnorm_kernel<<<(unsigned)(npad / 32), 256, 0, st>>>(W, npad, (int)n, (int)npad, sv);
  QB_LAUNCH_CHECK();
  std::vector<double> hs(npad);
  double hnegl = 0.0;
  QB_CUDA_CHECK(cudaMemcpyAsync(hs.data(), sv, sizeof(double) * npad,
                                cudaMemcpyDeviceToHost, st));
  QB_CUDA_CHECK(cudaMemcpyAsync(&hnegl, negl, sizeof(double), cudaMemcpyDeviceToHost, st));
  QB_CUDA_CHECK(cudaStreamSynchronize(st));
  // numerically zero columns (they took no part in the iteration): singular
  // value 0, so the caller completes their vectors to isometries
  bool zeroed = false;
  for (int64_t i = 0; i < n; ++i)
    if (hs[i] > 0.0 && hs[i] * hs[i] <= hnegl) { hs[i] = 0.0; zeroed = true; }
  if (zeroed)
    QB_CUDA_CHECK(cudaMemcpyAsync(sv, hs.data(), sizeof(double) * n, cudaMemcpyHostToDevice, st));
  std::vector<int> hp(npad);
  for (int i = 0; i < npad; ++i) hp[i] = i;
  std::stable_sort(hp.begin(), hp.end(), [&](int a, int b) {
    const bool pa = a >= n, pb = b >= n;  // padding columns last
    if (pa != pb) return pb;
    return hs[a] > hs[b];
  });
  // sorted singular values: ss in the caller's units, ssc in those of 2^-e X
  std::vector<double> ss(n), ssc(n);
  for (int i = 0; i < n; ++i) {
    ssc[i] = hs[hp[i]];
    ss[i] = e ? ldexp(ssc[i], e) : ssc[i];
  }
  // ---- the reference's keep rule / renormalisation on the sorted values ----
  int64_t nk = n;
  double f = 1.0, err = 0.0;
  if (cutoff_mode != 0) {
    rc = qb_svals_to_keep(ss.data(), n, cutoff, cutoff_mode, max_bond, renorm, &nk, &f, &err);
    if (rc) return rc;
  }
  int64_t n_null = 0;
  for (int64_t i = 0; i < nk; ++i) n_null += !(ss[i] > 0.0);
  if (n_keep_out) *n_keep_out = nk;
  if (err_out) *err_out = err;
  if (n_null_out) *n_null_out = n_null;
  // scales of the kept columns / rows: (f s)^lpow, (f s)^rpow
  std::vector<double> sc(2 * nk), sk(nk);
  for (int64_t i = 0; i < nk; ++i) {
    const double v = ss[i] * f;
    sk[i] = v;
    sc[i] = ap.lpow == 0.0 ? 1.0 : (ap.lpow == 1.0 ? v : sqrt(v));
    sc[nk + i] = ap.rpow == 0.0 ? 1.0 : (ap.rpow == 1.0 ? v : sqrt(v));
  }
  QB_CUDA_CHECK(cudaMemcpyAsync(perm, hp.data(), sizeof(int) * nk, cudaMemcpyHostToDevice, st));
  QB_CUDA_CHECK(cudaMemcpyAsync(d_scale, sc.data(), sizeof(double) * 2 * nk,
                                cudaMemcpyHostToDevice, st));
  if (S && ap.want_s)
    QB_CUDA_CHECK(cudaMemcpyAsync(S, sk.data(), sizeof(double) * nk, cudaMemcpyHostToDevice, st));
  const bool need_v = ap.want_r && VH;
  if (!accumulate) {
    if (vals_only) {
      QB_CUDA_CHECK(cudaStreamSynchronize(st));
      return 0;
    }
    if (right_family) {
      // U_R (n x nk) = normalised rotated columns of R (scale 1 / s, null
      // columns stay zero); U = Q1 U_R; (f S) V^T = f U_R^T R (R scaled by
      // 2^-e, so the GEMM takes f 2^e)
      std::vector<double> inv(nk);
      for (int64_t i = 0; i < nk; ++i) inv[i] = ssc[i] > 0.0 ? 1.0 / ssc[i] : 0.0;
      QB_CUDA_CHECK(cudaMemcpyAsync(d_scale, inv.data(), sizeof(double) * nk,
                                    cudaMemcpyHostToDevice, st));
      gather_scaled_kernel<<<blocks, 256, 0, st>>>(W, W, npad, (int)n, (int)nk, perm, sv,
                                                   d_scale, d_scale, UR, nullptr);
      QB_LAUNCH_CHECK();
      QB_CUDA_CHECK(cudaStreamSynchronize(st));  // host vectors go out of scope
      if (need_u) {
        rc = gemm_f64(Q1, n, 1, UR, nk, 1, U, nk, 1, m, nk, n, 1.0, 0.0, st);
        if (rc) return rc;
      }
      if (need_v) {
        rc = gemm_f64(UR, 1, nk, R, n, 1, VH, n, 1, nk, n, n, e ? ldexp(f, e) : f, 0.0, st);
        if (rc) return rc;
      }
      return 0;
    }
    // Y^T (nk x n, rows = normalised rotated columns): the caller's VH, or
    // scratch when only the left factor is wanted
    double *Yt = need_v ? VH : UR;
    gather_scaled_kernel<<<blocks, 256, 0, st>>>(W, W, npad, (int)n, (int)nk, perm, sv,
                                                 d_scale, d_scale + nk, nullptr, Yt);
    QB_LAUNCH_CHECK();
    QB_CUDA_CHECK(cudaStreamSynchronize(st));  // host vectors go out of scope
    if (need_u) {
      // U (f S) = f X Y :  (m x n) . (n x nk), Y[i, j] = Yt[j, i]
      rc = gemm_f64(X, n, 1, Yt, 1, n, U, nk, 1, m, nk, n, f, 0.0, st);
      if (rc) return rc;
    }
    return 0;
  }
  if (need_u || need_v) {
    gather_scaled_kernel<<<blocks, 256, 0, st>>>(W, Z, npad, (int)n, (int)nk, perm, sv,
                                                 d_scale, d_scale + nk,
                                                 need_u ? UR : nullptr, need_v ? VH : nullptr);
    QB_LAUNCH_CHECK();
  }
  QB_CUDA_CHECK(cudaStreamSynchronize(st));  // host vectors go out of scope
  if (need_u) {
    // U (m x nk) = Q1 (m x n) . UR (n x nk)
    rc = gemm_f64(Q1, n, 1, UR, nk, 1, U, nk, 1, m, nk, n, 1.0, 0.0, st);
    if (rc) return rc;
  }
  return 0;
}

}  // namespace qb

using namespace qb;

extern "C" {

int64_t qb_svd_workspace(int dtype, int64_t m, int64_t n) {
  if (dtype != QB_F64) return -1;
  jac2::Geom g;
  const int64_t mm = std::max(m, n), nn = std::min(m, n);
  if (!jac2::geometry(mm, nn, g)) return -2;
  return g.total * 8;
}

static int svd_check(const char *who, int dtype, int64_t m, int64_t n, void *workspace,
                     size_t workspace_bytes) {
  if (dtype != QB_F64) {
    set_error("%s: only f64 is implemented (got dtype %d)", who, dtype);
    return -1;
  }
  if (m < n) {
    set_error("%s: m < n -- pass the transpose (m >= n required)", who);
    return -2;
  }
  const int64_t need = qb_svd_workspace(dtype, m, n);
  if (need < 0) {
    set_error("%s: unsupported shape %lld x %lld", who, (long long)m, (long long)n);
    return -2;
  }
  if (!workspace || (int64_t)workspace_bytes < need) {
    set_error("%s: workspace too small (need %lld bytes)", who, (long long)need);
    return -8;
  }
  return 0;
}

int qb_svd(int dtype, int64_t m, int64_t n, const void *X, void *U, void *S,
           void *VH, void *workspace, size_t workspace_bytes, int *sweeps_out,
           void *stream) {
  if (m <= 0 || n <= 0) return 0;
  int rc = svd_check("qb_svd", dtype, m, n, workspace, workspace_bytes);
  if (rc) return rc;
  return svd_trunc_tall(m, n, (const double *)X, -1.0, 0, -1, QB_ABSORB_FULL, 0,
                        (double *)U, (double *)S, (double *)VH, nullptr, nullptr, nullptr,
                        static_cast<double *>(workspace), sweeps_out,
                        static_cast<cudaStream_t>(stream));
}

// TEST / debug entry, host only: the sweep schedule of the Jacobi SVD for
// `nblk` column blocks and `groups` independent streams.  Writes one record
// (phase, group, round, p, q) of five int32 per column-block pair into `out`
// (capacity in records) and returns the number of records (negative: capacity
// too small).  `*groups_used` receives the group count actually used.
int64_t qb_debug_jacobi_schedule(int nblk, int groups, int32_t *out, int64_t capacity,
                                 int *groups_used) {
  jac2::Schedule S;
  jac2::build_schedule(nblk, groups, S);
  if (groups_used) *groups_used = S.ngroups;
  int64_t n = 0;
  for (size_t ph = 0; ph < S.phases.size(); ++ph)
    for (size_t g = 0; g < S.phases[ph].rounds.size(); ++g)
      for (size_t r = 0; r < S.phases[ph].rounds[g].size(); ++r) {
        const auto &rd = S.phases[ph].rounds[g][r];
        for (int i = 0; i < rd.second; ++i) {
          if (n >= capacity) return -1;
          const int2 pr = S.pairs[rd.first + i];
          int32_t *o = out + 5 * n++;
          o[0] = (int32_t)ph; o[1] = (int32_t)g; o[2] = (int32_t)r; o[3] = pr.x; o[4] = pr.y;
        }
      }
  return n;
}

// Host only: what qb_svd_trunc (qb_svd: absorb = QB_ABSORB_FULL) launches for
// a tall m x n matrix (m >= n), from the decisions of the launch path.
int qb_svd_route(int64_t m, int64_t n, int absorb, int64_t *out) {
  jac2::Geom g;
  QrRoute q;
  AbsorbPlan ap;
  if (m < n || n <= 0 || !jac2::geometry(m, n, g) || !qr_route(m, n, q)) {
    set_error("qb_svd_route: unsupported shape %lld x %lld", (long long)m, (long long)n);
    return -2;
  }
  if (!absorb_plan(absorb, ap)) {
    set_error("qb_svd_route: invalid absorb code %d", absorb);
    return -8;
  }
  const int nblk = (int)(g.npad / jac2::JB);
  jac2::Schedule S;
  jac2::build_schedule(nblk, jac2::pick_groups(nblk), S);
  int64_t rounds = 0;
  for (const auto &ph : S.phases)
    for (const auto &gr : ph.rounds) rounds += (int64_t)gr.size();
  out[0] = g.npad; out[1] = nblk; out[2] = S.ngroups; out[3] = jac2::kJacCs;
  out[4] = jac2::kJacCh; out[5] = jac2::kJacStg; out[6] = epilogue_kind(absorb);
  out[7] = jac2::sweep_graph_eligible(S.ngroups) ? jac2::kGraphSweeps - 1 : 0;
  out[8] = q.panel_mask; out[9] = q.wy_t; out[10] = rounds;
  return 0;
}

int qb_svd_trunc(int dtype, int64_t m, int64_t n, const void *X, double cutoff,
                 int cutoff_mode, int64_t max_bond, int absorb, int renorm, void *U,
                 void *S, void *VH, int64_t *n_keep, double *trunc_error,
                 int64_t *n_null, void *workspace, size_t workspace_bytes,
                 int *sweeps_out, void *stream) {
  if (m <= 0 || n <= 0) {
    if (n_keep) *n_keep = 0;
    return 0;
  }
  int rc = svd_check("qb_svd_trunc", dtype, m, n, workspace, workspace_bytes);
  if (rc) return rc;
  if (cutoff_mode < 1 || cutoff_mode > 6) {
    set_error("qb_svd_trunc: invalid cutoff_mode %d", cutoff_mode);
    return -6;
  }
  return svd_trunc_tall(m, n, (const double *)X, cutoff, cutoff_mode, max_bond, absorb,
                        renorm, (double *)U, (double *)S, (double *)VH, n_keep,
                        trunc_error, n_null, static_cast<double *>(workspace), sweeps_out,
                        static_cast<cudaStream_t>(stream));
}

}  // extern "C"
