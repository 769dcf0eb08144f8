// Dense factorizations of the split half of quimb's hot path, fp64:
//
//   qb_qr_stab  <- qr_stabilized (quimb/tensor/decomp.py:2055-2216): blocked
//                  Householder QR (compact WY).  The panel factorization is
//                  ONE CTA that keeps the whole tall panel in registers
//                  (1024 threads x RPT rows x NB columns) and needs a single
//                  NB-wide block reduction per column; trailing updates and
//                  the formation of Q are GEMMs on the contraction kernel.
//                  The stabilisation (diag(R) >= 0, phase into Q) is a fused
//                  epilogue kernel.
//   qb_svd      <- the LAPACK gesdd call inside svd_truncated
//                  (decomp.py:1032-1055): one-sided block Jacobi on the
//                  R factor of a QR preconditioner.  Per round, one CTA per
//                  column-block pair: Gram matrix with DMMA-free register
//                  tiles, cyclic Jacobi eigen-solve of the 2b x 2b Gram in
//                  shared memory, rotation applied to the columns of the
//                  working matrix and of V.  The working set (n x n twice)
//                  is 64 MB at n = 2048 (the H100's L2 holds 50 MB).
//   qb_svals_to_keep <- _compute_number_svals_to_keep_numba + renorm factor
//                  (decomp.py:901-965), host side, bit-for-bit the same
//                  summation order as the reference.
#include <cooperative_groups.h>
#include <math.h>
#include <stdlib.h>

#include <algorithm>
#include <vector>

#include "internal.h"

namespace qb {

// =========================================================================
//                                   QR
// =========================================================================

// reduce NB per-thread partials over the warp: lane c (< NB) ends up with
// the sum over all lanes of p[c] (recursive halving, NB-1 shuffles)
template <int NB>
__device__ __forceinline__ double warp_multi_reduce(double (&p)[NB], int lane) {
#pragma unroll
  for (int off = NB / 2, cnt = NB / 2; off >= 1; off >>= 1, cnt >>= 1) {
    const bool upper = (lane & off) != 0;
#pragma unroll
    for (int i = 0; i < cnt; ++i) {
      double send = upper ? p[i] : p[i + cnt];
      double keep = upper ? p[i + cnt] : p[i];
      p[i] = keep + __shfl_xor_sync(0xffffffffu, send, off);
    }
  }
  double v = p[0];  // lane L holds index L % NB, partial over its NB-lane group
#pragma unroll
  for (int off = NB; off < 32; off <<= 1) v += __shfl_xor_sync(0xffffffffu, v, off);
  return v;
}

// Householder factorization of an m x nbw panel (nbw <= NB), row-major with
// leading dimension lda, m <= 2048 * RPT.  One thread-block CLUSTER of 8 CTAs
// (256 threads each) keeps the whole panel in registers: thread t of CTA r
// owns rows i*2048 + r*256 + t.  Per column there is ONE cluster-wide
// reduction of NB partial dot products through distributed shared memory
// (double buffered, so a single cluster.sync per column).
// In place: R on/above the diagonal, Householder vectors below.  Also writes
// the explicit V (m x NB, unit diagonal, zeros above; row-major ld NB) and
// the NB x NB upper triangular T of the compact WY form  Q = I - V T V^T.
constexpr int QR_CLUSTER = 8;
constexpr int QR_THREADS = 256;

template <int NB, int RPT>
__global__ void __cluster_dims__(QR_CLUSTER, 1, 1) __launch_bounds__(QR_THREADS, 1)
    qr_panel_kernel(double *__restrict__ A, int64_t lda, int m, int nbw,
                    double *__restrict__ Vout, int64_t ldv, double *__restrict__ Tout) {
  namespace cg = cooperative_groups;
  cg::cluster_group cluster = cg::this_cluster();
  const int rank = (int)cluster.block_rank();
  constexpr int NW = QR_THREADS / 32;
  __shared__ double red[NW][NB + 1];
  __shared__ double part[2][NB];   // this CTA's partial dots (DSMEM-visible)
  __shared__ double rowj_s[2][NB]; // row j of the panel if this CTA owns it
  __shared__ double dots[NB];
  __shared__ double rowj[NB];
  __shared__ double Ts[NB][NB + 1];
  __shared__ double hh[3];  // tau, scale, beta
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  constexpr int ROWS_PER_PASS = QR_CLUSTER * QR_THREADS;

  double a[RPT][NB];
#pragma unroll
  for (int i = 0; i < RPT; ++i) {
    const int row = i * ROWS_PER_PASS + rank * QR_THREADS + tid;
#pragma unroll
    for (int c = 0; c < NB; ++c)
      a[i][c] = (row < m && c < nbw) ? A[(int64_t)row * lda + c] : 0.0;
  }
  for (int i = tid; i < NB * (NB + 1); i += QR_THREADS) (&Ts[0][0])[i] = 0.0;
  __syncthreads();

#pragma unroll 1
  for (int j = 0; j < nbw; ++j) {
    const int buf = j & 1;
    // ---- partial u_c = sum_{row > j} a[row][j] * a[row][c]  for all c ----
    double p[NB];
#pragma unroll
    for (int c = 0; c < NB; ++c) p[c] = 0.0;
#pragma unroll
    for (int i = 0; i < RPT; ++i) {
      const int row = i * ROWS_PER_PASS + rank * QR_THREADS + tid;
      if (row > j && row < m) {
        // a[i][j] with runtime j: select through an unrolled scan
        double x = 0.0;
#pragma unroll
        for (int c = 0; c < NB; ++c) x = (c == j) ? a[i][c] : x;
#pragma unroll
        for (int c = 0; c < NB; ++c) p[c] += x * a[i][c];
      }
      if (row == j) {
#pragma unroll
        for (int c = 0; c < NB; ++c) rowj_s[buf][c] = a[i][c];
      }
    }
    double r = warp_multi_reduce<NB>(p, lane);
    if (lane < NB) red[warp][lane] = r;
    __syncthreads();
    if (tid < NB) {
      double s = 0.0;
#pragma unroll
      for (int w = 0; w < NW; ++w) s += red[w][tid];
      part[buf][tid] = s;
    }
    cluster.sync();
    // ---- every CTA: total dots, row j, Householder scalars, T column -----
    if (warp == 0) {
      if (lane < NB) {
        double s = 0.0;
#pragma unroll
        for (int q = 0; q < QR_CLUSTER; ++q) {
          const double *rp = cluster.map_shared_rank(&part[buf][0], q);
          s += rp[lane];
        }
        dots[lane] = s;
        const int owner = (j % ROWS_PER_PASS) / QR_THREADS;
        const double *rr = cluster.map_shared_rank(&rowj_s[buf][0], owner);
        rowj[lane] = rr[lane];
      }
      __syncwarp();
      // LAPACK dlarfg
      const double alpha = rowj[j];
      const double xnorm2 = dots[j];
      double tau, scale, beta;
      if (xnorm2 == 0.0) {
        tau = 0.0; scale = 0.0; beta = alpha;
      } else {
        beta = -copysign(sqrt(alpha * alpha + xnorm2), alpha);
        tau = (beta - alpha) / beta;
        scale = 1.0 / (alpha - beta);
      }
      if (lane == 0) { hh[0] = tau; hh[1] = scale; hh[2] = beta; }
      // T(0:j, j) = -tau * T(0:j,0:j) * (V^T v_j),
      // z_c = v_c^T v_j = rowj[c] + scale * u_c   (c < j)
      double acc = 0.0;
      if (lane < j && lane < NB) {
        for (int k = lane; k < j; ++k)
          acc += Ts[lane][k] * (rowj[k] + scale * dots[k]);
      }
      __syncwarp();
      if (lane < j && lane < NB) Ts[lane][j] = -tau * acc;
      if (lane == j) Ts[j][j] = tau;
    }
    __syncthreads();
    const double tau = hh[0], scale = hh[1], beta = hh[2];
    // ---- apply H_j to the trailing panel columns, store v_j --------------
#pragma unroll
    for (int i = 0; i < RPT; ++i) {
      const int row = i * ROWS_PER_PASS + rank * QR_THREADS + tid;
      if (row >= j && row < m) {
        double x = 0.0;
#pragma unroll
        for (int c = 0; c < NB; ++c) x = (c == j) ? a[i][c] : x;
        const double v = (row == j) ? 1.0 : x * scale;
#pragma unroll
        for (int c = 0; c < NB; ++c) {
          if (c > j) {
            const double w = rowj[c] + scale * dots[c];  // v^T a_c
            a[i][c] -= tau * v * w;
          } else if (c == j) {
            a[i][c] = (row == j) ? beta : v;
          }
        }
      }
    }
    __syncthreads();
  }
  // nobody may exit while peers can still read its shared memory
  cluster.sync();

  // ---- write back: factored panel, explicit V, T -------------------------
#pragma unroll
  for (int i = 0; i < RPT; ++i) {
    const int row = i * ROWS_PER_PASS + rank * QR_THREADS + tid;
    if (row < m) {
#pragma unroll
      for (int c = 0; c < NB; ++c) {
        if (c < nbw) {
          A[(int64_t)row * lda + c] = a[i][c];
          double v = (row > c) ? a[i][c] : (row == c ? 1.0 : 0.0);
          Vout[(int64_t)row * ldv + c] = v;
        }
      }
    }
  }
  if (rank == 0) {
    for (int i = tid; i < NB * NB; i += QR_THREADS) {
      int r = i / NB, c = i % NB;
      Tout[i] = (r < nbw && c < nbw) ? Ts[r][c] : 0.0;
    }
  }
}

// R = upper triangle of the factored matrix (first n rows), zeros below,
// scaled back by 2^e (e from the input's max|x|, 0 when not scaled)
__global__ void extract_r_kernel(const double *__restrict__ F, int64_t ldf,
                                 int k, int n, double *__restrict__ R,
                                 const unsigned long long *__restrict__ maxbits) {
  const int e = maxbits ? decomp_scale_exp(*maxbits) : 0;
  int64_t total = (int64_t)k * n;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total;
       i += (int64_t)gridDim.x * blockDim.x) {
    int r = (int)(i / n), c = (int)(i - (int64_t)r * n);
    const double v = (c >= r) ? F[(int64_t)r * ldf + c] : 0.0;
    R[i] = e ? ldexp(v, e) : v;
  }
}

// *out = max(*out, bits of max|X|): the bits of non-negative doubles order
// as unsigned integers, and |NaN| sorts above +inf
__global__ void __launch_bounds__(256)
    maxabs_bits_kernel(const double *__restrict__ X, int64_t total,
                       unsigned long long *__restrict__ out) {
  unsigned long long mx = 0;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total;
       i += (int64_t)gridDim.x * blockDim.x)
    mx = max(mx, (unsigned long long)__double_as_longlong(fabs(X[i])));
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) mx = max(mx, __shfl_xor_sync(0xffffffffu, mx, o));
  if ((threadIdx.x & 31) == 0 && mx) atomicMax(out, mx);
}

// F = 2^-e X (a plain copy when e = 0)
__global__ void __launch_bounds__(256)
    scale_copy_kernel(const double *__restrict__ X, int64_t total, double *__restrict__ F,
                      const unsigned long long *__restrict__ maxbits) {
  const int e = decomp_scale_exp(*maxbits);
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total;
       i += (int64_t)gridDim.x * blockDim.x)
    F[i] = e ? ldexp(X[i], -e) : X[i];
}

__global__ void set_identity_kernel(double *Q, int64_t m, int64_t n) {
  int64_t total = m * n;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total;
       i += (int64_t)gridDim.x * blockDim.x) {
    int64_t r = i / n, c = i - r * n;
    Q[i] = (r == c) ? 1.0 : 0.0;
  }
}

// stabilisation: phase_i = sgn(R_ii) (sgn(0) = 1);  Q[:, i] *= phase_i,
// R[i, :] *= phase_i  (decomp.py:2108-2124 / 2147-2178 for real dtypes)
__global__ void qr_phase_kernel(double *__restrict__ Q, int64_t m, int64_t kq,
                                double *__restrict__ R, int64_t k, int64_t n,
                                const double *__restrict__ Rdiag_src,
                                int64_t ld_src) {
  const int64_t totq = Q ? m * kq : 0, totr = R ? k * n : 0;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
       i < totq + totr; i += (int64_t)gridDim.x * blockDim.x) {
    if (i < totq) {
      int64_t c = i % kq;
      if (Rdiag_src[c * ld_src + c] < 0.0) Q[i] = -Q[i];
    } else {
      int64_t j = i - totq, r = j / n;
      if (Rdiag_src[r * ld_src + r] < 0.0) R[j] = -R[j];
    }
  }
}

template <int NB, int RPT>
static int launch_panel(double *A, int64_t lda, int m, int nbw, double *V, int64_t ldv,
                        double *T, cudaStream_t st) {
  qr_panel_kernel<NB, RPT><<<QR_CLUSTER, QR_THREADS, 0, st>>>(A, lda, m, nbw, V, ldv, T);
  QB_LAUNCH_CHECK();
  return 0;
}

// Outer (aggregated) panel width: the narrow register-resident panels (8-32
// columns) only update the rest of their own outer panel; the trailing matrix
// is updated once per outer panel with K = QR_NBO GEMMs (compact WY form of the
// whole outer panel), so it is streamed n / QR_NBO times instead of n / nb.
constexpr int QR_NBO = 128;

struct QrGeom {
  int nb;
  int64_t f_off, v_off, t_off, to_off, g_off, w_off, w2_off, sk_off, sk_elems, total;  // doubles
};

// inner panel width: one row per thread up to 2048 rows, (NB, rows/thread) =
// (32,1) or (32,2) up to 4096 rows, (16,4) up to 8192, (8,8) up to 16384
static int qr_inner_width(int64_t m) {
  if (m <= 4096) return 32;
  if (m <= 8192) return 16;
  if (m <= 16384) return 8;
  return 0;
}

// panel instantiation for a panel of `rows` rows: 0 (32,1), 1 (32,2),
// 2 (16,4), 3 (8,8)
static int qr_panel_kind(int nb, int64_t rows) {
  if (nb == 32) return rows <= 2048 ? 0 : 1;
  return nb == 16 ? 2 : 3;
}

// Aggregation pays when the trailing matrix does not stay in L2; for an
// L2-resident matrix the extra Gram GEMM + triangular inverse per outer
// panel cost more than the narrower updates save, so there every inner
// panel is its own outer panel and its T is used as it comes.  Measured on
// an H100 SXM at a 400 W power limit, Q and R, without / with aggregation:
// 2048 x 1024 (16 MiB) 9.3 / 11.2 ms, 2048^2 (32 MiB) 19.7 / 22.7 ms,
// 3072 x 2048 (48 MiB) 25.5 / 27.1 ms, 4096 x 2048 (64 MiB) 31.2 / 31.4 ms,
// 4096^2 (128 MiB) 66.3 / 60.3 ms.
static int qr_outer_width(int64_t m, int64_t n, int nb) {
  return (m > 4096 || m * n * 8 > (int64_t)48 << 20) ? QR_NBO : nb;
}

bool qr_route(int64_t m, int64_t n, QrRoute &r) {
  r = QrRoute{0, 0, 0, 0, 0, 0};
  r.nb = qr_inner_width(m);
  if (!r.nb || m <= 0 || n <= 0) return false;
  const int64_t k = std::min(m, n);
  r.nbo = qr_outer_width(m, n, r.nb);
  for (int64_t j0 = 0; j0 < k; j0 += r.nbo) {
    const int64_t w = std::min<int64_t>(r.nbo, k - j0);
    ++r.nout;
    if (w > r.nb) r.wy_t = 1;
    for (int64_t ji = 0; ji < w; ji += r.nb) {
      ++r.npan;
      r.panel_mask |= 1 << qr_panel_kind(r.nb, m - (j0 + ji));
    }
  }
  return true;
}

static bool qr_geometry(int64_t m, int64_t n, QrGeom &g) {
  const int64_t k = std::min(m, n);
  g.nb = qr_inner_width(m);
  if (!g.nb) return false;
  const int64_t npan = (k + g.nb - 1) / g.nb;
  const int64_t nout = (k + QR_NBO - 1) / QR_NBO;
  auto al = [](int64_t x) { return (x + 31) / 32 * 32; };  // 256-byte sections
  int64_t off = 32;                                // [0]: bits of max|X| (qr_maxbits)
  g.f_off = off; off += al(m * n);                 // factored copy of X
  g.v_off = off; off += al(m * (nout * QR_NBO));   // explicit V, one m x w slab per outer panel
  g.t_off = off; off += al(npan * g.nb * g.nb);    // T per inner panel (tau on the diagonal)
  g.to_off = off; off += al(nout * QR_NBO * QR_NBO);  // T per outer panel
  g.g_off = off; off += al((int64_t)QR_NBO * QR_NBO);
  g.w_off = off; off += al((int64_t)QR_NBO * std::max(n, k));
  g.w2_off = off; off += al((int64_t)QR_NBO * std::max(n, k));
  g.sk_elems = al((int64_t)16 * QR_NBO * std::max(n, k));  // split-K partials
  g.sk_off = off; off += g.sk_elems;
  g.total = off;
  return true;
}

// T of the compact WY form of w aggregated reflectors from the Gram matrix of
// their vectors:  T^-1 = striu(V^T V) + diag(1 / tau)  (Puglisi 1992; Joffrain
// et al. 2006).  One CTA, thread j back-substitutes column j of T.  tau_i sits
// on the diagonal of the inner panels' T (tin: [panel][nb][nb]); tau_i = 0
// (H_i = I) drops reflector i.
__global__ void __launch_bounds__(QR_NBO)
    wy_t_kernel(const double *__restrict__ G, int w, const double *__restrict__ tin, int nb,
                double *__restrict__ T) {
  extern __shared__ double ti[];       // [w][w + 1]: T^-1 (upper), dropped rows = identity
  const int j = threadIdx.x;
  const int ld = w + 1;
  if (j < w) {
    const double tj = tin[(int64_t)(j / nb) * nb * nb + (j % nb) * nb + (j % nb)];
    for (int i = 0; i < w; ++i) {
      const double tau_i = tin[(int64_t)(i / nb) * nb * nb + (i % nb) * nb + (i % nb)];
      double v = 0.0;
      if (i == j) v = (tj != 0.0) ? 1.0 / tj : 1.0;
      else if (i < j && tj != 0.0 && tau_i != 0.0) v = G[(int64_t)i * w + j];
      ti[i * ld + j] = v;
    }
  }
  __syncthreads();
  if (j < w) {
    const double tj = tin[(int64_t)(j / nb) * nb * nb + (j % nb) * nb + (j % nb)];
    // column j of T: solve (T^-1) x = e_j, x_i = 0 for i > j
    double x[QR_NBO];
#pragma unroll 1
    for (int i = j; i >= 0; --i) {
      double acc = (i == j) ? 1.0 : 0.0;
#pragma unroll 1
      for (int k = i + 1; k <= j; ++k) acc -= ti[i * ld + k] * x[k];
      x[i] = acc / ti[i * ld + i];
    }
    if (tj == 0.0) x[j] = 0.0;   // dropped reflector
    for (int i = 0; i < w; ++i) T[(int64_t)i * w + j] = (i <= j) ? x[i] : 0.0;
  }
}

// Householder QR of row-major X (m x n) -> factored F (in workspace), V, T.
// Q (m x k) and/or R (k x n) formed on request.  k = min(m, n).  X is
// factored as 2^-e X (decomp_scale_exp); R is scaled back unless keep_scaled.
int qr_f64(int64_t m, int64_t n, const double *X, double *Q, double *R,
           int stabilized, double *ws, cudaStream_t st, bool keep_scaled) {
  QrGeom g;
  if (!qr_geometry(m, n, g)) {
    set_error("qb_qr_stab: m = %lld exceeds the register-panel limit 16384",
              (long long)m);
    return -2;
  }
  const int64_t k = std::min(m, n);
  const int nb = g.nb;
  double *F = ws + g.f_off, *V = ws + g.v_off, *T = ws + g.t_off, *TO = ws + g.to_off;
  double *G = ws + g.g_off;
  double *W = ws + g.w_off, *W2 = ws + g.w2_off;
  double *SK = ws + g.sk_off;
  const int64_t SKN = g.sk_elems;
  static bool attr_set = false;
  if (!attr_set) {
    QB_CUDA_CHECK(cudaFuncSetAttribute(wy_t_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                       QR_NBO * (QR_NBO + 1) * 8));
    attr_set = true;
  }
  const int blocks = sm_count() * 4;
  // F = 2^-e X: one max|X| pass decides e on the device (no host round trip)
  unsigned long long *maxbits = qr_maxbits(ws);
  QB_CUDA_CHECK(cudaMemsetAsync(maxbits, 0, sizeof(*maxbits), st));
  maxabs_bits_kernel<<<blocks, 256, 0, st>>>(X, m * n, maxbits);
  QB_LAUNCH_CHECK();
  scale_copy_kernel<<<blocks, 256, 0, st>>>(X, m * n, F, maxbits);
  QB_LAUNCH_CHECK();
  int rc;
  int64_t po = 0;
  const int64_t nbo = qr_outer_width(m, n, nb);
  for (int64_t j0 = 0; j0 < k; j0 += nbo, ++po) {
    const int w = (int)std::min<int64_t>(nbo, k - j0);   // outer panel width
    const int64_t mp = m - j0;
    double *Vo = V + j0 * m;            // (m - j0) x w slab, leading dimension w
    double *To = TO + j0 * QR_NBO;      // w x w, leading dimension w
    double *Ti = T + (j0 / nb) * nb * nb;     // inner T's of this outer panel (w / nb of them)
    QB_CUDA_CHECK(cudaMemsetAsync(Vo, 0, sizeof(double) * mp * w, st));
    for (int ji = 0; ji < w; ji += nb) {
      const int64_t col = j0 + ji;
      const int nbw = (int)std::min<int64_t>(nb, w - ji);
      const int mpi = (int)(m - col);
      double *Fp = F + col * n + col;
      double *Vp = Vo + (int64_t)ji * w + ji;   // rows from `col`, columns ji.., ld w
      double *Tp = Ti + (int64_t)(ji / nb) * nb * nb;
      switch (qr_panel_kind(nb, mpi)) {
        case 0: rc = launch_panel<32, 1>(Fp, n, mpi, nbw, Vp, w, Tp, st); break;
        case 1: rc = launch_panel<32, 2>(Fp, n, mpi, nbw, Vp, w, Tp, st); break;
        case 2: rc = launch_panel<16, 4>(Fp, n, mpi, nbw, Vp, w, Tp, st); break;
        default: rc = launch_panel<8, 8>(Fp, n, mpi, nbw, Vp, w, Tp, st); break;
      }
      if (rc) return rc;
      const int64_t nti = w - (ji + nbw);   // rest of the OUTER panel only
      if (nti > 0) {
        double *A2 = F + col * n + col + nbw;
        // W = Vp^T A2 (nbw x nti); W2 = Tp^T W; A2 -= Vp W2
        if ((rc = gemm_f64(Vp, 1, w, A2, n, 1, W, nti, 1, nbw, nti, mpi, 1.0, 0.0, st, SK, SKN, 16))) return rc;
        if ((rc = gemm_f64(Tp, 1, nb, W, nti, 1, W2, nti, 1, nbw, nti, nbw, 1.0, 0.0, st))) return rc;
        if ((rc = gemm_f64(Vp, w, 1, W2, nti, 1, A2, n, 1, mpi, nti, nbw, -1.0, 1.0, st))) return rc;
      }
    }
    if (w <= nb) {
      // a single inner panel: its own T (nb x nb, leading dimension nb) is the
      // outer T; copy the w x w block into the outer slot (leading dimension w)
      QB_CUDA_CHECK(cudaMemcpy2DAsync(To, sizeof(double) * w, Ti, sizeof(double) * nb,
                                      sizeof(double) * w, w, cudaMemcpyDeviceToDevice, st));
    } else {
      // compact WY form of the whole outer panel: G = Vo^T Vo, T from its inverse
      if ((rc = gemm_f64(Vo, 1, w, Vo, w, 1, G, w, 1, w, w, mp, 1.0, 0.0, st, SK, SKN, 16))) return rc;
      wy_t_kernel<<<1, QR_NBO, (size_t)w * (w + 1) * 8, st>>>(G, w, Ti, nb, To);
      QB_LAUNCH_CHECK();
    }
    const int64_t nt = n - (j0 + w);
    if (nt > 0) {
      double *C = F + j0 * n + j0 + w;
      // C <- (I - Vo To Vo^T)^T C = C - Vo (To^T (Vo^T C))
      if ((rc = gemm_f64(Vo, 1, w, C, n, 1, W, nt, 1, w, nt, mp, 1.0, 0.0, st, SK, SKN, 16))) return rc;
      if ((rc = gemm_f64(To, 1, w, W, nt, 1, W2, nt, 1, w, nt, w, 1.0, 0.0, st))) return rc;
      if ((rc = gemm_f64(Vo, w, 1, W2, nt, 1, C, n, 1, mp, nt, w, -1.0, 1.0, st))) return rc;
    }
  }
  if (R) {
    extract_r_kernel<<<blocks, 256, 0, st>>>(F, n, (int)k, (int)n, R,
                                             keep_scaled ? nullptr : maxbits);
    QB_LAUNCH_CHECK();
  }
  if (Q) {
    set_identity_kernel<<<blocks, 256, 0, st>>>(Q, m, k);
    QB_LAUNCH_CHECK();
    // Q = H_1 ... H_p [I; 0], outer panels applied last to first on Q[j0:, j0:]
    const int64_t nout = (k + nbo - 1) / nbo;
    for (int64_t pj = nout - 1; pj >= 0; --pj) {
      const int64_t j0 = pj * nbo;
      const int w = (int)std::min<int64_t>(nbo, k - j0);
      const int64_t mp = m - j0;
      const int64_t nq = k - j0;
      double *Vo = V + j0 * m, *To = TO + j0 * QR_NBO;
      double *Qs = Q + j0 * k + j0;
      if ((rc = gemm_f64(Vo, 1, w, Qs, k, 1, W, nq, 1, w, nq, mp, 1.0, 0.0, st, SK, SKN, 16))) return rc;
      if ((rc = gemm_f64(To, w, 1, W, nq, 1, W2, nq, 1, w, nq, w, 1.0, 0.0, st))) return rc;
      if ((rc = gemm_f64(Vo, w, 1, W2, nq, 1, Qs, k, 1, mp, nq, w, -1.0, 1.0, st))) return rc;
    }
  }
  if (stabilized && (Q || R)) {
    qr_phase_kernel<<<blocks, 256, 0, st>>>(Q, m, k, R, k, n, F, n);
    QB_LAUNCH_CHECK();
  }
  return 0;
}

int64_t qr_workspace_doubles(int64_t m, int64_t n) {
  QrGeom g;
  if (!qr_geometry(m, n, g)) return -1;
  return g.total;
}

}  // namespace qb

using namespace qb;

extern "C" {

int64_t qb_qr_workspace(int dtype, int64_t m, int64_t n) {
  if (dtype != QB_F64) return -1;
  QrGeom g;
  if (!qr_geometry(m, n, g)) return -2;
  return g.total * 8;
}

int qb_qr_route(int64_t m, int64_t n, int64_t *out) {
  QrRoute r;
  if (!qr_route(m, n, r)) {
    set_error("qb_qr_route: unsupported shape %lld x %lld", (long long)m, (long long)n);
    return -2;
  }
  out[0] = r.nb; out[1] = r.nbo; out[2] = r.nout; out[3] = r.panel_mask;
  out[4] = r.wy_t; out[5] = r.npan;
  return 0;
}

int qb_qr_stab(int dtype, int64_t m, int64_t n, const void *X, void *Q,
               void *R, int stabilized, void *workspace,
               size_t workspace_bytes, void *stream) {
  if (dtype != QB_F64) {
    set_error("qb_qr_stab: only f64 is implemented (got dtype %d)", dtype);
    return -1;
  }
  if (m <= 0 || n <= 0) return 0;
  int64_t need = qb_qr_workspace(dtype, m, n);
  if (need < 0) {
    set_error("qb_qr_stab: unsupported shape %lld x %lld", (long long)m, (long long)n);
    return -2;
  }
  if (!workspace || (int64_t)workspace_bytes < need) {
    set_error("qb_qr_stab: workspace too small (need %lld bytes)", (long long)need);
    return -8;
  }
  return qr_f64(m, n, (const double *)X, (double *)Q, (double *)R, stabilized,
                (double *)workspace, static_cast<cudaStream_t>(stream));
}

int qb_svals_to_keep(const double *s, int64_t n, double cutoff,
                     int cutoff_mode, int64_t max_bond, int renorm,
                     int64_t *n_keep, double *renorm_factor,
                     double *trunc_error) {
  if (!s || n <= 0) {
    set_error("qb_svals_to_keep: empty spectrum (n = %lld)", (long long)n);
    return -1;
  }
  if (cutoff_mode < 1 || cutoff_mode > 6) {
    set_error("invalid cutoff_mode %d", cutoff_mode);
    return -4;
  }
  int64_t n_chi = n;
  double f = 1.0, err = 0.0;
  if (cutoff > 0.0 || renorm > 0) {
    // decomp.py:901-937
    if (cutoff_mode == QB_CUTOFF_ABS) {
      n_chi = 0;
      for (int64_t i = 0; i < n; ++i) n_chi += s[i] > cutoff;
    } else if (cutoff_mode == QB_CUTOFF_REL) {
      n_chi = 0;
      for (int64_t i = 0; i < n; ++i) n_chi += s[i] > cutoff * s[0];
    } else {
      const int pw = (cutoff_mode == QB_CUTOFF_SUM2 || cutoff_mode == QB_CUTOFF_RSUM2) ? 2 : 1;
      double target = cutoff;
      if (cutoff_mode == QB_CUTOFF_RSUM2 || cutoff_mode == QB_CUTOFF_RSUM1) {
        double tot = 0.0;
        for (int64_t i = 0; i < n; ++i) tot += (pw == 2) ? s[i] * s[i] : s[i];
        target *= tot;
      }
      n_chi = n;
      double ssum = 0.0;
      for (int64_t i = n - 1; i >= 0; --i) {
        double s2 = (pw == 2) ? s[i] * s[i] : s[i];
        if (!isnan(s2)) ssum += s2;
        if (ssum > target) break;
        --n_chi;
      }
    }
    if (n_chi < 1) n_chi = 1;
    if (max_bond > 0 && n_chi > max_bond) n_chi = max_bond;
    if (n_chi < n) {
      for (int64_t i = n_chi; i < n; ++i) err += s[i] * s[i];
      err = sqrt(err);
      if (renorm > 0) {
        // decomp.py:940-965
        double keep = 0.0, lose = 0.0;
        for (int64_t i = 0; i < n; ++i) {
          double s2 = s[i];
          if (renorm >= 2) s2 = pow(s2, (double)renorm);
          if (!isnan(s2)) { if (i < n_chi) keep += s2; else lose += s2; }
        }
        f = (keep + lose) / keep;
        if (renorm >= 2) f = pow(f, 1.0 / renorm);
      }
    }
  } else if (max_bond != -1 && max_bond < n) {
    n_chi = max_bond;
    for (int64_t i = n_chi; i < n; ++i) err += s[i] * s[i];
    err = sqrt(err);
  }
  if (n_keep) *n_keep = n_chi;
  if (renorm_factor) *renorm_factor = f;
  if (trunc_error) *trunc_error = err;
  return 0;
}

}  // extern "C"

// =========================================================================
//                      one-sided block Jacobi SVD
// =========================================================================
namespace qb {

constexpr int JB = 16;          // columns per block
constexpr int JP = 2 * JB;      // columns per pair
constexpr int JCH = 64;         // rows per streamed chunk
constexpr int JPITCH = JP + 4;  // smem pitch (== 4 mod 16 doubles)

struct JacobiParams {
  double *W;       // rows_w x ld  working matrix (columns get orthogonalised)
  double *V;       // rows_v x ld  accumulated right rotations
  int64_t ld;
  int rows_w, rows_v;
  int nblk;        // number of column blocks (even)
  int round;       // 0 .. nblk-2
  double tol;
  int *flag;       // set to 1 when any pair still needed rotating
  int inner_max;   // max inner Jacobi sweeps per visit
  unsigned long long *trace;  // tuning (QB_TRACE): phase stamps of cluster 0
  int trace_slot;             // ring of 1024 rounds
};

__device__ __forceinline__ unsigned long long jac_ns() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}
#define JAC_TRACE(ph)                                                     \
  do {                                                                    \
    if (P.trace && blockIdx.x == 0 && threadIdx.x == 0)                   \
      P.trace[(size_t)P.trace_slot * 8 + (ph)] = jac_ns();             \
  } while (0)

__device__ __forceinline__ void rr_pair(int k, int round, int nblk, int &p, int &q) {
  // circle-method round robin over nblk players
  const int m = nblk - 1;
  int a, b;
  if (k == 0) { a = m; b = round; }
  else { a = (round + k) % m; b = (round - k + m) % m; }
  p = min(a, b); q = max(a, b);
}

__device__ __forceinline__ void jac_load_chunk(double (*Xs)[JPITCH], const double *M,
                                               int64_t ld, int rows, int row0,
                                               int cp, int cq, int tid) {
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int idx = tid + 256 * i;       // 1024 double2 per chunk
    const int r = idx >> 4, c2 = (idx & 15) * 2;
    const int gc = (c2 < JB) ? (cp + c2) : (cq + c2 - JB);
    const int gr = row0 + r;
    const bool ok = gr < rows;
    const double *src = ok ? (M + (int64_t)gr * ld + gc) : M;
    cp_async16(smem_u32(&Xs[r][c2]), src, ok ? 16 : 0);
  }
}

constexpr int JCSZ = 2;         // CTAs (one cluster) per column-block pair

// One round-robin round of the one-sided block Jacobi method.  A CLUSTER of
// JCSZ CTAs owns one pair of column blocks (2 x 16 columns); the rows of W
// and V are dealt round-robin (64-row chunks) to the CTAs of the cluster:
//   1. partial Gram of the 32 columns by DMMA from a 4-stage cp.async stream,
//      reduced over warps and then over the cluster through distributed
//      shared memory (fixed order: deterministic);
//   2. every CTA diagonalises the same 32 x 32 Gram by parallel-ordered
//      cyclic Jacobi (two-sided rotations fused into one pass over a
//      ping-pong copy of the Gram: one barrier per step), sorted descending;
//   3. the rotation is applied by DMMA to this CTA's rows of W and of V.
template <int JSTG>  // cp.async stages of the row-chunk stream
__global__ void __cluster_dims__(JCSZ, 1, 1) __launch_bounds__(256)
    jacobi_pair_kernel(const JacobiParams P) {
  namespace cg = cooperative_groups;
  cg::cluster_group cluster = cg::this_cluster();
  const int rank = (int)cluster.block_rank();
  extern __shared__ __align__(16) unsigned char jac_smem[];
  double(*Xs)[JCH][JPITCH] = reinterpret_cast<double(*)[JCH][JPITCH]>(jac_smem);
  __shared__ double Gbuf[2][JP][JP + 1];
  double(*G)[JP + 1] = Gbuf[0];   // current Gram; the eigen-solve ping-pongs
  double(*Gn)[JP + 1] = Gbuf[1];
  __shared__ double Gpart[JP][JP];
  __shared__ __align__(16) double Jm[JP][JPITCH];
  __shared__ double redmax[8];
  __shared__ int rank_s[JP];

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int g = lane >> 2, t = lane & 3;
  int bp, bq;
  rr_pair(blockIdx.x / JCSZ, P.round, P.nblk, bp, bq);
  const int cp = bp * JB, cq = bq * JB;

  JAC_TRACE(0);
  // ---------------- phase 1: partial Gram over this CTA's row chunks --------
  double acc[2][4][4];
#pragma unroll
  for (int i = 0; i < 2; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j)
#pragma unroll
      for (int v = 0; v < 4; ++v) acc[i][j][v] = 0.0;
  {
    const int nch_all = (P.rows_w + JCH - 1) / JCH;
    const int nmine = (nch_all - rank + JCSZ - 1) / JCSZ;  // chunks rank, rank+JCSZ, ...
    auto issue = [&](int i) {
      if (i < nmine)
        jac_load_chunk(Xs[i % JSTG], P.W, P.ld, P.rows_w, (rank + i * JCSZ) * JCH, cp, cq, tid);
      cp_async_commit();
    };
    for (int s = 0; s < JSTG - 1; ++s) issue(s);
    for (int i = 0; i < nmine; ++i) {
      cp_async_wait<JSTG - 2>();
      __syncthreads();
      issue(i + JSTG - 1);
      const double(*X)[JPITCH] = Xs[i % JSTG];
      const int kb = warp * 8;
      double af[2][4], bf[4][2];
#pragma unroll
      for (int a = 0; a < 2; ++a) {
        af[a][0] = X[kb + t][a * 16 + g];
        af[a][1] = X[kb + t][a * 16 + g + 8];
        af[a][2] = X[kb + t + 4][a * 16 + g];
        af[a][3] = X[kb + t + 4][a * 16 + g + 8];
      }
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        bf[j][0] = X[kb + t][j * 8 + g];
        bf[j][1] = X[kb + t + 4][j * 8 + g];
      }
      // the Gram is symmetric: the lower-left 16 x 16 block (a = 1, j < 2)
      // is the mirror of the upper-right one and is not computed
#pragma unroll
      for (int a = 0; a < 2; ++a)
#pragma unroll
        for (int j = 0; j < 4; ++j)
          if (a == 0 || j >= 2) dmma_16x8x8(acc[a][j], af[a], bf[j]);
    }
    cp_async_wait<0>();
    __syncthreads();
  }
  JAC_TRACE(1);
  // deterministic reduction over the 8 warps into Gpart: every warp parks its
  // fragment in the (now idle) stream buffers, one barrier, then each thread
  // sums four entries over the warps in a fixed order
  {
    double *scr = &Xs[0][0][0];  // 8 x 32 x 32 doubles <= JSTG * JCH * JPITCH
#pragma unroll
    for (int i = 0; i < 2; ++i)
#pragma unroll
      for (int j = 0; j < 4; ++j)
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int r = i * 16 + g + h * 8, c = j * 8 + 2 * t;
          *reinterpret_cast<double2 *>(&scr[(warp * JP + r) * JP + c]) =
              make_double2(acc[i][j][2 * h], acc[i][j][2 * h + 1]);
        }
    __syncthreads();
    for (int idx = tid; idx < JP * JP; idx += 256) {
      const int r = idx / JP, c = idx % JP;
      const int src = (r >= 16 && c < 16) ? (c * JP + r) : idx;  // mirrored block
      double sum = 0.0;
#pragma unroll
      for (int w = 0; w < 8; ++w) sum += scr[w * JP * JP + src];
      Gpart[r][c] = sum;
    }
  }
  cluster.sync();
  // full Gram = sum over the cluster (same order everywhere), symmetrised
  for (int idx = tid; idx < JP * JP; idx += 256) {
    const int r = idx / JP, c = idx % JP;
    double s = 0.0;
#pragma unroll
    for (int q = 0; q < JCSZ; ++q) {
      const double *gp = cluster.map_shared_rank(&Gpart[0][0], q);
      s += 0.5 * (gp[r * JP + c] + gp[c * JP + r]);
    }
    G[r][c] = s;
    Jm[r][c] = (r == c) ? 1.0 : 0.0;
  }
  __syncthreads();
  auto offmax = [&]() -> double {
    double mx = 0.0;
    for (int idx = tid; idx < JP * JP; idx += 256) {
      const int r = idx / JP, c = idx % JP;
      if (r < c) {
        const double d = G[r][r] * G[c][c];
        const double v = fabs(G[r][c]);
        if (d > 0.0) mx = fmax(mx, v / sqrt(d));
        else if (v > 0.0) mx = fmax(mx, 1.0);
      }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) mx = fmax(mx, __shfl_xor_sync(0xffffffffu, mx, o));
    if (lane == 0) redmax[warp] = mx;
    __syncthreads();
    double m2 = 0.0;
    for (int w = 0; w < 8; ++w) m2 = fmax(m2, redmax[w]);
    __syncthreads();
    return m2;
  };
  const double off0 = offmax();
  JAC_TRACE(2);
  // all CTAs of the cluster take the same decision (same G)
  if (off0 <= P.tol) {
    cluster.sync();  // peers may still be reading our Gpart
    return;
  }
  if (tid == 0 && rank == 0) atomicOr(P.flag, 1);

  // ---------------- phase 2: J^T G J = diag by cyclic Jacobi ----------------
  // inner sweeps: stop at round-off, or once this visit has reduced the
  // pair's off-diagonal mass by 1e-4 (at most 3 sweeps): block Jacobi
  // converges with inexact inner solves, and near convergence one sweep is
  // enough to reach round-off (quadratic convergence)
  for (int sweep = 0; sweep < P.inner_max; ++sweep) {
    if (sweep > 0) {
      const double off = offmax();
      if (off <= 1e-15 || off <= 1e-4 * off0) break;
    }
    for (int step = 0; step < JP - 1; ++step) {
      // One barrier per step: thread (k1, k2) owns the 2x2 block (rows of pair
      // k1) x (columns of pair k2).  The 16 rotations of the step are computed
      // once per warp (lanes 0-15, pinned arithmetic so that all warps get
      // bit-identical c, s) and handed out by shuffles; the rotated block goes
      // to the other Gram buffer; J <- J R for column pair k2, rows k1, k1+16.
      const int k1 = tid >> 4, k2 = tid & 15;
      int p1, q1, p2, q2;
      rr_pair(k1, step, JP, p1, q1);
      rr_pair(k2, step, JP, p2, q2);
      double c = 1.0, s = 0.0;
      if (lane < 16) {  // lane == k2 here
        const double app = G[p2][p2], aqq = G[q2][q2], apq = G[p2][q2];
        if (fabs(apq) > 1e-300) {
          // t = sgn(z) / (|z| + sqrt(1 + z^2)), z = (aqq - app) / (2 apq)
          const double a = __dsub_rn(aqq, app), b = __dmul_rn(2.0, apq);
          const double h = sqrt(__fma_rn(a, a, __dmul_rn(b, b)));
          const double tt = __ddiv_rn(copysign(fabs(b), __dmul_rn(a, b)), __dadd_rn(fabs(a), h));
          c = rsqrt(__fma_rn(tt, tt, 1.0));
          s = __dmul_rn(c, tt);
        }
      }
      const double c2 = __shfl_sync(0xffffffffu, c, k2), s2 = __shfl_sync(0xffffffffu, s, k2);
      const double c1 = __shfl_sync(0xffffffffu, c, k1), s1 = __shfl_sync(0xffffffffu, s, k1);
      {
        const double gpp = G[p1][p2], gpq = G[p1][q2], gqp = G[q1][p2], gqq = G[q1][q2];
        // columns first
        const double a0 = c2 * gpp - s2 * gpq, a1 = s2 * gpp + c2 * gpq;
        const double b0 = c2 * gqp - s2 * gqq, b1 = s2 * gqp + c2 * gqq;
        // then rows
        double n00 = c1 * a0 - s1 * b0, n01 = c1 * a1 - s1 * b1;
        double n10 = s1 * a0 + c1 * b0, n11 = s1 * a1 + c1 * b1;
        if (k1 == k2) { n01 = 0.0; n10 = 0.0; }  // the annihilated pair
        Gn[p1][p2] = n00; Gn[p1][q2] = n01; Gn[q1][p2] = n10; Gn[q1][q2] = n11;
#pragma unroll
        for (int it = 0; it < 2; ++it) {
          const int r = k1 + 16 * it;
          const double jp = Jm[r][p2], jq = Jm[r][q2];
          Jm[r][p2] = c2 * jp - s2 * jq;
          Jm[r][q2] = s2 * jp + c2 * jq;
        }
      }
      __syncthreads();
      { double(*tmp)[JP + 1] = G; G = Gn; Gn = tmp; }
    }
  }
  JAC_TRACE(3);
  // sort: larger column norms first (ties by index) -> new column order
  if (tid < JP) {
    const double d = G[tid][tid];
    int rk = 0;
    for (int j = 0; j < JP; ++j) {
      const double dj = G[j][j];
      rk += (dj > d) || (dj == d && j < tid);
    }
    rank_s[tid] = rk;
  }
  __syncthreads();
  for (int idx = tid; idx < JP * JP; idx += 256) {
    const int r = idx / JP, c = idx % JP;
    G[r][rank_s[c]] = Jm[r][c];
  }
  __syncthreads();
  for (int idx = tid; idx < JP * JP; idx += 256) {
    const int r = idx / JP, c = idx % JP;
    Jm[r][c] = G[r][c];
  }
  __syncthreads();

  JAC_TRACE(4);
  // ---------------- phase 3: apply J to this CTA's rows of W and V ----------
  {
    const int nchw = (P.rows_w + JCH - 1) / JCH, nchv = (P.rows_v + JCH - 1) / JCH;
    const int ntot = nchw + nchv;
    const int nmine = (ntot - rank + JCSZ - 1) / JCSZ;
    auto chunk_src = [&](int i, double *&M, int &rows, int &row0) {
      const int ch = rank + i * JCSZ;
      if (ch < nchw) { M = P.W; rows = P.rows_w; row0 = ch * JCH; }
      else { M = P.V; rows = P.rows_v; row0 = (ch - nchw) * JCH; }
    };
    auto issue = [&](int i) {
      if (i < nmine) {
        double *M; int rows, row0;
        chunk_src(i, M, rows, row0);
        jac_load_chunk(Xs[i % JSTG], M, P.ld, rows, row0, cp, cq, tid);
      }
      cp_async_commit();
    };
    for (int s = 0; s < JSTG - 1; ++s) issue(s);
    const int mt = warp & 3, nh = warp >> 2;  // 16 rows x 16 cols per warp
    for (int i = 0; i < nmine; ++i) {
      cp_async_wait<JSTG - 2>();
      __syncthreads();
      issue(i + JSTG - 1);
      double *M; int rows, row0;
      chunk_src(i, M, rows, row0);
      const double(*X)[JPITCH] = Xs[i % JSTG];
      double c2[2][4];
#pragma unroll
      for (int j = 0; j < 2; ++j)
#pragma unroll
        for (int v = 0; v < 4; ++v) c2[j][v] = 0.0;
#pragma unroll
      for (int kk = 0; kk < JP; kk += 8) {
        double af[4], bf[2][2];
        af[0] = X[mt * 16 + g][kk + t];
        af[1] = X[mt * 16 + g + 8][kk + t];
        af[2] = X[mt * 16 + g][kk + t + 4];
        af[3] = X[mt * 16 + g + 8][kk + t + 4];
#pragma unroll
        for (int j = 0; j < 2; ++j) {
          bf[j][0] = Jm[kk + t][nh * 16 + j * 8 + g];
          bf[j][1] = Jm[kk + t + 4][nh * 16 + j * 8 + g];
        }
#pragma unroll
        for (int j = 0; j < 2; ++j) dmma_16x8x8(c2[j], af, bf[j]);
      }
#pragma unroll
      for (int j = 0; j < 2; ++j)
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int r = row0 + mt * 16 + g + h * 8;
          const int c = nh * 16 + j * 8 + 2 * t;  // column within the pair
          if (r < rows) {
            const int gc = (c < JB) ? (cp + c) : (cq + c - JB);
            *reinterpret_cast<double2 *>(M + (int64_t)r * P.ld + gc) =
                make_double2(c2[j][2 * h], c2[j][2 * h + 1]);
          }
        }
    }
    cp_async_wait<0>();
  }
  JAC_TRACE(5);
  cluster.sync();  // nobody exits while peers may read its shared memory
  JAC_TRACE(6);
}

// column norms of W (rows x ld, first ncols columns)
__global__ void __launch_bounds__(256)
    colnorm_kernel(const double *__restrict__ W, int64_t ld, int rows, int ncols,
                   double *__restrict__ out) {
  // one warp per 32 columns chunk-row: simple and coalesced: block handles
  // 32 columns, threads (32 x 8) walk rows
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

// U_R[:, k] = W[:, perm[k]] / s[perm[k]]   (n x nk, row-major), and
// VH[k, :] = V[:, perm[k]]^T  (nk x ncols_v rows of V)
__global__ void __launch_bounds__(256)
    svd_gather_kernel(const double *__restrict__ W, const double *__restrict__ V,
                      int64_t ld, int rows_w, int rows_v, int nk,
                      const int *__restrict__ perm, const double *__restrict__ s,
                      double *__restrict__ UR, double *__restrict__ VH) {
  const int64_t tot_u = (int64_t)rows_w * nk, tot_v = (int64_t)nk * rows_v;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < tot_u + tot_v;
       i += (int64_t)gridDim.x * blockDim.x) {
    if (i < tot_u) {
      const int64_t r = i / nk;
      const int k = (int)(i - r * nk);
      const int c = perm[k];
      // W = R^T was orthogonalised: R = Z S Y^T with Z the accumulated
      // rotations (-> U_R) and Y the normalised columns of W (-> V)
      UR[i] = V[r * ld + c];
    } else {
      const int64_t j = i - tot_u;
      const int k = (int)(j / rows_v);
      const int64_t r = j - (int64_t)k * rows_v;
      const int c = perm[k];
      const double sv = s[c];
      VH[j] = (sv > 0.0) ? W[r * ld + c] / sv : 0.0;
    }
  }
}

__global__ void pad_copy_kernel(const double *__restrict__ src, int64_t rows,
                                int64_t cols, int64_t ld_src, double *__restrict__ dst,
                                int64_t ld_dst, int64_t rows_dst, int identity) {
  // dst (rows_dst x ld_dst) = [src | 0] (or the identity when src == null)
  const int64_t tot = rows_dst * ld_dst;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < tot;
       i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t r = i / ld_dst, c = i - r * ld_dst;
    double v = 0.0;
    if (identity == 1) v = (r == c) ? 1.0 : 0.0;
    else if (r < rows && c < cols)
      v = (identity == 2) ? src[c * ld_src + r] : src[r * ld_src + c];  // 2: transposed
    dst[i] = v;
  }
}

struct SvdGeom {
  int64_t npad, qr_off, q1_off, r_off, w_off, v_off, s_off, ur_off, perm_off,
      flag_off, xt_off, total;
};

static bool svd_geometry(int64_t m, int64_t n, SvdGeom &g) {
  // m >= n here
  QrGeom q;
  if (!qr_geometry(m, n, q)) return false;
  g.npad = ((n + JP - 1) / JP) * JP;
  auto al = [](int64_t x) { return (x + 31) / 32 * 32; };  // 256-byte sections
  int64_t off = 0;
  g.qr_off = off; off += al(q.total);
  g.q1_off = off; off += al(m * n);
  g.r_off = off; off += al(n * n);
  g.w_off = off; off += al(n * g.npad);
  g.v_off = off; off += al(g.npad * g.npad);
  g.s_off = off; off += al(g.npad);
  g.ur_off = off; off += al(n * n);
  g.perm_off = off; off += al((g.npad + 1) / 2 + 1);   // ints
  g.flag_off = off; off += 32;
  g.xt_off = off; off += 0;
  g.total = off;
  return true;
}

// SVD of row-major X (m x n), m >= n.  U (m x n), S (n), VH (n x n).
int svd_tall_f64_v1(int64_t m, int64_t n, const double *X, double *U,
                        double *S, double *VH, double *ws, int *sweeps_out,
                        cudaStream_t st) {
  SvdGeom g;
  if (!svd_geometry(m, n, g)) {
    set_error("qb_svd: unsupported shape %lld x %lld", (long long)m, (long long)n);
    return -2;
  }
  double *Q1 = ws + g.q1_off, *R = ws + g.r_off, *W = ws + g.w_off;
  double *V = ws + g.v_off, *sv = ws + g.s_off, *UR = ws + g.ur_off;
  int *perm = reinterpret_cast<int *>(ws + g.perm_off);
  int *flag = reinterpret_cast<int *>(ws + g.flag_off);
  const int blocks = sm_count() * 4;
  int rc = qr_f64(m, n, X, Q1, R, /*stabilized=*/0, ws + g.qr_off, st);
  if (rc) return rc;
  const int64_t npad = g.npad;
  pad_copy_kernel<<<blocks, 256, 0, st>>>(R, n, n, n, W, npad, n, 2);  // W = R^T
  QB_LAUNCH_CHECK();
  pad_copy_kernel<<<blocks, 256, 0, st>>>(nullptr, 0, 0, 0, V, npad, npad, 1);
  QB_LAUNCH_CHECK();
  // stream depth (QB_JAC_STAGES: 4, 8 or 10): measured identical -- the row
  // streams are bound by the DMMA rate (64 rows x 32 x 32 FMAs per chunk =
  // 1024 pipe clocks per SM), not by bytes in flight
  static const int jstg = [] {
    const char *e = getenv("QB_JAC_STAGES");
    const int v = e ? atoi(e) : 4;
    return v <= 4 ? 4 : (v <= 8 ? 8 : 10);
  }();
  const int kJacSmem = jstg * JCH * JPITCH * 8;
  static bool attr_set = false;
  if (!attr_set) {
    QB_CUDA_CHECK(cudaFuncSetAttribute(jacobi_pair_kernel<4>,
                                       cudaFuncAttributeMaxDynamicSharedMemorySize,
                                       4 * JCH * JPITCH * 8));
    QB_CUDA_CHECK(cudaFuncSetAttribute(jacobi_pair_kernel<8>,
                                       cudaFuncAttributeMaxDynamicSharedMemorySize,
                                       8 * JCH * JPITCH * 8));
    QB_CUDA_CHECK(cudaFuncSetAttribute(jacobi_pair_kernel<10>,
                                       cudaFuncAttributeMaxDynamicSharedMemorySize,
                                       10 * JCH * JPITCH * 8));
    attr_set = true;
  }
  JacobiParams P;
  P.W = W; P.V = V; P.ld = npad; P.rows_w = (int)n; P.rows_v = (int)npad;
  P.nblk = (int)(npad / JB);
  P.tol = 1e-15 * sqrt((double)n) * 8.0;
  P.flag = flag;
  P.trace = trace_buffer() ? trace_buffer() + 16 * 8192 : nullptr;
  {
    static const int inner = [] { const char *e = getenv("QB_JAC_INNER"); return e ? atoi(e) : 1; }();
    P.inner_max = inner;
  }
  int sweeps = 0;
  const int max_sweeps = 60;
  const int inner0 = P.inner_max;
  for (; sweeps < max_sweeps; ++sweeps) {
    // one inner sweep per visit is fastest; fall back to fuller inner solves
    // if the outer iteration is unusually slow
    P.inner_max = (sweeps < 25) ? inner0 : std::max(inner0, 4);
    QB_CUDA_CHECK(cudaMemsetAsync(flag, 0, sizeof(int), st));
    for (int r = 0; r < P.nblk - 1; ++r) {
      P.round = r;
      P.trace_slot = (sweeps * (P.nblk - 1) + r) & 1023;
      const unsigned grid = (unsigned)(P.nblk / 2) * JCSZ;
      if (jstg == 4) jacobi_pair_kernel<4><<<grid, 256, kJacSmem, st>>>(P);
      else if (jstg == 8) jacobi_pair_kernel<8><<<grid, 256, kJacSmem, st>>>(P);
      else jacobi_pair_kernel<10><<<grid, 256, kJacSmem, st>>>(P);
      QB_LAUNCH_CHECK();
    }
    int h = 0;
    QB_CUDA_CHECK(cudaMemcpyAsync(&h, flag, sizeof(int), cudaMemcpyDeviceToHost, st));
    QB_CUDA_CHECK(cudaStreamSynchronize(st));
    if (!h) break;
  }
  if (sweeps_out) *sweeps_out = sweeps;
  if (sweeps >= max_sweeps) {
    set_error("qb_svd: Jacobi did not converge in %d sweeps", max_sweeps);
    return 2;
  }
  colnorm_kernel<<<(unsigned)(npad / 32), 256, 0, st>>>(W, npad, (int)n, (int)npad, sv);
  QB_LAUNCH_CHECK();
  std::vector<double> hs(npad);
  QB_CUDA_CHECK(cudaMemcpyAsync(hs.data(), sv, sizeof(double) * npad,
                                cudaMemcpyDeviceToHost, st));
  QB_CUDA_CHECK(cudaStreamSynchronize(st));
  std::vector<int> hp(npad);
  for (int i = 0; i < npad; ++i) hp[i] = i;
  std::stable_sort(hp.begin(), hp.end(), [&](int a, int b) {
    const bool pa = a >= n, pb = b >= n;  // padding columns last
    if (pa != pb) return pb;
    return hs[a] > hs[b];
  });
  QB_CUDA_CHECK(cudaMemcpyAsync(perm, hp.data(), sizeof(int) * n,
                                cudaMemcpyHostToDevice, st));
  // sorted singular values
  std::vector<double> ss(n);
  for (int i = 0; i < n; ++i) ss[i] = hs[hp[i]];
  if (S) QB_CUDA_CHECK(cudaMemcpyAsync(S, ss.data(), sizeof(double) * n,
                                       cudaMemcpyHostToDevice, st));
  // U_R, VH (VH rows: the first n rows of V only -- the rest is padding)
  svd_gather_kernel<<<blocks, 256, 0, st>>>(W, V, npad, (int)n, (int)n, (int)n,
                                            perm, sv, UR, VH ? VH : UR);
  QB_LAUNCH_CHECK();
  QB_CUDA_CHECK(cudaStreamSynchronize(st));  // host vectors go out of scope
  if (U) {
    rc = gemm_f64(Q1, n, 1, UR, n, 1, U, n, 1, m, n, n, 1.0, 0.0, st);
    if (rc) return rc;
  }
  return 0;
}

int64_t svd_v1_workspace_doubles(int64_t m, int64_t n) {
  SvdGeom g;
  if (!svd_geometry(m, n, g)) return -1;
  return g.total;
}

}  // namespace qb
