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
//   qb_svals_to_keep <- _compute_number_svals_to_keep_numba + renorm factor
//                  (decomp.py:901-965), host side, bit-for-bit the same
//                  summation order as the reference.
// The SVD (qb_svd, qb_svd_trunc) is in svd_jacobi.cu.
#include <cooperative_groups.h>
#include <math.h>

#include <algorithm>

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
