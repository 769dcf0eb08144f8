/*
 * quimb_b200 -- C ABI of the H100-native tensor-network contraction engine.
 *
 * This header is the drop-in boundary.  Every entry point replaces one
 * library call that quimb's hot path bottoms out in (all reference citations
 * are relative to the quimb source tree):
 *
 *   qb_contract_pair      <- autoray do("tensordot") / do("einsum") issued by the
 *                            cotengra pairwise loop under
 *                            quimb/tensor/contraction.py:272-292 (array_contract)
 *                            and by Tensor.__matmul__, quimb/tensor/tensor_core.py:3786-3808
 *   qb_permute            <- do("transpose")+do("reshape") materialisation in
 *                            quimb/tensor/array_ops.py:148-180 (fuse)
 *   qb_svd_trunc          <- svd_truncated incl. the keep rule, renormalisation
 *                            and absorb, quimb/tensor/decomp.py:829-1118, :901-1029,
 *                            :693-721 (qb_svd + qb_svals_to_keep are its parts)
 *   qb_qr_stab            <- qr_stabilized, quimb/tensor/decomp.py:2055-2216
 *   qb_dot / qb_axpby / qb_scale / qb_multi_dot / qb_multi_axpy
 *                         <- ARPACK dsaupd vector algebra behind
 *                            quimb/linalg/scipy_linalg.py:113-128 (eigs_scipy);
 *                            the Krylov control loop itself is host Python
 *                            (quimb_b200/lanczos.py) -- there is no qb_lanczos_*
 *                            and no plan_create/execute/destroy entry: cached
 *                            chains are CUDA graphs captured by the host layer
 *   qb_sample_select      <- the per-site probability / choice / projection of
 *                            MatrixProductState.sample_configuration,
 *                            quimb/tensor/tn1d/core.py:3871-3990, for a whole
 *                            batch of samples at once
 *   qb_rdm_reduce         <- the final contraction of
 *                            MatrixProductState.partial_trace_to_dense_canonical
 *                            and of the local expectations, core.py:2827-3087
 *   qb_plaquette_expec    <- the per-term contractions of
 *                            PEPS.compute_local_expectation,
 *                            quimb/tensor/tn2d/core.py:4335-4348
 *   qb_sketch_env         <- the noise-sketched left environments of
 *                            tensor_network_1d_compress_src,
 *                            quimb/tensor/tn1d/compress.py:1787-1826
 *
 * Conventions
 *   - plain C, no C++/torch types; device pointers are borrowed, never freed
 *     or retained by the library beyond the call.
 *   - all strides are in ELEMENTS (not bytes) and may describe any
 *     non-overlapping strided view (torch.Tensor.stride()).
 *   - `stream` is a cudaStream_t passed as void* (0 = legacy default stream).
 *   - return value: 0 = success; <0 = invalid argument (-(index+1));
 *     >0 = CUDA / numerical failure.  qb_last_error() gives a message.
 *   - thread safety: no global mutable state except the thread-local error
 *     string; calls on different streams may run concurrently.
 */
#ifndef QUIMB_B200_H
#define QUIMB_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define QB_MAX_RANK 32
#define QB_ABI_VERSION 1

typedef enum {
  QB_F32 = 0,
  QB_F64 = 1,
  QB_C64 = 2,
  QB_C128 = 3
} qb_dtype_t;

/* A strided device tensor view (mirrors what quimb keeps in Tensor._data). */
typedef struct {
  void *ptr;
  int32_t dtype; /* qb_dtype_t */
  int32_t rank;
  int64_t shape[QB_MAX_RANK];
  int64_t stride[QB_MAX_RANK]; /* elements */
} qb_tensor_t;

/* quimb's absorb codes, decomp.py:201-211 (QB_ABSORB_FULL stands for None). */
enum {
  QB_ABSORB_FULL = 100, /* 'U,s,VH' : return the three parts */
  QB_ABSORB_S = 2,      /* 's' */
  QB_ABSORB_LSQRT = -12,
  QB_ABSORB_RORTHOG = -11,
  QB_ABSORB_LFACTOR = -10,
  QB_ABSORB_LEFT = -1,
  QB_ABSORB_BOTH = 0,
  QB_ABSORB_RIGHT = 1,
  QB_ABSORB_LORTHOG = 10,
  QB_ABSORB_RFACTOR = 11,
  QB_ABSORB_RSQRT = 12
};

/* quimb's cutoff modes, decomp.py:265-270 */
enum {
  QB_CUTOFF_ABS = 1,
  QB_CUTOFF_REL = 2,
  QB_CUTOFF_SUM2 = 3,
  QB_CUTOFF_RSUM2 = 4,
  QB_CUTOFF_SUM1 = 5,
  QB_CUTOFF_RSUM1 = 6
};

/* contraction engine selection for qb_contract_pair */
enum {
  QB_ENGINE_AUTO = 0, /* heuristic                                    */
  QB_ENGINE_DMMA = 1, /* native fp64 tensor-core path (DMMA)          */
  QB_ENGINE_OZAKI = 2, /* int8 tensor-core (wgmma) error-free-split path */
  QB_ENGINE_STREAM = 3, /* HBM-bound streaming path for small-operator
                         * steps (after mode grouping N, K <= 32 for f64,
                         * N, K <= 16 for c128: gate application); other
                         * shapes take the DMMA path.  Opt-in: not timed
                         * on the H100.                                 */
  /* OR-able flag: the caller guarantees that bytes [0, 1024) of `workspace`
   * (the stream-K flag words) were zero before its first use and are written
   * by this library only -- which always leaves them zero again -- so the
   * per-launch clear of those words is skipped (saves one memset node per
   * contraction; matters for back-to-back launches and CUDA graphs). */
  QB_ENGINE_WS_ZEROED = 0x100
};

/* ---- library ---------------------------------------------------------- */
int qb_abi_version(void);
const char *qb_last_error(void);
/* number of kernels launched by this library in this process (monotonic) */
int64_t qb_launch_count(void);

/* ---- pairwise contraction --------------------------------------------- */
/*
 * C[labelsC] = sum over labels not in C of  op(A)[labelsA] * op(B)[labelsB]
 *
 * Labels are arbitrary int32 mode names (the integer image of quimb's index
 * names).  A label in A and B but not C is contracted; in A, B and C it is a
 * batch ("hyper") index; in only one input and not C it is summed over; a
 * label repeated inside one input takes that input's diagonal.  Every label
 * of C must appear in A or B.  No operand is transposed or copied: the index
 * permutation is folded into the kernel's tile loads / stores.
 * conjA / conjB conjugate complex inputs on load.
 * workspace may be NULL when qb_contract_pair_workspace() returns 0.
 */
int qb_contract_pair(const qb_tensor_t *A, const int32_t *labelsA,
                     const qb_tensor_t *B, const int32_t *labelsB,
                     qb_tensor_t *C, const int32_t *labelsC, int conjA,
                     int conjB, int engine, void *workspace,
                     size_t workspace_bytes, void *stream);

/* as qb_contract_pair, but C = alpha * op(A).op(B) + beta * C (real scalars;
 * beta != 0 accumulates into the existing contents of C).  This is the
 * building block of the Lanczos orthogonalisation and of the blocked
 * Householder updates. */
int qb_contract_pair_ab(const qb_tensor_t *A, const int32_t *labelsA,
                        const qb_tensor_t *B, const int32_t *labelsB,
                        qb_tensor_t *C, const int32_t *labelsC, int conjA,
                        int conjB, double alpha, double beta, void *workspace,
                        size_t workspace_bytes, void *stream);

int64_t qb_contract_pair_workspace(const qb_tensor_t *A,
                                   const int32_t *labelsA,
                                   const qb_tensor_t *B,
                                   const int32_t *labelsB, const qb_tensor_t *C,
                                   const int32_t *labelsC, int engine);

/*
 * Host-only: run the planner and report the GEMM view it derived.
 * out[0..7] = M, N, K, batch, n_m_modes, n_n_modes, n_k_modes, n_batch_modes
 * out[8] = tile config id, out[9] = split-k factor, out[10] = vecA,
 * out[11] = vecB, out[12] = vecC.  Needs no GPU; used by the CPU test-suite.
 */
int qb_contract_pair_plan(const qb_tensor_t *A, const int32_t *labelsA,
                          const qb_tensor_t *B, const int32_t *labelsB,
                          const qb_tensor_t *C, const int32_t *labelsC,
                          int64_t *out16);

/*
 * Host-only: the kernel route qb_contract_pair takes for these operands and
 * this engine argument (given a large enough workspace).  The launch path
 * and this report come from the same decision function.
 * out[0] = route kind: 0 empty output, 1 zero fill, 2 widen (single
 *          precision below the int8 engine's minimum: the caller widens),
 *          3 int8 engine, 4 streaming engine, 5 DMMA classic grid,
 *          6 DMMA stream-K grid
 * out[1] = DMMA tile config (-1 otherwise), out[2] = split-K factor,
 * out[3] = stream-K grid (CTAs, 0 otherwise), out[4] = stream-K head cost
 * (k-blocks), out[5] = DMMA k-block depth, out[6] = cfg-0 shared-memory
 * layout of real operands (a_kmajor * 2 + b_kmajor; -1: runtime layout),
 * out[7] = SM count the planner used, out[8] = kernels launched (beta = 0),
 * out[9] / out[10] = compiled (KMAX, NMAX) variant of the streaming engine
 * (0 for every other route).  The caller provides 16 slots.
 */
int qb_contract_pair_route(const qb_tensor_t *A, const int32_t *labelsA,
                           const qb_tensor_t *B, const int32_t *labelsB,
                           const qb_tensor_t *C, const int32_t *labelsC,
                           int engine, int64_t *out16);

/*
 * Host-only: how the route of qb_contract_pair_route (engine = auto) feeds
 * each operand into the DMMA large real tile.  out[0] / out[1] = feed of A /
 * B: 1 affine (a per-thread address advanced by constant steps), 0 offset
 * tables, -1 the route does not run the large real tile.
 */
int qb_contract_pair_feed(const qb_tensor_t *A, const int32_t *labelsA,
                          const qb_tensor_t *B, const int32_t *labelsB,
                          const qb_tensor_t *C, const int32_t *labelsC,
                          int64_t *out2);

/*
 * Host-only: how the stream-K grid of qb_contract_pair_route (engine = auto)
 * splits its work.  out[0] = 1 pair schedule (2-CTA clusters, one per tile,
 * each CTA one k-half, summed in distributed shared memory), 0 the segment
 * loop (equal-cost k-block ranges, partial tiles summed through the
 * workspace), -1 the route is not stream-K.  Without a device it assumes
 * that half the planner's grid can run as clusters at once.
 */
int qb_contract_pair_schedule(const qb_tensor_t *A, const int32_t *labelsA,
                              const qb_tensor_t *B, const int32_t *labelsB,
                              const qb_tensor_t *C, const int32_t *labelsC,
                              int64_t *out1);

/*
 * TEST / debug entry, host pointers only: runs the streaming engine's row
 * code (shared __host__ __device__ functions of contract_stream.cu) in a
 * host loop so that its index bookkeeping can be checked without a device.
 * Never called by the product; returns -9 for shapes the engine does not take.
 */
int qb_debug_contract_stream_host(const qb_tensor_t *A, const int32_t *labelsA,
                                  const qb_tensor_t *B, const int32_t *labelsB,
                                  qb_tensor_t *C, const int32_t *labelsC,
                                  int conjA, int conjB, double alpha,
                                  double beta);

/*
 * Many independent same-signature contractions in one launch: A[i], B[i], C[i]
 * share shape/stride/labels (taken from A0/B0/C0) but have their own base
 * pointers given in device arrays of `count` pointers.
 */
int qb_contract_batched(const qb_tensor_t *A0, const int32_t *labelsA,
                        const qb_tensor_t *B0, const int32_t *labelsB,
                        qb_tensor_t *C0, const int32_t *labelsC,
                        const void *const *dA, const void *const *dB,
                        void *const *dC, int64_t count, int conjA, int conjB,
                        void *stream);

/* ---- layout / element-wise -------------------------------------------- */
/* dst (any strides) = src (any strides), same shape; optional conjugation */
int qb_permute(const qb_tensor_t *src, qb_tensor_t *dst, int conj,
               void *stream);
/* y = alpha * x + beta * y over n contiguous elements (alpha,beta: re,im);
 * beta = 0 does not read y, so y may hold NaN / Inf or be uninitialised */
int qb_axpby(int dtype, int64_t n, const double alpha[2], const void *x,
             const double beta[2], void *y, void *stream);
/* x *= alpha / (*dev_scalar)  (dev_scalar may be NULL); Lanczos normalise */
int qb_scale(int dtype, int64_t n, const double alpha[2],
             const void *dev_div_scalar, void *x, void *stream);
/* y = x * alpha / (*dev_div_scalar) (divisor optional; zero divisor -> zeros):
 * the normalised copy of a Krylov residual in one pass. */
int qb_scale_into(int dtype, int64_t n, double alpha, const void *dev_div_scalar,
                  const void *x, void *y, void *stream);
/* out[0] (device, same dtype as x; complex: conj(x).y) = <x|y>; deterministic
 * two-stage reduction; workspace >= qb_dot_workspace(n) bytes */
int qb_dot(int dtype, int64_t n, const void *x, const void *y, void *out,
           void *workspace, void *stream);
int64_t qb_dot_workspace(int64_t n);
/* Krylov block algebra (one pass over V each; f64): V is m x n row-major with
 * leading dimension ldv, m <= 16.
 *   qb_multi_dot :  out[j] = <V[j], w>            (device out, deterministic)
 *   qb_multi_axpy:  w += alpha * sum_j h[j] V[j]  (h on the device)
 * Together: one classical Gram-Schmidt pass of the Lanczos vector w. */
int qb_multi_dot(int dtype, int m, int64_t n, const void *V, int64_t ldv,
                 const void *w, void *out, void *workspace, void *stream);
int64_t qb_multi_dot_workspace(void);
int qb_multi_axpy(int dtype, int m, int64_t n, const void *V, int64_t ldv,
                  const void *h, double alpha, void *w, void *stream);
/* x (rows x cols, row-major contiguous) *= d[col]^p  (side=1) or d[row]^p
 * (side=0); p in {1, 0.5}; d is real (f32 for F32/C64, f64 otherwise) */
int qb_scale_diag(int dtype, int64_t rows, int64_t cols, void *x,
                  const void *d, int side, int sqrt_d, void *stream);

/* contiguous precision conversion f32<->f64, c64<->c128 (n elements).  f32 /
 * c64 operands are widened (exactly) for the fp64 engines and the result is
 * rounded once. */
int qb_convert(int src_dtype, int dst_dtype, int64_t n, const void *src,
               void *dst, void *stream);

/* complex128 <-> interleaved real embedding E[2i+a, 2j+b] (row-major
 * 2m x 2n): complex QR / SVD run on the real kernels through it.
 * qb_extract_complex: out[i, c] = E[2i, c*col_step] + 1j E[2i+1, c*col_step]. */
int qb_embed_complex(int64_t m, int64_t n, const void *z, void *E, void *stream);
int qb_extract_complex(int64_t m, int64_t ncols, int64_t col_step, const void *E,
                       int64_t ld, void *out, void *stream);

/* ---- decompositions ---------------------------------------------------- */
/*
 * Stabilised thin QR of a row-major contiguous m x n matrix X (m >= n):
 * Q (m x n, row-major), R (n x n, row-major, upper triangular, diag >= 0).
 * Either output may be NULL.  decomp.py:2055-2216.
 */
int qb_qr_stab(int dtype, int64_t m, int64_t n, const void *X, void *Q,
               void *R, int stabilized, void *workspace,
               size_t workspace_bytes, void *stream);
int64_t qb_qr_workspace(int dtype, int64_t m, int64_t n);
/* Host only: the kernels qb_qr_stab launches for an m x n matrix, from the
 * decisions of the launch path.  out[0] = inner panel width, out[1] = outer
 * (aggregated) panel width, out[2] = outer panels, out[3] = bitmask of the
 * panel instantiations launched (bit 0: (32 columns, 1 row per thread),
 * 1: (32, 2), 2: (16, 4), 3: (8, 8)), out[4] = 1 when wy_t_kernel forms the
 * aggregated T factors, out[5] = inner panels.  The caller provides 16 slots.
 * qb_qr_stab and the SVD factor 2^-e X when max|X| lies outside
 * [2^-200, 2^200] (e = ilogb(max|X|)) and scale the results back. */
int qb_qr_route(int64_t m, int64_t n, int64_t *out16);

/*
 * Thin SVD of a row-major contiguous m x n matrix X by one-sided block
 * Jacobi: U (m x k), S (k, real, descending), VH (k x n), k = min(m, n).
 * sweeps_out / offnorm_out (host) report convergence.
 */
int qb_svd(int dtype, int64_t m, int64_t n, const void *X, void *U, void *S,
           void *VH, void *workspace, size_t workspace_bytes,
           int *sweeps_out, void *stream);
int64_t qb_svd_workspace(int dtype, int64_t m, int64_t n);

/*
 * Truncated SVD with the reference's epilogue fused in: svd_truncated,
 * quimb/tensor/decomp.py:829-898 with the keep rule
 * _compute_number_svals_to_keep (:901-937; cutoff_mode 1..6 = QB_CUTOFF_*,
 * cutoff <= 0 and renorm == 0: only max_bond applies, max_bond = -1: none),
 * _compute_svals_renorm_factor (:940-965), the trim (:968-1029) and
 * _do_absorb (:693-721; `absorb` = QB_ABSORB_*).  X is row-major m x n with
 * m >= n (the host layer passes the transpose of a wide matrix and swaps the
 * roles of the factors).  Only the kept rank k = *n_keep is written, compactly:
 * U as m x k (leading dimension k), S as k values (renormalised), VH as
 * k x n; factors the absorb mode does not request are not touched and may be
 * NULL.  The caller provides room for k = n.  *trunc_error = sqrt(sum of the
 * discarded s^2) (info["error"]); *n_null = number of kept singular values
 * that are exactly zero (their rows of VH are zero: complete them if an
 * isometry is needed).  Workspace: qb_svd_workspace(dtype, m, n) bytes.
 */
/* TEST / debug entry, host only: the sweep schedule of the Jacobi SVD (which
 * column-block pairs rotate in which round of which stream); five int32 per
 * pair: phase, group, round, p, q.  Returns the number of pairs. */
int64_t qb_debug_jacobi_schedule(int nblk, int groups, int32_t *out,
                                 int64_t capacity, int *groups_used);

int qb_svd_trunc(int dtype, int64_t m, int64_t n, const void *X, double cutoff,
                 int cutoff_mode, int64_t max_bond, int absorb, int renorm,
                 void *U, void *S, void *VH, int64_t *n_keep,
                 double *trunc_error, int64_t *n_null, void *workspace,
                 size_t workspace_bytes, int *sweeps_out, void *stream);
/* qb_svd / qb_svd_trunc return -9 (before any Jacobi sweep) when X holds a
 * NaN or an infinity. */

/* Host only: what qb_svd_trunc launches for a tall m x n matrix (m >= n) and
 * absorb mode (qb_svd: QB_ABSORB_FULL), from the decisions of the launch
 * path.  out[0] = padded column count, out[1] = column blocks, out[2] =
 * independent stream groups of a sweep, out[3] = cluster size, out[4] = rows
 * per streamed chunk, out[5] = cp.async stages, out[6] = epilogue (0
 * accumulated rotations, 1 left family, 2 right family, 3 values only),
 * out[7] = sweeps that may replay the cached sweep graph (0: none),
 * out[8] / out[9] = panel mask / wy_t of the QR preconditioner (as
 * qb_qr_route), out[10] = round launches per sweep.  16 slots. */
int qb_svd_route(int64_t m, int64_t n, int absorb, int64_t *out16);

/*
 * Host-side truncation rule of svd_truncated's numba core,
 * decomp.py:901-937 (_compute_number_svals_to_keep_numba) followed by the
 * max_bond clamp of decomp.py:1000-1004.  s: host array, descending.
 */
int qb_svals_to_keep(const double *s, int64_t n, double cutoff,
                     int cutoff_mode, int64_t max_bond, int renorm,
                     int64_t *n_keep, double *renorm_factor,
                     double *trunc_error);

/* ---- MPS sampling ------------------------------------------------------- */
/*
 * One site of batched MPS sampling, the selection after the contraction
 * W = V . A_i (MatrixProductState.sample / sample_configuration,
 * quimb/tensor/tn1d/core.py:3871-3990).  W is C x d x r, contiguous, of
 * dtype QB_F64 or QB_C128 (16-byte aligned for complex).  For every sample c:
 *   pi[s] = sum_j |W[c, s, j]|^2 (fp64), p = pi / sum(pi) with numpy's
 *   pairwise sum, cdf = cumsum(p) / cdf[d-1], x = #{s : cdf[s] <= u[c*ldu]}
 *   (numpy's Generator.choice(d, p=p) for the uniform u: searchsorted
 *   side='right'; a zero-probability outcome is never chosen),
 *   config[c*ldc] = x, omega[c] *= p[x], V[c, :] = W[c, x, :] / sqrt(pi[x])
 *   (C x r, contiguous: the selected row at unit norm).
 * A row whose sum(pi) is zero or not finite, or whose u lies outside [0, 1),
 * gets config = -1, omega = NaN and a zero V row.  The arithmetic of a row
 * depends on d and r only (never on C or the launch shape).  1 <= d <= 256
 * (-3 otherwise), r >= 1; C == 0 launches nothing.  One launch.
 */
int qb_sample_select(int dtype, int64_t C, int64_t d, int64_t r, const void *W,
                     const double *u, int64_t ldu, int64_t *config, int64_t ldc,
                     double *omega, void *V, void *stream);

/* ---- MPS reduced density matrices -------------------------------------- */
/*
 * The reduction that ends every reduced density matrix of an MPS
 * (partial_trace_to_dense_canonical / local expectations,
 * quimb/tensor/tn1d/core.py:2827-3087):
 *   out[m, n] = sum_{a < n1, b < n2} U[a, m, b] * conj(V[a, n, b])
 * U and V are strided views (strides in elements, any sign; permuted views
 * need no copy) of dtype QB_F64 (conj is the identity) or QB_C128 (16-byte
 * aligned); out is M x N, contiguous.  Accumulation is fp64 (pairs of fp64
 * for complex); NaN and Inf propagate.  When U == V with equal strides each
 * element is loaded once.  At most two launches on `stream` (partials over
 * fixed K-tiles, then a fixed-order reduction), no allocation and no host
 * synchronisation, so the call can be captured in a graph.  The grid and the
 * summation order depend on (n1, M, N, n2) only: the same input gives the
 * same bits on any device or stream, and whether or not U aliases V.
 * 1 <= M, N <= 64 (-2), n1, n2 >= 1 (-3), U, V, out or a stride array null
 * or misaligned (-4), workspace smaller than qb_rdm_workspace (-6), any
 * other dtype (-1); nothing is launched when a call is rejected.
 * qb_rdm_workspace returns the bytes needed (0 for a single block) or the
 * same negative codes.
 */
int64_t qb_rdm_workspace(int64_t n1, int64_t M, int64_t N, int64_t n2);
int qb_rdm_reduce(int dtype, int64_t n1, int64_t M, int64_t N, int64_t n2,
                  const void *U, const int64_t ustride[3],
                  const void *V, const int64_t vstride[3],
                  void *out, void *workspace, int64_t ws_bytes, void *stream);

/* ---- PEPS local expectations from plaquette density matrices ----------- */
/*
 * The per-term evaluation of PEPS.compute_local_expectation
 * (quimb/tensor/tn2d/core.py:4335-4348), for every term of a call in one
 * launch.  Term t reads row t of the host table `desc` (QB_PLAQ_DESC_WORDS
 * int64 words):
 *   [0] offset of its plaquette's rho (elements) in `rho`, a row-major D x D
 *       matrix, ket index first; D = prod of the site dimensions <= 64
 *   [1] offset of its G (elements) in `G`, a row-major dg x dg matrix over
 *       the term's sites in increasing position order (out index first)
 *   [2] number of plaquette sites, 1 .. QB_PLAQ_MAX_SITES
 *   [3] number of term sites, 1 or 2
 *   [4], [5] the term's site positions within the plaquette, increasing
 *       ([5] unused for one site)
 *   [6 .. 11] the plaquette's per-site dimensions
 * and writes out[2 t] = Tr[G_t rho_p] with the other plaquette sites traced,
 * out[2 t + 1] = Tr[rho_p].  rho, G and out are device arrays of one dtype,
 * QB_F64 or QB_C128.  The table is copied once to the device buffer
 * `desc_dev` (n_terms * QB_PLAQ_DESC_WORDS int64) on `stream`, then one
 * kernel runs there; no allocation, no host synchronisation.  Pageable `desc`
 * may be reused when the call returns.  Every sum has a fixed order set by
 * the descriptor alone: the same input gives the same bits on any device or
 * stream, and NaN / Inf reach only the terms that read them.
 * Unknown dtype (-1), n_terms < 0 (-2), an invalid descriptor: counts,
 * positions, dimensions, D > 64 or an offset out of rho_elems / g_elems (-3),
 * a pointer null or misaligned (-4); nothing is copied or launched when a
 * call is rejected, and n_terms == 0 does nothing.
 */
#define QB_PLAQ_DESC_WORDS 12
#define QB_PLAQ_MAX_SITES 6
#define QB_PLAQ_MAX_DIM 64
int qb_plaquette_expec(int dtype, int64_t n_terms, const int64_t *desc, void *desc_dev,
                       const void *rho, int64_t rho_elems, const void *G, int64_t g_elems,
                       void *out, void *stream);

/* ---- sketched left environments of successive randomized compression --- */
/*
 * The first half of one left-environment step of SRC on an MPS / MPO ladder
 * (tensor_network_1d_compress_src, quimb/tensor/tn1d/compress.py:1653-1840):
 *   H[B, a, u, p] = sum_{v < nv, o < no} LE[B, a, v] W[v, u, o, p] Om[B, o]
 * with nB samples B; the step ends with LE'[B, b, u] = sum H[B, a, u, p]
 * A[a, p, b], one ordinary contraction.  Every operand is a strided view
 * (strides in elements, any sign, 0 allowed on the inputs; H must not
 * overlap an input), all of one dtype: QB_F32, QB_F64, QB_C64 or QB_C128;
 * no conjugation.  Single precision is accumulated in fp64 and rounded once.
 * Exactly one launch on `stream`, no allocation, no host synchronisation.
 * Every output is a sum over v in order of products with the sum over o in
 * order, and the grid depends on (nB, na, nu np) alone, so the same input
 * gives the same bits on any device or stream; NaN and Inf propagate.
 * Unknown dtype (-1), an extent below 1 (-2), a pointer or stride array null
 * or misaligned (-3), a grid of more than 2^31 - 1 blocks (-4); nothing is
 * launched when a call is rejected.
 */
int qb_sketch_env(int dtype, int64_t nB, int64_t na, int64_t nv, int64_t nu, int64_t no,
                  int64_t np, const void *LE, const int64_t lestride[3], const void *W,
                  const int64_t wstride[4], const void *Om, const int64_t omstride[2],
                  void *H, const int64_t hstride[4], void *stream);

/* ---- device queries / microbenchmarks ---------------------------------- */
/* ------------------------------------------------------------------------
 * Peer-memory exchange of the bond-sharded two-site eigensolve (multi-GPU,
 * one process per GPU).  Replaces, on the data path, the ncclAllGather of the
 * Lanczos vector and the ncclAllReduce of the Gram-Schmidt inner products
 * that a sharded TNLinearOperator._matvec / eigsh would issue
 * (quimb/tensor/tensor_core.py:12393-12417, quimb/linalg/scipy_linalg.py:
 * 113-128): ONE kernel each, storing into the peers' HBM over NVLink.
 *
 * Every rank allocates one block (qb_p2p_alloc: cudaMalloc'ed and zeroed by
 * the library -- the only allocation the library owns, released by
 * qb_p2p_free), exports it (64-byte CUDA IPC handle) and imports the blocks
 * of its peers; `peer_bufs[world]` lists the block bases in rank order, the
 * caller's own block at index `rank`.  `epoch` counts the calls of each kind
 * (1, 2, ...; the same sequence on every rank; epoch 0 is rejected because
 * the flags start at 0); `scratch` is 8 bytes of zeroed device memory (CTA
 * counter, error word: non-zero after a kernel gave up waiting ~4 s for a
 * peer).  Every accepted call launches exactly one kernel.
 *
 * Error codes of the two exchange calls (nothing is launched): -1 world or
 * rank out of range (at most 16 ranks), -2 null peer block, -3 null scratch,
 * -4 epoch 0, -5 bad slab / vector (negative, not 16-byte granular or
 * aligned, null; for the all-reduce m outside [0, 64] or x not 8-byte
 * aligned), -6 slab past the gather buffer (dst_off + bytes above
 * gather_bytes rounded up to 256).
 */
int64_t qb_p2p_block_bytes(int64_t gather_bytes);
int64_t qb_p2p_data_offset(int64_t gather_bytes, int parity);
int qb_p2p_alloc(int64_t bytes, void **ptr);
int qb_p2p_free(void *ptr);
int qb_p2p_export(void *ptr, unsigned char *handle64);
int qb_p2p_import(const unsigned char *handle64, void **peer_ptr);
int qb_p2p_unimport(void *peer_ptr);
/* all ranks: slab `x` (bytes, 16-byte granular) -> byte offset dst_off of the
 * gather buffer of parity (epoch & 1) on EVERY rank; when the kernel has
 * completed the whole vector is resident in the local block.  An empty slab
 * (bytes == 0, x may be null) is legal and still raises this rank's flags. */
int qb_p2p_allgather(void *const *peer_bufs, int world, int rank, const void *x,
                     int64_t bytes, int64_t dst_off, int64_t gather_bytes,
                     uint64_t epoch, void *scratch, void *stream);
/* in-place sum over the ranks of m <= 64 doubles, bit-identical everywhere:
 * x[t] = ((p_0 + p_1) + p_2) + ... in rank order from rank 0's partial, so one
 * rank is the identity and -0.0 partials sum to -0.0.  Every rank passes the
 * same m; m == 0 still launches and raises the epoch's flags. */
int qb_p2p_allreduce_small(void *const *peer_bufs, int world, int rank, void *x,
                           int m, uint64_t epoch, void *scratch, void *stream);

/* sustained DMMA (fp64 tensor core) rate of the current device in TFLOP/s */
int qb_measure_dmma_peak(double *tflops, void *stream);
/* tuning hook: with QB_TRACE=1 in the environment the contraction kernels stamp
 * %globaltimer at their phase boundaries (entry, tables, prologue issued,
 * first tile landed, main loop done, stream-K fix-up done, stores issued) into
 * a device buffer laid out [cta][4 segments][8 phases]; this copies the first
 * `count` uint64 entries to `host_out`, clears the buffer and returns 0
 * (1 if tracing is off). */
int qb_debug_trace_read(unsigned long long *host_out, int64_t count);

#ifdef __cplusplus
}
#endif
#endif /* QUIMB_B200_H */
