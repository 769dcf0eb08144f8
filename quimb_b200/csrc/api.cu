// extern "C" entry points declared in include/quimb_b200.h
#include <stdarg.h>
#include <stdlib.h>
#include <string.h>

#include <vector>

#include "internal.h"

namespace qb {

static thread_local char g_err[1024] = "";
std::atomic<int64_t> g_launch_count{0};

void set_error(const char *fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}

int sm_count() {
  static int n = 0;
  if (!n) {
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess ||
        cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) !=
            cudaSuccess)
      n = 132;  // H100 SXM
  }
  return n;
}

int gemm_f64(const double *A, int64_t a_rs, int64_t a_cs, const double *B,
             int64_t b_rs, int64_t b_cs, double *C, int64_t c_rs, int64_t c_cs,
             int64_t M, int64_t N, int64_t K, double alpha, double beta,
             cudaStream_t st, double *splitk_ws, int64_t splitk_ws_elems,
             int max_splitk) {
  if (M <= 0 || N <= 0) return 0;
  qb_tensor_t a, b, c;
  memset(&a, 0, sizeof(a)); memset(&b, 0, sizeof(b)); memset(&c, 0, sizeof(c));
  a.ptr = const_cast<double *>(A); a.dtype = QB_F64; a.rank = 2;
  a.shape[0] = M; a.shape[1] = K; a.stride[0] = a_rs; a.stride[1] = a_cs;
  b.ptr = const_cast<double *>(B); b.dtype = QB_F64; b.rank = 2;
  b.shape[0] = K; b.shape[1] = N; b.stride[0] = b_rs; b.stride[1] = b_cs;
  c.ptr = C; c.dtype = QB_F64; c.rank = 2;
  c.shape[0] = M; c.shape[1] = N; c.stride[0] = c_rs; c.stride[1] = c_cs;
  const int32_t la[2] = {0, 1}, lb[2] = {1, 2}, lc[2] = {0, 2};
  PairPlan plan;
  if (!splitk_ws) max_splitk = 1;
  int rc = plan_pair(&a, la, &b, lb, &c, lc, 0, 0, plan, max_splitk);
  if (rc) return rc;
  plan.streamk = 0;  // internal GEMMs use classic launches (small scratch)
  if (plan.p.splitk > 1) {
    if (plan_scratch_bytes(plan) > splitk_ws_elems * 8) {
      // not enough scratch: redo the plan without split-K
      rc = plan_pair(&a, la, &b, lb, &c, lc, 0, 0, plan, 1);
      if (rc) return rc;
      plan.streamk = 0;
    } else {
      plan.p.partial = splitk_ws;
    }
  }
  if (plan.zero_fill) {
    if (beta == 0.0) return launch_fill_zero(&c, st);
    return 0;
  }
  plan.p.alpha = alpha; plan.p.beta = beta;
  return launch_contract_f64(plan, st);
}

static bool is_single(int dt) { return dt == QB_F32 || dt == QB_C64; }

// f64 / c128: every engine.  f32 / c64: the int8 engine only (4 int8
// slices, float epilogue); shapes below its tile minimum are refused with
// QB_NO_NATIVE_SINGLE and the host layer widens them instead.
constexpr int QB_NO_NATIVE_SINGLE = -101;
static int check_device_dtype(const PairPlan &plan) {
  if (is_single(plan.dtype) && !(plan.empty_out || plan.zero_fill) && !ozaki_eligible(plan)) {
    set_error("single-precision contraction M=%lld N=%lld K=%lld batch=%lld is below the "
              "int8 engine's minimum (M >= 128, N >= 64, K >= 128 real units, no "
              "batch modes): widen it", (long long)plan.p.M, (long long)plan.p.N,
              (long long)plan.p.K, (long long)plan.p.nbatch);
    return QB_NO_NATIVE_SINGLE;
  }
  return 0;
}

}  // namespace qb

using namespace qb;

// engine policy: explicit request, or QB_ENGINE=ozaki|dmma|stream in the
// environment
static int env_engine() {
  static const int v = [] {
    const char *e = getenv("QB_ENGINE");
    if (e && !strcmp(e, "ozaki")) return (int)QB_ENGINE_OZAKI;
    if (e && !strcmp(e, "dmma")) return (int)QB_ENGINE_DMMA;
    if (e && !strcmp(e, "stream")) return (int)QB_ENGINE_STREAM;
    return (int)QB_ENGINE_AUTO;
  }();
  return v;
}
// float64 / complex128 take the int8 engine only on request: on the H100 its
// 36 slice products bound it to ~55 TFLOP/s fp64-equivalent (1979 int8 TOPS /
// 36), below the 67 TFLOP/s DMMA peak at every size, and it was measured
// slower than the DMMA kernel at 2048^3 and 4096^3 (DESIGN.md section 4.6).
static bool want_ozaki(int engine, const PairPlan &plan) {
  if (is_single(plan.dtype)) return ozaki_eligible(plan);   // the only native engine
  if (engine == QB_ENGINE_AUTO) engine = env_engine();
  return engine == QB_ENGINE_OZAKI && ozaki_eligible(plan);
}
// streaming engine (contract_stream.cu): small-operator steps, N, K <= 32
// (real) or <= 16 (complex)
static bool want_stream(int engine, const PairPlan &plan) {
  if (engine == QB_ENGINE_AUTO) engine = env_engine();
  return engine == QB_ENGINE_STREAM && stream_eligible(plan);
}

// The one dispatch decision of a pairwise contraction (engine = the low byte
// of the caller's engine argument).  contract_pair_impl launches what this
// returns and qb_contract_pair_route reports it.
static Route select_route(const PairPlan &plan, int engine) {
  Route r{ROUTE_DMMA, -1, 1, 0, 0, 0, -1, 0};
  if (plan.empty_out) { r.kind = ROUTE_EMPTY; return r; }
  if (plan.zero_fill) {
    r.kind = ROUTE_ZERO_FILL;
    r.launches = plan.out_elems > 0 ? 1 : 0;
    return r;
  }
  if (is_single(plan.dtype) && !ozaki_eligible(plan)) { r.kind = ROUTE_WIDEN; return r; }
  if (want_ozaki(engine, plan)) {
    r.kind = ROUTE_INT8;
    r.launches = 5;  // rowmax + split of each operand, then the int8 GEMM
    return r;
  }
  if (want_stream(engine, plan)) {
    const StreamVariant v = stream_variant(plan.p);
    r.kind = ROUTE_STREAM;
    r.launches = 1;
    r.stream_k = v.kmax;
    r.stream_n = v.nmax;
    return r;
  }
  return dmma_route(plan, true);
}


extern "C" {

int qb_abi_version(void) { return QB_ABI_VERSION; }
const char *qb_last_error(void) { return g_err; }
int64_t qb_launch_count(void) { return g_launch_count.load(); }

int qb_contract_pair_plan(const qb_tensor_t *A, const int32_t *la,
                          const qb_tensor_t *B, const int32_t *lb,
                          const qb_tensor_t *C, const int32_t *lc,
                          int64_t *out) {
  PairPlan plan;
  int rc = plan_pair(A, la, B, lb, C, lc, 0, 0, plan);
  if (rc) return rc;
  const ContractParams &p = plan.p;
  out[0] = p.M; out[1] = p.N; out[2] = p.K; out[3] = p.nbatch;
  out[4] = p.m.n; out[5] = p.n.n; out[6] = p.k.n; out[7] = p.b.n;
  out[8] = plan.cfg; out[9] = p.splitk; out[10] = p.vecA; out[11] = p.vecB;
  out[12] = p.vecC; out[13] = p.thrA; out[14] = p.thrB;
  out[15] = plan.empty_out ? 2 : (plan.zero_fill ? 1 : 0);
  return 0;
}

int qb_contract_pair_route(const qb_tensor_t *A, const int32_t *la,
                           const qb_tensor_t *B, const int32_t *lb,
                           const qb_tensor_t *C, const int32_t *lc, int engine,
                           int64_t *out) {
  PairPlan plan;
  int rc = plan_pair(A, la, B, lb, C, lc, 0, 0, plan);
  if (rc) return rc;
  const Route r = select_route(plan, engine & 0xff);
  out[0] = r.kind; out[1] = r.cfg; out[2] = r.splitk; out[3] = r.streamk;
  out[4] = r.sk_head; out[5] = r.bk; out[6] = r.layout; out[7] = sm_count();
  out[8] = r.launches; out[9] = r.stream_k; out[10] = r.stream_n;
  return 0;
}

int qb_contract_pair_feed(const qb_tensor_t *A, const int32_t *la,
                          const qb_tensor_t *B, const int32_t *lb,
                          const qb_tensor_t *C, const int32_t *lc, int64_t *out) {
  PairPlan plan;
  int rc = plan_pair(A, la, B, lb, C, lc, 0, 0, plan);
  if (rc) return rc;
  const Route r = select_route(plan, QB_ENGINE_AUTO);
  const bool large_real = (r.kind == ROUTE_DMMA || r.kind == ROUTE_DMMA_STREAMK) &&
                          r.cfg == 0 && r.layout >= 0;
  out[0] = large_real ? plan.p.feedA : -1;
  out[1] = large_real ? plan.p.feedB : -1;
  return 0;
}

int qb_contract_pair_schedule(const qb_tensor_t *A, const int32_t *la,
                              const qb_tensor_t *B, const int32_t *lb,
                              const qb_tensor_t *C, const int32_t *lc, int64_t *out) {
  PairPlan plan;
  int rc = plan_pair(A, la, B, lb, C, lc, 0, 0, plan);
  if (rc) return rc;
  const Route r = select_route(plan, QB_ENGINE_AUTO);
  out[0] = r.kind != ROUTE_DMMA_STREAMK ? -1 : (streamk_pair(plan) ? 1 : 0);
  return 0;
}

int64_t qb_contract_pair_workspace(const qb_tensor_t *A, const int32_t *la,
                                   const qb_tensor_t *B, const int32_t *lb,
                                   const qb_tensor_t *C, const int32_t *lc,
                                   int engine) {
  PairPlan plan;
  int rc = plan_pair(A, la, B, lb, C, lc, 0, 0, plan);
  if (rc) return rc;
  if ((rc = check_device_dtype(plan))) return rc;
  int64_t need = plan_workspace_bytes(plan);
  if (want_ozaki(engine & 0xff, plan))
    need = std::max(need, ozaki_workspace_bytes(plan) + kWsHeaderBytes);
  return need;
}

int qb_debug_contract_stream_host(const qb_tensor_t *A, const int32_t *la,
                                  const qb_tensor_t *B, const int32_t *lb,
                                  qb_tensor_t *C, const int32_t *lc, int conjA,
                                  int conjB, double alpha, double beta) {
  PairPlan plan;
  int rc = plan_pair(A, la, B, lb, C, lc, conjA, conjB, plan);
  if (rc) return rc;
  if (plan.empty_out) return 0;
  if (plan.zero_fill) {
    set_error("qb_debug_contract_stream_host: zero-extent contraction");
    return -10;
  }
  plan.p.alpha = alpha; plan.p.beta = beta;
  rc = contract_stream_host(plan);
  if (rc)
    set_error("qb_debug_contract_stream_host: needs f64 with N, K <= 32 or c128 with "
              "N, K <= 16");
  return rc;
}

// QB_TRACE=1: device buffer the kernels stamp their phase times into
static constexpr int64_t kTraceEntries = 1 << 20;
}  // extern "C"
namespace qb {
unsigned long long *trace_buffer() {
  static unsigned long long *buf = [] () -> unsigned long long * {
    const char *e = getenv("QB_TRACE");
    if (!e || atoi(e) == 0) return nullptr;
    unsigned long long *b = nullptr;
    if (cudaMalloc(&b, kTraceEntries * 8) != cudaSuccess) return nullptr;
    cudaMemset(b, 0, kTraceEntries * 8);
    return b;
  }();
  return buf;
}
}  // namespace qb
extern "C" {

static int contract_pair_impl(const qb_tensor_t *A, const int32_t *la,
                              const qb_tensor_t *B, const int32_t *lb,
                              qb_tensor_t *C, const int32_t *lc, int conjA,
                              int conjB, double alpha, double beta, int engine,
                              void *workspace, size_t workspace_bytes,
                              void *stream) {
  PairPlan plan;
  const bool ws_zeroed = (engine & QB_ENGINE_WS_ZEROED) != 0;
  engine &= 0xff;
  int rc = plan_pair(A, la, B, lb, C, lc, conjA, conjB, plan);
  if (rc) return rc;
  const Route route = select_route(plan, engine);
  if (route.kind == ROUTE_WIDEN) return check_device_dtype(plan);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (route.kind == ROUTE_EMPTY) return 0;
  if (route.kind == ROUTE_ZERO_FILL) {
    if (beta == 0.0) return launch_fill_zero(C, st);
    if (beta == 1.0) return 0;
    set_error("zero-extent contraction with beta not in {0, 1}");
    return -10;
  }
  plan.p.alpha = alpha; plan.p.beta = beta;
  if (unsigned long long *tb = trace_buffer()) {
    static unsigned trace_launch = 0;  // 16 rotating slots of 8192 stamps
    plan.p.trace = tb + (size_t)(trace_launch++ % 16) * 8192;
  }
  if (route.kind == ROUTE_INT8) {
    int64_t need = ozaki_workspace_bytes(plan) + kWsHeaderBytes;
    if (!workspace || (int64_t)workspace_bytes < need) {
      set_error("workspace too small: need %lld bytes, got %lld",
                (long long)need, (long long)workspace_bytes);
      return -10;
    }
    return launch_contract_ozaki(plan, static_cast<char *>(workspace) + kWsHeaderBytes, st);
  }
  if (route.kind == ROUTE_STREAM) return launch_contract_stream(plan, st);
  int64_t need = plan_workspace_bytes(plan);
  if (need > 0) {
    if (!workspace || (int64_t)workspace_bytes < need) {
      set_error("workspace too small: need %lld bytes, got %lld",
                (long long)need, (long long)workspace_bytes);
      return -10;
    }
    // header = stream-K flag words, scratch behind it
    plan.p.flags = static_cast<int *>(workspace);
    plan.p.partial = reinterpret_cast<double *>(static_cast<char *>(workspace) + kWsHeaderBytes);
    plan.flags_clean = ws_zeroed;
  }
  if (plan.dtype == QB_F64) return launch_contract_f64(plan, st);
  return launch_contract_c128(plan, st);
}

int qb_contract_pair(const qb_tensor_t *A, const int32_t *la,
                     const qb_tensor_t *B, const int32_t *lb, qb_tensor_t *C,
                     const int32_t *lc, int conjA, int conjB, int engine,
                     void *workspace, size_t workspace_bytes, void *stream) {
  return contract_pair_impl(A, la, B, lb, C, lc, conjA, conjB, 1.0, 0.0, engine,
                            workspace, workspace_bytes, stream);
}

int qb_contract_pair_ab(const qb_tensor_t *A, const int32_t *la,
                        const qb_tensor_t *B, const int32_t *lb,
                        qb_tensor_t *C, const int32_t *lc, int conjA,
                        int conjB, double alpha, double beta, void *workspace,
                        size_t workspace_bytes, void *stream) {
  return contract_pair_impl(A, la, B, lb, C, lc, conjA, conjB, alpha, beta,
                            QB_ENGINE_AUTO, workspace, workspace_bytes, stream);
}

int qb_contract_batched(const qb_tensor_t *A0, const int32_t *la,
                        const qb_tensor_t *B0, const int32_t *lb,
                        qb_tensor_t *C0, const int32_t *lc,
                        const void *const *dA, const void *const *dB,
                        void *const *dC, int64_t count, int conjA, int conjB,
                        void *stream) {
  PairPlan plan;
  int rc = plan_pair(A0, la, B0, lb, C0, lc, conjA, conjB, plan);
  if (rc) return rc;
  if (is_single(plan.dtype)) {
    set_error("qb_contract_batched: single precision has no batched engine: widen");
    return QB_NO_NATIVE_SINGLE;
  }
  if (plan.p.b.n) {
    set_error("qb_contract_batched: batch labels are not allowed inside the "
              "per-item signature");
    return -2;
  }
  if (count <= 0 || plan.empty_out) return 0;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (plan.zero_fill) {
    set_error("qb_contract_batched: zero-extent contracted index");
    return -2;
  }
  // pointer-array batch: no split-K (tiles x count is the parallelism)
  plan.streamk = 0;
  plan.p.splitk = 1;
  // whole (real-unit) contracted extent in one pass
  plan.p.k_per_split = cdiv(plan.p.K * (plan.dtype == QB_C128 ? 2 : 1), 32) * 32;
  plan.p.dA = dA; plan.p.dB = dB; plan.p.dC = dC;
  int64_t done = 0;
  while (done < count) {
    int64_t chunk = std::min<int64_t>(count - done, 65535);
    plan.p.nbatch = chunk;
    plan.p.dA = dA + done; plan.p.dB = dB + done; plan.p.dC = dC + done;
    if (plan.dtype == QB_F64) rc = launch_contract_f64(plan, st);
    else rc = launch_contract_c128(plan, st);
    if (rc) return rc;
    done += chunk;
  }
  return 0;
}

}  // extern "C"

extern "C" int qb_debug_trace_read(unsigned long long *host_out, int64_t count) {
  unsigned long long *buf = trace_buffer();
  if (!buf) return 1;
  if (count > kTraceEntries) count = kTraceEntries;
  cudaDeviceSynchronize();
  if (cudaMemcpy(host_out, buf, count * 8, cudaMemcpyDeviceToHost) != cudaSuccess) return 2;
  cudaMemset(buf, 0, kTraceEntries * 8);
  return 0;
}

