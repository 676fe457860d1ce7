// extern "C" surface of libparo_b200.so (declared in include/paro_b200.h): argument checks with
// the reference's error behaviour (TORCH_CHECK -> message, here: code + paro_last_error()),
// dispatch to the sm_90a kernels.  No allocation, no host synchronisation.
#include <atomic>
#include <cstdarg>
#include <cstdio>
#include <cstdlib>

#include "paro_common.cuh"
#include "paro_launch.h"

namespace paro {

static thread_local char g_err[512] = "";
static thread_local int g_launches = 0;

void set_error(const char *fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}
void note_launches(int n) { g_launches += n; }

const Knobs &knobs() {
  static const Knobs k = [] {
    auto env = [](const char *name, int dflt) {
      const char *v = getenv(name);
      return v && *v ? atoi(v) : dflt;
    };
    Knobs x;
    const int m = env("PARO_SMALL_M_MAX", 16);
    x.small_m_max = m < 0 ? 0 : m > 16 ? 16 : m;
    x.decode_stream = env("PARO_DECODE_STREAM", 0) != 0;
    x.prerot_m = env("PARO_DECODE_PREROT_M", 0);
    x.no_cluster = env("PARO_NO_CLUSTER", 0);
    x.force_c = env("PARO_DECODE_C", 0);
    x.stages = env("PARO_DECODE_STAGES", 0);
    x.inflight = env("PARO_DECODE_INFLIGHT", 6);
    x.b8 = env("PARO_DECODE_B8", 1);
    x.no_pdl = env("PARO_NO_PDL", 0);
    x.trace = env("PARO_DECODE_TRACE", 0);
    x.verbose = env("PARO_DECODE_VERBOSE", 0);
    return x;
  }();
  return k;
}

int device_sms() {
  static std::atomic<int> sms_of[64];   // per device; threads that race on a first query store the same value
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess) return 0;
  if (dev < 64) {
    const int n = sms_of[dev].load(std::memory_order_relaxed);
    if (n) return n;
  }
  int n = 0;
  if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess) return 0;
  if (dev < 64) sms_of[dev].store(n, std::memory_order_relaxed);
  return n;
}

cudaError_t smem_opt_in(const void *kernel, int bytes) {
  static std::mutex mu;
  static std::map<std::pair<const void *, int>, int> granted;   // (kernel, device) -> bytes
  int dev = 0;
  cudaError_t e = cudaGetDevice(&dev);
  if (e == cudaSuccess) {
    std::lock_guard<std::mutex> lock(mu);
    int &have = granted[{kernel, dev}];
    if (have >= bytes) return cudaSuccess;
    e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes);
    if (e == cudaSuccess) have = bytes;
  }
  if (e != cudaSuccess) (void)cudaGetLastError();
  return e;
}

int ring_stages(int room, int stage_bytes, int max_stages, int multiple, int minimum, bool stages_knob) {
  int n = room / stage_bytes;
  if (n > max_stages) n = max_stages;
  const int want = knobs().stages;
  if (stages_knob && want >= multiple && want < n) n = want;
  n = n / multiple * multiple;
  return n < minimum ? 0 : n;
}

static bool valid_dtype(int d) { return d == PARO_F32 || d == PARO_F16 || d == PARO_BF16; }
static bool aligned(const void *p, size_t a) { return (reinterpret_cast<uintptr_t>(p) & (a - 1)) == 0; }
// the layout of a linear's shape; on a null or unsupported shape false, with the error "<what>: <reason>"
static bool layout_of(const paro_linear_shape *shape, const char *what, Layout &L) {
  const char *why = "null shape";
  if (shape && make_layout(*shape, L, &why)) return true;
  set_error("%s: %s", what, why);
  return false;
}

}  // namespace paro

using namespace paro;

extern "C" {

int paro_abi_version(void) { return PARO_ABI_VERSION; }
const char *paro_last_error(void) { return g_err; }
int paro_last_launch_count(void) { return g_launches; }

int paro_rotate(const void *x, void *out, const int16_t *idx_ij, const void *theta, int32_t theta_dtype,
                const void *scales, int32_t scales_dtype, int64_t M, int32_t K, int32_t krot, int32_t group_size,
                int32_t dtype, paro_stream_t stream) {
  g_launches = 0;
  if (!x || !out || !idx_ij || !theta) { set_error("rotate: null pointer argument"); return PARO_EINVAL; }
  if (!valid_dtype(dtype)) { set_error("rotate supports Float, Half, and BFloat16, got dtype code %d", dtype); return PARO_EINVAL; }
  if (!valid_dtype(theta_dtype) || (scales && !valid_dtype(scales_dtype))) { set_error("rotate: bad theta/scales dtype"); return PARO_EINVAL; }
  if (group_size != 64 && group_size != 128) {  // rotation.cu:123
    set_error("Unsupported group_size: %d; expected 64 or 128", group_size);
    return PARO_EUNSUPPORTED;
  }
  if (K <= 0 || K % group_size) { set_error("h must be divisible by GROUP_SIZE"); return PARO_EINVAL; }  // rotation.cu:66
  if (krot < 1 || krot > 16) { set_error("Unsupported KROT = %d; supported: 1..16", krot); return PARO_EUNSUPPORTED; }
  if (M < 0) { set_error("rotate: negative row count"); return PARO_EINVAL; }
  if (!aligned(x, 16) || !aligned(out, 16) || !aligned(idx_ij, 4)) { set_error("rotate: x/out must be 16-byte aligned, idx_ij 4-byte"); return PARO_EINVAL; }
  return rotate_launch(x, out, idx_ij, theta, theta_dtype, scales, scales_dtype, M, K, krot, group_size, dtype,
                       static_cast<cudaStream_t>(stream));
}

int paro_rotate_backward(const void *y, const void *grad_out, const void *x, const int16_t *idx_ij, const void *theta, int32_t theta_dtype,
                         const void *scales, int32_t scales_dtype, void *grad_x, float *grad_theta, float *grad_scale, int64_t M, int32_t K,
                         int32_t krot, int32_t group_size, int32_t dtype, int32_t theta_formula, paro_stream_t stream) {
  g_launches = 0;
  if (theta_formula != PARO_THETA_GRADIENT && theta_formula != PARO_THETA_REFERENCE_EXPRESSION) { set_error("rotate_backward: unknown theta_formula %d", theta_formula); return PARO_EINVAL; }
  if (!y || !grad_out || !idx_ij || !theta || !grad_x || !grad_theta) { set_error("rotate_backward: null pointer argument"); return PARO_EINVAL; }
  if (grad_scale && (!x || !scales)) { set_error("rotate_backward: grad_scale needs x and scales"); return PARO_EINVAL; }
  if (!valid_dtype(dtype)) { set_error("rotate supports Float, Half, and BFloat16, got dtype code %d", dtype); return PARO_EINVAL; }
  if (!valid_dtype(theta_dtype) || (scales && !valid_dtype(scales_dtype))) { set_error("rotate_backward: bad theta/scales dtype"); return PARO_EINVAL; }
  if (group_size != 64 && group_size != 128) { set_error("Unsupported group_size: %d; expected 64 or 128", group_size); return PARO_EUNSUPPORTED; }
  if (K <= 0 || K % group_size) { set_error("h must be divisible by GROUP_SIZE"); return PARO_EINVAL; }
  if (krot < 1 || krot > 16) { set_error("Unsupported KROT = %d; supported: 1..16", krot); return PARO_EUNSUPPORTED; }
  if (M < 0) { set_error("rotate_backward: negative row count"); return PARO_EINVAL; }
  if (grad_x == y || grad_x == grad_out) { set_error("rotate_backward: grad_x must not alias y / grad_out"); return PARO_EINVAL; }
  if (!aligned(idx_ij, 4)) { set_error("rotate_backward: idx_ij must be 4-byte aligned"); return PARO_EINVAL; }
  return rotate_backward_launch(y, grad_out, x, idx_ij, theta, theta_dtype, scales, scales_dtype, grad_x, grad_theta, grad_scale, M, K, krot, group_size,
                                dtype, theta_formula, static_cast<cudaStream_t>(stream));
}

int paro_debug_rotate_backward_plan(int64_t M, int32_t K, int32_t krot, int32_t group_size, int32_t dtype, int32_t theta_formula, int32_t sms,
                                    int64_t *out) {
  if (!out || sms < 1 || M < 1) { set_error("debug_rotate_backward_plan: bad arguments"); return PARO_EINVAL; }
  if (theta_formula != PARO_THETA_GRADIENT && theta_formula != PARO_THETA_REFERENCE_EXPRESSION) { set_error("rotate_backward: unknown theta_formula %d", theta_formula); return PARO_EINVAL; }
  if (!valid_dtype(dtype)) { set_error("rotate supports Float, Half, and BFloat16, got dtype code %d", dtype); return PARO_EINVAL; }
  if (group_size != 64 && group_size != 128) { set_error("Unsupported group_size: %d; expected 64 or 128", group_size); return PARO_EUNSUPPORTED; }
  if (K <= 0 || K % group_size) { set_error("h must be divisible by GROUP_SIZE"); return PARO_EINVAL; }
  if (krot < 1 || krot > 16) { set_error("Unsupported KROT = %d; supported: 1..16", krot); return PARO_EUNSUPPORTED; }
  return rotate_backward_debug_plan(M, K, krot, group_size, theta_formula, sms, out);
}

size_t paro_packed_bytes(const paro_linear_shape *shape) {
  Layout L;
  if (!layout_of(shape, "packed_bytes", L)) return 0;
  return L.total_bytes;
}

int paro_prepack(const paro_linear_shape *shape, const int32_t *qweight, const int32_t *qzeros, const void *scales,
                 int32_t scales_dtype, const int16_t *pairs, const void *theta, int32_t theta_dtype,
                 const void *channel_scales, int32_t cs_dtype, void *packed, paro_stream_t stream) {
  g_launches = 0;
  Layout L;
  if (!layout_of(shape, "prepack", L)) return PARO_EINVAL;
  if (!qweight || !qzeros || !scales || !pairs || !theta || !channel_scales || !packed) { set_error("prepack: null pointer argument"); return PARO_EINVAL; }
  if (!valid_dtype(scales_dtype) || !valid_dtype(theta_dtype) || !valid_dtype(cs_dtype)) { set_error("prepack: bad parameter dtype"); return PARO_EINVAL; }
  if (!aligned(packed, 128)) { set_error("prepack: packed buffer must be 128-byte aligned"); return PARO_EINVAL; }
  return prepack_launch(*shape, L, qweight, qzeros, scales, scales_dtype, pairs, theta, theta_dtype, channel_scales,
                        cs_dtype, packed, static_cast<cudaStream_t>(stream));
}

size_t paro_workspace_bytes(const paro_linear_shape *shape, int64_t max_m) {
  Layout L;
  if (!layout_of(shape, "workspace_bytes", L)) return 0;
  // head: sync words + block counters of the small-M kernel (zero between calls); behind them scratch: the partial slots
  // of the small-M kernel or the rotated activations of the M > 16 path
  size_t b = stream_workspace_bytes(L, max_m);
  {
    const size_t d = stream_sync_bytes(L) + decode_scratch_bytes(L, max_m);
    if (d > b) b = d;
  }
  if (max_m > knobs().small_m_max) {
    const size_t g = stream_sync_bytes(L) + gemm_workspace_bytes(L, max_m);
    if (g > b) b = g;
  }
  return b > 256 ? b : 256;
}

int paro_linear_forward(const paro_linear_shape *shape, const void *packed, const void *x, int64_t M, const void *bias,
                        void *y, void *workspace, size_t workspace_bytes, paro_stream_t stream) {
  g_launches = 0;
  Layout L;
  if (!layout_of(shape, "linear_forward", L)) return PARO_EINVAL;
  if (M < 0) { set_error("linear_forward: negative row count"); return PARO_EINVAL; }
  if (M == 0) return PARO_OK;
  if (!packed || !x || !y || !workspace) { set_error("linear_forward: null pointer argument"); return PARO_EINVAL; }
  if (!aligned(packed, 128) || !aligned(x, 16) || !aligned(y, 16) || !aligned(workspace, 256)) {
    set_error("linear_forward: packed must be 128-byte, workspace 256-byte, x / y 16-byte aligned");
    return PARO_EINVAL;
  }
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  // outside the cluster kernel a single linear runs as a one-step chain: the chain kernel up to 16 rows, the prefill chain above
  HostStep h = {};
  h.shape = shape;
  h.L = L;
  h.packed = packed; h.bias = bias; h.x = x; h.y = y;
  h.x_op = PARO_XOP_NONE; h.epi_op = PARO_EPI_STORE;
  if (M <= knobs().small_m_max) {
    // A single linear: the cluster kernel (paro_decode.cu: K slices reduced through distributed shared memory) has the shorter
    // tail -- measured 7.4 / 9.9 / 22.0 / 15.6 us on the Llama-3-8B shapes at M = 1 against 11.1 / 12.3 / 24.3 / 16.2 us for
    // the chain kernel run as a one-step chain, whose cross-CTA sums travel through L2.  The chain kernel takes over where the
    // cluster kernel has no launch plan (very long K) and for chains / tensor-parallel steps (paro_chain_forward).
    if (!knobs().decode_stream) {
      const size_t head = stream_sync_bytes(L);   // the pre-rotated rows of the M >= 4 pre-pass live behind the epoch word
      const int rc = decode_forward(*shape, L, packed, x, M, bias, y, static_cast<uint8_t *>(workspace) + head,
                                    workspace_bytes > head ? workspace_bytes - head : 0, st);
      if (rc != PARO_EUNSUPPORTED) return rc;
    }
    return stream_forward(&h, 1, M, workspace, workspace_bytes, st);
  }
  const size_t head = stream_sync_bytes(L);   // never touched by the large-M path
  if (workspace_bytes < head) { set_error("workspace too small: have %zu, need %zu", workspace_bytes, head); return PARO_EWORKSPACE; }
  return prefill_chain_forward(&h, 1, M, static_cast<uint8_t *>(workspace) + head, workspace_bytes - head, st);
}

int paro_unpack_dense(const paro_linear_shape *shape, const void *packed, void *W_out, paro_stream_t stream) {
  g_launches = 0;
  Layout L;
  if (!layout_of(shape, "unpack_dense", L)) return PARO_EINVAL;
  if (!packed || !W_out) { set_error("unpack_dense: null pointer argument"); return PARO_EINVAL; }
  return unpack_dense_launch(*shape, L, packed, W_out, static_cast<cudaStream_t>(stream));
}

int paro_debug_silu_mul(int32_t dtype, const void *gate_up, void *act, int64_t M, int32_t I, paro_stream_t stream) {
  g_launches = 0;
  if (dtype != PARO_F16 && dtype != PARO_BF16) { set_error("debug_silu_mul: dtype must be F16 or BF16, got code %d", dtype); return PARO_EINVAL; }
  if (M < 0 || I < 2 || I % 2) { set_error("debug_silu_mul: M >= 0 and an even I >= 2 needed, got M = %lld, I = %d", static_cast<long long>(M), I); return PARO_EINVAL; }
  if (!gate_up || !act) { set_error("debug_silu_mul: null pointer argument"); return PARO_EINVAL; }
  if (!aligned(gate_up, 4) || !aligned(act, 4)) { set_error("debug_silu_mul: gate_up / act must be 4-byte aligned"); return PARO_EINVAL; }
  return moe_debug_silu_mul(dtype, gate_up, act, M, I, static_cast<cudaStream_t>(stream));
}

int paro_debug_decode_plan(const paro_linear_shape *shape, int64_t M, int32_t sets, int32_t sms, const int32_t *resident_clusters,
                            int32_t *out) {
  Layout L;
  if (!layout_of(shape, "debug_decode_plan", L)) return PARO_EINVAL;
  if (!resident_clusters || !out || sms < 1) { set_error("debug_decode_plan: bad arguments"); return PARO_EINVAL; }
  return decode_debug_plan(L, M, sets, sms, resident_clusters, out);
}

int paro_debug_gemm_plan(const paro_linear_shape *shape, int64_t M, int32_t sms, int32_t *out) {
  Layout L;
  if (!layout_of(shape, "debug_gemm_plan", L)) return PARO_EINVAL;
  if (!out) { set_error("debug_gemm_plan: bad arguments"); return PARO_EINVAL; }
  return gemm_debug_plan(L, M, sms, out);
}

// The checks both chains share: every descriptor on its own here, the hand-offs between steps in chain_check_links.  The row
// bound is the caller's: 16 for the decode chain's one launch, the GEMM's int row index for the prefill chain.
static int chain_to_host(const paro_chain_step *steps, int32_t n, int64_t M, int64_t max_m, HostStep *hs) {
  if (!steps || n < 1 || n > PARO_CHAIN_MAX_STEPS) { set_error("chain: 1..%d steps supported", PARO_CHAIN_MAX_STEPS); return PARO_EINVAL; }
  if (M < 1 || M > max_m) {
    set_error("chain: 1 <= M <= %lld rows supported, got %lld", static_cast<long long>(max_m), static_cast<long long>(M));
    return PARO_EUNSUPPORTED;
  }
  for (int i = 0; i < n; ++i) {
    const paro_chain_step &c = steps[i];
    const char *why = "";
    if (!c.shape || !make_layout(*c.shape, hs[i].L, &why)) { set_error("chain: step %d: %s", i, c.shape ? why : "null shape"); return PARO_EINVAL; }
    if (!c.packed) { set_error("chain: step %d: null packed buffer", i); return PARO_EINVAL; }
    if (c.x_op < PARO_XOP_NONE || c.x_op > PARO_XOP_RMSNORM || c.epilogue < PARO_EPI_STORE || c.epilogue > PARO_EPI_ADD_RESIDUAL) {
      set_error("chain: step %d: unknown x_op / epilogue", i);
      return PARO_EINVAL;
    }
    if (!aligned(c.packed, 128) || !aligned(c.x, 16) || !aligned(c.y, 16) || !aligned(c.residual_in, 16) || !aligned(c.residual_out, 16)) {
      set_error("chain: step %d: packed must be 128-byte, activations 16-byte aligned", i);
      return PARO_EINVAL;
    }
    if (c.epilogue == PARO_EPI_ADD_RESIDUAL && c.residual_in == c.residual_out && c.residual_in) {
      set_error("chain: step %d: residual_out must not alias residual_in", i);
      return PARO_EINVAL;
    }
    hs[i].shape = c.shape;
    hs[i].packed = c.packed; hs[i].bias = c.bias; hs[i].x = c.x; hs[i].y = c.y;
    hs[i].x_op = c.x_op; hs[i].epi_op = c.epilogue;
    hs[i].res_in = c.residual_in; hs[i].res_out = c.residual_out; hs[i].norm_w = c.norm_weight; hs[i].eps = c.eps;
    hs[i].tp = c.tp;
    if (c.tp) {
      if (c.tp->world < 1 || c.tp->world > PARO_TP_MAX_RANKS || c.tp->rank < 0 || c.tp->rank >= c.tp->world) {
        set_error("chain: step %d: tensor-parallel world must be 1..%d and 0 <= rank < world", i, PARO_TP_MAX_RANKS);
        return PARO_EINVAL;
      }
      for (int r = 0; r < c.tp->world; ++r)
        if (c.tp->world > 1 && (!c.tp->peer_slots[r] || !aligned(c.tp->peer_slots[r], 256))) {
          set_error("chain: step %d: peer_slots[%d] must be a 256-byte aligned device address", i, r);
          return PARO_EINVAL;
        }
    }
  }
  return PARO_OK;
}

// what one step hands the next: an input for every step, the statistics an RMSNORM step needs, matching widths, one dtype
static int chain_check_links(const HostStep *hs, int n) {
  const int dtype = hs[0].L.dtype;
  for (int i = 0; i < n; ++i) {
    const HostStep &h = hs[i];
    if (h.L.dtype != dtype) { set_error("chain: every step must use the same activation dtype"); return PARO_EINVAL; }
    const bool consumed = i + 1 < n && !hs[i + 1].x;
    if (h.x) {
      if (h.x_op == PARO_XOP_RMSNORM) { set_error("chain: step %d: RMSNORM needs the statistics of the previous step (x must be NULL)", i); return PARO_EUNSUPPORTED; }
    } else {
      if (i == 0) { set_error("chain: step 0 needs an input"); return PARO_EINVAL; }
      const HostStep &P = hs[i - 1];
      const int x_ld = h.x_op == PARO_XOP_SILU_MUL ? 2 * h.L.K : h.L.K;
      if (h.x_op == PARO_XOP_RMSNORM && P.epi_op != PARO_EPI_ADD_RESIDUAL) { set_error("chain: step %d: RMSNORM follows an ADD_RESIDUAL epilogue", i); return PARO_EINVAL; }
      if (P.L.N != x_ld) { set_error("chain: step %d produces %d columns, step %d consumes %d", i - 1, P.L.N, i, x_ld); return PARO_EINVAL; }
    }
    if (h.epi_op == PARO_EPI_ADD_RESIDUAL && (!h.res_in || !h.res_out)) { set_error("chain: step %d: ADD_RESIDUAL needs residual_in and residual_out", i); return PARO_EINVAL; }
    if (h.epi_op == PARO_EPI_STORE && !h.y && !consumed) { set_error("chain: step %d has no output", i); return PARO_EINVAL; }
    if (h.x_op == PARO_XOP_RMSNORM && !h.norm_w) { set_error("chain: step %d: RMSNORM needs norm_weight", i); return PARO_EINVAL; }
  }
  return PARO_OK;
}

size_t paro_chain_workspace_bytes(const paro_chain_step *steps, int32_t n_steps, int64_t M) {
  HostStep hs[PARO_CHAIN_MAX_STEPS] = {};
  if (chain_to_host(steps, n_steps, M, 16, hs) != PARO_OK) return 0;
  return stream_chain_workspace_bytes(hs, n_steps, M);
}

int paro_chain_forward(const paro_chain_step *steps, int32_t n_steps, int64_t M, void *workspace, size_t workspace_bytes,
                       paro_stream_t stream) {
  g_launches = 0;
  HostStep hs[PARO_CHAIN_MAX_STEPS] = {};
  int rc = chain_to_host(steps, n_steps, M, 16, hs);
  if (rc != PARO_OK) return rc;
  if (!workspace || !aligned(workspace, 256)) { set_error("chain: workspace must be a 256-byte aligned device buffer"); return PARO_EINVAL; }
  if ((rc = chain_check_links(hs, n_steps)) != PARO_OK) return rc;
  return stream_forward(hs, n_steps, M, workspace, workspace_bytes, static_cast<cudaStream_t>(stream));
}

// the prefill chain: the same descriptors for any M >= 1 (paro_gemm.cu); tensor-parallel steps stay with the decode chain
static int prefill_chain_to_host(const paro_chain_step *steps, int32_t n, int64_t M, HostStep *hs) {
  int rc = chain_to_host(steps, n, M, 0x7FFFFFFF, hs);
  if (rc != PARO_OK) return rc;
  for (int i = 0; i < n; ++i)
    if (hs[i].tp && hs[i].tp->world > 1) {
      set_error("prefill_chain: step %d: tensor-parallel steps run only in the decode chain (M <= 16)", i);
      return PARO_EUNSUPPORTED;
    }
  return chain_check_links(hs, n);
}

size_t paro_prefill_chain_workspace_bytes(const paro_chain_step *steps, int32_t n_steps, int64_t M) {
  HostStep hs[PARO_CHAIN_MAX_STEPS] = {};
  if (prefill_chain_to_host(steps, n_steps, M, hs) != PARO_OK) return 0;
  return prefill_chain_workspace_bytes(hs, n_steps, M);
}

int paro_prefill_chain_forward(const paro_chain_step *steps, int32_t n_steps, int64_t M, void *workspace, size_t workspace_bytes,
                               paro_stream_t stream) {
  g_launches = 0;
  HostStep hs[PARO_CHAIN_MAX_STEPS] = {};
  const int rc = prefill_chain_to_host(steps, n_steps, M, hs);
  if (rc != PARO_OK) return rc;
  if (!workspace || !aligned(workspace, 256)) { set_error("chain: workspace must be a 256-byte aligned device buffer"); return PARO_EINVAL; }
  return prefill_chain_forward(hs, n_steps, M, workspace, workspace_bytes, static_cast<cudaStream_t>(stream));
}

size_t paro_tp_slot_bytes(const paro_linear_shape *shape, int64_t M, int32_t world) {
  Layout L;
  if (!layout_of(shape, "tp_slot_bytes", L)) return 0;
  if (M < 1 || M > 16 || world < 1 || world > PARO_TP_MAX_RANKS) { set_error("tp_slot_bytes: 1 <= M <= 16, 1 <= world <= %d", PARO_TP_MAX_RANKS); return 0; }
  return static_cast<size_t>(2) * L.blocks_total * world * M * 128 * 8;
}

int paro_debug_stream_plan(const paro_linear_shape *shape, int64_t M, int32_t sets, int32_t ctas, int32_t *out) {
  Layout L;
  if (!layout_of(shape, "debug_stream_plan", L)) return PARO_EINVAL;
  if (!out) { set_error("debug_stream_plan: bad arguments"); return PARO_EINVAL; }
  return stream_debug_plan(L, M, sets, ctas, out);
}

size_t paro_moe_workspace_bytes(const paro_moe_desc *d, int64_t T, int32_t top_k) { return moe_workspace_bytes(d, T, top_k); }

int paro_moe_forward(const paro_moe_desc *d, const void *x, const int32_t *topk_ids, const float *topk_weights, int64_t T, int32_t top_k,
                     void *h, void *y, void *workspace, size_t workspace_bytes, paro_stream_t stream) {
  g_launches = 0;
  return moe_forward(d, x, topk_ids, topk_weights, T, top_k, h, y, workspace, workspace_bytes, static_cast<cudaStream_t>(stream));
}

int paro_debug_moe_plan(const paro_moe_desc *d, int64_t T, int32_t top_k, int32_t sms, int32_t *out) {
  if (!out || sms < 1) { set_error("debug_moe_plan: bad arguments"); return PARO_EINVAL; }
  return moe_debug_plan(d, T, top_k, sms, out);
}

size_t paro_moe_grouped_workspace_bytes(const paro_moe_desc *d, int64_t T, int32_t top_k) { return moe_grouped_workspace_bytes(d, T, top_k); }

int paro_moe_grouped_forward(const paro_moe_desc *d, const void *x, const int32_t *topk_ids, const float *topk_weights, int64_t T, int32_t top_k,
                             void *h, void *y, void *workspace, size_t workspace_bytes, paro_stream_t stream) {
  g_launches = 0;
  return moe_grouped_forward(d, x, topk_ids, topk_weights, T, top_k, h, y, workspace, workspace_bytes, static_cast<cudaStream_t>(stream));
}

int paro_debug_moe_grouped_plan(const paro_moe_desc *d, int64_t T, int32_t top_k, int32_t sms, int32_t *out) {
  if (!out || sms < 1) { set_error("debug_moe_grouped_plan: bad arguments"); return PARO_EINVAL; }
  return moe_grouped_debug_plan(d, T, top_k, out);
}

int paro_moe_route(const void *x, const void *router_w, int32_t dtype, int64_t T, int32_t hidden, int32_t n_experts, int32_t top_k,
                   int32_t renormalize, int32_t *topk_ids, float *topk_weights, float *logits_or_null, paro_stream_t stream) {
  g_launches = 0;
  return moe_route_forward(x, router_w, dtype, T, hidden, n_experts, top_k, renormalize, topk_ids, topk_weights, logits_or_null,
                           static_cast<cudaStream_t>(stream));
}

int paro_debug_moe_route_plan(int64_t T, int32_t hidden, int32_t n_experts, int32_t top_k, int32_t sms, int32_t *out) {
  if (!out || sms < 1) { set_error("debug_moe_route_plan: bad arguments"); return PARO_EINVAL; }
  return moe_route_debug_plan(T, hidden, n_experts, top_k, sms, out);
}

int paro_debug_stream_trace(unsigned long long *host_out, int32_t max_ctas) {
  if (!host_out || max_ctas <= 0) { set_error("debug_trace: bad arguments"); return PARO_EINVAL; }
  return stream_trace_read(host_out, max_ctas);
}

int paro_debug_trace(unsigned long long *host_out, int32_t max_ctas) {
  if (!host_out || max_ctas <= 0) { set_error("debug_trace: bad arguments"); return PARO_EINVAL; }
  return decode_trace_read(host_out, max_ctas);
}

}  // extern "C"
