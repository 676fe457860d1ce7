// Shared helpers for the sm_90a ParoQuant kernels: error plumbing and launch setup on the host (SM count, shared-memory opt-in,
// ring depth, plan cache), dtype traits with the reference's rounding points, mbarrier / bulk-copy (TMA) / PDL PTX wrappers.
#pragma once

#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include <array>
#include <map>
#include <mutex>

#include "../../include/paro_b200.h"
#include "paro_layout.h"

namespace paro {

// ------------------------------------------------------------------ host-side error plumbing
void set_error(const char *fmt, ...);
void note_launches(int n);
#define PARO_CUDA_OK(expr)                                                                   \
  do {                                                                                       \
    cudaError_t _e = (expr);                                                                 \
    if (_e != cudaSuccess) {                                                                 \
      paro::set_error("%s failed: %s", #expr, cudaGetErrorString(_e));                       \
      return PARO_ECUDA;                                                                     \
    }                                                                                        \
  } while (0)

// Every PARO_* environment knob the library reads, read once per process (paro_capi.cu)
struct Knobs {
  int small_m_max;     // PARO_SMALL_M_MAX (0..16, default 16): rows up to which the small-M kernels serve a linear
  int decode_stream;   // PARO_DECODE_STREAM: a single linear takes the chain kernel, not the cluster kernel
  int prerot_m;        // PARO_DECODE_PREROT_M: 0 the built-in rule, n >= 2 pre-rotate from n rows on, 1 never
  int no_cluster;      // PARO_NO_CLUSTER: the cluster kernel runs without clusters
  int force_c;         // PARO_DECODE_C: K slices per linear (0: planned)
  int stages;          // PARO_DECODE_STAGES: ring depth cap (0: as deep as shared memory allows)
  int inflight;        // PARO_DECODE_INFLIGHT (default 6): the chain kernel's bulk copies outstanding per SM
  int b8;              // PARO_DECODE_B8 (default 1): the chain kernel stores 8 B-operand rows for M <= 8
  int no_pdl;          // PARO_NO_PDL: the small-M kernels launch without programmatic dependent launch
  int trace;           // PARO_DECODE_TRACE: the small-M kernels write their phase timestamps
  int verbose;         // PARO_DECODE_VERBOSE: the small-M kernels print their launch plans
};
const Knobs &knobs();

// SM count of the current device, asked once per device; 0 without a device
int device_sms();

// the SM count plans are made for: the device's, or an H100's 132 without a device (workspace queries then size for an H100)
inline int planning_sms() { const int n = device_sms(); return n > 0 ? n : 132; }

// Lets `kernel` use `bytes` of dynamic shared memory on the current device.  The driver is asked only when this (kernel, device)
// has not been granted that much yet, so a grant is never lowered; a failure is returned, not remembered: the next call asks again.
cudaError_t smem_opt_in(const void *kernel, int bytes);
template <typename F> cudaError_t smem_opt_in(F *kernel, int bytes) { return smem_opt_in(reinterpret_cast<const void *>(kernel), bytes); }

// Depth of a weight ring: the `room` bytes left after the fixed regions in stages of `stage_bytes`, at most `max_stages`, capped by
// PARO_DECODE_STAGES if `stages_knob`, rounded down to a multiple of `multiple` (the worker sets); 0 if below `minimum`.
int ring_stages(int room, int stage_bytes, int max_stages, int multiple, int minimum, bool stages_knob);

// Rotation warps of the prologue: one per task up to 4 per set, then 8, 4, 2 until `fits(warps)` takes the carve-up (and fills it in)
template <typename Fits> bool fit_rot_warps(int tasks, int sets, Fits fits) {
  for (int rw = tasks < 4 * sets ? tasks : 4 * sets;; rw = rw > 8 ? 8 : rw / 2) {
    if (fits(rw)) return true;
    if (rw <= 2) return false;
  }
}

// Plans that depend only on a layout's shape, M and one kernel-specific int: `search(plan)` runs once per key, its result (a
// failure too) is looked up after that.
template <typename Plan> struct PlanCache {
  using Key = std::array<int, 7 + PARO_MAX_PARTS>;   // K, N, krot, qhalves, n_parts, M, extra, partition sizes
  template <typename Search> bool get(const Layout &L, int M, int extra, Plan &out, Search search) {
    Key k = {L.K, L.N, L.krot, L.qhalves, L.n_parts, M, extra};
    for (int p = 0; p < L.n_parts; ++p) k[7 + p] = L.part_col_begin[p + 1] - L.part_col_begin[p];
    std::lock_guard<std::mutex> lock(mu);
    auto it = plans.find(k);
    if (it == plans.end()) {
      Entry e = {};
      e.found = search(e.plan);
      it = plans.emplace(k, e).first;
    }
    out = it->second.plan;
    return it->second.found;
  }
  struct Entry { bool found; Plan plan; };
  std::mutex mu;
  std::map<Key, Entry> plans;
};

// cfg for `grid` CTAs of `threads` threads with `smem` bytes of dynamic shared memory; attr (cfg points at it) gets a cluster
// dimension of `cluster` CTAs when cluster > 0 and programmatic stream serialization when pdl
inline void launch_config(cudaLaunchConfig_t &cfg, cudaLaunchAttribute (&attr)[2], int grid, int threads, size_t smem, cudaStream_t stream,
                          int cluster, bool pdl) {
  cfg = {};
  cfg.gridDim = dim3(grid);
  cfg.blockDim = dim3(threads);
  cfg.dynamicSmemBytes = smem;
  cfg.stream = stream;
  cfg.attrs = attr;
  cfg.numAttrs = 0;
  if (cluster > 0) {
    attr[cfg.numAttrs].id = cudaLaunchAttributeClusterDimension;
    attr[cfg.numAttrs].val.clusterDim.x = cluster;
    attr[cfg.numAttrs].val.clusterDim.y = 1;
    attr[cfg.numAttrs].val.clusterDim.z = 1;
    ++cfg.numAttrs;
  }
  if (pdl) {
    attr[cfg.numAttrs].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[cfg.numAttrs].val.programmaticStreamSerializationAllowed = 1;
    ++cfg.numAttrs;
  }
}

// ------------------------------------------------------------------ dtype traits
// Every conversion below is one round-to-nearest-even, matching rotation.cuh's Traits
// (/root/reference/paroquant/kernels/cuda/rotation.cuh:177-205).
template <typename T> struct Traits;

template <> struct Traits<__half> {
  using T2 = __half2;
  static constexpr int code = PARO_F16;
  __device__ static __forceinline__ float to_float(__half v) { return __half2float(v); }
  __device__ static __forceinline__ __half from_float(float v) { return __float2half_rn(v); }
  __device__ static __forceinline__ float2 to_float2(__half2 v) { return __half22float2(v); }
  __device__ static __forceinline__ __half2 from_floats(float a, float b) { return __floats2half2_rn(a, b); }
};

template <> struct Traits<float> {   // fp32 rotate (the optimiser's dtype): no rounding anywhere
  static constexpr int code = PARO_F32;
  __device__ static __forceinline__ float to_float(float v) { return v; }
  __device__ static __forceinline__ float from_float(float v) { return v; }
};

template <> struct Traits<__nv_bfloat16> {
  using T2 = __nv_bfloat162;
  static constexpr int code = PARO_BF16;
  __device__ static __forceinline__ float to_float(__nv_bfloat16 v) { return __bfloat162float(v); }
  __device__ static __forceinline__ __nv_bfloat16 from_float(float v) { return __float2bfloat16_rn(v); }
  __device__ static __forceinline__ float2 to_float2(__nv_bfloat162 v) { return __bfloat1622float2(v); }
  __device__ static __forceinline__ __nv_bfloat162 from_floats(float a, float b) { return __floats2bfloat162_rn(a, b); }
};

template <typename T> __device__ __forceinline__ uint32_t pack2(typename Traits<T>::T2 v) {
  return *reinterpret_cast<uint32_t *>(&v);
}
template <typename T> __device__ __forceinline__ typename Traits<T>::T2 unpack2(uint32_t u) {
  return *reinterpret_cast<typename Traits<T>::T2 *>(&u);
}

// Load one element of a parameter tensor stored as `src_dtype` and return it as float AFTER
// the cast to T that rotation.cu:75-78 performs with `.to(x.dtype)`.
template <typename T> __device__ __forceinline__ float load_param_as(const void *p, int64_t i, int src_dtype) {
  float f;
  if (src_dtype == PARO_F32) f = reinterpret_cast<const float *>(p)[i];
  else if (src_dtype == PARO_F16) f = __half2float(reinterpret_cast<const __half *>(p)[i]);
  else f = __bfloat162float(reinterpret_cast<const __nv_bfloat16 *>(p)[i]);
  return Traits<T>::to_float(Traits<T>::from_float(f));
}
template <> __device__ __forceinline__ float load_param_as<float>(const void *p, int64_t i, int src_dtype) {
  if (src_dtype == PARO_F32) return reinterpret_cast<const float *>(p)[i];
  if (src_dtype == PARO_F16) return __half2float(reinterpret_cast<const __half *>(p)[i]);
  return __bfloat162float(reinterpret_cast<const __nv_bfloat16 *>(p)[i]);
}

// The reference's Givens update (rotation.cuh:46-58,136-153; SASS of its build):
//   yi = fma(c, a, s*b)   yj = fma(c, b, s*(-a))     -- fp32, .ftz under --use_fast_math
__device__ __forceinline__ void givens(float c, float s, float a, float b, float &yi, float &yj) {
  yi = fmaf(c, a, s * b);
  yj = fmaf(c, b, s * -a);
}

// ------------------------------------------------------------------ PTX wrappers
__device__ __forceinline__ uint32_t smem_u32(const void *p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count));
}
__device__ __forceinline__ void fence_mbar_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint32_t bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(ok)
      : "r"(bar), "r"(parity)
      : "memory");
  return ok != 0;
}
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
  while (!mbar_try_wait(bar, parity)) {
  }
}

// L2 policy for data streamed exactly once (the packed weights)
__device__ __forceinline__ uint64_t policy_evict_first() {
  uint64_t pol;
  asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(pol));
  return pol;
}

// TMA bulk copy global -> shared, completion on an mbarrier (SASS: UBLKCP)
__device__ __forceinline__ void bulk_g2s(uint32_t dst_smem, const void *src, uint32_t bytes, uint32_t bar,
                                         uint64_t policy) {
  asm volatile(
      "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1], %2, [%3], %4;"
      ::"r"(dst_smem), "l"(src), "r"(bytes), "r"(bar), "l"(policy)
      : "memory");
}

// generic-proxy writes to shared memory must be fenced before the async proxy (TMA) reuses it
__device__ __forceinline__ void fence_proxy_async_smem() {
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}

// Programmatic dependent launch: everything before pdl_wait() may overlap the previous kernel in
// the stream; nothing written by that kernel may be read before it.
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void pdl_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }

__device__ __forceinline__ uint4 lds128(uint32_t addr) {
  uint4 v;
  asm volatile("ld.shared.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "r"(addr));
  return v;
}
__device__ __forceinline__ uint32_t lds32(uint32_t addr) {
  uint32_t v;
  asm volatile("ld.shared.u32 %0, [%1];" : "=r"(v) : "r"(addr));
  return v;
}
__device__ __forceinline__ uint32_t lds16(uint32_t addr) {
  uint16_t v;
  asm volatile("ld.shared.u16 %0, [%1];" : "=h"(v) : "r"(addr));
  return v;
}
__device__ __forceinline__ void sts32(uint32_t addr, uint32_t v) {
  asm volatile("st.shared.u32 [%0], %1;" ::"r"(addr), "r"(v) : "memory");
}
__device__ __forceinline__ void sts16(uint32_t addr, uint16_t v) {
  asm volatile("st.shared.u16 [%0], %1;" ::"r"(addr), "h"(v) : "memory");
}

}  // namespace paro
