// Fused small-M path (M <= 16): scaled pairwise rotation of x + INT4 group dequant + GEMV/GEMM, for ONE linear
// or a CHAIN of up to PARO_CHAIN_MAX_STEPS linears with their element-wise neighbours folded in, in ONE launch of ONE
// persistent CTA per SM.  Replaces the reference's rotate -> Marlin kernel pairs
// (/root/reference/paroquant/inference/backends/vllm/plugin.py:281-311) and, for a chain, the launches vLLM puts
// between them (fused_add_rms_norm before qkv / gate_up, silu_and_mul before down; call sites of plugin.py:304-310).
//
// Formulation (operand-swapped, as the large-M kernel): D[n, m] += W[n, k] * x_rot[m, k]
//   A = 128 output columns x 128 channels (one quantisation group) per ROUND, dequantised by CUDA cores straight
//       into mma.sync A fragments (registers); warp = one 16-row tile of the block x one 64-channel half of every round.
//   B = x_rot of the CTA's K-slice, written once per step after the in-kernel rotation, K-major core-matrix order, read
//       as mma.sync B fragments.  For M <= 8 only 8 token rows are stored (one n8 tile).
//   D = fp32 [16 x 16] per warp in registers over the rounds of a SEGMENT (a run of one 128-column block's groups); at
//       the segment's end every warp writes its k half to one of kStmDBufs shared-memory accumulators and a dedicated
//       epilogue warp group adds the two halves (fixed order) off the workers' critical path.
//
// Work split (no clusters; every SM works): the CTAs are dealt to `c` K-slices (whole groups, ragged), inside a slice
// to the partitions of a merged linear (proportional to their 128-column blocks), and inside such a TEAM the rounds
// (block-major, group-minor) are cut into equal contiguous runs -- a CTA's run may start and end in the middle of a
// block.  Every (block, contributor) partial goes to its own fp32 slot in the workspace; the LAST contributor to
// arrive on the block's counter adds the slots in their fixed order (bit-reproducible whoever comes last), rounds once
// to T, adds the bias in T (plugin.py:309-310), applies the step's epilogue and stores.
//
// Chain: step i + 1 may take its x from step i.  The weight stream does not depend on activations, so the TMA
// producer runs ahead across step boundaries (the ring holds the next step's first records while the current step
// drains); barrier initialisation and the instruction cache are paid once.  The only serial part
// left between dependent steps is: last block fixed up -> step counter -> x load -> rotation -> first MMA.
//   x ops:     NONE | SILU_MUL (x = T(silu(g)) * u of the [M, 2K] gate_up output) | RMSNORM (x = T(T(h * rstd) * w))
//   epilogues: STORE | ADD_RESIDUAL (h = T(y + residual) -> residual_out, per-block sum of h^2 -> the next step's rstd)
//
// Roles: warps 0..15 workers (tile = warp % 8, k half = warp / 8; they also run the rotation prologue); 4 epilogue
// warps; 1 TMA producer warp (ONE 8576-byte record per round per cp.async.bulk).
//
// Numerics: x_rot as paro_rotate.cu; W = T((q - z) * T(s)) with ONE rounding (the operand Marlin / AWQ form); fp32
// accumulation; one rounding to T.
#include <cstdio>
#include <cstring>
#include <type_traits>
#include <vector>

#include "paro_launch.h"
#include "paro_tc_common.cuh"

namespace paro {

constexpr int kStmMaxSteps = PARO_CHAIN_MAX_STEPS;
constexpr int kStmMaxStages = 24;
constexpr int kStmSets = 4;    // worker warps = 4 x sets = 8 row tiles x 2 k halves
constexpr int kStmDBufs = 2;   // segment accumulators handed to the epilogue group: [kStmDBufs][k half][M][128] fp32
constexpr int kStmSmemLimit = 227 * 1024;
// ring stage = one record: StreamParams::stage_bytes = the largest record of the chain's steps (8576, or 8960 with group_size 64)
constexpr int kStmBarBytes = 16 * kStmMaxStages + 320;   // barriers (32 bytes after the ring's) + 16 rstd floats at +224
constexpr int kStmMiscBytes = 4096;              // epilogue scratch: per warp, 64 segments x {block, global block, contributors, my slot | reducer}

constexpr int kStmTraceSlots = 12;
constexpr int kStmTraceCtas = 160;
__device__ unsigned long long g_stm_trace[kStmTraceCtas * kStmMaxSteps * kStmTraceSlots];
#define STM_TRACE(step, slot)                                                                                            \
  do {                                                                                                                   \
    if (p.trace && lane == 0 && blockIdx.x < kStmTraceCtas)                                                              \
      g_stm_trace[(blockIdx.x * kStmMaxSteps + (step)) * kStmTraceSlots + (slot)] = static_cast<unsigned long long>(clock64() - t_entry); \
  } while (0)

struct StepDesc {
  const uint8_t *packed;
  const void *x;            // [M, x_ld] of T (SILU_MUL: gate at column k, up at column K + k)
  void *y;                  // [M, N] of T, may be null with ADD_RESIDUAL
  const void *bias;
  const void *res_in;       // ADD_RESIDUAL: [M, N]
  void *res_out;            // ADD_RESIDUAL: [M, N]  h = T(y + res_in)
  const void *norm_w;       // RMSNORM: [K]
  const uint2 *x_ll;        // x produced by an earlier step of this launch: [M, x_ld] {T bits, tag} words (else null: read x)
  const uint2 *stats_in;    // RMSNORM: [stats_in_blocks = 4 x blocks][M] {partial sum of h^2, tag} written by the producing step
  uint2 *stats_ll;          // ADD_RESIDUAL whose h a later step normalises: [blocks_total][4 warps][M] {sum of h^2, tag}
  uint2 *out_ll;            // a later step consumes this step's output: [M, N] {T bits, tag}
  uint2 *slots;             // [blocks_total][max_slots][M][128] {fp32 partial, tag}
  uint2 *tp_slots[PARO_TP_MAX_RANKS];   // row-parallel step under tensor parallelism: every rank's [2][blocks_total][world][M][128]
  int tp_world, tp_rank;    // {this rank's block sum, tag} buffer (peer memory over NVLink); tp_world <= 1: none
  float eps;
  int x_op, epi_op;
  int stats_in_blocks;
  int x_ld;
  Layout L;                 // the packed linear (paro_layout.h)
  int c, T, max_slots;
  int part_cta_begin[PARO_MAX_PARTS + 1];   // members u of a slice (u = cta / c) dealt to the partitions
};

struct StreamParams {
  int n_steps, M;
  int nstages, nrows_b;       // ring stages; B-operand rows stored per group (8 or 16)
  int rot_bytes, rot_warps;
  int xb_off, rot_off, misc_off, dbuf_off, bar_off;
  int trace, inflight;        // inflight: bulk copies outstanding per SM
  int stage_bytes;            // ring stage stride
  uint32_t *sync;             // [0] epoch (tag of a launch = epoch + 1), [1] CTAs done
  StepDesc steps[kStmMaxSteps];
};
static_assert(sizeof(StreamParams) <= 4096, "kernel parameters are limited to 4 KB");

// ---- where a CTA works in a step
struct StepGeom {
  int active, part, slice, t, Tp;
  int g_begin, ng, blocks_p, r0, r1;
};

__device__ __forceinline__ StepGeom step_geom(const StepDesc &S, int cta) {
  StepGeom g;
  g.active = 0; g.part = 0; g.slice = 0; g.t = 0; g.Tp = 1; g.g_begin = 0; g.ng = 0; g.blocks_p = 0; g.r0 = 0; g.r1 = 0;
  if (cta >= S.c * S.T) return g;
  const int u = static_cast<int>(static_cast<unsigned>(cta) / static_cast<unsigned>(S.c));
  g.slice = cta - u * S.c;
  int part = 0;
  while (u >= S.part_cta_begin[part + 1]) ++part;
  g.part = part;
  g.t = u - S.part_cta_begin[part];
  g.Tp = S.part_cta_begin[part + 1] - S.part_cta_begin[part];
  g.g_begin = static_cast<int>(static_cast<unsigned>(g.slice * S.L.groups) / static_cast<unsigned>(S.c));
  g.ng = static_cast<int>(static_cast<unsigned>((g.slice + 1) * S.L.groups) / static_cast<unsigned>(S.c)) - g.g_begin;
  g.blocks_p = S.L.part_block_begin[part + 1] - S.L.part_block_begin[part];
  // 32-bit on purpose (a 64-bit division is a ~150-instruction subroutine on the GPU): the host checks Rp * Tp < 2^31
  const unsigned Rp = static_cast<unsigned>(g.blocks_p * g.ng), Tp = static_cast<unsigned>(g.Tp);
  g.r0 = static_cast<int>(static_cast<unsigned>(g.t) * Rp / Tp);
  g.r1 = static_cast<int>(static_cast<unsigned>(g.t + 1) * Rp / Tp);
  g.active = g.r1 > g.r0;
  return g;
}
// member of a team of Tp over Rp rounds that owns round r (inverse of r0 = t * Rp / Tp)
__host__ __device__ __forceinline__ int round_owner(int r, int Rp, int Tp) {
  return static_cast<int>((static_cast<unsigned>(r + 1) * static_cast<unsigned>(Tp) - 1u) / static_cast<unsigned>(Rp));
}

// The segments of a CTA's run, in the order every role walks them: the run is cut at block boundaries; when it holds whole
// blocks AND a trailing partial one, the trailing partial block goes right after the leading one -- the blocks shared with
// the neighbouring team members are then finished early in the step and only whole blocks (which need the other K slices'
// partials, nothing else) are left for the end.
struct SegWalk {
  int r0, r1, ng, a, z, nseg, lead, trail_at;   // a / z: first / last block boundary inside the run
};
__device__ __forceinline__ SegWalk seg_walk(const StepGeom &g) {
  SegWalk w;
  w.r0 = g.r0; w.r1 = g.r1; w.ng = g.ng;
  const unsigned ng = static_cast<unsigned>(g.ng);
  w.a = static_cast<int>((static_cast<unsigned>(g.r0) + ng - 1u) / ng * ng);
  w.z = static_cast<int>(static_cast<unsigned>(g.r1) / ng * ng);
  if (w.a >= g.r1) {   // the run lies inside one block
    w.nseg = 1; w.lead = 1; w.trail_at = -1; w.a = g.r1; w.z = g.r1;
    return w;
  }
  const int nfull = (w.z - w.a) / g.ng;
  w.lead = g.r0 < w.a ? 1 : 0;
  const int trail = w.z < g.r1 ? 1 : 0;
  w.nseg = w.lead + nfull + trail;
  w.trail_at = trail ? (nfull > 0 ? w.lead : w.nseg - 1) : -1;
  return w;
}
__device__ __forceinline__ void seg_range(const SegWalk &w, int k, int &ra, int &rb) {
  if (w.trail_at == k) { ra = w.z; rb = w.r1; return; }
  if (k < w.lead) { ra = w.r0; rb = w.a; return; }
  const int f = k - w.lead - (w.trail_at >= 0 && k > w.trail_at ? 1 : 0);
  ra = w.a + f * w.ng;
  rb = ra + w.ng;
}

// {value, tag} words: relaxed, naturally aligned 8-byte vector accesses at GPU scope; the tag validates the value.  (The hardware
// performs an aligned .v2.u32 as one 8-byte transaction -- the property NCCL's LL protocol is built on.  Scalar .u64 accesses,
// which the PTX model guarantees to be single-copy atomic, were measured: same results, but the chain got 13 % slower.)
__device__ __forceinline__ uint32_t ld_relaxed_u32(const uint32_t *ptr) {
  uint32_t v;
  asm volatile("ld.relaxed.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(ptr) : "memory");
  return v;
}
__device__ __forceinline__ uint2 ld_relaxed_v2(const uint2 *ptr) {
  uint2 v;
  asm volatile("ld.relaxed.gpu.global.v2.u32 {%0, %1}, [%2];" : "=r"(v.x), "=r"(v.y) : "l"(ptr) : "memory");
  return v;
}
__device__ __forceinline__ uint4 ld_relaxed_v4(const uint4 *ptr) {
  uint4 v;
  asm volatile("ld.relaxed.gpu.global.v4.u32 {%0, %1, %2, %3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(ptr) : "memory");
  return v;
}
__device__ __forceinline__ void st_relaxed_v2(uint2 *ptr, uint32_t a, uint32_t b) {
  asm volatile("st.relaxed.gpu.global.v2.u32 [%0], {%1, %2};" ::"l"(ptr), "r"(a), "r"(b) : "memory");
}

// Adds n sources of {fp32 value, tag} words, source k / row m at src[(k * M + m) * 128], into acc[m] in source order.  A word
// whose tag is not this launch's is re-read (`wait`) or makes the function give up (returns false).  SYS: the words are
// written by peer GPUs over NVLink (system scope).
template <bool SYS> __device__ __forceinline__ uint2 ll_load(const uint2 *ptr) {
  uint2 v;
  if constexpr (SYS) asm volatile("ld.relaxed.sys.global.v2.u32 {%0, %1}, [%2];" : "=r"(v.x), "=r"(v.y) : "l"(ptr) : "memory");
  else asm volatile("ld.relaxed.gpu.global.v2.u32 {%0, %1}, [%2];" : "=r"(v.x), "=r"(v.y) : "l"(ptr) : "memory");
  return v;
}
template <bool SYS, int MB>
__device__ __forceinline__ bool ll_sum(const uint2 *src, int n, int M, uint32_t tag, bool wait, float (&acc)[MB]) {
  bool ready = true;
  if constexpr (MB == 1) {
    for (int k0 = 0; k0 < n && ready; k0 += 8) {   // 8 sources in flight
      uint2 w[8];
      bool ok;
      do {
        ok = true;
#pragma unroll
        for (int kk = 0; kk < 8; ++kk)
          if (k0 + kk < n) {
            w[kk] = ll_load<SYS>(src + (k0 + kk) * 128);
            ok = ok && w[kk].y == tag;
          }
      } while (!ok && wait);
      ready = ok;
#pragma unroll
      for (int kk = 0; kk < 8; ++kk)
        if (k0 + kk < n) acc[0] += __uint_as_float(w[kk].x);
    }
  } else {
    constexpr int RB = MB < 8 ? MB : 8;   // rows in flight
    for (int k = 0; k < n && ready; ++k) {   // one source at a time
#pragma unroll
      for (int h = 0; h < MB / RB; ++h) {
        if (RB * h < M && ready) {
          uint2 w[RB];
          bool ok;
          do {
            ok = true;
#pragma unroll
            for (int m = 0; m < RB; ++m)
              if (RB * h + m < M) {
                w[m] = ll_load<SYS>(src + (k * M + RB * h + m) * 128);
                ok = ok && w[m].y == tag;
              }
          } while (!ok && wait);
          ready = ok;
#pragma unroll
          for (int m = 0; m < RB; ++m)
            if (RB * h + m < M) acc[RB * h + m] += __uint_as_float(w[m].x);
        }
      }
    }
  }
  return __all_sync(0xFFFFFFFFu, ready);   // a warp handles its 32 columns on its own
}
__device__ __forceinline__ void st_relaxed_sys_v2(uint2 *ptr, uint32_t a, uint32_t b) {
  asm volatile("st.relaxed.sys.global.v2.u32 [%0], {%1, %2};" ::"l"(ptr), "r"(a), "r"(b) : "memory");
}

// ------------------------------------------------------------------ prologue: the x op (rotation_tasks does the rest; norm2 and
// silu_mul2 are in paro_tc_common.cuh)
// rstd[m] = rsqrt(mean(h^2) + eps) of every row from the producing step's per-(block, warp) partial sums, in a fixed order:
// lane-strided serial sums, then a butterfly.  ONE warp per CTA polls the words (every consumer CTA needs the same 1 KB: all
// warps of all CTAs polling it made those L2 lines a hot spot) and leaves the result in shared memory.
__device__ __forceinline__ void stm_rstd(const StepDesc &S, int M, int lane, uint32_t tag, uint32_t rstd_smem) {
  const int nb = S.stats_in_blocks;
  for (int m = 0; m < M; ++m) {
    float s = 0.f;
    for (int b0 = lane; b0 < nb; b0 += 128) {   // four words in flight per lane (o / down: 4 x 32 blocks = 128 words)
      uint2 e[4];
      bool ok;
      do {
        ok = true;
#pragma unroll
        for (int u = 0; u < 4; ++u)
          if (b0 + 32 * u < nb) {
            e[u] = ld_relaxed_v2(S.stats_in + (b0 + 32 * u) * M + m);
            ok = ok && e[u].y == tag;
          }
      } while (!ok);
#pragma unroll
      for (int u = 0; u < 4; ++u)
        if (b0 + 32 * u < nb) s += __uint_as_float(e[u].x);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xFFFFFFFFu, s, o);
    if (lane == 0) sts_f32(rstd_smem + 4 * m, rsqrtf(s / static_cast<float>(S.L.K) + S.eps));
  }
}

// 4 consecutive {T bits, tag} words -> two packed T2 words; false if any tag is stale
__device__ __forceinline__ bool ll_unpack4(uint4 a, uint4 b, uint32_t tag, uint2 &out) {
  out.x = (a.x & 0xFFFFu) | (a.z << 16);
  out.y = (b.x & 0xFFFFu) | (b.z << 16);
  return a.y == tag && a.w == tag && b.y == tag && b.w == tag;
}

// this lane's 4 channels of group gk for rows m0 .. m0 + ROWS - 1, after the step's x op.  When x comes from an earlier
// step of this launch it is read as {value, tag} words and re-read until every tag is this launch's.
template <typename T, int ROWS>
__device__ __forceinline__ void stm_load_x(const StepDesc &S, int M, int gk, int lane, uint2 (&raw)[ROWS], int m0, uint32_t tag, uint32_t rstd_smem) {
  const int col = gk * kGroup + 4 * lane;
  const bool silu = S.x_op == PARO_XOP_SILU_MUL;
  uint2 nw = make_uint2(0u, 0u);   // RMSNorm weights: fetched before x is waited for (x arrives last)
  if (S.x_op == PARO_XOP_RMSNORM) nw = *reinterpret_cast<const uint2 *>(static_cast<const T *>(S.norm_w) + col);
  uint2 up[ROWS];
  if (S.x_ll) {
    bool ok;
    do {
      ok = true;
#pragma unroll
      for (int m = 0; m < ROWS; ++m) {
        raw[m] = make_uint2(0u, 0u);
        up[m] = make_uint2(0u, 0u);
        if (m0 + m < M) {
          const uint4 *src = reinterpret_cast<const uint4 *>(S.x_ll + static_cast<int64_t>(m0 + m) * S.x_ld + col);
          ok = ll_unpack4(ld_relaxed_v4(src), ld_relaxed_v4(src + 1), tag, raw[m]) && ok;
          if (silu) {
            const uint4 *su = reinterpret_cast<const uint4 *>(S.x_ll + static_cast<int64_t>(m0 + m) * S.x_ld + S.L.K + col);
            ok = ll_unpack4(ld_relaxed_v4(su), ld_relaxed_v4(su + 1), tag, up[m]) && ok;
          }
        }
      }
      if (!ok) __nanosleep(64);   // every CTA of a K slice polls the same words: do not hammer their L2 lines
    } while (!ok);
  } else {
    const T *xg = static_cast<const T *>(S.x) + col;
#pragma unroll
    for (int m = 0; m < ROWS; ++m) {
      raw[m] = make_uint2(0u, 0u);
      up[m] = make_uint2(0u, 0u);
      if (m0 + m < M) {
        raw[m] = __ldcg(reinterpret_cast<const uint2 *>(xg + static_cast<int64_t>(m0 + m) * S.x_ld));
        if (silu) up[m] = __ldcg(reinterpret_cast<const uint2 *>(xg + static_cast<int64_t>(m0 + m) * S.x_ld + S.L.K));
      }
    }
  }
  if (silu) {
#pragma unroll
    for (int m = 0; m < ROWS; ++m) {
      if (m0 + m < M) {
        raw[m].x = silu_mul2<T>(raw[m].x, up[m].x);
        raw[m].y = silu_mul2<T>(raw[m].y, up[m].y);
      }
    }
  } else if (S.x_op == PARO_XOP_RMSNORM) {
    const uint2 w = nw;
#pragma unroll
    for (int m = 0; m < ROWS; ++m) {
      if (m0 + m < M) {   // warp-uniform
        const float rstd = lds_f32(rstd_smem + 4 * (m0 + m));   // one warp per CTA formed it (stm_rstd)
        raw[m].x = norm2<T>(raw[m].x, rstd, w.x);
        raw[m].y = norm2<T>(raw[m].y, rstd, w.y);
      }
    }
  }
}

// ------------------------------------------------------------------ the kernel
// MB: compile-time bound on the rows (M <= MB in {1, 4, 16}) -- sizes the epilogue's per-row registers
template <typename T, int SETS, int MB>
__global__ void __launch_bounds__(32 * (4 * SETS + 5), 1) stream_kernel(const __grid_constant__ StreamParams p) {
  static_assert(SETS == 4, "the workers are 8 row tiles x 2 k halves");
  static_assert(SETS % 2 == 0, "the ring depth is a multiple of SETS; the round loop takes records in pairs that must not wrap");
  extern __shared__ __align__(128) uint8_t smem[];
  constexpr int kWorkers = 4 * SETS;
  constexpr int kEpiWarp0 = kWorkers, kProdWarp = kWorkers + 4;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int cta = blockIdx.x;
  const long long t_entry = clock64();
  const int NS = p.nstages, NR = p.nrows_b, M = p.M, nsteps = p.n_steps;
  const uint32_t smem0 = smem_u32(smem);
  const uint32_t xb = smem0 + p.xb_off, bars = smem0 + p.bar_off, dbuf = smem0 + p.dbuf_off;
  const uint32_t bar_wfull = bars, bar_wempty = bars + 8 * kStmMaxStages;
  const uint32_t bar_dfull = bars + 16 * kStmMaxStages, bar_dfree = bar_dfull + 16;
  const uint32_t dbuf_bytes = 2u * M * 512;   // one segment accumulator: [k half][M][128] fp32

  if (warp == kProdWarp) {
    // every worker warp consumes every ring stage and contributes to every segment accumulator
    ring_init(bar_wfull, bar_wempty, NS, kWorkers, lane);
    if (lane < kStmDBufs) {
      mbar_init(bar_dfull + 8 * lane, kWorkers);
      mbar_init(bar_dfree + 8 * lane, 4);
    }
    fence_mbar_init();
  }
  __syncthreads();
  pdl_launch_dependents();   // the next kernel in the stream may start its own prologue as soon as SMs free up

  if (warp == kProdWarp) {
    // ================= producer: ONE bulk copy per round; nothing here depends on activations, so it runs ahead across
    // step boundaries.  The whole warp runs the loop, an elected lane issues.
    const uint64_t pol = policy_evict_first();
    RingProducer prod = {bar_wfull, bar_wempty, smem0, static_cast<uint32_t>(p.stage_bytes), NS, 0, 0};
    int lag_st = 0, lag_it = 0;   // stage / wrap of copy number (issued - inflight)
    uint32_t issued = 0;
#pragma unroll 1
    for (int i = 0; i < nsteps; ++i) {
      const StepDesc &S = p.steps[i];
      const StepGeom g = step_geom(S, cta);
      if (!g.active) continue;
      const uint32_t rec_bytes = static_cast<uint32_t>(S.L.rec_bytes);
      const uint8_t *rec_part = S.packed + S.L.rec_off + (static_cast<size_t>(S.L.part_block_begin[g.part]) * S.L.groups + g.g_begin) * rec_bytes;
      const SegWalk sw = seg_walk(g);
#pragma unroll 1
      for (int k = 0; k < sw.nseg; ++k) {
        int ra, rb;
        seg_range(sw, k, ra, rb);
        const int jb = static_cast<int>(static_cast<unsigned>(ra) / static_cast<unsigned>(g.ng));
        int gi = ra - jb * g.ng;
#pragma unroll 1
        for (int r = ra; r < rb; ++r, ++gi) {
          // at most `inflight` records outstanding per SM (the stage of copy n - inflight has not been reused yet)
          if (issued >= static_cast<uint32_t>(p.inflight)) mbar_wait(bar_wfull + 8 * lag_st, lag_it & 1);
          prod.issue([=, &S] { return rec_part + (static_cast<size_t>(jb) * S.L.groups + gi) * rec_bytes; }, rec_bytes, pol, [] {});
          if (++issued > static_cast<uint32_t>(p.inflight)) {
            if (++lag_st == NS) { lag_st = 0; ++lag_it; }
          }
        }
      }
    }
  } else if (warp >= kEpiWarp0) {
    // ================= epilogue group (4 warps, thread = one of the block's 128 columns; each warp works alone on its 32 columns):
    // D -> {partial, tag} slot; the block's REDUCER (in K slice `block mod c`, the contributor that holds the block's last round)
    // looks at the other contributors' slots, adds them in fixed order, finishes the block and publishes it for the next step,
    // again as {value, tag} words.  No fences, no counters: every 8-byte word carries the launch's tag, a reader retries
    // until the tag matches.
    const int q = warp & 3;
    const int L128 = 32 * q + lane;
    int d = 0, duse = 0;
    uint32_t tag = 0;
    bool have_tag = false;
#pragma unroll 1
    for (int i = 0; i < nsteps; ++i) {
      const StepDesc &S = p.steps[i];
      const StepGeom g = step_geom(S, cta);
      if (!g.active) continue;
      const int n_end = S.L.part_col_begin[g.part + 1];
      const SegWalk sw = seg_walk(g);
      const bool tp = S.tp_world > 1;
      // Every segment's accumulator goes to its slot as soon as it completes -- nothing ever waits before that, so
      // contributors cannot queue behind each other.  A block this CTA reduces stays PENDING until all its contributors'
      // slots carry this launch's tag; pending blocks are looked at (one non-blocking look each) while the group waits for
      // the next accumulator, and after the last segment until none is left.
      unsigned long long pending = 0ull, pushed_mask = 0ull;

      // who contributes to a segment's block: per slice, the team members whose runs overlap it (fixed order); am I its
      // reducer.  Integer divisions galore, so every lane works this out for two segments while the warp has nothing else to
      // do (before the step's first accumulator) and parks it in shared memory: one 16-byte load per look afterwards.
      const uint32_t seg_tab = smem0 + p.misc_off + q * 1024;
      for (int k = lane; k < sw.nseg && k < 64; k += 32) {
        int ra, rb;
        seg_range(sw, k, ra, rb);
        const int jb = static_cast<int>(static_cast<unsigned>(ra) / static_cast<unsigned>(g.ng));
        const int gb = S.L.part_block_begin[g.part] + jb;
        int total = 0, myslot = 0;
        unsigned gs0 = 0;
        for (int sl = 0; sl < S.c; ++sl) {
          const unsigned gs1 = static_cast<unsigned>((sl + 1) * S.L.groups) / static_cast<unsigned>(S.c);
          const int ngs = static_cast<int>(gs1 - gs0);
          gs0 = gs1;
          const int Rp = g.blocks_p * ngs;
          const int lo = round_owner(jb * ngs, Rp, g.Tp), hi = round_owner((jb + 1) * ngs - 1, Rp, g.Tp);
          // a team with more members than rounds (Tp > Rp) has members without a round between lo and hi: then every round
          // of the block has its own owner, who contributes slot (round - first round of the block)
          const int n = hi - lo + 1 < ngs ? hi - lo + 1 : ngs;
          if (sl == g.slice) myslot = total + (n < hi - lo + 1 ? ra - jb * ngs : g.t - lo);
          total += n;
        }
        // the reducer: in slice (block mod c), the member that holds the block's last round there (spread over the slices)
        const bool reducer = static_cast<unsigned>(g.slice) == static_cast<unsigned>(gb) % static_cast<unsigned>(S.c) && rb == (jb + 1) * g.ng;
        sts128u(seg_tab + 16 * k, make_uint4(static_cast<uint32_t>(jb), static_cast<uint32_t>(gb), static_cast<uint32_t>(total),
                                             static_cast<uint32_t>(myslot) | (reducer ? 0x80000000u : 0u)));
      }
      __syncwarp();
      auto block_info = [&](int k, int &jb, int &gb, int &total, int &myslot, bool &reducer) {
        const uint4 e = lds128(seg_tab + 16 * k);
        jb = static_cast<int>(e.x);
        gb = static_cast<int>(e.y);
        total = static_cast<int>(e.z);
        myslot = static_cast<int>(e.w & 0x7FFFFFFFu);
        reducer = (e.w >> 31) != 0u;
      };

      // add the block's slots: stage 1 this GPU's contributors, stage 2 (tensor parallelism) the ranks' sums.  Returns false
      // if something is missing (`wait` = false: one look).
      auto sum_block = [&](int gb, int total, unsigned long long bit, float (&acc)[MB]) -> bool {
        const bool pushed = (pushed_mask & bit) != 0ull;
        if (S.epi_op == PARO_EPI_ADD_RESIDUAL) {   // warm the residual lines this block's finish will read (they sit in L2)
          const int n = S.L.part_col_begin[g.part] + (gb - S.L.part_block_begin[g.part]) * kBlockN + L128;
          if (n < n_end) asm volatile("prefetch.global.L2 [%0];" ::"l"(static_cast<const T *>(S.res_in) + n));
        }
        if (!pushed) {
#pragma unroll
          for (int m = 0; m < MB; ++m) acc[m] = 0.f;
          if (!ll_sum<false, MB>(S.slots + static_cast<size_t>(gb) * S.max_slots * (M * 128) + L128, total, M, tag, false, acc)) return false;
        }
        if (tp) {
          // my block sum goes to every rank (mine included), then the `world` sums are added in rank order -- every rank
          // computes the same bits.  Nothing waits before the push.  Buffers alternate with the launch parity: a rank that
          // is one launch ahead writes the other half while this one is still reading.
          const size_t blk = (static_cast<size_t>(tag & 1u) * S.L.blocks_total + gb) * S.tp_world;
          if (!pushed) {
            for (int rk = 0; rk < S.tp_world; ++rk) {
              uint2 *dst = S.tp_slots[rk] + (blk + S.tp_rank) * (M * 128) + L128;
#pragma unroll
              for (int m = 0; m < MB; ++m)
                if (m < M) st_relaxed_sys_v2(dst + m * 128, __float_as_uint(acc[m]), tag);
            }
            pushed_mask |= bit;
          }
#pragma unroll
          for (int m = 0; m < MB; ++m) acc[m] = 0.f;
          if (!ll_sum<true, MB>(S.tp_slots[S.tp_rank] + blk * (M * 128) + L128, S.tp_world, M, tag, false, acc)) return false;
        }
        return true;
      };

      // round once to T, bias, epilogue, publish for the next step
      auto finish_block = [&](int jb, int gb, float (&acc)[MB]) {
        if (warp == kEpiWarp0) STM_TRACE(i, 9);
        const int n = S.L.part_col_begin[g.part] + jb * kBlockN + L128;
        const bool ok = n < n_end;
        const bool add_res = S.epi_op == PARO_EPI_ADD_RESIDUAL;
#pragma unroll
        for (int m = 0; m < MB; ++m) {
          float sq = 0.f;
          if (m < M && ok) {
            T t = Traits<T>::from_float(acc[m]);
            if (S.bias) t = Traits<T>::from_float(Traits<T>::to_float(t) + Traits<T>::to_float(static_cast<const T *>(S.bias)[n]));  // plugin.py:309-310
            const int64_t o = static_cast<int64_t>(m) * S.L.N + n;
            if (S.y) static_cast<T *>(S.y)[o] = t;
            if (add_res) {
              t = Traits<T>::from_float(Traits<T>::to_float(t) + Traits<T>::to_float(static_cast<const T *>(S.res_in)[o]));
              static_cast<T *>(S.res_out)[o] = t;
              const float hf = Traits<T>::to_float(t);
              sq = hf * hf;
            }
            if (S.out_ll) st_relaxed_v2(S.out_ll + o, T_to_bits<T>(t), tag);   // what the next step consumes
          }
          acc[m] = sq;
        }
        if (add_res && S.stats_ll) {
          // per-row sum of h^2 over this warp's 32 columns (butterfly): one {sum, tag} word per (block, warp, row)
#pragma unroll
          for (int m = 0; m < MB; ++m) {
            if (m < M) {
              float sm = acc[m];
#pragma unroll
              for (int o = 16; o > 0; o >>= 1) sm += __shfl_xor_sync(0xFFFFFFFFu, sm, o);
              if (lane == 0) st_relaxed_v2(S.stats_ll + (gb * 4 + q) * M + m, __float_as_uint(sm), tag);
            }
          }
        }
      };

#pragma unroll 1
      for (int k = 0; k <= sw.nseg; ++k) {     // k == nseg: drain what is still pending
        // ---- wait for D of segment k; meanwhile (except before the step's last segment, whose D must not be kept waiting)
        // look at the pending blocks, one non-blocking look each
#pragma unroll 1
        for (;;) {
          if (k < sw.nseg) {
            if (mbar_try_wait(bar_dfull + 8 * d, duse & 1)) break;
            if (k + 1 == sw.nseg || pending == 0ull) {
              mbar_wait(bar_dfull + 8 * d, duse & 1);
              break;
            }
          } else if (pending == 0ull) {
            break;
          }
#pragma unroll 1
          for (int kk = 0; kk < sw.nseg; ++kk) {
            const unsigned long long pb = 1ull << kk;
            if (pending & pb) {
              int jb, gb, total, myslot;
              bool reducer;
              block_info(kk, jb, gb, total, myslot, reducer);
              float acc[MB];
              if (sum_block(gb, total, pb, acc)) {
                finish_block(jb, gb, acc);
                pending &= ~pb;
              }
            }
          }
        }
        if (k == sw.nseg) break;
        if (warp == kEpiWarp0) STM_TRACE(i, 8);
        if (!have_tag) {   // the workers are past griddepcontrol.wait: the previous launch has bumped the epoch
          tag = ld_relaxed_u32(p.sync) + 1u;
          have_tag = true;
        }
        uint32_t v[MB] = {};
        {
          const uint32_t db = dbuf + d * dbuf_bytes + L128 * 4;   // the two k halves, added in a fixed order
#pragma unroll
          for (int m = 0; m < MB; ++m)
            if (m < M) v[m] = __float_as_uint(lds_f32(db + m * 512) + lds_f32(db + (M + m) * 512));
        }
        __syncwarp();
        if (lane == 0) mbar_arrive(bar_dfree + 8 * d);
        if (++d == kStmDBufs) { d = 0; ++duse; }
        if (warp == kEpiWarp0) STM_TRACE(i, 7);
        int jb, gb, total, myslot;
        bool reducer;
        block_info(k, jb, gb, total, myslot, reducer);
        float acc[MB];
#pragma unroll
        for (int m = 0; m < MB; ++m) acc[m] = __uint_as_float(v[m]);
        if (total == 1 && !tp) {
          finish_block(jb, gb, acc);     // nobody else contributes: straight from the accumulator
        } else {
          uint2 *slot = S.slots + (static_cast<size_t>(gb) * S.max_slots + myslot) * (M * 128) + L128;
#pragma unroll
          for (int m = 0; m < MB; ++m)
            if (m < M) st_relaxed_v2(slot + m * 128, v[m], tag);
          if (reducer) pending |= 1ull << k;
          if (warp == kEpiWarp0 && k + 1 == sw.nseg) STM_TRACE(i, 11);
        }
      }
      if (warp == kEpiWarp0) STM_TRACE(i, 6);
    }
  } else {
    // ================= workers: warp = (16-row tile of the block, k half of every record); each takes every round
    const int wi = warp, tile = warp & 7, kh = warp >> 3;
    const uint32_t rot = smem0 + p.rot_off + wi * p.rot_bytes;
    const int nq = M > 4 ? (M + 3) >> 2 : 1;   // rotation tasks: row blocks of 4 for M > 4
    uint32_t tag = 0;
    const uint32_t rstd_smem = bars + 16 * kStmMaxStages + 224;   // 16 floats behind the barriers
    const int g8 = lane >> 2, t4 = lane & 3;
    int st = 0, par = 0, d = 0, duse = 0;
#pragma unroll 1
    for (int i = 0; i < nsteps; ++i) {
      const StepDesc &S = p.steps[i];
      const StepGeom g = step_geom(S, cta);
      const int ntasks = g.active ? g.ng * nq : 0;
      const bool mine = wi < ntasks && wi < p.rot_warps;
      RotMeta rm;
      if (mine) fetch_meta(S.packed + S.L.meta_off + (static_cast<size_t>(g.part) * S.L.groups + g.g_begin + wi / nq) * S.L.meta_group_bytes, S.L.krot, lane, rm);   // flies during the waits below
      if (i == 0) {
        // rows [M, NR) of every group are zero padding of the MMA's N: cleared once (M is the same for every step)
        if (M < NR) {
          const int words = (p.rot_off - p.xb_off) >> 4;
          for (int k = threadIdx.x; k < words; k += 32 * kWorkers) sts128u(xb + k * 16, make_uint4(0u, 0u, 0u, 0u));
          named_bar_sync(1, 32 * kWorkers);
        }
        if (wi == 0) STM_TRACE(0, 0);
        pdl_wait();   // x may have been written by the previous kernel in the stream
        tag = ld_relaxed_u32(p.sync) + 1u;   // ... which has also bumped the epoch
      } else {
        named_bar_sync(2, 32 * kWorkers);   // every worker is done with the previous step's B operand
      }
      if (wi == 0) STM_TRACE(i, 1);
      if (mine) {
        if (S.x_op == PARO_XOP_RMSNORM) {
          const int nrot = ntasks < p.rot_warps ? ntasks : p.rot_warps;   // the warps that rotate in this step (warp 0 is one)
          if (wi == 0) stm_rstd(S, M, lane, tag, rstd_smem);
          named_bar_sync(3, 32 * nrot);
        }
        if (wi == 0) STM_TRACE(i, 2);
        auto stage_x = [&](auto rows, int gi, int m0, uint2 csw) {
          uint2 raw[decltype(rows)::value];
          stm_load_x<T>(S, M, g.g_begin + gi, lane, raw, m0, tag, rstd_smem);
          scale_and_stage<T>(rot, lane, raw, csw);
        };
        const uint8_t *meta = S.packed + S.L.meta_off;
        const int mi0 = g.part * S.L.groups + g.g_begin, mg = S.L.meta_group_bytes, rw = p.rot_warps;
        if constexpr (MB == 1) {
          rotation_tasks<T, 1, true>(rm, meta, mg, S.L.krot, mi0, ntasks, nq, M, wi, rw, lane, rot, xb, NR, stage_x);
        } else if constexpr (MB == 4) {
          if (M == 2) rotation_tasks<T, 2, true>(rm, meta, mg, S.L.krot, mi0, ntasks, nq, M, wi, rw, lane, rot, xb, NR, stage_x);
          else rotation_tasks<T, 4, true>(rm, meta, mg, S.L.krot, mi0, ntasks, nq, M, wi, rw, lane, rot, xb, NR, stage_x);
        } else {
          rotation_tasks<T, 4, true>(rm, meta, mg, S.L.krot, mi0, ntasks, nq, M, wi, rw, lane, rot, xb, NR, stage_x);
        }
      }
      named_bar_sync(2, 32 * kWorkers);   // B operand of this step complete
      if (wi == 0) STM_TRACE(i, 3);
      if (!g.active) continue;

      const SegWalk sw = seg_walk(g);
      if (p.trace && wi == 0 && sw.nseg > 0) {   // the step's first record has landed (waiting twice on one phase is harmless)
        mbar_wait(bar_wfull + 8 * st, par);
        STM_TRACE(i, 4);
      }
      // The round loop, specialised on the token tiles and the B rows so that neither is a per-round branch or multiply;
      // stage and parity advance by increments (`fb`: the stage's full barrier, its empty barrier sits 8 * kStmMaxStages
      // above).  Records are taken in pairs from an even stage: the ring depth is a multiple of SETS (even), so a pair
      // never wraps.  A segment starting at an odd stage takes its first record alone, an odd remainder its last.
      auto segments = [&](auto ntt, auto nr) {
        constexpr int NTT = decltype(ntt)::value, NRC = decltype(nr)::value;
        const RoundLane lo = round_lane<NRC>(S.L.qhalves == 2, tile, kh, lane);
        const uint32_t ring_end = bar_wfull + 8 * NS, stage_bytes = p.stage_bytes;
        // a stage's record from its full barrier: smem0 + (fb - bar_wfull) / 8 * stage_bytes (a multiple of 8)
        const uint32_t rec_per_bar = stage_bytes / 8, rec_at_bar0 = smem0 - bar_wfull * rec_per_bar;
        uint32_t fb = bar_wfull + 8 * st, bx;   // bx: this lane's ldmatrix row in the B operand of the next group
        float acc[2][4];
        auto take = [&](auto nrec) {
          constexpr int NREC = decltype(nrec)::value;
#pragma unroll
          for (int i = 0; i < NREC; ++i) mbar_wait(fb + 8 * i, par);
          mma_rounds<T, NTT, NREC, NRC>(fb * rec_per_bar + rec_at_bar0, stage_bytes, bx, lo, acc);
          __syncwarp();
          if (elect_one()) {
#pragma unroll
            for (int i = 0; i < NREC; ++i) mbar_arrive(fb + 8 * i + 8 * kStmMaxStages);
          }
          bx += NREC * (NRC * 256);
          fb += 8 * NREC;
          if (fb == ring_end) { fb = bar_wfull; par ^= 1; }
        };
#pragma unroll 1
        for (int k = 0; k < sw.nseg; ++k) {
          int ra, rb;
          seg_range(sw, k, ra, rb);
          const int gi = ra - static_cast<int>(static_cast<unsigned>(ra) / static_cast<unsigned>(g.ng)) * g.ng;
          bx = xb + gi * (NRC * 256) + lo.x;
#pragma unroll
          for (int e = 0; e < 8; ++e) acc[e >> 2][e & 3] = 0.f;
          int left = rb - ra;
          if (left > 0 && ((fb - bar_wfull) & 8)) { take(std::integral_constant<int, 1>{}); --left; }
          const uint32_t pairs_end = bx + (left >> 1) * (2 * NRC * 256);   // the pair loop counts with bx
#pragma unroll 1
          while (bx != pairs_end) take(std::integral_constant<int, 2>{});
          if (left & 1) take(std::integral_constant<int, 1>{});
          // ---- segment done: my k half of the accumulator to the epilogue group
          if (duse > 0) mbar_wait(bar_dfree + 8 * d, (duse - 1) & 1);
          const uint32_t db = dbuf + d * dbuf_bytes + (kh * M) * 512;
#pragma unroll
          for (int e = 0; e < 8; ++e) {
            const int col = 16 * tile + g8 + 8 * ((e >> 1) & 1), m = 8 * (e >> 2) + 2 * t4 + (e & 1);
            if (m < M) sts_f32(db + m * 512 + col * 4, acc[e >> 2][e & 3]);
          }
          __syncwarp();
          if (lane == 0) mbar_arrive(bar_dfull + 8 * d);
          if (++d == kStmDBufs) { d = 0; ++duse; }
        }
        st = static_cast<int>((fb - bar_wfull) >> 3);
      };
      using I1 = std::integral_constant<int, 1>;
      using I2 = std::integral_constant<int, 2>;
      if (M > 8) segments(I2{}, std::integral_constant<int, 16>{});
      else if (NR == 8) segments(I1{}, std::integral_constant<int, 8>{});
      else segments(I1{}, std::integral_constant<int, 16>{});
      if (wi == 0) STM_TRACE(i, 5);
    }
  }

  // ================= common tail
  __syncwarp();
  __syncthreads();
  if (threadIdx.x == 0) {
    // the last CTA to get here bumps the epoch: every tag of this launch becomes stale, the next launch on this workspace
    // (which reads the epoch after griddepcontrol.wait, i.e. after this grid has completed) uses a fresh one
    __threadfence();
    const uint32_t old = atomicAdd(p.sync + 1, 1u);
    if (old == gridDim.x - 1) {
      p.sync[1] = 0u;
      p.sync[0] = p.sync[0] + 1u;
      __threadfence();
    }
  }
}

int stream_trace_read(unsigned long long *host, int max_ctas) {
  const size_t n = static_cast<size_t>(max_ctas < kStmTraceCtas ? max_ctas : kStmTraceCtas) * kStmMaxSteps * kStmTraceSlots;
  PARO_CUDA_OK(cudaMemcpyFromSymbol(host, g_stm_trace, n * sizeof(unsigned long long)));
  return PARO_OK;
}

// ------------------------------------------------------------------ host side: plan (pure, cached), carve-up, launch
struct StepPlan {
  int c, T, max_slots, ng_max, max_rounds;
  int part_cta_begin[PARO_MAX_PARTS + 1];
};

static int stm_rot_rows(int M) { return M == 1 ? 1 : M == 2 ? 2 : 4; }
static int stm_b_rows(int M) { return (M <= 8 && knobs().b8) ? 8 : 16; }

// The plan of one step on `ctas` CTAs: the number of K slices c.  Pure host logic (tests drive it through
// paro_debug_stream_plan).  Cost in "round units" (8 per dequant round): the busiest CTA's rounds, the rotation passes of
// the prologue, a charge per contributor slot (the fix-up reads them) and a penalty when the B operand crowds the ring.
static bool stm_choose_plan(const Layout &L, int M, int sets, int ctas, int force_c, StepPlan &best) {
  long best_cost = -1;
  const int nq = M > 4 ? (M + 3) / 4 : 1;
  const int NR = stm_b_rows(M);
  for (int c = 1; c <= 16; ++c) {
    if (c > L.groups) break;
    if (force_c && c != force_c) continue;
    StepPlan pl = {};
    pl.c = c;
    pl.T = ctas / c;
    if (pl.T < 1) break;
    if (!apportion(L, pl.T, pl.part_cta_begin)) continue;   // the slice's members dealt to the partitions
    pl.ng_max = (L.groups + c - 1) / c;
    const int xb_bytes = pl.ng_max * NR * 256;
    const int nst_room = ring_stages(kStmSmemLimit - xb_bytes - 4 * sets * kGroup * 2 * stm_rot_rows(M) - kStmBarBytes - kStmMiscBytes - kStmDBufs * M * 1024 - 256,
                                     kBlockBytesMax, kStmMaxStages, sets, sets, false);
    if (!nst_room) continue;
    pl.max_rounds = 0;
    pl.max_slots = 1;
    for (int p = 0; p < L.n_parts; ++p) {
      const int blocks = L.part_block_begin[p + 1] - L.part_block_begin[p];
      const int Tp = pl.part_cta_begin[p + 1] - pl.part_cta_begin[p];
      const int mr = (blocks * pl.ng_max + Tp - 1) / Tp;
      if (mr > pl.max_rounds) pl.max_rounds = mr;
      for (int jb = 0; jb < blocks; ++jb) {
        int total = 0;
        for (int s = 0; s < c; ++s) {
          const int ngs = (s + 1) * L.groups / c - s * L.groups / c;
          const int Rp = blocks * ngs;
          // members lo..hi: an upper bound of the contributors the kernel counts (equal unless a team has more members than
          // rounds); slots are sized and the plan is priced by it
          total += round_owner((jb + 1) * ngs - 1, Rp, Tp) - round_owner(jb * ngs, Rp, Tp) + 1;
        }
        if (total > pl.max_slots) pl.max_slots = total;
      }
    }
    if (static_cast<long long>(L.blocks_total) * pl.ng_max * (ctas + 1) >= (1ll << 31)) continue;   // the kernel's 32-bit round arithmetic
    if (pl.max_rounds / (L.groups / c) + 3 > 64) continue;   // segments of a CTA's run: the epilogue's pending mask is 64 bits
    const int passes = (pl.ng_max * nq + 4 * sets - 1) / (4 * sets);
    long cost = static_cast<long>(pl.max_rounds) * 8 + passes * 24 + pl.max_slots;
    if (nst_room < 2 * sets) cost += cost / 4;
    if (best_cost < 0 || cost < best_cost) { best = pl; best_cost = cost; }
  }
  return best_cost >= 0;
}

static bool stm_cached_plan(const Layout &L, int M, int ctas, StepPlan &out) {
  static PlanCache<StepPlan> cache;
  return cache.get(L, M, ctas, out, [&](StepPlan &pl) { return stm_choose_plan(L, M, kStmSets, ctas, knobs().force_c, pl); });
}

// test hook: out[0..4] = c, T, max_slots, ng_max, max_rounds; out[5..13] = part_cta_begin
int stream_debug_plan(const Layout &L, int64_t M, int sets, int ctas, int32_t *out) {
  if (M < 1 || M > 16 || sets < 4 || sets > 6 || ctas < 1) { set_error("debug_stream_plan: bad M / sets / ctas"); return PARO_EINVAL; }
  StepPlan pl;
  if (!stm_choose_plan(L, static_cast<int>(M), sets, ctas, 0, pl)) {
    set_error("decode: no launch configuration fits (in_features=%d, M=%d)", L.K, static_cast<int>(M));
    return PARO_EUNSUPPORTED;
  }
  out[0] = pl.c; out[1] = pl.T; out[2] = pl.max_slots; out[3] = pl.ng_max; out[4] = pl.max_rounds;
  for (int i = 0; i <= PARO_MAX_PARTS; ++i) out[5 + i] = pl.part_cta_begin[i];
  return PARO_OK;
}

// Workspace: [sync words: epoch, CTAs-done counter][per step: statistics words, output words, partial slots].  Only the
// sync words carry state between launches (the epoch); everything else is validated by its tag, so linears of different
// shapes may share one workspace (the single-linear entry point does) and stale bytes are harmless.
constexpr size_t kStmSyncBytes = 256;
struct StepWs { size_t stats_off, out_off, slots_off, end; };
static StepWs stm_step_ws(const Layout &L, const StepPlan &pl, int M, size_t base, bool consumed) {
  StepWs w;
  w.stats_off = base;
  w.out_off = w.stats_off + (consumed ? (static_cast<size_t>(L.blocks_total) * 4 * M * 8 + 255) / 256 * 256 : 0);
  w.slots_off = w.out_off + (consumed ? (static_cast<size_t>(M) * L.N * 8 + 255) / 256 * 256 : 0);
  w.end = w.slots_off + static_cast<size_t>(L.blocks_total) * pl.max_slots * M * 1024;
  w.end = (w.end + 255) / 256 * 256;
  return w;
}

bool stream_supported(const Layout &L, int64_t M) { return M >= 1 && M <= 16 && L.groups >= 1; }

// bytes a single linear needs in its workspace for any M <= max_m (the sync words at the head must start as zeros and are
// never touched by the large-M path, which keeps its scratch behind them)
size_t stream_sync_bytes(const Layout &) { return kStmSyncBytes; }
size_t stream_workspace_bytes(const Layout &L, int64_t max_m) {
  size_t need = kStmSyncBytes;
  const int top = max_m < 16 ? static_cast<int>(max_m) : 16;
  for (int M = 1; M <= top; ++M) {
    StepPlan pl;
    if (!stm_cached_plan(L, M, planning_sms(), pl)) continue;
    const StepWs w = stm_step_ws(L, pl, M, kStmSyncBytes, false);
    if (w.end > need) need = w.end;
  }
  return need;
}

template <typename T, int SETS, int MB>
static int stm_launch(StreamParams &p, int max_ng, int ctas, cudaStream_t stream) {
  auto kern = stream_kernel<T, SETS, MB>;
  const Knobs &kn = knobs();
  const int M = p.M;
  p.nrows_b = stm_b_rows(M);
  p.rot_bytes = kGroup * 2 * stm_rot_rows(M);
  const int xb_bytes = max_ng * p.nrows_b * 256;
  const bool fits = fit_rot_warps(max_ng * (M > 4 ? (M + 3) / 4 : 1), SETS, [&](int rw) {
    const int rot_total = (rw * p.rot_bytes + 127) / 128 * 128;
    const int fixed = xb_bytes + rot_total + kStmMiscBytes + kStmDBufs * M * 1024 + kStmBarBytes + 128;
    const int nst = ring_stages(kStmSmemLimit - fixed, p.stage_bytes, kStmMaxStages, SETS, SETS, true);
    if (!nst) return false;
    p.nstages = nst;
    p.inflight = kn.inflight < 1 ? 1 : kn.inflight > nst - 1 ? nst - 1 : kn.inflight;
    p.rot_warps = rw;
    p.xb_off = (nst * p.stage_bytes + 127) / 128 * 128;
    p.rot_off = p.xb_off + xb_bytes;
    p.misc_off = p.rot_off + rot_total;
    p.dbuf_off = p.misc_off + kStmMiscBytes;
    p.bar_off = p.dbuf_off + kStmDBufs * M * 1024;
    return true;
  });
  if (!fits) { set_error("decode: no launch configuration fits (M=%d, %d groups per CTA)", M, max_ng); return PARO_EUNSUPPORTED; }
  const int smem_total = p.bar_off + kStmBarBytes;
  PARO_CUDA_OK(smem_opt_in(kern, kStmSmemLimit));
  if (kn.verbose) {
    for (int i = 0; i < p.n_steps; ++i)
      fprintf(stderr, "[paro stream] step %d K=%d N=%d M=%d: %d slices x %d members, <= %d slots/block, xop %d epi %d wait %d\n", i, p.steps[i].L.K,
              p.steps[i].L.N, M, p.steps[i].c, p.steps[i].T, p.steps[i].max_slots, p.steps[i].x_op, p.steps[i].epi_op, p.steps[i].x_ll ? 1 : 0);
    fprintf(stderr, "[paro stream] %d CTAs, %d stages, B rows %d, rot warps %d, smem %d\n", ctas, p.nstages, p.nrows_b, p.rot_warps, smem_total);
  }
  cudaLaunchConfig_t cfg;
  cudaLaunchAttribute attr[2];
  launch_config(cfg, attr, ctas, 32 * (4 * SETS + 5), smem_total, stream, 0, !kn.no_pdl);
  PARO_CUDA_OK(cudaLaunchKernelEx(&cfg, kern, p));
  note_launches(1);
  return PARO_OK;
}

size_t stream_chain_workspace_bytes(const HostStep *steps, int n, int64_t M) {
  size_t off = kStmSyncBytes;
  for (int i = 0; i < n; ++i) {
    StepPlan pl;
    if (!stm_cached_plan(steps[i].L, static_cast<int>(M), planning_sms(), pl)) return 0;
    const bool consumed = i + 1 < n && !steps[i + 1].x;
    off = stm_step_ws(steps[i].L, pl, static_cast<int>(M), off, consumed).end;
  }
  return off;
}

int stream_forward(const HostStep *steps, int n, int64_t M, void *workspace, size_t workspace_bytes, cudaStream_t stream) {
  const Knobs &kn = knobs();
  const int sms = device_sms();
  if (sms <= 0) { set_error("decode: no CUDA device"); return PARO_ECUDA; }
  StreamParams p;
  memset(&p, 0, sizeof(p));
  p.n_steps = n;
  p.M = static_cast<int>(M);
  p.trace = kn.trace;
  uint8_t *ws = static_cast<uint8_t *>(workspace);
  p.sync = reinterpret_cast<uint32_t *>(ws);
  size_t off = kStmSyncBytes;
  int max_ng = 1;
  const int dtype = steps[0].L.dtype;
  for (int i = 0; i < n; ++i) {
    const HostStep &h = steps[i];
    const Layout &L = h.L;
    StepPlan pl;
    if (!stm_cached_plan(L, p.M, sms, pl)) {
      set_error("decode: no launch configuration fits (in_features=%d, M=%d)", L.K, p.M);
      return PARO_EUNSUPPORTED;
    }
    const bool consumed = i + 1 < n && !steps[i + 1].x;
    const StepWs w = stm_step_ws(L, pl, p.M, off, consumed);
    if (w.end > workspace_bytes) { set_error("workspace too small: have %zu, need %zu", workspace_bytes, w.end); return PARO_EWORKSPACE; }
    off = w.end;
    StepDesc &S = p.steps[i];
    S.packed = static_cast<const uint8_t *>(h.packed);
    S.bias = h.bias;
    S.y = h.y;
    S.res_in = h.res_in; S.res_out = h.res_out; S.norm_w = h.norm_w; S.eps = h.eps;
    S.x_op = h.x_op; S.epi_op = h.epi_op;
    S.stats_ll = consumed && h.epi_op == PARO_EPI_ADD_RESIDUAL ? reinterpret_cast<uint2 *>(ws + w.stats_off) : nullptr;
    S.out_ll = consumed ? reinterpret_cast<uint2 *>(ws + w.out_off) : nullptr;
    S.slots = reinterpret_cast<uint2 *>(ws + w.slots_off);
    S.L = L;
    S.c = pl.c; S.T = pl.T; S.max_slots = pl.max_slots;
    if (L.rec_bytes > p.stage_bytes) p.stage_bytes = L.rec_bytes;
    for (int k = 0; k <= PARO_MAX_PARTS; ++k) S.part_cta_begin[k] = pl.part_cta_begin[k];
    if (h.tp && h.tp->world > 1) {
      S.tp_world = h.tp->world;
      S.tp_rank = h.tp->rank;
      for (int r = 0; r < h.tp->world; ++r) S.tp_slots[r] = static_cast<uint2 *>(h.tp->peer_slots[r]);
    }
    S.x_ld = h.x_op == PARO_XOP_SILU_MUL ? 2 * L.K : L.K;
    if (h.x) {   // the steps passed chain_check_links (paro_capi.cu)
      S.x = h.x;
    } else {
      const StepDesc &P = p.steps[i - 1];
      S.x_ll = P.out_ll;
      S.stats_in = P.stats_ll;
      S.stats_in_blocks = 4 * P.L.blocks_total;   // one partial sum per (block, epilogue warp)
    }
    if (pl.ng_max > max_ng) max_ng = pl.ng_max;
  }
  const bool bf16 = dtype == PARO_BF16;
  if (p.M == 1) return bf16 ? stm_launch<__nv_bfloat16, kStmSets, 1>(p, max_ng, sms, stream) : stm_launch<__half, kStmSets, 1>(p, max_ng, sms, stream);
  if (p.M <= 4) return bf16 ? stm_launch<__nv_bfloat16, kStmSets, 4>(p, max_ng, sms, stream) : stm_launch<__half, kStmSets, 4>(p, max_ng, sms, stream);
  return bf16 ? stm_launch<__nv_bfloat16, kStmSets, 16>(p, max_ng, sms, stream) : stm_launch<__half, kStmSets, 16>(p, max_ng, sms, stream);
}

}  // namespace paro
