// Fused small-M path (M <= 16): scaled pairwise rotation of x + INT4 group dequant + GEMV/GEMM in ONE
// launch per (merged) linear, ONE persistent CTA per SM.  Replaces the reference's
// rotate -> Marlin kernel pairs (/root/reference/paroquant/inference/backends/vllm/plugin.py:281-311).
//
// Formulation (operand-swapped, as the large-M kernel): D[n, m] += W[n, k] * x_rot[m, k]
//   A = 128 output columns x 128 channels (one quantisation group) per ROUND, dequantised by CUDA cores straight
//       into mma.sync A fragments (registers); warp = one 16-row tile of the block x one 64-channel half of every round.
//   B = x_rot of the CTA's K-slice, 16 token rows (zero-padded), written once per CTA after the in-kernel
//       rotation, K-major core-matrix order; read as mma.sync B fragments.
//   D = fp32 [16 x 16] per warp in registers over all rounds of a 128-column block; at the block's end the two
//       k-half warps of a tile add their partials through shared memory (fixed order) -- the in-CTA part of the
//       split-K reduction.
//
// Work split: the `c` CTAs of a cluster cover K (ragged slices of whole groups); a cluster walks a range
// of 128-column blocks of one partition.  Cross-slice partials are pushed through distributed shared
// memory to rank (block mod c); one cluster barrier; fixed summation order (bit-reproducible).
//
// Roles (16 worker warps + 1): warps 0..15 workers (tile = warp % 8, k half = warp / 8): the prologue rotates the
// slice's groups (tasks of one group x up to 4 token rows per warp, __syncwarp only); the main loop takes every
// round.  Warp 16: TMA producer (ONE 8576-byte record = weights + scales + zeros of a round per cp.async.bulk, into
// an mbarrier ring, issued before griddepcontrol.wait).
//
// Numerics: x_rot as paro_rotate.cu; W = T((q - z) * T(s)) with ONE rounding (the operand Marlin / AWQ
// form); fp32 accumulation; one rounding to T; bias added in T (plugin.py:309-310).
#include <cstdio>
#include <type_traits>

#include "paro_launch.h"
#include "paro_tc_common.cuh"

namespace paro {

constexpr int kDecMaxStages = 24;
constexpr int kDecSets = 4;                     // worker warps = 4 x sets = 8 row tiles x 2 k halves
constexpr int kDecWorkers = 4 * kDecSets;
constexpr int kDecN = 16;            // B operand rows per group: token rows, zero-padded
constexpr int kDecSmemLimit = 227 * 1024;
constexpr int kDecBarBytes = 16 * kDecMaxStages + 256;   // ring barriers + the x-load barrier
constexpr int kDecXchgBytes = 2 * 8 * 8 * 128;           // k-half partials: [2][8 tiles][8 values][32 lanes] fp32 (in the rotation tiles)
// one record per ring stage: 8576 bytes (group_size 128) or 8960 (group_size 64), both multiples of 64 -> Layout::rec_bytes

constexpr int kDecTraceSlots = 12;
constexpr int kDecTraceCtas = 200;       // rows 200.. of the trace double as a per-round log of CTA 0 (issued / full / consumed)
constexpr int kDecTraceRows = 256;
__device__ unsigned long long g_dec_trace[kDecTraceRows * kDecTraceSlots];
#define DEC_TRACE(slot)                                                                                      \
  do {                                                                                                       \
    if (p.trace && warp == 0 && lane == 0 && blockIdx.x < kDecTraceCtas)                                      \
      g_dec_trace[blockIdx.x * kDecTraceSlots + (slot)] = static_cast<unsigned long long>(clock64() - t_entry); \
  } while (0)

struct DecParams {
  const uint8_t *packed;
  const void *x;
  void *y;
  const void *bias;
  Layout L;                       // the packed linear (paro_layout.h); a record is one ring stage
  int M;
  int c, c_shift;                 // cluster size (K slices of this launch), log2
  int nstages, rot_bytes, rot_warps, trace;   // rot_warps: worker warps that take rotation tasks (each owns one rot_bytes tile)
  int pre_rotated;                // x is the pre-pass's output: [n_parts][M][K], already scaled and rotated (no stages here)
  long long x_part_stride;        // elements between partitions of a pre-rotated x (0 otherwise)
  int xb_off, rot_off, recv_off, bar_off;   // shared-memory carve-up (bytes)
  int part_range_begin[PARO_MAX_PARTS + 1];
};

template <typename T>
__device__ __forceinline__ void dec_store(const DecParams &p, float v, int m, int n) {
  T t = Traits<T>::from_float(v);
  if (p.bias) t = Traits<T>::from_float(Traits<T>::to_float(t) + Traits<T>::to_float(static_cast<const T *>(p.bias)[n]));  // plugin.py:309-310
  static_cast<T *>(p.y)[static_cast<int64_t>(m) * p.L.N + n] = t;
}

template <typename T>
__global__ void __launch_bounds__(32 * (kDecWorkers + 1), 1) decode_kernel(const DecParams p) {
  extern __shared__ __align__(128) uint8_t smem[];
  constexpr int kWorkers = kDecWorkers;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const long long t_entry = clock64();
  if (p.trace && threadIdx.x == 0 && blockIdx.x < kDecTraceCtas) g_dec_trace[blockIdx.x * kDecTraceSlots + 10] = globaltimer_ns();
  const int NS = p.nstages;
  const uint32_t smem0 = smem_u32(smem);
  const uint32_t xb = smem0 + p.xb_off, recv = smem0 + p.recv_off, bars = smem0 + p.bar_off;
  const uint32_t bar_wfull = bars, bar_wempty = bars + 8 * kDecMaxStages;
  const uint32_t bar_xload = bars + 16 * kDecMaxStages;   // pre-rotated x: one bulk copy fills the whole B operand
  // k-half partials, [block parity][tile][8 values][32 lanes] fp32: in the rotation tiles' space, free once the B operand is complete
  const uint32_t xchg = smem0 + p.rot_off;

  // ---- my range of 128-column blocks (within one partition) and my K-slice (whole groups, ragged)
  const int range = blockIdx.x >> p.c_shift;
  const int slice = blockIdx.x & (p.c - 1);   // == %cluster_ctarank
  int part = 0;
  while (range >= p.part_range_begin[part + 1]) ++part;
  const int jl = range - p.part_range_begin[part];
  const int cp = p.part_range_begin[part + 1] - p.part_range_begin[part];
  const int cbp = p.L.part_block_begin[part + 1] - p.L.part_block_begin[part];
  const int cb_begin = static_cast<int>(static_cast<unsigned>(jl) * static_cast<unsigned>(cbp) / static_cast<unsigned>(cp));
  const int cb_end = static_cast<int>(static_cast<unsigned>(jl + 1) * static_cast<unsigned>(cbp) / static_cast<unsigned>(cp));
  const int nj = cb_end - cb_begin;
  const int g_begin = static_cast<int>(static_cast<unsigned>(slice) * static_cast<unsigned>(p.L.groups) >> p.c_shift);
  const int g_end = static_cast<int>(static_cast<unsigned>(slice + 1) * static_cast<unsigned>(p.L.groups) >> p.c_shift);
  const int ng = g_end - g_begin;
  const int nrounds = nj * ng;
  // first output column of my first block, and the end of my partition (a last partial block is masked at the stores)
  const int n_first = p.L.part_col_begin[part] + cb_begin * kBlockN, n_end = p.L.part_col_begin[part + 1];
  // record of (block j, group gi) of mine: rec0 + (j * groups + gi) * rec_bytes
  const uint32_t rec_bytes = static_cast<uint32_t>(p.L.rec_bytes);
  const uint8_t *rec0 = p.packed + p.L.rec_off + (static_cast<size_t>(p.L.part_block_begin[part] + cb_begin) * p.L.groups + g_begin) * rec_bytes;

  // A rotation task = (group of the slice, block of up to 4 token rows); worker warp w takes tasks w, w + rot_warps, ...  (M = 16:
  // four tasks per group, so all warps share the rotation instead of 16-row tiles on a few)
  RotMeta rm;
  const int nq = p.M > 4 ? (p.M + 3) >> 2 : 1, ntasks = ng * nq;
  const int mi0 = part * p.L.groups + g_begin;   // metadata block of the slice's first group
  if (!p.pre_rotated && warp < kWorkers && warp < ntasks && warp < p.rot_warps)
    fetch_meta(p.packed + p.L.meta_off + static_cast<size_t>(mi0 + warp / nq) * p.L.meta_group_bytes, p.L.krot, lane, rm);   // flies during the barrier initialisation

  if (warp == kWorkers) {
    ring_init(bar_wfull, bar_wempty, NS, kWorkers, lane);   // every worker warp consumes every ring stage
    if (lane == 0) mbar_init(bar_xload, 1);
    fence_mbar_init();
  }
  __syncthreads();
  DEC_TRACE(1);
  if (p.c > 1) cluster_arrive_relaxed();   // #1 "this CTA runs" -- waited on before the first DSMEM push into a peer's receive buffer
  pdl_launch_dependents();                 // let the next linear in the stream start prefetching its weights
  bool cluster_ready = false;

  if (warp == kWorkers) {
    // ================= producer: ONE bulk copy per round (weights + scales + zeros of a (block, group), 8576 contiguous
    // bytes); nothing here depends on the previous kernel.  The whole warp runs the loop, an elected lane issues.
    const uint64_t pol = policy_evict_first();
    RingProducer prod = {bar_wfull, bar_wempty, smem0, rec_bytes, NS, 0, 0};
    int j = 0, gi = 0;
#pragma unroll 1
    for (int r = 0; r < nrounds; ++r) {
      // (hooks that capture the loop counters by reference change the instructions nvcc makes of this loop)
      prod.issue([=, &p] { return rec0 + (static_cast<size_t>(j) * p.L.groups + gi) * rec_bytes; }, rec_bytes, pol, [=, &p] {
        if (p.trace && blockIdx.x == 0 && r < 100) g_dec_trace[kDecTraceCtas * kDecTraceSlots + 3 * r] = clock64() - t_entry;
      });
      if (++gi == ng) { gi = 0; ++j; }
    }
  } else {
    // ================= workers: warp = (16-row tile of the block, k half of every record)
    const int wi = warp, tile = warp & 7, kh = warp >> 3;
    if (p.pre_rotated) {
      // the pre-pass (paro_rotate.cu, tiled for 16 rows) wrote x_rot in exactly the B-operand order of this kernel, zero padding
      // rows included: the K-slice's groups are ONE contiguous range -> one bulk copy, no rotation tasks
      if (wi == 0) {
        pdl_wait();   // ... written by the previous kernel in the stream
        if (elect_one()) {
          const uint32_t bytes = static_cast<uint32_t>(ng) * (kDecN * 256);
          mbar_arrive_expect_tx(bar_xload, bytes);
          bulk_g2s(xb, static_cast<const uint8_t *>(p.x) + (static_cast<size_t>(part) * p.x_part_stride + static_cast<size_t>(g_begin) * (kDecN * kGroup)) * 2,
                   bytes, bar_xload, policy_evict_first());
        }
        __syncwarp();
      }
      mbar_wait(bar_xload, 0);
    } else {
      // rows [M, 16) of every group are the zero padding of the N = 16 MMA: all workers clear the B operand before the
      // dependency wait (it does not depend on x); the rotation tasks then write only token rows
      if (p.M < kDecN) {
        for (int i = threadIdx.x; i < ng * (kDecN * 16); i += 32 * kWorkers) sts128u(xb + i * 16, make_uint4(0u, 0u, 0u, 0u));
        named_bar_sync(1, 32 * kWorkers);
      }
      DEC_TRACE(2);
      pdl_wait();  // x may have been written by the previous kernel
      DEC_TRACE(3);
      if (wi < ntasks && wi < p.rot_warps) {
        const uint32_t rot = smem0 + p.rot_off + wi * p.rot_bytes;
        const int M = p.M, rw = p.rot_warps;
        const uint8_t *meta = p.packed + p.L.meta_off;
        auto stage_x = [&](auto rows, int gi, int m0, uint2 csw) {
          constexpr int ROWS = decltype(rows)::value;
          const T *xg = static_cast<const T *>(p.x) + (g_begin + gi) * kGroup + 4 * lane;
          uint2 raw[ROWS];
#pragma unroll
          for (int m = 0; m < ROWS; ++m) {
            raw[m] = make_uint2(0u, 0u);
            if (m0 + m < M) raw[m] = __ldcg(reinterpret_cast<const uint2 *>(xg + static_cast<int64_t>(m0 + m) * p.L.K));
          }
          scale_and_stage<T, ROWS>(rot, lane, raw, csw);
          if (p.trace && threadIdx.x == 0 && blockIdx.x < kDecTraceCtas) g_dec_trace[blockIdx.x * kDecTraceSlots + 0] = clock64() - t_entry;
        };
        if (M == 1) rotation_tasks<T, 1, true>(rm, meta, p.L.meta_group_bytes, p.L.krot, mi0, ntasks, nq, M, wi, rw, lane, rot, xb, kDecN, stage_x);
        else if (M == 2) rotation_tasks<T, 2, true>(rm, meta, p.L.meta_group_bytes, p.L.krot, mi0, ntasks, nq, M, wi, rw, lane, rot, xb, kDecN, stage_x);
        else rotation_tasks<T, 4, true>(rm, meta, p.L.meta_group_bytes, p.L.krot, mi0, ntasks, nq, M, wi, rw, lane, rot, xb, kDecN, stage_x);
        if (p.trace && threadIdx.x == 0 && blockIdx.x < kDecTraceCtas) g_dec_trace[blockIdx.x * kDecTraceSlots + 9] = clock64() - t_entry;
      }
      named_bar_sync(2, 32 * kWorkers);   // B operand complete
    }
    DEC_TRACE(4);

    const int M = p.M;
    const int g = lane >> 2, t = lane & 3;
    const RoundLane lo = round_lane<kDecN>(p.L.qhalves == 2, tile, kh, lane);
    // The round loop (segment_rounds: one segment = one 128-column block), specialised on the token tiles (NTT) and on
    // tracing, so that neither is a per-round branch.
    using One = std::integral_constant<int, 1>;
    using Two = std::integral_constant<int, 2>;
    auto rounds = [&](auto ntt, auto trace) {
      constexpr int NTT = decltype(ntt)::value;
      constexpr bool TRACE = decltype(trace)::value;
      RingCursor rg = {bar_wfull, 0u, bar_wfull, bar_wfull + 8 * NS, 8 * kDecMaxStages, rec_bytes / 8, smem0 - bar_wfull * (rec_bytes / 8), rec_bytes};
      int tr_seen = 0, tr_done = 0;   // records of CTA 0's per-round log written
      auto seen = [&](int n) {
        if constexpr (TRACE) {
          if (tr_seen == 0) DEC_TRACE(5);
          if (blockIdx.x == 0 && warp == 0 && lane == 0)
            for (int i = 0; i < n; ++i)
              if (tr_seen + i < 100) g_dec_trace[kDecTraceCtas * kDecTraceSlots + 3 * (tr_seen + i) + 1] = clock64() - t_entry;   // seen full
          tr_seen += n;
        }
      };
      auto done = [&](int n) {
        if constexpr (TRACE) {
          if (blockIdx.x == 0 && warp == 0 && lane == 0)
            for (int i = 0; i < n; ++i)
              if (tr_done + i < 100) g_dec_trace[kDecTraceCtas * kDecTraceSlots + 3 * (tr_done + i) + 2] = clock64() - t_entry;   // MMAs issued
          tr_done += n;
        }
      };
      auto seg_begin = [&](int, uint32_t &bx, int &len) {
        bx = xb + lo.x;
        len = ng;
      };
      auto seg_end = [&](int j, float (&acc)[2][4]) {
        // ---- block j closed: the k-half-1 warp hands its partial to its tile's k-half-0 warp, which adds it (fixed order)
        // and stores or pushes the sum.  Two buffers by block parity: a warp writes buffer j & 1 again only after the pair
        // barrier of block j + 1, which its partner reaches after reading it.
        khalf_meet(acc, xchg + ((j & 1) * 8 + tile) * (8 * 128) + lane * 4, kh, 4 + tile, [&] {
          if (p.c > 1 && !cluster_ready) { cluster_wait_acquire(); cluster_ready = true; }  // #1: every peer CTA is running
          const uint32_t dst = p.c > 1 ? map_to_rank(recv + (((j >> p.c_shift) << p.c_shift) + slice) * (M * 512), j & (p.c - 1)) : 0u;
#pragma unroll
          for (int i = 0; i < 8; ++i) {
            const int col = 16 * tile + g + 8 * ((i >> 1) & 1), m = 8 * (i >> 2) + 2 * t + (i & 1);
            if (m < M) {
              const float v = acc[i >> 2][i & 3];
              if (p.c == 1) {
                const int n = n_first + j * kBlockN + col;
                if (n < n_end) dec_store<T>(p, v, m, n);
              } else {
                st_cluster_f32(dst + m * 512 + col * 4, v);
              }
            }
          }
        });
      };
      segment_rounds<T, NTT, kDecN>(rg, lo, nj, seg_begin, seg_end, seen, done);
    };
    if (p.trace) {
      if (M > 8) rounds(Two{}, std::true_type{});
      else rounds(One{}, std::true_type{});
    } else {
      if (M > 8) rounds(Two{}, std::false_type{});
      else rounds(One{}, std::false_type{});
    }
    DEC_TRACE(6);
  }

  // ================= common tail (all threads; warps reconverge first)
  __syncwarp();
  if (p.c > 1) {
    if (!cluster_ready) cluster_wait_acquire();
    cluster_arrive_release();                              // #2: all my pushes are done
    cluster_wait_acquire();
    DEC_TRACE(7);
    if (warp < kWorkers) {
      // finish the blocks that were sent to me (j % c == slice); fixed order over the K-slices
      const int M = p.M;
      const int nmine = nj > slice ? ((nj - slice + p.c - 1) >> p.c_shift) : 0;
      const int per = M * 128;
      for (int idx = threadIdx.x; idx < nmine * per; idx += 32 * kWorkers) {
        const int jo = idx / per, o = idx - jo * per;
        const int m = o >> 7, col = o & 127;
        float acc = 0.f;
        for (int src = 0; src < p.c; ++src) acc += lds_f32(recv + ((jo << p.c_shift) + src) * (M * 512) + o * 4);
        const int n = n_first + ((jo << p.c_shift) + slice) * kBlockN + col;
        if (n < n_end) dec_store<T>(p, acc, m, n);
      }
    }
  }
  DEC_TRACE(8);
  if (p.trace && threadIdx.x == 0 && blockIdx.x < kDecTraceCtas) g_dec_trace[blockIdx.x * kDecTraceSlots + 11] = globaltimer_ns();
}

int decode_trace_read(unsigned long long *host, int max_ctas) {
  const size_t n = static_cast<size_t>(max_ctas < kDecTraceRows ? max_ctas : kDecTraceRows) * kDecTraceSlots;
  PARO_CUDA_OK(cudaMemcpyFromSymbol(host, g_dec_trace, n * sizeof(unsigned long long)));
  return PARO_OK;
}

// ------------------------------------------------------------------ host side
struct DecPlan {
  int c, c_shift, ranges, grid;
  int part_range_begin[PARO_MAX_PARTS + 1];
  int nj_max, ng_max;
};

// `ranges` block ranges over the partitions, proportional to their 128-column blocks, at most one per block
static bool dec_split_ranges(const Layout &L, int ranges, DecPlan &plan) {
  if (!apportion(L, ranges < L.blocks_total ? ranges : L.blocks_total, plan.part_range_begin)) return false;
  plan.nj_max = 0;
  for (int p = 0; p < L.n_parts; ++p) {
    const int cb = L.part_block_begin[p + 1] - L.part_block_begin[p], n = plan.part_range_begin[p + 1] - plan.part_range_begin[p];
    const int mx = (cb + n - 1) / n;
    if (mx > plan.nj_max) plan.nj_max = mx;
  }
  plan.ranges = plan.part_range_begin[L.n_parts];
  return true;
}

struct DecSmem { int xb_off, rot_off, recv_off, bar_off, nstages, rot_warps, total; };

static bool dec_carve_with(const DecPlan &plan, int M, int rot_bytes, int sets, int rot_warps, int stage_bytes, DecSmem &s) {
  const int xb_bytes = plan.ng_max * kDecN * 256;
  const int rot_total = rot_warps * rot_bytes > kDecXchgBytes ? (rot_warps * rot_bytes + 127) / 128 * 128 : kDecXchgBytes;
  const int recv = plan.c > 1 ? ((plan.nj_max + plan.c - 1) / plan.c) * plan.c * M * 512 : 0;
  const int bar_bytes = kDecBarBytes;
  const int fixed = xb_bytes + rot_total + recv + bar_bytes + 128;
  const int nst = ring_stages(kDecSmemLimit - fixed, stage_bytes, kDecMaxStages, sets, sets, true);
  if (!nst) return false;
  s.nstages = nst;
  s.rot_warps = rot_warps;
  s.xb_off = (nst * stage_bytes + 127) / 128 * 128;
  s.rot_off = s.xb_off + xb_bytes;
  s.recv_off = s.rot_off + rot_total;
  s.bar_off = s.recv_off + (recv + 127) / 128 * 128;
  s.total = s.bar_off + bar_bytes;
  return s.total <= kDecSmemLimit;
}

// every group gets its own rotating warp when the tiles fit; otherwise fewer warps take several groups each
static bool dec_carve(const DecPlan &plan, int M, int rot_bytes, int sets, int stage_bytes, DecSmem &s) {
  return fit_rot_warps(plan.ng_max * (M > 4 ? (M + 3) / 4 : 1), sets,
                       [&](int rw) { return dec_carve_with(plan, M, rot_bytes, sets, rw, stage_bytes, s); });
}

// how many clusters of `c` CTAs with this footprint the device keeps resident (GPC granularity); 0 when that cannot be asked
template <typename T>
static int max_resident_clusters(int c, int smem_bytes, int sms) {
  if (c == 1) return sms;
  auto kern = decode_kernel<T>;
  if (smem_opt_in(kern, kDecSmemLimit) != cudaSuccess) return 0;
  cudaLaunchConfig_t cfg;
  cudaLaunchAttribute attr[2];
  launch_config(cfg, attr, (sms / c) * c, 32 * (kDecWorkers + 1), smem_bytes, 0, c, false);
  int n = 0;
  if (cudaOccupancyMaxActiveClusters(&n, kern, &cfg) != cudaSuccess) { (void)cudaGetLastError(); return 0; }
  return n;   // (the caller caches the whole plan per shape, M and device)
}

// The launch plan: cluster size c (K slices), block ranges per partition, shared-memory carve-up.  Pure host logic --
// `resident(c, smem_bytes)` says how many clusters of c CTAs with that footprint the device keeps resident (all clusters
// must be co-resident: one wave) -- so tests can drive it without a GPU (paro_debug_decode_plan).
template <typename ResidentFn>
static bool dec_choose_plan(const Layout &L, int M, int rot_bytes, int sets, int sms, bool cluster_ok, int force_c, ResidentFn resident,
                            DecPlan &best, DecSmem &best_s) {
  long best_cost = -1;
  for (int cs = 0; cs <= 3; ++cs) {
    const int c = 1 << cs;
    if (c > 1 && !cluster_ok) break;
    if (c > L.groups) break;
    if (force_c && c != force_c) continue;
    DecPlan plan = {};
    plan.c = c; plan.c_shift = cs;
    plan.ng_max = (L.groups + c - 1) / c;
    if (!dec_split_ranges(L, sms / c, plan)) continue;
    DecSmem s;
    if (!dec_carve(plan, M, rot_bytes, sets, L.rec_bytes, s)) continue;
    const int res = resident(c, s.total);
    if (res < L.n_parts) continue;
    if (res < plan.ranges) {
      if (!dec_split_ranges(L, res, plan)) continue;
      if (!dec_carve(plan, M, rot_bytes, sets, L.rec_bytes, s)) continue;
    }
    plan.grid = plan.ranges * c;
    // critical path in rounds: main loop of the busiest CTA + rotation passes + a small charge per doubling of the cluster
    const int passes = (plan.ng_max * (M > 4 ? (M + 3) / 4 : 1) + 4 * sets - 1) / (4 * sets);
    long cost = static_cast<long>(plan.nj_max) * plan.ng_max * 8 + passes * 24 + cs * 2;
    if (s.nstages < 2 * sets) cost += cost / 4;   // a ring shallower than two rounds per set starves the dequant warps (large M: the receive buffer crowds it out)
    if (best_cost < 0 || cost < best_cost) { best = plan; best_s = s; best_cost = cost; }
  }
  return best_cost >= 0;
}

static int dec_rot_bytes(int64_t M) { return kGroup * 2 * (M == 1 ? 1 : M == 2 ? 2 : 4); }   // rotation tile of one task: 128 channels x up to 4 rows

// test hook: the plan for given resident-cluster counts (index log2 c), no device involved
int decode_debug_plan(const Layout &L, int64_t M, int sets, int sms, const int32_t *resident4, int32_t *out20) {
  if (M < 1 || M > 16 || sets < 4 || sets > 7) { set_error("debug_plan: bad M / sets"); return PARO_EINVAL; }
  DecPlan plan = {};
  DecSmem sm = {};
  auto res = [&](int c, int) { int i = 0; while ((1 << i) < c) ++i; return static_cast<int>(resident4[i]); };
  if (!dec_choose_plan(L, static_cast<int>(M), dec_rot_bytes(M), sets, sms, true, 0, res, plan, sm)) {
    set_error("decode: no launch configuration fits (in_features=%d, M=%d)", L.K, static_cast<int>(M));
    return PARO_EUNSUPPORTED;
  }
  const int32_t v[11] = {plan.c, plan.ranges, plan.grid, plan.nj_max, plan.ng_max, sm.nstages, sm.rot_warps, sm.total, sm.xb_off, sm.recv_off, sm.bar_off};
  for (int i = 0; i < 11; ++i) out20[i] = v[i];
  for (int i = 0; i <= PARO_MAX_PARTS; ++i) out20[11 + i] = plan.part_range_begin[i];
  return PARO_OK;
}

struct DecCached { DecPlan plan; DecSmem smem; };

// the plan (cluster size, block ranges, shared-memory carve-up) depends on the shape, M and the device only: searched once
// (the search asks the occupancy API), then looked up -- an eager launch is a map lookup
template <typename T>
static bool dec_cached_plan(const Layout &L, int M, int sms, DecCached &out) {
  static PlanCache<DecCached> cache;
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess) dev = 0;
  const Knobs &kn = knobs();
  return cache.get(L, M, dev, out, [&](DecCached &c) {
    return dec_choose_plan(L, M, dec_rot_bytes(M), kDecSets, sms, !kn.no_cluster, kn.force_c,
                           [&](int cc, int smem) { return max_resident_clusters<T>(cc, smem, sms); }, c.plan, c.smem);
  });
}

template <typename T>
static int launch_decode(DecParams &p, const DecCached &c, cudaStream_t stream) {
  auto kern = decode_kernel<T>;
  const Knobs &kn = knobs();
  const DecPlan &best = c.plan;
  const DecSmem &best_s = c.smem;
  if (kn.verbose)
    fprintf(stderr, "[paro decode] K=%d N=%d M=%d: cluster %d x %d ranges (grid %d), blocks/CTA <= %d, groups/CTA <= %d, %d stages, smem %d\n",
            p.L.K, p.L.N, p.M, best.c, best.ranges, best.grid, best.nj_max, best.ng_max, best_s.nstages, best_s.total);

  PARO_CUDA_OK(smem_opt_in(kern, kDecSmemLimit));
  cudaLaunchConfig_t cfg;
  cudaLaunchAttribute attr[2];
  launch_config(cfg, attr, best.grid, 32 * (kDecWorkers + 1), best_s.total, stream, best.c > 1 ? best.c : 0, !kn.no_pdl);
  p.c = best.c; p.c_shift = best.c_shift;
  p.nstages = best_s.nstages;
  p.rot_warps = best_s.rot_warps;
  p.xb_off = best_s.xb_off; p.rot_off = best_s.rot_off; p.recv_off = best_s.recv_off; p.bar_off = best_s.bar_off;
  for (int i = 0; i <= PARO_MAX_PARTS; ++i) p.part_range_begin[i] = best.part_range_begin[i];
  PARO_CUDA_OK(cudaLaunchKernelEx(&cfg, kern, p));
  note_launches(1);
  return PARO_OK;
}

bool decode_supported(const Layout &L, int64_t M) { return M >= 1 && M <= 16 && L.groups >= 1; }

// From 5 rows on (3 when K >= 8192) the rotation runs ONCE, in a pre-pass (paro_rotate.cu: rotate_tile_kernel, one launch for all
// partitions, ~2.5 us) that writes x_rot in this kernel's B-operand order, and the kernel fetches its K slice with one bulk copy.
// Inside the kernel a 4-row rotation task is ~1000 dependent instructions of one warp (7-14 k cycles with 20 warps contending) and
// at M = 16 a CTA has 32-56 of them: 28 k of o_proj's 40 k cycles, 48 k of down_proj's 80 k (tools/trace_decode.py).  Measured
// (us, in-kernel -> pre-pass): M = 16: o 21.7 -> 13.4, qkv 18.2 -> 16.4, gate_up 38.1 -> 29.1, down 42.3 -> 23.8; M = 8: 14.0 ->
// 11.8, 16.7 -> 15.0, 29.7 -> 27.5, 38.2 -> 20.3; M = 4: o 10.0 -> 11.4 (stays in-kernel), down 25.1 -> 18.7.
static bool decode_wants_prerot(const Layout &L, int64_t M) {
  const int k = knobs().prerot_m;   // 0: the rule below; n >= 2: from n rows on; 1: never
  if (k == 1) return false;
  if (k >= 2) return M >= k;
  return M >= 5 || (M >= 3 && L.groups >= 64);
}
size_t decode_scratch_bytes(const Layout &L, int64_t max_m) {
  bool any = false;
  for (int64_t m = 1; m <= (max_m < 16 ? max_m : 16); ++m) any = any || decode_wants_prerot(L, m);
  return any ? static_cast<size_t>(L.n_parts) * kDecN * L.K * 2 : 0;
}

int decode_forward(const paro_linear_shape &s, const Layout &L, const void *packed, const void *x, int64_t M,
                   const void *bias, void *y, void *scratch, size_t scratch_bytes, cudaStream_t stream) {
  const int sms = device_sms();
  if (sms <= 0) { set_error("decode: no CUDA device"); return PARO_ECUDA; }
  // no plan (e.g. K too long for one CTA without clusters): the caller falls back to the stream kernel, before any launch
  DecCached plan;
  const bool found = s.dtype == PARO_BF16 ? dec_cached_plan<__nv_bfloat16>(L, static_cast<int>(M), sms, plan)
                                          : dec_cached_plan<__half>(L, static_cast<int>(M), sms, plan);
  if (!found) { set_error("decode: no launch configuration fits (in_features=%d, M=%d)", L.K, static_cast<int>(M)); return PARO_EUNSUPPORTED; }
  const size_t part_bytes = static_cast<size_t>(kDecN) * L.K * 2;   // 16 rows (zero padded) x K of T, B-operand order
  const bool prerot = decode_wants_prerot(L, M) && scratch && scratch_bytes >= L.n_parts * part_bytes;
  if (prerot) {   // one launch for all partitions (paro_rotate.cu: rotate_tile_kernel)
    const int rc = rotate_chain_launch(L, packed, PARO_XOP_NONE, x, nullptr, nullptr, 0, 0.f, scratch, M, kDecN, kDecN, stream);
    if (rc) return rc;
  }
  DecParams p = {};
  p.packed = static_cast<const uint8_t *>(packed);
  p.x = prerot ? scratch : x; p.y = y; p.bias = bias;
  p.pre_rotated = prerot ? 1 : 0;
  p.x_part_stride = prerot ? static_cast<long long>(kDecN) * L.K : 0;
  p.L = L;
  p.M = static_cast<int>(M);
  p.rot_bytes = dec_rot_bytes(M);
  p.trace = knobs().trace;
  return s.dtype == PARO_BF16 ? launch_decode<__nv_bfloat16>(p, plan, stream) : launch_decode<__half>(p, plan, stream);
}

}  // namespace paro
