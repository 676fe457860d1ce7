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
#include <cstring>
#include <map>
#include <mutex>
#include <type_traits>

#include "paro_tc_common.cuh"

namespace paro {

constexpr int kDecMaxStages = 24;
constexpr int kDecSets = 4;                     // worker warps = 4 x sets = 8 row tiles x 2 k halves
constexpr int kDecWorkers = 4 * kDecSets;
static_assert(kDecSets % 2 == 0, "the ring depth is a multiple of kDecSets; the round loop takes records in pairs that must not wrap");
constexpr int kDecN = 16;            // B operand rows per group: token rows, zero-padded
constexpr int kDecSmemLimit = 227 * 1024;
constexpr int kDecBarBytes = 16 * kDecMaxStages + 256;   // ring barriers + the x-load barrier
constexpr int kDecXchgBytes = 2 * 8 * 8 * 128;           // k-half partials: [2][8 tiles][8 values][32 lanes] fp32 (in the rotation tiles)
// one record per ring stage: 8576 bytes (group_size 128) or 8960 (group_size 64), both multiples of 64 -> DecParams::rec_bytes

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
  int M, K, N;
  int n_parts, groups, krot;
  int c, c_shift;                 // cluster size (K slices of this launch), log2
  int nstages, rot_bytes, rot_warps, trace;   // rot_warps: worker warps that take rotation tasks (each owns one rot_bytes tile)
  int rec_bytes, q2;              // record (= ring stage) size; q2: group_size 64, two scale / zero sets per record (paro_layout.h)
  int pre_rotated;                // x is the pre-pass's output: [n_parts][M][K], already scaled and rotated (no stages here)
  long long x_part_stride;        // elements between partitions of a pre-rotated x (0 otherwise)
  int xb_off, rot_off, recv_off, bar_off;   // shared-memory carve-up (bytes)
  int part_col_begin[PARO_MAX_PARTS + 1];
  int part_block_begin[PARO_MAX_PARTS + 1];
  int part_range_begin[PARO_MAX_PARTS + 1];
  int meta_group_bytes;
  long long meta_off, rec_off;
};

// ---- prologue.  A rotation TASK = (group gi of the CTA's slice, block of up to ROWS <= 4 token rows); worker warp w takes
// tasks w, w + W, ...  (M = 16: four tasks per group, so all warps share the rotation instead of 16-row tiles on a few).
// B[gi][k16 step s][k half h][row m][8 k]: 16 rows x 16 bytes per core-matrix pair, 512 bytes per step.
template <typename T, int ROWS>
__device__ __forceinline__ void dec_write_b_rows(uint32_t xb_group, uint32_t rot, int m0, int nrows, int lane) {
  for (int idx = lane; idx < 16 * nrows; idx += 32) {
    const int ml = idx >> 4, s = (idx >> 1) & 7, h = idx & 1;
    const int c0 = 16 * s + 8 * h, m = m0 + ml;
    uint4 v;
    if constexpr (ROWS == 1) {
      v = lds128(rot + c0 * 2);
    } else {
      uint32_t e[8];
#pragma unroll
      for (int k = 0; k < 8; ++k) e[k] = lds16(rot + (c0 + k) * (ROWS * 2) + 2 * ml);
      v = make_uint4(e[0] | (e[1] << 16), e[2] | (e[3] << 16), e[4] | (e[5] << 16), e[6] | (e[7] << 16));
    }
    sts128u(xb_group + s * (kDecN * 32) + h * (kDecN * 16) + (m >> 3) * 128 + (m & 7) * 16, v);
  }
}
struct DecRotMeta {
  uint32_t idxw[8], tw[8];
  uint2 csw;
  const uint8_t *meta;
};

__device__ __forceinline__ void dec_fetch_meta(const DecParams &p, int part, int gk, int lane, DecRotMeta &rm) {
  rm.meta = p.packed + p.meta_off + (static_cast<size_t>(part) * p.groups + gk) * p.meta_group_bytes;
  if (p.pre_rotated) return;   // no rotation tasks at all
  rm.csw = *reinterpret_cast<const uint2 *>(rm.meta + p.krot * 256 + 8 * lane);
  if (p.krot == 8) {
#pragma unroll
    for (int r = 0; r < 8; ++r) {
      rm.idxw[r] = *reinterpret_cast<const uint32_t *>(rm.meta + r * 128 + 4 * lane);
      rm.tw[r] = *reinterpret_cast<const uint32_t *>(rm.meta + 8 * 128 + r * 128 + 4 * lane);
    }
  }
}

template <typename T, int ROWS>
__device__ __forceinline__ void dec_rotate_task(const DecParams &p, const DecRotMeta &rm, const void *xpart, int gk, int m0, int lane, uint32_t rot,
                                                uint32_t xb_group, long long t_entry) {
  uint2 raw[ROWS];
  struct { const void *x; int M, K; } px = {xpart, p.M, p.K};   // my partition's rows (a pre-rotated x has one copy per partition)
  load_x<T, ROWS>(px, gk, lane, raw, m0);
  scale_and_stage<T, ROWS>(rot, lane, raw, rm.csw);
  __syncwarp();
  if (p.trace && threadIdx.x == 0 && blockIdx.x < kDecTraceCtas) g_dec_trace[blockIdx.x * kDecTraceSlots + 0] = clock64() - t_entry;
  if (p.krot == 8) {
#pragma unroll
    for (int r = 0; r < 8; ++r) {
      // (keeping all 32 coefficients live across griddepcontrol.wait was tried: it spills at 80 registers and the
      // stages get slower than with the MUFU work inline)
      float c0, s0, c1, s1;
      sincos2<T>(rm.tw[r], c0, s0, c1, s1);
      rotate_stage<T, ROWS>(rot, rm.idxw[r], c0, s0, c1, s1);
      __syncwarp();
    }
  } else {
    const int krot = p.krot;
    for (int r = 0; r < krot; ++r) {
      const uint32_t iw = *reinterpret_cast<const uint32_t *>(rm.meta + r * 128 + 4 * lane);
      const uint32_t tw = *reinterpret_cast<const uint32_t *>(rm.meta + krot * 128 + r * 128 + 4 * lane);
      float c0, s0, c1, s1;
      sincos2<T>(tw, c0, s0, c1, s1);
      rotate_stage<T, ROWS>(rot, iw, c0, s0, c1, s1);
      __syncwarp();
    }
  }
  if (p.trace && threadIdx.x == 0 && blockIdx.x < kDecTraceCtas) g_dec_trace[blockIdx.x * kDecTraceSlots + 9] = clock64() - t_entry;
  const int left = p.M - m0;
  dec_write_b_rows<T, ROWS>(xb_group, rot, m0, left < ROWS ? left : ROWS, lane);
  __syncwarp();
}

// tasks t = wi, wi + nwarps, ... of ng * nq (nq row blocks per group); the first task's metadata was fetched before the wait
template <typename T, int ROWS>
__device__ __forceinline__ void dec_prologue(const DecParams &p, DecRotMeta &rm, int part, int g_begin, int ntasks, int nq, int wi, int nwarps,
                                             int lane, uint32_t rot, uint32_t xb, long long t_entry) {
  const void *xpart = static_cast<const T *>(p.x) + static_cast<long long>(part) * p.x_part_stride;
  for (int t = wi; t < ntasks; t += nwarps) {
    const int gi = t / nq, rq = t - gi * nq;
    if (t != wi) dec_fetch_meta(p, part, g_begin + gi, lane, rm);
    dec_rotate_task<T, ROWS>(p, rm, xpart, g_begin + gi, rq * ROWS, lane, rot, xb + gi * (kDecN * 256), t_entry);
  }
}

template <typename T>
__device__ __forceinline__ void dec_store(const DecParams &p, float v, int m, int n) {
  T t = Traits<T>::from_float(v);
  if (p.bias) t = Traits<T>::from_float(Traits<T>::to_float(t) + Traits<T>::to_float(static_cast<const T *>(p.bias)[n]));  // plugin.py:309-310
  static_cast<T *>(p.y)[static_cast<int64_t>(m) * p.N + n] = t;
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
  const int cbp = p.part_block_begin[part + 1] - p.part_block_begin[part];
  const int cb_begin = static_cast<int>(static_cast<unsigned>(jl) * static_cast<unsigned>(cbp) / static_cast<unsigned>(cp));
  const int cb_end = static_cast<int>(static_cast<unsigned>(jl + 1) * static_cast<unsigned>(cbp) / static_cast<unsigned>(cp));
  const int nj = cb_end - cb_begin;
  const int g_begin = static_cast<int>(static_cast<unsigned>(slice) * static_cast<unsigned>(p.groups) >> p.c_shift);
  const int g_end = static_cast<int>(static_cast<unsigned>(slice + 1) * static_cast<unsigned>(p.groups) >> p.c_shift);
  const int ng = g_end - g_begin;
  const int nrounds = nj * ng;
  // first output column of my first block, and the end of my partition (a last partial block is masked at the stores)
  const int n_first = p.part_col_begin[part] + cb_begin * kBlockN, n_end = p.part_col_begin[part + 1];
  // record of (block j, group gi) of mine: rec0 + (j * groups + gi) * rec_bytes
  const uint32_t rec_bytes = static_cast<uint32_t>(p.rec_bytes);
  const uint8_t *rec0 = p.packed + p.rec_off + (static_cast<size_t>(p.part_block_begin[part] + cb_begin) * p.groups + g_begin) * rec_bytes;

  DecRotMeta rm;
  const int nq = p.M > 4 ? (p.M + 3) >> 2 : 1, ntasks = ng * nq;   // rotation tasks: row blocks of 4 for M > 4
  if (warp < kWorkers && warp < ntasks && warp < p.rot_warps)
    dec_fetch_meta(p, part, g_begin + warp / nq, lane, rm);   // flies during the barrier initialisation

  if (warp == kWorkers) {
    // one barrier per lane; every worker warp consumes every ring stage
    if (lane < NS) {
      mbar_init(bar_wfull + 8 * lane, 1);
      mbar_init(bar_wempty + 8 * lane, kWorkers);
    }
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
    int st = 0, it = 0, j = 0, gi = 0;
#pragma unroll 1
    for (int r = 0; r < nrounds; ++r) {
      if (it > 0) mbar_wait(bar_wempty + 8 * st, (it - 1) & 1);
      if (elect_one()) {
        mbar_arrive_expect_tx(bar_wfull + 8 * st, rec_bytes);
        bulk_g2s(smem0 + st * rec_bytes, rec0 + (static_cast<size_t>(j) * p.groups + gi) * rec_bytes, rec_bytes, bar_wfull + 8 * st, pol);
        if (p.trace && blockIdx.x == 0 && r < 100) g_dec_trace[kDecTraceCtas * kDecTraceSlots + 3 * r] = clock64() - t_entry;
      }
      __syncwarp();
      if (++st == NS) { st = 0; ++it; }
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
        if (M == 1) dec_prologue<T, 1>(p, rm, part, g_begin, ntasks, nq, wi, rw, lane, rot, xb, t_entry);
        else if (M == 2) dec_prologue<T, 2>(p, rm, part, g_begin, ntasks, nq, wi, rw, lane, rot, xb, t_entry);
        else dec_prologue<T, 4>(p, rm, part, g_begin, ntasks, nq, wi, rw, lane, rot, xb, t_entry);
      }
      named_bar_sync(2, 32 * kWorkers);   // B operand complete
    }
    DEC_TRACE(4);

    const int M = p.M;
    const int g = lane >> 2, t = lane & 3;
    const RoundLane lo = round_lane<kDecN>(p.q2 != 0, tile, kh, lane);
    const uint32_t ring_end = bar_wfull + 8 * NS;
    // a stage's record from its full barrier: smem0 + (fb - bar_wfull) / 8 * rec_bytes (rec_bytes is a multiple of 8)
    const uint32_t rec_per_bar = rec_bytes / 8, rec_at_bar0 = smem0 - bar_wfull * rec_per_bar;
    // The round loop, specialised on the token tiles (NTT) and on tracing, so that neither is a per-round branch.  Stage
    // and parity advance by increments: `fb` is the stage's full barrier, its empty barrier sits 8 * kDecMaxStages above.
    // Records are taken in pairs from an even stage: the ring depth is a multiple of kDecSets (even), so a pair never
    // wraps.  A block starting at an odd stage (ng odd) takes its first record alone, an odd count its last.
    using One = std::integral_constant<int, 1>;
    using Two = std::integral_constant<int, 2>;
    auto rounds = [&](auto ntt, auto trace) {
      constexpr int NTT = decltype(ntt)::value;
      constexpr bool TRACE = decltype(trace)::value;
      uint32_t fb = bar_wfull, par = 0;
      int tr = 0;   // rounds of CTA 0's per-round log written
      float acc[2][4];
      uint32_t bx;   // this lane's ldmatrix row in the B operand of the next group
      auto take = [&](auto nrec) {
        constexpr int NREC = decltype(nrec)::value;
#pragma unroll
        for (int i = 0; i < NREC; ++i) mbar_wait(fb + 8 * i, par);
        if constexpr (TRACE) {
          if (tr == 0) DEC_TRACE(5);
          if (blockIdx.x == 0 && warp == 0 && lane == 0)
            for (int i = 0; i < NREC; ++i)
              if (tr + i < 100) g_dec_trace[kDecTraceCtas * kDecTraceSlots + 3 * (tr + i) + 1] = clock64() - t_entry;   // seen full
        }
        mma_rounds<T, NTT, NREC, kDecN>(fb * rec_per_bar + rec_at_bar0, rec_bytes, bx, lo, acc);
        __syncwarp();
        if (elect_one()) {
#pragma unroll
          for (int i = 0; i < NREC; ++i) mbar_arrive(fb + 8 * i + 8 * kDecMaxStages);
        }
        if constexpr (TRACE) {
          if (blockIdx.x == 0 && warp == 0 && lane == 0)
            for (int i = 0; i < NREC; ++i)
              if (tr + i < 100) g_dec_trace[kDecTraceCtas * kDecTraceSlots + 3 * (tr + i) + 2] = clock64() - t_entry;   // consumed
          tr += NREC;
        }
        bx += NREC * (kDecN * 256);
        fb += 8 * NREC;
        if (fb == ring_end) { fb = bar_wfull; par ^= 1; }
      };
#pragma unroll 1
      for (int j = 0; j < nj; ++j) {
#pragma unroll
        for (int i = 0; i < 8; ++i) acc[i >> 2][i & 3] = 0.f;
        bx = xb + lo.x;
        int left = ng;
        if ((fb - bar_wfull) & 8) { take(One{}); --left; }
        const uint32_t pairs_end = bx + (left >> 1) * (2 * kDecN * 256);   // the pair loop counts with bx
#pragma unroll 1
        while (bx != pairs_end) take(Two{});
        if (left & 1) take(One{});
        // ---- block j closed: the k-half-1 warp hands its partial to its tile's k-half-0 warp, which adds it (fixed order)
        // and stores or pushes the sum.  Two buffers by block parity: a warp writes buffer j & 1 again only after the pair
        // barrier of block j + 1, which its partner reaches after reading it.
        const uint32_t xc = xchg + ((j & 1) * 8 + tile) * (8 * 128) + lane * 4;
        if (kh == 1) {
#pragma unroll
          for (int i = 0; i < 8; ++i) sts_f32(xc + i * 128, acc[i >> 2][i & 3]);
        }
        named_bar_sync(4 + tile, 64);
        if (kh == 0) {
#pragma unroll
          for (int i = 0; i < 8; ++i) acc[i >> 2][i & 3] += lds_f32(xc + i * 128);
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
        }
      }
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
static int dec_env_int(const char *name, int dflt) {
  const char *v = getenv(name);
  return v && *v ? atoi(v) : dflt;
}
// environment knobs are read ONCE per process (every launch used to pay half a dozen getenv calls)
struct DecKnobs { int stages, no_cluster, force_c, verbose, no_pdl, trace; };
static const DecKnobs &dec_knobs() {
  static const DecKnobs k = {dec_env_int("PARO_DECODE_STAGES", 0), dec_env_int("PARO_NO_CLUSTER", 0), dec_env_int("PARO_DECODE_C", 0),
                             dec_env_int("PARO_DECODE_VERBOSE", 0), dec_env_int("PARO_NO_PDL", 0), dec_env_int("PARO_DECODE_TRACE", 0)};
  return k;
}

struct DecPlan {
  int c, c_shift, ranges, grid;
  int part_range_begin[PARO_MAX_PARTS + 1];
  int nj_max, ng_max;
};

// `ranges` block ranges over the partitions, proportional to their 128-column block counts (largest remainder)
static bool dec_split_ranges(const Layout &L, int ranges, DecPlan &plan) {
  int cb[PARO_MAX_PARTS], alloc[PARO_MAX_PARTS], total = 0;
  double frac[PARO_MAX_PARTS];
  for (int p = 0; p < L.n_parts; ++p) {
    cb[p] = L.part_block_begin[p + 1] - L.part_block_begin[p];
    total += cb[p];
  }
  if (ranges > total) ranges = total;
  if (ranges < L.n_parts) return false;
  int used = 0;
  for (int p = 0; p < L.n_parts; ++p) {
    const double exact = static_cast<double>(ranges) * cb[p] / total;
    alloc[p] = static_cast<int>(exact);
    if (alloc[p] < 1) alloc[p] = 1;
    if (alloc[p] > cb[p]) alloc[p] = cb[p];
    frac[p] = exact - alloc[p];
    used += alloc[p];
  }
  while (used < ranges) {
    int best = -1;
    for (int p = 0; p < L.n_parts; ++p)
      if (alloc[p] < cb[p] && (best < 0 || frac[p] > frac[best])) best = p;
    if (best < 0) break;
    alloc[best]++; frac[best] -= 1.0; used++;
  }
  while (used > ranges) {
    int best = -1;
    for (int p = 0; p < L.n_parts; ++p)
      if (alloc[p] > 1 && (best < 0 || frac[p] < frac[best])) best = p;
    if (best < 0) return false;
    alloc[best]--; frac[best] += 1.0; used--;
  }
  plan.part_range_begin[0] = 0;
  plan.nj_max = 0;
  for (int p = 0; p < PARO_MAX_PARTS; ++p) {
    plan.part_range_begin[p + 1] = plan.part_range_begin[p] + (p < L.n_parts ? alloc[p] : 0);
    if (p < L.n_parts) {
      const int mx = (cb[p] + alloc[p] - 1) / alloc[p];
      if (mx > plan.nj_max) plan.nj_max = mx;
    }
  }
  plan.ranges = plan.part_range_begin[L.n_parts];
  return plan.ranges > 0;
}

struct DecSmem { int xb_off, rot_off, recv_off, bar_off, nstages, rot_warps, total; };

static bool dec_carve_with(const DecPlan &plan, int M, int rot_bytes, int sets, int rot_warps, int stage_bytes, DecSmem &s) {
  const int xb_bytes = plan.ng_max * kDecN * 256;
  const int rot_total = rot_warps * rot_bytes > kDecXchgBytes ? (rot_warps * rot_bytes + 127) / 128 * 128 : kDecXchgBytes;
  const int recv = plan.c > 1 ? ((plan.nj_max + plan.c - 1) / plan.c) * plan.c * M * 512 : 0;
  const int bar_bytes = kDecBarBytes;
  const int fixed = xb_bytes + rot_total + recv + bar_bytes + 128;
  int nst = (kDecSmemLimit - fixed) / stage_bytes;
  if (nst > kDecMaxStages) nst = kDecMaxStages;
  const int want = dec_knobs().stages;
  if (want >= sets && want < nst) nst = want;
  nst = nst / sets * sets;   // a stage is always consumed by the same set
  if (nst < sets) return false;
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
  const int ntasks = plan.ng_max * (M > 4 ? (M + 3) / 4 : 1);
  int rw = ntasks < 4 * sets ? ntasks : 4 * sets;
  for (;;) {
    if (dec_carve_with(plan, M, rot_bytes, sets, rw, stage_bytes, s)) return true;
    if (rw <= 2) return false;
    rw = rw > 8 ? 8 : rw / 2;
  }
}

// how many clusters of `c` CTAs with this footprint the device keeps resident (GPC granularity); cached per thread
template <typename T>
static int max_resident_clusters(int c, int smem_bytes, int sms) {
  if (c == 1) return sms;
  int slot = 0;
  while ((1 << slot) < c) ++slot;
  auto kern = decode_kernel<T>;
  if (cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, kDecSmemLimit) != cudaSuccess) { (void)cudaGetLastError(); return 0; }   // never lowered: cached plans keep launching
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3((sms / c) * c);
  cfg.blockDim = dim3(32 * (kDecWorkers + 1));
  cfg.dynamicSmemBytes = smem_bytes;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeClusterDimension;
  attr[0].val.clusterDim.x = c;
  attr[0].val.clusterDim.y = 1;
  attr[0].val.clusterDim.z = 1;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
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

struct DecCached { bool found; DecPlan plan; DecSmem smem; };

// the plan (cluster size, block ranges, shared-memory carve-up) depends on the shape, M and the device only: searched once
// (the search asks the occupancy API and sets the function attribute), then looked up -- an eager launch is a map lookup
template <typename T>
static DecCached dec_cached_plan(const Layout &L, int M, int sms) {
  auto kern = decode_kernel<T>;
  const DecKnobs &kn = dec_knobs();
  struct Key {
    int K, N, krot, n_parts, M, dev, qhalves, parts[PARO_MAX_PARTS];
    bool operator<(const Key &o) const { return memcmp(this, &o, sizeof(Key)) < 0; }
  };
  static std::mutex mu;
  static std::map<Key, DecCached> cache;
  Key key;
  memset(&key, 0, sizeof(key));
  key.K = L.K; key.N = L.N; key.krot = L.krot; key.n_parts = L.n_parts; key.M = M; key.qhalves = L.qhalves;
  if (cudaGetDevice(&key.dev) != cudaSuccess) key.dev = 0;
  for (int i = 0; i < L.n_parts; ++i) key.parts[i] = L.part_col_begin[i + 1] - L.part_col_begin[i];
  DecCached c;
  {
    std::lock_guard<std::mutex> lock(mu);
    auto it = cache.find(key);
    if (it == cache.end()) {
      DecCached fresh = {};
      fresh.found = dec_choose_plan(L, M, dec_rot_bytes(M), kDecSets, sms, !kn.no_cluster, kn.force_c,
                                    [&](int cc, int smem) { return max_resident_clusters<T>(cc, smem, sms); }, fresh.plan, fresh.smem);
      if (fresh.found && cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, kDecSmemLimit) != cudaSuccess) {
        (void)cudaGetLastError();
        fresh.found = false;
      }
      it = cache.emplace(key, fresh).first;
    }
    c = it->second;
  }
  return c;
}

template <typename T>
static int launch_decode(DecParams &p, const Layout &L, const DecCached &c, cudaStream_t stream) {
  auto kern = decode_kernel<T>;
  const DecKnobs &kn = dec_knobs();
  const DecPlan &best = c.plan;
  const DecSmem &best_s = c.smem;
  if (kn.verbose)
    fprintf(stderr, "[paro decode] K=%d N=%d M=%d: cluster %d x %d ranges (grid %d), blocks/CTA <= %d, groups/CTA <= %d, %d stages, smem %d\n",
            L.K, L.N, p.M, best.c, best.ranges, best.grid, best.nj_max, best.ng_max, best_s.nstages, best_s.total);

  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3(best.grid);
  cfg.blockDim = dim3(32 * (kDecWorkers + 1));
  cfg.dynamicSmemBytes = best_s.total;
  cfg.stream = stream;
  cudaLaunchAttribute attr[2];
  int na = 0;
  if (best.c > 1) {
    attr[na].id = cudaLaunchAttributeClusterDimension;
    attr[na].val.clusterDim.x = best.c;
    attr[na].val.clusterDim.y = 1;
    attr[na].val.clusterDim.z = 1;
    ++na;
  }
  if (!kn.no_pdl) {
    attr[na].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[na].val.programmaticStreamSerializationAllowed = 1;
    ++na;
  }
  cfg.attrs = attr;
  cfg.numAttrs = na;
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

// From 5 rows on (3 when K >= 8192) the rotation runs ONCE, in a pre-pass (paro_rotate.cu: rotate_small_kernel, one launch for all
// partitions, ~2.5 us) that writes x_rot in this kernel's B-operand order, and the kernel fetches its K slice with one bulk copy.
// Inside the kernel a 4-row rotation task is ~1000 dependent instructions of one warp (7-14 k cycles with 20 warps contending) and
// at M = 16 a CTA has 32-56 of them: 28 k of o_proj's 40 k cycles, 48 k of down_proj's 80 k (tools/trace_decode.py).  Measured
// (us, in-kernel -> pre-pass): M = 16: o 21.7 -> 13.4, qkv 18.2 -> 16.4, gate_up 38.1 -> 29.1, down 42.3 -> 23.8; M = 8: 14.0 ->
// 11.8, 16.7 -> 15.0, 29.7 -> 27.5, 38.2 -> 20.3; M = 4: o 10.0 -> 11.4 (stays in-kernel), down 25.1 -> 18.7.
static int dec_prerot_knob() {
  static const int v = dec_env_int("PARO_DECODE_PREROT_M", 0);   // 0: the rule below; n >= 2: from n rows on; 1: never
  return v;
}
static bool decode_wants_prerot(const Layout &L, int64_t M) {
  const int k = dec_prerot_knob();
  if (k == 1) return false;
  if (k >= 2) return M >= k;
  return M >= 5 || (M >= 3 && L.groups >= 64);
}
size_t decode_scratch_bytes(const Layout &L, int64_t max_m) {
  bool any = false;
  for (int64_t m = 1; m <= (max_m < 16 ? max_m : 16); ++m) any = any || decode_wants_prerot(L, m);
  return any ? static_cast<size_t>(L.n_parts) * kDecN * L.K * 2 : 0;
}

int rotate_small_launch(const void *x, void *out, const void *raw_base, long long raw_part_bytes, int n_parts, int64_t M, int64_t M_store, int nt,
                        int K, int krot, int dtype, cudaStream_t stream);

int decode_forward(const paro_linear_shape &s, const Layout &L, const void *packed, const void *x, int64_t M,
                   const void *bias, void *y, void *scratch, size_t scratch_bytes, cudaStream_t stream) {
  int dev = 0;
  PARO_CUDA_OK(cudaGetDevice(&dev));
  static thread_local int sms_of[64] = {};   // SM count per device, asked once
  if (!sms_of[dev & 63]) PARO_CUDA_OK(cudaDeviceGetAttribute(&sms_of[dev & 63], cudaDevAttrMultiProcessorCount, dev));
  const int sms = sms_of[dev & 63];
  // no plan (e.g. K too long for one CTA without clusters): the caller falls back to the stream kernel, before any launch
  const DecCached plan = s.dtype == PARO_BF16 ? dec_cached_plan<__nv_bfloat16>(L, static_cast<int>(M), sms)
                                              : dec_cached_plan<__half>(L, static_cast<int>(M), sms);
  if (!plan.found) { set_error("decode: no launch configuration fits (in_features=%d, M=%d)", L.K, static_cast<int>(M)); return PARO_EUNSUPPORTED; }
  const size_t part_bytes = static_cast<size_t>(kDecN) * L.K * 2;   // 16 rows (zero padded) x K of T, B-operand order
  const bool prerot = decode_wants_prerot(L, M) && scratch && scratch_bytes >= L.n_parts * part_bytes;
  if (prerot) {   // one launch for all partitions (paro_rotate.cu: rotate_small_kernel)
    const int rc = rotate_small_launch(x, scratch, static_cast<const uint8_t *>(packed) + L.raw_off, static_cast<long long>(L.raw_part_bytes), L.n_parts, M,
                                       kDecN, kDecN, L.K, L.krot, s.dtype, stream);
    if (rc) return rc;
  }
  DecParams p = {};
  p.packed = static_cast<const uint8_t *>(packed);
  p.x = prerot ? scratch : x; p.y = y; p.bias = bias;
  p.pre_rotated = prerot ? 1 : 0;
  p.x_part_stride = prerot ? static_cast<long long>(kDecN) * L.K : 0;
  p.M = static_cast<int>(M); p.K = L.K; p.N = L.N;
  p.n_parts = L.n_parts; p.groups = L.groups; p.krot = L.krot;
  p.rec_bytes = L.rec_bytes; p.q2 = L.qhalves == 2;
  p.rot_bytes = dec_rot_bytes(M);
  p.trace = dec_knobs().trace;
  for (int i = 0; i <= PARO_MAX_PARTS; ++i) {
    p.part_col_begin[i] = L.part_col_begin[i];
    p.part_block_begin[i] = L.part_block_begin[i];
  }
  p.meta_group_bytes = L.meta_group_bytes;
  p.meta_off = static_cast<long long>(L.meta_off);
  p.rec_off = static_cast<long long>(L.rec_off);
  return s.dtype == PARO_BF16 ? launch_decode<__nv_bfloat16>(p, L, plan, stream) : launch_decode<__half>(p, L, plan, stream);
}

}  // namespace paro
