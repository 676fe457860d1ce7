// Large-M path (M > 16): rotation pre-pass + INT4-dequant wgmma GEMM, tensor-core bound.
//
//   y^T[n, m] = sum_k W[n, k] * x_rot[m, k]          (operand-swapped: the quantised weights are the
//                                                      M = 64 side of wgmma, the tokens the N side)
//   A  = W block of 128 output columns x 128 channels per round, dequantised by the consumer warpgroups straight
//        into wgmma's register A fragments: T((q - z) * T(s)), one rounding, the operand Marlin / AWQ form.
//        No shared-memory round trip for the weight operand.
//   B  = x_rot tile [NT tokens x 64 channels] per stage, produced by the rotation pre-pass
//        (paro_rotate.cu, the reference's rounding points) directly in wgmma's K-major core-matrix
//        order, so ONE 1-D bulk copy (TMA) per stage fills the operand -- no tensor map needed.
//   D  = fp32 [64 x NT] per consumer warpgroup in registers, one rounding to T in the epilogue, bias in T.
//
// CTA = one (128-column block of N) x (NT-token block of M) output tile over the whole K.
// Warpgroup 0: warp 0 TMA producer of the weight records (one 8576-byte record per round), warp 1 TMA producer of the
// x_rot stages.  Warpgroups 1 and 2: consumers of output columns 0-63 / 64-127 of the block; a consumer dequantises
// round r + 1 while the wgmmas of round r run (two register sets of A fragments).
//
// The same kernel serves the MoE block's grouped GEMMs (paro_moe_grouped.cu) through its tile source: there a token block is a
// tile slot of the routing table -- NT sorted (token, slot) rows of one expert -- the weights are that expert's, and the
// epilogue scatters each row to its (token, slot) output row.  It also serves the prefill chain (prefill_chain_forward below), whose
// ADD_RESIDUAL steps take the residual tile source: the residual add and the next RMSNorm's row statistics in the epilogue.
#include "paro_launch.h"
#include "paro_tc_common.cuh"

namespace paro {

constexpr int kGemmConsumers = 2;                         // warpgroups of 64 output columns
constexpr int kGemmThreads = 128 * (1 + kGemmConsumers);
constexpr int kWStages = 8;   // rounds of weights in flight (8.5 KB each)
constexpr int kBStages = 4;   // k64 stages of x_rot in flight (NT * 128 bytes each): two rounds
constexpr int kWStage = kBlockBytesMax;   // one (block, group) record per ring stage (8576 bytes, 8960 with group_size 64)

struct GemmParams {
  const uint8_t *packed;
  const uint8_t *xr;       // [n_parts][token blocks][K/16 steps][2][NT/8][8][8] elements
  void *y;
  const void *bias;
  Layout L;                // the packed linear (paro_layout.h)
  int M, NT, tok_blocks;
  long long xr_part_stride;
};

// Tile source of a linear: token block tb is rows tb * NT .. tb * NT + NT - 1 of x and y, the weights are p.packed.
struct DenseTiles {
  static constexpr bool kGrouped = false, kResidual = false;
};
// The same tiles with a prefill chain step's ADD_RESIDUAL epilogue (paro_stream.cu finish_block's order): t = T(acc) (+ bias in T),
// y = t where y is given, h = T(t + residual_in) -> residual_out.  With `stats`, also stats[block * M + m] = the sum of the T-rounded
// h^2 over the block's 128 columns, for the next step's RMSNorm: per warp the thread's two columns, then a butterfly over the 8 g
// lanes, then the 8 consumer warps in warp order through shared memory -- an order fixed by the column alone, so a row's sums do
// not depend on NT, M or the other rows.
struct ResidualTiles {
  static constexpr bool kGrouped = false, kResidual = true;
  const void *res_in;
  void *res_out;
  float *stats;   // [blocks_total][M] or NULL
};
// Tile source of a MoE block's grouped GEMM: tile slot tb is positions tb * NT .. of the routing table, all of one expert
// (paro_moe_grouped.cu writes the table on the device).  Slots from *live_tiles on are empty and exit at once.
struct GroupedTiles {
  static constexpr bool kGrouped = true, kResidual = false;
  const int32_t *rows;          // [slots * NT]: output row (token * top_k + slot) of each position, -1 for padding
  const int32_t *tile_expert;   // [slots]
  const int32_t *live_tiles;
  long long expert_stride;      // bytes from one expert's packed buffer to the next
};

// the A fragments of one round (8 k16 steps x 4 registers) for this warp's 16-row tile: two 128-bit loads per lane
template <typename T>
__device__ __forceinline__ void gemm_dequant_round(uint32_t rec, bool q2, uint32_t zero_off, int tile, int lane, uint32_t (&a)[32]) {
  const int q = qparam_index(16 * tile + (lane >> 2));
  const uint4 w0 = lds128(rec + frag_offset(tile, 0, lane)), w1 = lds128(rec + frag_offset(tile, 1, lane));
  FragDequant<T> d;
  d.prep(lds32(rec + kBlockScaleOff + 2 * q), lds16(rec + zero_off + q));
  d.frag(w0.x, a + 0); d.frag(w0.y, a + 4); d.frag(w0.z, a + 8); d.frag(w0.w, a + 12);
  if (q2)   // group_size 64: channels 64..127 of the record have their own scale / zero
    d.prep(lds32(rec + kBlockScaleOff + 256 + 2 * q), lds16(rec + zero_off + 128 + q));
  d.frag(w1.x, a + 16); d.frag(w1.y, a + 20); d.frag(w1.z, a + 24); d.frag(w1.w, a + 28);
}

// ResidualTiles' epilogue for this thread's output columns n (n + 8 the other half) and its NT / 4 tokens; `red`: 8 x NT fp32 of
// shared memory behind the barriers
template <typename T, int NT>
__device__ __forceinline__ void residual_epilogue(const GemmParams &p, const ResidualTiles &tiles, const float (&acc)[NT / 2], int tb, int block,
                                                  int n, int n_end, int tile, int t, int lane, uint32_t red) {
  T *yout = static_cast<T *>(p.y);
  const T *rin = static_cast<const T *>(tiles.res_in);
  T *rout = static_cast<T *>(tiles.res_out);
  float sq[NT / 4];   // token 8j + 2t + e: h^2 of this thread's two columns
#pragma unroll
  for (int i = 0; i < NT / 4; ++i) sq[i] = 0.f;
#pragma unroll
  for (int hi = 0; hi < 2; ++hi) {
    const int nn = n + 8 * hi;
    if (nn >= n_end) continue;
    const bool has_bias = p.bias != nullptr;
    const float bias_f = has_bias ? Traits<T>::to_float(static_cast<const T *>(p.bias)[nn]) : 0.f;
#pragma unroll
    for (int j = 0; j < NT / 8; ++j) {
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const int64_t m = static_cast<int64_t>(tb) * NT + 8 * j + 2 * t + e;
        if (m < p.M) {
          T v = Traits<T>::from_float(acc[4 * j + 2 * hi + e]);
          if (has_bias) v = Traits<T>::from_float(Traits<T>::to_float(v) + bias_f);
          const int64_t o = m * p.L.N + nn;
          if (yout) yout[o] = v;
          const T h = Traits<T>::from_float(Traits<T>::to_float(v) + Traits<T>::to_float(rin[o]));
          rout[o] = h;
          const float hf = Traits<T>::to_float(h);
          sq[2 * j + e] += hf * hf;
        }
      }
    }
  }
  if (!tiles.stats) return;
  const int g = lane >> 2;
#pragma unroll
  for (int i = 0; i < NT / 4; ++i) {
    float v = sq[i];
#pragma unroll
    for (int o = 4; o < 32; o <<= 1) v += __shfl_xor_sync(0xFFFFFFFFu, v, o);   // the 8 g lanes: 16 columns of this warp
    if (g == 0) sts_f32(red + 4 * (tile * NT + 8 * (i >> 1) + 2 * t + (i & 1)), v);
  }
  named_bar_sync(1, 128 * kGemmConsumers);
  const int c = threadIdx.x - 128;   // consumer thread 0 .. 255: token c of the tile
  const int64_t m = static_cast<int64_t>(tb) * NT + c;
  if (c < NT && m < p.M) {
    float s = lds_f32(red + 4 * c);
#pragma unroll
    for (int w = 1; w < 4 * kGemmConsumers; ++w) s += lds_f32(red + 4 * (w * NT + c));   // warp order
    tiles.stats[static_cast<int64_t>(block) * p.M + m] = s;
  }
}

template <typename T, int NT, typename Tiles>
__global__ void __launch_bounds__(kGemmThreads, 1) wg_gemm_kernel(const GemmParams p, const Tiles tiles) {
  extern __shared__ __align__(128) uint8_t smem[];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const uint32_t smem0 = smem_u32(smem);
  constexpr uint32_t b_stage_bytes = NT * 128;
  const uint32_t w_ring = smem0, b_ring = smem0 + kWStages * kWStage;
  const uint32_t bars = b_ring + kBStages * b_stage_bytes;
  const uint32_t bar_wfull = bars, bar_wempty = bars + 64, bar_bfull = bars + 128, bar_bempty = bars + 160;

  const int block = blockIdx.x % p.L.blocks_total, tb = blockIdx.x / p.L.blocks_total;   // 128-column block (over all partitions), token block
  int part = 0;
  while (block >= p.L.part_block_begin[part + 1]) ++part;
  const int n0 = p.L.part_col_begin[part] + (block - p.L.part_block_begin[part]) * kBlockN, n_end = p.L.part_col_begin[part + 1];
  const int rounds = p.L.groups;
  const uint8_t *packed = p.packed;
  if constexpr (Tiles::kGrouped) {
    pdl_wait();   // the routing table (written two launches back) names the tile's expert
    if (tb >= *tiles.live_tiles) return;
    packed += tiles.tile_expert[tb] * tiles.expert_stride;
  }

  if (threadIdx.x == 0) {
    for (int s = 0; s < kWStages; ++s) { mbar_init(bar_wfull + 8 * s, 1); mbar_init(bar_wempty + 8 * s, 4 * kGemmConsumers); }
    for (int s = 0; s < kBStages; ++s) { mbar_init(bar_bfull + 8 * s, 1); mbar_init(bar_bempty + 8 * s, kGemmConsumers); }
    fence_mbar_init();
  }
  __syncthreads();

  if (warp == 0) {
    // ================= weight producer: independent of the pre-pass; every 128-column block is re-read by
    // all token blocks, so the records stay under the normal L2 policy (no evict-first here)
    if (lane == 0) {
      const uint32_t rec_bytes = static_cast<uint32_t>(p.L.rec_bytes);
      const uint8_t *rec = packed + p.L.rec_off + static_cast<size_t>(block) * p.L.groups * rec_bytes;
      for (int r = 0; r < rounds; ++r) {
        const int ws = r % kWStages, wit = r / kWStages;
        if (wit > 0) mbar_wait(bar_wempty + 8 * ws, (wit - 1) & 1);
        mbar_arrive_expect_tx(bar_wfull + 8 * ws, rec_bytes);
        asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                     ::"r"(w_ring + ws * kWStage), "l"(rec + static_cast<size_t>(r) * rec_bytes), "r"(rec_bytes), "r"(bar_wfull + 8 * ws)
                     : "memory");
      }
    }
  } else if (warp == 1) {
    // ================= x_rot producer: one contiguous NT x 64 operand tile per stage
    if (lane == 0) {
      const uint8_t *xr_tile = p.xr + static_cast<size_t>(part) * p.xr_part_stride +
                               static_cast<size_t>(tb) * (p.L.K / 64) * b_stage_bytes;
      pdl_wait();   // x_rot is written by the pre-pass kernel
      for (int bi = 0; bi < 2 * rounds; ++bi) {
        const int bs = bi % kBStages, bit = bi / kBStages;
        if (bit > 0) mbar_wait(bar_bempty + 8 * bs, (bit - 1) & 1);
        mbar_arrive_expect_tx(bar_bfull + 8 * bs, b_stage_bytes);
        asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                     ::"r"(b_ring + bs * b_stage_bytes), "l"(xr_tile + static_cast<size_t>(bi) * b_stage_bytes), "r"(b_stage_bytes),
                       "r"(bar_bfull + 8 * bs)
                     : "memory");
      }
    }
  } else if (warp >= 4) {
    // ================= consumers: warpgroup wg owns output columns 64 wg .. 64 wg + 63 of the block
    const int wg = (warp >> 2) - 1, w = warp & 3;
    const int g = lane >> 2, t = lane & 3;
    const int tile = 4 * wg + w, r = 16 * tile + g;   // my 16-row tile, rows r and r + 8 inside the block
    const bool q2 = p.L.qhalves == 2;
    const uint32_t zero_off = q2 ? block_zero_off(2) : block_zero_off(1);
    const uint64_t desc_hi = smem_desc_kmajor(0, NT * 16, 128);
    float acc[NT / 2];
#pragma unroll
    for (int i = 0; i < NT / 2; ++i) acc[i] = 0.f;
    uint32_t a0[32], a1[32];

    // dequantise round rr into `a` (the record's ring stage is released as soon as the fragments are in registers)
    auto dequant = [&](int rr, uint32_t (&a)[32]) {
      const int ws = rr % kWStages;
      mbar_wait(bar_wfull + 8 * ws, (rr / kWStages) & 1);
      gemm_dequant_round<T>(w_ring + ws * kWStage, q2, zero_off, tile, lane, a);
      __syncwarp();
      if (lane == 0) mbar_arrive(bar_wempty + 8 * ws);
    };
    // issue the 8 wgmmas of round rr (B: its two x_rot stages), one commit group
    auto issue = [&](int rr, const uint32_t (&a)[32]) {
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int bi = 2 * rr + h, bs = bi % kBStages;
        mbar_wait(bar_bfull + 8 * bs, (bi / kBStages) & 1);
      }
      fence_operands(acc);
      wgmma_fence();
#pragma unroll
      for (int s = 0; s < 8; ++s) {
        const int bs = (2 * rr + (s >> 2)) % kBStages;
        const uint64_t desc = desc_hi | static_cast<uint64_t>(((b_ring + bs * b_stage_bytes + (s & 3) * (NT * 32)) >> 4) & 0x3FFF);
        Wgmma<T, NT>::mma(acc, a + 4 * s, desc);
      }
      wgmma_commit();
      fence_operands(acc);
    };
    // round rr's wgmmas have completed: its x_rot stages go back to the producer
    auto release = [&](int rr) {
      if (w == 0 && lane == 0) {
        mbar_arrive(bar_bempty + 8 * ((2 * rr) % kBStages));
        mbar_arrive(bar_bempty + 8 * ((2 * rr + 1) % kBStages));
      }
    };

    dequant(0, a0);
    for (int rr = 0; rr < rounds; rr += 2) {
      issue(rr, a0);
      if (rr + 1 < rounds) dequant(rr + 1, a1);
      wgmma_wait<0>();
      fence_operands(acc);
      release(rr);
      if (rr + 1 >= rounds) break;
      issue(rr + 1, a1);
      if (rr + 2 < rounds) dequant(rr + 2, a0);
      wgmma_wait<0>();
      fence_operands(acc);
      release(rr + 1);
    }

    // ---- epilogue: acc[4j + e] = rows r (e < 2) / r + 8, tokens 8j + 2t + (e & 1)
    if constexpr (Tiles::kResidual) {
      residual_epilogue<T, NT>(p, tiles, acc, tb, block, n0 + r, n_end, tile, t, lane, bars + 256);
      return;
    }
    T *yout = static_cast<T *>(p.y);
    const bool has_bias = p.bias != nullptr;
#pragma unroll
    for (int hi = 0; hi < 2; ++hi) {
      const int n = n0 + r + 8 * hi;
      if (n >= n_end) continue;
      const float bias_f = has_bias ? Traits<T>::to_float(static_cast<const T *>(p.bias)[n]) : 0.f;
#pragma unroll
      for (int j = 0; j < NT / 8; ++j) {
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const int64_t m = static_cast<int64_t>(tb) * NT + 8 * j + 2 * t + e;
          if constexpr (Tiles::kGrouped) {
            const int row = tiles.rows[m];
            if (row >= 0) yout[static_cast<int64_t>(row) * p.L.N + n] = Traits<T>::from_float(acc[4 * j + 2 * hi + e]);
          } else if (m < p.M) {
            T v = Traits<T>::from_float(acc[4 * j + 2 * hi + e]);
            if (has_bias) v = Traits<T>::from_float(Traits<T>::to_float(v) + bias_f);
            yout[m * p.L.N + n] = v;
          }
        }
      }
    }
  }
}

// ------------------------------------------------------------------ host side
// Tokens per output tile.  A round is 8 wgmmas of m64 x NT x k16 per consumer warpgroup (~NT * 8 tensor cycles for both) against
// ~400 cycles of dequant per warpgroup: NT = 128 tiles keep the tensor pipe busy, but a small batch x few column blocks gives fewer
// tiles than SMs (256 tokens x 4096 columns = 64 tiles) and is better cut finer -- pick the size with the shortest critical path
// (waves x (rounds x max(dequant, MMA) + per-tile prologue / epilogue)).
// Pure host logic: `sms` is the device's SM count (tests drive it through paro_debug_gemm_plan).
static int pick_nt(int64_t M, const Layout &L, int sms) {
  // from the largest tile the batch allows downwards: a finer tile must be CLEARLY better on paper (>= 25 %) -- finer tiles
  // re-read the weights more often and sit at the dequant limit, which the model prices optimistically
  int best = 0;
  double best_t = 0;
  for (int nt = 128; nt >= 32; nt /= 2) {
    if (nt > 32 && M <= nt / 2) continue;   // never pad the batch more than 2x
    const int64_t tiles = (M + nt - 1) / nt * L.blocks_total;
    const int64_t waves = (tiles + sms - 1) / sms;
    const double per_round = nt * 8.0 > 400.0 ? nt * 8.0 : 400.0;
    const double t = static_cast<double>(waves) * (L.groups * per_round + 4000.0 + 16.0 * nt);
    if (!best || t < 0.75 * best_t) { best = nt; best_t = t; }
  }
  return best;
}

// test hook: out[0] = tokens per tile (NT), out[1] = token blocks
int gemm_debug_plan(const Layout &L, int64_t M, int sms, int32_t *out) {
  if (M < 1 || sms < 1) { set_error("debug_gemm_plan: bad M / sms"); return PARO_EINVAL; }
  const int nt = pick_nt(M, L, sms);
  out[0] = nt;
  out[1] = static_cast<int32_t>((M + nt - 1) / nt);
  return PARO_OK;
}

size_t gemm_workspace_bytes(const Layout &L, int64_t max_m) {
  const int64_t m_pad = (max_m + 255) / 256 * 256;           // whatever tile size a later call picks
  return static_cast<size_t>(L.n_parts) * m_pad * L.K * 2;   // x_rot per partition, B-operand tile order
}

template <typename T, int NT, typename Tiles>
static int launch_gemm(const GemmParams &p, const Tiles &tiles, cudaStream_t stream) {
  auto kern = wg_gemm_kernel<T, NT, Tiles>;
  const size_t smem = static_cast<size_t>(kWStages) * kWStage + static_cast<size_t>(kBStages) * NT * 128 + 256 +
                      (Tiles::kResidual ? static_cast<size_t>(4 * kGemmConsumers) * NT * 4 : 0);   // the residual epilogue's warp sums
  PARO_CUDA_OK(smem_opt_in(kern, static_cast<int>(smem)));
  cudaLaunchConfig_t cfg;
  cudaLaunchAttribute attr[2];
  launch_config(cfg, attr, p.L.blocks_total * p.tok_blocks, kGemmThreads, smem, stream, 0, true);   // PDL: prologue + first weight stages overlap the pre-pass
  PARO_CUDA_OK(cudaLaunchKernelEx(&cfg, kern, p, tiles));
  note_launches(1);
  return PARO_OK;
}

template <typename T, typename Tiles = DenseTiles>
static int launch_gemm_nt(const GemmParams &p, cudaStream_t stream, const Tiles &tiles = Tiles{}) {
  if (p.NT == 128) return launch_gemm<T, 128>(p, tiles, stream);
  if (p.NT == 64) return launch_gemm<T, 64>(p, tiles, stream);
  return launch_gemm<T, 32>(p, tiles, stream);
}

// a linear's GEMM over M rows in tiles of NT, x_rot (m_pad rows per partition) at xr
static GemmParams dense_params(const Layout &L, const void *packed, const void *xr, void *y, const void *bias, int64_t M, int NT, int64_t m_pad) {
  GemmParams p;
  p.packed = static_cast<const uint8_t *>(packed);
  p.xr = static_cast<const uint8_t *>(xr);
  p.y = y;
  p.bias = bias;
  p.L = L;
  p.M = static_cast<int>(M); p.NT = NT;
  p.tok_blocks = static_cast<int>(m_pad / NT);
  p.xr_part_stride = static_cast<long long>(m_pad) * L.K * 2;
  return p;
}

// ------------------------------------------------------------------ prefill chain (paro_prefill_chain_forward)
// Workspace: the rotated operand, sized for the largest step and shared by all (a step's pre-pass runs after the previous GEMM
// is done with it), then one fp32 [blocks][M] statistics region per ADD_RESIDUAL step an RMSNORM step consumes, then the
// output of every consumed STORE step without y.  Offsets 256-byte aligned; 0 = no region.
struct PrefillWs {
  size_t stats_off[PARO_CHAIN_MAX_STEPS], out_off[PARO_CHAIN_MAX_STEPS], end;
};

static PrefillWs prefill_ws(const HostStep *steps, int n, int64_t M) {
  auto up = [](size_t b) { return (b + 255) / 256 * 256; };
  PrefillWs w = {};
  size_t off = 0;
  for (int i = 0; i < n; ++i) {
    const size_t b = gemm_workspace_bytes(steps[i].L, M);
    if (b > off) off = b;
  }
  off = up(off);
  for (int i = 0; i < n; ++i) {
    const HostStep &h = steps[i];
    const bool consumed = i + 1 < n && !steps[i + 1].x;
    if (consumed && h.epi_op == PARO_EPI_ADD_RESIDUAL && steps[i + 1].x_op == PARO_XOP_RMSNORM) {
      w.stats_off[i] = off;
      off += up(static_cast<size_t>(h.L.blocks_total) * M * 4);
    }
    if (consumed && h.epi_op == PARO_EPI_STORE && !h.y) {
      w.out_off[i] = off;
      off += up(static_cast<size_t>(M) * h.L.N * 2);
    }
  }
  w.end = off;
  return w;
}

size_t prefill_chain_workspace_bytes(const HostStep *steps, int n, int64_t M) { return prefill_ws(steps, n, M).end; }

// Per step two launches: the pre-pass with the step's x op as a plain launch (it reads what the previous GEMM wrote and
// overwrites the operand that GEMM read; one launch rotates x for every partition, where one rotate launch per partition
// cost 3 x ~7 us at 256 tokens), then the GEMM with PDL.  A single linear above 16 rows runs as a one-step chain.
int prefill_chain_forward(const HostStep *steps, int n, int64_t M, void *workspace, size_t workspace_bytes, cudaStream_t stream) {
  const PrefillWs w = prefill_ws(steps, n, M);
  if (workspace_bytes < w.end) { set_error("workspace too small: have %zu, need %zu", workspace_bytes, w.end); return PARO_EWORKSPACE; }
  uint8_t *ws = static_cast<uint8_t *>(workspace);
  const void *prev_out = nullptr;
  const float *prev_stats = nullptr;
  int prev_blocks = 0;
  for (int i = 0; i < n; ++i) {
    const HostStep &h = steps[i];
    const Layout &L = h.L;
    const int NT = pick_nt(M, L, planning_sms());
    const int64_t m_pad = (M + NT - 1) / NT * NT;
    int rc = rotate_chain_launch(L, h.packed, h.x_op, h.x ? h.x : prev_out, h.norm_w, prev_stats, prev_blocks, h.eps, ws, M, m_pad, NT, stream);
    if (rc) return rc;
    void *y = h.y ? h.y : w.out_off[i] ? ws + w.out_off[i] : nullptr;
    const GemmParams p = dense_params(L, h.packed, ws, y, h.bias, M, NT, m_pad);
    const bool bf16 = L.dtype == PARO_BF16;
    if (h.epi_op == PARO_EPI_ADD_RESIDUAL) {
      float *stats = w.stats_off[i] ? reinterpret_cast<float *>(ws + w.stats_off[i]) : nullptr;
      const ResidualTiles tiles = {h.res_in, h.res_out, stats};
      rc = bf16 ? launch_gemm_nt<__nv_bfloat16>(p, stream, tiles) : launch_gemm_nt<__half>(p, stream, tiles);
      prev_out = h.res_out;
      prev_stats = stats;
    } else {
      rc = bf16 ? launch_gemm_nt<__nv_bfloat16>(p, stream) : launch_gemm_nt<__half>(p, stream);
      prev_out = y;
      prev_stats = nullptr;
    }
    if (rc) return rc;
    prev_blocks = L.blocks_total;
  }
  return PARO_OK;
}

// One grouped GEMM of a MoE block (paro_moe_grouped.cu): y[rows[m], :] = x_rot[m, :] . W[expert of m's tile] for every live tile
// slot.  `xr` holds `slots` tiles of NT rows in B-operand order, written by the pre-pass; every partition of L reads it (a MoE
// block's gate and up share one rotation).  `packed` is expert 0's buffer, expert e's lies `expert_stride` bytes further on.
int gemm_grouped_launch(const Layout &L, const void *packed, long long expert_stride, const void *xr, void *y, int NT, int slots,
                        const int32_t *rows, const int32_t *tile_expert, const int32_t *live_tiles, int dtype, cudaStream_t stream) {
  GemmParams p = {};
  p.L = L;
  p.packed = static_cast<const uint8_t *>(packed);
  p.xr = static_cast<const uint8_t *>(xr);
  p.y = y;
  p.bias = nullptr;
  p.M = slots * NT; p.NT = NT;
  p.tok_blocks = slots;
  p.xr_part_stride = 0;
  const GroupedTiles tiles = {rows, tile_expert, live_tiles, expert_stride};
  if (dtype == PARO_BF16) return launch_gemm_nt<__nv_bfloat16>(p, stream, tiles);
  return launch_gemm_nt<__half>(p, stream, tiles);
}

}  // namespace paro
