// MoE expert block for any batch (T >= 1 tokens, top-k routing) as grouped INT4 wgmma GEMMs, routing read on the device.
// Same semantics as paro_moe_forward (paro_moe.cu), which serves decode batches only:
//
//   h[t, s]  = T(rotate_gu(x[t]) . W_gu[e_s])                      for every valid slot s of token t
//   y_s      = T(rotate_d(T(T(silu(gate)) * up)) . W_d[e_s])
//   y[t]     = T(sum over (expert id, slot) ascending of fp32(y_s) * w_s, from 0, product rounded first)
//
// Six launches, no host synchronisation, no allocation:
//   1. route     one CTA: counts the valid entries (t, s) of every expert, gives each expert a run of NT-row tiles and writes
//                the routing table -- the entries sorted by (expert, token, slot), each expert's run padded with -1 to a
//                whole tile, the expert of every tile and the live tile count.  Rewritten in full every launch.
//   2. pre-pass  rotate_tile_kernel (paro_rotate.cu) with a gather row source: x[t] of every table position, rotated by the
//                block's gate_up rotation, straight into the B-operand tile order of the GEMM; padding rows zero.
//   3. GEMM      wg_gemm_kernel (paro_gemm.cu) with the grouped tile source: CTA = (tile slot, 128-column block), the weights
//                of the tile's expert, the epilogue scatters row (t, s) to h[t, s].  Slots past the live count exit at once.
//   4. pre-pass  the same kernel with a SiLU * up row source over h (silu_mul2, the decode kernel's), the down rotation.
//   5. GEMM      the down projection, y_s rounded to T into a [T * k, hidden] workspace region.
//   6. combine   one CTA per token: its valid slots in (expert id, slot) order, fp32 products and sums as above.
// Each output row is the dot product of one rotated row with one expert's columns, whatever tile it shares, so the result
// does not depend on the tiling: permuting tokens or slots permutes the outputs bit for bit.
//
// The grids are sized for the worst routing: at most floor(T k / NT) + min(E, T k) tiles are live.  NT is chosen on the host
// from (T, k, E) only, so one plan serves every routing and a captured CUDA graph stays valid while the ids change.
#include "paro_launch.h"
#include "paro_tc_common.cuh"

namespace paro {

constexpr int kGroupedMaxEntries = PARO_MOE_GROUPED_MAX_ENTRIES;   // T * top_k
constexpr int kGroupedMaxExperts = PARO_MOE_GROUPED_MAX_EXPERTS;   // one route thread per expert
constexpr int kRouteThreads = 1024, kRouteWarps = kRouteThreads / 32;
constexpr int kCombineThreads = 128;

// ------------------------------------------------------------------ 1. route
// Warp w owns a contiguous segment of the n = T * k entries.  Pass one counts each expert's entries per segment; a scan over the
// experts gives expert e its first tile; pass two places every entry at its expert's start + the entries of e in earlier segments
// + earlier lanes of the same 32-entry step (__match_any_sync): a stable sort by (expert, entry index) without atomics.
__global__ void __launch_bounds__(kRouteThreads, 1) moe_route_kernel(const int32_t *__restrict__ ids, int n, int E, int nt, int32_t *__restrict__ rows,
                                                                     int32_t *__restrict__ tile_expert, int32_t *__restrict__ live_tiles) {
  extern __shared__ int s_pos[];   // [warp][E]: entries of expert e in warp w's segment, then where the next of them goes
  __shared__ int s_warp_tiles[kRouteWarps];
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  for (int i = tid; i < kRouteWarps * E; i += kRouteThreads) s_pos[i] = 0;
  __syncthreads();
  const int seg = (n + kRouteWarps - 1) / kRouteWarps, b0 = min(n, warp * seg), b1 = min(n, b0 + seg);
  int *mine = s_pos + warp * E;
  auto walk = [&](bool place) {
#pragma unroll 1
    for (int i0 = b0; i0 < b1; i0 += 32) {
      const int i = i0 + lane;
      int e = i < b1 ? ids[i] : -1;
      if (e < 0 || e >= E) e = -1;
      const uint32_t peers = __match_any_sync(0xFFFFFFFFu, e);
      if (place && e >= 0) rows[mine[e] + __popc(peers & ((1u << lane) - 1u))] = i;
      __syncwarp();
      if (e >= 0 && lane == __ffs(peers) - 1) mine[e] += __popc(peers);
      __syncwarp();
    }
  };
  walk(false);
  __syncthreads();
  int count = 0;
  if (tid < E)
    for (int w = 0; w < kRouteWarps; ++w) count += s_pos[w * E + tid];
  const int tiles = (count + nt - 1) / nt;
  // exclusive scan of the tile counts over the experts (thread e = expert e)
  int incl = tiles;
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) {
    const int v = __shfl_up_sync(0xFFFFFFFFu, incl, d);
    if (lane >= d) incl += v;
  }
  if (lane == 31) s_warp_tiles[warp] = incl;
  __syncthreads();
  if (warp == 0) {
    int v = s_warp_tiles[lane];
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
      const int u = __shfl_up_sync(0xFFFFFFFFu, v, d);
      if (lane >= d) v += u;
    }
    s_warp_tiles[lane] = v;
  }
  __syncthreads();
  if (tid < E) {
    const int first = (warp ? s_warp_tiles[warp - 1] : 0) + incl - tiles;
    int pos = first * nt;
    for (int w = 0; w < kRouteWarps; ++w) {
      const int c = s_pos[w * E + tid];
      s_pos[w * E + tid] = pos;
      pos += c;
    }
    for (int p = pos; p < (first + tiles) * nt; ++p) rows[p] = -1;
    for (int j = 0; j < tiles; ++j) tile_expert[first + j] = tid;
  }
  if (tid == 0) *live_tiles = s_warp_tiles[kRouteWarps - 1];
  __syncthreads();
  walk(true);
}

// ------------------------------------------------------------------ 6. combine
template <typename T>
__global__ void __launch_bounds__(kCombineThreads) moe_combine_kernel(const int32_t *__restrict__ ids, const float *__restrict__ wts,
                                                                      const T *__restrict__ ys, T *__restrict__ y, int k, int E, int H) {
  __shared__ int s_order[16];   // the token's valid slots in (expert id, slot) order
  const int t = blockIdx.x, tid = threadIdx.x;
  const int32_t *tok_ids = ids + static_cast<int64_t>(t) * k;
  bool ok = false;
  if (tid < k) {
    const int e = tok_ids[tid];
    ok = e >= 0 && e < E;
    if (ok) {
      int r = 0;
      for (int s = 0; s < k; ++s) {
        const int f = tok_ids[s];
        r += f >= 0 && f < E && (f < e || (f == e && s < tid));
      }
      s_order[r] = tid;
    }
  }
  const int nv = __syncthreads_count(ok);
  for (int c = tid * 8; c < H; c += kCombineThreads * 8) {
    float acc[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    for (int r = 0; r < nv; ++r) {
      const int s = s_order[r];
      const float w = wts[static_cast<int64_t>(t) * k + s];
      const uint4 v = *reinterpret_cast<const uint4 *>(ys + (static_cast<int64_t>(t) * k + s) * H + c);
      const T *pv = reinterpret_cast<const T *>(&v);
#pragma unroll
      for (int i = 0; i < 8; ++i) acc[i] = __fadd_rn(acc[i], __fmul_rn(Traits<T>::to_float(pv[i]), w));
    }
    uint4 o;
    T *po = reinterpret_cast<T *>(&o);
#pragma unroll
    for (int i = 0; i < 8; ++i) po[i] = Traits<T>::from_float(acc[i]);
    *reinterpret_cast<uint4 *>(y + static_cast<int64_t>(t) * H + c) = o;
  }
}

// ------------------------------------------------------------------ host side
static size_t align256(size_t b) { return (b + 255) / 256 * 256; }

struct GroupedPlan {
  int nt, slots;                                          // rows per tile, tile slots (the worst case's tile count)
  size_t table_bytes, operand_bytes, ys_bytes, total;     // workspace: routing table, B operand (both pre-passes), y_s
  int grid[6];                                            // route, gate_up pre-pass, gate_up GEMM, down pre-pass, down GEMM, combine
};

// Rows per tile from (n = T * k, E) alone.  With U = min(E, n) experts of a = n / U entries each, about max(U, n / NT + U / 2)
// tiles are live (each expert's last tile half full); a tile costs its rounds (16 nominal, each the larger of the NT * 8 tensor
// cycles and the ~400-cycle dequant, as in paro_gemm.cu's pick_nt) plus its prologue and epilogue.  Small per-expert batches take
// NT = 32 (less padding), large ones 128 (fewer rounds per row).
static int grouped_pick_nt(int64_t n, int E) {
  const double U = static_cast<double>(E < n ? E : n);
  int best = 0;
  double best_cost = 0;
  for (int nt = 32; nt <= 128; nt *= 2) {
    const double tiles = U > n / static_cast<double>(nt) + U / 2 ? U : n / static_cast<double>(nt) + U / 2;
    const double per_round = nt * 8.0 > 400.0 ? nt * 8.0 : 400.0;
    const double cost = tiles * (16 * per_round + 4000.0 + 16.0 * nt);
    if (!best || cost < best_cost) { best = nt; best_cost = cost; }
  }
  return best;
}

static int grouped_check(const paro_moe_desc *d, int64_t T, int32_t k, MoeShapes &ms, GroupedPlan &gp) {
  int rc = moe_check_desc(d, ms);
  if (rc) return rc;
  if (T < 1 || k < 1 || k > 16 || T * k > kGroupedMaxEntries) {
    set_error("moe_grouped: T >= 1, 1 <= top_k <= 16 and T * top_k <= %d supported, got T = %lld, top_k = %d", kGroupedMaxEntries,
              static_cast<long long>(T), k);
    return PARO_EUNSUPPORTED;
  }
  if (ms.E > kGroupedMaxExperts) {
    set_error("moe_grouped: n_experts <= %d supported, got %d", kGroupedMaxExperts, ms.E);
    return PARO_EUNSUPPORTED;
  }
  const int n = static_cast<int>(T * k);
  gp.nt = grouped_pick_nt(n, ms.E);
  gp.slots = n / gp.nt + (ms.E < n ? ms.E : n);
  const int64_t rows = static_cast<int64_t>(gp.slots) * gp.nt;
  gp.table_bytes = align256(static_cast<size_t>(rows + gp.slots + 1) * 4);
  gp.operand_bytes = align256(static_cast<size_t>(rows) * (ms.H > ms.I ? ms.H : ms.I) * 2);
  gp.ys_bytes = align256(static_cast<size_t>(n) * ms.H * 2);
  gp.total = gp.table_bytes + gp.operand_bytes + gp.ys_bytes;
  const int64_t rot_gu = (rows / 8 * (ms.H / 128) + 3) / 4, rot_d = (rows / 8 * (ms.I / 128) + 3) / 4;
  gp.grid[0] = 1;
  gp.grid[1] = static_cast<int>(rot_gu);
  gp.grid[2] = ms.gu.blocks_total * gp.slots;
  gp.grid[3] = static_cast<int>(rot_d);
  gp.grid[4] = ms.dn.blocks_total * gp.slots;
  gp.grid[5] = static_cast<int>(T);
  return PARO_OK;
}

size_t moe_grouped_workspace_bytes(const paro_moe_desc *d, int64_t T, int32_t k) {
  MoeShapes ms;
  GroupedPlan gp;
  if (grouped_check(d, T, k, ms, gp)) return 0;
  return gp.total;
}

int moe_grouped_debug_plan(const paro_moe_desc *d, int64_t T, int32_t k, int32_t *out) {
  MoeShapes ms;
  GroupedPlan gp;
  const int rc = grouped_check(d, T, k, ms, gp);
  if (rc) return rc;
  out[0] = gp.nt;
  out[1] = gp.slots;
  for (int i = 0; i < 6; ++i) out[2 + i] = gp.grid[i];
  out[8] = static_cast<int32_t>(gp.table_bytes / 256);
  out[9] = static_cast<int32_t>(gp.operand_bytes / 256);
  out[10] = static_cast<int32_t>(gp.ys_bytes / 256);
  out[11] = static_cast<int32_t>(gp.total / 256);
  return PARO_OK;
}

int moe_grouped_forward(const paro_moe_desc *d, const void *x, const int32_t *ids, const float *wts, int64_t T, int32_t k, void *h, void *y,
                        void *workspace, size_t workspace_bytes, cudaStream_t stream) {
  MoeShapes ms;
  GroupedPlan gp;
  int rc = grouped_check(d, T, k, ms, gp);
  if (rc) return rc;
  if (!x || !ids || !wts || !h || !y || !workspace || !d->gate_up_packed || !d->down_packed) { set_error("moe_grouped: null pointer argument"); return PARO_EINVAL; }
  if ((reinterpret_cast<uintptr_t>(d->gate_up_packed) | reinterpret_cast<uintptr_t>(d->down_packed) | reinterpret_cast<uintptr_t>(workspace)) & 255 ||
      (reinterpret_cast<uintptr_t>(x) | reinterpret_cast<uintptr_t>(h) | reinterpret_cast<uintptr_t>(y)) & 15 ||
      (reinterpret_cast<uintptr_t>(ids) | reinterpret_cast<uintptr_t>(wts)) & 3) {
    set_error("moe_grouped: packed buffers and workspace must be 256-byte, x / h / y 16-byte, ids / weights 4-byte aligned");
    return PARO_EINVAL;
  }
  if (workspace_bytes < gp.total) {
    set_error("moe_grouped: workspace too small: have %zu, need %zu", workspace_bytes, gp.total);
    return PARO_EWORKSPACE;
  }
  const int n = static_cast<int>(T * k), rows_max = gp.slots * gp.nt, dtype = d->gate_up->dtype;
  uint8_t *ws = static_cast<uint8_t *>(workspace);
  int32_t *rows = reinterpret_cast<int32_t *>(ws), *tile_expert = rows + rows_max, *live = tile_expert + gp.slots;
  uint8_t *operand = ws + gp.table_bytes, *ys = operand + gp.operand_bytes;
  const uint8_t *gu = static_cast<const uint8_t *>(d->gate_up_packed), *dn = static_cast<const uint8_t *>(d->down_packed);

  PARO_CUDA_OK(smem_opt_in(moe_route_kernel, kRouteWarps * kGroupedMaxExperts * 4));
  moe_route_kernel<<<1, kRouteThreads, kRouteWarps * ms.E * 4, stream>>>(ids, n, ms.E, gp.nt, rows, tile_expert, live);
  PARO_CUDA_OK(cudaGetLastError());
  note_launches(1);
  if ((rc = rotate_routed_launch(ms.gu, gu, false, x, rows, live, k, operand, rows_max, gp.nt, stream))) return rc;
  if ((rc = gemm_grouped_launch(ms.gu, gu, static_cast<long long>(d->gate_up_stride), operand, h, gp.nt, gp.slots, rows, tile_expert, live, dtype,
                                stream)))
    return rc;
  if ((rc = rotate_routed_launch(ms.dn, dn, true, h, rows, live, k, operand, rows_max, gp.nt, stream))) return rc;
  if ((rc = gemm_grouped_launch(ms.dn, dn, static_cast<long long>(d->down_stride), operand, ys, gp.nt, gp.slots, rows, tile_expert, live, dtype,
                                stream)))
    return rc;
  if (dtype == PARO_BF16)
    moe_combine_kernel<__nv_bfloat16><<<static_cast<unsigned>(T), kCombineThreads, 0, stream>>>(
        ids, wts, reinterpret_cast<const __nv_bfloat16 *>(ys), static_cast<__nv_bfloat16 *>(y), k, ms.E, ms.H);
  else
    moe_combine_kernel<__half><<<static_cast<unsigned>(T), kCombineThreads, 0, stream>>>(ids, wts, reinterpret_cast<const __half *>(ys),
                                                                                          static_cast<__half *>(y), k, ms.E, ms.H);
  PARO_CUDA_OK(cudaGetLastError());
  note_launches(1);
  return PARO_OK;
}

}  // namespace paro
