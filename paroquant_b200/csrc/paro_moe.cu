// MoE expert block for decode batches (T <= 16 tokens, top-k routing) in TWO launches with the routing read on the device.
// Replaces the reference's RotateSwitchGLU (/root/reference/paroquant/inference/backends/mlx/modules.py:159-212) on the
// expert format of cli/convert.py:281-406 (one gate_up and one down rotation shared by all experts).
//
//   launch 1 (gate_up):  h[t, s]  = T(rotate_gu(x[t]) . W_gu[e_s])                      for every valid slot s of token t
//   launch 2 (down):     y_s      = T(rotate_d(T(T(silu(gate)) * up)) . W_d[e_s])
//                        out[t]   = T(sum over (expert id, slot) ascending of fp32(y_s) * w_s, from 0, product rounded first)
//
// Both launches are one kernel template built from decode_kernel's pieces (paro_tc_common.cuh): 16 worker warps (8 row tiles x 2
// k halves, mma.sync with dequantised A fragments in registers, B = token rows rotated by rotation_tasks in shared memory) and
// a TMA producer warp streaming ONE record per ring stage.
//
// Routing.  After griddepcontrol.wait every CTA ranks the T * k <= 128 ids in shared memory: the ascending list of distinct
// valid experts u = 0..U-1 (ids outside [0, E) are dropped) and, per (u, token), the mask of slots that chose it.  The launch
// plan is fixed on the host for U_max = min(E, T * k); the work list below is built from the runtime U, so one plan serves every
// routing and a captured graph stays valid when the ids change.  The producer cannot prefetch before the routing is known.
//
// Work split.  One cluster of c CTAs per 128-column output block b.  The cluster's work items are (expert slot u, K slice s)
// for u < U, s < S (S slices of whole groups), u-major.  Item i runs on rank i mod c in wave i / c: the rank rotates the rows
// of expert u (its distinct tokens) over the slice's groups, streams that expert's records of block b and pushes its fp32
// partial [rows x 128] into rank 0's receive buffer through distributed shared memory.  One cluster barrier per wave; rank 0
// then adds the wave's partials in item order, i.e. for every expert its slices in ascending order, and finishes an expert
// after its last slice: launch 1 rounds and stores h for each of its slots, launch 2 rounds y_s and accumulates w_s * y_s.
// Fixed order everywhere, no global atomics: bit-reproducible for a given routing.  Receive buffers alternate by wave
// parity, so one barrier per wave suffices (a rank writes buffer w & 1 again only after the barrier of wave w + 1, which
// rank 0 reaches after reading it).
#include <cstdio>
#include <cstring>
#include <type_traits>

#include "paro_launch.h"
#include "paro_tc_common.cuh"

namespace paro {

constexpr int kMoeWorkers = 16;                  // 8 row tiles x 2 k halves
constexpr int kMoeThreads = 32 * (kMoeWorkers + 1);
constexpr int kMoeN = 16;                        // B operand rows per group (token rows of one expert, zero padded)
constexpr int kMoeMaxStages = 16;
constexpr int kMoeMaxEntries = 128;              // T * k: one thread per routing entry builds the table
constexpr int kMoeSmemLimit = 227 * 1024;
constexpr int kMoeRotBytes = kMoeWorkers * 1024; // rotation tiles (128 channels x 4 rows of T per warp); k-half exchange after
constexpr int kMoeTabBytes = 3 * 512 + kMoeMaxEntries * 16 * 4;   // ids, expert list, first-occurrence flags, slot masks [u][t]
constexpr int kMoeBarBytes = 16 * kMoeMaxStages;

struct MoeParams {
  const uint8_t *packed;        // expert e at packed + e * stride
  long long stride;
  const void *x;                // launch 1: x [T, K]; launch 2: h [T, k, 2 K] (gate | up)
  void *y;                      // launch 1: h [T, k, N]; launch 2: out [T, N]
  const int32_t *ids;
  const float *wts;
  int T, k, E;
  Layout L;                     // one expert's linear (gate_up: 2 partitions; down: 1)
  int c, S, nstages;
  int xb_off, rot_off, recv_off, tab_off, bar_off;
};

// ---- the work list, shared by the kernels and the host plan check (paro_debug_moe_plan)
// item i = (expert slot i / S, K slice i % S); slice s covers groups [s * G / S, (s + 1) * G / S)
PARO_HD inline int moe_slice_begin(int s, int S, int G) { return static_cast<int>(static_cast<long long>(s) * G / S); }
PARO_HD inline void moe_item(int i, int S, int G, int &u, int &g0, int &g1) {
  u = i / S;
  const int s = i - u * S;
  g0 = moe_slice_begin(s, S, G);
  g1 = moe_slice_begin(s + 1, S, G);
}
PARO_HD inline int moe_waves(int U, int S, int c) { return (U * S + c - 1) / c; }

__device__ __forceinline__ int nth_bit(uint32_t mask, int m) {
  for (int j = 0; j < m; ++j) mask &= mask - 1;
  return __ffs(mask) - 1;
}

template <typename T, bool DOWN>
__global__ void __launch_bounds__(kMoeThreads, 1) moe_kernel(const MoeParams p) {
  extern __shared__ __align__(128) uint8_t smem[];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const uint32_t smem0 = smem_u32(smem);
  const uint32_t xb = smem0 + p.xb_off, rot0 = smem0 + p.rot_off, recv = smem0 + p.recv_off;
  const uint32_t bar_wfull = smem0 + p.bar_off, bar_wempty = bar_wfull + 8 * kMoeMaxStages;
  int *s_ids = reinterpret_cast<int *>(smem + p.tab_off);
  int *s_uexp = s_ids + kMoeMaxEntries;
  int *s_first = s_uexp + kMoeMaxEntries;
  uint32_t *s_mask = reinterpret_cast<uint32_t *>(s_first + kMoeMaxEntries);   // [u][16 tokens]: slots of token t that chose u
  const int NS = p.nstages, c = p.c, S = p.S, G = p.L.groups;
  const int b = blockIdx.x / c, rank = blockIdx.x - b * c;   // rank == %cluster_ctarank
  const uint32_t rec_bytes = static_cast<uint32_t>(p.L.rec_bytes);

  if (warp == kMoeWorkers) {
    ring_init(bar_wfull, bar_wempty, NS, kMoeWorkers, lane);
    fence_mbar_init();
  }
  for (int i = threadIdx.x; i < kMoeMaxEntries * 16; i += kMoeThreads) s_mask[i] = 0u;
  __syncthreads();
  cluster_arrive_relaxed();   // phase 0: "this CTA runs" -- waited on before the first DSMEM push
  pdl_launch_dependents();
  pdl_wait();                 // ids, weights, x / h may come from the previous kernels in the stream

  // ---- routing table: distinct valid ids ascending (rank among first occurrences), slot masks per (expert slot, token)
  const int n = p.T * p.k, tid = threadIdx.x;
  if (tid < n) {
    const int e = p.ids[tid];
    s_ids[tid] = e >= 0 && e < p.E ? e : -1;
  }
  __syncthreads();
  if (tid < n) {
    const int e = s_ids[tid];
    int f = e >= 0;
    for (int j = 0; j < tid && f; ++j) f = s_ids[j] != e;
    s_first[tid] = f;
  }
  __syncthreads();
  if (tid < n) {
    const int e = s_ids[tid];
    if (e >= 0) {
      int u = 0;
      for (int j = 0; j < n; ++j) u += s_first[j] && s_ids[j] < e;
      if (s_first[tid]) s_uexp[u] = e;
      const int t = tid / p.k;
      atomicOr(&s_mask[u * 16 + t], 1u << (tid - t * p.k));
    }
  }
  const int U = __syncthreads_count(tid < n && s_first[tid]);
  const int nitems = U * S, nw = moe_waves(U, S, c);

  if (warp == kMoeWorkers) {
    // ================= producer: the records of my items, one bulk copy per ring stage.  It joins the cluster barrier of
    // every wave after issuing the wave's records, so it runs up to a ring ahead of the workers across waves.
    const uint64_t pol = policy_evict_first();
    RingProducer prod = {bar_wfull, bar_wempty, smem0, rec_bytes, NS, 0, 0};
#pragma unroll 1
    for (int w = 0; w < nw; ++w) {
      const int i = w * c + rank;
      if (i < nitems) {
        int u, g0, g1;
        moe_item(i, S, G, u, g0, g1);
        const uint8_t *src = p.packed + s_uexp[u] * p.stride + p.L.rec_off + (static_cast<size_t>(b) * G + g0) * rec_bytes;
#pragma unroll 1
        for (int g = g0; g < g1; ++g) {
          prod.issue([src] { return src; }, rec_bytes, pol, [] {});
          src += rec_bytes;
        }
      }
      cluster_wait_acquire();
      cluster_arrive_relaxed();
    }
    cluster_wait_acquire();
    return;
  }

  // ================= workers
  const int tile = warp & 7, kh = warp >> 3;
  const int g = lane >> 2, t4 = lane & 3;
  const RoundLane lo = round_lane<kMoeN>(p.L.qhalves == 2, tile, kh, lane);
  // the ring position persists across items and waves; a stage's record from its full barrier: smem0 + (fb - bar_wfull) / 8 * rec_bytes
  RingCursor rg = {bar_wfull, 0u, bar_wfull, bar_wfull + 8 * NS, 8 * kMoeMaxStages, rec_bytes / 8, smem0 - bar_wfull * (rec_bytes / 8), rec_bytes};
  const int ntok = p.T, nel = ntok * kBlockN;
  float yacc[4] = {0.f, 0.f, 0.f, 0.f}, oacc[4] = {0.f, 0.f, 0.f, 0.f};   // rank 0: elements tid + 512 q = (token, column)
  // my output columns (launch 1: gate_up has two partitions; a last partial block is masked at the stores)
  const int part = b >= p.L.part_block_begin[1] ? 1 : 0;
  const int n0 = p.L.part_col_begin[part] + (b - p.L.part_block_begin[part]) * kBlockN, n_end = p.L.part_col_begin[part + 1];
  cluster_wait_acquire();   // phase 0: every CTA of the cluster runs

#pragma unroll 1
  for (int w = 0; w < nw; ++w) {
    const int i = w * c + rank;
    if (i < nitems) {
      int u, g0, g1;
      moe_item(i, S, G, u, g0, g1);
      const int ng = g1 - g0;
      const uint32_t *umask = s_mask + u * 16;
      const uint32_t tokmask = __ballot_sync(0xFFFFFFFFu, lane < ntok && umask[lane & 15] != 0u);
      const int R = __popc(tokmask);
      // ---- B operand of the item: zero rows [R, 16), then the rotation tasks (group x block of up to 4 rows) of the expert's
      // rows: its tokens (`tokmask`) ascending.  Launch 1 reads x[t]; launch 2 reads h[t, first slot of t] and applies SiLU * up.
      const uint8_t *meta = p.packed + s_uexp[u] * p.stride + p.L.meta_off;   // partition 0 (gate and up share it)
      const int nq = R > 4 ? (R + 3) >> 2 : 1, ntasks = ng * nq;
      RotMeta rm;
      if (warp < ntasks) fetch_meta<false>(meta + static_cast<size_t>(g0 + warp / nq) * p.L.meta_group_bytes, p.L.krot, lane, rm);
      for (int idx = tid; idx < ng * (kMoeN * 16); idx += 32 * kMoeWorkers) sts128u(xb + idx * 16, make_uint4(0u, 0u, 0u, 0u));
      named_bar_sync(1, 32 * kMoeWorkers);
      {
        const uint32_t rot = rot0 + warp * 1024;
        auto stage_x = [&](auto rows, int gi, int m0, uint2 csw) {
          constexpr int ROWS = decltype(rows)::value;
          const int gk = g0 + gi;
          uint2 raw[ROWS];
#pragma unroll
          for (int j = 0; j < ROWS; ++j) {
            raw[j] = make_uint2(0u, 0u);
            if (m0 + j < R) {
              const int t = nth_bit(tokmask, m0 + j);
              if constexpr (DOWN) {
                const int slot = __ffs(umask[t]) - 1;   // duplicate slots of one token carry the same h row
                const T *row = static_cast<const T *>(p.x) + (static_cast<int64_t>(t) * p.k + slot) * (2 * p.L.K) + gk * kGroup + 4 * lane;
                const uint2 gate = __ldcg(reinterpret_cast<const uint2 *>(row)), up = __ldcg(reinterpret_cast<const uint2 *>(row + p.L.K));
                raw[j].x = silu_mul2<T>(gate.x, up.x);
                raw[j].y = silu_mul2<T>(gate.y, up.y);
              } else {
                raw[j] = __ldcg(reinterpret_cast<const uint2 *>(static_cast<const T *>(p.x) + static_cast<int64_t>(t) * p.L.K + gk * kGroup + 4 * lane));
              }
            }
          }
          scale_and_stage<T, ROWS>(rot, lane, raw, csw);
        };
        const int mg = p.L.meta_group_bytes;
        if (R == 1) rotation_tasks<T, 1, false>(rm, meta, mg, p.L.krot, g0, ntasks, nq, R, warp, kMoeWorkers, lane, rot, xb, kMoeN, stage_x);
        else if (R == 2) rotation_tasks<T, 2, false>(rm, meta, mg, p.L.krot, g0, ntasks, nq, R, warp, kMoeWorkers, lane, rot, xb, kMoeN, stage_x);
        else rotation_tasks<T, 4, false>(rm, meta, mg, p.L.krot, g0, ntasks, nq, R, warp, kMoeWorkers, lane, rot, xb, kMoeN, stage_x);
      }
      named_bar_sync(2, 32 * kMoeWorkers);   // B operand complete
      // ---- rounds: the item is one segment of the round loop
      auto seg_begin = [&](int, uint32_t &bx, int &len) {
        bx = xb + lo.x;
        len = ng;
      };
      auto seg_end = [&](int, float (&acc)[2][4]) {
        // the k halves meet in the (now free) rotation tiles in a fixed order; the k-half-0 warp pushes the sum to rank 0
        khalf_meet(acc, rot0 + tile * (8 * 128) + lane * 4, kh, 4 + tile, [&] {
          const uint32_t dst = map_to_rank(recv + ((w & 1) * c + rank) * (ntok * 512), 0);
#pragma unroll
          for (int q = 0; q < 8; ++q) {
            const int col = 16 * tile + g + 8 * ((q >> 1) & 1), m = 8 * (q >> 2) + 2 * t4 + (q & 1);
            if (m < R) st_cluster_f32(dst + nth_bit(tokmask, m) * 512 + col * 4, acc[q >> 2][q & 3]);
          }
        });
      };
      auto none = [](int) {};
      if (R > 8) segment_rounds<T, 2, kMoeN>(rg, lo, 1, seg_begin, seg_end, none, none);
      else segment_rounds<T, 1, kMoeN>(rg, lo, 1, seg_begin, seg_end, none, none);
    }
    cluster_arrive_release();   // my pushes of wave w are done
    cluster_wait_acquire();
    if (rank == 0) {
      // ---- the wave's partials in item order: slices of an expert ascending; an expert is finished after its last slice
#pragma unroll 1
      for (int pos = 0; pos < c; ++pos) {
        const int ii = w * c + pos;
        if (ii >= nitems) break;
        const int u = ii / S, s = ii - u * S;
        const uint32_t src = recv + ((w & 1) * c + pos) * (ntok * 512);
#pragma unroll
        for (int q = 0; q < 4; ++q) {
          const int e = tid + 32 * kMoeWorkers * q;
          if (e < nel) {
            const int t = e >> 7, col = e & 127;
            const uint32_t m = s_mask[u * 16 + t];
            if (m) yacc[q] += lds_f32(src + e * 4);
            if (s == S - 1) {
              if (m) {
                const T v = Traits<T>::from_float(yacc[q]);
                if constexpr (DOWN) {
                  const float yv = Traits<T>::to_float(v);
                  for (uint32_t mm = m; mm; mm &= mm - 1) oacc[q] = __fadd_rn(oacc[q], __fmul_rn(yv, p.wts[t * p.k + __ffs(mm) - 1]));
                } else {
                  const int nn = n0 + col;
                  if (nn < n_end)
                    for (uint32_t mm = m; mm; mm &= mm - 1) static_cast<T *>(p.y)[(static_cast<int64_t>(t) * p.k + __ffs(mm) - 1) * p.L.N + nn] = v;
                }
              }
              yacc[q] = 0.f;
            }
          }
        }
      }
    }
  }
  if constexpr (DOWN) {
    if (rank == 0) {
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        const int e = tid + 32 * kMoeWorkers * q;
        if (e < nel && n0 + (e & 127) < n_end) static_cast<T *>(p.y)[static_cast<int64_t>(e >> 7) * p.L.N + n0 + (e & 127)] = Traits<T>::from_float(oacc[q]);
      }
    }
  }
}

// ------------------------------------------------------------------ host side
struct MoePlan {
  int c, S, grid, nb, groups, ng_max, nstages, smem;
  int xb_off, rot_off, recv_off, tab_off, bar_off;
};

static bool moe_carve(const Layout &L, int T, int c, int S, MoePlan &m) {
  m.c = c; m.S = S; m.nb = L.blocks_total; m.groups = L.groups;
  m.ng_max = (L.groups + S - 1) / S;
  m.grid = m.nb * c;
  const int xb = m.ng_max * kMoeN * 256, recv = 2 * c * T * 512;
  const int fixed = xb + kMoeRotBytes + recv + kMoeTabBytes + kMoeBarBytes + 128;
  const int nst = ring_stages(kMoeSmemLimit - fixed, L.rec_bytes, kMoeMaxStages, 2, 4, false);   // even: segment_rounds
  if (!nst) return false;
  m.nstages = nst;
  m.xb_off = (nst * L.rec_bytes + 127) / 128 * 128;
  m.rot_off = m.xb_off + xb;
  m.recv_off = m.rot_off + kMoeRotBytes;
  m.tab_off = m.recv_off + recv;
  m.bar_off = m.tab_off + kMoeTabBytes;
  m.smem = m.bar_off + kMoeBarBytes;
  return m.smem <= kMoeSmemLimit;
}

// (cluster size c, K slices S) minimising the critical path in rounds at U_max experts: CTA waves of the grid x item waves x
// (rounds of an item + its rotation passes + the wave's barrier).  Small experts with short K want c = 8 and S = 1 (one
// expert per rank); few big experts want their K split (S > 1) so that every rank of every cluster has work.
static bool moe_choose_plan(const Layout &L, int T, int umax, int sms, MoePlan &best) {
  long best_cost = -1;
  for (int cs = 0; cs <= 3; ++cs) {
    const int c = 1 << cs;
    for (int S = 1; S <= L.groups; ++S) {
      MoePlan m;
      if (!moe_carve(L, T, c, S, m)) continue;
      const long cta_waves = (m.grid + sms - 1) / sms;
      const int nq = T > 4 ? (T + 3) / 4 : 1;
      const long passes = (m.ng_max * nq + kMoeWorkers - 1) / kMoeWorkers;
      const long cost = cta_waves * moe_waves(umax, S, c) * (m.ng_max * 8L + passes * 24 + 8);
      if (best_cost < 0 || cost < best_cost) { best = m; best_cost = cost; }
    }
  }
  return best_cost >= 0;
}

int moe_check_desc(const paro_moe_desc *d, MoeShapes &ms) {
  const char *why = "";
  if (!d || !d->gate_up || !d->down) { set_error("moe: null descriptor or shape"); return PARO_EINVAL; }
  if (!make_layout(*d->gate_up, ms.gu, &why)) { set_error("moe: gate_up: %s", why); return PARO_EINVAL; }
  if (!make_layout(*d->down, ms.dn, &why)) { set_error("moe: down: %s", why); return PARO_EINVAL; }
  const paro_linear_shape &gu = *d->gate_up, &dn = *d->down;
  ms.I = dn.in_features; ms.H = gu.in_features; ms.E = d->n_experts;
  if (d->n_experts < 1) { set_error("moe: n_experts must be >= 1, got %d", d->n_experts); return PARO_EINVAL; }
  if (gu.n_parts != 2 || gu.part_sizes[0] != ms.I || gu.part_sizes[1] != ms.I) {
    set_error("moe: gate_up must have two partitions {I, I} with I = down.in_features = %d", ms.I);
    return PARO_EINVAL;
  }
  if (dn.n_parts != 1 || dn.out_features != ms.H) { set_error("moe: down must have one partition of out_features = hidden = %d", ms.H); return PARO_EINVAL; }
  if (gu.dtype != dn.dtype || gu.group_size != dn.group_size || gu.krot != dn.krot) {
    set_error("moe: gate_up and down must agree on dtype, group_size and krot");
    return PARO_EINVAL;
  }
  if (d->gate_up_stride < ms.gu.total_bytes || d->down_stride < ms.dn.total_bytes || d->gate_up_stride % 256 || d->down_stride % 256) {
    set_error("moe: expert strides must be >= paro_packed_bytes of their shape and multiples of 256 (gate_up %zu, down %zu)",
              d->gate_up_stride, d->down_stride);
    return PARO_EINVAL;
  }
  return PARO_OK;
}

static int moe_check(const paro_moe_desc *d, int64_t T, int32_t k, MoeShapes &ms) {
  const int rc = moe_check_desc(d, ms);
  if (rc) return rc;
  if (T < 1 || T > 16 || k < 1 || k > 16 || T * k > kMoeMaxEntries) {
    set_error("moe: 1 <= T <= 16, 1 <= top_k <= 16 and T * top_k <= %d supported, got T = %lld, top_k = %d", kMoeMaxEntries,
              static_cast<long long>(T), k);
    return PARO_EUNSUPPORTED;
  }
  return PARO_OK;
}

static void moe_fill(MoeParams &p, const Layout &L, const MoePlan &m, const void *packed, size_t stride) {
  p.packed = static_cast<const uint8_t *>(packed);
  p.stride = static_cast<long long>(stride);
  p.L = L;
  p.c = m.c; p.S = m.S; p.nstages = m.nstages;
  p.xb_off = m.xb_off; p.rot_off = m.rot_off; p.recv_off = m.recv_off; p.tab_off = m.tab_off; p.bar_off = m.bar_off;
}

template <typename T, bool DOWN>
static int moe_launch(const MoeParams &p, const MoePlan &m, cudaStream_t stream) {
  auto kern = moe_kernel<T, DOWN>;
  PARO_CUDA_OK(smem_opt_in(kern, kMoeSmemLimit));
  cudaLaunchConfig_t cfg;
  cudaLaunchAttribute attr[2];
  launch_config(cfg, attr, m.grid, kMoeThreads, m.smem, stream, m.c, true);   // a cluster launch also at c = 1
  PARO_CUDA_OK(cudaLaunchKernelEx(&cfg, kern, p));
  return PARO_OK;
}

int moe_forward(const paro_moe_desc *d, const void *x, const int32_t *ids, const float *wts, int64_t T, int32_t k, void *h, void *y,
                void *workspace, size_t workspace_bytes, cudaStream_t stream) {
  MoeShapes ms;
  int rc = moe_check(d, T, k, ms);
  if (rc) return rc;
  if (!x || !ids || !wts || !h || !y || !workspace || !d->gate_up_packed || !d->down_packed) { set_error("moe: null pointer argument"); return PARO_EINVAL; }
  if ((reinterpret_cast<uintptr_t>(d->gate_up_packed) | reinterpret_cast<uintptr_t>(d->down_packed)) & 255 ||
      (reinterpret_cast<uintptr_t>(x) | reinterpret_cast<uintptr_t>(h) | reinterpret_cast<uintptr_t>(y)) & 15 ||
      (reinterpret_cast<uintptr_t>(ids) | reinterpret_cast<uintptr_t>(wts)) & 3) {
    set_error("moe: packed buffers must be 256-byte, x / h / y 16-byte, ids / weights 4-byte aligned");
    return PARO_EINVAL;
  }
  if (workspace_bytes < 256) { set_error("moe: workspace too small: have %zu, need 256", workspace_bytes); return PARO_EWORKSPACE; }
  const int Ti = static_cast<int>(T), umax = ms.E < Ti * k ? ms.E : Ti * k, sms = planning_sms();
  MoePlan m1, m2;
  if (!moe_choose_plan(ms.gu, Ti, umax, sms, m1) || !moe_choose_plan(ms.dn, Ti, umax, sms, m2)) {
    set_error("moe: no launch configuration fits (hidden=%d, I=%d, T=%d)", ms.H, ms.I, Ti);
    return PARO_EUNSUPPORTED;
  }
  MoeParams p1 = {}, p2 = {};
  moe_fill(p1, ms.gu, m1, d->gate_up_packed, d->gate_up_stride);
  moe_fill(p2, ms.dn, m2, d->down_packed, d->down_stride);
  p1.x = x; p1.y = h;
  p2.x = h; p2.y = y;
  for (MoeParams *p : {&p1, &p2}) {
    p->ids = ids; p->wts = wts; p->T = Ti; p->k = k; p->E = ms.E;
  }
  const bool bf = d->gate_up->dtype == PARO_BF16;
  rc = bf ? moe_launch<__nv_bfloat16, false>(p1, m1, stream) : moe_launch<__half, false>(p1, m1, stream);
  if (rc) return rc;
  rc = bf ? moe_launch<__nv_bfloat16, true>(p2, m2, stream) : moe_launch<__half, true>(p2, m2, stream);
  if (rc) return rc;
  note_launches(2);
  return PARO_OK;
}

size_t moe_workspace_bytes(const paro_moe_desc *d, int64_t T, int32_t k) {
  MoeShapes ms;
  if (moe_check(d, T, k, ms)) return 0;
  return 256;   // the routing table and the cross-CTA sums live in shared memory; the workspace is reserved
}

// Test hook: both plans and a walk of the kernels' work list.  For every U = 1..U_max and both launches, every (expert slot,
// group) round of a block must be taken by exactly one (rank, wave) and none beyond U; rank 0 must read, in every wave, only
// the receive slots of ranks that had an item in that wave.  out[0..7] gate_up plan, out[8..15] down plan (cluster size, K
// slices, grid, blocks, groups, groups per item, ring stages, shared-memory bytes), out[16] = U_max, out[17] = violations.
int moe_debug_plan(const paro_moe_desc *d, int64_t T, int32_t k, int32_t sms, int32_t *out) {
  MoeShapes ms;
  const int rc = moe_check(d, T, k, ms);
  if (rc) return rc;
  const int Ti = static_cast<int>(T), umax = ms.E < Ti * k ? ms.E : Ti * k;
  MoePlan mp[2];
  if (!moe_choose_plan(ms.gu, Ti, umax, sms, mp[0]) || !moe_choose_plan(ms.dn, Ti, umax, sms, mp[1])) {
    set_error("moe: no launch configuration fits (hidden=%d, I=%d, T=%d)", ms.H, ms.I, Ti);
    return PARO_EUNSUPPORTED;
  }
  int bad = 0;
  for (int l = 0; l < 2; ++l) {
    const MoePlan &m = mp[l];
    const int v[8] = {m.c, m.S, m.grid, m.nb, m.groups, m.ng_max, m.nstages, m.smem};
    for (int i = 0; i < 8; ++i) out[8 * l + i] = v[i];
    for (int U = 1; U <= umax; ++U) {
      int count[kMoeMaxEntries * 128] = {};   // groups <= 128 checked below
      if (m.groups > 128) { ++bad; continue; }
      const int nw = moe_waves(U, m.S, m.c);
      for (int w = 0; w < nw; ++w) {
        bool had[8] = {};
        for (int r = 0; r < m.c; ++r) {   // what every rank's producer and workers take (moe_kernel)
          const int i = w * m.c + r;
          if (i >= U * m.S) continue;
          had[r] = true;
          int u, g0, g1;
          moe_item(i, m.S, m.groups, u, g0, g1);
          if (u >= U || g1 - g0 > m.ng_max || g0 > g1) ++bad;
          for (int g = g0; g < g1; ++g) ++count[u * 128 + g];
        }
        for (int pos = 0; pos < m.c; ++pos) {   // what rank 0 reads
          if (w * m.c + pos >= U * m.S) break;
          if (!had[pos]) ++bad;
        }
      }
      for (int u = 0; u < kMoeMaxEntries; ++u)
        for (int g = 0; g < 128; ++g) bad += count[u * 128 + g] != ((u < U && g < m.groups) ? 1 : 0);
    }
  }
  out[16] = umax;
  out[17] = bad;
  return PARO_OK;
}

// Test hook: act[m, i] = silu_mul2(gate[m, i], up[m, i]) -- the down launch's operand before its rotation, from the same
// device function compiled with the same flags, so tests can rebuild it bit for bit.  One thread per element pair.
template <typename T>
__global__ void silu_mul_kernel(const uint32_t *__restrict__ gu, uint32_t *__restrict__ act, int64_t M, int I2) {
  const int64_t idx = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
  if (idx >= M * I2) return;
  const int64_t m = idx / I2;
  const int j = static_cast<int>(idx - m * I2);
  act[idx] = silu_mul2<T>(gu[m * 2 * I2 + j], gu[m * 2 * I2 + I2 + j]);
}

int moe_debug_silu_mul(int dtype, const void *gate_up, void *act, int64_t M, int I, cudaStream_t stream) {
  if (M == 0) return PARO_OK;
  const int I2 = I / 2;
  const int B = 256;
  const unsigned grid = static_cast<unsigned>((M * I2 + B - 1) / B);
  const uint32_t *gu = static_cast<const uint32_t *>(gate_up);
  uint32_t *out = static_cast<uint32_t *>(act);
  if (dtype == PARO_BF16) silu_mul_kernel<__nv_bfloat16><<<grid, B, 0, stream>>>(gu, out, M, I2);
  else silu_mul_kernel<__half><<<grid, B, 0, stream>>>(gu, out, M, I2);
  PARO_CUDA_OK(cudaGetLastError());
  note_launches(1);
  return PARO_OK;
}

}  // namespace paro
