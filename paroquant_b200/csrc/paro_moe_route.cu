// MoE router in ONE launch for any T >= 1: router logits, softmax and top-k, written straight into the buffers the expert-block
// kernels (paro_moe.cu, paro_moe_grouped.cu) read.  For x [T, H] and the router weight w [E, H] (row-major, as a checkpoint
// stores mlp.gate.weight), both of dtype D:
//
//   logit[t, e] = D(sum_h x[t, h] * w[e, h])        fp32 accumulation, one rounding to D
//   p[t, :]     = softmax(fp32(logit[t, :]))        fp32, max subtracted first
//   slots       = the top_k experts by descending logit, equal logits -> lower id first
//   weight[t,s] = p[t, id_s]   or   p[t, id_s] / sum_s' p[t, id_s'] (renormalize, summed in slot order)
//
// Operand-swapped like the other kernels: w rows are the mma.m16n8k16 A operand (E padded to 16 inside the kernel; padded rows
// never reach the softmax), a tile of NT tokens is the B operand.  Both are read from global memory with 16-byte loads: a lane
// (g, t) takes 8 consecutive columns of its row, which feed the k slots {2t, 2t+1, 2t+8, 2t+9} of two k16 steps -- the MMA sums
// over k, so any assignment of columns to slots that A and B share computes the dot product.
//
// H is cut into S K slices, S fixed by H alone (route_slices).  A slice's partial sum starts from zero and walks its columns in
// ascending order; the S partial sums of an output are added in slice order, p_0 + p_1 + ... .  One cluster of c CTAs serves a
// token tile, rank r taking slices [r S / c, (r + 1) S / c): every rank pushes its slices' partial sums into rank 0's shared
// memory (DSMEM), one cluster barrier, and rank 0 folds them.  The cluster size and the tile only decide WHO computes a partial
// sum, never its value or the order of the fold: logit[t, :], and with it the ids and weights, depend on row t of x and on w
// only -- the same bits at T = 1, inside a 16-row step and inside a 4096-token prefill chunk.
//
// Epilogue on rank 0, one warp per token row: fold, round to D, row max and sum of exp by shuffles, top_k rounds of a warp
// arg-max, renormalise, store.  No atomics, no global scratch, no workspace.
#include <vector>

#include "paro_launch.h"
#include "paro_tc_common.cuh"

namespace paro {

constexpr int kRouteWarpsPerCta = 8, kRouteCtaThreads = 32 * kRouteWarpsPerCta;
constexpr int kRouteMaxExperts = 256, kRouteMaxTopK = 16;
constexpr int kRouteSmemLimit = 227 * 1024;

// K slices of H: 8 where a slice is a whole number of the 32-column steps the kernel walks, else 4 (H is a multiple of 128)
PARO_HD inline int route_slices(int H) { return H % 256 == 0 ? 8 : 4; }
// the slices of rank r of a cluster of c CTAs (c divides S): [s0, s1)
PARO_HD inline void route_rank_slices(int r, int c, int S, int &s0, int &s1) {
  s0 = r * (S / c);
  s1 = s0 + S / c;
}
// row stride (floats) of a token's partial sums in the receive buffer: + 4 keeps the fragment stores off each other's banks
PARO_HD inline int route_recv_stride(int E16) { return E16 + 4; }

struct RouteParams {
  const void *x, *w;
  int32_t *ids;
  float *wts, *logits;
  long long T;
  int H, E, E16, k, renorm;
  int c, S;
};

// (v, e) beats (bv, be): larger logit, equal logits -> lower id
__device__ __forceinline__ bool route_better(float v, int e, float bv, int be) { return v > bv || (v == bv && e < be); }

template <typename T, int NB>   // NB n8 token tiles per CTA (NT = 8 NB)
__global__ void __launch_bounds__(kRouteCtaThreads, NB == 4 ? 1 : 2) moe_router_kernel(const RouteParams p) {
  extern __shared__ __align__(16) float recv[];   // [S][NT][E16 + 4]: partial sums, used on rank 0
  constexpr int NT = 8 * NB;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, t4 = lane & 3;
  const int c = p.c, S = p.S, H = p.H, E = p.E, E16 = p.E16, EP = route_recv_stride(E16);
  const long long tile = blockIdx.x / c;
  const int rank = blockIdx.x - static_cast<int>(tile) * c;   // == %cluster_ctarank
  cluster_arrive_relaxed();   // "this CTA runs": waited on before the first DSMEM store
  pdl_launch_dependents();    // the expert-block kernels wait for this grid's completion before they read the routing

  // warps over (16-expert tile, 8-token tile): up to 2 x NB per warp
  const int MT = E16 / 16;
  const int WM = MT >= 5 ? 8 : MT >= 3 ? 4 : MT, WN = kRouteWarpsPerCta / WM;
  const int wm = warp % WM, wn = warp / WM;
  const T *xw = static_cast<const T *>(p.x), *ww = static_cast<const T *>(p.w);
  const T *a_row[2][2];
  const T *b_row[NB];
  bool m_on[2], n_on[NB];
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    const int mt = wm + i * WM;
    m_on[i] = mt < MT;
#pragma unroll
    for (int hh = 0; hh < 2; ++hh) {
      const int e = mt * 16 + g + 8 * hh;
      a_row[i][hh] = ww + static_cast<long long>(e < E ? e : E - 1) * H + 8 * t4;   // padded rows: any row, never read back
    }
  }
#pragma unroll
  for (int j = 0; j < NB; ++j) {
    const int nb = wn + j * WN;
    n_on[j] = nb < NB;
    const long long tok = tile * NT + nb * 8 + g;
    b_row[j] = xw + (tok < p.T ? tok : p.T - 1) * H + 8 * t4;
  }
  const bool busy = m_on[0] && n_on[0];

  int s0, s1;
  route_rank_slices(rank, c, S, s0, s1);
  const int slice = H / S;
  const uint32_t recv0 = map_to_rank(smem_u32(recv), 0);
  bool waited = false;
#pragma unroll 1
  for (int s = s0; s < s1; ++s) {
    float acc[2][NB][4];
#pragma unroll
    for (int i = 0; i < 2; ++i)
#pragma unroll
      for (int j = 0; j < NB; ++j)
#pragma unroll
        for (int q = 0; q < 4; ++q) acc[i][j][q] = 0.f;
    if (busy) {
#pragma unroll 2
      for (int k = s * slice; k < (s + 1) * slice; k += 32) {
        uint4 a[2][2], b[NB];
#pragma unroll
        for (int i = 0; i < 2; ++i)
          if (m_on[i]) {
            a[i][0] = __ldg(reinterpret_cast<const uint4 *>(a_row[i][0] + k));
            a[i][1] = __ldg(reinterpret_cast<const uint4 *>(a_row[i][1] + k));
          }
#pragma unroll
        for (int j = 0; j < NB; ++j)
          if (n_on[j]) b[j] = __ldg(reinterpret_cast<const uint4 *>(b_row[j] + k));
#pragma unroll
        for (int i = 0; i < 2; ++i)
          if (m_on[i]) {
            const uint32_t f0[4] = {a[i][0].x, a[i][1].x, a[i][0].y, a[i][1].y};
            const uint32_t f1[4] = {a[i][0].z, a[i][1].z, a[i][0].w, a[i][1].w};
#pragma unroll
            for (int j = 0; j < NB; ++j)
              if (n_on[j]) {
                mma16816<T>(acc[i][j], f0, b[j].x, b[j].y);
                mma16816<T>(acc[i][j], f1, b[j].z, b[j].w);
              }
          }
      }
    }
    if (!waited) {   // every CTA of the cluster runs: rank 0's shared memory may be written
      cluster_wait_acquire();
      waited = true;
    }
    if (busy) {
#pragma unroll
      for (int i = 0; i < 2; ++i)
        if (m_on[i])
#pragma unroll
          for (int j = 0; j < NB; ++j)
            if (n_on[j]) {
              const int e = (wm + i * WM) * 16 + g, n = (wn + j * WN) * 8 + 2 * t4;
              const uint32_t at = recv0 + 4u * static_cast<uint32_t>((s * NT + n) * EP + e);
              st_cluster_f32(at, acc[i][j][0]);
              st_cluster_f32(at + 4u * EP, acc[i][j][1]);
              st_cluster_f32(at + 32u, acc[i][j][2]);
              st_cluster_f32(at + 4u * EP + 32u, acc[i][j][3]);
            }
    }
  }
  cluster_arrive_release();
  cluster_wait_acquire();
  if (rank != 0) return;

  // ---- rank 0: one warp per token row; lane l holds experts l, l + 32, ...
  constexpr int PER = kRouteMaxExperts / 32;
#pragma unroll 1
  for (int n = warp; n < NT; n += kRouteWarpsPerCta) {
    const long long tok = tile * NT + n;
    if (tok >= p.T) break;
    float v[PER];
    float vmax = -INFINITY;
#pragma unroll
    for (int j = 0; j < PER; ++j) {
      const int e = lane + 32 * j;
      v[j] = -INFINITY;
      if (e < E) {
        float sum = recv[n * EP + e];
        for (int s = 1; s < S; ++s) sum = __fadd_rn(sum, recv[(s * NT + n) * EP + e]);
        const float l = Traits<T>::to_float(Traits<T>::from_float(sum));
        if (p.logits) p.logits[tok * E + e] = l;
        v[j] = l == l ? l : -INFINITY;   // a NaN logit ranks last
        vmax = fmaxf(vmax, v[j]);
      }
    }
#pragma unroll
    for (int d = 16; d; d >>= 1) vmax = fmaxf(vmax, __shfl_xor_sync(0xFFFFFFFFu, vmax, d));
    if (vmax == -INFINITY) vmax = 0.f;   // every logit -inf or NaN: exp(v - vmax) stays defined
    float den = 0.f;
#pragma unroll
    for (int j = 0; j < PER; ++j)
      if (lane + 32 * j < E) den += __expf(v[j] - vmax);
#pragma unroll
    for (int d = 16; d; d >>= 1) den += __shfl_xor_sync(0xFFFFFFFFu, den, d);
    const float inv = 1.f / den;

    uint32_t taken = 0u;
    int my_id = 0;
    float my_p = 0.f, psum = 0.f;
#pragma unroll 1
    for (int slot = 0; slot < p.k; ++slot) {
      float bv = -INFINITY;
      int be = 0x7FFFFFFF;
#pragma unroll
      for (int j = 0; j < PER; ++j) {
        const int e = lane + 32 * j;
        if (e < E && !(taken >> j & 1u) && route_better(v[j], e, bv, be)) { bv = v[j]; be = e; }
      }
#pragma unroll
      for (int d = 16; d; d >>= 1) {
        const float ov = __shfl_xor_sync(0xFFFFFFFFu, bv, d);
        const int oe = __shfl_xor_sync(0xFFFFFFFFu, be, d);
        if (route_better(ov, oe, bv, be)) { bv = ov; be = oe; }
      }
      if ((be & 31) == lane) taken |= 1u << (be >> 5);
      const float pr = __expf(bv - vmax) * inv;
      psum += pr;   // slot order, the same on every lane
      if (lane == slot) { my_id = be; my_p = pr; }
    }
    if (lane < p.k) {
      p.ids[tok * p.k + lane] = my_id;
      p.wts[tok * p.k + lane] = p.renorm ? my_p / psum : my_p;
    }
  }
}

// ------------------------------------------------------------------ host side
struct RoutePlan {
  int nt, c, S, e16, smem;
  long long tiles, grid;
};

static size_t route_smem(int S, int nt, int e16) { return static_cast<size_t>(S) * nt * route_recv_stride(e16) * 4; }

static int route_check(int64_t T, int hidden, int E, int k) {
  if (T < 0) { set_error("moe_route: negative token count"); return PARO_EINVAL; }
  if (hidden < 128 || hidden % 128) { set_error("moe_route: hidden must be a positive multiple of 128, got %d", hidden); return PARO_EUNSUPPORTED; }
  if (E < 1 || E > kRouteMaxExperts) { set_error("moe_route: 1 <= n_experts <= %d supported, got %d", kRouteMaxExperts, E); return PARO_EUNSUPPORTED; }
  if (k < 1 || k > kRouteMaxTopK || k > E) {
    set_error("moe_route: 1 <= top_k <= min(n_experts, %d) supported, got top_k = %d with %d experts", kRouteMaxTopK, k, E);
    return PARO_EUNSUPPORTED;
  }
  if (T > 0x7FFFFFFFLL) { set_error("moe_route: T <= %d supported, got %lld", 0x7FFFFFFF, static_cast<long long>(T)); return PARO_EUNSUPPORTED; }
  return PARO_OK;
}

// The plan from (T, H, E, SM count) alone.  Few tokens: 8-token tiles and the widest cluster, so that as many SMs as possible pull
// the weight; once those no longer fit one wave: the largest tile whose receive buffer fits shared memory (the weight is read
// once per tile) and the widest cluster that keeps the grid within one wave, down to c = 1.
static void route_plan(int64_t T, int H, int E, int sms, RoutePlan &r) {
  r.S = route_slices(H);
  r.e16 = (E + 15) / 16 * 16;
  const long long tiles8 = (T + 7) / 8;
  if (tiles8 * r.S <= sms) r.nt = 8;
  else r.nt = route_smem(r.S, 32, r.e16) <= static_cast<size_t>(kRouteSmemLimit) ? 32 : 16;
  r.tiles = (T + r.nt - 1) / r.nt;
  r.c = r.S;
  while (r.c > 1 && r.tiles * r.c > sms) r.c /= 2;
  r.grid = r.tiles * r.c;
  r.smem = static_cast<int>(route_smem(r.S, r.nt, r.e16));
}

template <typename T, int NB>
static int route_launch(const RouteParams &p, const RoutePlan &r, cudaStream_t stream) {
  auto kern = moe_router_kernel<T, NB>;
  PARO_CUDA_OK(smem_opt_in(kern, kRouteSmemLimit));
  cudaLaunchConfig_t cfg;
  cudaLaunchAttribute attr[2];
  launch_config(cfg, attr, static_cast<int>(r.grid), kRouteCtaThreads, r.smem, stream, r.c, false);   // a cluster launch also at c = 1
  PARO_CUDA_OK(cudaLaunchKernelEx(&cfg, kern, p));
  return PARO_OK;
}

int moe_route_forward(const void *x, const void *w, int dtype, int64_t T, int hidden, int E, int k, int renormalize, int32_t *ids, float *wts,
                      float *logits, cudaStream_t stream) {
  if (dtype != PARO_F16 && dtype != PARO_BF16) { set_error("moe_route: dtype must be F16 or BF16, got code %d", dtype); return PARO_EINVAL; }
  if (renormalize != 0 && renormalize != 1) { set_error("moe_route: renormalize must be 0 or 1, got %d", renormalize); return PARO_EINVAL; }
  const int rc = route_check(T, hidden, E, k);
  if (rc) return rc;
  if (T == 0) return PARO_OK;
  if (!x || !w || !ids || !wts) { set_error("moe_route: null pointer argument"); return PARO_EINVAL; }
  if ((reinterpret_cast<uintptr_t>(x) | reinterpret_cast<uintptr_t>(w)) & 15 ||
      (reinterpret_cast<uintptr_t>(ids) | reinterpret_cast<uintptr_t>(wts) | reinterpret_cast<uintptr_t>(logits)) & 3) {
    set_error("moe_route: x / router_w must be 16-byte, ids / weights / logits 4-byte aligned");
    return PARO_EINVAL;
  }
  RoutePlan r;
  route_plan(T, hidden, E, planning_sms(), r);
  RouteParams p = {};
  p.x = x; p.w = w; p.ids = ids; p.wts = wts; p.logits = logits;
  p.T = T; p.H = hidden; p.E = E; p.E16 = r.e16; p.k = k; p.renorm = renormalize; p.c = r.c; p.S = r.S;
  const bool bf = dtype == PARO_BF16;
  int lrc;
  if (r.nt == 8) lrc = bf ? route_launch<__nv_bfloat16, 1>(p, r, stream) : route_launch<__half, 1>(p, r, stream);
  else if (r.nt == 16) lrc = bf ? route_launch<__nv_bfloat16, 2>(p, r, stream) : route_launch<__half, 2>(p, r, stream);
  else lrc = bf ? route_launch<__nv_bfloat16, 4>(p, r, stream) : route_launch<__half, 4>(p, r, stream);
  if (lrc) return lrc;
  note_launches(1);
  return PARO_OK;
}

// Test hook: the plan and a walk of it as the kernel reads it -- CTA b is rank b % c of tile b / c and takes
// route_rank_slices; every (token tile, K slice) must be owned exactly once.
int moe_route_debug_plan(int64_t T, int hidden, int E, int k, int sms, int32_t *out) {
  const int rc = route_check(T, hidden, E, k);
  if (rc) return rc;
  if (T < 1) { set_error("moe_route: the plan of an empty batch does not exist (T = 0 launches nothing)"); return PARO_EINVAL; }
  RoutePlan r;
  route_plan(T, hidden, E, sms, r);
  std::vector<uint8_t> owned(static_cast<size_t>(r.tiles) * r.S, 0);
  int bad = 0;
  for (long long b = 0; b < r.grid; ++b) {
    const long long tile = b / r.c;
    int s0, s1;
    route_rank_slices(static_cast<int>(b - tile * r.c), r.c, r.S, s0, s1);
    for (int s = s0; s < s1; ++s) {
      if (tile >= r.tiles || s >= r.S) { ++bad; continue; }
      if (owned[tile * r.S + s]++) ++bad;
    }
  }
  for (uint8_t o : owned) bad += o == 0;
  if (r.tiles * r.nt < T || hidden % (r.S * 32)) ++bad;   // tokens past the last tile; a slice that is not whole 32-column steps
  out[0] = r.nt; out[1] = r.c; out[2] = r.S; out[3] = static_cast<int32_t>(r.grid); out[4] = r.smem; out[5] = bad;
  out[6] = static_cast<int32_t>(r.tiles); out[7] = kRouteCtaThreads;
  return PARO_OK;
}

}  // namespace paro
