// Scaled pairwise (Givens) rotation for sm_90a: ONE tile kernel, rotate_tile_kernel, serves the torch.ops.rotation.rotate
// surface (/root/reference/paroquant/kernels/cuda/rotation.cu:10-43,62-135) and the activation pre-pass of the tensor-core
// kernels (paro_decode.cu from 5 rows, paro_gemm.cu, paro_moe_grouped.cu).
//
// Arithmetic is the reference's, rounding point for rounding point (rotation.cuh:91-173 for
// fp16/bf16, :16-75 for fp32): v = T(x * T(scale)); per rotation r and pair (i, j):
// (s, c) = __sincosf(float(T(theta))), vi' = T(fma(c, vi, s*vj)), vj' = T(fma(c, vj, s*-vi)).
//
// Mapping (not the reference's): one WARP owns one (block of RB rows, group) tile, so the
// krot rotations need only __syncwarp().  The tile lives in shared memory channel-major --
// rot[channel][RB rows] = one 16-byte vector per channel -- so a pair update is two 128-bit
// loads and two 128-bit stores for all RB rows at once.  The 16-byte slot of channel c is
// c ^ ((c >> 3) & 7), which makes the coalesced transpose-in / transpose-out conflict free.
#include "paro_common.cuh"
#include "paro_launch.h"
#include "paro_tc_common.cuh"   // silu_mul2: the MoE down pre-pass

namespace paro {

__device__ __forceinline__ int rot_slot(int c) { return c ^ ((c >> 3) & 7); }

// ---- half / bf16: a channel vector is 4 x T2 words, word u = rows (2u, 2u+1)
template <typename T>
__device__ __forceinline__ void pair_update(uint4 &vi, uint4 &vj, float c, float s) {
  uint32_t *pi = reinterpret_cast<uint32_t *>(&vi), *pj = reinterpret_cast<uint32_t *>(&vj);
#pragma unroll
  for (int u = 0; u < 4; ++u) {
    const float2 a = Traits<T>::to_float2(unpack2<T>(pi[u]));
    const float2 b = Traits<T>::to_float2(unpack2<T>(pj[u]));
    float yix, yiy, yjx, yjy;
    givens(c, s, a.x, b.x, yix, yjx);
    givens(c, s, a.y, b.y, yiy, yjy);
    pi[u] = pack2<T>(Traits<T>::from_floats(yix, yiy));
    pj[u] = pack2<T>(Traits<T>::from_floats(yjx, yjy));
  }
}
template <>
__device__ __forceinline__ void pair_update<float>(uint4 &vi, uint4 &vj, float c, float s) {
  float *pi = reinterpret_cast<float *>(&vi), *pj = reinterpret_cast<float *>(&vj);
#pragma unroll
  for (int u = 0; u < 4; ++u) {
    float yi, yj;
    givens(c, s, pi[u], pj[u], yi, yj);
    pi[u] = yi;
    pj[u] = yj;
  }
}

// x * scale: one rounding to T (rotation.cuh:112-113), fp32 as is (:24-32)
template <typename T> __device__ __forceinline__ T scale_mul(T x, T s) { return __hmul(x, s); }
template <> __device__ __forceinline__ float scale_mul<float>(float x, float s) { return x * s; }

// A lane's share of one row of a group: its CPL = G / 32 channels of T in one word
template <int Bytes> struct Bits;
template <> struct Bits<4> { using type = uint32_t; };
template <> struct Bits<8> { using type = uint2; };
template <> struct Bits<16> { using type = uint4; };
template <typename T, int G> using Chunk = typename Bits<G / 32 * static_cast<int>(sizeof(T))>::type;

// ------------------------------------------------------------------ row sources
// A row source says what feeds output row m: `skip(row0)` -- the block of RB rows from row0 on is never read, leave it;
// `padding_block(row0)` -- all RB rows are padding, store zeros; `valid(m)` -- row m has an input (else it is a zero row);
// `load(m, k)` -- the lane's channels k .. k + CPL - 1 of row m's input, before the channel scale; `finish(row0, k, lane, xr)`
// -- called once per block of rows by the whole warp with the loaded channels of rows row0 .. row0 + RB - 1, before the
// channel scale (a no-op except for RMSNorm, whose rows need the block's statistics).  Each source takes rows as its own
// index type `Row`: int for the pre-pass (at most 2^31 rows), int64 for the op.

// the rotate op's x [M, K], row-major and 16-byte aligned (paro_rotate checks it); rows >= M are neither read nor stored, and
// the grid ends at the block of row M - 1
template <typename T, int G>
struct OpRows {
  using Row = int64_t;
  const T *x;
  int64_t M;
  int K;
  __device__ bool skip(int64_t) const { return false; }
  __device__ bool padding_block(int64_t) const { return false; }
  __device__ bool valid(int64_t m) const { return m < M; }
  __device__ Chunk<T, G> load(int64_t m, int k) const { return *reinterpret_cast<const Chunk<T, G> *>(x + m * K + k); }
  __device__ void finish(int64_t, int, int, Chunk<T, G> (&)[16 / sizeof(T)]) const {}
};

// SiLU * up of the [gate | up] row whose gate channel k .. k + 3 `row` points at, K channels per half -- silu_mul2, the MoE
// decode kernel's and the decode chain's
template <typename T>
__device__ __forceinline__ uint2 silu_mul_load(const T *row, int K) {
  const uint2 gate = __ldcg(reinterpret_cast<const uint2 *>(row)), up = __ldcg(reinterpret_cast<const uint2 *>(row + K));
  return make_uint2(silu_mul2<T>(gate.x, up.x), silu_mul2<T>(gate.y, up.y));
}

// The pre-pass sources below feed 16-bit T in groups of 128: 8 rows per block, 4 channels (one uint2) per lane.
// a linear's activations x [M, K]; rows >= M are padding
template <typename T>
struct DenseRows {
  using Row = int;
  const T *x;
  int M, K;
  __device__ bool skip(int) const { return false; }
  __device__ bool padding_block(int row0) const { return row0 >= M; }
  __device__ bool valid(int m) const { return m < M; }
  __device__ uint2 load(int m, int k) const { return *reinterpret_cast<const uint2 *>(x + static_cast<int64_t>(m) * K + k); }
  __device__ void finish(int, int, int, uint2 (&)[8]) const {}
};
// a chain step's SILU_MUL x op: x [M, 2K] (gate | up)
template <typename T>
struct DenseSiluMulRows : DenseRows<T> {
  __device__ uint2 load(int m, int k) const { return silu_mul_load<T>(this->x + static_cast<int64_t>(m) * (2 * this->K) + k, this->K); }
};
// a chain step's RMSNORM x op: h = x [M, K], norm weights w [K]; stats[b * M + m] = the producing GEMM's sum of h^2 over the
// columns of its 128-column block b (paro_gemm.cu, ResidualTiles).  rstd of a row adds the nb partials in block order, whatever
// the tiles, the batch or the row's neighbours, then T(T(h * rstd) * w) as the decode chain's norm2.
template <typename T>
struct RmsNormRows : DenseRows<T> {
  const T *w;
  const float *stats;
  int nb;
  float eps;
  __device__ void finish(int row0, int k, int lane, uint2 (&xr)[8]) const {
    const int m = row0 + (lane & 7);
    float s = 0.f;
    if (lane < 8 && m < this->M)
      for (int b = 0; b < nb; ++b) s += __ldcg(stats + static_cast<int64_t>(b) * this->M + m);
    const float rstd = rsqrtf(s / static_cast<float>(this->K) + eps);   // lane r: row row0 + r
    const uint2 w2 = *reinterpret_cast<const uint2 *>(w + k);
#pragma unroll
    for (int r = 0; r < 8; ++r) {
      const float rs = __shfl_sync(0xFFFFFFFFu, rstd, r);
      xr[r].x = norm2<T>(xr[r].x, rs, w2.x);
      xr[r].y = norm2<T>(xr[r].y, rs, w2.y);
    }
  }
};

// The MoE grouped pre-passes (paro_moe_grouped.cu): output row m is routing entry rows[m] = token * top_k + slot, -1 for padding.
// Padding runs from an expert's last entry to the end of its tile, so a block of 8 rows starting on padding is all padding.
// Rows from live_tiles * nt on belong to no tile the GEMM runs.
struct RoutedRows {
  using Row = int;
  const int32_t *rows, *live_tiles;
  int nt;
  __device__ bool skip(int row0) const { return row0 >= *live_tiles * nt; }
  __device__ bool padding_block(int row0) const { return rows[row0] < 0; }
  __device__ bool valid(int m) const { return rows[m] >= 0; }
  __device__ void finish(int, int, int, uint2 (&)[8]) const {}
};
// gate_up: x [T, K], entry e reads token e / top_k
template <typename T>
struct GatherRows : RoutedRows {
  const T *x;
  int top_k, K;
  __device__ uint2 load(int m, int k) const { return *reinterpret_cast<const uint2 *>(x + static_cast<int64_t>(rows[m] / top_k) * K + k); }
};
// down: T(T(silu(gate)) * up) of h [T * top_k, 2K] (gate | up), entry e reads row e
template <typename T>
struct SiluMulRows : RoutedRows {
  const T *h;
  int K;
  __device__ uint2 load(int m, int k) const { return silu_mul_load<T>(h + static_cast<int64_t>(rows[m]) * (2 * K) + k, K); }
};

// ------------------------------------------------------------------ metadata sources
// `at(b)` -- the source narrowed to block b = partition * groups + group; `scales(lane, s)` -- the lane's CPL channel scales as
// T; `stage(r, lane)` -- what the lane needs of rotation r, as loaded; `pair(st, q, i, j, theta)` -- the lane's pair q of that
// rotation, theta as float(T(theta)); `kAhead` -- how many rotations' stages the kernel fetches at a time.  Lane l owns pairs
// l * PPL .. l * PPL + PPL - 1 of every rotation.

// The packed layout's per-group blocks (paro_layout.h), read with the loads fetch_meta makes in the fused kernels (G = 128).
// 8 rotations at a time: a pre-pass launch costs one load round trip, not one per rotation.
template <typename T>
struct PackedMeta {
  const uint8_t *blk;
  int group_bytes, krot;
  struct Stage { uint32_t iw, th; };   // bytes (i0, j0, i1, j1) of pairs 2 lane, 2 lane + 1, and their two angles
  static constexpr int kAhead = 8;
  __device__ PackedMeta at(int b) const { return {blk + static_cast<long long>(b) * group_bytes, group_bytes, krot}; }
  __device__ bool scaled() const { return true; }
  __device__ void scales(int lane, T (&s)[4]) const {
    const uint2 w = *reinterpret_cast<const uint2 *>(blk + meta_scales_off(krot) + 8 * lane);
    const T *p = reinterpret_cast<const T *>(&w);
#pragma unroll
    for (int c = 0; c < 4; ++c) s[c] = p[c];
  }
  __device__ Stage stage(int r, int lane) const {
    return {*reinterpret_cast<const uint32_t *>(blk + meta_pairs_off(r) + 4 * lane),
            *reinterpret_cast<const uint32_t *>(blk + meta_theta_off(krot, r) + 4 * lane)};
  }
  __device__ void pair(const Stage &st, int q, int &i, int &j, float &theta) const {
    const float2 t2 = Traits<T>::to_float2(unpack2<T>(st.th));
    theta = q ? t2.y : t2.x;
    i = (st.iw >> (16 * q)) & 0xFF;
    j = (st.iw >> (16 * q + 8)) & 0xFF;
  }
};

// The reference's tensors, as the op takes them: idx_ij [krot, K] int16 (pair t of a group at 2t, 2t + 1, 4-byte aligned),
// theta [krot, K / 2] and scales [K] (optional) in any float dtype, read element by element and cast to T (rotation.cu:75-78).
// The op has one partition, so block b is group b.  One rotation at a time: 8 at a time took the op from 40-53 registers to
// 72-116 and, measured on an H100 SXM (700 W), made it slower at 4096 x 4096 bf16 (69 vs 62 us) and at 1 and 16 rows (5.4
// and 5.8 vs 5.2 and 5.5 us per launch in a CUDA graph).
template <typename T, int G>
struct RefMeta {
  const int16_t *idx;
  const void *theta, *sc;
  int theta_dtype, sc_dtype, K, krot, g;
  static constexpr int CPL = G / 32, PPL = G / 64;
  struct Stage { int ij[PPL]; float th[PPL]; };
  static constexpr int kAhead = 1;
  __device__ RefMeta at(int b) const { RefMeta m = *this; m.g = b; return m; }
  __device__ bool scaled() const { return sc != nullptr; }
  __device__ void scales(int lane, T (&s)[CPL]) const {
#pragma unroll
    for (int c = 0; c < CPL; ++c)
      s[c] = sc ? Traits<T>::from_float(load_param_as<T>(sc, static_cast<int64_t>(g) * G + lane * CPL + c, sc_dtype)) : T{};
  }
  __device__ Stage stage(int r, int lane) const {
    Stage st;
#pragma unroll
    for (int q = 0; q < PPL; ++q) {
      const int t = lane * PPL + q;
      st.ij[q] = *reinterpret_cast<const int *>(idx + static_cast<int64_t>(r) * K + g * G + 2 * t);
      st.th[q] = load_param_as<T>(theta, static_cast<int64_t>(r) * (K / 2) + g * (G / 2) + t, theta_dtype);
    }
    return st;
  }
  __device__ void pair(const Stage &st, int q, int &i, int &j, float &theta) const {
    theta = st.th[q];
    i = st.ij[q] & 0xFFFF;
    j = (st.ij[q] >> 16) & 0xFFFF;
  }
};

// ------------------------------------------------------------------ outputs
// `partition(p)` -- the output narrowed to partition p; `put(m, k, ok, w)` -- the lane's channels k .. of output row m, w (zero
// when !ok, the row had no input)

// the op: y [M, K], row-major; rows without input are not stored
template <typename T>
struct RowMajorOut {
  T *y;
  int K;
  __device__ RowMajorOut partition(int) const { return *this; }
  template <typename W>
  __device__ void put(int64_t m, int k, bool ok, W w) const {
    if (ok) *reinterpret_cast<W *>(y + m * K + k) = w;
  }
};

// the pre-pass: the B operand of the tensor-core kernels, [token block of nt][k16 step][k half][row / 8][row % 8][8 elements],
// partition p at y + p * part_elems; rows without input are zero rows
template <typename T>
struct TiledOut {
  T *y;
  long long part_elems;
  int nt, K;
  __device__ TiledOut partition(int p) const { return {y + p * part_elems, part_elems, nt, K}; }
  __device__ void put(int m, int k, bool, uint2 w) const {
    const int tb = m / nt, n = m - tb * nt;
    const int64_t e = (static_cast<int64_t>(tb) * (K / 16) + (k >> 4)) * (static_cast<int64_t>(nt) * 16) + ((k >> 3) & 1) * (nt * 8) + (n >> 3) * 64 +
                      (n & 7) * 8 + (k & 7);
    *reinterpret_cast<uint2 *>(y + e) = w;
  }
};

// ------------------------------------------------------------------ the tile kernel
// One warp per (partition, block of RB = 16 / sizeof(T) rows, group of G channels), the group minor.  The warp issues its rows,
// its scales and the first Meta::kAhead rotations' stages together.  The rows are scaled and transposed in before the rotation
// loop, so that they are not live across its iterations.  Its global loads are plain ld.global, not the read-only path: with
// __ldg on every read-only input, measured on an H100 SXM (700 W), the op took 64-66 us instead of 61-62 us at 4096 x 4096
// bf16 and 5.5-5.7 us instead of 5.2-5.3 us per launch at 1 row, and the decode pre-pass gave up its 1-4 % over the parent's.
template <typename T, int G, typename Rows, typename Meta, typename Out>
__global__ void __launch_bounds__(128) rotate_tile_kernel(const Rows src, const Meta meta_all, const Out out_all, long long row_blocks, int K,
                                                          int n_parts) {
  constexpr int RB = 16 / sizeof(T), CPL = G / 32, PPL = G / 64;
  using W = Chunk<T, G>;
  __shared__ __align__(16) uint4 tile[4][G];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int groups = K / G;
  const long long task = static_cast<long long>(blockIdx.x) * 4 + warp;
  if (task >= n_parts * row_blocks * groups) return;
  const int g = static_cast<int>(task % groups), part = static_cast<int>(task / (row_blocks * groups));
  const typename Rows::Row row0 = static_cast<typename Rows::Row>((task / groups) % row_blocks) * RB;
  const Meta meta = meta_all.at(part * groups + g);
  const Out out = out_all.partition(part);
  const int krot = meta.krot, k = g * G + lane * CPL;
  uint4 *rot = tile[warp];
  if (src.skip(row0)) return;
  if (src.padding_block(row0)) {   // a block of padding rows: zeros, in place
#pragma unroll
    for (int r = 0; r < RB; ++r) out.put(row0 + r, k, false, W{});
    return;
  }
  W xr[RB];
  bool ok[RB];
#pragma unroll
  for (int r = 0; r < RB; ++r) {
    ok[r] = src.valid(row0 + r);
    xr[r] = ok[r] ? src.load(row0 + r, k) : W{};
  }
  T sc[CPL];
  meta.scales(lane, sc);
  typename Meta::Stage st[Meta::kAhead];   // rotations r0 .. r0 + kAhead - 1
  auto fetch = [&](int r0) {
#pragma unroll
    for (int r = 0; r < Meta::kAhead; ++r)
      if (r0 + r < krot) st[r] = meta.stage(r0 + r, lane);
  };
  fetch(0);
  src.finish(row0, k, lane, xr);
  // ---- scale, transpose into rot[channel]
  {
    T v[RB][CPL];
#pragma unroll
    for (int r = 0; r < RB; ++r) {
      const T *pr = reinterpret_cast<const T *>(&xr[r]);
#pragma unroll
      for (int c = 0; c < CPL; ++c) v[r][c] = meta.scaled() ? scale_mul<T>(pr[c], sc[c]) : pr[c];
    }
#pragma unroll
    for (int c = 0; c < CPL; ++c) {
      uint4 w;
      T *pw = reinterpret_cast<T *>(&w);
#pragma unroll
      for (int r = 0; r < RB; ++r) pw[r] = v[r][c];
      rot[rot_slot(lane * CPL + c)] = w;
    }
  }
  __syncwarp();
  // ---- krot rotations, kAhead fetched at a time
  for (int r0 = 0; r0 < krot; r0 += Meta::kAhead) {
    if (r0 > 0) fetch(r0);
#pragma unroll
    for (int r = 0; r < Meta::kAhead; ++r) {
      if (r0 + r < krot) {
#pragma unroll
        for (int q = 0; q < PPL; ++q) {
          int pi, pj;
          float th, sn, cs;
          meta.pair(st[r], q, pi, pj, th);
          __sincosf(th, &sn, &cs);
          uint4 vi = rot[rot_slot(pi)], vj = rot[rot_slot(pj)];
          pair_update<T>(vi, vj, cs, sn);
          rot[rot_slot(pi)] = vi;
          rot[rot_slot(pj)] = vj;
        }
        __syncwarp();
      }
    }
  }
  // ---- transpose out
  T v[RB][CPL];
#pragma unroll
  for (int c = 0; c < CPL; ++c) {
    const uint4 w = rot[rot_slot(lane * CPL + c)];
    const T *pw = reinterpret_cast<const T *>(&w);
#pragma unroll
    for (int r = 0; r < RB; ++r) v[r][c] = pw[r];
  }
#pragma unroll
  for (int r = 0; r < RB; ++r) {
    W w{};
    if (ok[r]) {
      T *pw = reinterpret_cast<T *>(&w);
#pragma unroll
      for (int c = 0; c < CPL; ++c) pw[c] = v[r][c];
    }
    out.put(row0 + r, k, ok[r], w);
  }
}

// n_parts partitions of row_blocks blocks of rows each, all in one launch
template <typename T, int G, typename Rows, typename Meta, typename Out>
static int launch_rotation(const Rows &src, const Meta &meta, const Out &out, long long row_blocks, int K, int n_parts, cudaStream_t stream) {
  const long long blocks = (n_parts * row_blocks * (K / G) + 3) / 4;
  if (blocks > 0x7FFFFFFF) { set_error("rotate: too many rows"); return PARO_EINVAL; }
  rotate_tile_kernel<T, G><<<static_cast<unsigned>(blocks), 128, 0, stream>>>(src, meta, out, row_blocks, K, n_parts);
  PARO_CUDA_OK(cudaGetLastError());
  note_launches(1);
  return PARO_OK;
}

// ------------------------------------------------------------------ pre-pass of the tensor-core kernels
// n_parts partitions of L, rows of `src` -> out: per partition M_store rows (a multiple of 8; rows without input zero) in tiles
// of `nt` tokens
template <typename T, typename Rows>
static int rotate_tiles(const Layout &L, const void *packed, int n_parts, const Rows &src, void *out, int64_t M_store, int nt, cudaStream_t stream) {
  const PackedMeta<T> meta = {static_cast<const uint8_t *>(packed) + L.meta_off, L.meta_group_bytes, L.krot};
  const TiledOut<T> o = {static_cast<T *>(out), static_cast<long long>(M_store) * L.K, nt, L.K};
  return launch_rotation<T, 128>(src, meta, o, M_store / 8, L.K, n_parts, stream);
}

template <typename T>
static int rotate_chain_T(const Layout &L, const void *packed, int x_op, const void *x, const void *norm_w, const float *stats, int stats_blocks,
                          float eps, void *out, int64_t M, int64_t M_store, int nt, cudaStream_t stream) {
  const DenseRows<T> dense = {static_cast<const T *>(x), static_cast<int>(M), L.K};
  if (x_op == PARO_XOP_SILU_MUL) {
    DenseSiluMulRows<T> r;
    static_cast<DenseRows<T> &>(r) = dense;
    return rotate_tiles<T>(L, packed, L.n_parts, r, out, M_store, nt, stream);
  }
  if (x_op == PARO_XOP_RMSNORM) {
    RmsNormRows<T> r;
    static_cast<DenseRows<T> &>(r) = dense;
    r.w = static_cast<const T *>(norm_w); r.stats = stats; r.nb = stats_blocks; r.eps = eps;
    return rotate_tiles<T>(L, packed, L.n_parts, r, out, M_store, nt, stream);
  }
  return rotate_tiles<T>(L, packed, L.n_parts, dense, out, M_store, nt, stream);
}

int rotate_chain_launch(const Layout &L, const void *packed, int x_op, const void *x, const void *norm_w, const float *stats, int stats_blocks,
                        float eps, void *out, int64_t M, int64_t M_store, int nt, cudaStream_t stream) {
  if (L.dtype == PARO_BF16) return rotate_chain_T<__nv_bfloat16>(L, packed, x_op, x, norm_w, stats, stats_blocks, eps, out, M, M_store, nt, stream);
  return rotate_chain_T<__half>(L, packed, x_op, x, norm_w, stats, stats_blocks, eps, out, M, M_store, nt, stream);
}

// The pre-pass of a MoE block's grouped GEMM (paro_moe_grouped.cu): the B operand of `rows_max` routing-table positions in tiles
// of nt, from x [T, K] (silu_mul false: the gate_up operand) or from h [T * top_k, 2K] (silu_mul true: the down operand).
// The rotation every expert shares is partition 0's of expert 0 (`packed`); gate and up share it.
template <typename T>
static int rotate_routed_T(const Layout &L, const void *packed, bool silu_mul, const void *src, const int32_t *rows, const int32_t *live_tiles,
                           int top_k, void *out, int rows_max, int nt, cudaStream_t stream) {
  const RoutedRows rr = {rows, live_tiles, nt};
  if (silu_mul) {
    SiluMulRows<T> r;
    static_cast<RoutedRows &>(r) = rr;
    r.h = static_cast<const T *>(src); r.K = L.K;
    return rotate_tiles<T>(L, packed, 1, r, out, rows_max, nt, stream);
  }
  GatherRows<T> r;
  static_cast<RoutedRows &>(r) = rr;
  r.x = static_cast<const T *>(src); r.top_k = top_k; r.K = L.K;
  return rotate_tiles<T>(L, packed, 1, r, out, rows_max, nt, stream);
}

int rotate_routed_launch(const Layout &L, const void *packed, bool silu_mul, const void *src, const int32_t *rows, const int32_t *live_tiles,
                         int top_k, void *out, int rows_max, int nt, cudaStream_t stream) {
  if (L.dtype == PARO_BF16) return rotate_routed_T<__nv_bfloat16>(L, packed, silu_mul, src, rows, live_tiles, top_k, out, rows_max, nt, stream);
  return rotate_routed_T<__half>(L, packed, silu_mul, src, rows, live_tiles, top_k, out, rows_max, nt, stream);
}

// ------------------------------------------------------------------ the rotate op
template <typename T, int G>
static int rotate_op(const void *x, void *out, const int16_t *idx, const void *theta, int theta_dtype, const void *scales, int scales_dtype,
                     int64_t M, int K, int krot, cudaStream_t stream) {
  constexpr int RB = 16 / sizeof(T);
  const OpRows<T, G> src = {static_cast<const T *>(x), M, K};
  const RefMeta<T, G> meta = {idx, theta, scales, theta_dtype, scales_dtype, K, krot, 0};
  const RowMajorOut<T> o = {static_cast<T *>(out), K};
  return launch_rotation<T, G>(src, meta, o, (M + RB - 1) / RB, K, 1, stream);
}

template <typename T>
static int rotate_op_T(const void *x, void *out, const int16_t *idx, const void *theta, int theta_dtype, const void *scales, int scales_dtype,
                       int64_t M, int K, int krot, int G, cudaStream_t stream) {
  if (G == 128) return rotate_op<T, 128>(x, out, idx, theta, theta_dtype, scales, scales_dtype, M, K, krot, stream);
  return rotate_op<T, 64>(x, out, idx, theta, theta_dtype, scales, scales_dtype, M, K, krot, stream);
}

int rotate_launch(const void *x, void *out, const int16_t *idx, const void *theta, int theta_dtype, const void *scales,
                  int scales_dtype, int64_t M, int K, int krot, int G, int dtype, cudaStream_t stream) {
  if (M == 0) return PARO_OK;
  switch (dtype) {
    case PARO_F32: return rotate_op_T<float>(x, out, idx, theta, theta_dtype, scales, scales_dtype, M, K, krot, G, stream);
    case PARO_F16: return rotate_op_T<__half>(x, out, idx, theta, theta_dtype, scales, scales_dtype, M, K, krot, G, stream);
    case PARO_BF16: return rotate_op_T<__nv_bfloat16>(x, out, idx, theta, theta_dtype, scales, scales_dtype, M, K, krot, G, stream);
  }
  set_error("rotate supports Float, Half, and BFloat16, got dtype code %d", dtype);
  return PARO_EINVAL;
}

// ------------------------------------------------------------------ backward of the rotate op (training side, SURVEY 8(f) rank 4)
// The reference walks the krot rotations in Python, last to first: two one-rotation rotate launches (t and g with -theta), five
// gathers and a row reduction per rotation (/root/reference/paroquant/kernels/cuda/autograd.py:20-61).  Here ONE launch does the
// whole walk: a warp owns a group and a strided set of 4-row blocks; the stage output t (from y) and its gradient g sit in two
// fp32 shared-memory tiles; per rotation and pair
//     dL/dtheta += sum_rows (g_i t_j - g_j t_i)          (identity on the stage OUTPUT: dy_i/dtheta = y_j, dy_j/dtheta = -y_i)
//     (t, g) <- Givens(-theta) (t, g)                    (orthogonal: the same update back-propagates g), rounded to T per
//                                                         rotation exactly where the per-rotation launches rounded
// and after the last un-rotation grad_x = g * scale, dL/dscale += x * g.  dL/dtheta and dL/dscale are accumulated per warp over
// its row blocks and added to fp32 buffers with one atomic per (rotation, pair) / channel and warp.  A warp keeps ONE group for
// all its row blocks, so the group's pair slots and (cos, sin) are computed once into shared memory: the first version re-read
// indices and angles from L2 in every rotation of every row block and sat on those loads (13 long-scoreboard stalls per issue).
template <typename T, int G>
__global__ void __launch_bounds__(128) rotate_backward_kernel(const T *__restrict__ y, const T *__restrict__ gout, const T *__restrict__ x,
                                                              const int16_t *__restrict__ idx, const void *__restrict__ theta, int theta_dtype,
                                                              const void *__restrict__ scales, int scales_dtype, T *__restrict__ grad_x,
                                                              float *__restrict__ grad_theta, float *__restrict__ grad_scale, int64_t M, int K,
                                                              int krot, int splits, int ref_formula) {
  constexpr int RB = 4, CPL = G / 32, PPL = G / 64;
  __shared__ __align__(16) float4 tile_t[4][G], tile_g[4][G];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int groups = K / G;
  const int64_t wid = static_cast<int64_t>(blockIdx.x) * 4 + warp;   // (split, group)
  if (wid >= static_cast<int64_t>(splits) * groups) return;
  const int g = static_cast<int>(wid % groups), split = static_cast<int>(wid / groups);
  const int64_t row_blocks = (M + RB - 1) / RB;
  float4 *tt = tile_t[warp], *tg = tile_g[warp];
  // per warp, dynamic shared memory: [rotation][q][lane] {cos, sin} (float2), pair slots (i | j << 16), dL/dtheta partial -- each
  // lane touches only the entries of its own pairs (shared memory, not registers: the rotation loop stays rolled; unrolled over
  // 16 rotations the kernel needed 160-190 registers)
  extern __shared__ __align__(16) uint8_t bw_dyn[];
  constexpr int kPerRot = G / 2;   // pairs per rotation = PPL * 32
  float2 *mcs = reinterpret_cast<float2 *>(bw_dyn) + static_cast<size_t>(warp) * krot * kPerRot;
  uint32_t *mij = reinterpret_cast<uint32_t *>(bw_dyn + static_cast<size_t>(4) * krot * kPerRot * 8) + static_cast<size_t>(warp) * krot * kPerRot;
  float *acc = reinterpret_cast<float *>(bw_dyn + static_cast<size_t>(4) * krot * kPerRot * 12) + static_cast<size_t>(warp) * krot * kPerRot;
  // ref_formula: also sum_rows (g . t) per pair, for the value the reference's expression takes (autograd.py:50-52 applied after
  // g was un-rotated: cos * dL/dtheta - sin * sum(g . t)); the array exists only then
  float *acc2 = reinterpret_cast<float *>(bw_dyn + static_cast<size_t>(4) * krot * kPerRot * 16) + static_cast<size_t>(warp) * krot * kPerRot;
  for (int r = 0; r < krot; ++r) {
#pragma unroll
    for (int q = 0; q < PPL; ++q) {
      const int t = lane * PPL + q, e = r * kPerRot + q * 32 + lane;
      const int ij = *reinterpret_cast<const int *>(idx + static_cast<int64_t>(r) * K + g * G + 2 * t);
      const float th = load_param_as<T>(theta, static_cast<int64_t>(r) * (K / 2) + g * (G / 2) + t, theta_dtype);
      float sn, cs;
      __sincosf(-th, &sn, &cs);
      mcs[e] = make_float2(cs, sn);
      mij[e] = static_cast<uint32_t>(rot_slot(ij & 0xFFFF)) | (static_cast<uint32_t>(rot_slot((ij >> 16) & 0xFFFF)) << 16);
      acc[e] = 0.f;
      if (ref_formula) acc2[e] = 0.f;
    }
  }
  __syncwarp();
  float acc_s[CPL], sc[CPL];
#pragma unroll
  for (int c = 0; c < CPL; ++c) {
    acc_s[c] = 0.f;
    sc[c] = scales ? load_param_as<float>(scales, static_cast<int64_t>(g) * G + lane * CPL + c, scales_dtype) : 1.0f;   // autograd.py:55: the scale as stored
  }
  auto rnd = [](float v) { return Traits<T>::to_float(Traits<T>::from_float(v)); };   // the per-rotation launches store T
  for (int64_t rb = split; rb < row_blocks; rb += splits) {
    const int64_t row0 = rb * RB;
    // ---- stage output and its gradient, channel-major fp32 vectors of 4 rows
#pragma unroll
    for (int c = 0; c < CPL; ++c) {
      float vt[RB], vg[RB];
#pragma unroll
      for (int r = 0; r < RB; ++r) {
        const bool ok = row0 + r < M;
        const int64_t o = (row0 + r) * K + g * G + lane * CPL + c;
        vt[r] = ok ? Traits<T>::to_float(y[o]) : 0.f;
        vg[r] = ok ? Traits<T>::to_float(gout[o]) : 0.f;
      }
      tt[rot_slot(lane * CPL + c)] = make_float4(vt[0], vt[1], vt[2], vt[3]);
      tg[rot_slot(lane * CPL + c)] = make_float4(vg[0], vg[1], vg[2], vg[3]);
    }
    __syncwarp();
#pragma unroll 1
    for (int r = krot - 1; r >= 0; --r) {
      {
#pragma unroll
        for (int q = 0; q < PPL; ++q) {
          const int e = r * kPerRot + q * 32 + lane;
          const uint32_t ijw = mij[e];
          const int pi = ijw & 0xFFFF, pj = ijw >> 16;
          const float2 csn = mcs[e];
          const float cs = csn.x, sn = csn.y;
          float4 ti = tt[pi], tj = tt[pj], gi = tg[pi], gj = tg[pj];
          acc[e] += (gi.x * tj.x - gj.x * ti.x) + (gi.y * tj.y - gj.y * ti.y) + (gi.z * tj.z - gj.z * ti.z) + (gi.w * tj.w - gj.w * ti.w);
          if (ref_formula)   // g . t of the pair (rotation invariant, like the cross product above)
            acc2[e] += (gi.x * ti.x + gj.x * tj.x) + (gi.y * ti.y + gj.y * tj.y) + (gi.z * ti.z + gj.z * tj.z) + (gi.w * ti.w + gj.w * tj.w);
          float4 ni, nj, mi, mj;
          givens(cs, sn, ti.x, tj.x, ni.x, nj.x); givens(cs, sn, ti.y, tj.y, ni.y, nj.y);
          givens(cs, sn, ti.z, tj.z, ni.z, nj.z); givens(cs, sn, ti.w, tj.w, ni.w, nj.w);
          givens(cs, sn, gi.x, gj.x, mi.x, mj.x); givens(cs, sn, gi.y, gj.y, mi.y, mj.y);
          givens(cs, sn, gi.z, gj.z, mi.z, mj.z); givens(cs, sn, gi.w, gj.w, mi.w, mj.w);
          if constexpr (sizeof(T) == 2) {
            ni = make_float4(rnd(ni.x), rnd(ni.y), rnd(ni.z), rnd(ni.w)); nj = make_float4(rnd(nj.x), rnd(nj.y), rnd(nj.z), rnd(nj.w));
            mi = make_float4(rnd(mi.x), rnd(mi.y), rnd(mi.z), rnd(mi.w)); mj = make_float4(rnd(mj.x), rnd(mj.y), rnd(mj.z), rnd(mj.w));
          }
          tt[pi] = ni; tt[pj] = nj; tg[pi] = mi; tg[pj] = mj;
        }
        __syncwarp();
      }
    }
    // ---- g is now dL/d(x * scale)
#pragma unroll
    for (int c = 0; c < CPL; ++c) {
      const float4 gv = tg[rot_slot(lane * CPL + c)];
      const float gr[RB] = {gv.x, gv.y, gv.z, gv.w};
#pragma unroll
      for (int r = 0; r < RB; ++r) {
        if (row0 + r < M) {
          const int64_t o = (row0 + r) * K + g * G + lane * CPL + c;
          grad_x[o] = Traits<T>::from_float(scales ? gr[r] * sc[c] : gr[r]);
          if (grad_scale) acc_s[c] += Traits<T>::to_float(x[o]) * gr[r];
        }
      }
    }
    __syncwarp();
  }
  for (int r = 0; r < krot; ++r) {
#pragma unroll
    for (int q = 0; q < PPL; ++q) {
      const int e = r * kPerRot + q * 32 + lane;
      float v = acc[e];
      if (ref_formula) v = mcs[e].x * v + mcs[e].y * acc2[e];   // {cos, sin}(-theta): cos(theta) * cross - sin(theta) * dot
      atomicAdd(grad_theta + static_cast<int64_t>(r) * (K / 2) + g * (G / 2) + lane * PPL + q, v);
    }
  }
  if (grad_scale) {
#pragma unroll
    for (int c = 0; c < CPL; ++c) atomicAdd(grad_scale + static_cast<int64_t>(g) * G + lane * CPL + c, acc_s[c]);
  }
}

// The backward's launch plan, pure host logic (paro_debug_rotate_backward_plan drives it without a GPU).  Per CTA: 4 warps x krot
// x G/2 pairs x ({cos, sin} 8 B + slots 4 B + partial 4 B) of dynamic shared memory (+ 4 B: the g . t sums of the reference's
// expression) next to the two static tiles; as many CTAs per SM as that leaves room for, at most 6 (the register limit).  Enough
// (split, group) warps to fill the machine, no more splits than row blocks: every warp then walks ~row_blocks / splits blocks of
// its group (split, split + splits, ...), computes the group's (cos, sin) once and pays its atomics once.
struct BackwardPlan {
  size_t dyn;
  int ctas_per_sm;
  int64_t row_blocks, splits, blocks;
};
static BackwardPlan backward_plan(int64_t M, int K, int krot, int G, int ref_formula, int sms) {
  BackwardPlan p;
  const int groups = K / G;
  p.row_blocks = (M + 3) / 4;
  p.dyn = static_cast<size_t>(4) * krot * (G / 2) * (ref_formula ? 20 : 16);
  const int resident = static_cast<int>((227 * 1024) / (p.dyn + static_cast<size_t>(8) * G * 16 + 1024));
  p.ctas_per_sm = resident < 1 ? 1 : resident > 6 ? 6 : resident;
  p.splits = (static_cast<int64_t>(sms) * p.ctas_per_sm * 4 + groups - 1) / groups;
  if (p.splits > p.row_blocks) p.splits = p.row_blocks;
  if (p.splits < 1) p.splits = 1;
  p.blocks = (p.splits * groups + 3) / 4;
  return p;
}

int rotate_backward_debug_plan(int64_t M, int K, int krot, int G, int ref_formula, int sms, int64_t *out) {
  const BackwardPlan p = backward_plan(M, K, krot, G, ref_formula, sms);
  out[0] = static_cast<int64_t>(p.dyn);
  out[1] = p.ctas_per_sm;
  out[2] = p.splits;
  out[3] = p.row_blocks;
  out[4] = (p.row_blocks + p.splits - 1) / p.splits;   // the most row blocks a warp walks
  out[5] = p.row_blocks / p.splits;                    // the fewest
  out[6] = p.blocks;
  return PARO_OK;
}

template <typename T>
static int launch_backward_T(const void *y, const void *gout, const void *x, const int16_t *idx, const void *theta, int theta_dtype, const void *scales,
                             int scales_dtype, void *grad_x, float *grad_theta, float *grad_scale, int64_t M, int K, int krot, int G, int ref_formula,
                             cudaStream_t stream) {
  const int sms = device_sms();
  if (sms <= 0) { set_error("rotate_backward: no CUDA device"); return PARO_ECUDA; }
  const BackwardPlan plan = backward_plan(M, K, krot, G, ref_formula, sms);
  const size_t dyn = plan.dyn;
  const int64_t splits = plan.splits, blocks = plan.blocks;
  if (blocks > 0x7FFFFFFF) { set_error("rotate_backward: too many groups"); return PARO_EINVAL; }
  const T *yp = static_cast<const T *>(y), *gp = static_cast<const T *>(gout), *xp = static_cast<const T *>(x);
  T *gx = static_cast<T *>(grad_x);
  if (G == 128) {
    PARO_CUDA_OK(smem_opt_in(rotate_backward_kernel<T, 128>, static_cast<int>(dyn)));
    rotate_backward_kernel<T, 128><<<static_cast<unsigned>(blocks), 128, dyn, stream>>>(yp, gp, xp, idx, theta, theta_dtype, scales, scales_dtype, gx, grad_theta,
                                                                                       grad_scale, M, K, krot, static_cast<int>(splits), ref_formula);
  } else {
    PARO_CUDA_OK(smem_opt_in(rotate_backward_kernel<T, 64>, static_cast<int>(dyn)));
    rotate_backward_kernel<T, 64><<<static_cast<unsigned>(blocks), 128, dyn, stream>>>(yp, gp, xp, idx, theta, theta_dtype, scales, scales_dtype, gx, grad_theta,
                                                                                      grad_scale, M, K, krot, static_cast<int>(splits), ref_formula);
  }
  PARO_CUDA_OK(cudaGetLastError());
  note_launches(1);
  return PARO_OK;
}

int rotate_backward_launch(const void *y, const void *gout, const void *x, const int16_t *idx, const void *theta, int theta_dtype, const void *scales,
                           int scales_dtype, void *grad_x, float *grad_theta, float *grad_scale, int64_t M, int K, int krot, int G, int dtype,
                           int ref_formula, cudaStream_t stream) {
  if (M == 0) return PARO_OK;
  switch (dtype) {
    case PARO_F32: return launch_backward_T<float>(y, gout, x, idx, theta, theta_dtype, scales, scales_dtype, grad_x, grad_theta, grad_scale, M, K, krot, G, ref_formula, stream);
    case PARO_F16: return launch_backward_T<__half>(y, gout, x, idx, theta, theta_dtype, scales, scales_dtype, grad_x, grad_theta, grad_scale, M, K, krot, G, ref_formula, stream);
    case PARO_BF16: return launch_backward_T<__nv_bfloat16>(y, gout, x, idx, theta, theta_dtype, scales, scales_dtype, grad_x, grad_theta, grad_scale, M, K, krot, G, ref_formula, stream);
  }
  set_error("rotate supports Float, Half, and BFloat16, got dtype code %d", dtype);
  return PARO_EINVAL;
}

}  // namespace paro
