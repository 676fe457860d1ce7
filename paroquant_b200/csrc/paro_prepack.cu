// One-time AWQ checkpoint layout -> streaming layout (see paro_layout.h), and its inverse for
// tests.  Integer work, bit-exact by construction; replaces the AWQ->Marlin repack the reference
// reaches through ParoQuantLinearMethod.process_weights_after_loading
// (/root/reference/paroquant/inference/backends/vllm/plugin.py:208-279).
#include "paro_common.cuh"
#include "paro_launch.h"

namespace paro {

// AWQ: nibble slot i of a word holds column 8c + (0,2,4,6,1,3,5,7)[i]  (cli/convert.py:19)
__device__ __forceinline__ uint32_t awq_nibble(const int32_t *packed, int64_t row, int n, int ncols8) {
  const uint32_t w = static_cast<uint32_t>(packed[row * ncols8 + (n >> 3)]);
  const int c = n & 7;
  const int slot = (c >> 1) + ((c & 1) << 2);
  return (w >> (4 * slot)) & 0xFu;
}

__device__ __forceinline__ uint16_t cast_to_T_bits(const void *p, int64_t i, int src_dtype, int dst_dtype) {
  float f;
  if (src_dtype == PARO_F32) f = reinterpret_cast<const float *>(p)[i];
  else if (src_dtype == PARO_F16) f = __half2float(reinterpret_cast<const __half *>(p)[i]);
  else f = __bfloat162float(reinterpret_cast<const __nv_bfloat16 *>(p)[i]);
  if (dst_dtype == PARO_F16) return __half_as_ushort(__float2half_rn(f));
  return __bfloat16_as_ushort(__float2bfloat16_rn(f));
}

__global__ void prepack_meta_kernel(Layout L, const int16_t *__restrict__ pairs, const void *__restrict__ theta,
                                    int theta_dtype, const void *__restrict__ cscales, int cs_dtype,
                                    uint8_t *__restrict__ packed) {
  // one thread per (part, group, channel c in 0..127)
  const int64_t idx = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
  const int64_t total = static_cast<int64_t>(L.n_parts) * L.groups * kGroup;
  if (idx >= total) return;
  const int c = idx % kGroup;
  const int gk = (idx / kGroup) % L.groups;
  const int part = idx / (static_cast<int64_t>(kGroup) * L.groups);
  uint8_t *blk = packed + L.meta_offset(part, gk);
  const int K = L.K;
  // group_size 64: indices are local to the 64-channel group; the second group of the record moves up by 64, so the two
  // rotations become ONE 128-channel rotation of identical arithmetic (theta: 2 x 32 consecutive values = the same 64)
  const int16_t lift = (L.qhalves == 2 && c >= 64) ? 64 : 0, imask = L.qhalves == 2 ? 0x3F : 0x7F;
  for (int r = 0; r < L.krot; ++r) {
    const int16_t v = static_cast<int16_t>((pairs[(static_cast<int64_t>(part) * L.krot + r) * K + gk * kGroup + c] & imask) + lift);
    blk[meta_pairs_off(r) + c] = static_cast<uint8_t>(v);
    if (c < 64) {
      const int64_t ti = (static_cast<int64_t>(part) * L.krot + r) * (K / 2) + gk * 64 + c;
      reinterpret_cast<uint16_t *>(blk + meta_theta_off(L.krot, r))[c] = cast_to_T_bits(theta, ti, theta_dtype, L.dtype);
    }
  }
  reinterpret_cast<uint16_t *>(blk + meta_scales_off(L.krot))[c] =
      cast_to_T_bits(cscales, static_cast<int64_t>(part) * K + gk * kGroup + c, cs_dtype, L.dtype);
}

// block index over all partitions -> partition
__device__ __forceinline__ int block_part(const Layout &L, int block) {
  int part = 0;
  while (block >= L.part_block_begin[part + 1]) ++part;
  return part;
}

__global__ void prepack_weight_kernel(Layout L, const int32_t *__restrict__ qweight, uint8_t *__restrict__ packed) {
  // one thread per output word: (record = (block, g), row tile, k half kh, lane, k16 step s of the half) -- paro_layout.h
  const int64_t idx = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
  const int64_t total = static_cast<int64_t>(L.blocks_total) * L.groups * 2048;
  if (idx >= total) return;
  const int s = idx & 3, lane = (idx >> 2) & 31, kh = (idx >> 7) & 1, tile = (idx >> 8) & 7;
  const int64_t rec = idx >> 11;
  const int block = static_cast<int>(rec / L.groups), g = static_cast<int>(rec % L.groups);
  const int part = block_part(L, block);
  const int n0 = L.part_col_begin[part] + (block - L.part_block_begin[part]) * kBlockN + tile * 16 + (lane >> 2);
  const int64_t k0 = static_cast<int64_t>(g) * kGroup + 16 * (4 * kh + s) + 2 * (lane & 3);
  const int nc8 = L.N / 8;
  uint32_t w = 0;
#pragma unroll
  for (int i = 0; i < 4; ++i) {   // A-fragment register i: row g (+ 8 for odd i), channels 2t, 2t + 1 (+ 8 for i >= 2)
    const int n = n0 + 8 * (i & 1);
    const int64_t k = k0 + 8 * (i >> 1);
    if (n < L.part_col_begin[part + 1])
      w |= (awq_nibble(qweight, k, n, nc8) << (4 * i)) | (awq_nibble(qweight, k + 1, n, nc8) << (16 + 4 * i));
  }
  reinterpret_cast<uint32_t *>(packed + L.rec_off + rec * L.rec_bytes)[idx & 2047] = w;
}

__global__ void prepack_qparam_kernel(Layout L, const int32_t *__restrict__ qzeros, const void *__restrict__ scales,
                                      int scales_dtype, uint8_t *__restrict__ packed) {
  // one thread per (record, quantisation group h of the record, column of the block)
  const int64_t idx = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
  const int64_t total = static_cast<int64_t>(L.blocks_total) * L.groups * L.qhalves * kBlockN;
  if (idx >= total) return;
  const int col = idx & 127;
  const int h = static_cast<int>((idx >> 7) % L.qhalves);
  const int64_t rec = (idx >> 7) / L.qhalves;
  const int block = static_cast<int>(rec / L.groups), g = static_cast<int>(rec % L.groups);
  const int part = block_part(L, block);
  const int n = L.part_col_begin[part] + (block - L.part_block_begin[part]) * kBlockN + col;
  uint16_t s = 0;
  uint8_t z = 0;
  if (n < L.part_col_begin[part + 1]) {
    const int64_t qg = static_cast<int64_t>(g) * L.qhalves + h;   // row of the checkpoint's scales / qzeros
    s = cast_to_T_bits(scales, qg * L.N + n, scales_dtype, L.dtype);
    z = static_cast<uint8_t>(awq_nibble(qzeros, qg, n, L.N / 8));
  }
  uint8_t *rb = packed + L.rec_off + rec * L.rec_bytes;
  reinterpret_cast<uint16_t *>(rb + kBlockScaleOff)[h * 128 + qparam_index(col)] = s;
  rb[block_zero_off(L.qhalves) + h * 128 + qparam_index(col)] = z;
}

// Inverse, for tests: dense W[k][n] = T((q - z) * s_T), the exact operand the GEMM consumes.
template <typename T>
__global__ void unpack_dense_kernel(Layout L, const uint8_t *__restrict__ packed, T *__restrict__ W) {
  const int64_t idx = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
  if (idx >= static_cast<int64_t>(L.K) * L.N) return;
  const int n = idx % L.N;
  const int k = idx / L.N;
  int part = 0;
  while (n >= L.part_col_begin[part + 1]) ++part;
  const int nl = n - L.part_col_begin[part];
  const int block = L.part_block_begin[part] + nl / kBlockN, col = nl % kBlockN;
  const int g = k / kGroup, kl = k % kGroup;
  // A-fragment position of (k, column): step kl / 16, lane (row % 8, channel pair), register (row / 8, channel / 8 of the step)
  const int step = kl >> 4, kk = kl & 15, row = col & 15;
  const int lane = 4 * (row & 7) + ((kk & 7) >> 1), i = (row >> 3) + 2 * (kk >> 3);
  const uint8_t *rb = packed + L.record_offset(block, g);
  const uint32_t w = reinterpret_cast<const uint32_t *>(rb + frag_offset(col >> 4, step >> 2, lane))[step & 3];
  const int q = (w >> (4 * i + 16 * (kk & 1))) & 0xF;
  const int h = L.qhalves == 2 ? kl >> 6 : 0;
  const int z = rb[block_zero_off(L.qhalves) + h * 128 + qparam_index(col)];
  const T s = reinterpret_cast<const T *>(rb + kBlockScaleOff)[h * 128 + qparam_index(col)];
  // (q - z) is exact in T; one rounding in the product, like the fused kernels
  W[idx] = Traits<T>::from_float(static_cast<float>(q - z) * Traits<T>::to_float(s));
}

int prepack_launch(const paro_linear_shape &s, const Layout &L, const int32_t *qweight, const int32_t *qzeros,
                   const void *scales, int scales_dtype, const int16_t *pairs, const void *theta, int theta_dtype,
                   const void *cscales, int cs_dtype, void *packed, cudaStream_t stream) {
  uint8_t *out = static_cast<uint8_t *>(packed);
  const int B = 256;
  {
    const int64_t total = static_cast<int64_t>(L.n_parts) * L.groups * kGroup;
    prepack_meta_kernel<<<static_cast<unsigned>((total + B - 1) / B), B, 0, stream>>>(L, pairs, theta, theta_dtype,
                                                                                     cscales, cs_dtype, out);
  }
  {
    const int64_t total = static_cast<int64_t>(L.blocks_total) * L.groups * 2048;
    prepack_weight_kernel<<<static_cast<unsigned>((total + B - 1) / B), B, 0, stream>>>(L, qweight, out);
  }
  {
    const int64_t total = static_cast<int64_t>(L.blocks_total) * L.groups * L.qhalves * kBlockN;
    prepack_qparam_kernel<<<static_cast<unsigned>((total + B - 1) / B), B, 0, stream>>>(L, qzeros, scales, scales_dtype, out);
  }
  PARO_CUDA_OK(cudaGetLastError());
  note_launches(3);
  return PARO_OK;
}

int unpack_dense_launch(const paro_linear_shape &s, const Layout &L, const void *packed, void *W, cudaStream_t stream) {
  const int64_t total = static_cast<int64_t>(L.K) * L.N;
  const int B = 256;
  const unsigned grid = static_cast<unsigned>((total + B - 1) / B);
  if (L.dtype == PARO_F16)
    unpack_dense_kernel<__half><<<grid, B, 0, stream>>>(L, static_cast<const uint8_t *>(packed), static_cast<__half *>(W));
  else
    unpack_dense_kernel<__nv_bfloat16><<<grid, B, 0, stream>>>(L, static_cast<const uint8_t *>(packed),
                                                               static_cast<__nv_bfloat16 *>(W));
  PARO_CUDA_OK(cudaGetLastError());
  note_launches(1);
  return PARO_OK;
}

}  // namespace paro
