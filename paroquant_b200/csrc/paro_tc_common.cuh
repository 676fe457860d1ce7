// Device helpers shared by the tensor-core kernels (paro_decode.cu, paro_stream.cu, paro_moe.cu, paro_gemm.cu):
// mma.sync / wgmma wrappers and operand fragments, cluster + DSMEM primitives, the INT4 -> T A-fragment dequant, the small-M
// kernels' weight ring (set-up, producer step, round loop),
// the in-warp pairwise rotation (rounding points of /root/reference/paroquant/kernels/cuda/rotation.cuh:91-173) and the
// small-M kernels' rotation prologue built from it (rotation_tasks).
#pragma once
#include <type_traits>

#include "paro_common.cuh"
#include "paro_layout.h"

namespace paro {

__device__ __forceinline__ unsigned long long globaltimer_ns() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}

// ------------------------------------------------------------------ tensor-core operands
// Both fused small-M kernels (paro_decode.cu, paro_stream.cu) and the large-M GEMM (paro_gemm.cu) work operand-swapped:
// D[n, m] += W[n, k] * x_rot[m, k], the dequantised weights are the register A operand, x_rot the shared-memory B operand.
// A warp owns a 16-row tile of the 128-column block; its A fragment (mma.m16n8k16 and one warp's slice of a wgmma m64) holds
// rows g = lane / 4 and g + 8, channels 2t, 2t + 1 and 2t + 8, 2t + 9 of each k16 step (t = lane % 4).

// D (fp32, 16 x 8) += A (16 x 16) * B (16 x 8)
template <typename T>
__device__ __forceinline__ void mma16816(float (&d)[4], const uint32_t *a, uint32_t b0, uint32_t b1) {
  if constexpr (Traits<T>::code == PARO_BF16)
    asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
  else
    asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

// K-major, no swizzle: 8-row x 16-byte core matrices; `lbo` = byte distance between the two k-halves of a k16 step,
// `sbo` = byte distance between 8-row groups (wgmma matrix descriptor, swizzle mode 0)
__device__ __forceinline__ uint64_t smem_desc_kmajor(uint32_t addr, uint32_t lbo, uint32_t sbo) {
  return static_cast<uint64_t>((addr >> 4) & 0x3FFF) | (static_cast<uint64_t>((lbo >> 4) & 0x3FFF) << 16) |
         (static_cast<uint64_t>((sbo >> 4) & 0x3FFF) << 32);
}

__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N> __device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
template <int R> __device__ __forceinline__ void fence_operands(float (&d)[R]) {
#pragma unroll
  for (int i = 0; i < R; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

// D (fp32, 64 x N, the warpgroup's registers) += A (64 x 16, registers) * B (16 x N, shared memory descriptor, K-major)
template <typename T, int N> struct Wgmma;
template <> struct Wgmma<__nv_bfloat16, 32> {
  __device__ static __forceinline__ void mma(float (&d)[16], const uint32_t *a, uint64_t desc) {
    asm volatile(
        "wgmma.mma_async.sync.aligned.m64n32k16.f32.bf16.bf16 "
        "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15}, {%16,%17,%18,%19}, %20, 1, 1, 1, 0;"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(desc));
  }
};
template <> struct Wgmma<__half, 32> {
  __device__ static __forceinline__ void mma(float (&d)[16], const uint32_t *a, uint64_t desc) {
    asm volatile(
        "wgmma.mma_async.sync.aligned.m64n32k16.f32.f16.f16 "
        "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15}, {%16,%17,%18,%19}, %20, 1, 1, 1, 0;"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(desc));
  }
};
template <> struct Wgmma<__nv_bfloat16, 64> {
  __device__ static __forceinline__ void mma(float (&d)[32], const uint32_t *a, uint64_t desc) {
    asm volatile(
        "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 "
        "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31}, {%32,%33,%34,%35}, %36, 1, 1, 1, 0;"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(desc));
  }
};
template <> struct Wgmma<__half, 64> {
  __device__ static __forceinline__ void mma(float (&d)[32], const uint32_t *a, uint64_t desc) {
    asm volatile(
        "wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 "
        "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31}, {%32,%33,%34,%35}, %36, 1, 1, 1, 0;"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(desc));
  }
};
template <> struct Wgmma<__nv_bfloat16, 128> {
  __device__ static __forceinline__ void mma(float (&d)[64], const uint32_t *a, uint64_t desc) {
    asm volatile(
        "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 "
        "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,%60,%61,%62,%63}, {%64,%65,%66,%67}, %68, 1, 1, 1, 0;"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(desc));
  }
};
template <> struct Wgmma<__half, 128> {
  __device__ static __forceinline__ void mma(float (&d)[64], const uint32_t *a, uint64_t desc) {
    asm volatile(
        "wgmma.mma_async.sync.aligned.m64n128k16.f32.f16.f16 "
        "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,%60,%61,%62,%63}, {%64,%65,%66,%67}, %68, 1, 1, 1, 0;"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(desc));
  }
};

// one lane of a converged warp (CUTLASS' elect_one_sync): ptxas treats the guarded region as single-threaded
__device__ __forceinline__ bool elect_one() {
  uint32_t pred;
  asm volatile("{\n\t.reg .pred P;\n\telect.sync _|P, 0xFFFFFFFF;\n\tselp.u32 %0, 1, 0, P;\n\t}" : "=r"(pred));
  return pred != 0;
}

__device__ __forceinline__ void named_bar_sync(int id, int nthreads) { asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(nthreads) : "memory"); }

// ------------------------------------------------------------------ cluster / DSMEM helpers
__device__ __forceinline__ void cluster_arrive_relaxed() { asm volatile("barrier.cluster.arrive.relaxed.aligned;" ::: "memory"); }
__device__ __forceinline__ void cluster_arrive_release() { asm volatile("barrier.cluster.arrive.release.aligned;" ::: "memory"); }
__device__ __forceinline__ void cluster_wait_acquire() { asm volatile("barrier.cluster.wait.acquire.aligned;" ::: "memory"); }
__device__ __forceinline__ uint32_t map_to_rank(uint32_t local_smem_addr, uint32_t rank) {
  uint32_t r;
  asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(r) : "r"(local_smem_addr), "r"(rank));
  return r;
}
__device__ __forceinline__ void st_cluster_f32(uint32_t addr, float v) {
  asm volatile("st.shared::cluster.f32 [%0], %1;" ::"r"(addr), "f"(v) : "memory");
}
__device__ __forceinline__ float lds_f32(uint32_t addr) {
  float v;
  asm volatile("ld.shared.f32 %0, [%1];" : "=f"(v) : "r"(addr));
  return v;
}
__device__ __forceinline__ void sts_f32(uint32_t addr, float v) { asm volatile("st.shared.f32 [%0], %1;" ::"r"(addr), "f"(v) : "memory"); }
__device__ __forceinline__ void sts128u(uint32_t addr, uint4 v) {
  asm volatile("st.shared.v4.u32 [%0], {%1,%2,%3,%4};" ::"r"(addr), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w) : "memory");
}

template <typename T> __device__ __forceinline__ T bits_to_T(uint32_t b) {
  const uint16_t h = static_cast<uint16_t>(b);
  return *reinterpret_cast<const T *>(&h);
}
template <typename T> __device__ __forceinline__ uint16_t T_to_bits(T v) { return *reinterpret_cast<const uint16_t *>(&v); }

// ------------------------------------------------------------------ INT4 -> T dequant of A fragments
// (a & mask) | magic in ONE LOP3: both constants must sit in registers (LOP3 takes one immediate)
__device__ __forceinline__ uint32_t and_or(uint32_t a, uint32_t mask, uint32_t magic) {
  uint32_t d;
  asm("lop3.b32 %0, %1, %2, %3, 0xEA;" : "=r"(d) : "r"(a), "r"(mask), "r"(magic));
  return d;
}

// Dequantiser of one lane's rows g and g + 8 of a 16-row tile (paro_layout.h: the two rows' scales are one 32-bit word of
// the record, their zeros one 16-bit word).  magic | q is the T value base + q (bf16 0x4300 = 128, half 0x6400 = 1024):
// (base + q) - (base + z) = q - z exactly, then one rounding in the multiply by the scale.
template <typename T>
struct FragDequant {
  static constexpr uint32_t kMagic = Traits<T>::code == PARO_BF16 ? 0x43004300u : 0x64006400u;
  uint32_t s0, s1, z0, z1;   // T x2 {s, s} and {base + z, base + z} of rows g (0) and g + 8 (1)
  __device__ __forceinline__ void prep(uint32_t s_pair, uint32_t z_pair) {
    s0 = __byte_perm(s_pair, 0u, 0x1010);
    s1 = __byte_perm(s_pair, 0u, 0x3232);
    z0 = __byte_perm(z_pair, kMagic >> 8, 0x4040);   // bytes {z, magic byte, z, magic byte}
    z1 = __byte_perm(z_pair, kMagic >> 8, 0x4141);
  }
  __device__ __forceinline__ uint32_t one(uint32_t w, uint32_t z, uint32_t sc) const {
    using T2 = typename Traits<T>::T2;
    const T2 d = __hsub2(unpack2<T>(and_or(w, 0x000F000Fu, kMagic)), unpack2<T>(z));
    return pack2<T>(__hmul2(d, unpack2<T>(sc)));
  }
  // the A fragment of one k16 step from its record word: register i = (w >> 4i) & 0x000F000F, rows g / g + 8 alternating
  __device__ __forceinline__ void frag(uint32_t w, uint32_t *a) const {
    a[0] = one(w, z0, s0);
    a[1] = one(w >> 4, z1, s1);
    a[2] = one(w >> 8, z0, s0);
    a[3] = one(w >> 12, z1, s1);
  }
};

// four 8 x 8 b16 matrices; lanes 8i .. 8i + 7 give the row addresses of matrix i, register i of lane l holds its row
// l / 4, elements 2 (l % 4) and + 1 -- for a K-major core matrix that is an mma.m16n8k16 .col B fragment register
__device__ __forceinline__ void ldsm_x4(uint32_t addr, uint32_t (&r)[4]) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];" : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(addr));
}

// Per-lane shared-memory offsets of a small-M worker warp's round: they depend on the warp's (tile, k half) and the lane
// only, so the round loop computes them once.  w / s / z are record-relative, x is relative to the group's B operand:
// the row this lane hands to ldmatrix.x4 for k16 steps (4 kh, 4 kh + 1) -- matrices {step, k half} = {0, 0}, {0, 1},
// {1, 0}, {1, 1}, i.e. b0, b1 of the first step and b0, b1 of the second.
struct RoundLane {
  uint32_t w, s, z, x;
};
template <int NR>
__device__ __forceinline__ RoundLane round_lane(bool q2, int tile, int kh, int lane) {
  const int g = lane >> 2;
  const bool second = q2 && kh;   // group_size 64: channels 64..127 (kh = 1) have the record's second scale / zero set
  RoundLane o;
  o.w = frag_offset(tile, kh, lane);
  o.s = kBlockScaleOff + (second ? 256 : 0) + 2 * qparam_index(16 * tile + g);
  o.z = block_zero_off(q2 ? 2 : 1) + (second ? 128 : 0) + qparam_index(16 * tile + g);
  o.x = (4 * kh + (lane >> 4)) * (NR * 32) + ((lane >> 3) & 1) * (NR * 16) + (lane & 7) * 16;
  return o;
}

// NREC (1 or 2) records of consecutive groups for a small-M worker warp: record i at rec + i * rec_stride, its B operand
// (x_rot of the group) at bx - o.x + i * NR * 256, where bx is this lane's ldmatrix row of the first group.  Per record the
// warp takes its 16-row tile, k16 steps 4 kh .. 4 kh + 3, NTT token tiles of 8.  B is K-major core matrices: [k16 step]
// [k half][row / 8][row % 8][8 elements], NR rows per step (8 or 16).  One 128-bit load brings a record's four A fragments
// (paro_layout.h), two ldmatrix.x4 its B fragments per token tile.  Every load of both records is issued first and the two
// dequants are independent, so one ring wait covers two records' worth of latency; the MMAs go into ONE accumulator in
// record, step order -- the sum order of one record per call, so the result does not depend on how records are paired.
template <typename T, int NTT, int NREC, int NR>
__device__ __forceinline__ void mma_rounds(uint32_t rec, uint32_t rec_stride, uint32_t bx, const RoundLane &o, float (&acc)[2][4]) {
  FragDequant<T> d[NREC];
  uint4 w[NREC];
  uint32_t b[NREC][NTT][2][4];   // [record][token tile][steps 0-1 / 2-3][b0, b1 of the first step, b0, b1 of the second]
#pragma unroll
  for (int i = 0; i < NREC; ++i) {
    const uint32_t r = rec + i * rec_stride;
    d[i].prep(lds32(r + o.s), lds16(r + o.z));
    w[i] = lds128(r + o.w);
#pragma unroll
    for (int nt = 0; nt < NTT; ++nt)
#pragma unroll
      for (int h = 0; h < 2; ++h) ldsm_x4(bx + i * (NR * 256) + h * (NR * 64) + nt * 128, b[i][nt][h]);
  }
#pragma unroll
  for (int i = 0; i < NREC; ++i) {
    const uint32_t ws[4] = {w[i].x, w[i].y, w[i].z, w[i].w};
#pragma unroll
    for (int s = 0; s < 4; ++s) {
      uint32_t a[4];
      d[i].frag(ws[s], a);
#pragma unroll
      for (int nt = 0; nt < NTT; ++nt) mma16816<T>(acc[nt], a, b[i][nt][s >> 1][2 * (s & 1)], b[i][nt][s >> 1][2 * (s & 1) + 1]);
    }
  }
}

// ------------------------------------------------------------------ weight ring of the small-M kernels (decode, stream, MoE)
// `nstages` stages of one record each, every stage with a full barrier (the producer's expect_tx, then the bulk copy's bytes)
// and an empty barrier (one arrival per consumer warp), 8 bytes apart from `full` / `empty`.  One barrier pair per lane of the
// calling warp; the caller initialises its own other barriers and then fences them all (fence_mbar_init).
__device__ __forceinline__ void ring_init(uint32_t full, uint32_t empty, int nstages, int consumers, int lane) {
  if (lane < nstages) {
    mbar_init(full + 8 * lane, 1);
    mbar_init(empty + 8 * lane, consumers);
  }
}

// The producer warp's place in the ring: stage `st` of wrap `it`.  The whole warp calls issue(), which waits until the stage's
// previous record was consumed, then one elected lane arms the full barrier, starts the bulk copy of `bytes` from src() into
// the stage and runs on_issue().  src is a hook so that the address arithmetic stays behind the wait, where the producer loops
// had it (computed ahead, it reorders decode_kernel's instructions).
struct RingProducer {
  uint32_t full, empty, stage0, stride;   // barrier bases, stage 0's address, stage stride
  int nstages, st, it;
  template <typename Src, typename OnIssue>
  __device__ __forceinline__ void issue(Src src, uint32_t bytes, uint64_t policy, OnIssue on_issue) {
    if (it > 0) mbar_wait(empty + 8 * st, (it - 1) & 1);
    if (elect_one()) {
      mbar_arrive_expect_tx(full + 8 * st, bytes);
      bulk_g2s(stage0 + st * stride, src(), bytes, full + 8 * st, policy);
      on_issue();
    }
    __syncwarp();
    if (++st == nstages) { st = 0; ++it; }
  }
};

// A worker warp's place in the weight ring: `fb` = full barrier of the next stage to take, its empty barrier sits `empty_off`
// above; stage records are rec_stride apart, the record of a stage is fb * rec_per_bar + rec_at_bar0.
struct RingCursor {
  uint32_t fb, par, bar0, end, empty_off, rec_per_bar, rec_at_bar0, rec_stride;
  __device__ __forceinline__ uint32_t rec() const { return fb * rec_per_bar + rec_at_bar0; }
  __device__ __forceinline__ void advance(int n) {
    fb += 8 * n;
    if (fb == end) { fb = bar0; par ^= 1; }
  }
  __device__ __forceinline__ void release(uint32_t first, int n) const {
    __syncwarp();
    if (elect_one()) {
      for (int i = 0; i < n; ++i) mbar_arrive(first + 8 * i + empty_off);
    }
  }
};

// The round loop of a worker warp over `nseg` segments (runs of consecutive records that go into one accumulator):
// seg_begin(k, bx, len) gives segment k's first B row and record count, seg_end(k, acc) hands its accumulator on.  Records
// are taken in pairs from an even stage; a segment that starts at an odd stage takes its first record alone, an odd remainder
// its last.  The loop counts the records left in the segment.
// The ring depth must be even, so that a pair never wraps: every caller's depth rule (ring_stages) rounds to a multiple of 2.
// seen(n) / done(n): tracing hooks after n records' full barriers were seen / their MMAs issued.
template <typename T, int NTT, int NR, typename SegBegin, typename SegEnd, typename Seen, typename Done>
__device__ __forceinline__ void segment_rounds(RingCursor &rg, const RoundLane &lo, int nseg, SegBegin seg_begin, SegEnd seg_end, Seen seen,
                                               Done done) {
  float acc[2][4];
  uint32_t bx = 0;   // this lane's ldmatrix row of the next record
  int left = 0;      // records of the segment not taken yet
  auto take = [&](auto nrec) {
    constexpr int NREC = decltype(nrec)::value;
    for (int i = 0; i < NREC; ++i) mbar_wait(rg.fb + 8 * i, rg.par);
    seen(NREC);
    mma_rounds<T, NTT, NREC, NR>(rg.rec(), rg.rec_stride, bx, lo, acc);
    rg.release(rg.fb, NREC);
    done(NREC);
    bx += NREC * (NR * 256);
    rg.advance(NREC);
    left -= NREC;
  };
  int k = 0;
#pragma unroll 1
  while (k < nseg) {
    seg_begin(k, bx, left);
#pragma unroll
    for (int e = 0; e < 8; ++e) acc[e >> 2][e & 3] = 0.f;
    if (left > 0 && ((rg.fb - rg.bar0) & 8)) take(std::integral_constant<int, 1>{});
    // The pair loop sits in its own branch, with the segment's close written out on both sides, on purpose.  In this shape
    // ptxas issues a pair's two full-barrier waits back to back (no YIELD and no address add between them) and hoists all of
    // the pair's shared-memory loads (scale / zero words, the 128-bit weight words, the first ldmatrix) right behind them,
    // ahead of the first dequant.  A plain `for (k) { ...; while (left >= 2) take(2); ... }` of the same operations
    // interleaves those loads with the dequant of the first k16 steps; on an H100 the per-linear M = 1 decode ran ~3.5 %
    // slower that way (DESIGN.md section 4).
    if (left >= 2) {
#pragma unroll 1
      while (left >= 2) take(std::integral_constant<int, 2>{});
      if (left == 1) take(std::integral_constant<int, 1>{});
      seg_end(k, acc);
      ++k;
    } else {
      if (left == 1) take(std::integral_constant<int, 1>{});
      seg_end(k, acc);
      ++k;
    }
  }
}

// The two k-half warps of a tile add their accumulators in a fixed order: the k-half-1 warp stores its 8 values per lane at
// xc, xc + 128, ..., both pass the tile's pair barrier `bar`, and the k-half-0 warp adds them to its own and runs sum().
template <typename Sum>
__device__ __forceinline__ void khalf_meet(float (&acc)[2][4], uint32_t xc, int kh, int bar, Sum sum) {
  if (kh == 1) {
#pragma unroll
    for (int i = 0; i < 8; ++i) sts_f32(xc + i * 128, acc[i >> 2][i & 3]);
  }
  named_bar_sync(bar, 64);
  if (kh == 0) {
#pragma unroll
    for (int i = 0; i < 8; ++i) acc[i >> 2][i & 3] += lds_f32(xc + i * 128);
    sum();
  }
}

// ------------------------------------------------------------------ in-warp rotation of one group
// Tile `rot` = this warp's [128 channels][ROWS] elements of T, channel-major.  Lane owns pairs
// 2*lane and 2*lane+1 of every rotation; idxw = bytes (i0, j0, i1, j1).
template <typename T, int ROWS>
__device__ __forceinline__ void rotate_stage(uint32_t rot, uint32_t idxw, float c0, float s0, float c1, float s1) {
  const uint32_t i0 = idxw & 0xFFu, j0 = (idxw >> 8) & 0xFFu, i1 = (idxw >> 16) & 0xFFu, j1 = idxw >> 24;
  if constexpr (ROWS == 1) {
    // all four loads first (the two pairs are disjoint), then the math, then the stores
    const uint32_t a0 = rot + i0 * 2, b0 = rot + j0 * 2, a1 = rot + i1 * 2, b1 = rot + j1 * 2;
    const float xa0 = Traits<T>::to_float(bits_to_T<T>(lds16(a0))), xb0 = Traits<T>::to_float(bits_to_T<T>(lds16(b0)));
    const float xa1 = Traits<T>::to_float(bits_to_T<T>(lds16(a1))), xb1 = Traits<T>::to_float(bits_to_T<T>(lds16(b1)));
    float yi0, yj0, yi1, yj1;
    givens(c0, s0, xa0, xb0, yi0, yj0);
    givens(c1, s1, xa1, xb1, yi1, yj1);
    sts16(a0, T_to_bits<T>(Traits<T>::from_float(yi0)));
    sts16(b0, T_to_bits<T>(Traits<T>::from_float(yj0)));
    sts16(a1, T_to_bits<T>(Traits<T>::from_float(yi1)));
    sts16(b1, T_to_bits<T>(Traits<T>::from_float(yj1)));
  } else {
    constexpr int MPW = ROWS / 2;
    const uint32_t ad[4] = {rot + i0 * (MPW * 4), rot + j0 * (MPW * 4), rot + i1 * (MPW * 4), rot + j1 * (MPW * 4)};
    uint32_t v[4][MPW];
#pragma unroll
    for (int k = 0; k < 4; ++k)
#pragma unroll
      for (int u = 0; u < MPW; ++u) v[k][u] = lds32(ad[k] + 4 * u);
#pragma unroll
    for (int q = 0; q < 2; ++q) {
      const float c = q ? c1 : c0, s = q ? s1 : s0;
#pragma unroll
      for (int u = 0; u < MPW; ++u) {
        const float2 a = Traits<T>::to_float2(unpack2<T>(v[2 * q][u]));
        const float2 b = Traits<T>::to_float2(unpack2<T>(v[2 * q + 1][u]));
        float yix, yiy, yjx, yjy;
        givens(c, s, a.x, b.x, yix, yjx);
        givens(c, s, a.y, b.y, yiy, yjy);
        sts32(ad[2 * q] + 4 * u, pack2<T>(Traits<T>::from_floats(yix, yiy)));
        sts32(ad[2 * q + 1] + 4 * u, pack2<T>(Traits<T>::from_floats(yjx, yjy)));
      }
    }
  }
}

// multiply by the channel scales in T (one rounding, rotation.cuh:112-113), lay out channel-major in `rot`
template <typename T, int ROWS>
__device__ __forceinline__ void scale_and_stage(uint32_t rot, int lane, const uint2 (&raw)[ROWS], uint2 csw) {
  using T2 = typename Traits<T>::T2;
  const T2 sc01 = unpack2<T>(csw.x), sc23 = unpack2<T>(csw.y);
  if constexpr (ROWS == 1) {
    const uint32_t v01 = pack2<T>(__hmul2(unpack2<T>(raw[0].x), sc01));
    const uint32_t v23 = pack2<T>(__hmul2(unpack2<T>(raw[0].y), sc23));
    asm volatile("st.shared.v2.u32 [%0], {%1,%2};" ::"r"(rot + 8 * lane), "r"(v01), "r"(v23) : "memory");
  } else {
    constexpr int MPW = ROWS / 2;
    uint32_t v01[ROWS], v23[ROWS];
#pragma unroll
    for (int m = 0; m < ROWS; ++m) {
      v01[m] = pack2<T>(__hmul2(unpack2<T>(raw[m].x), sc01));
      v23[m] = pack2<T>(__hmul2(unpack2<T>(raw[m].y), sc23));
    }
#pragma unroll
    for (int u = 0; u < MPW; ++u) {  // word u of a channel = rows (2u, 2u+1)
      const uint32_t base = rot + (4 * lane) * (MPW * 4) + 4 * u;
      sts32(base + 0 * (MPW * 4), __byte_perm(v01[2 * u], v01[2 * u + 1], 0x5410));
      sts32(base + 1 * (MPW * 4), __byte_perm(v01[2 * u], v01[2 * u + 1], 0x7632));
      sts32(base + 2 * (MPW * 4), __byte_perm(v23[2 * u], v23[2 * u + 1], 0x5410));
      sts32(base + 3 * (MPW * 4), __byte_perm(v23[2 * u], v23[2 * u + 1], 0x7632));
    }
  }
}

// silu as vLLM's silu_and_mul computes it: T(x / (1 + exp(-x))) in fp32, then the product in T (paro_stream.cu's SILU_MUL x op
// and paro_moe.cu's down prologue)
template <typename T> __device__ __forceinline__ uint32_t silu_mul2(uint32_t g2, uint32_t u2) {
  const float2 g = Traits<T>::to_float2(unpack2<T>(g2));
  const float a = g.x / (1.0f + __expf(-g.x)), b = g.y / (1.0f + __expf(-g.y));
  return pack2<T>(__hmul2(Traits<T>::from_floats(a, b), unpack2<T>(u2)));
}

// RMSNorm as vLLM's (fused_add_)rms_norm: T(T(h * rstd) * w) (paro_stream.cu's RMSNORM x op and the prefill chain's pre-pass)
template <typename T> __device__ __forceinline__ uint32_t norm2(uint32_t h2, float rstd, uint32_t w2) {
  const float2 h = Traits<T>::to_float2(unpack2<T>(h2));
  return pack2<T>(__hmul2(Traits<T>::from_floats(h.x * rstd, h.y * rstd), unpack2<T>(w2)));
}

template <typename T>
__device__ __forceinline__ void sincos2(uint32_t theta_pair_bits, float &c0, float &s0, float &c1, float &s1) {
  const float2 th = Traits<T>::to_float2(unpack2<T>(theta_pair_bits));
  __sincosf(th.x, &s0, &c0);
  __sincosf(th.y, &s1, &c1);
}

// ------------------------------------------------------------------ rotation prologue of the small-M kernels
// One group's rotation metadata (paro_layout.h) as this lane uses it: its 4 channel scales and, for krot = 8, its pair-index
// and theta words of every stage -- fetched with the scales, so they fly during whatever the kernel waits for before x.
// Here and in rotation_tasks the block offsets meta_pairs_off(r), meta_theta_off(krot, r) and meta_scales_off(krot) are written
// out: through the helpers nvcc orders the address arithmetic differently and the fused kernels' SASS changes.
struct RotMeta {
  uint32_t idxw[8], tw[8];
  uint2 csw;
  const uint8_t *meta;
};

template <bool REGS8 = true>
__device__ __forceinline__ void fetch_meta(const uint8_t *meta, int krot, int lane, RotMeta &rm) {
  rm.meta = meta;
  rm.csw = *reinterpret_cast<const uint2 *>(meta + krot * 256 + 8 * lane);
  if (REGS8 && krot == 8) {
#pragma unroll
    for (int r = 0; r < 8; ++r) {
      rm.idxw[r] = *reinterpret_cast<const uint32_t *>(meta + r * 128 + 4 * lane);
      rm.tw[r] = *reinterpret_cast<const uint32_t *>(meta + 8 * 128 + r * 128 + 4 * lane);
    }
  }
}

// rows m0 .. m0 + nrows - 1 of a rotation tile into the group's B operand, B[k16 step s][k half h][row m][8 k]: NR rows x 16 bytes
// per core-matrix column, NR * 32 bytes per step (NR = 8 or 16; a literal 16 folds into the addressing)
template <typename T, int ROWS>
__device__ __forceinline__ void write_b_rows(uint32_t xb_group, uint32_t rot, int NR, int m0, int nrows, int lane) {
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
    sts128u(xb_group + s * (NR * 32) + h * (NR * 16) + (m >> 3) * 128 + (m & 7) * 16, v);
  }
}

// A warp's rotation tasks t = wi, wi + nwarps, ... < ntasks: task t is group gi = t / nq of the warp's groups (metadata block
// mi0 + gi of `meta`, meta_group_bytes each) x token rows m0 = ROWS * (t % nq) .. of `rows`.  The kernel's x loader
// stage_x(ROWS tag, gi, m0, csw) loads this lane's 4 channels of those rows after the kernel's x op and stages them in `rot`
// (scale_and_stage); here they go through the krot stages into group gi's B operand, xb + gi * NR * 256.  rm holds the first
// task's metadata, which the caller fetched ahead of its waits (fetch_meta<REGS8>).  REGS8: krot = 8 takes its stage words from
// rm's registers; without it every krot reads them in the stage loop (the MoE kernel: its tasks follow no wait to hide them
// behind, and the register path costs it ~15 registers and ~80 % more SASS).
template <typename T, int ROWS, bool REGS8, typename StageX>
__device__ __forceinline__ void rotation_tasks(RotMeta &rm, const uint8_t *meta, int meta_group_bytes, int krot, int mi0, int ntasks, int nq,
                                               int rows, int wi, int nwarps, int lane, uint32_t rot, uint32_t xb, int NR, StageX stage_x) {
  for (int t = wi; t < ntasks; t += nwarps) {
    const int gi = t / nq, m0 = (t - gi * nq) * ROWS;
    if (t != wi) fetch_meta<REGS8>(meta + static_cast<size_t>(mi0 + gi) * meta_group_bytes, krot, lane, rm);
    stage_x(std::integral_constant<int, ROWS>{}, gi, m0, rm.csw);
    __syncwarp();
    if (REGS8 && krot == 8) {
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
      for (int r = 0; r < krot; ++r) {
        const uint32_t iw = *reinterpret_cast<const uint32_t *>(rm.meta + r * 128 + 4 * lane);
        const uint32_t tw = *reinterpret_cast<const uint32_t *>(rm.meta + krot * 128 + r * 128 + 4 * lane);
        float c0, s0, c1, s1;
        sincos2<T>(tw, c0, s0, c1, s1);
        rotate_stage<T, ROWS>(rot, iw, c0, s0, c1, s1);
        __syncwarp();
      }
    }
    const int left = rows - m0;
    write_b_rows<T, ROWS>(xb + gi * (NR * 256), rot, NR, m0, left < ROWS ? left : ROWS, lane);
    __syncwarp();
  }
}

}  // namespace paro
