// The streaming layout paro_prepack writes and both fused kernels read.  Host + device.
//
//   packed := [ rotation metadata ][ weight records ]
//
// Rotation metadata, one block per (partition p, group gk), groups of 128 channels (offsets: meta_pairs_off & co. below):
//   [r = 0..krot-1][128] uint8   pair indices: (i, j) of pair t at bytes 2t, 2t+1, always inside the 128-channel group
//   [r = 0..krot-1][ 64] T       theta, already cast to the activation dtype T (rotation.cu:75)
//   [128]                T       channel scales, cast to T (rotation.cu:76-78)
//   -> krot*256 + 256 bytes; lane l of the warp that owns the group reads 4 bytes of each stage's pair and theta rows
//   (pairs 2l and 2l + 1) and 8 bytes of the scales (channels 4l .. 4l + 3).  Every rotation path reads these blocks.
//
// Weight records.  N is cut into BLOCKS of 128 output columns per partition (a last partial block is
// zero-filled), K into the quantisation groups of 128 channels.  One record = one (block, group gk) =
// exactly what one dequant ROUND of either fused kernel consumes, and ONE cp.async.bulk (TMA) copy:
//   weights  [tile = 0..7][kh = 0..1][lane = 0..31] 16 bytes = 4 words: lane-private A fragments.  Word s is the whole
//            mma.m16n8k16 A fragment of lane (g = lane / 4, t = lane % 4) for row tile `tile` and k16 step 4 kh + s:
//            (w >> 4i) & 0x000F000F is register i, rows n = 128*block + 16*tile + g + 8*(i & 1), channels
//            kb + 2t + 8*(i >> 1) (low half) and + 1 (high half), kb = 128*gk + 16*(4 kh + s) -- the pair sits in the low
//            mantissa bits of a bf16x2 / half2 word.  A warp reads its (tile, k half) as one conflict-free 128-bit shared
//            load per lane, 512 contiguous bytes; the wgmma GEMM's warps read both k halves.           (8192 bytes)
//   scales   [128] T       s[gk][n], entry 16*tile + 2*g + hi for row 16*tile + g + 8*hi: a lane's two rows   (256 bytes)
//            are one 32-bit word
//   zeros    [128] uint8   z[gk][n], same order: a lane's two rows are one 16-bit word                        (128 bytes)
// -> 8576 bytes.  group_size 64 (the converter rotates AND quantises in groups of `group_size`, cli/convert.py:176-182):
// a record still covers 128 channels = TWO groups; it carries both groups' scales ([2][128] T at 8192) and then both
// groups' zeros ([2][128] uint8) -> 8960 bytes; the pair indices of the second group are stored + 64, which makes the two
// 64-channel rotations one 128-channel rotation of the same arithmetic (pairs never cross the halves).
// Records are ordered partition-major, then block, then group: the groups one CTA streams for a block are one
// contiguous byte range.  (Measured: a bulk copy costs ~90 SM cycles of
// issue whatever its size, so 8 x 1 KB pieces per round capped the stream at ~11 B/clk/SM.)
#pragma once

#include <stddef.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>

#include "../../include/paro_b200.h"

#if defined(__CUDACC__)
#define PARO_HD __host__ __device__
#else
#define PARO_HD
#endif

namespace paro {

constexpr int kGroup = 128;
constexpr int kBlockN = 128;               // output columns per block = rows of the weight operand per round
constexpr int kBlockWeightBytes = 8192;    // 128 columns x 128 channels of INT4
constexpr int kBlockScaleOff = 8192;        // [qhalves][128] T, then [qhalves][128] uint8 zeros
constexpr int kBlockBytes = 8192 + 256 + 128;      // group_size 128: one scale / zero set per record
constexpr int kBlockBytes64 = 8192 + 512 + 256;    // group_size 64: two
constexpr int kBlockBytesMax = kBlockBytes64;
PARO_HD constexpr int block_bytes(int qhalves) { return kBlockWeightBytes + qhalves * 384; }
PARO_HD constexpr int block_zero_off(int qhalves) { return kBlockScaleOff + qhalves * 256; }
// byte offset of lane `lane`'s 16-byte A-fragment chunk of (row tile, k half) inside a record
PARO_HD constexpr int frag_offset(int tile, int kh, int lane) { return ((tile * 2 + kh) * 32 + lane) * 16; }
// entry of block column `col` (0..127) in a scale / zero set: rows g and g + 8 of a 16-row tile side by side
PARO_HD constexpr int qparam_index(int col) { return (col & ~15) | ((col & 7) << 1) | ((col >> 3) & 1); }
// byte offsets inside one group's rotation metadata block: stage r's pair indices ([128] uint8) and theta ([64] T), the channel
// scales ([128] T)
PARO_HD constexpr int meta_pairs_off(int r) { return r * 128; }
PARO_HD constexpr int meta_theta_off(int krot, int r) { return krot * 128 + r * 128; }
PARO_HD constexpr int meta_scales_off(int krot) { return krot * 256; }

// Every kernel's parameters carry one.  The field order sets which ints ptxas loads from the parameter bank in pairs: this one
// keeps decode_kernel at 78 registers.
struct Layout {
  int K, N, n_parts;
  int groups;                               // K / 128: 128-channel record groups (each holds `qhalves` quantisation groups)
  int krot;
  int meta_group_bytes;                     // krot*256 + 256
  int rec_bytes, qhalves;                   // group_size 128: 8576, 1;  group_size 64: 8960, 2
  int blocks_total;                         // sum over partitions of ceil(size / 128)
  int dtype;
  int part_col_begin[PARO_MAX_PARTS + 1];   // first output column of each partition
  int part_block_begin[PARO_MAX_PARTS + 1]; // cumulative blocks per partition
  size_t meta_off, rec_off, total_bytes;

  PARO_HD size_t meta_offset(int part, int gk) const {
    return meta_off + (static_cast<size_t>(part) * groups + gk) * meta_group_bytes;
  }
  // record of (block index over all partitions, group)
  PARO_HD size_t record_offset(int block, int g) const {
    return rec_off + (static_cast<size_t>(block) * groups + g) * rec_bytes;
  }
};

// Returns false (and leaves `why` pointing at a static message) on an unsupported shape.
inline bool make_layout(const paro_linear_shape &s, Layout &L, const char **why) {
  static const char *msgs[] = {
      "group_size must be 64 or 128",
      "in_features must be a positive multiple of 128",
      "n_parts must be in 1..8",
      "every partition size must be a positive multiple of 16",
      "sum(part_sizes) != out_features",
      "krot must be in 1..16",
      "dtype must be PARO_F16 or PARO_BF16",
  };
  if (s.group_size != kGroup && s.group_size != 64) { *why = msgs[0]; return false; }
  if (s.in_features <= 0 || s.in_features % kGroup) { *why = msgs[1]; return false; }
  if (s.n_parts < 1 || s.n_parts > PARO_MAX_PARTS) { *why = msgs[2]; return false; }
  if (s.krot < 1 || s.krot > 16) { *why = msgs[5]; return false; }
  if (s.dtype != PARO_F16 && s.dtype != PARO_BF16) { *why = msgs[6]; return false; }
  L.K = s.in_features; L.N = s.out_features; L.krot = s.krot; L.n_parts = s.n_parts; L.dtype = s.dtype;
  L.groups = L.K / kGroup;
  L.qhalves = kGroup / s.group_size;
  L.rec_bytes = block_bytes(L.qhalves);
  int n = 0, nb = 0;
  L.part_col_begin[0] = 0;
  L.part_block_begin[0] = 0;
  for (int p = 0; p < s.n_parts; ++p) {
    if (s.part_sizes[p] <= 0 || s.part_sizes[p] % 16) { *why = msgs[3]; return false; }
    n += s.part_sizes[p];
    nb += (s.part_sizes[p] + kBlockN - 1) / kBlockN;
    L.part_col_begin[p + 1] = n;
    L.part_block_begin[p + 1] = nb;
  }
  for (int p = s.n_parts; p < PARO_MAX_PARTS; ++p) {
    L.part_col_begin[p + 1] = n;
    L.part_block_begin[p + 1] = nb;
  }
  if (n != s.out_features) { *why = msgs[4]; return false; }
  L.blocks_total = nb;
  L.meta_group_bytes = meta_scales_off(s.krot) + 256;
  L.meta_off = 0;
  size_t meta = static_cast<size_t>(s.n_parts) * L.groups * L.meta_group_bytes;
  L.rec_off = (meta + 127) / 128 * 128;
  L.total_bytes = L.rec_off + static_cast<size_t>(L.blocks_total) * L.groups * L.rec_bytes;
  return true;
}

// `count` units (CTAs, block ranges) dealt to the partitions in proportion to their 128-column blocks, at least one each
// (largest remainder): partition p gets begin[p] .. begin[p + 1] - 1.  False if count < n_parts.
inline bool apportion(const Layout &L, int count, int *begin) {
  int alloc[PARO_MAX_PARTS];
  double frac[PARO_MAX_PARTS];
  if (count < L.n_parts) return false;
  int used = 0;
  for (int p = 0; p < L.n_parts; ++p) {
    const double exact = static_cast<double>(count) * (L.part_block_begin[p + 1] - L.part_block_begin[p]) / L.blocks_total;
    alloc[p] = static_cast<int>(exact);
    if (alloc[p] < 1) alloc[p] = 1;
    frac[p] = exact - alloc[p];
    used += alloc[p];
  }
  while (used < count) {
    int best = 0;
    for (int p = 1; p < L.n_parts; ++p)
      if (frac[p] > frac[best]) best = p;
    alloc[best]++; frac[best] -= 1.0; used++;
  }
  while (used > count) {
    int best = -1;
    for (int p = 0; p < L.n_parts; ++p)
      if (alloc[p] > 1 && (best < 0 || frac[p] < frac[best])) best = p;
    if (best < 0) return false;
    alloc[best]--; frac[best] += 1.0; used--;
  }
  begin[0] = 0;
  for (int p = 0; p < PARO_MAX_PARTS; ++p) begin[p + 1] = begin[p] + (p < L.n_parts ? alloc[p] : 0);
  return true;
}

// A MoE block's two layouts (every expert's gate_up and down), the expert count, intermediate and hidden size.  moe_check_desc
// (paro_moe.cu) validates a paro_moe_desc into it for both MoE paths, with the error message set on failure.
struct MoeShapes { Layout gu, dn; int E, I, H; };
int moe_check_desc(const paro_moe_desc *d, MoeShapes &ms);

}  // namespace paro
