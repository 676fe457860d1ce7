"""Selection weights: checkpoint-format layers whose output is one exact product per element (a helper module: pytest does not
collect it).

Column n of a selection layer has exactly one non-zero weight, at input channel sigma(n) (a seeded permutation of the K
channels, shifted by `shift`), worth d_n * s with d_n in {+-1, +-2, +-4, -8} and s = 2^e (e in -2..2 by default) the fp16
scale of that (group, column); every (group, column) has a random zero z in 0..15 and q = z everywhere except the selected entry, q = z + d_n.
The layer is packed with oracle.np_awq_pack, independently of the library's prepack.  Every product x * d_n * s of a value in T
is exact in fp32 and every other term is an exact zero, so for any K split and any summation order

    y[m, n] = T(xr[m, sigma(n)] * d_n * s)

exactly, xr the rotated activations.  A misplaced nibble, zero or scale gives a second non-zero term or a wrong factor; a wrong
operand element of row m reaches every column that selects it.  Where N < K, `cover` gives the shifts of layers that together
select every channel.  The identity needs finite operands: one inf in a row of xr meets the exact zeros (inf * 0 = NaN), so
steps stacked in fp16 (a SiLU * up squares magnitudes) take a lower `exps` range.
"""
from __future__ import annotations

from dataclasses import dataclass

import numpy as np
import torch

from paroquant_b200.checkpoint import ParoLayerBuffers, make_synthetic_layer

_D = np.array([1, -1, 2, -2, 4, -4, -8])


@dataclass
class Selection:
    L: ParoLayerBuffers       # checkpoint-format buffers (rotation from make_synthetic_layer, selection weights)
    sigma: torch.Tensor       # [N] int64: the input channel column n selects
    w: torch.Tensor           # [N] fp32: d_n * s, the selected weight (exact in fp16 and bf16)

    def apply(self, xr_parts, dtype: torch.dtype) -> torch.Tensor:
        """y [M, N] in T from the rotated activations [M, K] of every partition: T(xr[m, sigma(n)] * w_n), fp32 product (exact)."""
        out, n0 = [], 0
        for xr, n in zip(xr_parts, self.L.part_sizes):
            sig, w = self.sigma[n0:n0 + n].to(xr.device), self.w[n0:n0 + n].to(xr.device)
            out.append((xr.float()[:, sig] * w).to(dtype))
            n0 += n
        return torch.cat(out, -1)

    def exact(self, xr_parts) -> torch.Tensor:
        """The same products in fp64 (exact), before the rounding to T: expert outputs for gpu_reference.check_combine."""
        out, n0 = [], 0
        for xr, n in zip(xr_parts, self.L.part_sizes):
            sig, w = self.sigma[n0:n0 + n].to(xr.device), self.w[n0:n0 + n].to(xr.device)
            out.append(xr.double()[:, sig] * w.double())
            n0 += n
        return torch.cat(out, -1)


def cover(K: int, N: int) -> list[int]:
    """Shifts of sigma for layers that together select every one of the K channels."""
    return list(range(0, K, N)) if N < K else [0]


def selection_layer(K: int, parts, *, group: int = 128, krot: int = 8, seed: int = 0, shift: int = 0, rotation: ParoLayerBuffers | None = None,
                    bias: bool = False, theta_uniform_pi: bool = False, exps: tuple[int, int] = (-2, 2)) -> Selection:
    """A selection layer on the CPU.  The rotation (theta, pairs, channel scales) and bias are make_synthetic_layer's for `seed`,
    or `rotation`'s (the layers of one MoE projection share one); the weights come from `seed` and sigma from `seed` and `shift`."""
    from oracle import oracle as O
    parts = [int(p) for p in parts]
    N, ng = sum(parts), K // group
    rot = rotation if rotation is not None else make_synthetic_layer(K, parts, group_size=group, krot=krot, seed=seed, bias=bias,
                                                                     theta_uniform_pi=theta_uniform_pi)
    rng = np.random.default_rng(seed)
    sigma = np.random.default_rng(seed + 7919).permutation(K)[(np.arange(N) + shift) % K]
    d = _D[rng.integers(0, len(_D), N)]
    e = rng.integers(exps[0], exps[1] + 1, (ng, N))
    z = rng.integers(0, 16, (ng, N))
    cols = np.arange(N)
    gsel = sigma // group
    z[gsel, cols] = rng.integers(np.maximum(0, -d), np.minimum(15, 15 - d) + 1)    # z + d in 0..15
    qweight = np.empty((K, N // 8), np.int32)
    for r0 in range(0, K, group):                         # one group of rows at a time: bounded host memory
        q = np.repeat(z[r0 // group][None], group, axis=0).astype(np.uint8)
        hit = (sigma >= r0) & (sigma < r0 + group)
        q[sigma[hit] - r0, cols[hit]] += d[hit].astype(np.uint8)
        qweight[r0:r0 + group] = O.np_awq_pack(q)
    qzeros = O.np_awq_pack(z.astype(np.uint8))
    scales = torch.from_numpy(np.exp2(e).astype(np.float16))
    L = ParoLayerBuffers(torch.from_numpy(qweight), torch.from_numpy(qzeros), scales, rot.theta, rot.pairs, rot.channel_scales, parts,
                         group, rot.bias if rotation is None else None)
    w = torch.from_numpy((d * np.exp2(e[gsel, cols])).astype(np.float32))
    return Selection(L, torch.from_numpy(sigma.astype(np.int64)), w)
