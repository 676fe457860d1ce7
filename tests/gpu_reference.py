"""Element-wise check of a fused linear's output against an fp64 reference (a helper module: pytest does not collect it).

The fused kernels compute y[m, n] = T(sum_k x_rot[m, k] * W[k, n]) with fp32 accumulation, then add the bias in T.  The
rotated activations (the standalone rotate kernel) and the dequantised operand (`dense_weight()`) are both checked bit for
bit elsewhere, so what is left is the fp32 summation order and the rounding to T.  Every element must satisfy

    |y - ref| <= ulp_T(ref_pre) [+ ulp_T(ref) with a bias] + 2^-16 * sum_k |x_rot[m, k] * W[k, n]|

with ref_pre = T(fp64 sum) and ref = T(ref_pre + bias) (= ref_pre without a bias).  The ulp terms cover each rounding to T
and a tie flip (the bias adds a second rounding, and a flip of the first one moves the sum by ulp_T(ref_pre), which exceeds
ulp_T(ref) where the bias cancels the product).  The last term covers any fp32 summation order with a margin of about 8x
over tensor-core fp32 accumulation at K = 14336.  A normwise bound averages over the whole output; this one catches a
single wrong element, e.g. one 16-column fragment of one row or a group dropped from one K slice of one column block.
"""
from __future__ import annotations

import torch

SUM_REL = 2.0 ** -16
_MANT_BITS = {torch.bfloat16: 7, torch.float16: 10}
_MIN_NORMAL_EXP = {torch.bfloat16: -126, torch.float16: -14}


def ulp(v: torch.Tensor, dtype: torch.dtype) -> torch.Tensor:
    """Spacing of `dtype` values at |v| (float64 in, float64 out); subnormals have the spacing of the smallest normal."""
    a = v.abs().double()
    _, e = torch.frexp(a)                                     # |v| = mant * 2^e, mant in [0.5, 1)
    e = torch.where(a > 0, e.double() - 1, float(_MIN_NORMAL_EXP[dtype])).clamp(min=_MIN_NORMAL_EXP[dtype])
    return torch.exp2(e - _MANT_BITS[dtype])


def check(y: torch.Tensor, xr_parts, W: torch.Tensor, part_sizes, bias: torch.Tensor | None = None, what: str = "",
          sum_rel: float = SUM_REL, show: int = 6) -> float:
    """y [M, N] in T; xr_parts: the rotated activations [M, K] of every partition; W [K, N] the dequantised operand; bias [N]
    or [M, N] in T, or None.  Raises AssertionError naming the violating elements as (row, column, 128-column block of its
    partition, partition) with got / ref / tol; returns the largest err / tol."""
    dt = y.dtype
    refs, mags = [], []
    n0 = 0
    for xr, n in zip(xr_parts, part_sizes):
        Wp = W[:, n0:n0 + n].double()
        xd = xr.reshape(-1, xr.shape[-1]).double()
        refs.append(xd @ Wp)
        mags.append(xd.abs() @ Wp.abs())
        n0 += n
    exact, mag = torch.cat(refs, -1), torch.cat(mags, -1)
    ref_pre = exact.to(dt)
    tol = ulp(ref_pre, dt) + sum_rel * mag
    ref = ref_pre
    if bias is not None:
        ref = (ref_pre.float() + bias.float()).to(dt)
        tol = tol + ulp(ref, dt)
    y2 = y.reshape(ref.shape)
    err = (y2.double() - ref.double()).abs()
    bad = ~(err <= tol)                                       # NaN / inf in y count as violations
    if bool(bad.any()):
        bounds = torch.tensor([0] + list(part_sizes)).cumsum(0).tolist()
        idx = bad.nonzero().tolist()
        lines = []
        for m, n in idx[:show]:
            p = max(i for i in range(len(part_sizes)) if bounds[i] <= n)
            lines.append(f"  (row {m}, col {n}, block {(n - bounds[p]) // 128}, part {p}): got {float(y2[m, n]):.6g} "
                         f"ref {float(ref[m, n]):.6g} tol {float(tol[m, n]):.3g}")
        raise AssertionError(f"{what}: {len(idx)} of {bad.numel()} elements outside the element-wise bound\n" + "\n".join(lines))
    return float((err / tol).max())


def rotated(L, x: torch.Tensor) -> list[torch.Tensor]:
    """x rotated for every partition of layer buffers L (on x's device) by the standalone rotate kernel."""
    import paroquant_b200.kernels.cuda  # noqa: F401  registers torch.ops.rotation.rotate
    return [torch.ops.rotation.rotate(x, L.pairs[p], L.theta[p], L.channel_scales[p], L.group_size) for p in range(len(L.part_sizes))]


def check_linear(k, L, x: torch.Tensor, y: torch.Tensor, bias: torch.Tensor | None = None, W: torch.Tensor | None = None,
                 what: str = "") -> float:
    """`check` for the output y of ParoLinearKernel k (layer buffers L on the GPU) on input x: the reference rotates x with the
    standalone rotate kernel and multiplies with k's own dequantised operand (pass W to reuse one)."""
    return check(y, rotated(L, x), k.dense_weight() if W is None else W, L.part_sizes, bias, what)
