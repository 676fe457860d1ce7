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


COMBINE_REL = 2.0 ** -24


def check_combine(y: torch.Tensor, tok: torch.Tensor, w: torch.Tensor, ys: torch.Tensor, mag: torch.Tensor, what: str = "",
                  show: int = 6) -> float:
    """Element-wise check of a MoE block's output y [T, N] in T (include/paro_b200.h: paro_moe_forward).  One entry j per valid
    slot (a duplicate id is one entry per occurrence): tok[j] its token, w[j] its weight, ys[j] [N] the exact fp64 expert output
    sum_k xr[k] * W[k, n] and mag[j] [N] = sum_k |xr[k] * W[k, n]|.  The block computes v_j = T(fp32 sum, any order),
    p_j = fp32(v_j * w_j) and out[t] = T(fp32 sum of p_j from 0, any order).  With ref[t] = T(sum_j w_j ys[j]) in fp64:

      |v_j - ys_j|   <= ulp_T(T(ys_j)) + 2^-16 mag_j         (rounding of the fp32 sum to T, a flip at a binade edge included,
                                                              plus `check`'s bound on the fp32 sum)
      |S - sum w v|  <= n 2^-24 sum_j |w_j v_j|              (n fp32 roundings: n products, n - 1 adds; first order)
      |T(S) - ref|   <= ulp_T(ref) + |S - sum_j w_j ys_j|    (the two roundings to T, a tie flip included)

    so every element of a token with n valid slots must satisfy

      |out - ref| <= ulp_T(ref) + sum_j |w_j| (ulp_T(T(ys_j)) + 2^-16 mag_j) + (n + 1) 2^-24 sum_j |w_j ys_j|

    where the + 1 covers |v_j| > |ys_j| and the second-order terms.  A token with no valid slot must be exactly 0.  Raises
    AssertionError naming the violating elements as (token, column, 128-column block) with got / ref / tol; returns the
    largest err / tol."""
    dt = y.dtype
    T, N = y.shape
    dev = ys.device
    tok, wd = tok.to(dev).long(), w.to(dev).double()
    ys, mag = ys.double(), mag.double()
    z = lambda: torch.zeros(T, N, dtype=torch.float64, device=dev)
    exact = z().index_add_(0, tok, wd[:, None] * ys)
    slot_tol = z().index_add_(0, tok, wd.abs()[:, None] * (ulp(ys.to(dt), dt) + SUM_REL * mag))
    absum = z().index_add_(0, tok, (wd[:, None] * ys).abs())
    n = torch.bincount(tok, minlength=T).double()[:, None]
    ref = exact.to(dt)
    tol = ulp(ref, dt) + slot_tol + (n + 1) * COMBINE_REL * absum
    y2 = y.to(dev)
    err = (y2.double() - ref.double()).abs()
    empty = (n == 0).expand(T, N)
    bad = torch.where(empty, y2.double() != 0, ~(err <= tol))   # NaN / inf count as violations
    if bool(bad.any()):
        idx = bad.nonzero().tolist()
        lines = [f"  (token {t}, col {c}, block {c // 128}): got {float(y2[t, c]):.6g} ref {float(ref[t, c]):.6g} "
                 f"tol {'0 (no valid slot)' if bool(empty[t, c]) else format(float(tol[t, c]), '.3g')}" for t, c in idx[:show]]
        raise AssertionError(f"{what}: {len(idx)} of {bad.numel()} elements outside the element-wise bound\n" + "\n".join(lines))
    full = ~empty
    return float((err[full] / tol[full]).max()) if bool(full.any()) else 0.0


def check_moe(y: torch.Tensor, h: torch.Tensor, ids: torch.Tensor, w: torch.Tensor, experts, down, what: str = "") -> float:
    """`check_combine` for the output y [T, N] of a MoE block (ParoExperts `experts`, down rotation buffers `down`) from the
    block's own gate|up output h [T, k, 2I]: for every valid slot (t, s), act = the library's SiLU * up of h[t, s] (bit-identical
    to the down launch's operand), xr = act rotated by the standalone rotate kernel, ys = xr . W_d[e] in fp64 with W_d[e]
    expert e's dequantised down operand.  Ids outside [0, E) are dropped.  With `check` on h per expert, both launches are
    checked element-wise."""
    from paroquant_b200 import _cabi
    dev = h.device
    ids, w = ids.to(dev).long(), w.to(dev).float()
    Ld = down.to(dev)
    tok, ws, ys, mag = [], [], [], []
    valid = (ids >= 0) & (ids < experts.n_experts)
    for e in torch.unique(ids[valid]).tolist():
        rows, slot = (ids == e).nonzero(as_tuple=True)
        xr = rotated(Ld, _cabi.debug_silu_mul(h[rows, slot]))[0].double()
        Wd = experts.down[e].dense_weight().double()
        ys.append(xr @ Wd)
        mag.append(xr.abs() @ Wd.abs())
        tok.append(rows)
        ws.append(w[rows, slot])
        del Wd
    N = y.shape[1]
    if not tok:
        tok, ws = [torch.zeros(0, dtype=torch.long, device=dev)], [torch.zeros(0, device=dev)]
        ys = mag = [torch.zeros(0, N, dtype=torch.float64, device=dev)]
    return check_combine(y, torch.cat(tok), torch.cat(ws), torch.cat(ys), torch.cat(mag), what)
