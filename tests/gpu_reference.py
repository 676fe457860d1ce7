"""Element-wise check of a fused linear's output against an fp64 reference (a helper module: pytest does not collect it).

The fused kernels compute y[m, n] = T(sum_k x_rot[m, k] * W[k, n]) with fp32 accumulation, then add the bias in T.  The
rotated activations (the standalone rotate kernel) and the dequantised operand (`dense_weight()`) are both pinned bit for bit:
the rotate op equals `exact_rotate` -- oracle.np_rotate on the GPU's own sin / cos table, which is bounded against fp64 -- on
every dtype, shape and edge value (tests/test_gpu_rotation_exact.py), and `dense_weight()` equals oracle.c_dequant at every
shape this suite uses it for (tests/test_gpu_selection_exact.py, which also checks every fused kernel's own rotated operand
bit for bit through selection weights).  So what is left is the fp32 summation order and the rounding to T.  Every element
must satisfy

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


def linear_bound(xr_parts, W: torch.Tensor, part_sizes, dt: torch.dtype, bias: torch.Tensor | None = None,
                 sum_rel: float = SUM_REL) -> tuple[torch.Tensor, torch.Tensor]:
    """(ref, tol) of `check`: ref [M, N] in T, tol [M, N] in float64."""
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
    return ref, tol


def _assert_within(y: torch.Tensor, ref: torch.Tensor, tol: torch.Tensor, part_sizes, what: str, show: int) -> float:
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


def check(y: torch.Tensor, xr_parts, W: torch.Tensor, part_sizes, bias: torch.Tensor | None = None, what: str = "",
          sum_rel: float = SUM_REL, show: int = 6) -> float:
    """y [M, N] in T; xr_parts: the rotated activations [M, K] of every partition; W [K, N] the dequantised operand; bias [N]
    or [M, N] in T, or None.  Raises AssertionError naming the violating elements as (row, column, 128-column block of its
    partition, partition) with got / ref / tol; returns the largest err / tol."""
    ref, tol = linear_bound(xr_parts, W, part_sizes, y.dtype, bias, sum_rel)
    return _assert_within(y, ref, tol, part_sizes, what, show)


def check_residual(h: torch.Tensor, t: tuple[torch.Tensor, torch.Tensor], r: torch.Tensor, what: str = "", show: int = 6) -> float:
    """The residual stream h = T(t + r) [M, N] of an ADD_RESIDUAL epilogue whose linear output t is not stored.  t = (ref_t,
    tol_t) of `linear_bound` for that linear, r the residual input in T.  t itself satisfies |t - ref_t| <= tol_t, and the
    kernel and the reference each round t + r once to T, so every element must satisfy

        |h - T(ref_t + r)| <= ulp_T(max(|h|, |T(ref_t + r)|)) + tol_t

    (the ulp term is the two half-ulp roundings, taken in the larger binade when they straddle a power of two)."""
    ref_t, tol_t = t
    ref = (ref_t.float() + r.reshape(ref_t.shape).float()).to(h.dtype)
    big = torch.maximum(h.reshape(ref.shape).double().abs(), ref.double().abs())
    return _assert_within(h, ref, ulp(big, h.dtype) + tol_t, [ref.shape[1]], what, show)


def check_residual_linear(k, L, x: torch.Tensor, h: torch.Tensor, r: torch.Tensor, bias: torch.Tensor | None = None,
                          W: torch.Tensor | None = None, what: str = "") -> float:
    """`check_residual` for ParoLinearKernel k (layer buffers L on the GPU) on input x: h = T(k(x, bias) + r)."""
    t = linear_bound(rotated(L, x), k.dense_weight() if W is None else W, L.part_sizes, h.dtype, bias)
    return check_residual(h, t, r, what)


# ---- RMSNorm statistics
RSTD_ULPS = 16


def _nudge(v: torch.Tensor, ulps: int) -> torch.Tensor:
    """fp32 v (all positive, normal) moved by `ulps` fp32 spacings."""
    return (v.view(torch.int32) + ulps).view(torch.float32)


def rms_operand(h: torch.Tensor, rstd: torch.Tensor, w: torch.Tensor | None) -> torch.Tensor:
    """The RMSNORM x op for rstd [M] in fp32: T(T(h * rstd) * w) (T(h * rstd) without w), every product in fp32."""
    n = (h.float() * rstd.float()[:, None]).to(h.dtype)
    return n if w is None else (n.float() * w.float()).to(h.dtype)


def rms_candidates(h: torch.Tensor, w: torch.Tensor, eps: float, ulps: int = RSTD_ULPS) -> tuple[torch.Tensor, torch.Tensor]:
    """Every operand the RMSNORM x op can produce from h [M, K] in T: the kernel adds the fp32 h^2 in its own order and forms
    rstd with fast division and rsqrtf, so its rstd is within a few fp32 ulps of r = fp32(1 / sqrt(mean(h^2) + eps)) (mean in
    fp64).  The operand is a step function of rstd, so the fp32 values r - ulps .. r + ulps give every operand it can produce.
    Returns (xs [R, K] in T, owner [R]): the distinct candidate rows and the row of h each belongs to; row m's first candidate
    is the one of r itself (oracle.rms_norm's operand)."""
    var = (h.double() ** 2).mean(-1)
    r = (1.0 / torch.sqrt(var + eps)).float()
    xs, owner = [rms_operand(h, r, w)], [torch.arange(h.shape[0], device=h.device)]
    seen = xs[0].clone()[:, None, :]                                           # [M, distinct so far, K]
    for i in [d for u in range(1, ulps + 1) for d in (-u, u)]:
        xi = rms_operand(h, _nudge(r, i), w)
        new = ~(seen == xi[:, None, :]).all(-1).any(-1)
        if bool(new.any()):
            rows = new.nonzero()[:, 0]
            xs.append(xi[rows])
            owner.append(rows)
            seen = torch.cat([seen, torch.where(new[:, None], xi, xs[0])[:, None, :]], 1)
    return torch.cat(xs), torch.cat(owner)


def check_rmsnorm(y: torch.Tensor, h: torch.Tensor, w: torch.Tensor, eps: float, rotate, W: torch.Tensor, part_sizes,
                  bias: torch.Tensor | None = None, what: str = "", show: int = 6) -> float:
    """`check` at full strength for the output y [M, N] of an RMSNORM step on random data, where the operand depends on the
    last fp32 bits of rstd: each row must satisfy `check`'s bound for at least one of its `rms_candidates` (h: the step's
    input in T, the GPU's own previous stage; rotate(x) -> the rotated activations of every partition).  A wrong statistics
    word (a missing block, a neighbour row's partial) moves rstd by far more than RSTD_ULPS and fails every candidate.
    Raises AssertionError naming the failing rows with the elements their first candidate violates; returns, over the rows,
    the largest of the best candidate's err / tol."""
    xs, owner = rms_candidates(h, w, eps)
    ref, tol = linear_bound(rotate(xs), W, part_sizes, y.dtype, bias)
    M = y.shape[0]
    y2 = y.reshape(M, -1)[owner]
    ratio = ((y2.double() - ref.double()).abs() / tol).nan_to_num(nan=float("inf")).amax(-1)   # [R]
    best = torch.full((M,), float("inf"), dtype=torch.float64, device=ratio.device).scatter_reduce(0, owner, ratio, "amin")
    if bool((~(best <= 1.0)).any()):
        bad = (~(best <= 1.0)).nonzero()[:, 0].tolist()
        first = [int((owner == m).nonzero()[0, 0]) for m in bad[:show]]
        detail = ""
        try:
            _assert_within(y2[first], ref[first], tol[first], part_sizes, "", show)
        except AssertionError as e:
            detail = str(e).split("\n", 1)[1]
        raise AssertionError(f"{what}: {len(bad)} of {M} rows outside the element-wise bound for every rstd within "
                             f"{RSTD_ULPS} fp32 ulps (rows {bad[:show]}); first candidate of the rows shown, as positions "
                             f"among them:\n{detail}")
    return float(best.max())


def check_rmsnorm_linear(k, L, h: torch.Tensor, w: torch.Tensor, eps: float, y: torch.Tensor, bias: torch.Tensor | None = None,
                         W: torch.Tensor | None = None, what: str = "") -> float:
    """`check_rmsnorm` for ParoLinearKernel k (layer buffers L on the GPU): y = k(RMSNorm(h) * w)."""
    return check_rmsnorm(y, h, w, eps, lambda x: rotated(L, x), k.dense_weight() if W is None else W, L.part_sizes, bias, what)


# exact-statistics rows: every value is +-2^j * c with c in {1.5, 0.5} (3/8 and 5/8 of a uniform row), times COLD off the hot
# block of an energy-concentrated row
_COLD = 2.0 ** -3


def exact_rms_rows(M: int, K: int, dtype: torch.dtype, seed: int, w: torch.Tensor | None = None, eps: float = 1e-8,
                   hot=None, ulps: int = 4) -> tuple[torch.Tensor, torch.Tensor]:
    """Residual rows h [M, K] in T (on the CPU) whose RMSNorm operand is known exactly, and that operand T(T(h * rstd) * w)
    (T(h * rstd) without w).  Row m is +-2^j_m * c_k with 3/8 of the c 1.5 and 5/8 0.5 in a per-row permutation and signs,
    j_m in {0, 1, 2}.  Every value is a multiple of u = 2^(j_m - 1) (2^(j_m - 4) in a hot row) and a row's sum of h^2 is below
    2^16 u^2, so every partial sum is exact in fp32 in any order.  A uniform row (hot[m] = -1) has mean square 4^j_m exactly: rstd = 2^-j_m up to the ulps of fast
    division and rsqrtf, and T(h * rstd) = +-c whatever those ulps.  A row with hot[m] = b keeps the scale only in 128-column
    block b and multiplies the rest by 2^-3: block b then holds half or more of the row's energy, so any one 32-column
    statistics word of it dropped or counted twice moves the operand (asserted here, row by row).  Every row is also asserted
    to give the same operand for every fp32 rstd within `ulps` ulps of the fp64 value; a row that does not is drawn again.
    hot: [M] block indices or -1; default: every third row uniform, the others hot in a seed-dependent block.
    Values are multiples of 2^-4 below 8, so h - b is exact in T for any bias b in {+-4, +-8} (`exact_bias`)."""
    assert K % 128 == 0
    nb = K // 128
    g = torch.Generator().manual_seed(seed)
    if hot is None:
        hot = [-1 if (m + seed) % 3 == 0 else (seed * 7 + m * 5) % nb for m in range(M)]
    hot = [int(b) for b in hot]
    assert len(hot) == M and all(-1 <= b < nb for b in hot)
    base = torch.full((K,), 0.5, dtype=torch.float64)
    base[: 3 * K // 8] = 1.5
    rows, ops = [], []
    wf = None if w is None else w.cpu()
    for m in range(M):
        for _attempt in range(20):
            c = base[torch.randperm(K, generator=g)] * (torch.randint(0, 2, (K,), generator=g) * 2 - 1)
            j = int(torch.randint(0, 3, (1,), generator=g))
            v = c * 2.0 ** j
            u = 2.0 ** (j - 1) * (_COLD if hot[m] >= 0 else 1.0)        # every value is a multiple of u
            if hot[m] >= 0:
                cold = torch.ones(K, dtype=torch.bool)
                cold[128 * hot[m]:128 * hot[m] + 128] = False
                v[cold] *= _COLD
            h = v.to(dtype)
            assert torch.equal(h.double(), v)
            sq = v * v
            s = float(sq.sum())
            assert s < 2.0 ** 24 * u * u and torch.equal(torch.fmod(sq / (u * u), 1.0), torch.zeros(K, dtype=torch.float64))
            r64 = 1.0 / (s / K + eps) ** 0.5
            r = torch.tensor([r64], dtype=torch.float32)
            x = rms_operand(h[None], r, wf)[0]
            if not all(torch.equal(rms_operand(h[None], _nudge(r, d), wf)[0], x) for d in range(-ulps, ulps + 1)):
                continue                                          # an operand element within `ulps` of a rounding edge
            if hot[m] >= 0:
                for q in range(4):                                 # one 32-column word of the hot block dropped or doubled
                    a = 128 * hot[m] + 32 * q
                    share = float(sq[a:a + 32].sum())
                    for s2 in (s - share, s + share):
                        r2 = torch.tensor([1.0 / (s2 / K + eps) ** 0.5], dtype=torch.float32)
                        assert not torch.equal(rms_operand(h[None], r2, wf)[0], x), (m, hot[m], q)
            rows.append(h)
            ops.append(x)
            break
        else:
            raise AssertionError(f"exact_rms_rows: row {m} found no draw whose operand is robust to {ulps} ulps of rstd")
    return torch.stack(rows), torch.stack(ops)


def exact_bias(N: int, seed: int, dtype: torch.dtype) -> torch.Tensor:
    """A bias of +-4 / +-8: with h from `exact_rms_rows`, r = h - bias is exact in T and T(bias + r) = h."""
    g = torch.Generator().manual_seed(seed)
    return (torch.tensor([4.0, 8.0])[torch.randint(0, 2, (N,), generator=g)] * (torch.randint(0, 2, (N,), generator=g) * 2 - 1)).to(dtype)


def rotated(L, x: torch.Tensor) -> list[torch.Tensor]:
    """x rotated for every partition of layer buffers L (on x's device) by the standalone rotate kernel (equal, value for value,
    to `exact_rotate` on every dtype, shape and edge value: tests/test_gpu_rotation_exact.py)."""
    import paroquant_b200.kernels.cuda  # noqa: F401  registers torch.ops.rotation.rotate
    return [torch.ops.rotation.rotate(x, L.pairs[p], L.theta[p], L.channel_scales[p], L.group_size) for p in range(len(L.part_sizes))]


# ---- exact restatement of the rotation on the GPU's own sin / cos
_ODT = {torch.float32: "float32", torch.float16: "float16", torch.bfloat16: "bfloat16"}
# CUDA's documented maximum absolute errors for |x| <= pi (CUDA Math API, intrinsic functions): __sinf 2^-21.41, __cosf 2^-21.19
# -- cos has the looser bound, and the H100 reaches past 2^-21.41 on it (2^-21.29 over the fp16 angles)
SIN_ABS, COS_ABS = 2.0 ** -21.41, 2.0 ** -21.19


def kernel_sincos(theta: torch.Tensor) -> tuple[torch.Tensor, torch.Tensor]:
    """(c, s) = __sincosf(theta) exactly as the kernels compute it, fp32 of theta's shape on the GPU.  Every kernel takes sin / cos
    of float(theta as it reads it) -- T(theta) in the fused kernels and the half / bf16 rotate op, the raw value in the fp32 op
    -- so pass theta already rounded to T, as fp32 values.  One fp32 rotate launch, krot = 1, no scales, identity pairs (pair t
    of a group is channels (2t, 2t + 1)), x = 1 on every i channel and 0 on every j channel: out_i = fmaf(c, 1, s * 0) = c and
    out_j = fmaf(c, 0, s * -1) = -s.  tests/test_gpu_rotation_exact.py bounds the table against fp64."""
    import paroquant_b200.kernels.cuda  # noqa: F401  registers torch.ops.rotation.rotate
    flat = theta.detach().to("cuda", torch.float32).reshape(-1)
    n = flat.numel()
    pad = (-n) % 64                                           # whole 128-channel groups
    th = torch.cat([flat, flat.new_zeros(pad)])[None]
    ch = 2 * th.shape[1]
    x = torch.zeros(1, ch, device="cuda")
    x[0, 0::2] = 1.0
    pairs = (torch.arange(ch, device="cuda") % 128).to(torch.int16)[None]
    out = torch.ops.rotation.rotate(x, pairs, th, None, 128)[0]
    return out[0::2][:n].reshape(theta.shape), (-out[1::2][:n]).reshape(theta.shape)


def exact_rotate(x: torch.Tensor, pairs: torch.Tensor, theta: torch.Tensor, scales: torch.Tensor | None, group: int) -> torch.Tensor:
    """The rotate op's result for x [.., K] in T (T = x.dtype), restated on the CPU by oracle.np_rotate -- error-free fp32 FMA,
    every rounding point of the kernels -- with the GPU's own sin / cos (`kernel_sincos` of T(theta)): the one input taken from
    the GPU, bounded against fp64 on its own.  theta [krot, K/2] and scales [K] / [1, K] in any float dtype, read as the kernels
    read them.  Returns x's shape and dtype on x's device."""
    from oracle import oracle as O
    dt = _ODT[x.dtype]
    th = theta.detach().float().cpu().numpy()
    c, s = kernel_sincos(torch.from_numpy(O.round_to(th, dt)))
    sc = None if scales is None else scales.detach().float().cpu().numpy()
    out = O.np_rotate(x.detach().float().cpu().numpy(), pairs.detach().cpu().numpy(), th, sc, group, dt,
                      sincos=(c.cpu().numpy(), s.cpu().numpy()))
    return torch.from_numpy(out).to(x.dtype).to(x.device)


def exact_rotated(L, x: torch.Tensor) -> list[torch.Tensor]:
    """`rotated` restated exactly: x [M, K] in T for every partition of layer buffers L, by `exact_rotate`."""
    return [exact_rotate(x, L.pairs[p], L.theta[p], L.channel_scales[p], L.group_size) for p in range(len(L.part_sizes))]


def sample_rows(M: int, block: int, seed: int, n: int = 64) -> torch.Tensor:
    """Rows a CPU restatement looks at: all of them up to 64; above, the first 16, every row of the last `block`-row block and n
    seeded random rows (sorted, distinct)."""
    if M <= 64:
        return torch.arange(M)
    g = torch.Generator().manual_seed(seed)
    last = torch.arange((M - 1) // block * block, M)
    return torch.unique(torch.cat([torch.arange(16), last, torch.randint(0, M, (n,), generator=g)]))


def assert_same_values(got: torch.Tensor, ref: torch.Tensor, what: str = "", show: int = 6) -> None:
    """got == ref as values: +0 == -0, NaN where and only where ref has NaN, inf as inf; nothing else may differ."""
    g, r = got.reshape(ref.shape), ref
    same = (g == r) | (torch.isnan(g) & torch.isnan(r))
    if not bool(same.all()):
        idx = (~same).nonzero().tolist()
        lines = [f"  {tuple(i)}: got {float(g[tuple(i)])!r} ref {float(r[tuple(i)])!r}" for i in idx[:show]]
        raise AssertionError(f"{what}: {len(idx)} of {same.numel()} elements differ\n" + "\n".join(lines))


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


# ---- the rotate op's backward (paro_rotate_backward)
U32 = 2.0 ** -24                  # fp32 unit roundoff
FTZ_PER_ROW = 2.0 ** -125         # the kernel flushes fp32 subnormals: two flushed products of at most 2^-126 each per row
_F64_SUM = 2.0 ** -52             # torch's fp64 row sums of exact products, per row (far below one fp32 step)


def backward_restated(x: torch.Tensor, pairs: torch.Tensor, theta: torch.Tensor, y: torch.Tensor, grad_out: torch.Tensor,
                      scales: torch.Tensor | None, group: int) -> dict:
    """The rotate op's backward restated, for x, y = rotate(x), grad_out [M, K] in T on the GPU.  The stage values come from
    the reference's walk (autograd.py:20-61): from rotation krot - 1 down to 0, t and g are un-rotated by one-rotation rotate-op
    launches with -theta, which round them to T where the fused kernel does (the rotate op equals `exact_rotate` value for value).
    Every product of two stage values, or of x and g, is a product of fp32 values and so exact in fp64.  Returns, on y's device:

      grad_x      T(fp32(g * scale as stored)) (g without scales), [M, K] in T
      S, D        per rotation and pair, sum_rows (g_i t_j - g_j t_i) and sum_rows (g_i t_i + g_j t_j) in fp64, [krot, K / 2]
      A, B        their magnitudes sum_rows |g_i t_j| + |g_j t_i| and sum_rows |g_i t_i| + |g_j t_j|
      xg, xg_abs  sum_rows x g and sum_rows |x g| per channel in fp64, [K] (None without scales)

    The pair slots are group-relative, as the op takes them."""
    import paroquant_b200.kernels.cuda  # noqa: F401  registers torch.ops.rotation.rotate
    krot, K = pairs.shape
    rows = y.numel() // K
    t, g = y.reshape(rows, K).contiguous(), grad_out.reshape(rows, K).contiguous()
    base = (torch.arange(K, device=y.device) // group * group).view(K // 2, 2)[:, 0]
    out = {k: torch.zeros(krot, K // 2, dtype=torch.float64, device=y.device) for k in "SDAB"}
    for r in reversed(range(krot)):
        pr = pairs[r].view(K // 2, 2).long()
        ci, cj = pr[:, 0] + base, pr[:, 1] + base
        gi, gj, ti, tj = g[:, ci].double(), g[:, cj].double(), t[:, ci].double(), t[:, cj].double()
        a, b, c, d = gi * tj, gj * ti, gi * ti, gj * tj
        out["S"][r], out["D"][r] = (a - b).sum(0), (c + d).sum(0)
        out["A"][r], out["B"][r] = (a.abs() + b.abs()).sum(0), (c.abs() + d.abs()).sum(0)
        del gi, gj, ti, tj, a, b, c, d
        inv = -theta[r:r + 1]
        t = torch.ops.rotation.rotate(t, pairs[r:r + 1], inv, None, group)
        g = torch.ops.rotation.rotate(g, pairs[r:r + 1], inv, None, group)
    if scales is None:
        out["grad_x"], out["xg"], out["xg_abs"] = g, None, None
    else:
        out["grad_x"] = (g.float() * scales.float().reshape(-1)).to(y.dtype)
        xg = x.reshape(rows, K).double() * g.double()
        out["xg"], out["xg_abs"] = xg.sum(0), xg.abs().sum(0)
    out["rows"] = rows
    return out


def backward_depths(max_blocks: int, splits: int) -> tuple[int, int]:
    """The fp32 steps a term of the backward's row sums goes through, for a plan whose warps walk at most `max_blocks` row blocks
    of 4 rows and whose `splits` warp partials per entry are added with fp32 atomics (paro_debug_rotate_backward_plan).
    grad_theta: 2 for the product difference, 3 within a 4-row block, one per block in the warp's running sum, one per atomic.
    grad_scale: 1 for the product, one per row in the warp's running sum (4 per block), one per atomic."""
    return 5 + max_blocks + splits, 1 + 4 * max_blocks + splits


def _gamma(d: int) -> float:
    return d * U32 / (1 - d * U32)


def _assert_entries(got: torch.Tensor, ref: torch.Tensor, tol: torch.Tensor, keep: torch.Tensor, label, what: str, show: int) -> float:
    err = (got.double() - ref).abs()
    bad = keep & ~(err <= tol)                                # NaN / inf in got count as violations
    if bool(bad.any()):
        idx = bad.nonzero().tolist()
        lines = [f"  ({label(*i)}): got {float(got[tuple(i)]):.9g} ref {float(ref[tuple(i)]):.9g} tol {float(tol[tuple(i)]):.3g}"
                 for i in idx[:show]]
        raise AssertionError(f"{what}: {len(idx)} of {int(keep.sum())} entries outside the element-wise bound\n" + "\n".join(lines))
    return float((err[keep] / tol[keep]).max()) if bool(keep.any()) else 0.0


def check_backward_theta(got: torch.Tensor, ref: dict, c: torch.Tensor, s: torch.Tensor, group: int, max_blocks: int, splits: int,
                         reference_formula: bool = False, skip_groups=(), cast: torch.dtype | None = None, what: str = "",
                         show: int = 6) -> float:
    """grad_theta [krot, K / 2] of the fused backward against `backward_restated`'s sums.  With d = backward_depths(...)[0] and
    M rows, every entry must satisfy

        gradient:              |got - S| <= gamma_d A + 2^-125 M
        reference expression:  |got - (c S + s D)| <= gamma_(d+2) (|c| A + |s| B) + 2^-124 M

    (gamma_d = d u / (1 - d u), u = 2^-24; the M terms cover flushed subnormal products and, far below them, the fp64 sums).
    (c, s) [krot, K / 2] is the kernel's own __sincosf(-T(theta)) (`kernel_sincos`); the expression's two extra steps are its
    product and sum.  cast: the dtype grad_theta was cast to after the sum (autograd returns it in theta's dtype): one more
    rounding, ulp_cast(got).  Entries of `skip_groups` are not checked; every other entry must be finite.  Raises AssertionError
    naming the violating entries as (rotation, group, pair) with got / ref / tol; returns the largest err / tol."""
    dev = ref["S"].device
    d = backward_depths(max_blocks, splits)[0]
    rows = ref["rows"]
    if reference_formula:
        cd, sd = c.to(dev).double(), s.to(dev).double()
        exact = cd * ref["S"] + sd * ref["D"]
        tol = _gamma(d + 2) * (cd.abs() * ref["A"] + sd.abs() * ref["B"]) + 2 * FTZ_PER_ROW * rows
    else:
        exact = ref["S"]
        tol = _gamma(d) * ref["A"] + FTZ_PER_ROW * rows
    tol = tol + _F64_SUM * rows * (ref["A"] + ref["B"])
    got = got.to(dev)
    if cast is not None:
        tol = tol + ulp(got, cast)
    per = group // 2
    keep = torch.ones_like(exact, dtype=torch.bool)
    for gr in skip_groups:
        keep[:, gr * per:(gr + 1) * per] = False
    return _assert_entries(got, exact, tol, keep, lambda r, p: f"rotation {r}, group {p // per}, pair {p % per}", what, show)


def check_backward_scale(got: torch.Tensor, ref: dict, group: int, max_blocks: int, splits: int, skip_groups=(),
                         cast: torch.dtype | None = None, what: str = "", show: int = 6) -> float:
    """grad_scale [K] of the fused backward against `backward_restated`'s sum_rows x g: with d = backward_depths(...)[1],
    |got - xg| <= gamma_d xg_abs + 2^-125 M per channel (cast, skip_groups as `check_backward_theta`).  Raises AssertionError
    naming the violating channels with got / ref / tol; returns the largest err / tol."""
    dev = ref["xg"].device
    rows = ref["rows"]
    d = backward_depths(max_blocks, splits)[1]
    tol = _gamma(d) * ref["xg_abs"] + FTZ_PER_ROW * rows + _F64_SUM * rows * ref["xg_abs"]
    got = got.to(dev).reshape(-1)
    if cast is not None:
        tol = tol + ulp(got, cast)
    keep = torch.ones_like(tol, dtype=torch.bool)
    for gr in skip_groups:
        keep[gr * group:(gr + 1) * group] = False
    return _assert_entries(got, ref["xg"], tol, keep, lambda ch: f"channel {ch}, group {ch // group}", what, show)
