"""The element-wise bounds of tests/gpu_reference.py, on the CPU.  `check` (a fused linear) accepts any fp32 summation order and
flags a single element that normwise relative error 1e-3 lets through (a 64-channel partial sum missing, or 3 ulps off).
`check_combine` (a MoE block's weighted sum of expert outputs) accepts any fp32 order of the expert sums and of the slot
combine, and flags faults of the block's reduction and combine that the oracle comparisons' normwise and per-row bounds let
through.  `check_backward_theta` / `check_backward_scale` (the rotate op's fused backward) accept the kernel's fp32 sums taken
over rows in any order, in 4-row blocks, per warp and across warps by atomics in any order, and flag a block missing or counted
twice, a pair's term from its neighbour and two rotations' sums swapped."""
import pytest
import torch

from gpu_reference import (_nudge, backward_depths, check, check_backward_scale, check_backward_theta, check_combine, check_residual,
                           check_rmsnorm, exact_bias, exact_rms_rows, linear_bound, rms_candidates, rms_operand, ulp)

M, K, PARTS = 32, 4096, [1024, 1024]


def _case(dt, seed=0):
    g = torch.Generator().manual_seed(seed)
    xr = torch.randn(M, K, generator=g)
    xr[:, torch.randperm(K, generator=g)[:K // 100]] *= 20.0                                  # outlier channels
    q = torch.randint(0, 16, (K, sum(PARTS)), generator=g) - torch.randint(0, 16, (1, sum(PARTS)), generator=g)
    W = (q * 0.002 * (0.5 + torch.rand(K // 128, 1, sum(PARTS), generator=g)).repeat_interleave(128, 0).view(K, -1)).to(dt)
    xr = xr.to(dt)
    bias = (0.1 * torch.randn(sum(PARTS), generator=g)).to(dt)
    return [xr, xr], W, bias


def _fp32_chunked(xr, W, chunk):
    """fp32 accumulation in another order: per-chunk fp32 products, chunk sums added in fp32."""
    acc = torch.zeros(xr.shape[0], W.shape[1])
    for k0 in range(0, xr.shape[1], chunk):
        acc += xr[:, k0:k0 + chunk].float() @ W[k0:k0 + chunk].float()
    return acc


def _exact(xr, W):
    return xr.double() @ W.double()


def _rel(a, b):
    return float((a.double() - b.double()).norm() / b.double().norm())


def test_ulp():
    v = torch.tensor([1.0, 1.5, 0.75, 2.0 ** -130, 0.0], dtype=torch.float64)
    assert ulp(v, torch.bfloat16).tolist() == [2.0 ** -7, 2.0 ** -7, 2.0 ** -8, 2.0 ** -133, 2.0 ** -133]
    assert ulp(v, torch.float16)[:3].tolist() == [2.0 ** -10, 2.0 ** -10, 2.0 ** -11]
    assert ulp(v, torch.float16)[4] == 2.0 ** -24


@pytest.mark.parametrize("dt", [torch.bfloat16, torch.float16])
@pytest.mark.parametrize("with_bias", [False, True])
def test_accepts_any_fp32_summation_order(dt, with_bias):
    xrs, W, bias = _case(dt)
    b = bias if with_bias else None
    for chunk in (16, 64, 1024, K):
        acc = _fp32_chunked(xrs[0], W, chunk)
        y = acc.to(dt)
        if with_bias:
            y = (y.float() + bias.float()).to(dt)
        assert check(y, xrs, W, PARTS, b, what=f"chunk {chunk}") <= 1.0


@pytest.mark.parametrize("dt", [torch.bfloat16, torch.float16])
def test_flags_one_missing_partial_sum_that_normwise_misses(dt):
    xrs, W, _ = _case(dt, seed=1)
    xr = xrs[0]
    y = _exact(xr, W).to(dt)
    # row 5, column 1500 (partition 1, block 3): channels 2048..2111 (one group_size-64 K slice) dropped from the sum
    m, n, k0 = 5, 1500, 2048
    part = _exact(xr[m:m + 1, k0:k0 + 64], W[k0:k0 + 64, n:n + 1])[0, 0]
    bad = y.clone()
    bad[m, n] = (_exact(xr[m:m + 1], W[:, n:n + 1])[0, 0] - part).to(dt)
    assert bad[m, n] != y[m, n]
    assert _rel(bad, y) < 1e-3                                   # the normwise criterion does not see it
    with pytest.raises(AssertionError, match=r"1 of 65536 elements.*\n.*row 5, col 1500, block 3, part 1"):
        check(bad, xrs, W, PARTS)


@pytest.mark.parametrize("dt", [torch.bfloat16, torch.float16])
def test_flags_three_ulps_on_one_element(dt):
    xrs, W, _ = _case(dt, seed=2)
    y = _exact(xrs[0], W).to(dt)
    m, n = divmod(int(y.float().abs().argmax()), y.shape[1])
    bad = y.clone()
    bad[m, n] = (y[m, n].double() + 3 * ulp(y[m, n].double(), dt)).to(dt)
    assert _rel(bad, y) < 1e-3
    assert check(y, xrs, W, PARTS) == 0.0
    with pytest.raises(AssertionError, match=f"1 of 65536 elements.*\n.*row {m}, col {n}, block {(n % 1024) // 128}"):
        check(bad, xrs, W, PARTS)


def test_flags_non_finite_output():
    xrs, W, _ = _case(torch.bfloat16, seed=3)
    y = _exact(xrs[0], W).to(torch.bfloat16)
    y[0, 0] = float("nan")
    with pytest.raises(AssertionError, match="1 of 65536"):
        check(y, xrs, W, PARTS)


# ---- the MoE combine bound (check_combine): T tokens x k slots of E experts, each slot's rotated row xr [K] against its
# expert's operand W[e] [K, N]; the block rounds every slot's fp32 sum to T and adds the weighted slots in fp32
MT, MK, ME, MKK, MN = 4, 4, 4, 2048, 1024


def _moe(dt, seed, ids=None, w=None):
    g = torch.Generator().manual_seed(seed)
    W = []
    for _ in range(ME):
        q = torch.randint(0, 16, (MKK, MN), generator=g) - torch.randint(0, 16, (1, MN), generator=g)
        W.append((q * 0.002 * (0.5 + torch.rand(MKK // 128, 1, MN, generator=g)).repeat_interleave(128, 0).view(MKK, MN)).to(dt))
    xr = torch.randn(MT, MK, MKK, generator=g)
    xr[..., torch.randperm(MKK, generator=g)[:MKK // 100]] *= 20.0
    ids = torch.stack([torch.randperm(ME, generator=g)[:MK] for _ in range(MT)]) if ids is None else ids
    w = torch.softmax(torch.randn(MT, MK, generator=g), -1) if w is None else w
    return {"dt": dt, "W": W, "xr": xr.to(dt), "ids": ids, "w": w}


def _moe_exact(c):
    rows = [(c["xr"][t, s].double(), c["W"][int(c["ids"][t, s])].double()) for t in range(MT) for s in range(MK)]
    return torch.stack([x @ Wd for x, Wd in rows]), torch.stack([x.abs() @ Wd.abs() for x, Wd in rows])   # [T * k, N]


def _moe_slots(c, chunk=128, skip_group=None):
    """v [T, k, N]: every slot's fp32 sum in chunks of `chunk` channels, rounded to T.  skip_group = (t, s, g, block): channels
    g * 128 .. + 127 left out of slot (t, s)'s sum in the 128 columns of `block`."""
    v = torch.zeros(MT, MK, MN)
    for t in range(MT):
        for s in range(MK):
            x, Wf = c["xr"][t, s].float(), c["W"][int(c["ids"][t, s])].float()
            for k0 in range(0, MKK, chunk):
                p = x[k0:k0 + chunk] @ Wf[k0:k0 + chunk]
                if skip_group is not None and skip_group[:2] == (t, s) and k0 // 128 == skip_group[2]:
                    p[128 * skip_group[3]:128 * skip_group[3] + 128] = 0.0
                v[t, s] += p
    return v.to(c["dt"]).float()


def _moe_combine(v, w, order=range(MK), skip=()):
    """out [T, N] = fp32 sum over slots in `order` of fp32(v * w), from 0 (slots (t, s) in `skip` left out)."""
    out = torch.zeros(MT, MN)
    for t in range(MT):
        acc = torch.zeros(MN)
        for s in order:
            if (t, s) not in skip:
                acc = acc + v[t, s] * w[t, s]
        out[t] = acc
    return out


def _moe_check(c, y, exact):
    ys, mag = exact
    return check_combine(y, torch.arange(MT).repeat_interleave(MK), c["w"].reshape(-1), ys, mag)


def _passes_old_bounds(c, bad, exact):
    """The normwise (2e-3) and per-row (2e-3, and so 1.5e-2) bounds of the MoE block's oracle comparisons, against the oracle's
    combine: fp64 sum of w * T(y_s), rounded to T."""
    ref = (c["w"].double()[..., None] * exact[0].view(MT, MK, MN).to(c["dt"]).double()).sum(1).to(c["dt"])
    return _rel(bad, ref) < 2e-3 and all(_rel(bad[t], ref[t]) < 2e-3 for t in range(MT))


@pytest.mark.parametrize("dt", [torch.bfloat16, torch.float16])
def test_moe_bound_accepts_any_fp32_order(dt):
    c = _moe(dt, seed=0)
    c["w"][1, 2] = 0.0                                                                        # a zero weight
    exact = _moe_exact(c)
    for chunk in (16, 128, MKK):
        v = _moe_slots(c, chunk)
        for order in ([0, 1, 2, 3], [3, 2, 1, 0], [2, 0, 3, 1]):
            assert _moe_check(c, _moe_combine(v, c["w"], order).to(dt), exact) <= 1.0, (chunk, order)


@pytest.mark.parametrize("dt", [torch.bfloat16, torch.float16])
def test_moe_bound_token_without_slot_must_be_zero(dt):
    c = _moe(dt, seed=4)
    ys, mag = _moe_exact(c)
    keep = torch.arange(MT).repeat_interleave(MK) != 3                                        # token 3: every id dropped
    y = _moe_combine(_moe_slots(c), c["w"], skip={(3, s) for s in range(MK)}).to(dt)
    assert check_combine(y, torch.arange(MT).repeat_interleave(MK)[keep], c["w"].reshape(-1)[keep], ys[keep], mag[keep]) <= 1.0
    y[3, 700] = 2.0 ** -20
    with pytest.raises(AssertionError, match=r"1 of 4096 elements.*\n.*token 3, col 700, block 5\).*no valid slot"):
        check_combine(y, torch.arange(MT).repeat_interleave(MK)[keep], c["w"].reshape(-1)[keep], ys[keep], mag[keep])


@pytest.mark.parametrize("dt", [torch.bfloat16, torch.float16])
def test_moe_bound_flags_one_group_missing_from_one_slot(dt):
    # token 2's slot 3 (weight 0.01) loses channels 640..767 in column block 3: a dropped K slice of one expert
    c = _moe(dt, seed=1)
    c["w"][2] = torch.tensor([0.55, 0.43, 0.01, 0.01])
    exact = _moe_exact(c)
    bad = _moe_combine(_moe_slots(c, skip_group=(2, 3, 5, 3)), c["w"]).to(dt)
    assert _passes_old_bounds(c, bad, exact)
    with pytest.raises(AssertionError, match=r"elements outside the element-wise bound\n.*token 2, col \d+, block 3\)"):
        _moe_check(c, bad, exact)


@pytest.mark.parametrize("dt", [torch.bfloat16, torch.float16])
def test_moe_bound_flags_duplicate_slot_counted_once(dt):
    # token 1 routes slots 1 and 2 to expert 2; the block adds only the first of them
    ids = torch.tensor([[0, 1, 2, 3], [0, 2, 2, 3], [3, 2, 1, 0], [1, 0, 3, 2]])
    c = _moe(dt, seed=2, ids=ids)
    c["w"][1] = torch.tensor([0.55, 0.00005, 0.0006, 0.44935])
    c["xr"][1, 2] = c["xr"][1, 1]                                                           # one h row feeds both duplicates
    exact = _moe_exact(c)
    bad = _moe_combine(_moe_slots(c), c["w"], skip={(1, 2)}).to(dt)
    assert _passes_old_bounds(c, bad, exact)
    with pytest.raises(AssertionError, match=r"elements outside the element-wise bound\n.*token 1, col"):
        _moe_check(c, bad, exact)


@pytest.mark.parametrize("dt", [torch.bfloat16, torch.float16])
def test_moe_bound_flags_slot_0_weight_on_slot_1(dt):
    c = _moe(dt, seed=3)
    c["w"][0] = torch.tensor([0.0204, 0.02, 0.5, 0.4596])
    exact = _moe_exact(c)
    wrong = c["w"].clone()
    wrong[0, 1] = wrong[0, 0]                                                               # token 0: slot 1 added with slot 0's weight
    bad = _moe_combine(_moe_slots(c), wrong).to(dt)
    assert _passes_old_bounds(c, bad, exact)
    with pytest.raises(AssertionError, match=r"elements outside the element-wise bound\n.*token 0, col"):
        _moe_check(c, bad, exact)


@pytest.mark.parametrize("dt", [torch.bfloat16, torch.float16])
def test_moe_bound_flags_three_ulps_on_one_element(dt):
    c = _moe(dt, seed=5)
    exact = _moe_exact(c)
    y = _moe_combine(_moe_slots(c), c["w"]).to(dt)
    t, n = divmod(int(y.float().abs().argmax()), MN)
    bad = y.clone()
    bad[t, n] = (y[t, n].double() + 3 * ulp(y[t, n].double(), dt)).to(dt)
    assert _passes_old_bounds(c, bad, exact)
    assert _moe_check(c, y, exact) <= 1.0
    with pytest.raises(AssertionError, match=f"1 of 4096 elements.*\n.*token {t}, col {n}, block {n // 128}\\)"):
        _moe_check(c, bad, exact)


# ---- the chain neighbours' bounds: the RMSNORM x op on exact-statistics rows (`exact_rms_rows` + `check`), on random data
# (`check_rmsnorm`), and the ADD_RESIDUAL epilogue without y (`check_residual`)
CK, CN = 2048, 256


def _rms_case(dt, M, K=CK, seed=0):
    g = torch.Generator().manual_seed(seed)
    h = (torch.randn(M, K, generator=g) * (0.5 + torch.rand(M, 1, generator=g)) * 4).to(dt)
    h[:, torch.randperm(K, generator=g)[:K // 100]] *= 20
    w = (1.0 + 0.1 * torch.randn(K, generator=g)).to(dt)
    q = torch.randint(0, 16, (K, CN), generator=g) - torch.randint(0, 16, (1, CN), generator=g)
    W = (q * 0.002 * (0.5 + torch.rand(K // 128, 1, CN, generator=g)).repeat_interleave(128, 0).view(K, -1)).to(dt)
    return h, w, W


def _block_stats(h, width=128):
    """fp32 sums of h^2 per (width-column block, row), as the epilogues write them: [K / width, M]."""
    hf = h.float()
    return (hf * hf).view(h.shape[0], -1, width).sum(-1).t().contiguous()


def _rstd(s, K, eps):
    """the kernels' rstd from fp32 row sums s: rsqrt(s / K + eps) in fp32."""
    return torch.rsqrt(s / float(K) + torch.tensor(eps, dtype=torch.float32))


def _gpu_like_y(x, W, bias=None, chunk=64):
    y = _fp32_chunked(x, W, chunk).to(x.dtype)
    return y if bias is None else (y.float() + bias.float()).to(x.dtype)


@pytest.mark.parametrize("dt", [torch.bfloat16, torch.float16])
@pytest.mark.parametrize("K", [512, 5120, 8192])
def test_exact_rows_invariants(dt, K):
    g = torch.Generator().manual_seed(K)
    w = (1.0 + 0.1 * torch.randn(K, generator=g)).to(dt)
    M, nb = 12, K // 128
    hot = [-1, 0, nb - 1, 1, -1, nb // 2, nb - 2, -1, 3 % nb, nb - 1, 2 % nb, -1]
    h, x = exact_rms_rows(M, K, dt, seed=K, w=w, hot=hot)
    hd = h.double() ** 2
    exact = hd.sum(-1)
    for order in (torch.arange(K), torch.arange(K).flip(0), torch.randperm(K, generator=g)):
        assert torch.equal(hd[:, order].float().cumsum(-1)[:, -1].double(), exact)                      # sequential fp32
    assert torch.equal(_block_stats(h).sum(0).double(), exact)                                          # per block, then blocks
    assert torch.equal(_block_stats(h, 32).flip(0).cumsum(0)[-1].double(), exact)                       # per word, reversed
    r = _rstd(exact.float(), K, 1e-8)
    for d in range(-4, 5):
        assert torch.equal(rms_operand(h, _nudge(r, d), w), x), d
    for m, b in enumerate(hot):
        if b < 0:   # uniform: mean square 4^j, T(h * rstd) = +-c exactly
            assert set(rms_operand(h[m:m + 1], r[m:m + 1], None).abs().unique().tolist()) == {0.5, 1.5}
            continue
        for q in range(4):
            a = 128 * b + 32 * q
            share = float(hd[m, a:a + 32].sum())
            for s2 in (exact[m] - share, exact[m] + share):
                assert not torch.equal(rms_operand(h[m:m + 1], _rstd(s2.float()[None], K, 1e-8), w), x[m:m + 1]), (m, q)


def test_exact_bias_keeps_rows_exact():
    for dt in (torch.bfloat16, torch.float16):
        h, _ = exact_rms_rows(8, 1024, dt, seed=3)
        b = exact_bias(1024, 4, dt)
        r = (h.double() - b.double()).to(dt)
        assert torch.equal(r.double(), h.double() - b.double())
        assert torch.equal((b.float() + r.float()).to(dt), h)


@pytest.mark.parametrize("dt", [torch.bfloat16, torch.float16])
def test_rmsnorm_bound_accepts_other_fp32_orders(dt):
    M, eps = 64, 1e-5
    h, w, W = _rms_case(dt, M)
    ident = lambda x: [x]   # noqa: E731  the bound is rotation-agnostic: the CPU cases use the operand as it is
    for width, chunk in ((128, 64), (32, 16), (CK, CK)):
        stats = _block_stats(h, width)
        for s in (stats.sum(0), stats.flip(0).cumsum(0)[-1]):
            y = _gpu_like_y(rms_operand(h, _rstd(s, CK, eps), w), W, chunk=chunk)
            assert check_rmsnorm(y, h, w, eps, ident, W, [CN]) <= 1.0


@pytest.mark.parametrize("dt", [torch.bfloat16, torch.float16])
@pytest.mark.parametrize("with_bias", [False, True])
def test_residual_bound_accepts_other_fp32_orders(dt, with_bias):
    xrs, W, bias = _case(dt, seed=6)
    b = bias if with_bias else None
    r = (torch.randn(M, sum(PARTS), generator=torch.Generator().manual_seed(7)) * 0.5).to(dt)
    t = linear_bound(xrs, W, PARTS, dt, b)
    for chunk in (16, 1024):
        y = _gpu_like_y(xrs[0], W, b, chunk)
        assert check_residual((y.float() + r.float()).to(dt), t, r) <= 1.0


# planted faults at M = 1000 that the whole-matrix 1e-3 lets through
FM = 1000


@pytest.mark.parametrize("dt", [torch.bfloat16, torch.float16])
def test_rmsnorm_bound_flags_one_row_missing_one_block(dt):
    eps = 1e-5
    h, w, W = _rms_case(dt, FM, seed=8)
    stats = _block_stats(h)
    s = stats.sum(0)
    ok = _gpu_like_y(rms_operand(h, _rstd(s, CK, eps), w), W)
    s[617] -= stats[CK // 128 - 1, 617]                                   # row 617's rstd without its last block
    bad = _gpu_like_y(rms_operand(h, _rstd(s, CK, eps), w), W)
    ref = _exact(rms_candidates(h, w, eps)[0][:FM], W).to(dt)             # oracle.rms_norm -> fp64 linear
    assert _rel(bad, ref) < 1e-3 and _rel(ok, ref) < 1e-3
    assert check_rmsnorm(ok, h, w, eps, lambda x: [x], W, [CN]) <= 1.0
    with pytest.raises(AssertionError, match=r"1 of 1000 rows .*\(rows \[617\]\)"):
        check_rmsnorm(bad, h, w, eps, lambda x: [x], W, [CN])


@pytest.mark.parametrize("dt", [torch.bfloat16, torch.float16])
def test_exact_rows_flag_one_statistics_word_from_the_next_row(dt):
    """The prefill pre-pass adds row m's block partials in block order; here row m reads block b's partial of row m + 1."""
    K = 4096
    nb = K // 128
    g = torch.Generator().manual_seed(9)
    w = (1.0 + 0.1 * torch.randn(K, generator=g)).to(dt)
    hot = [-1 if m % 3 == 0 else (m * 5) % nb for m in range(FM)]
    h, x = exact_rms_rows(FM, K, dt, seed=9, w=w, hot=hot)
    q = torch.randint(0, 16, (K, CN), generator=g) - torch.randint(0, 16, (1, CN), generator=g)
    W = (q * 0.002 * (0.5 + torch.rand(K // 128, 1, CN, generator=g)).repeat_interleave(128, 0).view(K, -1)).to(dt)
    stats = _block_stats(h)
    m = 400
    s = stats.sum(0)
    assert torch.equal(rms_operand(h, _rstd(s, K, 1e-8), w), x)
    # the first block outside both rows' hot blocks whose partials differ enough to move the operand: a cold block, so the
    # whole-matrix error stays small
    for b in range(nb):
        if b in (hot[m], hot[m + 1]):
            continue
        s2 = s.clone()
        s2[m] = s[m] - stats[b, m] + stats[b, m + 1]
        op = rms_operand(h, _rstd(s2, K, 1e-8), w)
        if not torch.equal(op, x):
            break
    else:
        raise AssertionError("no cold block moves the operand")
    y = _gpu_like_y(op, W)
    ref = _exact(x, W).to(dt)
    assert _rel(y, ref) < 1e-3
    assert check(_gpu_like_y(x, W), [x], W, [CN]) <= 1.0
    with pytest.raises(AssertionError, match=rf"elements outside the element-wise bound\n.*\(row {m}, col"):
        check(y, [x], W, [CN])


@pytest.mark.parametrize("dt", [torch.bfloat16, torch.float16])
def test_residual_bound_flags_one_block_of_one_row(dt):
    g = torch.Generator().manual_seed(10)
    x = torch.randn(FM, 1024, generator=g).to(dt)
    q = torch.randint(0, 16, (1024, CN), generator=g) - torch.randint(0, 16, (1, CN), generator=g)
    W = (q * 0.002 * (0.5 + torch.rand(8, 1, CN, generator=g)).repeat_interleave(128, 0).view(1024, -1)).to(dt)
    r = (torch.randn(FM, CN, generator=g) * 0.3).to(dt)
    h = (_gpu_like_y(x, W).float() + r.float()).to(dt)
    t = linear_bound([x], W, [CN], dt)
    assert check_residual(h, t, r) <= 1.0
    bad = h.clone()
    m, b = 733, 1
    blk = bad[m, 128 * b:128 * b + 128].double()
    pattern = torch.tensor([4.0, -4.0], dtype=torch.float64).repeat(64)      # +-4 ulps, alternating
    bad[m, 128 * b:128 * b + 128] = (blk + pattern * ulp(blk, dt)).to(dt)
    assert _rel(bad, h) < 1e-3
    with pytest.raises(AssertionError, match=rf"elements outside the element-wise bound\n.*\(row {m}, col \d+, block {b}, part 0\)"):
        check_residual(bad, t, r)


# ---- the rotate op's fused backward: grad_theta and grad_scale
BG, BK, BKROT, BM = 128, 256, 3, 2003                     # 2 groups; 501 row blocks, the last one ragged


def _bwd_case(seed=0):
    """Stage values t_r, g_r [krot, M, K] (fp32, independent per rotation: the bound does not care where they come from), x, the
    absolute pair channels [krot, K / 2] of random group-relative pairs, (c, s) of random angles, and the fp64 sums of
    `backward_restated`."""
    g = torch.Generator().manual_seed(seed)
    t = torch.randn(BKROT, BM, BK, generator=g)
    gr = torch.randn(BKROT, BM, BK, generator=g) * 0.01
    x = torch.randn(BM, BK, generator=g)
    base = (torch.arange(BK) // BG * BG).view(BK // 2, 2)[:, 0]
    ci, cj = [], []
    for _ in range(BKROT):
        perm = torch.cat([torch.randperm(BG, generator=g) + q * BG for q in range(BK // BG)]).view(BK // 2, 2) - base[:, None]
        ci.append(perm[:, 0] + base)
        cj.append(perm[:, 1] + base)
    ci, cj = torch.stack(ci), torch.stack(cj)
    ang = (torch.rand(BKROT, BK // 2, generator=g) * 2 - 1) * 3.0
    c, s = ang.cos(), ang.sin()
    ref = {k: torch.zeros(BKROT, BK // 2, dtype=torch.float64) for k in "SDAB"}
    for r in range(BKROT):
        gi, gj, ti, tj = (v.double() for v in (gr[r][:, ci[r]], gr[r][:, cj[r]], t[r][:, ci[r]], t[r][:, cj[r]]))
        a, b, cc, d = gi * tj, gj * ti, gi * ti, gj * tj
        ref["S"][r], ref["D"][r], ref["A"][r], ref["B"][r] = (a - b).sum(0), (cc + d).sum(0), (a.abs() + b.abs()).sum(0), (cc.abs() + d.abs()).sum(0)
    xg = x.double() * gr[0].double()                      # grad_scale: x times the last un-rotated g
    ref["xg"], ref["xg_abs"], ref["rows"] = xg.sum(0), xg.abs().sum(0), BM
    return t, gr, x, ci, cj, c, s, ref


def _warp_sums(rows_terms, splits, block_sum, fault=None):
    """The kernel's per-warp fp32 running sums: rows_terms [M, E] fp32 -> [splits, E].  Row blocks of 4 (zero rows pad the last),
    block b summed by block_sum([4, E]) and added to warp b % splits in block order.  fault: ("drop" | "twice", block)."""
    M, E = rows_terms.shape
    rb = (M + 3) // 4
    nb = (rb + splits - 1) // splits
    padded = torch.zeros(nb * splits * 4, E)
    padded[:M] = rows_terms
    blocks = padded.view(nb, splits, 4, E)
    acc = torch.zeros(splits, E)
    for i in range(nb):
        for w in range(splits):
            b = i * splits + w
            if fault == ("drop", b):
                continue
            part = block_sum(blocks[i, w])
            acc[w] = acc[w] + part
            if fault == ("twice", b):
                acc[w] = acc[w] + part
    return acc


def _atomics(parts, g):
    """fp32 atomics of the warp partials [splits, E] into a zeroed buffer, in a random order."""
    out = torch.zeros(parts.shape[1])
    for w in torch.randperm(parts.shape[0], generator=g).tolist():
        out = out + parts[w]
    return out


def _theta_rows(t, gr, ci, cj, r):
    gi, gj, ti, tj = gr[r][:, ci[r]], gr[r][:, cj[r]], t[r][:, ci[r]], t[r][:, cj[r]]
    return gi * tj - gj * ti, gi * ti + gj * tj            # fp32: two products and a difference per row


def _block4(v):
    return ((v[0] + v[1]) + v[2]) + v[3]


def _kernel_like_theta(case, splits, seed, reference_formula=False, fault=None, rotation=None):
    """grad_theta [krot, K / 2] summed as the kernel does, rows taken in a random order (fault applied in rotation `rotation`, or
    all rotations when None: a block a warp drops or repeats is dropped or repeated for all its entries)."""
    t, gr, x, ci, cj, c, s, ref = case
    g = torch.Generator().manual_seed(seed)
    perm = torch.randperm(BM, generator=g)
    out = torch.zeros(BKROT, BK // 2)
    for r in range(BKROT):
        f = fault if rotation in (None, r) else None
        cross, dot = (v[perm] for v in _theta_rows(t, gr, ci, cj, r))
        acc = _warp_sums(cross, splits, _block4, f)
        if reference_formula:
            acc = c[r] * acc + s[r] * _warp_sums(dot, splits, _block4, f)
        out[r] = _atomics(acc, g)
    return out


def _kernel_like_scale(case, splits, seed, fault=None):
    t, gr, x, ci, cj, c, s, ref = case
    g = torch.Generator().manual_seed(seed)
    perm = torch.randperm(BM, generator=g)
    prods = (x * gr[0])[perm]                              # acc_s += x * g row by row: one fp32 step per row
    M, E = prods.shape
    rb = (M + 3) // 4
    nb = (rb + splits - 1) // splits
    padded = torch.zeros(nb * splits * 4, E)
    padded[:M] = prods
    blocks = padded.view(nb, splits, 4, E)
    acc = torch.zeros(splits, E)
    for i in range(nb):
        for w in range(splits):
            b = i * splits + w
            reps = 0 if fault == ("drop", b) else 2 if fault == ("twice", b) else 1
            for _ in range(reps):
                for q in range(4):
                    acc[w] = acc[w] + blocks[i, w, q]
    return _atomics(acc, g)


def _plan_depth(splits):
    rb = (BM + 3) // 4
    return (rb + splits - 1) // splits, splits


@pytest.mark.parametrize("splits", [1, 7, 66, 251, 501])
@pytest.mark.parametrize("reference_formula", [False, True])
def test_backward_bounds_accept_any_row_order_and_atomic_order(splits, reference_formula):
    case = _bwd_case()
    c, s, ref = case[5], case[6], case[7]
    nb, sp = _plan_depth(splits)
    for seed in (1, 2):
        got = _kernel_like_theta(case, splits, seed, reference_formula)
        assert check_backward_theta(got, ref, c, s, BG, nb, sp, reference_formula, what=f"splits {splits}") <= 1.0
        assert check_backward_scale(_kernel_like_scale(case, splits, seed), ref, BG, nb, sp) <= 1.0


def test_backward_depths():
    assert backward_depths(16, 66) == (5 + 16 + 66, 1 + 64 + 66)


@pytest.mark.parametrize("fault", ["drop", "twice"])
@pytest.mark.parametrize("reference_formula", [False, True])
def test_backward_bound_flags_one_block_missing_or_duplicated_in_one_warp(fault, reference_formula):
    case = _bwd_case(seed=3)
    c, s, ref = case[5], case[6], case[7]
    splits = 66
    nb, sp = _plan_depth(splits)
    blk = 66 * 4 + 67                                      # row block 331: warp 1 (group 0 in this layout of the rows), 6th block
    got = _kernel_like_theta(case, splits, 5, reference_formula, fault=(fault, blk), rotation=1)
    with pytest.raises(AssertionError, match=r"entries outside the element-wise bound\n.*\(rotation 1, group \d, pair \d+\)"):
        check_backward_theta(got, ref, c, s, BG, nb, sp, reference_formula)
    with pytest.raises(AssertionError, match=r"entries outside the element-wise bound\n.*\(channel \d+, group \d\)"):
        check_backward_scale(_kernel_like_scale(case, splits, 5, fault=(fault, blk)), ref, BG, nb, sp)


@pytest.mark.parametrize("reference_formula", [False, True])
def test_backward_bound_flags_one_pair_from_its_neighbour(reference_formula):
    case = _bwd_case(seed=4)
    c, s, ref = case[5], case[6], case[7]
    nb, sp = _plan_depth(66)
    got = _kernel_like_theta(case, 66, 6, reference_formula)
    assert check_backward_theta(got, ref, c, s, BG, nb, sp, reference_formula) <= 1.0
    r, p = 2, 64 + 17                                      # group 1, pair 17 takes pair 18's sums
    t, gr, x, ci, cj = case[:5]
    ci2, cj2 = ci.clone(), cj.clone()
    ci2[r, p], cj2[r, p] = ci[r, p + 1], cj[r, p + 1]
    bad = _kernel_like_theta((t, gr, x, ci2, cj2, c, s, ref), 66, 6, reference_formula)
    with pytest.raises(AssertionError, match=r"1 of 384 entries outside the element-wise bound\n  \(rotation 2, group 1, pair 17\)"):
        check_backward_theta(bad, ref, c, s, BG, nb, sp, reference_formula)


@pytest.mark.parametrize("reference_formula", [False, True])
def test_backward_bound_flags_two_rotations_swapped(reference_formula):
    case = _bwd_case(seed=5)
    c, s, ref = case[5], case[6], case[7]
    nb, sp = _plan_depth(7)
    got = _kernel_like_theta(case, 7, 8, reference_formula)
    bad = got.clone()
    bad[[0, 1]] = got[[1, 0]]
    with pytest.raises(AssertionError, match=r"entries outside the element-wise bound\n  \(rotation 0, group 0, pair \d+\)"):
        check_backward_theta(bad, ref, c, s, BG, nb, sp, reference_formula)


def test_backward_bound_skips_only_the_named_groups():
    case = _bwd_case(seed=6)
    c, s, ref = case[5], case[6], case[7]
    nb, sp = _plan_depth(66)
    got = _kernel_like_theta(case, 66, 9)
    gsc = _kernel_like_scale(case, 66, 9)
    got[:, 64 + 5], gsc[BG + 9] = float("nan"), float("inf")
    assert check_backward_theta(got, ref, c, s, BG, nb, sp, skip_groups=[1]) <= 1.0
    assert check_backward_scale(gsc, ref, BG, nb, sp, skip_groups=[1]) <= 1.0
    with pytest.raises(AssertionError, match=r"3 of 384 entries.*\n  \(rotation 0, group 1, pair 5\): got nan"):
        check_backward_theta(got, ref, c, s, BG, nb, sp)
    with pytest.raises(AssertionError, match=r"1 of 128 entries.*\n  \(channel 137, group 1\): got inf"):
        check_backward_scale(gsc, ref, BG, nb, sp, skip_groups=[0])


def test_rotate_backward_plan_reaches_every_case_at_132_sms():
    """paro_debug_rotate_backward_plan (the function the launch uses) on an H100 SXM's 132 SMs: every case of the GPU suite gets
    the blocks per warp, the uneven split or the dynamic shared memory it is there for."""
    from paroquant_b200 import _cabi
    from rotate_backward_cases import CASES, assert_plan_reaches, case_id
    for c in CASES:
        dt, G, krot, M, K, forms, kind = c
        for f in forms:
            plan = _cabi.debug_rotate_backward_plan(M, K, krot, G, dt, f, sms=132)
            assert_plan_reaches(plan, kind, M, f"{case_id(c)} reference_formula={f}")
            assert plan["row_blocks"] == (M + 3) // 4
            assert plan["grid"] == (plan["splits"] * (K // G) + 3) // 4
    # the 48 KB opt-in: the krot-13 and krot-16 group-128 cases and the reference formula's krot 10, not krot 8
    dyn = lambda krot, f=False: _cabi.debug_rotate_backward_plan(4096, 4096, krot, 128, torch.float32, f, sms=132)["dyn_smem"]
    assert dyn(13) == 53248 and dyn(16) == 65536 and dyn(16, True) == 81920 and dyn(10, True) == 51200
    assert dyn(8) <= 48 * 1024 and dyn(8, True) <= 48 * 1024 and dyn(12) <= 48 * 1024 and dyn(9, True) <= 48 * 1024
    # what the old stage-wise cases (K 1024) got: one block per warp
    for dt, G, krot, M in ((torch.float32, 128, 8, 1037), (torch.float32, 64, 8, 333), (torch.bfloat16, 128, 8, 260)):
        assert _cabi.debug_rotate_backward_plan(M, 1024, krot, G, dt, sms=132)["max_blocks_per_warp"] == 1
    for bad in ((0, 4096, 8, 128), (1, 4096, 17, 128), (1, 100, 8, 64), (1, 4096, 8, 32)):
        with pytest.raises(RuntimeError, match="debug_rotate_backward_plan"):
            _cabi.debug_rotate_backward_plan(*bad, torch.float32, sms=132)
