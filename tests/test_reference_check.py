"""The element-wise bound of tests/gpu_reference.py, on the CPU: it accepts any fp32 summation order, and it flags a single
element that normwise relative error 1e-3 lets through (a 64-channel partial sum missing, or 3 ulps off)."""
import pytest
import torch

from gpu_reference import check, ulp

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
