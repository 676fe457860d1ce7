"""The standalone rotate op (torch.ops.rotation.rotate) bit for bit against an exact CPU restatement, on the GPU's own sin / cos.

The CPU oracle restates the rotation with an error-free fp32 FMA and every rounding point of the kernels; it differs from them
only in where sin / cos come from (libm there, MUFU __sincosf here), which is why test_gpu_rotate.py compares it normwise.
`gpu_reference.kernel_sincos` reads the exact __sincosf values the kernels use, and this module

  * bounds that table against fp64 (CUDA's documented 2^-21.41 for __sinf and 2^-21.19 for __cosf, |theta| <= pi) over
    every fp16 and bf16 angle in
    [-pi, pi], random fp32 angles and the synthetic layers' angles -- the one GPU-sourced input of the reference;
  * requires the rotate op to equal oracle.np_rotate on that table value for value (+0 == -0, inf / NaN at the same
    positions, nothing else may differ) over dtypes, group sizes, krot, K up to 14336, ragged row blocks (4 rows for fp32, 8
    for fp16 / bf16) up to 4096 rows, every scale form, theta dtypes, 3-D inputs, subnormals and overflow.

Above 64 rows the CPU side looks at the first 16 rows, every row of the last block and 64 seeded random rows.
"""
import math

import numpy as np
import pytest
import torch

from gpu_reference import COS_ABS, SIN_ABS, assert_same_values, exact_rotate, kernel_sincos, sample_rows
from paroquant_b200.checkpoint import make_synthetic_activations, make_synthetic_layer

pytestmark = pytest.mark.gpu
F32, F16, BF16 = torch.float32, torch.float16, torch.bfloat16
RB = {F32: 4, F16: 8, BF16: 8}
KROTS = [1, 2, 3, 7, 8, 9, 16]


@pytest.fixture(scope="module")
def ops():
    import paroquant_b200.kernels.cuda as k  # registers torch.ops.rotation.rotate
    return k


# ---------------------------------------------------------------- the sin / cos table
def _every_value_in_pi(dtype):
    """Every finite value of a 16-bit float type with |v| <= pi, as fp32."""
    v = torch.from_numpy(np.arange(1 << 16, dtype=np.uint16).view(np.int16)).view(dtype).float()
    return v[torch.isfinite(v) & (v.abs() <= math.pi)]


def test_kernel_sincos_within_the_documented_bound_of_fp64(ops):
    g = torch.Generator().manual_seed(3)
    layers = [make_synthetic_layer(1024, [64], krot=16, seed=s, theta_uniform_pi=u) for s, u in ((1, False), (2, True))]
    thetas = {"fp16": _every_value_in_pi(F16), "bf16": _every_value_in_pi(BF16),
              "fp32": (torch.rand(1 << 16, generator=g, dtype=torch.float64) * 2 - 1).mul(math.pi).float(),
              "layers": torch.cat([L.theta.float().reshape(-1) for L in layers])}
    for name, th in thetas.items():
        c, s = kernel_sincos(th)
        t64 = th.double()
        ec = (c.double().cpu() - torch.cos(t64)).abs()
        es = (s.double().cpu() - torch.sin(t64)).abs()
        print(f"[sincos] {name}: {th.numel()} angles, max |theta| {float(th.abs().max()):.6f}, "
              f"max |cos err| 2^{math.log2(max(float(ec.max()), 1e-300)):.2f}, max |sin err| 2^{math.log2(max(float(es.max()), 1e-300)):.2f}")
        assert float(ec.max()) <= COS_ABS and float(es.max()) <= SIN_ABS, name


# ---------------------------------------------------------------- rotate op == np_rotate on the table
def _compare(x, pairs, theta, scales, G, what, seed=0):
    """Rotate x on the GPU; compare the sampled rows with exact_rotate."""
    got = torch.ops.rotation.rotate(x, pairs, theta, scales, G)
    assert got.shape == x.shape and got.dtype == x.dtype
    K = x.shape[-1]
    g2, x2 = got.reshape(-1, K), x.reshape(-1, K)
    rows = sample_rows(x2.shape[0], RB[x.dtype], seed).cuda()
    ref = exact_rotate(x2[rows], pairs, theta, scales, G)
    assert_same_values(g2[rows], ref, what)
    return got


def _layer(K, G, krot, seed, **kw):
    L = make_synthetic_layer(K, [64], group_size=G, krot=krot, seed=seed, device="cuda", **kw)
    return L.pairs[0], L.theta[0], L.channel_scales[0]


@pytest.mark.parametrize("dt", [F32, F16, BF16])
@pytest.mark.parametrize("G", [64, 128])
@pytest.mark.parametrize("krot", KROTS)
def test_dtypes_groups_krot(ops, dt, G, krot):
    pr, th, cs = _layer(1024, G, krot, seed=100 + krot)
    for M in (1, 9):
        x = make_synthetic_activations(M, 1024, seed=110 + M, device="cuda", dtype=dt)
        _compare(x, pr, th, cs, G, f"{dt} g{G} krot{krot} M={M}")


@pytest.mark.parametrize("dt", [F32, F16, BF16])
@pytest.mark.parametrize("K", [128, 256, 1024, 4096, 11008, 14336])
def test_K(ops, dt, K):
    for G, krot in ((128, 8), (64, 9)):
        pr, th, cs = _layer(K, G, krot, seed=K + G)
        x = make_synthetic_activations(17, K, seed=K, device="cuda", dtype=dt)
        _compare(x, pr, th, cs, G, f"{dt} K={K} g{G} krot{krot}")


@pytest.mark.parametrize("dt", [F32, F16, BF16])
@pytest.mark.parametrize("M", [1, 3, 4, 5, 7, 8, 9, 17, 1037, 4096])
def test_M_ragged_row_blocks(ops, dt, M):
    K = 4096 if M < 1000 else 2048
    pr, th, cs = _layer(K, 128, 8, seed=200 + M, theta_uniform_pi=True)
    x = make_synthetic_activations(M, K, seed=210 + M, device="cuda", dtype=dt)
    _compare(x, pr, th, cs, 128, f"{dt} M={M}", seed=M)


@pytest.mark.parametrize("dt", [F32, F16, BF16])
def test_scales_theta_forms_and_3d_input(ops, dt):
    K, G = 512, 64
    pr, th, cs = _layer(K, G, 3, seed=300, theta_uniform_pi=True)
    x = make_synthetic_activations(2 * 5, K, seed=301, device="cuda", dtype=dt)
    g = torch.Generator(device="cuda").manual_seed(302)
    cs32 = torch.exp(torch.randn(1, K, generator=g, device="cuda") * 0.3)             # values an fp16 scale cannot hold
    th32 = th.float() + torch.randn(th.shape, generator=g, device="cuda") * 1e-3     # angles between fp16 values
    for name, sc in (("none", None), ("[1,K] fp16", cs), ("[K] fp16", cs.reshape(-1)), ("[1,K] fp32", cs32),
                     ("[K] bf16", cs32.reshape(-1).to(BF16))):
        for tname, t in (("fp16", th), ("fp32", th32), ("bf16", th32.to(BF16))):
            _compare(x, pr, t, sc, G, f"{dt} scales {name} theta {tname}")
    # a 3-D input is its rows
    y3 = _compare(x.reshape(2, 5, K), pr, th32, cs32, G, f"{dt} 3-D")
    assert torch.equal(y3.reshape(10, K), torch.ops.rotation.rotate(x, pr, th32, cs32, G))


@pytest.mark.parametrize("dt", [F32, F16, BF16])
def test_subnormal_inputs(ops, dt):
    """Subnormal inputs next to normal ones (fp32 subnormals are flushed, as --use_fast_math does and the oracle's _ftz
    mirrors; fp16 / bf16 ones go through their scale product in T and are exact in fp32)."""
    K, G = 1024, 128
    pr, th, cs = _layer(K, G, 8, seed=400, theta_uniform_pi=True)
    g = torch.Generator(device="cuda").manual_seed(401)
    tiny = torch.finfo(dt).smallest_normal
    x = torch.randn(13, K, generator=g, device="cuda", dtype=torch.float64) * tiny * 0.25
    x[::2, ::3] *= 256.0                                              # normal values in every other row
    x = x.to(dt)
    assert bool(((x.abs() < tiny) & (x != 0)).any()) and bool((x.abs() >= tiny).any())
    for sc in (cs, None):
        y = _compare(x, pr, th, sc, G, f"{dt} subnormal, scales {sc is not None}")
        assert bool((y != 0).any())


@pytest.mark.parametrize("dt", [F32, F16, BF16])
def test_overflow(ops, dt):
    """Values near the largest finite one in group 0 of every other row: the scale product or a rotation overflows to inf, and
    inf meets finite values and other infs (inf - inf = NaN) in later stages; the other groups stay finite.  Same values,
    same positions."""
    K, G = 1024, 128
    pr, th, cs = _layer(K, G, 8, seed=402, theta_uniform_pi=True)
    g = torch.Generator(device="cuda").manual_seed(403)
    big = torch.finfo(dt).max * 0.9
    x = torch.randn(13, K, generator=g, device="cuda")
    x[::2, 0:G:5] = big * torch.sign(torch.randn(7, (G + 4) // 5, generator=g, device="cuda"))
    x = x.to(dt)
    assert bool(torch.isfinite(x).all())
    for sc in (cs, None):
        y = _compare(x, pr, th, sc, G, f"{dt} overflow, scales {sc is not None}")
        assert bool((~torch.isfinite(y[::2, :G])).any()) and bool(torch.isfinite(y[:, G:]).all())
