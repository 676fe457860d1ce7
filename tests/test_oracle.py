"""CPU tests of the oracle itself: two independent restatements agree bit for bit, algebraic
known-answer tests (SURVEY.md section 4), and -- when present -- the fixtures captured from the
unmodified reference kernels on an H100 (tests/golden/ref_gpu_*.npz)."""
import numpy as np
import pytest
import torch

from paroquant_b200.checkpoint import (make_synthetic_activations, make_synthetic_layer, pack_awq, unpack_awq)

from conftest import GOLDEN

DTYPES = ["bfloat16", "float16", "float32"]


def _layer(K=512, parts=(256, 128), seed=7, **kw):
    L = make_synthetic_layer(K, list(parts), seed=seed, **kw)
    return L, L.numpy_dict()


def test_awq_pack_unpack_roundtrip(oracle):
    L, d = _layer()
    v = oracle.np_awq_unpack(d["qweight"])
    assert v.min() >= 0 and v.max() <= 15
    assert (oracle.c_awq_unpack(d["qweight"]) == v).all()
    assert (oracle.np_awq_pack(v) == d["qweight"]).all()
    assert (oracle.c_awq_pack(v) == d["qweight"]).all()
    # product-side helpers use the same nibble order (convert.py:19)
    assert (unpack_awq(L.qweight).numpy() == v).all()
    assert (pack_awq(torch.from_numpy(v.astype(np.int32))).numpy() == d["qweight"]).all()


def test_awq_known_word():
    # columns 0..7 = 0..7 -> nibbles in slot order (0,2,4,6,1,3,5,7): 0x75316420
    from oracle import oracle as O
    w = O.np_awq_pack(np.arange(8, dtype=np.uint8)[None, :])
    assert (w.view(np.uint32)[0, 0]) == 0x75316420


def test_half_conversions_match_numpy_and_torch(oracle):
    rng = np.random.default_rng(0)
    x = np.concatenate([rng.standard_normal(20000).astype(np.float32) * 10.0 ** rng.integers(-8, 5, 20000),
                        np.array([0.0, -0.0, 65504.0, 65520.0, 1e-8, 6e-8, 2.0 ** -24, 2.0 ** -25, 3.0 * 2.0 ** -25], np.float32)]).astype(np.float32)
    import ctypes
    for dt, code in (("float16", 1), ("bfloat16", 2)):
        out = np.empty(x.size, np.uint16)
        oracle._c().paro_oracle_f32_to_half(oracle._p(x), oracle._p(out), ctypes.c_int64(x.size), ctypes.c_int(code))
        ref = torch.from_numpy(x).to(torch.float16 if code == 1 else torch.bfloat16).view(torch.int16).numpy().view(np.uint16)
        assert (out == ref).all(), dt
        assert (oracle.to_bits(oracle.round_to(x, dt), dt) == ref).all(), dt


@pytest.mark.parametrize("dt", DTYPES)
def test_c_and_numpy_restatements_agree(oracle, dt):
    L, d = _layer()
    assert (oracle.np_dequant(d["qweight"], d["qzeros"], d["scales"], 128, dt)
            == oracle.c_dequant(d["qweight"], d["qzeros"], d["scales"], 128, dt)).all()
    x = make_synthetic_activations(9, 512, dtype=torch.float32).numpy()
    for p in range(2):
        a = oracle.np_rotate(x, d["pairs"][p], d["theta"][p], d["channel_scales"][p], 128, dt)
        b = oracle.c_rotate(x, d["pairs"][p], d["theta"][p], d["channel_scales"][p], 128, dt)
        assert (a == b).all()
    assert (oracle.linear(x, d, dt, "np") == oracle.linear(x, d, dt, "c")).all()


@pytest.mark.parametrize("dt", DTYPES)
@pytest.mark.parametrize("G,krot", [(128, 8), (64, 3), (128, 16)])
def test_np_rotate_sincos_table_of_the_default_values_is_the_default(oracle, dt, G, krot):
    """np_rotate(sincos=(fp32(cos T(theta)), fp32(sin T(theta)))) is np_rotate bit for bit: the table replaces exactly the
    sin / cos and nothing else.  A table of other values changes the result."""
    L = make_synthetic_layer(512, [64], group_size=G, krot=krot, seed=11, theta_uniform_pi=True)
    d = L.numpy_dict()
    x = make_synthetic_activations(7, 512, dtype=torch.float32).numpy()
    th = oracle.round_to(d["theta"][0], dt).astype(np.float64)
    table = (np.cos(th).astype(np.float32), np.sin(th).astype(np.float32))
    for sc in (d["channel_scales"][0], None):
        a = oracle.np_rotate(x, d["pairs"][0], d["theta"][0], sc, G, dt)
        b = oracle.np_rotate(x, d["pairs"][0], d["theta"][0], sc, G, dt, sincos=table)
        assert np.array_equal(a.view(np.uint32), b.view(np.uint32))
    off = (table[0], np.nextafter(table[1], np.float32(2)) * np.float32(1.01))
    assert not np.array_equal(a, oracle.np_rotate(x, d["pairs"][0], d["theta"][0], None, G, dt, sincos=off))


@pytest.mark.parametrize("dt", DTYPES)
def test_rotate_theta_zero_is_identity(oracle, dt):
    _, d = _layer()
    x = make_synthetic_activations(4, 512, dtype=torch.float32).numpy()
    y = oracle.c_rotate(x, d["pairs"][0], np.zeros_like(d["theta"][0]), None, 128, dt)
    assert (y == oracle.round_to(x, dt)).all()


def test_rotate_inverse_and_norm_fp32(oracle):
    """rotate(theta) then rotate(reversed order, -theta) is the identity; each 128-group keeps its
    norm (qlinear.py:111-119)."""
    _, d = _layer(theta_uniform_pi=True)
    x = make_synthetic_activations(3, 512, dtype=torch.float32).numpy()
    pr, th = d["pairs"][0], d["theta"][0]
    y = oracle.c_rotate(x, pr, th, None, 128, "float32")
    nx = np.linalg.norm(x.reshape(3, 4, 128), axis=-1)
    ny = np.linalg.norm(y.reshape(3, 4, 128), axis=-1)
    assert np.allclose(nx, ny, rtol=1e-5)
    back = oracle.c_rotate(y, pr[::-1].copy(), -th[::-1].copy(), None, 128, "float32")
    assert np.allclose(back, x, rtol=0, atol=1e-4 * np.abs(x).max())


def test_rotate_group64_and_krot1(oracle):
    L = make_synthetic_layer(256, [64], group_size=64, krot=1, seed=3)
    d = L.numpy_dict()
    x = make_synthetic_activations(2, 256, dtype=torch.float32).numpy()
    a = oracle.np_rotate(x, d["pairs"][0], d["theta"][0], d["channel_scales"][0], 64, "float16")
    b = oracle.c_rotate(x, d["pairs"][0], d["theta"][0], d["channel_scales"][0], 64, "float16")
    assert (a == b).all()
    # one rotation, pair (i, j): explicit 2x2 check on the first pair of row 0, group 0
    i, j = int(d["pairs"][0][0, 0]), int(d["pairs"][0][0, 1])
    th = float(oracle.round_to(d["theta"][0][0, :1], "float16")[0])
    v = oracle.round_to(oracle.round_to(x[0, :64], "float16") * oracle.round_to(d["channel_scales"][0][0, :64], "float16"), "float16")
    exp_i = np.float32(np.cos(th)) * v[i] + np.float32(np.sin(th)) * v[j]
    assert abs(float(a[0, i]) - float(exp_i)) <= 2e-3 * max(1.0, abs(float(exp_i)))


@pytest.mark.parametrize("G,krot,with_scale", [(128, 8, True), (64, 3, True), (128, 2, False)])
def test_rotate_backward_matches_autograd_of_the_dense_formulation(oracle, G, krot, with_scale):
    """oracle.np_rotate_backward (the reference's backward formulas, autograd.py:20-61, in float64) against torch autograd
    through an explicit dense float64 formulation of the same rotation: gradients w.r.t. x, theta and the channel scales."""
    K, M = 256, 5
    L = make_synthetic_layer(K, [64], group_size=G, krot=krot, seed=23)
    pr = L.pairs[0]
    th = L.theta[0].double().requires_grad_(True)
    sc = L.channel_scales[0].double().view(-1).requires_grad_(with_scale)
    g = torch.Generator().manual_seed(3)
    x = torch.randn(M, K, generator=g, dtype=torch.float64, requires_grad=True)
    w = torch.randn(M, K, generator=g, dtype=torch.float64)

    def dense(x, th, sc):
        v = x * sc if with_scale else x
        base = (torch.arange(K) // G * G).view(K // 2, 2)[:, 0]
        for r in range(krot):
            p = pr[r].view(K // 2, 2).long()
            i, j = p[:, 0] + base, p[:, 1] + base
            c, s = th[r].cos(), th[r].sin()
            vi, vj = v[:, i], v[:, j]
            v = v.clone()
            v[:, i] = c * vi + s * vj                            # Appendix A.2: [[c, s], [-s, c]]
            v[:, j] = c * vj - s * vi
        return v

    y = dense(x, th, sc)
    (y * w).sum().backward()
    gx, gth, gsc = oracle.np_rotate_backward(x.detach().numpy(), pr.numpy(), th.detach().numpy(), y.detach().numpy(), w.numpy(),
                                             sc.detach().numpy() if with_scale else None, G)
    assert np.allclose(gx, x.grad.numpy(), rtol=1e-10, atol=1e-12)
    assert np.allclose(gth, th.grad.numpy(), rtol=1e-9, atol=1e-11)
    if with_scale:
        assert np.allclose(gsc, sc.grad.numpy(), rtol=1e-10, atol=1e-12)
    else:
        assert gsc is None
    # the expression the reference evaluates (autograd.py:50-52, after un-rotating g as well) is NOT this gradient: it returns
    # cos * dL/dtheta - sin * sum_rows(g . t); same grad_x / grad_scale
    gx2, gth_ref, _ = oracle.np_rotate_backward(x.detach().numpy(), pr.numpy(), th.detach().numpy(), y.detach().numpy(), w.numpy(),
                                                sc.detach().numpy() if with_scale else None, G, reference_formula=True)
    assert np.array_equal(gx2, gx)
    assert not np.allclose(gth_ref, th.grad.numpy(), rtol=1e-3, atol=1e-6)
    last = th.detach().numpy()[krot - 1]
    base = (np.arange(K) // G * G).reshape(K // 2, 2)[:, 0]
    pl = pr[krot - 1].numpy().astype(np.int64).reshape(K // 2, 2)
    i, j = pl[:, 0] + base, pl[:, 1] + base
    yn, wn = y.detach().numpy(), w.numpy()
    dot = (wn[:, i] * yn[:, i] + wn[:, j] * yn[:, j]).sum(0)      # g . t of a pair is rotation invariant: use the stage output
    assert np.allclose(gth_ref[krot - 1], np.cos(last) * th.grad.numpy()[krot - 1] - np.sin(last) * dot, rtol=1e-9, atol=1e-11)


def test_linear_equals_pseudo_weight_identity(oracle):
    """Appendix A.4: rotate(x * cs) . W == x . (cs * R^T W) -- checked in fp32 on a tiny layer."""
    _, d = _layer(K=256, parts=(32,), seed=11)
    x = make_synthetic_activations(2, 256, dtype=torch.float32).numpy()
    W = oracle.c_dequant(d["qweight"], d["qzeros"], d["scales"], 128, "float32").astype(np.float64)
    xr = oracle.c_rotate(x, d["pairs"][0], d["theta"][0], d["channel_scales"][0], 128, "float32").astype(np.float64)
    # R as an explicit matrix: rotate the identity rows
    R = oracle.c_rotate(np.eye(256, dtype=np.float32), d["pairs"][0], d["theta"][0], None, 128, "float32").astype(np.float64)
    cs = oracle.round_to(d["channel_scales"][0][0], "float32").astype(np.float64)
    lhs = xr @ W
    rhs = (x.astype(np.float64) * cs) @ R @ W
    assert np.allclose(lhs, rhs, rtol=1e-4, atol=1e-5)


def test_bias_added_in_T(oracle):
    _, d = _layer(K=256, parts=(32,), seed=5, bias=True)
    x = make_synthetic_activations(1, 256, dtype=torch.float32).numpy()
    y = oracle.linear(x, d, "bfloat16")
    d2 = dict(d, bias=None)
    y0 = oracle.linear(x, d2, "bfloat16")
    assert (y == oracle.round_to(y0 + oracle.round_to(d["bias"], "bfloat16"), "bfloat16")).all()


# ---------------------------------------------------------------- fixtures from the real reference
_rot_golden = sorted(GOLDEN.glob("ref_gpu_rotate_*.npz"))
_lin_golden = sorted(GOLDEN.glob("ref_gpu_linear_*.npz"))


@pytest.mark.skipif(not _rot_golden, reason="reference GPU fixtures not generated yet")
@pytest.mark.parametrize("path", _rot_golden, ids=lambda p: p.stem)
def test_oracle_vs_reference_rotate_kernel(oracle, path):
    """Oracle against the UNMODIFIED reference rotate kernel's output.  The only modelled
    difference is MUFU sin/cos vs correctly rounded sin/cos: a small fraction of elements may
    differ, each by at most a few ulps of T."""
    z = np.load(path)
    dt = str(z["dtype"])
    scales = z["scales"] if "scales" in z.files else None
    got = oracle.c_rotate(oracle.from_bits(z["x"], dt), z["pairs"], oracle.from_bits(z["theta"], str(z["theta_dtype"])),
                          None if scales is None else oracle.from_bits(scales, str(z["theta_dtype"])), int(z["group"]), dt)
    ref = oracle.from_bits(z["out"], dt)
    frac = float((got != ref).mean())
    assert oracle.rel_err(got, ref) < (2e-6 if dt == "float32" else 1.5e-3), (frac, oracle.rel_err(got, ref))
    if dt != "float32":
        assert frac < 0.03, frac


@pytest.mark.skipif(not _lin_golden, reason="reference GPU fixtures not generated yet")
@pytest.mark.parametrize("path", _lin_golden, ids=lambda p: p.stem)
def test_oracle_vs_reference_rotate_marlin(oracle, path):
    z = np.load(path)
    dt = str(z["dtype"])
    layer = {"qweight": z["qweight"], "qzeros": z["qzeros"], "scales": oracle.from_bits(z["scales"], "float16"),
             "theta": oracle.from_bits(z["theta"], "float16"), "pairs": z["pairs"],
             "channel_scales": oracle.from_bits(z["channel_scales"], "float16"),
             "part_sizes": [int(v) for v in z["part_sizes"]], "group": 128, "bias": None}
    got = oracle.linear(oracle.from_bits(z["x"], dt), layer, dt)
    ref = oracle.from_bits(z["y"], dt)
    assert oracle.rel_err(got, ref) < 1e-3, oracle.rel_err(got, ref)
    if "w_onehot" in z.files:   # Marlin's dequantised operand, read out with one-hot activations
        W = oracle.c_dequant(z["qweight"], z["qzeros"], layer["scales"], 128, dt)
        rows = z["w_rows"]
        assert (W[rows] == oracle.from_bits(z["w_onehot"], dt)).all()
