"""The fused rotate backward (paro_rotate_backward, the op behind scaled_pairwise_rotation's backward) element by element, at
the shapes it is built for: every warp sums several 4-row blocks of its group before its atomics.

The stage values t_r and g_r the kernel works on are restated exactly by the reference's walk (`backward_restated`: one-rotation
rotate-op launches with -theta, equal to `exact_rotate` value for value), so

  * grad_x must equal T(g * scale) of that walk value for value;
  * grad_theta and grad_scale are fp32 sums in an order the atomics decide: every entry must lie within
    `check_backward_theta` / `check_backward_scale`'s bound of the exact fp64 sum, whose depth comes from the launch plan
    (paro_debug_rotate_backward_plan) at the device's SM count.  Each case also asserts, through that plan, the blocks per warp
    or the dynamic shared memory it is there for (tests/rotate_backward_cases.py).

An integer case with theta = 0 pins all three outputs bit for bit, and run to run; a non-finite gradient must stay in its group.
Random data stays in the normal range: the kernel flushes fp32 subnormals, torch's reference products do not.
"""
import pytest
import torch

from gpu_reference import assert_same_values, backward_restated, check_backward_scale, check_backward_theta, kernel_sincos
from paroquant_b200.checkpoint import make_synthetic_layer
from rotate_backward_cases import CASES, assert_plan_reaches, case_id

pytestmark = pytest.mark.gpu
F32, F16, BF16 = torch.float32, torch.float16, torch.bfloat16


@pytest.fixture(scope="module")
def ops():
    import paroquant_b200.kernels.cuda as k  # registers torch.ops.rotation.rotate
    return k


def _plan(M, K, krot, G, dt, ref):
    from paroquant_b200 import _cabi
    return _cabi.debug_rotate_backward_plan(M, K, krot, G, dt, ref)


def _normal(shape, g, dt):
    """randn in dt with |v| >= 2^-8: no product of two values is an fp32 subnormal."""
    v = torch.randn(*shape, generator=g)
    return (v.sign() + (v == 0)) * v.abs().clamp(min=2.0 ** -8)


def _layer(dt, G, krot, M, K, seed, theta_dtype=F32, scale_dtype=F32):
    L = make_synthetic_layer(K, [64], group_size=G, krot=krot, seed=seed)
    g = torch.Generator().manual_seed(seed + 1)
    pr = L.pairs[0].cuda()
    th = L.theta[0].float().to(theta_dtype).cuda()
    sc = None if scale_dtype is None else L.channel_scales[0].float().to(scale_dtype).cuda().view(-1)
    x = _normal((M, K), g, dt).to(dt).cuda()
    go = _normal((M, K), g, dt).to(dt).cuda()
    y = torch.ops.rotation.rotate(x, pr, th, sc, G)
    return x, pr, th, sc, y, go


def _sincos(th, dt):
    """The kernel's own {cos, sin}(-T(theta)) (the fp32 kernel reads theta as stored)."""
    return kernel_sincos(-(th.float().to(dt).float()))


def _check(dt, G, krot, M, K, ref_formula, x, pr, th, sc, y, go, what, R=None, skip_groups=()):
    """One launch of the backward checked against the restated walk; returns (grad_theta ratio, grad_scale ratio, outputs)."""
    from paroquant_b200 import _cabi
    plan = _plan(M, K, krot, G, dt, ref_formula)
    gx, gth, gsc = _cabi.rotate_backward(y, go, x, pr, th, sc, G, reference_formula=ref_formula)
    if R is None:
        R = backward_restated(x, pr, th, y, go, sc, G)
    assert_same_values(gx, R["grad_x"], f"{what}: grad_x")
    c, s = _sincos(th, dt)
    rt = check_backward_theta(gth, R, c, s, G, plan["max_blocks_per_warp"], plan["splits"], ref_formula, skip_groups,
                              what=f"{what}: grad_theta")
    rs = None
    if sc is None:
        assert gsc is None
    else:
        rs = check_backward_scale(gsc, R, G, plan["max_blocks_per_warp"], plan["splits"], skip_groups, what=f"{what}: grad_scale")
    print(f"[bwd] {what}: splits {plan['splits']}, blocks per warp {plan['min_blocks_per_warp']}..{plan['max_blocks_per_warp']}, "
          f"dyn smem {plan['dyn_smem']} B; max err/tol grad_theta {rt:.3g}" + ("" if rs is None else f", grad_scale {rs:.3g}"))
    return rt, rs, (gx, gth, gsc)


@pytest.mark.parametrize("case", CASES, ids=case_id)
def test_backward_elementwise(ops, case):
    dt, G, krot, M, K, forms, kind = case
    for f in forms:
        assert_plan_reaches(_plan(M, K, krot, G, dt, f), kind, M, f"{case_id(case)} reference_formula={f}")
    x, pr, th, sc, y, go = _layer(dt, G, krot, M, K, seed=700 + krot)
    R = backward_restated(x, pr, th, y, go, sc, G)
    for f in forms:
        _check(dt, G, krot, M, K, f, x, pr, th, sc, y, go, f"{case_id(case)} ref={int(f)}", R)


SCALE_M, SCALE_K = 4099, 2048        # G 128: 16 groups, every warp walks 7 or 8 row blocks at 132 SMs, the last one ragged


@pytest.mark.parametrize("dt", [F32, F16, BF16])
@pytest.mark.parametrize("form", [None, F16, BF16, F32], ids=["no-scales", "f16", "bf16", "f32"])
def test_backward_scale_and_theta_forms(ops, dt, form):
    """No channel scales, or scales and theta both stored as f16, bf16 or f32, for every x dtype."""
    M, K, G, krot = SCALE_M, SCALE_K, 128, 8
    assert_plan_reaches(_plan(M, K, krot, G, dt, False), "multi", M)
    x, pr, th, sc, y, go = _layer(dt, G, krot, M, K, seed=810, theta_dtype=form or F32, scale_dtype=form)
    _check(dt, G, krot, M, K, False, x, pr, th, sc, y, go, f"{dt} scales/theta {form}")


@pytest.mark.parametrize("dt,G,M,K", [(F32, 128, 14333, 4096), (BF16, 128, 16383, 128)])
def test_backward_exact_on_integers(ops, dt, G, M, K):
    """theta = 0 and integer data: every product and partial sum is exact in fp32 in any order, so all three outputs equal the
    integer sums bit for bit, for both theta formulas, launch after launch."""
    from paroquant_b200 import _cabi
    c0, s0 = kernel_sincos(torch.tensor([-0.0]))
    assert float(c0[0]) == 1.0 and float(s0[0]) == 0.0
    krot = 8
    gen = torch.Generator().manual_seed(900 + M)
    L = make_synthetic_layer(K, [64], group_size=G, krot=krot, seed=901)
    pr = L.pairs[0].cuda()
    th = torch.zeros(krot, K // 2, device="cuda")
    sc = (2.0 ** torch.randint(-2, 3, (K,), generator=gen).float()).cuda()
    x, y, go = (torch.randint(-8, 9, (M, K), generator=gen).float().to(dt).cuda() for _ in range(3))
    plan = _plan(M, K, krot, G, dt, False)
    assert plan["max_blocks_per_warp"] >= 2
    # expected: the stage values never change, so every rotation sums the same t = y, g = go over its own pairs
    base = (torch.arange(K, device="cuda") // G * G).view(K // 2, 2)[:, 0]
    want = torch.zeros(krot, K // 2, dtype=torch.float64, device="cuda")
    for r in range(krot):
        p = pr[r].view(K // 2, 2).long()
        ci, cj = p[:, 0] + base, p[:, 1] + base
        want[r] = (go[:, ci].double() * y[:, cj].double() - go[:, cj].double() * y[:, ci].double()).sum(0)
    assert float(want.abs().max()) < 2.0 ** 24
    want_sc = (x.double() * go.double()).sum(0)
    want_x = (go.float() * sc).to(dt)
    bits = lambda t: t.contiguous().view(torch.int32 if t.dtype == F32 else torch.int16)
    for ref in (False, True):
        for launch in range(2):
            gx, gth, gsc = _cabi.rotate_backward(y, go, x, pr, th, sc, G, reference_formula=ref)
            assert torch.equal(bits(gx), bits(want_x)), (ref, launch)
            assert torch.equal(bits(gth), bits(want.float())), (ref, launch, int((gth != want.float()).sum()))
            assert torch.equal(bits(gsc), bits(want_sc.float())), (ref, launch)


def test_backward_non_finite_stays_in_its_group(ops):
    """One inf in dL/dy at (row m, group g): grad_x is the restated walk's as values (inf / NaN where the walk has them); every
    other group's grad_theta and grad_scale is finite and within the bound."""
    dt, G, krot, M, K = F32, 128, 8, SCALE_M, SCALE_K
    x, pr, th, sc, y, go = _layer(dt, G, krot, M, K, seed=820)
    m, grp = 2901, 11
    go[m, grp * G + 37] = float("inf")
    _, _, (gx, gth, gsc) = _check(dt, G, krot, M, K, False, x, pr, th, sc, y, go, "inf in dL/dy", skip_groups=[grp])
    assert not bool(torch.isfinite(gx[m, grp * G:(grp + 1) * G]).all())
    assert not bool(torch.isfinite(gth[:, grp * G // 2:(grp + 1) * G // 2]).all())
    assert not bool(torch.isfinite(gsc[grp * G:(grp + 1) * G]).all())


def test_backward_reproducibility_as_it_is(ops):
    """grad_x is the same launch after launch; grad_theta and grad_scale are fp32 atomics in no fixed order, so they are only
    required to lie within the bound every time."""
    dt, G, krot, M, K = F32, 128, 8, 14333, 4096
    x, pr, th, sc, y, go = _layer(dt, G, krot, M, K, seed=830)
    R = backward_restated(x, pr, th, y, go, sc, G)
    runs = [_check(dt, G, krot, M, K, False, x, pr, th, sc, y, go, f"launch {i}", R)[2] for i in range(3)]
    for gx, gth, gsc in runs[1:]:
        assert torch.equal(gx.view(torch.int32), runs[0][0].view(torch.int32))
    print(f"[bwd] grad_theta entries that differ between launches 0 and 1: {int((runs[0][1] != runs[1][1]).sum())} of {runs[0][1].numel()}")


@pytest.mark.parametrize("theta_dtype,with_scale,reference", [(F32, True, False), (F16, True, False), (F32, False, False),
                                                               (F16, True, True)])
def test_autograd_at_a_training_shape(ops, monkeypatch, theta_dtype, with_scale, reference):
    """scaled_pairwise_rotation on x [4, 1024, 4096] bf16 with a non-contiguous upstream gradient: gradient dtypes and shapes,
    x.grad equal to the fused launch's grad_x bit for bit, theta.grad and scale.grad (cast to the parameters' dtype) within
    the bound."""
    from paroquant_b200 import _cabi
    from paroquant_b200.kernels.cuda import autograd, scaled_pairwise_rotation
    monkeypatch.setattr(autograd, "REFERENCE_THETA_EXPRESSION", reference)
    B, N, K, G, krot, dt = 4, 1024, 4096, 128, 8, BF16
    M = B * N
    L = make_synthetic_layer(K, [64], group_size=G, krot=krot, seed=840)
    gen = torch.Generator().manual_seed(841)
    pr = L.pairs[0].cuda()
    th = L.theta[0].float().to(theta_dtype).cuda().requires_grad_(True)
    sc = L.channel_scales[0].float().to(theta_dtype).reshape(1, K).cuda().requires_grad_(True) if with_scale else None
    x = _normal((B, N, K), gen, dt).to(dt).cuda().requires_grad_(True)
    w = _normal((B, K, N), gen, dt).to(dt).cuda().transpose(1, 2)
    assert not w.is_contiguous()
    y = scaled_pairwise_rotation(x, pr, th, sc, G)
    y.backward(w)
    assert x.grad.shape == x.shape and x.grad.dtype == dt
    assert th.grad.shape == th.shape and th.grad.dtype == theta_dtype
    if with_scale:
        assert sc.grad.shape == sc.shape and sc.grad.dtype == theta_dtype
    yd, wd, xd = y.detach().reshape(M, K), w.reshape(M, K).contiguous(), x.detach().reshape(M, K)
    scd = None if sc is None else sc.detach().reshape(-1)
    gx = _cabi.rotate_backward(yd, wd, xd, pr, th.detach(), scd, G, reference_formula=reference)[0]
    assert torch.equal(x.grad.reshape(M, K).view(torch.int16), gx.view(torch.int16))
    plan = _plan(M, K, krot, G, dt, reference)
    assert_plan_reaches(plan, "multi", M)
    R = backward_restated(xd, pr, th.detach(), yd, wd, scd, G)
    c, s = _sincos(th.detach(), dt)
    cast = None if theta_dtype == F32 else theta_dtype
    rt = check_backward_theta(th.grad, R, c, s, G, plan["max_blocks_per_warp"], plan["splits"], reference, cast=cast,
                              what="theta.grad")
    rs = check_backward_scale(sc.grad, R, G, plan["max_blocks_per_warp"], plan["splits"], cast=cast,
                              what="scale.grad") if with_scale else None
    print(f"[bwd] autograd theta {theta_dtype} scales {with_scale} reference {reference}: max err/tol theta.grad {rt:.3g}"
          + ("" if rs is None else f", scale.grad {rs:.3g}"))
