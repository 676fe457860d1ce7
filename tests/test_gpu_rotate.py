"""GPU parity of the standalone rotation kernel (torch.ops.rotation.rotate surface), called
through the C-ABI.

Three references:
  * tests/golden/ref_gpu_rotate_*.npz -- outputs of the UNMODIFIED reference kernel captured on a
    H100: BIT-EXACT equality is required (same rounding points, same MUFU sin/cos);
  * the CPU oracle: identical except for MUFU vs correctly rounded sin/cos (bounded fraction of
    one-ulp flips);
  * size-independent properties at BASELINE sizes (theta = 0 identity, rotate / un-rotate
    round trip, per-group norm preservation).
"""
import numpy as np
import pytest
import torch

from paroquant_b200.checkpoint import make_synthetic_activations, make_synthetic_layer

from conftest import GOLDEN
from gpu_reference import backward_restated

pytestmark = pytest.mark.gpu
_TD = {"float32": torch.float32, "float16": torch.float16, "bfloat16": torch.bfloat16}


@pytest.fixture(scope="module")
def ops():
    import paroquant_b200.kernels.cuda as k  # registers torch.ops.rotation.rotate
    return k


def _from_bits(a, dt):
    t = torch.from_numpy(np.ascontiguousarray(a))
    return t if dt == "float32" else t.view(torch.int16).view(_TD[dt])


def _bits(t):
    t = t.detach().cpu().contiguous()
    return t.numpy() if t.dtype == torch.float32 else t.view(torch.int16).numpy().view(np.uint16)


_rot_golden = sorted(GOLDEN.glob("ref_gpu_rotate_*.npz"))


@pytest.mark.skipif(not _rot_golden, reason="reference GPU fixtures not generated yet")
@pytest.mark.parametrize("path", _rot_golden, ids=lambda p: p.stem)
def test_bit_exact_vs_reference_kernel_fixture(ops, path):
    z = np.load(path)
    dt = str(z["dtype"])
    x = _from_bits(z["x"], dt).cuda()
    th = _from_bits(z["theta"], "float16").cuda()
    sc = _from_bits(z["scales"], "float16").cuda() if "scales" in z.files else None
    out = torch.ops.rotation.rotate(x, torch.from_numpy(z["pairs"]).cuda(), th, sc, int(z["group"]))
    assert np.array_equal(_bits(out), z["out"]), f"{(_bits(out) != z['out']).mean():.4%} of elements differ"


@pytest.mark.parametrize("dt", ["bfloat16", "float16", "float32"])
@pytest.mark.parametrize("M,K,G,krot", [(1, 4096, 128, 8), (16, 4096, 128, 8), (37, 1024, 128, 8), (9, 512, 64, 1), (5, 256, 64, 8),
                                         (4, 1024, 128, 2), (7, 512, 64, 3), (17, 1024, 128, 9), (3, 2048, 64, 16)])
def test_vs_oracle(ops, oracle, dt, M, K, G, krot):
    L = make_synthetic_layer(K, [64], group_size=G, krot=krot, seed=21)
    x = make_synthetic_activations(M, K, seed=5, dtype=_TD[dt])
    got = torch.ops.rotation.rotate(x.cuda(), L.pairs[0].cuda(), L.theta[0].cuda(), L.channel_scales[0].cuda(), G).float().cpu().numpy()
    d = L.numpy_dict()
    ref = oracle.c_rotate(x.float().numpy(), d["pairs"][0], d["theta"][0], d["channel_scales"][0], G, dt)
    # MUFU sin/cos vs libm: rare one-ulp flips after the per-stage rounding to T
    assert oracle.rel_err(got, ref) < (3e-6 if dt == "float32" else 1.5e-3)
    if dt != "float32":
        assert (got != ref).mean() < 0.03


@pytest.mark.parametrize("dt", [torch.bfloat16, torch.float16, torch.float32])
def test_properties_at_full_size(ops, dt):
    M, K = 256, 4096
    L = make_synthetic_layer(K, [64], seed=33, theta_uniform_pi=True)
    x = make_synthetic_activations(M, K, seed=6, dtype=dt).cuda()
    pr, th = L.pairs[0].cuda(), L.theta[0].cuda()
    # theta = 0, no scale: exact identity
    assert torch.equal(torch.ops.rotation.rotate(x, pr, torch.zeros_like(th), None, 128), x)
    y = torch.ops.rotation.rotate(x, pr, th, None, 128)
    tol = {torch.float32: 1e-5, torch.float16: 4e-3, torch.bfloat16: 3e-2}[dt]
    nx = x.float().view(M, -1, 128).norm(dim=-1)
    ny = y.float().view(M, -1, 128).norm(dim=-1)
    assert ((nx - ny).abs() <= tol * nx).all()
    # un-rotate: reversed order, negated angles (qlinear.py:111-119 uses the same construction)
    back = torch.ops.rotation.rotate(y, pr.flip(0).contiguous(), (-th).flip(0).contiguous(), None, 128)
    err = (back.float() - x.float()).norm() / x.float().norm()
    assert err < tol
    # linear in x (same parameters): rotate(2x) == 2 rotate(x) exactly (power-of-two scaling; fp16 is
    # excluded: its subnormal range makes tiny products round differently after scaling)
    if dt != torch.float16:
        assert torch.equal(torch.ops.rotation.rotate(x * 2, pr, th, None, 128), y * 2)


def test_shapes_dtypes_and_errors(ops):
    L = make_synthetic_layer(512, [64], seed=2)
    pr, th, cs = L.pairs[0].cuda(), L.theta[0].cuda(), L.channel_scales[0].cuda()
    x = torch.randn(2, 3, 512, device="cuda", dtype=torch.bfloat16)
    y = torch.ops.rotation.rotate(x, pr, th, cs)
    assert y.shape == x.shape and y.dtype == x.dtype
    assert torch.equal(y.view(6, 512), torch.ops.rotation.rotate(x.view(6, 512), pr, th, cs))
    # scales given as [K] or [1, K]; theta given in another float dtype is cast like theta.to(x.dtype)
    assert torch.equal(torch.ops.rotation.rotate(x, pr, th, cs.view(-1)), y)
    assert torch.equal(torch.ops.rotation.rotate(x, pr, th.to(torch.bfloat16), cs.to(torch.bfloat16)), y)
    assert torch.ops.rotation.rotate(x[:0], pr, th, cs).shape == (0, 3, 512)
    with pytest.raises(RuntimeError, match="Unsupported group_size"):
        torch.ops.rotation.rotate(x, pr, th, cs, 32)
    with pytest.raises(RuntimeError, match="theta.size\\(0\\) must equal idx_ij.size\\(0\\)"):
        torch.ops.rotation.rotate(x, pr[:4], th, cs)
    with pytest.raises(RuntimeError, match="Float, Half, and BFloat16"):
        torch.ops.rotation.rotate(x.to(torch.float64), pr, th, cs)


def test_autograd_matches_dense_jacobian(ops):
    """RotateTensorFunc: gradients w.r.t. x, theta and scale against autograd through an explicit
    fp32 dense formulation of the same rotation."""
    from paroquant_b200.kernels.cuda import scaled_pairwise_rotation

    torch.manual_seed(0)
    K, G, R, M = 256, 128, 8, 6
    L = make_synthetic_layer(K, [64], seed=8)
    pr = L.pairs[0].cuda()
    th = L.theta[0].float().cuda().requires_grad_(True)
    sc = L.channel_scales[0].float().cuda().view(-1).requires_grad_(True)
    x = torch.randn(M, K, device="cuda", requires_grad=True)
    w = torch.randn(M, K, device="cuda")

    def dense(x, th, sc):
        v = x * sc
        base = (torch.arange(K, device="cuda") // G * G).view(K // 2, 2)[:, 0]
        for r in range(R):
            p = pr[r].view(K // 2, 2).long()
            i, j = p[:, 0] + base, p[:, 1] + base
            c, s = th[r].cos(), th[r].sin()
            vi, vj = v[:, i], v[:, j]
            v = v.clone()
            v[:, i] = c * vi + s * vj
            v[:, j] = c * vj - s * vi
        return v

    (dense(x, th, sc) * w).sum().backward()
    gx, gt, gs = x.grad.clone(), th.grad.clone(), sc.grad.clone()
    x.grad = th.grad = sc.grad = None
    (scaled_pairwise_rotation(x, pr, th, sc, G) * w).sum().backward()
    for a, b in ((x.grad, gx), (th.grad, gt), (sc.grad, gs)):
        assert (a - b).norm() / b.norm() < 2e-5


@pytest.mark.parametrize("dt,G,krot,M,with_scale", [
    (torch.float32, 128, 8, 1037, True),       # ragged last block; at K 1024 every warp walks one row block (multi-block sums:
                                               # tests/test_gpu_rotate_backward.py)
    (torch.float32, 64, 8, 333, True),
    (torch.float32, 128, 3, 5, False),         # no channel scales, krot != 8
    (torch.bfloat16, 128, 8, 260, True),       # t and g rounded to bf16 after every rotation, like the per-rotation launches
    (torch.float16, 64, 16, 77, True),
])
def test_fused_backward_equals_the_stagewise_walk(ops, dt, G, krot, M, with_scale):
    from paroquant_b200 import _cabi
    K = 1024
    L = make_synthetic_layer(K, [64], group_size=G, krot=krot, seed=31)
    pr, th = L.pairs[0].cuda(), L.theta[0].float().cuda()
    sc = L.channel_scales[0].float().cuda().view(-1) if with_scale else None
    x = torch.randn(M, K, device="cuda").to(dt)
    go = torch.randn(M, K, device="cuda").to(dt)
    y = torch.ops.rotation.rotate(x, pr, th, sc, G)
    gx, gth, gsc = _cabi.rotate_backward(y, go, x, pr, th, sc, G)
    R = backward_restated(x, pr, th, y, go, sc, G)    # the reference's walk: one-rotation rotate launches with -theta
    rx, rth, rsc = R["grad_x"], R["S"], R["xg"]
    # grad_x: the same arithmetic at the same rounding points -> identical
    assert torch.equal(gx, rx)
    # row sums: fp32 atomics in another order than torch's reduction
    assert (gth - rth).norm() / rth.norm() < 1e-5
    if with_scale:
        assert (gsc - rsc).norm() / rsc.norm() < 1e-5
    else:
        assert gsc is None


def test_autograd_group64_bf16_runs_through_the_op(ops):
    from paroquant_b200.kernels.cuda import scaled_pairwise_rotation
    K, G, M = 512, 64, 9
    L = make_synthetic_layer(K, [64], group_size=G, seed=12)
    pr = L.pairs[0].cuda()
    th = L.theta[0].cuda().requires_grad_(True)                       # fp16 parameter: grad comes back in fp16
    sc = L.channel_scales[0].cuda().requires_grad_(True)              # [1, K]
    x = torch.randn(2, M, K, device="cuda", dtype=torch.bfloat16, requires_grad=True)
    scaled_pairwise_rotation(x, pr, th, sc, G).float().square().sum().backward()
    assert x.grad.shape == x.shape and x.grad.dtype == torch.bfloat16
    assert th.grad.shape == th.shape and th.grad.dtype == th.dtype and sc.grad.shape == sc.shape
    # an orthogonal map preserves the norm: d/dtheta of |y|^2 vanishes up to rounding, d/dx = 2 x s^2
    ref = 2 * x.detach().float() * sc.detach().float().reshape(-1) ** 2
    assert (x.grad.float() - ref).norm() / ref.norm() < 2e-2
    assert th.grad.float().abs().max() < 0.05 * x.detach().float().square().sum().sqrt()


@pytest.mark.parametrize("G", [128, 64])
def test_fused_backward_vs_oracle_both_theta_formulas(ops, oracle, G):
    """fp32 kernel against the float64 oracle (oracle.np_rotate_backward, pinned to autograd on the CPU): the gradient, and the
    value of the reference's expression (autograd.py:50-52 after un-rotating g: cos * gradient - sin * sum_rows(g . t))."""
    from paroquant_b200 import _cabi
    torch.manual_seed(7)
    K, M = 512, 37
    L = make_synthetic_layer(K, [64], group_size=G, krot=8, seed=33)
    pr, th = L.pairs[0].cuda(), L.theta[0].float().cuda()
    sc = L.channel_scales[0].float().cuda().view(-1)
    x = torch.randn(M, K, device="cuda")
    go = torch.randn(M, K, device="cuda")
    y = torch.ops.rotation.rotate(x, pr, th, sc, G)
    args = (x.cpu().numpy(), pr.cpu().numpy(), th.cpu().numpy(), y.cpu().numpy(), go.cpu().numpy(), sc.cpu().numpy(), G)
    for ref in (False, True):
        gx, gth, gsc = _cabi.rotate_backward(y, go, x, pr, th, sc, G, reference_formula=ref)
        ox, oth, osc = oracle.np_rotate_backward(*args, reference_formula=ref)
        # fp32 kernel with MUFU sin / cos against float64: the dense-Jacobian test above sees ~1e-5
        assert oracle.rel_err(gx.cpu().numpy(), ox) < 5e-5
        assert oracle.rel_err(gth.cpu().numpy(), oth) < 2e-4, ref
        assert oracle.rel_err(gsc.cpu().numpy(), osc) < 5e-5
    a = _cabi.rotate_backward(y, go, x, pr, th, sc, G)[1]
    b = _cabi.rotate_backward(y, go, x, pr, th, sc, G, reference_formula=True)[1]
    assert (a - b).norm() / a.norm() > 1e-2          # the two really differ on random data


# (K, partitions, M, group, krot, dtype): the decode pre-pass (M <= 16: 16 rows in tiles of 16) and the GEMM's (M > 16: m_pad rows in
# tiles of the GEMM's NT); krot 9 and 16 run a second chunk of 8 stages
PREPASS_CASES = [
    (1024, [512], 5, 128, 9, torch.bfloat16),
    (2048, [256, 128, 384], 16, 64, 16, torch.float16),
    (1024, [384], 48, 64, 3, torch.bfloat16),
    (1536, [1024, 256, 256], 300, 128, 16, torch.float16),
    (512, [256], 300, 64, 9, torch.bfloat16),
]


@pytest.mark.parametrize("K,parts,M,G,krot,dt", PREPASS_CASES)
def test_prepass_operand_is_the_rotate_op_bit_for_bit(ops, K, parts, M, G, krot, dt):
    """The tensor-core kernels' pre-pass (rotate_tile_kernel, reading the packed layout's metadata blocks) writes, for every
    partition, exactly torch.ops.rotation.rotate of the same rows in the B-operand tile order, padding rows zero."""
    import ctypes
    from paroquant_b200 import _cabi
    from paroquant_b200.linear import ParoLinearKernel
    L = make_synthetic_layer(K, parts, group_size=G, krot=krot, seed=600 + M, device="cuda")
    k = ParoLinearKernel.from_buffers(L, dt, max_m=M, private_workspace=True)
    x = make_synthetic_activations(M, K, seed=610 + M, device="cuda", dtype=dt)
    k(x)
    assert _cabi.last_launch_count() == 2   # pre-pass + consumer: the rows below were rotated by the pre-pass
    if M <= 16:
        nt = rows = 16
    else:
        plan = (ctypes.c_int32 * 2)()
        sms = torch.cuda.get_device_properties(0).multi_processor_count
        assert _cabi.lib().paro_debug_gemm_plan(ctypes.byref(k.shape), M, sms, plan) == 0
        nt = plan[0]
        rows = (M + nt - 1) // nt * nt
    P = len(parts)
    # behind the 256-byte epoch head: [partition][token block][k16 step][k half][row / 8][row % 8][8 channels]
    op = k.workspace[256:256 + P * rows * K * 2].view(dt).view(P, rows // nt, K // 16, 2, nt // 8, 8, 8)
    op = op.permute(0, 1, 4, 5, 2, 3, 6).reshape(P, rows, K)
    for p in range(P):
        ref = torch.ops.rotation.rotate(x, L.pairs[p], L.theta[p], L.channel_scales[p], G)
        assert torch.equal(op[p, :M].view(torch.int16), ref.view(torch.int16)), p
        assert not op[p, M:].view(torch.int16).any(), p
