"""Every fused path's own rotated operand, bit for bit, through selection weights (tests/selection_layers.py), and the dequantised
operand `dense_weight()` against oracle.c_dequant at every shape the element-wise suite relies on it.

With a selection layer, y[m, n] = T(xr[m, sigma(n)] * d_n * s) exactly whatever the K split or summation order, so the output is
compared for equality with a reference built without the library: xr from oracle.np_rotate on the GPU's own sin / cos
(gpu_reference.exact_rotate), the weights from oracle.np_awq_pack.  The element-wise bound of gpu_reference.check absorbs a
wrong low bit in scattered operand elements and even a wrong element whose |xr_k W_k| is small; here each one shows.  Outputs
start as NaN, so an element not written shows too.  Paths:

  * the single linear at every default plan: in-kernel rotation (M 1..4), the pre-pass (M 5..16), the GEMM at every token
    tile with a ragged last tile; merged partitions with distinct rotations, partial blocks, K up to 14336, group 64 / 128,
    krot 1 .. 16, bf16 / fp16, bias (ref = T(fp32(t + b)));
  * the stream kernel as a one-step chain; decode (M <= 16) and prefill (M > 16) chains with an ADD_RESIDUAL step, an RMSNORM
    step on exact-statistics rows (its operand is exact whatever rstd's last bits), a SILU_MUL step and an ADD_RESIDUAL step
    without y (h = T(fp32(t + r)));
  * the MoE block, decode_step and prefill_step, each expert with its own sigma: every valid h[t, s] exactly, and y exactly
    where a token's one valid slot has weight 1.0, gpu_reference.check_combine on the exact expert outputs otherwise.
The forced launch plans run a selection case each in tests/variant_child.py.
"""
import pytest
import torch

from gpu_reference import assert_same_values, check_combine, exact_bias, exact_rms_rows, exact_rotated, sample_rows
from paroquant_b200 import _cabi
from paroquant_b200.checkpoint import make_synthetic_activations, make_synthetic_layer
from selection_layers import cover, selection_layer
from test_gpu_variants import GEMM_CASES

pytestmark = pytest.mark.gpu
BF, FP = torch.bfloat16, torch.float16
_TD = {"bfloat16": BF, "float16": FP}
# scale exponents of stacked steps: in fp16 a SiLU * up of selection outputs would overflow with the default -2..2
EXPS = {BF: (-2, 2), FP: (-6, -2)}


@pytest.fixture(scope="module")
def mods():
    import paroquant_b200.kernels.cuda  # noqa: F401  registers torch.ops.rotation.rotate
    from paroquant_b200 import chain
    from paroquant_b200.linear import ParoLinearKernel
    return chain, ParoLinearKernel


def _nan(*shape, dt):
    return torch.full(shape, float("nan"), dtype=dt, device="cuda")


def _ref(S, x, dt, bias=None, rows=None):
    """Selection output of x (rows `rows` of it) through S's rotation, bias added in T as T(fp32(t + b))."""
    xs = x if rows is None else x[rows]
    y = S.apply(exact_rotated(S.L, xs), dt)
    return y if bias is None else (y.float() + bias.float()).to(dt)


def _check_linear(S, x, y, dt, bias, what):
    rows = sample_rows(x.shape[0], 8, seed=x.shape[0]).cuda()
    assert_same_values(y[rows], _ref(S, x, dt, bias, rows), what)


# ---------------------------------------------------------------- single linear, default dispatch
# (K, parts, group, krot, dtype, bias)
SINGLE = [
    (1024, [256, 128], 128, 8, "bfloat16", True),
    (640, [48, 16, 32], 64, 3, "float16", False),
    (128, [272, 16], 128, 1, "bfloat16", True),
    (2048, [384], 64, 9, "bfloat16", False),
    (4096, [4096, 1024, 1024], 128, 16, "float16", True),
    (14336, [4096], 128, 8, "bfloat16", False),
]
DECODE_M = (1, 2, 3, 4, 5, 8, 9, 16)


def _cid(c):
    return "-".join(str(v) for v in c)


@pytest.mark.parametrize("case", SINGLE, ids=_cid)
def test_single_linear_decode(mods, case):
    """M 1..4: the decode kernel's in-kernel rotation (ROWS 1 / 2 / 4); M 5..16: the pre-pass (earlier at K >= 8192)."""
    chain, PK = mods
    K, parts, group, krot, dt, with_bias = case
    T = _TD[dt]
    plans = set()
    for shift in cover(K, sum(parts)):
        S = selection_layer(K, parts, group=group, krot=krot, seed=K + krot, shift=shift, bias=with_bias)
        L = S.L.to("cuda")
        k = PK.from_buffers(L, T, check_pairs=False, max_m=16)
        bias = None if L.bias is None else L.bias.to(T)
        for M in DECODE_M:
            x = make_synthetic_activations(M, K, seed=M + shift, device="cuda", dtype=T)
            y = _nan(M, sum(parts), dt=T)
            k.forward_into(x, y, bias)
            plans.add((M, _cabi.last_launch_count()))
            _check_linear(S, x, y, T, bias, f"{_cid(case)} shift {shift} M={M}")
    print(f"[plan] single linear {_cid(case)}: (M, launches) {sorted(plans)}")
    if K < 8192:                                  # in-kernel rotation below 5 rows, the pre-pass from 5
        assert all(n == (2 if M >= 5 else 1) for M, n in plans), plans


@pytest.mark.parametrize("K,parts,M,nt,group,dt,with_bias", GEMM_CASES)
def test_single_linear_gemm_tiles(mods, K, parts, M, nt, group, dt, with_bias):
    chain, PK = mods
    T = _TD[dt]
    for shift in cover(K, sum(parts))[:2]:
        S = selection_layer(K, parts, group=group, krot=8, seed=M, shift=shift, bias=with_bias)
        L = S.L.to("cuda")
        k = PK.from_buffers(L, T, check_pairs=False, max_m=M)
        bias = None if L.bias is None else L.bias.to(T)
        x = make_synthetic_activations(M, K, seed=M + 1, device="cuda", dtype=T)
        y = _nan(M, sum(parts), dt=T)
        k.forward_into(x, y, bias)
        assert _cabi.last_launch_count() == 2
        _check_linear(S, x, y, T, bias, f"GEMM NT={nt} K={K} {parts} M={M} shift {shift}")


# ---------------------------------------------------------------- chains
@pytest.mark.parametrize("dt", [BF, FP])
def test_stream_kernel_one_step_chain(mods, dt):
    chain, PK = mods
    for K, parts, group, krot in ((1024, [256, 128], 128, 8), (2048, [384], 64, 3), (4096, [4096, 1024, 1024], 128, 9)):
        for shift in cover(K, sum(parts)):
            S = selection_layer(K, parts, group=group, krot=krot, seed=K, shift=shift, bias=True)
            L = S.L.to("cuda")
            k = PK.from_buffers(L, dt, check_pairs=False)
            bias = L.bias.to(dt)
            for M in (1, 4, 16):
                x = make_synthetic_activations(M, K, seed=M, device="cuda", dtype=dt)
                y = _nan(M, sum(parts), dt=dt)
                chain.ParoChain([chain.ChainStep(k, x=x, y=y, bias=bias)], M)()
                _check_linear(S, x, y, dt, bias, f"stream K={K} {parts} shift {shift} M={M}")


A_K = 256
# (hidden, intermediate, group, krot of the RMSNORM step)
CHAIN_SHAPES = [(512, 384, 128, 8), (2048, 1024, 64, 3)]


@pytest.mark.parametrize("dt", [BF, FP])
@pytest.mark.parametrize("shape", CHAIN_SHAPES, ids=_cid)
@pytest.mark.parametrize("kind", ["decode", "prefill"])
def test_chain_steps(mods, kind, shape, dt):
    """A: x = 0, bias, ADD_RESIDUAL (h = the exact-statistics rows) -> B: RMSNORM -> gate_up -> C: SILU_MUL -> down ->
    D: a linear of C's y with ADD_RESIDUAL on h and no y.  Every output of B, C and D exactly."""
    chain, PK = mods
    H, I, group, krot = shape
    eps = 1e-8
    seed = H + (1 if dt == FP else 0)
    Sa = selection_layer(A_K, [H], seed=seed)
    Sb = selection_layer(H, [I, I], group=group, krot=krot, seed=seed + 1, exps=EXPS[dt])
    Sc = selection_layer(I, [H], seed=seed + 2, krot=9, exps=EXPS[dt])
    Sd = selection_layer(H, [H], group=64, krot=16, seed=seed + 3, exps=EXPS[dt])
    Ls = [S.L.to("cuda") for S in (Sa, Sb, Sc, Sd)]
    ka, kb, kc, kd = (PK.from_buffers(L, dt, check_pairs=False) for L in Ls)
    w = (1.0 + 0.1 * torch.randn(H, generator=torch.Generator().manual_seed(seed))).to(dt)
    bias = exact_bias(H, seed, dt).cuda()
    wd = w.cuda()
    for M in ((1, 3, 8, 16) if kind == "decode" else (17, 100, 257)):
        h, xop = exact_rms_rows(M, H, dt, seed=seed * 100 + M, w=w, eps=eps)
        h, xop = h.cuda(), xop.cuda()
        r = (h.double() - bias.double()).to(dt)
        ya, hres, yb, yc, hd = _nan(M, H, dt=dt), _nan(M, H, dt=dt), _nan(M, 2 * I, dt=dt), _nan(M, H, dt=dt), _nan(M, H, dt=dt)
        steps = [chain.ChainStep(ka, x=torch.zeros(M, A_K, dtype=dt, device="cuda"), y=ya, bias=bias, epilogue="add_residual",
                                 residual_in=r, residual_out=hres),
                 chain.ChainStep(kb, x_op="rmsnorm", norm_weight=wd, eps=eps, y=yb),
                 chain.ChainStep(kc, x_op="silu_mul", y=yc),
                 chain.ChainStep(kd, epilogue="add_residual", residual_in=hres, residual_out=hd)]
        (chain.ParoChain if kind == "decode" else chain.ParoPrefillChain)(steps, M)()
        torch.cuda.synchronize()
        what = f"{kind} {_cid(shape)} {dt} M={M}"
        assert torch.equal(hres, h), f"{what}: residual_out of step A is not T(bias + residual_in)"
        assert all(bool(torch.isfinite(t).all()) for t in (yb, yc, hd)), f"{what}: the data overflows {dt}"
        rows = sample_rows(M, 8, seed=M).cuda()
        assert_same_values(yb[rows], Sb.apply(exact_rotated(Ls[1], xop[rows]), dt), f"{what}: RMSNORM step")
        act = _cabi.debug_silu_mul(yb[rows])
        assert_same_values(yc[rows], Sc.apply(exact_rotated(Ls[2], act), dt), f"{what}: SILU_MUL step")
        t = Sd.apply(exact_rotated(Ls[3], yc[rows]), dt)
        assert_same_values(hd[rows], (t.float() + hres[rows].float()).to(dt), f"{what}: ADD_RESIDUAL step without y")


# ---------------------------------------------------------------- MoE
def _moe_blocks(E, H, I, group, krot, seed, exps):
    """Selection experts sharing one rotation per projection (gate and up the same); sigma differs per expert."""
    gu = make_synthetic_layer(H, [I, I], group_size=group, krot=krot, seed=seed)
    for n in ("theta", "pairs", "channel_scales"):
        getattr(gu, n)[1] = getattr(gu, n)[0]
    d = make_synthetic_layer(I, [H], group_size=group, krot=krot, seed=seed + 1)
    sels = [(selection_layer(H, [I, I], group=group, seed=seed + 10 + 2 * e, rotation=gu, exps=exps),
             selection_layer(I, [H], group=group, seed=seed + 11 + 2 * e, rotation=d, exps=exps)) for e in range(E)]
    return sels, [{"gate_up": g.L, "down": dn.L} for g, dn in sels]


def _single_routing(T, k, E, seed):
    """Exactly one valid slot per token, weight 1.0; the other slots -1 or >= E with random weights."""
    g = torch.Generator().manual_seed(seed)
    ids = torch.tensor([-1, E, E + 3])[torch.randint(0, 3, (T, k), generator=g)]
    slot = torch.randint(0, k, (T,), generator=g)
    ids[torch.arange(T), slot] = torch.randint(0, E, (T,), generator=g)
    w = torch.rand(T, k, generator=g)
    w[torch.arange(T), slot] = 1.0
    return ids.int(), w.float()


# (T, k, E, dtype, group, krot, H, I)
MOE_CASES = [
    (1, 1, 1, BF, 128, 8, 256, 384),
    (5, 2, 8, FP, 64, 3, 256, 256),
    (16, 2, 64, BF, 128, 8, 512, 384),
    (17, 8, 64, FP, 64, 3, 256, 256),
    (129, 2, 8, BF, 128, 8, 256, 384),
    (1000, 8, 64, BF, 64, 8, 256, 256),
]


def _mid(c):
    T, k, E, dt, g, r, H, I = c
    return f"T{T}-k{k}-E{E}-{'bf16' if dt == BF else 'fp16'}-g{g}-r{r}-H{H}-I{I}"


@pytest.mark.parametrize("case", MOE_CASES, ids=_mid)
def test_moe_steps(case):
    from paroquant_b200.experts import ParoExperts
    from test_gpu_moe_grouped import KINDS, routing
    T, k, E, dt, group, krot, H, I = case
    sels, blocks = _moe_blocks(E, H, I, group, krot, seed=T + E, exps=EXPS[dt])
    ex = ParoExperts(blocks, dt)
    Lgu, Ld = blocks[0]["gate_up"].to("cuda"), blocks[0]["down"].to("cuda")
    x = make_synthetic_activations(T, H, seed=T, device="cuda", dtype=dt) * (0.25 if dt == FP else 1.0)
    toks = sample_rows(T, 8, seed=T)
    xr = exact_rotated(Lgu, x[toks.cuda()])                     # [len(toks), H] per partition (the same rotation)
    steps = [("decode_step", ex.decode_step(T, k))] if T <= 16 else []
    steps.append(("prefill_step", ex.prefill_step(T, k)))
    for kind in (*KINDS, "single"):
        ids, w = _single_routing(T, k, E, seed=T) if kind == "single" else routing(kind, T, k, E, seed=T)
        for name, st in steps:
            st.x.copy_(x)
            st.topk_ids.copy_(ids.cuda())
            st.topk_weights.copy_(w.cuda())
            st.h.fill_(float("nan"))
            st.y.fill_(float("nan"))
            st.step()
            torch.cuda.synchronize()
            what = f"{_mid(case)} {kind} {name}"
            assert bool(torch.isfinite(st.y).all()), f"{what}: the data overflows {dt}"
            idt = ids[toks]
            valid = (idt >= 0) & (idt < E)
            ti, si = valid.nonzero(as_tuple=True)                  # positions among the sampled tokens
            h_got = st.h[toks[ti].cuda(), si.cuda()]
            eids = idt[ti, si].tolist()
            for e in sorted(set(eids)):
                j = torch.tensor([n for n, v in enumerate(eids) if v == e])
                assert_same_values(h_got[j.cuda()], sels[e][0].apply([r[ti[j].cuda()] for r in xr], dt), f"{what}: h of expert {e}")
            yd = exact_rotated(Ld, _cabi.debug_silu_mul(h_got))[0] if len(eids) else None
            ys = torch.zeros(len(eids), H, dtype=torch.float64, device="cuda")
            for e in sorted(set(eids)):
                j = torch.tensor([n for n, v in enumerate(eids) if v == e]).cuda()
                ys[j] = sels[e][1].exact([yd[j]])
            y = st.y[toks.cuda()]
            if kind == "single":                                    # one entry per token, in token order
                assert torch.equal(ti, torch.arange(len(toks)))
                assert_same_values(y, ys.to(dt), f"{what}: y")
            else:
                check_combine(y, ti, w[toks][ti, si], ys, ys.abs(), what=f"{what}: y")


# ---------------------------------------------------------------- dense_weight() == oracle.c_dequant
def _dequant_equal(oracle, L, W, dt, what, chunk=2048):
    """W [K, N] in T on the GPU against oracle.c_dequant of L's checkpoint buffers, column chunk by column chunk."""
    qw, qz, sc = L.qweight.cpu().numpy(), L.qzeros.cpu().numpy(), L.scales.float().cpu().numpy()
    name = "bfloat16" if dt == BF else "float16"
    N = W.shape[1]
    for c0 in range(0, N, chunk):
        c1 = min(N, c0 + chunk)
        ref = oracle.c_dequant(qw[:, c0 // 8:c1 // 8], qz[:, c0 // 8:c1 // 8], sc[:, c0:c1], L.group_size, name)
        got = W[:, c0:c1].float().cpu().numpy()
        if not (got == ref).all():
            bad = (got != ref).nonzero()
            raise AssertionError(f"{what}: {len(bad[0])} elements of columns {c0}..{c1} differ, first (k {bad[0][0]}, n {c0 + bad[1][0]}): "
                                 f"got {got[bad[0][0], bad[1][0]]} ref {ref[bad[0][0], bad[1][0]]}")


DENSE_SHAPES = [(4096, [4096, 1024, 1024], 128), (4096, [14336, 14336], 128), (14336, [4096], 128), (11008, [4096], 128),
                (11008, [512], 128), (14336, [640], 128), (128, [272, 16], 128), (1152, [4096, 1024, 1024], 64)]


@pytest.mark.parametrize("dt", [BF, FP])
@pytest.mark.parametrize("K,parts,group", DENSE_SHAPES)
def test_dense_weight_is_c_dequant(mods, oracle, K, parts, group, dt):
    chain, PK = mods
    L = make_synthetic_layer(K, parts, group_size=group, krot=1, seed=K + len(parts), device="cuda")
    k = PK.from_buffers(L, dt, check_pairs=False)
    _dequant_equal(oracle, L, k.dense_weight(), dt, f"K={K} {parts} g{group}")


@pytest.mark.parametrize("name,H,I,E,dt,group,krot", [("64 experts", 4096, 128, 64, BF, 128, 8),
                                                      ("64 experts, group 64", 4096, 1536, 64, FP, 64, 3),
                                                      ("mixtral_8x7b", 4096, 14336, 8, BF, 128, 8)])
def test_dense_weight_every_stacked_expert(oracle, name, H, I, E, dt, group, krot):
    """Every expert's row of the stacked per-projection buffers (moe_cases.py shapes)."""
    from paroquant_b200.experts import ParoExperts
    from test_gpu_moe import _blocks
    blocks = _blocks(E, H, I, group, krot, device="cuda")
    ex = ParoExperts(blocks, dt)
    for e in range(E):
        for proj, ks in (("gate_up", ex.gate_up), ("down", ex.down)):
            _dequant_equal(oracle, blocks[e][proj], ks[e].dense_weight(), dt, f"{name}: expert {e} {proj}")
    del ex, blocks
    torch.cuda.empty_cache()
