"""Every step of both chain kernels element-wise against fp64 (tests/gpu_reference.py), the x ops and epilogues included, each
stage teacher-forced on the GPU's own previous output:

  * exact statistics: a step with x = 0 and ADD_RESIDUAL (its bias the only output) hands an RMSNORM step residual rows whose
    normalised operand is known exactly (`exact_rms_rows`): the norm step must meet `check` at full strength on that operand
    and equal the same linear launched on it bit for bit.  Hidden sizes up to 8192 (above 4096 the decode chain's rstd makes
    a second pass over its statistics words); every M of the decode chain, every GEMM tile size of the prefill chain with
    ragged last tiles; rows whose energy sits in one 128-column block, which block moving from row to row until every block
    has been hit, so one statistics word dropped, duplicated or taken from another row moves the operand;
  * random data through the decoder tail (Llama-3-8B and 8192-hidden shapes) and a 6-step chain with three RMSNORM steps and
    a residual step without y: SiLU * up steps with `check_linear` on the library's SiLU * up, residual steps with `check` on y
    and a bitwise residual add, or `check_residual` without y, RMSNORM steps with `check_rmsnorm` (`check` for some rstd
    within a few fp32 ulps of the fp64 one).
"""
import ctypes

import pytest
import torch

from gpu_reference import (check_linear, check_residual_linear, check_rmsnorm_linear, exact_bias, exact_rms_rows)
from paroquant_b200 import _cabi
from paroquant_b200.checkpoint import make_synthetic_activations, make_synthetic_layer

pytestmark = pytest.mark.gpu
HIDDENS = [512, 2048, 4096, 5120, 8192]
DECODE_M = list(range(1, 17))
PREFILL_M = [17, 40, 100, 257, 1000]
A_K, NORM_PARTS, EPS = 256, [256, 128], 1e-8


def _report(area, ratio):
    print(f"[max err/tol] {area}: {ratio:.3f}")


@pytest.fixture(scope="module")
def mods():
    import paroquant_b200.kernels.cuda  # noqa: F401  registers torch.ops.rotation.rotate
    from paroquant_b200 import chain
    from paroquant_b200.linear import ParoLinearKernel
    return chain, ParoLinearKernel


def _plan_nt(shape, M):
    out = (ctypes.c_int32 * 2)()
    assert _cabi.lib().paro_debug_gemm_plan(ctypes.byref(shape), M, torch.cuda.get_device_properties(0).multi_processor_count, out) == 0
    return out[0]


def _hot_blocks(n_rows, nb):
    """Row g of the test (over all its launches): uniform every third row, else hot in the next block in turn."""
    hot, k = [], 0
    for g in range(n_rows):
        if g % 3 == 2:
            hot.append(-1)
        else:
            hot.append(k % nb)
            k += 1
    return hot


# ---------------------------------------------------------------- exact statistics
def test_exact_statistics_prefill_tiles():
    """The prefill cases reach every GEMM tile size with a ragged last tile in the step whose epilogue writes the statistics
    (K = A_K), and the two smaller ones in the RMSNORM step."""
    for dt in (torch.bfloat16, torch.float16):
        a = {(_plan_nt(_cabi.make_shape(A_K, [h], 128, 8, dt), M), M) for h in HIDDENS for M in PREFILL_M}
        b = {(_plan_nt(_cabi.make_shape(h, NORM_PARTS, 64, 3, dt), M), M) for h in HIDDENS for M in PREFILL_M}
        assert {nt for nt, M in a if M % nt} == {32, 64, 128}, a
        assert {nt for nt, M in b if M % nt} >= {32, 64}, b


@pytest.mark.parametrize("dt", [torch.bfloat16, torch.float16])
@pytest.mark.parametrize("hidden", HIDDENS)
@pytest.mark.parametrize("kind", ["decode", "prefill"])
def test_rmsnorm_step_on_exact_statistics(mods, kind, hidden, dt):
    """A (x = 0, bias, ADD_RESIDUAL) -> B (RMSNORM, group 64, krot 3): B == `check` on the exact operand, and == the same
    linear on that operand bit for bit (decode: a one-step chain; prefill: the single linear, the same pre-pass and GEMM)."""
    chain, PK = mods
    seed = hidden + (1 if dt == torch.float16 else 0)
    La = make_synthetic_layer(A_K, [hidden], seed=seed)
    Lb = make_synthetic_layer(hidden, NORM_PARTS, group_size=64, krot=3, seed=seed + 1).to("cuda")
    ka, kb = PK.from_buffers(La.to("cuda"), dt, check_pairs=False), PK.from_buffers(Lb, dt, check_pairs=False)
    Wb = kb.dense_weight()
    w = (1.0 + 0.1 * torch.randn(hidden, generator=torch.Generator().manual_seed(seed))).to(dt)
    bias = exact_bias(hidden, seed, dt)
    Ms = DECODE_M if kind == "decode" else PREFILL_M
    nb = hidden // 128
    hot = _hot_blocks(sum(Ms), nb)
    assert set(hot) >= set(range(nb))
    worst, row0 = 0.0, 0
    for M in Ms:
        h, xop = exact_rms_rows(M, hidden, dt, seed=seed * 100 + M, w=w, eps=EPS, hot=hot[row0:row0 + M])
        row0 += M
        h, xop, wd, bd = h.cuda(), xop.cuda(), w.cuda(), bias.cuda()
        r = (h.double() - bd.double()).to(dt)
        assert torch.equal(r.double(), h.double() - bd.double())
        ya, hres = torch.full_like(h, float("nan")), torch.full_like(h, float("nan"))
        yb = torch.full((M, sum(NORM_PARTS)), float("nan"), dtype=dt, device="cuda")
        steps = [chain.ChainStep(ka, x=torch.zeros(M, A_K, dtype=dt, device="cuda"), y=ya, bias=bd, epilogue="add_residual",
                                 residual_in=r, residual_out=hres),
                 chain.ChainStep(kb, x_op="rmsnorm", norm_weight=wd, eps=EPS, y=yb)]
        if kind == "decode":
            chain.ParoChain(steps, M)()
            one = torch.empty_like(yb)
            chain.ParoChain([chain.ChainStep(kb, x=xop, y=one)], M)()
        else:
            chain.ParoPrefillChain(steps, M)()
            one = kb(xop)
        torch.cuda.synchronize()
        assert torch.equal(ya, bd.expand(M, -1)), f"M={M}: y of the x = 0 step is not its bias"
        assert torch.equal(hres, h), f"M={M}: residual_out is not T(bias + residual_in)"
        worst = max(worst, check_linear(kb, Lb, xop, yb, W=Wb, what=f"{kind} hidden={hidden} {dt} M={M} RMSNORM step"))
        assert torch.equal(yb, one), f"M={M}: the RMSNORM step differs from the same linear on its exact operand"
    _report(f"{kind} exact-statistics RMSNORM step, hidden {hidden}, {dt}", worst)


# ---------------------------------------------------------------- random data
def _layer(K, parts, seed, **kw):
    return make_synthetic_layer(K, parts, seed=seed, device="cuda", **kw)


@pytest.mark.parametrize("hidden,inter,qkv,Ms", [
    (4096, 14336, [4096, 1024, 1024], (1, 16, 64, 1024)),        # Llama-3-8B
    (8192, 28672, [8192, 1024, 1024], (1, 16, 64, 1024)),        # Llama-2/3-70B
])
def test_decoder_tail_every_stage(mods, hidden, inter, qkv, Ms):
    chain, PK = mods
    T, eps = torch.bfloat16, 1e-5
    Ls = {"o": _layer(hidden, [hidden], 41), "gate_up": _layer(hidden, [inter, inter], 42), "down": _layer(inter, [hidden], 43),
          "qkv": _layer(hidden, qkv, 44)}
    ks = {n: PK.from_buffers(L, T, check_pairs=False) for n, L in Ls.items()}
    g = torch.Generator().manual_seed(45)
    w1 = (1.0 + 0.1 * torch.randn(hidden, generator=g)).to(T).cuda()
    w2 = (1.0 + 0.1 * torch.randn(hidden, generator=g)).to(T).cuda()
    worst = {}
    for M in Ms:
        attn = make_synthetic_activations(M, hidden, seed=46 + M, dtype=T).cuda()
        resid = make_synthetic_activations(M, hidden, seed=47 + M, dtype=T).cuda()
        ch, b = chain.decoder_tail(ks["o"], ks["gate_up"], ks["down"], ks["qkv"], attn_out=attn, residual=resid,
                                   post_attn_norm=w1, next_input_norm=w2, eps=eps)
        assert isinstance(ch, chain.ParoChain if M <= 16 else chain.ParoPrefillChain)
        ch()
        torch.cuda.synchronize()
        kind = "decode" if M <= 16 else "prefill"
        what = f"hidden {hidden} M={M}"
        res = {
            "o + residual": check_residual_linear(ks["o"], Ls["o"], attn, b["residual_mid"], resid, what=f"{what} o + residual"),
            "RMSNorm -> gate_up": check_rmsnorm_linear(ks["gate_up"], Ls["gate_up"], b["residual_mid"], w1, eps, b["mlp_act"],
                                                       what=f"{what} gate_up"),
            "SiLU*up -> down + residual": check_residual_linear(ks["down"], Ls["down"], _cabi.debug_silu_mul(b["mlp_act"]),
                                                                b["residual_out"], b["residual_mid"], what=f"{what} down + residual"),
            "RMSNorm -> qkv": check_rmsnorm_linear(ks["qkv"], Ls["qkv"], b["residual_out"], w2, eps, b["qkv"], what=f"{what} qkv"),
        }
        for area, v in res.items():
            worst[(kind, area)] = max(worst.get((kind, area), 0.0), v)
        del ch, b
    for (kind, area), v in worst.items():
        _report(f"{kind} tail hidden {hidden}: {area}", v)


@pytest.mark.parametrize("M", [1, 7, 16, 33, 300])
def test_six_step_chain_every_stage(mods, M):
    """o (+bias, y kept) + residual -> RMSNorm -> gate_up -> SiLU*up -> down (y kept) + residual -> RMSNorm -> a square
    projection -> its output through a linear + residual without y -> RMSNorm -> qkv; hidden 5120 (Qwen2.5-32B,
    Mistral-Nemo)."""
    chain, PK = mods
    T, eps, H, I = torch.bfloat16, 1e-5, 5120, 3072
    Ls = [_layer(H, [H], 51, bias=True), _layer(H, [I, I], 52), _layer(I, [H], 53), _layer(H, [H], 54), _layer(H, [H], 55),
          _layer(H, [1024, 256, 256], 56)]
    ks = [PK.from_buffers(L, T, check_pairs=False) for L in Ls]
    g = torch.Generator().manual_seed(57)
    w1, w2, w3 = ((1.0 + 0.1 * torch.randn(H, generator=g)).to(T).cuda() for _ in range(3))
    bias = Ls[0].bias.to("cuda", T)
    x0 = make_synthetic_activations(M, H, seed=58, dtype=T).cuda()
    r0 = make_synthetic_activations(M, H, seed=59, dtype=T).cuda()
    e = lambda n: torch.full((M, n), float("nan"), dtype=T, device="cuda")   # noqa: E731
    y0, h0, y1, y2, h2, y3, h4, y5 = e(H), e(H), e(2 * I), e(H), e(H), e(H), e(H), e(1536)
    steps = [chain.ChainStep(ks[0], x=x0, y=y0, bias=bias, epilogue="add_residual", residual_in=r0, residual_out=h0),
             chain.ChainStep(ks[1], x_op="rmsnorm", norm_weight=w1, eps=eps, y=y1),
             chain.ChainStep(ks[2], x_op="silu_mul", y=y2, epilogue="add_residual", residual_in=h0, residual_out=h2),
             chain.ChainStep(ks[3], x_op="rmsnorm", norm_weight=w2, eps=eps, y=y3),
             chain.ChainStep(ks[4], epilogue="add_residual", residual_in=h2, residual_out=h4),
             chain.ChainStep(ks[5], x_op="rmsnorm", norm_weight=w3, eps=eps, y=y5)]
    (chain.ParoChain if M <= 16 else chain.ParoPrefillChain)(steps, M)()
    torch.cuda.synchronize()
    kind = "decode" if M <= 16 else "prefill"
    res = {"0 linear (bias)": check_linear(ks[0], Ls[0], x0, y0, bias, what=f"M={M} step 0")}
    assert torch.equal(h0, (y0.float() + r0.float()).to(T)), "step 0: residual_out != T(y + residual_in)"
    res["1 RMSNorm"] = check_rmsnorm_linear(ks[1], Ls[1], h0, w1, eps, y1, what=f"M={M} step 1")
    res["2 SiLU*up"] = check_linear(ks[2], Ls[2], _cabi.debug_silu_mul(y1), y2, what=f"M={M} step 2")
    assert torch.equal(h2, (y2.float() + h0.float()).to(T)), "step 2: residual_out != T(y + residual_in)"
    res["3 RMSNorm"] = check_rmsnorm_linear(ks[3], Ls[3], h2, w2, eps, y3, what=f"M={M} step 3")
    res["4 + residual, no y"] = check_residual_linear(ks[4], Ls[4], y3, h4, h2, what=f"M={M} step 4")
    res["5 RMSNorm"] = check_rmsnorm_linear(ks[5], Ls[5], h4, w3, eps, y5, what=f"M={M} step 5")
    for area, v in res.items():
        _report(f"{kind} 6-step chain M={M}: {area}", v)
