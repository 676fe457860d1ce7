"""GPU parity of prefill chains (paro_prefill_chain_forward, ParoPrefillChain): the chain descriptors for any M as a rotation
pre-pass + INT4 wgmma GEMM per step, the x op in the pre-pass and the epilogue in the GEMM.

  * every stage of the decoder tail vs the oracle applied to the GPU's own previous stage (teacher forcing), normwise 1e-3,
    over ragged last tiles and every tile size the GEMM picks; the Llama-3-8B tail vs the unfused GPU path;
  * a step computes what the single linear computes BIT FOR BIT (same pre-pass, same GEMM): plain chains, SiLU * up against
    paro_debug_silu_mul, the residual epilogue against a torch add of the linear's output;
  * a row's results do not depend on the other rows of the batch; repeated launches and graph replays give identical bits.
"""
import ctypes

import pytest
import torch

from paroquant_b200 import _cabi
from paroquant_b200.checkpoint import make_synthetic_activations, make_synthetic_layer
from test_gpu_chain import _np, _tail, _torch_rms, _torch_silu_mul

pytestmark = pytest.mark.gpu
TOL = 1e-3


@pytest.fixture(scope="module")
def mods():
    from paroquant_b200 import chain
    from paroquant_b200.linear import ParoLinearKernel
    return chain, ParoLinearKernel


def _nt(k, M):
    out = (ctypes.c_int32 * 2)()
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    assert _cabi.lib().paro_debug_gemm_plan(ctypes.byref(k.shape), M, sms, out) == 0
    return out[0]


def _err(a, b):
    return float((a.double() - b.double()).norm() / b.double().norm())


def test_tile_sizes_covered(mods):
    """The sizes of test_decoder_tail_vs_oracle_stagewise reach every tile size of the GEMM, ragged last tiles included."""
    chain, PK = mods
    ks = [PK.from_buffers(make_synthetic_layer(K, p, seed=1).to("cuda"), torch.bfloat16, check_pairs=False)
          for K, p in ((512, [512]), (512, [1024, 1024]), (1024, [512]), (512, [512, 128, 128]))]
    nts = {(_nt(k, M), M % _nt(k, M) != 0) for k in ks for M in (17, 40, 100, 256, 1000)}
    assert {nt for nt, _ in nts} == {32, 64, 128}, nts
    assert any(ragged for _, ragged in nts)


@pytest.mark.parametrize("dt", ["bfloat16", "float16"])
@pytest.mark.parametrize("M", [17, 40, 100, 256, 1000])
def test_decoder_tail_vs_oracle_stagewise(mods, oracle, dt, M):
    chain, _ = mods
    Ls, ks, ch, bufs, attn, resid, w1, w2 = _tail(mods, 512, 1024, [512, 128, 128], M, dt)
    assert isinstance(ch, chain.ParoPrefillChain)
    ch()
    assert _cabi.last_launch_count() == 8
    torch.cuda.synchronize()
    O = oracle
    d = {n: L.numpy_dict() for n, L in Ls.items()}
    h1 = O.add_residual(O.linear(_np(attn), d["o"], dt), _np(resid), dt)
    assert O.rel_err(_np(bufs["residual_mid"]), h1) < TOL
    act = O.linear(O.rms_norm(_np(bufs["residual_mid"]), _np(w1), 1e-5, dt), d["gate_up"], dt)
    assert O.rel_err(_np(bufs["mlp_act"]), act) < TOL
    h2 = O.add_residual(O.linear(O.silu_and_mul(_np(bufs["mlp_act"]), dt), d["down"], dt), _np(bufs["residual_mid"]), dt)
    assert O.rel_err(_np(bufs["residual_out"]), h2) < TOL
    qkv = O.linear(O.rms_norm(_np(bufs["residual_out"]), _np(w2), 1e-5, dt), d["qkv"], dt)
    assert O.rel_err(_np(bufs["qkv"]), qkv) < TOL


@pytest.mark.parametrize("M", [64, 1024])
def test_decoder_tail_llama_shapes_vs_unfused_gpu(mods, M):
    """Llama-3-8B shapes: each stage vs the single-linear kernel + plain torch element-wise ops on the same inputs."""
    Ls, ks, ch, bufs, attn, resid, w1, w2 = _tail(mods, 4096, 14336, [4096, 1024, 1024], M, "bfloat16", seed=21)
    ch()
    torch.cuda.synchronize()
    h1 = (ks["o"](attn).float() + resid.float()).to(attn.dtype)
    assert _err(bufs["residual_mid"], h1) < TOL
    act = ks["gate_up"](_torch_rms(bufs["residual_mid"], w1, 1e-5))
    assert _err(bufs["mlp_act"], act) < TOL
    h2 = (ks["down"](_torch_silu_mul(bufs["mlp_act"])).float() + bufs["residual_mid"].float()).to(attn.dtype)
    assert _err(bufs["residual_out"], h2) < TOL
    qkv = ks["qkv"](_torch_rms(bufs["residual_out"], w2, 1e-5))
    assert _err(bufs["qkv"], qkv) < TOL


@pytest.mark.parametrize("M", [17, 300])
def test_plain_chain_equals_single_linears_bitwise(mods, M):
    """NONE / STORE steps: a merged projection with a partial block, a bias, a group-64 step among group-128 ones and krot 3,
    fed forward (one output kept only in the workspace) == the same linears through paro_linear_forward, bit for bit."""
    chain, PK = mods
    T = torch.bfloat16
    Ls = [make_synthetic_layer(1024, [256, 128], seed=60, bias=True), make_synthetic_layer(384, [1024], group_size=64, seed=61),
          make_synthetic_layer(1024, [640], krot=3, seed=62), make_synthetic_layer(640, [48, 16, 32], seed=63)]
    ks = [PK.from_buffers(L.to("cuda"), T, check_pairs=False) for L in Ls]
    bias = Ls[0].bias.to("cuda", T)
    x0 = make_synthetic_activations(M, 1024, seed=3, dtype=T).cuda()
    ys = [torch.empty(M, k.shape.out_features, dtype=T, device="cuda") for k in ks]
    steps = [chain.ChainStep(ks[0], x=x0, y=ys[0], bias=bias), chain.ChainStep(ks[1], y=ys[1]), chain.ChainStep(ks[2]),
             chain.ChainStep(ks[3], y=ys[3])]
    chain.ParoPrefillChain(steps, M)()
    ref = ks[0](x0, bias)
    assert torch.equal(ys[0], ref)
    ref = ks[1](ref)
    assert torch.equal(ys[1], ref)
    ref = ks[3](ks[2](ref))   # step 2's output lives in the chain's workspace
    assert torch.equal(ys[3], ref)


@pytest.mark.parametrize("dt", [torch.bfloat16, torch.float16])
@pytest.mark.parametrize("M", [40, 257])
def test_silu_mul_and_residual_steps_bitwise(mods, dt, M):
    chain, PK = mods
    L = make_synthetic_layer(512, [384], seed=70, bias=True)
    k = PK.from_buffers(L.to("cuda"), dt, check_pairs=False)
    bias = L.bias.to("cuda", dt)
    gu = make_synthetic_activations(M, 1024, seed=71, dtype=dt).cuda()
    y = torch.empty(M, 384, dtype=dt, device="cuda")
    chain.ParoPrefillChain([chain.ChainStep(k, x=gu, y=y, x_op="silu_mul")], M)()
    assert torch.equal(y, k(_cabi.debug_silu_mul(gu)))
    x = make_synthetic_activations(M, 512, seed=72, dtype=dt).cuda()
    r = make_synthetic_activations(M, 384, seed=73, dtype=dt).cuda()
    y, h = torch.empty_like(r), torch.empty_like(r)
    chain.ParoPrefillChain([chain.ChainStep(k, x=x, y=y, bias=bias, epilogue="add_residual", residual_in=r, residual_out=h)], M)()
    lin = k(x, bias)
    assert torch.equal(y, lin)
    assert torch.equal(h, (lin.float() + r.float()).to(dt))
    h2 = torch.empty_like(r)   # without y
    chain.ParoPrefillChain([chain.ChainStep(k, x=x, bias=bias, epilogue="add_residual", residual_in=r, residual_out=h2)], M)()
    assert torch.equal(h2, h)


def test_rows_do_not_depend_on_the_batch(mods):
    """Every output row of the tail at M = 300 equals the same row of a run on its first 40 rows, bit for bit (both M give
    every step the same tile size)."""
    chain, _ = mods
    Ls, ks, ch, bufs, attn, resid, w1, w2 = _tail(mods, 512, 1024, [512, 128, 128], 300, "bfloat16", seed=9)
    for k in ks.values():
        assert _nt(k, 300) == _nt(k, 40)
    ch()
    ch40, bufs40 = chain.decoder_tail(ks["o"], ks["gate_up"], ks["down"], ks["qkv"], attn_out=attn[:40].contiguous(),
                                      residual=resid[:40].contiguous(), post_attn_norm=w1, next_input_norm=w2, eps=1e-5)
    ch40()
    torch.cuda.synchronize()
    for name, b in bufs.items():
        assert torch.equal(b[:40], bufs40[name]), name


def test_repeated_launches_and_graph_replay_reproduce_eager(mods):
    chain, _ = mods
    Ls, ks, ch, bufs, attn, resid, w1, w2 = _tail(mods, 1024, 2048, [1024, 256, 256], 100, "bfloat16", seed=33)
    outs = []
    for _ in range(3):
        ch()
        assert _cabi.last_launch_count() == 2 * len(ch.steps)
        torch.cuda.synchronize()
        outs.append({n: b.clone() for n, b in bufs.items()})
    for o in outs[1:]:
        assert all(torch.equal(o[n], outs[0][n]) for n in bufs)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        ch()
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        ch()
    for _ in range(3):
        for b in bufs.values():
            b.zero_()
        g.replay()
        torch.cuda.synchronize()
        assert all(torch.equal(bufs[n], outs[0][n]) for n in bufs)


def test_decoder_tail_dispatch(mods):
    chain, PK = mods
    k = {n: PK.from_buffers(make_synthetic_layer(K, p, seed=5).to("cuda"), torch.bfloat16, check_pairs=False)
         for n, (K, p) in {"o": (256, [256]), "gu": (256, [512, 512]), "d": (512, [256]), "qkv": (256, [256, 128, 128])}.items()}
    w = torch.ones(256, dtype=torch.bfloat16, device="cuda")

    def tail(m, **kw):
        a = torch.zeros(m, 256, dtype=torch.bfloat16, device="cuda")
        return chain.decoder_tail(k["o"], k["gu"], k["d"], k["qkv"], attn_out=a, residual=a.clone(), post_attn_norm=w,
                                  next_input_norm=w, **kw)[0]

    assert isinstance(tail(16), chain.ParoChain)
    assert isinstance(tail(17), chain.ParoPrefillChain)
    with pytest.raises(RuntimeError, match="tensor-parallel"):
        tail(17, tensor_parallel=True)
