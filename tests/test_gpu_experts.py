"""MoE expert block on the fused kernels (paroquant_b200/experts.py) vs the oracle: every expert is rotate -> gate | up ->
SiLU * up -> rotate -> down with the block's shared rotations (reference semantics: mlx/modules.py:159-212, RotateSwitchGLU;
format: convert.py:281-406).  Decode batches run each selected expert as ONE two-step chain, larger ones as two launches."""
import numpy as np
import pytest
import torch

from paroquant_b200.checkpoint import ParoLayerBuffers, make_synthetic_activations, make_synthetic_layer

pytestmark = pytest.mark.gpu
TOL = 2e-3       # two fused linears and an activation deep (each stage within 1e-3 of the oracle on the same inputs)


def _blocks(E, H, I):
    shared_gu = make_synthetic_layer(H, [I, I], seed=70)
    shared_d = make_synthetic_layer(I, [H], seed=71)
    blocks = []
    for e in range(E):
        gu, d = make_synthetic_layer(H, [I, I], seed=80 + e), make_synthetic_layer(I, [H], seed=90 + e)
        gu = ParoLayerBuffers(gu.qweight, gu.qzeros, gu.scales, shared_gu.theta, shared_gu.pairs, shared_gu.channel_scales, [I, I], 128, None)
        gu.theta[1], gu.pairs[1], gu.channel_scales[1] = gu.theta[0], gu.pairs[0], gu.channel_scales[0]     # ONE rotation for gate and up
        d = ParoLayerBuffers(d.qweight, d.qzeros, d.scales, shared_d.theta, shared_d.pairs, shared_d.channel_scales, [H], 128, None)
        blocks.append({"gate_up": gu, "down": d})
    return blocks


@pytest.mark.parametrize("T,k", [(1, 2), (5, 2), (40, 3)])
def test_experts_vs_oracle(oracle, T, k):
    from paroquant_b200.experts import ParoExperts

    E, H, I = 4, 256, 384
    blocks = _blocks(E, H, I)
    ex = ParoExperts(blocks, torch.bfloat16)
    g = torch.Generator().manual_seed(T)
    x = make_synthetic_activations(T, H, seed=3 + T, dtype=torch.bfloat16)
    ids = torch.stack([torch.randperm(E, generator=g)[:k] for _ in range(T)])
    w = torch.softmax(torch.randn(T, k, generator=g), -1)
    y = ex(x.cuda(), ids.cuda(), w.cuda()).float().cpu().numpy()
    ref = np.zeros((T, H), np.float64)
    for e in range(E):
        rows, slot = (ids == e).nonzero(as_tuple=True)
        if not len(rows):
            continue
        xe = x[rows].float().numpy()
        act = oracle.silu_and_mul(oracle.linear(xe, blocks[e]["gate_up"].numpy_dict(), "bfloat16"), "bfloat16")
        ye = oracle.linear(act, blocks[e]["down"].numpy_dict(), "bfloat16")
        ref[rows.numpy()] += ye.astype(np.float64) * w[rows, slot].numpy()[:, None].astype(np.float64)
    assert oracle.rel_err(y, oracle.round_to(ref.astype(np.float32), "bfloat16")) < TOL


@pytest.mark.parametrize("T", [5, 40])
def test_experts_drop_ids_outside_range(oracle, T):
    """Slots whose id lies outside [0, E) contribute nothing on the eager path too (T <= 16: one chain per expert; T = 40: the
    GEMM path), as in decode_step and include/paro_b200.h; a token with no valid id gives an exact 0 row.  At T = 5 the eager
    path and decode_step are each checked element-wise against fp64 from their own gate|up output (`check` on h, `check_moe` on
    y): both meet the same derived bounds of the same block.  The eager path's h is taken from a copy of its per-expert chain
    that also stores the gate_up step's output, after checking that the copy reproduces the chain's result bit for bit."""
    from gpu_reference import check, check_moe, rotated
    from paroquant_b200.chain import ChainStep, ParoChain
    from paroquant_b200.experts import ParoExperts

    E, H, I, k = 4, 256, 384, 3
    blocks = _blocks(E, H, I)
    ex = ParoExperts(blocks, torch.bfloat16)
    g = torch.Generator().manual_seed(50 + T)
    x = make_synthetic_activations(T, H, seed=60 + T, dtype=torch.bfloat16)
    ids = torch.stack([torch.randperm(E, generator=g)[:k] for _ in range(T)])
    ids[0, 0], ids[1, 2], ids[T - 1, 1] = -1, E, -1
    ids[2] = torch.tensor([-1, E, E + 3])                                                 # no valid id
    w = torch.softmax(torch.randn(T, k, generator=g), -1)
    y = ex(x.cuda(), ids.cuda(), w.cuda())
    assert not bool(y[2].any()), "a token with no valid id must give 0"
    ref = np.zeros((T, H), np.float64)
    for e in range(E):
        rows, slot = (ids == e).nonzero(as_tuple=True)
        if not len(rows):
            continue
        xe = x[rows].float().numpy()
        act = oracle.silu_and_mul(oracle.linear(xe, blocks[e]["gate_up"].numpy_dict(), "bfloat16"), "bfloat16")
        ye = oracle.linear(act, blocks[e]["down"].numpy_dict(), "bfloat16")
        np.add.at(ref, rows.numpy(), ye.astype(np.float64) * w[rows, slot].numpy()[:, None].astype(np.float64))
    assert oracle.rel_err(y.float().cpu().numpy(), oracle.round_to(ref.astype(np.float32), "bfloat16")) < TOL
    if T <= 16:
        xc, idc, wc = x.cuda(), ids.cuda(), w.cuda()
        Lgu = blocks[0]["gate_up"].to("cuda")
        xr = rotated(Lgu, xc)
        h_eager = torch.full((T, k, 2 * I), float("nan"), dtype=torch.bfloat16, device="cuda")
        for e in range(E):
            rows, slot = (idc == e).nonzero(as_tuple=True)
            if not len(rows):
                continue
            m = len(rows)
            xin = xc[rows].contiguous()
            hbuf = torch.empty(m, 2 * I, dtype=torch.bfloat16, device="cuda")
            ybuf = torch.empty(m, H, dtype=torch.bfloat16, device="cuda")
            ParoChain([ChainStep(ex.gate_up[e], x=xin, y=hbuf), ChainStep(ex.down[e], x_op="silu_mul", y=ybuf)], m)()
            assert torch.equal(ybuf, ex.expert_forward(e, xin)), f"expert {e}: the chain copy differs from the eager path"
            h_eager[rows, slot] = hbuf
        st = ex.decode_step(T, k)
        st.x.copy_(xc)
        st.topk_ids.copy_(idc.int())
        st.topk_weights.copy_(wc)
        st.step()
        for what, h in (("eager path", h_eager), ("decode_step", st.h)):
            for e in range(E):
                rows, slot = (idc == e).nonzero(as_tuple=True)
                if len(rows):
                    check(h[rows, slot], [r[rows] for r in xr], ex.gate_up[e].dense_weight(), Lgu.part_sizes, what=f"{what}: h of expert {e}")
        check_moe(y, h_eager, ids, w, ex, blocks[0]["down"], what="eager path")
        check_moe(st.y, st.h, ids, w, ex, blocks[0]["down"], what="decode_step")
