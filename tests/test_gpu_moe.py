"""The MoE expert block in two launches with device-side routing (ParoExperts.decode_step, include/paro_b200.h:
paro_moe_forward) against the oracle composed per expert (oracle.linear / oracle.silu_and_mul, fp64 combine), element-wise
against fp64 (h against the standalone rotate kernel and each expert's dequantised operand, y against the library's own SiLU *
up of that h, rotated, times each expert's dense down operand; tests/gpu_reference.py) over a table of shapes whose launch
plans cover the planner's features (tests/moe_cases.py), over routing edge cases, for bit invariance, under CUDA-graph replay
with changing routings, and with no host work.  Reference semantics: mlx/modules.py:159-212 (RotateSwitchGLU) on the format of
convert.py:281-406."""
import numpy as np
import pytest
import torch

from gpu_reference import check, check_moe, rotated, ulp
from moe_cases import CASES, ROUTINGS, routing
from paroquant_b200.checkpoint import ParoLayerBuffers, make_synthetic_activations, make_synthetic_layer

pytestmark = pytest.mark.gpu
TOL = 2e-3       # two fused linears and an activation deep (the existing experts test's bound)
ROW_TOL = 1.5e-2  # one token's row: a few bf16 roundings (2^-8 each) deep; a missing expert moves a row by tens of percent


def _blocks(E, H, I, group=128, krot=8, device="cpu"):
    shared_gu = make_synthetic_layer(H, [I, I], group_size=group, krot=krot, seed=70, device=device)
    shared_d = make_synthetic_layer(I, [H], group_size=group, krot=krot, seed=71, device=device)
    blocks = []
    for e in range(E):
        gu = make_synthetic_layer(H, [I, I], group_size=group, krot=krot, seed=80 + e, device=device)
        d = make_synthetic_layer(I, [H], group_size=group, krot=krot, seed=90 + e, device=device)
        gu = ParoLayerBuffers(gu.qweight, gu.qzeros, gu.scales, shared_gu.theta.clone(), shared_gu.pairs.clone(), shared_gu.channel_scales.clone(),
                              [I, I], group, None)
        gu.theta[1], gu.pairs[1], gu.channel_scales[1] = gu.theta[0], gu.pairs[0], gu.channel_scales[0]
        d = ParoLayerBuffers(d.qweight, d.qzeros, d.scales, shared_d.theta, shared_d.pairs, shared_d.channel_scales, [H], group, None)
        blocks.append({"gate_up": gu, "down": d})
    return blocks


_cache = {}


def _experts(E, H, I, dtype=torch.bfloat16, group=128, krot=8):
    from paroquant_b200.experts import ParoExperts
    key = (E, H, I, dtype, group, krot)
    if key not in _cache:
        blocks = _blocks(E, H, I, group, krot)
        _cache[key] = (blocks, ParoExperts(blocks, dtype))
    return _cache[key]


def _dname(dtype):
    return "bfloat16" if dtype == torch.bfloat16 else "float16"


def _oracle(oracle, blocks, x, ids, w, dtype):
    """fp64 combine of oracle experts in (expert, slot) order; slots with ids outside [0, E) dropped."""
    E = len(blocks)
    T, H = x.shape
    ref = np.zeros((T, H), np.float64)
    for e in range(E):
        rows, slot = (ids == e).nonzero(as_tuple=True)
        if not len(rows):
            continue
        xe = x[rows].float().numpy()
        act = oracle.silu_and_mul(oracle.linear(xe, blocks[e]["gate_up"].numpy_dict(), _dname(dtype)), _dname(dtype))
        ye = oracle.linear(act, blocks[e]["down"].numpy_dict(), _dname(dtype))
        np.add.at(ref, rows.numpy(), ye.astype(np.float64) * w[rows, slot].numpy()[:, None].astype(np.float64))
    return oracle.round_to(ref.astype(np.float32), _dname(dtype))


def _run(ex, x, ids, w):
    st = ex.decode_step(x.shape[0], ids.shape[1])
    st.x.copy_(x.cuda())
    st.topk_ids.copy_(ids.cuda())
    st.topk_weights.copy_(w.cuda())
    st.step()
    return st


def _routing(T, k, E, seed):
    g = torch.Generator().manual_seed(seed)
    ids = torch.stack([torch.randperm(E, generator=g)[:k] for _ in range(T)]) if k <= E else torch.randint(0, E, (T, k), generator=g)
    w = torch.softmax(torch.randn(T, k, generator=g), -1)
    return ids.int(), w


def _compare(oracle, blocks, x, ids, w, y, dtype, what=""):
    ref = _oracle(oracle, blocks, x, ids.long(), w, dtype)
    got = y.float().cpu().numpy()
    assert oracle.rel_err(got, ref) < TOL, what
    for t in range(x.shape[0]):
        if np.linalg.norm(ref[t]) > 0:
            assert oracle.rel_err(got[t], ref[t]) < ROW_TOL, f"{what}: token {t}"
        else:
            assert not np.any(got[t]), f"{what}: token {t} has no expert and must be 0"


@pytest.mark.parametrize("E", [4, 16])
@pytest.mark.parametrize("k", [1, 2, 8])
@pytest.mark.parametrize("T", [1, 3, 8, 16])
def test_moe_vs_oracle(oracle, T, k, E):
    if k > E:
        pytest.skip("top-k above the expert count")
    blocks, ex = _experts(E, 256, 384)
    x = make_synthetic_activations(T, 256, seed=3 + T, dtype=torch.bfloat16)
    ids, w = _routing(T, k, E, seed=100 * T + k)
    st = _run(ex, x, ids, w)
    _compare(oracle, blocks, x, ids, w, st.y, torch.bfloat16, f"T={T} k={k} E={E}")


@pytest.mark.parametrize("dtype,group,krot", [(torch.float16, 128, 8), (torch.bfloat16, 64, 8), (torch.float16, 64, 3), (torch.bfloat16, 128, 3)])
@pytest.mark.parametrize("T", [1, 5, 16])
def test_moe_variants_vs_oracle(oracle, dtype, group, krot, T):
    blocks, ex = _experts(8, 256, 384, dtype, group, krot)
    x = make_synthetic_activations(T, 256, seed=7 + T, dtype=dtype)
    ids, w = _routing(T, 2, 8, seed=T)
    st = _run(ex, x, ids, w)
    _compare(oracle, blocks, x, ids, w, st.y, dtype, f"{dtype} g{group} krot{krot} T={T}")


@pytest.mark.parametrize("T", [1, 16])
def test_moe_qwen3_shaped_block(oracle, T):
    blocks, ex = _experts(16, 2048, 768)
    x = make_synthetic_activations(T, 2048, seed=11 + T, dtype=torch.bfloat16)
    ids, w = _routing(T, 8, 16, seed=5 + T)
    st = _run(ex, x, ids, w)
    _compare(oracle, blocks, x, ids, w, st.y, torch.bfloat16, f"qwen3 T={T}")


@pytest.mark.parametrize("T,k", [(1, 2), (6, 8), (16, 4)])
def test_moe_stagewise(T, k):
    """Every valid h[t, s] element-wise against the rotate kernel and the expert's dense operand; y element-wise against the
    library's SiLU * up of the GPU's own h, rotated, times each expert's dense down operand in fp64, combined in fp64."""
    E, H, I = 8, 256, 384
    blocks, ex = _experts(E, H, I)
    x = make_synthetic_activations(T, H, seed=21 + T, dtype=torch.bfloat16)
    ids, w = _routing(T, k, E, seed=T * k)
    st = _run(ex, x, ids, w)
    xc = x.cuda()
    for e in range(E):
        rows, slot = (ids.long() == e).nonzero(as_tuple=True)
        if not len(rows):
            continue
        L = blocks[e]["gate_up"].to("cuda")
        xr = [r[rows.cuda()] for r in rotated(L, xc)]
        check(st.h[rows.cuda(), slot.cuda()], xr, ex.gate_up[e].dense_weight(), L.part_sizes, what=f"h of expert {e}")
    check_moe(st.y, st.h, ids, w, ex, blocks[0]["down"], what="y")


def _edge_routings(T, k, E):
    g = torch.Generator().manual_seed(9)
    w = torch.softmax(torch.randn(T, k, generator=g), -1)
    one = torch.full((T, k), 3, dtype=torch.int32)                                       # all tokens on one expert (with duplicates)
    distinct = torch.arange(T * k, dtype=torch.int32).reshape(T, k) % E                  # all slots on distinct experts when T*k <= E
    dup = torch.randint(0, E, (T, k), generator=g).int()
    dup[:, 1] = dup[:, 0]                                                                # duplicate ids in every token
    invalid = torch.randint(0, E, (T, k), generator=g).int()
    invalid[0, 0], invalid[-1, -1] = -1, E                                               # dropped slots
    invalid[T // 2, :] = -1                                                              # a token with no local expert
    zero_w = w.clone()
    zero_w[:, 0] = 0.0
    return {"one_expert": (one, w), "distinct": (distinct, w), "duplicates": (dup, w), "invalid_ids": (invalid, w),
            "zero_weight": (torch.randint(0, E, (T, k), generator=g).int(), zero_w)}


@pytest.mark.parametrize("case", ["one_expert", "distinct", "duplicates", "invalid_ids", "zero_weight"])
@pytest.mark.parametrize("T,k,E", [(16, 2, 32), (16, 8, 128)])
def test_moe_routing_edge_cases(oracle, case, T, k, E):
    blocks, ex = _experts(E, 256, 384) if E <= 32 else _experts(E, 256, 128)
    ids, w = _edge_routings(T, k, E)[case]
    x = make_synthetic_activations(T, 256, seed=31, dtype=torch.bfloat16)
    st = _run(ex, x, ids, w)
    _compare(oracle, blocks, x, ids, w, st.y, torch.bfloat16, case)


def test_moe_bit_invariance_and_graph_replay():
    from paroquant_b200.chain import ChainStep, ParoChain
    E, H, I, T, k = 16, 256, 384, 5, 4
    blocks, ex = _experts(E, H, I)
    x = make_synthetic_activations(T, H, seed=41, dtype=torch.bfloat16).cuda()
    ids, w = _routing(T, k, E, seed=77)
    st = _run(ex, x, ids, w)
    y0 = st.y.clone()
    st.step()
    assert torch.equal(st.y, y0), "two launches differ"
    perm = torch.stack([torch.randperm(k) for _ in range(T)])
    st.topk_ids.copy_(torch.gather(ids, 1, perm).cuda())
    st.topk_weights.copy_(torch.gather(w, 1, perm).cuda())
    st.step()
    assert torch.equal(st.y, y0), "permuting a token's slots changed the output"

    # a preceding chain (x of the block = a ParoChain's output, PDL edge) and three routings replayed through one graph
    pre = ex.gate_up[0]
    from paroquant_b200.linear import ParoLinearKernel
    dn = ParoLinearKernel.from_buffers(make_synthetic_layer(I, [H], seed=5).to("cuda"), torch.bfloat16)
    xin = make_synthetic_activations(T, H, seed=42, dtype=torch.bfloat16).cuda()
    chain = ParoChain([ChainStep(pre, x=xin), ChainStep(dn, x_op="silu_mul", y=st.x)], T)
    routings = [_routing(T, k, E, seed=s) for s in (1, 2, 3)]
    eager = []
    for r_ids, r_w in routings:
        chain()
        st.topk_ids.copy_(r_ids.cuda())
        st.topk_weights.copy_(r_w.cuda())
        st.step()
        eager.append((st.y.clone(), st.h.clone()))
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        chain()
        st.step()
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        chain()
        st.step()
    for (r_ids, r_w), (ye, he) in zip(routings, eager):
        st.topk_ids.copy_(r_ids.cuda())
        st.topk_weights.copy_(r_w.cuda())
        st.y.zero_()
        g.replay()
        torch.cuda.synchronize()
        assert torch.equal(st.y, ye), "graph replay differs from the eager launch"
        valid = (r_ids >= 0) & (r_ids < E)
        assert torch.equal(st.h[valid.cuda()], he[valid.cuda()])


def test_moe_no_host_work():
    from paroquant_b200 import _cabi
    E, T, k = 8, 4, 2
    blocks, ex = _experts(E, 256, 384)
    ids, w = _routing(T, k, E, seed=3)
    st = _run(ex, make_synthetic_activations(T, 256, seed=1, dtype=torch.bfloat16), ids, w)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        st.step()
        assert _cabi.last_launch_count() == 2
    finally:
        torch.cuda.set_sync_debug_mode("default")
    torch.cuda.synchronize()


def test_moe_from_disk_checkpoint(oracle, tmp_path):
    from paroquant_b200 import checkpoint_io as cio
    from paroquant_b200.experts import ParoExperts
    E, H, I, T, k = 4, 256, 256, 3, 2
    shared_gu, shared_d = make_synthetic_layer(H, [I, I], seed=70), make_synthetic_layer(I, [H], seed=71)
    tensors = {}
    for e in range(E):
        gu, d = make_synthetic_layer(H, [I, I], seed=80 + e), make_synthetic_layer(I, [H], seed=90 + e)
        for proj, sl in (("gate_proj", slice(0, I // 8)), ("up_proj", slice(I // 8, 2 * I // 8))):
            tensors[f"model.layers.0.mlp.experts.{e}.{proj}.qweight"] = gu.qweight[:, sl].contiguous()
            tensors[f"model.layers.0.mlp.experts.{e}.{proj}.qzeros"] = gu.qzeros[:, sl].contiguous()
            tensors[f"model.layers.0.mlp.experts.{e}.{proj}.scales"] = gu.scales[:, sl.start * 8:sl.stop * 8].contiguous()
        for leaf in ("qweight", "qzeros", "scales"):
            tensors[f"model.layers.0.mlp.experts.{e}.down_proj.{leaf}"] = getattr(d, leaf)
    for tag, L in (("gate_up", shared_gu), ("down", shared_d)):
        tensors[f"model.layers.0.mlp.experts.{tag}_weight_theta"] = L.theta[0]
        tensors[f"model.layers.0.mlp.experts.{tag}_weight_pairs"] = L.pairs[0]
        tensors[f"model.layers.0.mlp.experts.{tag}_weight_channel_scales"] = L.channel_scales[0]
    cio.save_paro_checkpoint(tmp_path, tensors, base_config={"model_type": "qwen3_moe"})
    blocks = cio.load_paro_checkpoint(tmp_path).experts["model.layers.0.mlp.experts"]
    ex = ParoExperts(blocks, torch.bfloat16)
    x = make_synthetic_activations(T, H, seed=2, dtype=torch.bfloat16)
    ids, w = _routing(T, k, E, seed=4)
    st = _run(ex, x, ids, w)
    _compare(oracle, blocks, x, ids, w, st.y, torch.bfloat16, "from disk")

    bad = [dict(b) for b in blocks]
    d = bad[2]["down"]
    bad[2]["down"] = ParoLayerBuffers(d.qweight, d.qzeros, d.scales, d.theta + 0.5, d.pairs, d.channel_scales, d.part_sizes, d.group_size, None)
    with pytest.raises(RuntimeError, match="rotation differs"):
        ParoExperts(bad, torch.bfloat16)


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
def test_debug_silu_mul_within_one_ulp_of_fp64_silu(dtype):
    """The test hook's SiLU * up (the library's own, with its fast exp): every element is T(s * u) with s within one ulp of
    T(silu(g)) computed in fp64, and the product rounded once to T; nearly all elements take s = T(silu(g)) itself.  (A one-ulp
    step of s can move the product by more than one ulp of the product, so the ulp is counted on s.)"""
    from paroquant_b200 import _cabi
    g = torch.Generator(device="cuda").manual_seed(0)
    gu = (torch.randn(48, 2 * 1024, generator=g, device="cuda") * 4).to(dtype)
    gu[0, :8] = torch.tensor([0.0, -0.0, 1e-3, -1e-3, 30.0, -30.0, 80.0, -80.0], dtype=dtype)
    act = _cabi.debug_silu_mul(gu)
    assert _cabi.last_launch_count() == 1
    gd, ud = gu[:, :1024].double(), gu[:, 1024:].double()
    s0 = (gd / (1.0 + torch.exp(-gd))).to(dtype).double()
    du = ulp(s0, dtype)
    hits = [act.double() == (c.to(dtype).double() * ud).to(dtype).double() for c in (s0, s0 - du, s0 - du / 2, s0 + du)]
    ok = hits[0] | hits[1] | hits[2] | hits[3]
    assert bool(ok.all()), f"{int((~ok).sum())} elements are not T(s * u) with s within one ulp of T(silu(g))"
    assert float(hits[0].double().mean()) > 0.99
    assert torch.equal(_cabi.debug_silu_mul(gu[5:9]), act[5:9])


_case_cache = {}


def _case_experts(case):
    """Weights generated on the device, one shape kept at a time (a Mixtral-shaped block is about 1.5 GB with its buffers)."""
    from paroquant_b200.experts import ParoExperts
    key = (case.H, case.I, case.E, case.dtype, case.group, case.krot)
    if key not in _case_cache:
        _case_cache.clear()
        torch.cuda.empty_cache()
        blocks = _blocks(case.E, case.H, case.I, case.group, case.krot, device="cuda")
        _case_cache[key] = (blocks, ParoExperts(blocks, case.dtype))
    return _case_cache[key]


def _plan_str(out, U):
    s = []
    for name, base in (("gate_up", 0), ("down", 8)):
        c, S, grid, nb, G, ng, nst, smem = out[base: base + 8]
        s.append(f"{name} c={c} S={S} waves={-(-U * S // c)} groups/item={ng} stages={nst}")
    return ", ".join(s)


@pytest.mark.parametrize("kind", ROUTINGS)
@pytest.mark.parametrize("case", CASES, ids=lambda c: c.name)
def test_moe_plan_space_elementwise(case, kind):
    """Every case of tests/moe_cases.py (together their plans at 132 SMs reach every cluster size, uneven and wave-crossing K
    slices, reused receive buffers, partial last waves and items longer than the ring) under four routings: h of every selected
    expert with `check`, y with `check_moe`, every output element written, and a second launch bit-identical."""
    from paroquant_b200 import _cabi
    blocks, ex = _case_experts(case)
    T, k = case.T, case.k
    x = make_synthetic_activations(T, case.H, seed=17 + T, dtype=case.dtype, device="cuda")
    ids, w = routing(case, kind)
    idc = ids.cuda()
    valid = (idc >= 0) & (idc < case.E)
    st = ex.decode_step(T, k)
    st.x.copy_(x)
    st.topk_ids.copy_(idc)
    st.topk_weights.copy_(w.cuda())
    outs = []
    for _ in range(2):
        st.h.fill_(float("nan"))
        st.y.fill_(float("nan"))   # every element of y and of the valid rows of h must be written
        st.step()
        outs.append((st.y.clone(), st.h[valid].clone()))
    assert torch.equal(outs[0][0], outs[1][0]) and torch.equal(outs[0][1], outs[1][1]), "a second launch differs"

    Lgu = blocks[0]["gate_up"]
    xr = rotated(Lgu, x)
    worst_h = 0.0
    for e in torch.unique(idc[valid]).tolist():
        rows, slot = (idc == e).nonzero(as_tuple=True)
        worst_h = max(worst_h, check(st.h[rows, slot], [r[rows] for r in xr], ex.gate_up[e].dense_weight(), Lgu.part_sizes,
                                     what=f"{case.name} {kind}: h of expert {e}"))
    worst_y = check_moe(st.y, st.h, idc, w, ex, blocks[0]["down"], what=f"{case.name} {kind}: y")
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    out = _cabi.debug_moe_plan(st._desc, T, k, sms)
    U = len(torch.unique(idc[valid]))
    print(f"\n[moe-case] {case.name} {kind}: U={U} of {out[16]}, {sms} SMs: {_plan_str(out, out[16])}; "
          f"max err/tol h {worst_h:.3f} y {worst_y:.3f}")
