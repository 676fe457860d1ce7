"""The MoE expert block for any batch as grouped wgmma GEMMs (ParoExperts.prefill_step, include/paro_b200.h:
paro_moe_grouped_forward).  Element-wise against fp64 (tests/gpu_reference.py: every valid h[t, s] against the standalone rotate
kernel and its expert's dequantised operand, y against the library's SiLU * up of that h, rotated, times each expert's dense down
operand) over batch sizes, top-k, expert counts, dtypes, group sizes, krot and routings; every output written; real Qwen3-30B-A3B-
and Mixtral-8x7B-shaped blocks also against the oracle; agreement with decode_step where both apply; bit reproducibility and
permutation invariance; CUDA-graph replay over changing routings; no host work.  Shapes and routings are defined here."""
import numpy as np
import pytest
import torch

from gpu_reference import check, check_moe, rotated
from paroquant_b200.checkpoint import make_synthetic_activations
from test_gpu_moe import _blocks, _oracle

pytestmark = pytest.mark.gpu
BF, FP = torch.bfloat16, torch.float16
TOL = 2e-3   # normwise against the oracle, as test_gpu_moe.py
LAUNCHES = 6

# (T, k, E, dtype, group, krot, H, I): together T in {1, 16, 17, 40, 129, 1000}, k in {1, 2, 8}, E in {1, 8, 64, 128}, both dtypes,
# group 64 / 128, krot 3 / 8, hidden above and below I
CASES = [
    (1, 1, 1, BF, 128, 8, 256, 384),
    (16, 2, 8, BF, 128, 8, 256, 384),
    (17, 8, 64, FP, 64, 3, 256, 256),
    (40, 2, 8, FP, 128, 8, 512, 384),
    (40, 8, 1, BF, 64, 3, 256, 384),
    (129, 8, 128, BF, 64, 8, 256, 128),
    (1000, 1, 8, BF, 128, 3, 256, 384),
    (1000, 8, 64, FP, 128, 8, 256, 256),
]
KINDS = ("balanced", "skewed", "one_expert", "duplicates", "invalid_ids", "none_valid")


def _cid(c):
    T, k, E, dt, g, r, H, I = c
    return f"T{T}-k{k}-E{E}-{'bf16' if dt == BF else 'fp16'}-g{g}-r{r}-H{H}-I{I}"


def routing(kind, T, k, E, seed=0):
    """(ids [T, k] int32, weights [T, k] fp32).  balanced: ids cycle over all experts; skewed: every token's slot 0 and a third
    of the others on one hot expert; one_expert: every slot on one expert (duplicates within a token when k > 1); duplicates:
    slot 1 repeats slot 0 in every token; invalid_ids: a quarter of the slots -1 or >= E and one token with no valid slot;
    none_valid: every id -1 or E.  The weights differ per slot, so a weight on the wrong slot changes the output."""
    g = torch.Generator().manual_seed(1000 * seed + KINDS.index(kind))
    w = torch.softmax(torch.randn(T, k, generator=g), -1)
    rnd = torch.randint(0, E, (T, k), generator=g)
    if kind == "balanced":
        ids = (torch.arange(T * k).reshape(T, k) + int(torch.randint(0, E, (1,), generator=g))) % E
    elif kind == "skewed":
        hot = int(torch.randint(0, E, (1,), generator=g))
        ids = torch.where(torch.rand(T, k, generator=g) < 0.33, hot, rnd)
        ids[:, 0] = hot
    elif kind == "one_expert":
        ids = torch.full((T, k), int(torch.randint(0, E, (1,), generator=g)))
    elif kind == "duplicates":
        ids = rnd
        if k > 1:
            ids[:, 1] = ids[:, 0]
    elif kind == "invalid_ids":
        bad = torch.tensor([-1, E, E + 7, -100])[torch.randint(0, 4, (T, k), generator=g)]
        ids = torch.where(torch.rand(T, k, generator=g) < 0.25, bad, rnd)
        ids[T // 2, :] = -1
    elif kind == "none_valid":
        ids = torch.where(torch.rand(T, k, generator=g) < 0.5, -1, E)
    else:
        raise ValueError(kind)
    return ids.int(), w.float()


def _distinct_routing(T, k, E, seed):
    g = torch.Generator().manual_seed(seed)
    ids = torch.stack([torch.randperm(E, generator=g)[:k] for _ in range(T)])
    return ids.int(), torch.softmax(torch.randn(T, k, generator=g), -1).float()


_cache = {}


def _experts(E, H, I, dtype=BF, group=128, krot=8, big=False):
    """Weights generated on the device.  A big (real-shaped) block is kept alone; small ones stay cached."""
    from paroquant_b200.experts import ParoExperts
    key = (E, H, I, dtype, group, krot)
    if key not in _cache:
        if big or any(k[1] * k[2] * k[0] > 1 << 26 for k in _cache):
            _cache.clear()
            torch.cuda.empty_cache()
        blocks = _blocks(E, H, I, group, krot, device="cuda")
        _cache[key] = (blocks, ParoExperts(blocks, dtype))
    return _cache[key]


def _launch(st, x, ids, w, nan=True):
    st.x.copy_(x)
    st.topk_ids.copy_(ids.cuda())
    st.topk_weights.copy_(w.cuda())
    if nan:
        st.h.fill_(float("nan"))   # every valid row of h and every element of y must be written
        st.y.fill_(float("nan"))
    st.step()
    return st


def _check_block(blocks, ex, st, x, ids, w, what):
    """`check` on every valid h[t, s] per expert, `check_moe` on y (exact zeros for a token without a valid slot)."""
    idc = ids.cuda()
    valid = (idc >= 0) & (idc < ex.n_experts)
    Lgu = blocks[0]["gate_up"]
    xr = rotated(Lgu, x)
    worst = 0.0
    for e in torch.unique(idc[valid]).tolist():
        rows, slot = (idc == e).nonzero(as_tuple=True)
        worst = max(worst, check(st.h[rows, slot], [r[rows] for r in xr], ex.gate_up[e].dense_weight(), Lgu.part_sizes, what=f"{what}: h of expert {e}"))
    return worst, check_moe(st.y, st.h, idc, w, ex, blocks[0]["down"], what=f"{what}: y")


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("case", CASES, ids=_cid)
def test_grouped_elementwise(case, kind):
    T, k, E, dtype, group, krot, H, I = case
    blocks, ex = _experts(E, H, I, dtype, group, krot)
    x = make_synthetic_activations(T, H, seed=T + k, dtype=dtype, device="cuda")
    ids, w = routing(kind, T, k, E)
    st = _launch(ex.prefill_step(T, k), x, ids, w)
    wh, wy = _check_block(blocks, ex, st, x, ids, w, f"{_cid(case)} {kind}")
    print(f"\n[moe-grouped] {_cid(case)} {kind}: max err/tol h {wh:.3f} y {wy:.3f}")


@pytest.mark.parametrize("T,E", [(32, 8), (33, 8), (96, 8), (64, 1), (65, 1), (128, 1), (512, 1), (513, 1)])
def test_grouped_one_expert_at_tile_edges(T, E):
    """All T * k entries on one expert with T * k = NT, NT + 1 or a multiple of NT, for every tile size: full tiles, a tile
    holding one entry, and several full tiles of one expert."""
    from paroquant_b200 import _cabi
    H, I, k = 256, 384, 1
    blocks, ex = _experts(E, H, I)
    st = ex.prefill_step(T, k)
    nt = _cabi.debug_moe_grouped_plan(st._desc, T, k, 132)[0]
    assert T % nt in (0, 1)
    x = make_synthetic_activations(T, H, seed=T, dtype=BF, device="cuda")
    ids = torch.full((T, k), E - 1, dtype=torch.int32)
    w = torch.rand(T, k) + 0.5
    _launch(st, x, ids, w)
    _check_block(blocks, ex, st, x, ids, w, f"one expert T={T} NT={nt}")


@pytest.mark.parametrize("name,H,I,E,k,T", [("qwen3_30b_a3b", 2048, 768, 128, 8, 512), ("mixtral_8x7b", 4096, 14336, 8, 2, 256)])
def test_grouped_real_shapes(oracle, name, H, I, E, k, T):
    """Element-wise over the whole batch; against the oracle (normwise, as test_gpu_moe.py) on the first 48 tokens, whose rows
    depend on no other token.  Fewer tokens make the normwise error a property of the sample: on the first 12 tokens of the
    Qwen3-shaped block it is 2.03e-3 for decode_step and prefill_step alike (H100), 1.87e-3 over 48."""
    blocks, ex = _experts(E, H, I, big=True)
    x = make_synthetic_activations(T, H, seed=5, dtype=BF, device="cuda")
    ids, w = _distinct_routing(T, k, E, seed=3)
    st = _launch(ex.prefill_step(T, k), x, ids, w)
    wh, wy = _check_block(blocks, ex, st, x, ids, w, name)
    n = 48
    cpu_blocks = [{p: b[p].to("cpu") for p in b} for b in blocks]
    ref = _oracle(oracle, cpu_blocks, x[:n].cpu(), ids[:n].long(), w[:n], BF)
    err = oracle.rel_err(st.y[:n].float().cpu().numpy(), ref)
    assert err < TOL, err
    print(f"\n[moe-grouped] {name} T={T}: max err/tol h {wh:.3f} y {wy:.3f}, oracle rel err {err:.2e}")


@pytest.mark.parametrize("T", [1, 7, 16])
@pytest.mark.parametrize("kind", ["balanced", "duplicates", "invalid_ids"])
def test_grouped_agrees_with_decode_step(T, kind):
    """Where both paths apply, both pass the element-wise checks on the same inputs, and their outputs lie within a few ulps."""
    E, H, I, k = 8, 256, 384, 2
    blocks, ex = _experts(E, H, I)
    x = make_synthetic_activations(T, H, seed=9 + T, dtype=BF, device="cuda")
    ids, w = routing(kind, T, k, E, seed=T)
    outs = []
    for st in (ex.decode_step(T, k), ex.prefill_step(T, k)):
        _launch(st, x, ids, w)
        _check_block(blocks, ex, st, x, ids, w, f"{type(st).__name__} T={T} {kind}")
        outs.append(st.y.float())
    assert torch.allclose(outs[0], outs[1], rtol=2e-2, atol=1e-3)


def test_grouped_deterministic_and_permutation_invariant():
    E, H, I, T, k = 16, 256, 384, 70, 4
    blocks, ex = _experts(E, H, I)
    x = make_synthetic_activations(T, H, seed=41, dtype=BF, device="cuda")
    ids, w = _distinct_routing(T, k, E, seed=77)
    st = _launch(ex.prefill_step(T, k), x, ids, w)
    y0, h0 = st.y.clone(), st.h.clone()
    _launch(st, x, ids, w)
    assert torch.equal(st.y, y0) and torch.equal(st.h, h0), "two launches differ"
    g = torch.Generator().manual_seed(5)
    pt = torch.randperm(T, generator=g)
    ps = torch.stack([torch.randperm(k, generator=g) for _ in range(T)])
    ids2, w2 = torch.gather(ids[pt], 1, ps), torch.gather(w[pt], 1, ps)
    _launch(st, x[pt.cuda()], ids2, w2)
    assert torch.equal(st.y, y0[pt.cuda()]), "permuting tokens and slots changed y beyond the permutation"
    h_perm = h0[pt.cuda()][torch.arange(T, device="cuda")[:, None], ps.cuda()]
    assert torch.equal(st.h, h_perm), "permuting tokens and slots changed h beyond the permutation"


def test_grouped_graph_replay_over_routings():
    E, H, I, T, k = 8, 256, 384, 45, 2
    blocks, ex = _experts(E, H, I)
    st = ex.prefill_step(T, k)
    x = make_synthetic_activations(T, H, seed=42, dtype=BF, device="cuda")
    routings = [routing(kind, T, k, E, seed=2) for kind in ("balanced", "one_expert", "none_valid")]
    eager = []
    for r_ids, r_w in routings:
        _launch(st, x, r_ids, r_w, nan=False)
        eager.append((st.y.clone(), st.h.clone()))
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        st.step()
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        st.step()
    for (r_ids, r_w), (ye, he) in zip(routings, eager):
        st.topk_ids.copy_(r_ids.cuda())
        st.topk_weights.copy_(r_w.cuda())
        st.y.fill_(float("nan"))
        g.replay()
        torch.cuda.synchronize()
        assert torch.equal(st.y, ye), "graph replay differs from the eager launch"
        valid = ((r_ids >= 0) & (r_ids < E)).cuda()
        assert torch.equal(st.h[valid], he[valid])
    assert not np.any(st.y.float().cpu().numpy()), "none_valid: every token must be exactly 0"


def test_grouped_no_host_work():
    from paroquant_b200 import _cabi
    E, H, I, T, k = 8, 256, 384, 300, 2
    blocks, ex = _experts(E, H, I)
    ids, w = routing("balanced", T, k, E)
    st = _launch(ex.prefill_step(T, k), make_synthetic_activations(T, H, seed=1, dtype=BF, device="cuda"), ids, w)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        st.step()
        assert _cabi.last_launch_count() == LAUNCHES
    finally:
        torch.cuda.set_sync_debug_mode("default")
    torch.cuda.synchronize()
