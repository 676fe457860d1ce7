"""The MoE router on the device (ParoRouter, include/paro_b200.h: paro_moe_route): router logits, softmax and top-k in one launch.

Logits element-wise against fp64 with the bound of a fused linear (tests/gpu_reference.py); the selection exactly and the weights
within a stated bound, both from the GPU's own logits (each stage is fed the previous stage's GPU output); ties and extreme
logits; bit-identical routing of a row whatever batch it is routed in; and the router inside decode_step / prefill_step on
Qwen3-30B-A3B- and Mixtral-8x7B-shaped blocks (tests/moe_cases.py): same y and h as the step fed the same routing by hand, 3 / 7
launches, one CUDA graph from hidden state to block output.  Outputs are NaN / -1 filled before every call.

The weight bound.  With d = logit - row max, the kernel forms exp(d) as ex2.approx(d * log2(e)): the fp32 product carries a
relative error of 2^-24 (and log2(e) itself 2^-25) on an exponent of magnitude |d| * 1.44, i.e. up to |d| * 2^-23 relative on the
result with margin, and ex2.approx adds 2^-22.  Only terms with d > -87.4 are non-zero in fp32 (the kernel flushes below), so
|d| counts up to min(row spread, 88).  A weight is exp(d_s) / sum_e exp(d_e), renormalised by a sum of at most 16 of them: one
exp error in the numerator, at most one in the denominator (a weighted mean of the terms' errors), and about 36 fp32 roundings
(13 adds of the denominator, a reciprocal, a product; 16 adds and a fast division of the renormalisation), taken as 48 * 2^-24.
So |w - ref| <= ref * (2 * (2^-22 + min(spread, 88) * 2^-23) + 48 * 2^-24) + 1e-37, ref the fp64 softmax of the same logits; the
absolute term covers a probability below the smallest normal fp32, which the kernel returns as zero."""
import numpy as np
import pytest
import torch

from gpu_reference import check
from moe_cases import CASES as MOE_CASES
from moe_route_reference import np_moe_route
from paroquant_b200 import _cabi
from paroquant_b200.checkpoint import make_synthetic_activations
from paroquant_b200.experts import ParoRouter

pytestmark = pytest.mark.gpu
BF, FP = torch.bfloat16, torch.float16
SHAPES = [(2048, 128, 8), (4096, 8, 2), (4096, 256, 8), (2048, 60, 4), (256, 1, 1), (8192, 64, 6)]   # (H, E, k)
TS = [1, 5, 16, 17, 40, 129, 1000, 4096]


def _dname(dt):
    return "bfloat16" if dt == BF else "float16"


def _weight(E, H, dt, seed=0, spread=2.0):
    """A router weight whose logits on unit-variance activations have a standard deviation of about `spread`."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    return (torch.randn(E, H, generator=g, device="cuda") * (spread / H ** 0.5)).to(dt)


def _route(x, w, k, renorm=True, logits=True):
    """(ids, weights, logits) of one paro_moe_route call into NaN / -1 filled outputs."""
    T, E = x.shape[0], w.shape[0]
    ids = torch.full((T, k), -1, dtype=torch.int32, device="cuda")
    wts = torch.full((T, k), float("nan"), dtype=torch.float32, device="cuda")
    lg = torch.full((T, E), float("nan"), dtype=torch.float32, device="cuda") if logits else None
    _cabi.moe_route(x, w, k, renorm, ids, wts, lg)
    assert _cabi.last_launch_count() == 1
    return ids, wts, lg


def _check_routing(ids, wts, lg, k, renorm, dt, what):
    """ids exactly and weights within the bound of the module docstring, both from the GPU's own logits."""
    l = lg.cpu().numpy()
    assert np.isfinite(l).all(), f"{what}: non-finite logits"
    ref_ids, ref_w, _ = np_moe_route(None, None, k, renorm, _dname(dt), logits=l)
    got_ids, got_w = ids.cpu().numpy(), wts.cpu().numpy().astype(np.float64)
    assert np.array_equal(got_ids, ref_ids), f"{what}: {int((got_ids != ref_ids).any(-1).sum())} rows select other experts or another slot order"
    spread = np.minimum(l.max(-1) - l.min(-1), 88.0).astype(np.float64)[:, None]
    tol = ref_w * (2 * (2.0 ** -22 + spread * 2.0 ** -23) + 48 * 2.0 ** -24) + 1e-37
    err = np.abs(got_w - ref_w)
    assert (err <= tol).all(), f"{what}: {int((~(err <= tol)).sum())} weights outside the bound, worst err/tol {np.nanmax(err / tol):.3g}"
    return float((err / tol).max())


@pytest.mark.parametrize("dt", [BF, FP], ids=["bf16", "fp16"])
@pytest.mark.parametrize("H,E,k", SHAPES)
def test_logits_elementwise_and_routing_from_them(H, E, k, dt):
    w = _weight(E, H, dt, seed=H + E)
    for T in TS:
        x = make_synthetic_activations(T, H, seed=T + k, dtype=dt, device="cuda")
        for renorm in (True, False):
            ids, wts, lg = _route(x, w, k, renorm)
            what = f"H{H}-E{E}-k{k}-T{T}-{_dname(dt)}-renorm{int(renorm)}"
            assert torch.equal(lg.to(dt).float(), lg), f"{what}: logits are not values of {dt}"
            worst_l = check(lg.to(dt), [x], w.t(), [E], what=f"{what}: logits")
            worst_w = _check_routing(ids, wts, lg, k, renorm, dt, what)
            ids2, wts2, _ = _route(x, w, k, renorm, logits=False)   # the logits output is optional and changes nothing
            assert torch.equal(ids, ids2) and torch.equal(wts, wts2), what
        print(f"\n[moe-route] {what}: max err/tol logits {worst_l:.3f} weights {worst_w:.3f}")


@pytest.mark.parametrize("dt", [BF, FP], ids=["bf16", "fp16"])
def test_ties_and_extremes(dt):
    H, E, k = 2048, 128, 8
    w = _weight(E, H, dt, seed=3)
    w[77], w[100] = w[5], w[5]                       # three experts with identical rows: exact ties, lower id first
    x = make_synthetic_activations(40, H, seed=9, dtype=dt, device="cuda")
    x[:, :] += w[5].float().mul(40.0).to(dt)        # ... and in the top k of every row
    ids, wts, lg = _route(x, w, k)
    assert torch.equal(lg[:, 5], lg[:, 77]) and torch.equal(lg[:, 5], lg[:, 100])
    _check_routing(ids, wts, lg, k, True, dt, "duplicate rows")
    pos = (ids == 5).nonzero()
    assert len(pos) == 40, "the duplicated expert must be selected in every row"
    for t, s in pos.tolist():
        assert ids[t, s:s + 3].tolist() == [5, 77, 100] and wts[t, s] == wts[t, s + 1] == wts[t, s + 2]

    # x = 0: every logit zero -> ids 0..k-1, weights 1/k renormalised and 1/E not
    z = torch.zeros(17, H, dtype=dt, device="cuda")
    for renorm, want in ((True, 1.0 / k), (False, 1.0 / E)):
        ids, wts, lg = _route(z, w, k, renorm)
        assert not lg.any() and torch.equal(ids, torch.arange(k, dtype=torch.int32, device="cuda").expand(17, k))
        assert torch.allclose(wts, torch.full_like(wts, want), rtol=1e-6, atol=0)

    # logits spanning +-60 (fp16) / +-300 (bf16): expert e's row is a multiple of one direction, x that direction
    span = 60.0 if dt == FP else 300.0
    E2 = 64
    u = torch.zeros(H, device="cuda")
    u[:128] = 1.0 / 128 ** 0.5
    scale = torch.linspace(-span, span, E2, device="cuda")
    w2 = (scale[:, None] * u[None, :]).to(dt)
    x2 = u[None, :].repeat(9, 1).to(dt)
    for renorm in (True, False):
        ids, wts, lg = _route(x2, w2, 6, renorm)
        assert float(lg.max()) > 0.9 * span and float(lg.min()) < -0.9 * span
        assert torch.isfinite(wts).all() and torch.isfinite(lg).all()
        _check_routing(ids, wts, lg, 6, renorm, dt, f"span {span}")
        if renorm:
            assert float((wts.double().sum(-1) - 1).abs().max()) <= 1e-6

    # top_k = E: every expert selected once, in descending logit order; the weights are the whole softmax
    for E3 in (1, 8, 16):
        w3 = _weight(E3, 256, dt, seed=E3)
        x3 = make_synthetic_activations(21, 256, seed=E3, dtype=dt, device="cuda")
        for renorm in (True, False):
            ids, wts, lg = _route(x3, w3, E3, renorm)
            assert torch.equal(ids.sort(-1).values, torch.arange(E3, dtype=torch.int32, device="cuda").expand(21, E3))
            _check_routing(ids, wts, lg, E3, renorm, dt, f"top_k = E = {E3}")
            assert float((wts.double().sum(-1) - 1).abs().max()) <= 1e-6


@pytest.mark.parametrize("H,E,k,dt", [(2048, 128, 8, BF), (4096, 8, 2, FP), (4096, 256, 8, BF), (2048, 60, 4, FP), (128, 8, 2, BF)])
def test_routing_of_a_row_does_not_depend_on_the_batch(H, E, k, dt):
    """Rows of a T = 1000 batch, alone (T = 1), inside a 16-row and a 129-row batch and in a permuted batch: bit-identical logits,
    ids and weights.  The plans differ in tile size, cluster size and the row's place in its tile (tests/test_moe_route_plan.py)."""
    w = _weight(E, H, dt, seed=11)
    x = make_synthetic_activations(1000, H, seed=5, dtype=dt, device="cuda")
    ids, wts, lg = _route(x, w, k)
    assert len({tuple(_cabi.debug_moe_route_plan(T, H, E, k, torch.cuda.get_device_properties(0).multi_processor_count)[:2])
                for T in (1, 16, 129, 1000)}) >= 2
    perm = torch.randperm(1000, generator=torch.Generator().manual_seed(1)).cuda()
    pi, pw, pl = _route(x[perm].contiguous(), w, k)
    assert torch.equal(pl, lg[perm]) and torch.equal(pi, ids[perm]) and torch.equal(pw, wts[perm])
    for t in (0, 7, 8, 531, 999):
        for rows in ([t], list(range(t - 15, t + 1)) if t >= 15 else list(range(t, t + 16)), list(range(min(max(0, t - 100), 871), min(max(0, t - 100), 871) + 129))):
            sel = torch.tensor(rows, device="cuda")
            si, sw, sl = _route(x[sel].contiguous(), w, k)
            j = rows.index(t)
            assert torch.equal(sl[j], lg[t]) and torch.equal(si[j], ids[t]) and torch.equal(sw[j], wts[t]), (t, len(rows))


def _block_case(name):
    from test_gpu_moe_grouped import _experts
    case = {"qwen3": MOE_CASES[8], "mixtral": MOE_CASES[3], "mixtral-fp16": MOE_CASES[4]}[name]
    blocks, ex = _experts(case.E, case.H, case.I, case.dtype, case.group, case.krot, big=True)
    return case, ex


def _fill(st):
    st.topk_ids.fill_(-1)
    st.topk_weights.fill_(float("nan"))
    st.h.fill_(float("nan"))
    st.y.fill_(float("nan"))
    if st.router is not None:
        st.logits.fill_(float("nan"))


@pytest.mark.parametrize("name", ["qwen3", "mixtral", "mixtral-fp16"])
def test_step_with_router(name, monkeypatch):
    case, ex = _block_case(name)
    counts = []
    for fn in ("moe_route", "moe_forward", "moe_grouped_forward"):
        orig = getattr(_cabi, fn)
        monkeypatch.setattr(_cabi, fn, lambda *a, _o=orig, **kw: (_o(*a, **kw), counts.append(_cabi.last_launch_count()))[0])
    for mode in ("decode", "prefill"):
        _step_with_router(case, ex, mode, counts)


def _step_with_router(case, ex, mode, counts):
    dt, k = case.dtype, case.k
    T = case.T if mode == "decode" else 40
    make = ex.decode_step if mode == "decode" else ex.prefill_step
    r = ParoRouter(_weight(case.E, case.H, dt, seed=21).cpu(), k, True, dtype=dt)
    st, plain = make(T, k, router=r), make(T, k)
    assert not hasattr(plain, "logits") and plain.router is None

    def run_both(x):
        for s in (st, plain):
            _fill(s)
            s.x.copy_(x)
        counts.clear()
        st.step()
        assert counts == ([1, 2] if mode == "decode" else [1, 6]), counts   # 3 / 7 launches
        ids, wts, lg = _route(x, r.weight, k)
        assert torch.equal(st.topk_ids, ids) and torch.equal(st.topk_weights, wts) and torch.equal(st.logits, lg)
        plain.topk_ids.copy_(st.topk_ids)
        plain.topk_weights.copy_(st.topk_weights)
        plain.step()
        assert torch.isfinite(st.y.float()).all() and torch.isfinite(st.h.float()).all()
        assert torch.equal(st.y, plain.y) and torch.equal(st.h, plain.h)

    x1 = make_synthetic_activations(T, case.H, seed=31, dtype=dt, device="cuda")
    run_both(x1)
    y1, ids1 = st.y.clone(), st.topk_ids.clone()

    # one CUDA graph from hidden state to block output: captured once, replayed on another x
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        st.step()
    torch.cuda.current_stream().wait_stream(side)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        st.step()
    x2 = make_synthetic_activations(T, case.H, seed=32, dtype=dt, device="cuda")
    run_both(x2)
    y2, ids2 = st.y.clone(), st.topk_ids.clone()
    assert not torch.equal(ids1, ids2), "the second input must route differently"
    for x, y in ((x1, y1), (x2, y2), (x1, y1)):
        _fill(st)
        st.x.copy_(x)
        graph.replay()
        torch.cuda.synchronize()
        assert torch.equal(st.y, y)
    assert torch.equal(st.topk_ids, ids1)


def test_router_mismatches_raise_at_construction():
    case, ex = _block_case("qwen3")
    k = case.k
    ok = _weight(case.E, case.H, case.dtype)
    for weight, kk, dt in ((ok[:64], k, BF), (ok[:, :1024], k, BF), (ok, k, FP), (ok, k - 1, BF)):
        with pytest.raises(RuntimeError, match="does not match"):
            ex.decode_step(4, k, router=ParoRouter(weight, kk, dtype=dt))
        with pytest.raises(RuntimeError, match="does not match"):
            ex.prefill_step(40, k, router=ParoRouter(weight, kk, dtype=dt))
