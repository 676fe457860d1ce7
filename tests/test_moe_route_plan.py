"""Host-side checks of the MoE router (paro_moe_route): the fp64 restatement of its semantics (np_moe_route in
tests/moe_route_reference.py) against a torch formulation and on ties, the launch plans (every (token tile, K slice) owned once;
the K slices a function of the hidden size alone), the C ABI's argument checks with their messages, and the Python wrappers'
rejections.  No GPU needed."""
import ctypes

import numpy as np
import pytest
import torch

from moe_route_reference import np_moe_route
from oracle.oracle import round_to
from paroquant_b200 import _cabi
from paroquant_b200.experts import ParoRouter

BF = torch.bfloat16


@pytest.mark.parametrize("dtype,tdt", [("bfloat16", torch.bfloat16), ("float16", torch.float16)])
@pytest.mark.parametrize("renorm", [True, False])
def test_oracle_agrees_with_torch(dtype, tdt, renorm):
    g = torch.Generator().manual_seed(7)
    T, H, E, k = 33, 256, 60, 4
    x, w = torch.randn(T, H, generator=g).to(tdt), (torch.randn(E, H, generator=g) * 0.1).to(tdt)
    ids, wts, logits = np_moe_route(x.float().numpy(), w.float().numpy(), k, renorm, dtype)
    ref_logits = (x.double() @ w.double().t()).to(tdt)
    assert np.array_equal(logits, ref_logits.float().numpy())
    p = torch.softmax(ref_logits.double(), -1)
    tw, ti = torch.topk(p, k, dim=-1)
    if renorm:
        tw = tw / tw.sum(-1, keepdim=True)
    distinct = np.array([len(set(r)) == E for r in logits.tolist()])      # torch.topk's order among equal values is unspecified
    assert distinct.sum() >= 5
    assert np.array_equal(ids[distinct], ti.numpy()[distinct])
    np.testing.assert_allclose(wts[distinct], tw.numpy()[distinct], rtol=1e-12)
    assert ids.dtype == np.int32 and wts.dtype == np.float64 and logits.dtype == np.float32


def test_oracle_tie_rule():
    rng = np.random.default_rng(0)
    H, E, k = 128, 16, 4
    w = round_to(rng.standard_normal((E, H)) * 0.1, "bfloat16")
    w[9], w[12] = w[3], w[3]                                              # duplicate router rows -> the lower id first
    x = round_to(rng.standard_normal((6, H)) + 8 * w[3], "bfloat16")
    ids, wts, logits = np_moe_route(x, w, k)
    assert np.array_equal(logits[:, 3], logits[:, 9]) and np.array_equal(logits[:, 3], logits[:, 12])
    assert (ids[:, :3] == [3, 9, 12]).all() and (wts[:, 0] == wts[:, 1]).all() and (wts[:, 1] == wts[:, 2]).all()
    assert (np.diff(np.take_along_axis(logits, ids, -1), axis=-1) <= 0).all()   # slot 0 is the largest
    # all-equal logits: ids 0..k-1, weights 1/k renormalised and 1/E not
    z = np.zeros((3, H), np.float32)
    for renorm, want in ((True, 1 / k), (False, 1 / E)):
        ids, wts, logits = np_moe_route(z, w, k, renorm)
        assert not logits.any() and (ids == np.arange(k)).all() and np.allclose(wts, want, rtol=1e-15)
    # routing of given logits: the first line of the semantics is skipped
    ids, wts, _ = np_moe_route(None, None, 2, True, logits=np.array([[1.0, 3.0, 3.0, -2.0]], np.float32))
    assert ids.tolist() == [[1, 2]] and wts.tolist() == [[0.5, 0.5]]


SHAPES = [(2048, 128), (4096, 8), (4096, 256), (2048, 60), (256, 1)]
TS = [1, 4, 16, 17, 129, 4096]


@pytest.mark.parametrize("H,E", SHAPES)
def test_plan_covers_every_tile_and_slice_once(H, E):
    slices = set()
    for T in TS:
        for sms in (132, 114, 16):
            nt, c, S, grid, smem, bad, tiles, threads = _cabi.debug_moe_route_plan(T, H, E, 1, sms)
            assert bad == 0, f"T={T} sms={sms}: {bad} coverage violations"
            assert nt in (8, 16, 32) and c in (1, 2, 4, 8) and S % c == 0 and H % (32 * S) == 0
            assert tiles == -(-T // nt) and grid == tiles * c and threads == 256
            assert smem == S * nt * ((E + 15) // 16 * 16 + 4) * 4 <= 227 * 1024
            slices.add(S)
    assert len(slices) == 1, "the K slices depend on the hidden size only"


def test_plan_shapes():
    # the slice count is a function of H: the same for every T, E and SM count
    for H in (128, 256, 384, 2048, 8192):
        assert {_cabi.debug_moe_route_plan(T, H, E, 1, sms)[2] for T in (1, 40, 5000) for E in (1, 64, 256) for sms in (8, 132)} == \
            {8 if H % 256 == 0 else 4}
    # few tokens: eight SMs pull the weight; many: one CTA per tile, many tiles
    assert _cabi.debug_moe_route_plan(1, 2048, 128, 8, 132)[:3] == [8, 8, 8]
    assert _cabi.debug_moe_route_plan(16, 2048, 128, 8, 132)[:4] == [8, 8, 8, 16]
    nt, c, S, grid = _cabi.debug_moe_route_plan(4096, 2048, 128, 8, 132)[:4]
    assert (nt, c, grid) == (32, 1, 128)
    assert _cabi.debug_moe_route_plan(4096, 4096, 256, 8, 132)[0] == 16        # the receive buffer of 32 tokens would not fit
    # the plan does not depend on top_k
    assert _cabi.debug_moe_route_plan(129, 2048, 128, 1, 132) == _cabi.debug_moe_route_plan(129, 2048, 128, 8, 132)


def _buf():
    buf = (ctypes.c_char * 4096)()
    return buf, (ctypes.addressof(buf) + 255) // 256 * 256


def test_abi_argument_checks():
    L = _cabi.lib()
    assert L.paro_abi_version() == _cabi.ABI_VERSION == 5
    buf, p = _buf()
    good = dict(x=p, w=p, dtype=_cabi.BF16, T=4, H=256, E=8, k=2, renorm=1, ids=p, wts=p, logits=p)
    for change, code, msg in (
            (dict(dtype=_cabi.F32), 1, "F16 or BF16"), (dict(dtype=7), 1, "F16 or BF16"), (dict(renorm=2), 1, "renormalize must be 0 or 1"),
            (dict(T=-1), 1, "negative token count"), (dict(H=200), 2, "multiple of 128"), (dict(H=0), 2, "multiple of 128"),
            (dict(E=0), 2, "n_experts <= 256"), (dict(E=257), 2, "n_experts <= 256"), (dict(k=0), 2, "top_k <= min(n_experts, 16)"),
            (dict(k=9), 2, "top_k <= min(n_experts, 16)"), (dict(E=64, k=17), 2, "top_k <= min(n_experts, 16)"),
            (dict(T=1 << 31), 2, "T <= 2147483647"),
            (dict(x=None), 1, "null pointer"), (dict(w=None), 1, "null pointer"), (dict(ids=None), 1, "null pointer"),
            (dict(wts=None), 1, "null pointer"), (dict(x=p + 8), 1, "16-byte"), (dict(w=p + 4), 1, "16-byte"),
            (dict(ids=p + 2), 1, "4-byte aligned"), (dict(wts=p + 1), 1, "4-byte aligned"), (dict(logits=p + 2), 1, "4-byte aligned")):
        a = dict(good, **change)
        rc = L.paro_moe_route(a["x"], a["w"], a["dtype"], a["T"], a["H"], a["E"], a["k"], a["renorm"], a["ids"], a["wts"], a["logits"], None)
        err = L.paro_last_error().decode()
        assert rc == code and msg in err, (change, rc, err)
        assert L.paro_last_launch_count() == 0
    # T = 0: success, nothing launched, no pointer looked at
    assert L.paro_moe_route(None, None, _cabi.F16, 0, 256, 8, 2, 0, None, None, None, None) == 0 and L.paro_last_launch_count() == 0
    # the plan hook: the same limits, its own arguments
    out = (ctypes.c_int32 * 8)()
    for args, code, msg in (((4, 200, 8, 2, 132), 2, "multiple of 128"), ((4, 256, 300, 2, 132), 2, "n_experts"), ((4, 256, 8, 9, 132), 2, "top_k"),
                            ((0, 256, 8, 2, 132), 1, "empty batch"), ((4, 256, 8, 2, 0), 1, "bad arguments")):
        rc = L.paro_debug_moe_route_plan(*args, out)
        assert rc == code and msg in L.paro_last_error().decode(), (args, rc, L.paro_last_error())
    assert L.paro_debug_moe_route_plan(4, 256, 8, 2, 132, None) == 1


def test_wrapper_rejections():
    T, H, E, k = 3, 256, 8, 2
    x, w = torch.zeros(T, H, dtype=BF), torch.zeros(E, H, dtype=BF)
    ids, wts, lg = torch.zeros(T, k, dtype=torch.int32), torch.zeros(T, k), torch.zeros(T, E)
    with pytest.raises(RuntimeError, match="CUDA-only"):
        _cabi.moe_route(x, w, k, True, ids, wts, lg)
    with pytest.raises(RuntimeError, match="CUDA-only"):
        _cabi.moe_route(x, w, k, True, ids, wts)
    with pytest.raises(RuntimeError, match="float16 or bfloat16"):
        _cabi.moe_route(x.float(), w.float(), k, True, ids, wts)
    with pytest.raises(RuntimeError, match="share"):
        _cabi.moe_route(x, w.half(), k, True, ids, wts)
    with pytest.raises(RuntimeError, match="int32"):
        _cabi.moe_route(x, w, k, True, ids.long(), wts)
    with pytest.raises(RuntimeError, match="float32"):
        _cabi.moe_route(x, w, k, True, ids, wts.half())
    with pytest.raises(RuntimeError, match="float32"):
        _cabi.moe_route(x, w, k, True, ids, wts, lg.double())


def test_router_construction_checks():
    with pytest.raises(RuntimeError, match=r"\[n_experts, hidden\]"):
        ParoRouter(torch.zeros(8), 2, device="cpu")
    with pytest.raises(RuntimeError, match="float16 or bfloat16"):
        ParoRouter(torch.zeros(8, 256), 2, dtype=torch.float32, device="cpu")
    for shape, k in (((8, 200), 2), ((257, 256), 2), ((8, 256), 9), ((8, 256), 0), ((64, 256), 17)):
        with pytest.raises(RuntimeError, match="supported"):
            ParoRouter(torch.zeros(*shape), k, device="cpu")
    r = ParoRouter(torch.randn(8, 256), 2, renormalize=False, dtype=torch.float16, device="cpu")
    assert (r.n_experts, r.hidden, r.top_k, r.renormalize) == (8, 256, 2, False) and r.weight.dtype == torch.float16 and r.weight.is_contiguous()


def test_router_from_checkpoint():
    class Ck:
        dense = {"model.layers.3.mlp.gate.weight": torch.randn(8, 256).half()}
    r = ParoRouter.from_checkpoint(Ck, "model.layers.3.mlp.experts", 2, dtype=torch.float16, device="cpu")
    assert torch.equal(r.weight, Ck.dense["model.layers.3.mlp.gate.weight"]) and r.top_k == 2 and r.renormalize
    with pytest.raises(RuntimeError, match=r"no router weight 'model\.layers\.4\.mlp\.gate\.weight'"):
        ParoRouter.from_checkpoint(Ck, "model.layers.4.mlp.experts", 2, device="cpu")
