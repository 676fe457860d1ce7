"""Host-side checks of the grouped MoE expert block (paro_moe_grouped_forward, ParoExperts.prefill_step): the C ABI rejects invalid
calls with a message before any device work, the tile size and tile bound of the plan, the workspace covers the regions the plan
reports, and the decode path keeps its own limit.  No GPU needed."""
import ctypes

import pytest
import torch

from paroquant_b200 import _cabi
from test_moe_plan import _desc

MAX_ENTRIES, MAX_EXPERTS = 65536, 1024


def _rc(fn, *args):
    rc = fn(*args)
    return rc, _cabi.lib().paro_last_error().decode()


def _forward(d, T, k, *, x=16, ids=16, w=16, h=16, y=16, ws=256, ws_bytes=None):
    L = _cabi.lib()
    if ws_bytes is None:
        ws_bytes = L.paro_moe_grouped_workspace_bytes(ctypes.byref(d), T, k) if d is not None else 256
    return _rc(L.paro_moe_grouped_forward, ctypes.byref(d) if d is not None else None, x, ids, w, T, k, h, y, ws, ws_bytes, None)


@pytest.mark.parametrize("T,k,E,code,msg", [
    (0, 2, 8, 2, "T >= 1"),
    (-3, 2, 8, 2, "T >= 1"),
    (4, 0, 8, 2, "top_k"),
    (4, 17, 8, 2, "top_k"),
    (MAX_ENTRIES + 1, 1, 8, 2, f"T * top_k <= {MAX_ENTRIES}"),
    (MAX_ENTRIES // 8 + 1, 8, 8, 2, f"T * top_k <= {MAX_ENTRIES}"),
    (4, 2, MAX_EXPERTS + 1, 2, f"n_experts <= {MAX_EXPERTS}"),
    (4, 2, 0, 1, "n_experts"),
])
def test_abi_rejects_unsupported_batches(T, k, E, code, msg):
    d = _desc(256, 384, E)
    L = _cabi.lib()
    out = (ctypes.c_int32 * 12)()
    rc, err = _rc(L.paro_debug_moe_grouped_plan, ctypes.byref(d), T, k, 132, out)
    assert rc == code and msg in err, (rc, err)
    assert L.paro_moe_grouped_workspace_bytes(ctypes.byref(d), T, k) == 0
    rc, err = _forward(d, T, k, ws_bytes=1 << 40)
    assert rc == code and msg in err, (rc, err)


def test_abi_accepts_the_limits():
    for T, k, E in ((MAX_ENTRIES, 1, 8), (MAX_ENTRIES // 16, 16, MAX_EXPERTS), (1, 16, 1)):
        assert _cabi.debug_moe_grouped_plan(_desc(256, 384, E), T, k, 132)[0] in (32, 64, 128)


@pytest.mark.parametrize("kw,msg", [
    ({"gu_parts": [384, 256]}, "two partitions"),
    ({"down_out": 384}, "out_features = hidden"),
    ({"down_krot": 3}, "krot"),
    ({"gu_stride": 256}, "strides"),
])
def test_abi_rejects_invalid_descriptors(kw, msg):
    rc, err = _forward(_desc(256, 384, **kw), 40, 2, ws_bytes=1 << 40)
    assert rc == 1 and msg in err, (rc, err)


def test_abi_rejects_null_and_misaligned():
    d = _desc(256, 384)
    rc, err = _forward(None, 40, 2)
    assert rc == 1 and "null" in err
    for arg in ("x", "ids", "w", "h", "y", "ws"):
        rc, err = _forward(d, 40, 2, **{arg: None})
        assert rc == 1 and "null pointer" in err, (arg, err)
    for arg, bad in (("x", 24), ("h", 8), ("y", 40), ("ids", 18), ("w", 2), ("ws", 128)):
        rc, err = _forward(d, 40, 2, **{arg: bad})
        assert rc == 1 and "aligned" in err, (arg, err)
    packed = _desc(256, 384)
    packed.down_packed = (1 << 30) + 128
    rc, err = _forward(packed, 40, 2)
    assert rc == 1 and "aligned" in err


def test_abi_rejects_a_short_workspace_naming_the_size():
    d = _desc(2048, 768, 128)
    need = _cabi.moe_grouped_workspace_bytes(d, 512, 8)
    rc, err = _forward(d, 512, 8, ws_bytes=need - 1)
    assert rc == 4 and f"need {need}" in err, (rc, err)


def test_tile_size_and_tile_bound():
    """NT is one of 32 / 64 / 128, depends on (T, k, E) only, and tiles_max = floor(T k / NT) + min(E, T k): an expert with c
    entries takes ceil(c / NT) <= floor(c / NT) + 1 tiles, and at most min(E, T k) experts have entries."""
    seen = set()
    for E in (1, 8, 64, 128, 1024):
        for k in (1, 2, 8, 16):
            for T in (1, 2, 7, 16, 17, 40, 129, 512, 1000, 4096):
                if T * k > MAX_ENTRIES:
                    continue
                plans = [_cabi.debug_moe_grouped_plan(_desc(H, I, E), T, k, 132) for H, I in ((256, 384), (4096, 1536))]
                nt, slots = plans[0][:2]
                assert nt in (32, 64, 128)
                assert plans[1][:2] == [nt, slots], "the tile plan depends on the expert shapes"
                n = T * k
                assert slots == n // nt + min(E, n), (T, k, E, nt, slots)
                seen.add(nt)
    assert seen == {32, 64, 128}


@pytest.mark.parametrize("H,I,E,k", [(256, 384, 8, 2), (2048, 768, 128, 8), (4096, 14336, 8, 2), (1024, 128, 64, 1)])
@pytest.mark.parametrize("T", [1, 17, 129, 1000, 4096])
def test_workspace_covers_the_regions(H, I, E, k, T):
    d = _desc(H, I, E)
    out = _cabi.debug_moe_grouped_plan(d, T, k, 132)
    nt, slots = out[:2]
    table, operand, ys, total = (v * 256 for v in out[8:12])
    rows = slots * nt
    assert table >= (rows + slots + 1) * 4
    assert operand >= rows * max(H, I) * 2
    assert ys >= T * k * H * 2
    assert total == table + operand + ys == _cabi.moe_grouped_workspace_bytes(d, T, k)
    blocks_gu, blocks_d = -(-2 * I // 128), -(-H // 128)
    assert out[2:8] == [1, -(-(rows // 8) * (H // 128) // 4), blocks_gu * slots, -(-(rows // 8) * (I // 128) // 4), blocks_d * slots, T]


def test_decode_path_still_rejects_more_than_16_tokens():
    d = _desc(256, 384)
    rc, err = _rc(_cabi.lib().paro_moe_forward, ctypes.byref(d), 16, 16, 16, 17, 2, 16, 16, 256, 256, None)
    assert rc == 2 and "T <= 16" in err
    assert _cabi.moe_grouped_workspace_bytes(d, 17, 2) > 0


def test_wrapper_rejects_cpu_tensors_and_wrong_dtypes():
    d = _desc(256, 384)
    T, k = 20, 2
    bf = torch.bfloat16
    x, h, y = torch.zeros(T, 256, dtype=bf), torch.zeros(T, k, 768, dtype=bf), torch.zeros(T, 256, dtype=bf)
    ids, w, ws = torch.zeros(T, k, dtype=torch.int32), torch.zeros(T, k), torch.zeros(256, dtype=torch.uint8)
    with pytest.raises(RuntimeError, match="CUDA-only"):
        _cabi.moe_grouped_forward(d, x, ids, w, h, y, ws)
    with pytest.raises(RuntimeError, match="moe_grouped_forward: topk_ids must be int32"):
        _cabi.moe_grouped_forward(d, x, ids.long(), w, h, y, ws)
    with pytest.raises(RuntimeError, match="moe_grouped_forward: h must be"):
        _cabi.moe_grouped_forward(d, x, ids, w, h.half(), y, ws)
    assert "paro_moe_grouped_forward" in _cabi.EXPORTED_SYMBOLS
