"""Host-side checks of the MoE expert block (paro_moe_forward): the launch plans cover every round exactly once for every
routing, the C ABI rejects invalid descriptors with a message, and the Python wrapper rejects CPU tensors and wrong dtypes.
No GPU needed."""
import ctypes

import pytest
import torch

from paroquant_b200 import _cabi

BF16 = torch.bfloat16


def _desc(H, I, E=8, *, dtype=BF16, group=128, krot=8, gu_parts=None, down_out=None, down_dtype=None, down_group=None, down_krot=None,
          gu_stride=None, down_stride=None):
    gu = _cabi.make_shape(H, gu_parts or [I, I], group, krot, dtype)
    dn = _cabi.make_shape(I, [down_out or H], down_group or group, down_krot or krot, down_dtype or dtype)
    d = _cabi.ParoMoEDesc()
    d.gate_up, d.down, d.n_experts = ctypes.pointer(gu), ctypes.pointer(dn), E
    d.gate_up_packed, d.down_packed = 1 << 20, 1 << 30   # never dereferenced by the host-only entry points
    d.gate_up_stride = gu_stride if gu_stride is not None else (_cabi.packed_bytes(gu) + 255) // 256 * 256
    d.down_stride = down_stride if down_stride is not None else (_cabi.packed_bytes(dn) + 255) // 256 * 256
    d._keep = (gu, dn)
    return d


@pytest.mark.parametrize("H,I,E", [(256, 384, 16), (2048, 768, 128), (4096, 14336, 8)])
@pytest.mark.parametrize("sms", [132, 114])
def test_plan_covers_every_round_once(H, I, E, sms):
    d = _desc(H, I, E)
    for T in range(1, 17):
        for k in (1, 2, 8):
            out = _cabi.debug_moe_plan(d, T, k, sms)
            assert out[16] == min(E, T * k)
            assert out[17] == 0, f"T={T} k={k}: {out[17]} coverage violations"
            for base, (K, N) in ((0, (H, 2 * I)), (8, (I, H))):
                c, S, grid, nb, groups, ng_max, nst, smem = out[base: base + 8]
                assert c in (1, 2, 4, 8) and grid == nb * c and nb == (N + 127) // 128 and groups == K // 128
                assert 1 <= S <= groups and ng_max == -(-groups // S)
                assert 4 <= nst <= 16 and nst % 2 == 0 and smem <= 227 * 1024   # even: the round loop's record pairs never wrap


def test_plan_keeps_both_reference_shapes_busy():
    # tiny experts with short K: one expert per rank; few big experts: K split so that every rank of a cluster has work
    q = _cabi.debug_moe_plan(_desc(2048, 768, 128), 1, 8, 132)
    assert q[8] * min(128, 8) * q[9] >= q[8] and q[10] >= 64            # down: >= 64 CTAs for 16 blocks
    m = _cabi.debug_moe_plan(_desc(4096, 14336, 8), 1, 2, 132)
    assert 2 * m[9] >= m[8], "every rank of a down cluster gets a K slice of one of the two experts"
    assert m[2] >= 132 and m[10] >= 64


def test_gpu_case_table_reaches_every_plan_feature():
    """The default plans at 132 SMs of the cases tests/test_gpu_moe.py runs (tests/moe_cases.py) cover every cluster size on
    each launch and the plan features where the kernel's cross-CTA reduction can go wrong; if the planner drifts away from
    one, this fails without a GPU."""
    from moe_cases import CASES
    cs = {0: set(), 8: set()}
    seen = set()
    for case in CASES:
        out = _cabi.debug_moe_plan(_desc(case.H, case.I, case.E, dtype=case.dtype, group=case.group, krot=case.krot), case.T, case.k, 132)
        assert out[17] == 0, f"{case.name}: {out[17]} coverage violations"
        U = out[16]
        for base in (0, 8):
            c, S, grid, nb, G, ng_max, nst, smem = out[base: base + 8]
            cs[base].add(c)
            waves = -(-U * S // c)
            if S > 1 and G % S:
                seen.add("uneven K slices")
            if any((u * S) // c != (u * S + S - 1) // c for u in range(U)):
                seen.add("an expert's slices split across a wave boundary")
            if waves >= 3:
                seen.add("three or more waves: both receive buffers reused")
            if (U * S) % c:
                seen.add("a partial last wave")
            if ng_max > nst:
                seen.add("a work item longer than the weight ring")
    assert cs[0] == {1, 2, 4, 8}, f"gate_up cluster sizes {sorted(cs[0])}"
    assert cs[8] == {1, 2, 4, 8}, f"down cluster sizes {sorted(cs[8])}"
    assert seen == {"uneven K slices", "an expert's slices split across a wave boundary", "three or more waves: both receive buffers reused",
                    "a partial last wave", "a work item longer than the weight ring"}, sorted(seen)


def _rc(fn, *args):
    rc = fn(*args)
    return rc, _cabi.lib().paro_last_error().decode()


@pytest.mark.parametrize("kw,T,k,code,msg", [
    ({}, 0, 2, 2, "T <= 16"),
    ({}, 17, 2, 2, "T <= 16"),
    ({}, 4, 0, 2, "top_k"),
    ({}, 4, 17, 2, "top_k"),
    ({}, 16, 9, 2, "T * top_k <= 128"),
    ({"gu_parts": [384, 256]}, 1, 2, 1, "two partitions"),
    ({"gu_parts": [768]}, 1, 2, 1, "two partitions"),
    ({"down_out": 384}, 1, 2, 1, "out_features = hidden"),
    ({"down_dtype": torch.float16}, 1, 2, 1, "agree on dtype"),
    ({"down_group": 64}, 1, 2, 1, "agree on dtype, group_size and krot"),
    ({"down_krot": 3}, 1, 2, 1, "krot"),
    ({"gu_stride": 256}, 1, 2, 1, "strides"),
    ({"down_stride": 1 << 20 | 128}, 1, 2, 1, "multiples of 256"),
    ({"E": 0}, 1, 2, 1, "n_experts"),
])
def test_abi_rejects_invalid(kw, T, k, code, msg):
    kw = dict(kw)
    E = kw.pop("E", 8)
    d = _desc(256, 384, E, **kw)
    L = _cabi.lib()
    out = (ctypes.c_int32 * 18)()
    rc, err = _rc(L.paro_debug_moe_plan, ctypes.byref(d), T, k, 132, out)
    assert rc == code and msg in err, (rc, err)
    assert L.paro_moe_workspace_bytes(ctypes.byref(d), T, k) == 0
    rc, err = _rc(L.paro_moe_forward, ctypes.byref(d), 16, 16, 16, T, k, 16, 16, 256, 256, None)
    assert rc == code and msg in err, (rc, err)


def test_abi_rejects_null_and_misaligned():
    d = _desc(256, 384)
    L = _cabi.lib()
    rc, err = _rc(L.paro_moe_forward, None, 16, 16, 16, 1, 2, 16, 16, 256, 256, None)
    assert rc == 1 and "null" in err
    rc, err = _rc(L.paro_moe_forward, ctypes.byref(d), None, 16, 16, 1, 2, 16, 16, 256, 256, None)
    assert rc == 1 and "null pointer" in err
    rc, err = _rc(L.paro_moe_forward, ctypes.byref(d), 18, 16, 16, 1, 2, 16, 16, 256, 256, None)
    assert rc == 1 and "aligned" in err


def test_wrapper_rejects_cpu_tensors_and_wrong_dtypes():
    d = _desc(256, 384)
    T, k = 2, 2
    x, h, y = torch.zeros(T, 256, dtype=BF16), torch.zeros(T, k, 768, dtype=BF16), torch.zeros(T, 256, dtype=BF16)
    ids, w, ws = torch.zeros(T, k, dtype=torch.int32), torch.zeros(T, k), torch.zeros(256, dtype=torch.uint8)
    with pytest.raises(RuntimeError, match="CUDA-only"):
        _cabi.moe_forward(d, x, ids, w, h, y, ws)
    with pytest.raises(RuntimeError, match="int32"):
        _cabi.moe_forward(d, x, ids.long(), w, h, y, ws)
    with pytest.raises(RuntimeError, match="float32"):
        _cabi.moe_forward(d, x, ids, w.half(), h, y, ws)
    with pytest.raises(RuntimeError, match="x must be"):
        _cabi.moe_forward(d, x.half(), ids, w, h, y, ws)
