"""Launch plan of the M <= 16 kernel (host logic of paroquant_b200/csrc/paro_decode.cu) through the test hook
paro_debug_decode_plan: no GPU.  The kernel's own index arithmetic is re-stated here and must cover every
(128-column block, group) of the layer exactly once, inside the shared-memory and barrier constraints the kernel relies on."""
import ctypes

import pytest
import torch

from paroquant_b200 import _cabi

SMEM_LIMIT = 227 * 1024
REC = {128: 8576, 64: 8960}   # record = ring stage: group_size 64 carries two scale / zero sets (paro_layout.h)


def plan(K, parts, M, sets=5, sms=132, resident=(132, 66, 32, 16), group=128):
    shape = _cabi.make_shape(K, parts, group, 8, torch.bfloat16)
    out = (ctypes.c_int32 * 20)()
    res = (ctypes.c_int32 * 4)(*resident)
    lib = _cabi.lib()
    lib.paro_debug_decode_plan.restype = ctypes.c_int
    rc = lib.paro_debug_decode_plan(ctypes.byref(shape), ctypes.c_int64(M), sets, sms, res, out)
    if rc:
        raise RuntimeError(lib.paro_last_error().decode())
    v = list(out)
    keys = ["c", "ranges", "grid", "nj_max", "ng_max", "nstages", "rot_warps", "smem", "xb_off", "recv_off", "bar_off"]
    return dict(zip(keys, v[:11])), v[11:20]


SHAPES = [(4096, [4096]), (4096, [4096, 1024, 1024]), (4096, [14336, 14336]), (14336, [4096]), (11008, [4096]), (8192, [1024]),
          (128, [128]), (256, [272, 16]), (640, [48, 16, 32]), (512, [512, 128, 128]), (1792, [4096]), (1024, [1024, 256, 256]),
          (3584, [4096]), (4096, [3584, 3584]), (12288, [4096]), (4096, [12288, 12288])]


@pytest.mark.parametrize("K,parts", SHAPES)
@pytest.mark.parametrize("M", [1, 3, 4, 8, 9, 16])
@pytest.mark.parametrize("sets,group", [(5, 128), (6, 128), (5, 64)])
def test_plan_covers_the_layer_once_and_fits(K, parts, M, sets, group):
    p, prb = plan(K, parts, M, sets, group=group)
    c, groups = p["c"], K // 128
    blocks = [(n + 127) // 128 for n in parts]
    assert c in (1, 2, 4, 8) and c <= groups
    assert p["grid"] == p["ranges"] * c and p["ranges"] <= (132, 66, 32, 16)[c.bit_length() - 1]
    assert p["ranges"] >= len(parts) and prb[0] == 0 and prb[len(parts)] == p["ranges"]
    # ---- the kernel's index arithmetic (decode_kernel prologue), CTA by CTA
    seen = {}
    nj_max = ng_max = 0
    for cta in range(p["grid"]):
        rng, sl = cta // c, cta % c
        part = 0
        while rng >= prb[part + 1]:
            part += 1
        jl, cp, cbp = rng - prb[part], prb[part + 1] - prb[part], blocks[part]
        cb0, cb1 = jl * cbp // cp, (jl + 1) * cbp // cp
        g0, g1 = sl * groups // c, (sl + 1) * groups // c
        assert cb1 > cb0 and g1 > g0, "a CTA without work would hang its cluster barrier"
        nj_max, ng_max = max(nj_max, cb1 - cb0), max(ng_max, g1 - g0)
        for cb in range(cb0, cb1):
            for g in range(g0, g1):
                key = (part, cb, g)
                assert key not in seen
                seen[key] = cta
    assert len(seen) == sum(blocks) * groups
    assert nj_max == p["nj_max"] and ng_max == p["ng_max"]
    # ---- constraints the kernel relies on
    assert p["nstages"] % sets == 0 and sets <= p["nstages"] <= 24          # a ring stage is always consumed by the same set
    ntasks = p["ng_max"] * ((M + 3) // 4 if M > 4 else 1)
    assert 1 <= p["rot_warps"] <= min(4 * sets, ntasks)
    assert p["smem"] <= SMEM_LIMIT
    assert p["xb_off"] >= p["nstages"] * REC[group] and p["xb_off"] % 128 == 0
    rot_bytes = 256 * (1 if M == 1 else 2 if M == 2 else 4)
    recv = ((p["nj_max"] + c - 1) // c) * c * M * 512 if c > 1 else 0
    assert p["recv_off"] >= p["xb_off"] + p["ng_max"] * 4096 + p["rot_warps"] * rot_bytes    # B operand, then the rotation tiles
    assert p["bar_off"] >= p["recv_off"] + recv and p["bar_off"] % 16 == 0
    assert p["smem"] >= p["bar_off"] + 16 * 24 + 224                                        # ring barriers + the fixed ones


def test_plan_uses_the_machine_for_the_llama_shapes():
    """Busiest CTA within 20 % of a perfect split for the big layers; small layers use at least 128 CTAs."""
    for K, parts, slack in ((4096, [14336, 14336], 1.2), (14336, [4096], 1.2), (4096, [4096], 1.2), (4096, [4096, 1024, 1024], 1.6)):
        p, _ = plan(K, parts, 1)
        units = sum((n + 127) // 128 for n in parts) * (K // 128)
        assert p["nj_max"] * p["ng_max"] <= slack * units / 132 + 1, (K, parts, p)
        assert p["grid"] >= 96
    # large M: the DSMEM receive buffer must not crowd the weight ring down to one stage per set
    for K, parts in ((4096, [14336, 14336]), (4096, [4096]), (14336, [4096])):
        p, _ = plan(K, parts, 16)
        assert p["nstages"] >= 10, (K, parts, p)


def test_plan_without_clusters_and_errors():
    p, _ = plan(4096, [4096], 1, resident=(132, 0, 0, 0))
    assert p["c"] == 1 and p["grid"] == 32 and p["ng_max"] == 32          # one CTA per block, whole K
    with pytest.raises(RuntimeError, match="no launch configuration fits"):
        plan(14336, [4096], 1, resident=(132, 0, 0, 0))                  # 112 groups of B operand do not fit one CTA
    with pytest.raises(RuntimeError, match="bad M"):
        plan(4096, [4096], 17)
