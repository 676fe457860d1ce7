"""Work split of the small-M kernel (host logic of paroquant_b200/csrc/paro_stream.cu) through the test hook
paro_debug_stream_plan: no GPU.  The kernel's own index arithmetic (step_geom, round_owner, the contributor slots of
the fix-up) is re-stated here and must cover every (128-column block, group) of the layer exactly once, give every
contributor of a block its own slot below max_slots, and agree with the arrival count the last-arriver test uses."""
import ctypes

import pytest
import torch

from paroquant_b200 import _cabi


def plan(K, parts, M, sets=5, ctas=132):
    shape = _cabi.make_shape(K, parts, 128, 8, torch.bfloat16)
    out = (ctypes.c_int32 * 16)()
    rc = _cabi.lib().paro_debug_stream_plan(ctypes.byref(shape), M, sets, ctas, out)
    if rc:
        raise RuntimeError(_cabi.lib().paro_last_error().decode())
    v = list(out)
    return dict(zip(["c", "T", "max_slots", "ng_max", "max_rounds"], v[:5])), v[5:14]


def round_owner(r, Rp, Tp):
    return ((r + 1) * Tp - 1) // Rp


def geom(cta, c, T, pcb, groups, blocks):
    """step_geom(): None for a CTA without a team."""
    if cta >= c * T:
        return None
    sl, u = cta % c, cta // c
    part = 0
    while u >= pcb[part + 1]:
        part += 1
    t, Tp = u - pcb[part], pcb[part + 1] - pcb[part]
    g0, g1 = sl * groups // c, (sl + 1) * groups // c
    ng = g1 - g0
    Rp = blocks[part] * ng
    return dict(part=part, slice=sl, t=t, Tp=Tp, g0=g0, ng=ng, r0=t * Rp // Tp, r1=(t + 1) * Rp // Tp, Rp=Rp)


SHAPES = [(4096, [4096]), (4096, [4096, 1024, 1024]), (4096, [14336, 14336]), (14336, [4096]), (11008, [4096]), (8192, [1024]),
          (128, [128]), (256, [272, 16]), (640, [48, 16, 32]), (512, [512, 128, 128]), (1792, [4096]), (1024, [1024, 256, 256]),
          (3584, [4096]), (4096, [3584, 3584]), (12288, [4096]), (4096, [12288, 12288]), (2048, [4096]), (512, [4096]),
          (4096, [512, 128, 128]), (4096, [1792, 1792])]


@pytest.mark.parametrize("K,parts", SHAPES)
@pytest.mark.parametrize("M", [1, 4, 8, 9, 16])
@pytest.mark.parametrize("ctas", [148, 132, 16])
def test_plan_covers_the_layer_once(K, parts, M, ctas):
    p, pcb = plan(K, parts, M, ctas=ctas)
    c, T, groups = p["c"], p["T"], K // 128
    blocks = [(n + 127) // 128 for n in parts]
    assert 1 <= c <= min(groups, 16) and c * T <= ctas and T >= len(parts)
    assert pcb[0] == 0 and pcb[len(parts)] == T and all(pcb[i + 1] > pcb[i] for i in range(len(parts)))
    seen, slots = {}, {}
    max_rounds = ng_max = 0
    for cta in range(ctas):
        g = geom(cta, c, T, pcb, groups, blocks)
        if g is None:
            continue
        ng_max = max(ng_max, g["ng"])
        max_rounds = max(max_rounds, g["r1"] - g["r0"])
        for r in range(g["r0"], g["r1"]):
            jb, gi = divmod(r, g["ng"])
            key = (g["part"], jb, g["g0"] + gi)
            assert key not in seen, f"round {key} dequantised twice"
            seen[key] = cta
            assert round_owner(r, g["Rp"], g["Tp"]) == g["t"]
        # the segments the epilogue group walks, and the slot each lands in
        r = g["r0"]
        while r < g["r1"]:
            jb = r // g["ng"]
            rb = min((jb + 1) * g["ng"], g["r1"])
            total = myslot = 0
            for s in range(c):
                ngs = (s + 1) * groups // c - s * groups // c
                Rp = blocks[g["part"]] * ngs
                lo, hi = round_owner(jb * ngs, Rp, g["Tp"]), round_owner((jb + 1) * ngs - 1, Rp, g["Tp"])
                if s == g["slice"]:
                    assert lo <= g["t"] <= hi
                    myslot = total + g["t"] - lo
                total += hi - lo + 1
            assert 0 <= myslot < total <= p["max_slots"]
            entry = slots.setdefault((g["part"], jb), {"total": total, "used": set()})
            assert entry["total"] == total, "contributors disagree on the arrival count"
            assert myslot not in entry["used"], "two contributors share a slot"
            entry["used"].add(myslot)
            r = rb
    assert len(seen) == sum(blocks) * groups, "some (block, group) is never dequantised"
    for key, e in slots.items():
        assert len(e["used"]) == e["total"], f"block {key}: {len(e['used'])} arrivals, the last-arriver test waits for {e['total']}"
    assert len(slots) == sum(blocks)
    assert ng_max == p["ng_max"] and max_rounds <= p["max_rounds"]


def test_llama_shapes_are_balanced():
    """Rounds of the busiest CTA stay within a few percent of the ideal share on the headline shapes (132 SMs)."""
    for K, parts in [(4096, [4096]), (4096, [4096, 1024, 1024]), (4096, [14336, 14336]), (14336, [4096])]:
        p, _ = plan(K, parts, 1)
        ideal = sum((n + 127) // 128 for n in parts) * (K // 128) / 132
        assert p["max_rounds"] <= ideal * 1.10 + 1, (K, parts, p, ideal)


def test_bad_arguments():
    shape = _cabi.make_shape(4096, [4096], 128, 8, torch.bfloat16)
    out = (ctypes.c_int32 * 16)()
    assert _cabi.lib().paro_debug_stream_plan(ctypes.byref(shape), 17, 5, 148, out) != 0
    assert _cabi.lib().paro_debug_stream_plan(ctypes.byref(shape), 1, 9, 148, out) != 0


def deal_members(T, blocks):
    """stm_deal_members: T members of a slice dealt to the partitions by 128-column blocks (largest remainder), >= 1 each."""
    exact = [T * b / sum(blocks) for b in blocks]
    alloc = [max(1, int(e)) for e in exact]
    frac = [e - a for e, a in zip(exact, alloc)]
    while sum(alloc) < T:
        best = max(range(len(blocks)), key=lambda i: (frac[i], -i))
        alloc[best] += 1
        frac[best] -= 1
    return [0] + [sum(alloc[:i + 1]) for i in range(len(blocks))]


@pytest.mark.parametrize("K,parts", [(1024, [256, 128]), (512, [64]), (640, [48, 16, 32]), (2048, [384]), (4096, [4096, 1024, 1024])])
@pytest.mark.parametrize("c", [1, 2, 3, 5, 8, 16])
def test_forced_slices_count_only_members_with_rounds(K, parts, c):
    """PARO_DECODE_C forces the number of K slices.  On a small layer a team then has more members than rounds, and members
    without a round lie between the first and the last owner of a block's rounds: the kernel's seg table counts only the
    owners (min(hi - lo + 1, ngs) per slice; a lone round's owner takes slot round - first round of the block).  Every block
    must then get exactly `total` distinct slots below the planner's bound (the sum of hi - lo + 1), or its reducer waits
    for ever."""
    groups = K // 128
    if c > groups:
        pytest.skip("more slices than groups")
    T = 132 // c
    blocks = [(n + 127) // 128 for n in parts]
    pcb = deal_members(T, blocks)
    holes = False
    for part, nb in enumerate(blocks):
        Tp = pcb[part + 1] - pcb[part]
        for jb in range(nb):
            total = bound = 0
            used = set()
            for s in range(c):
                ngs = (s + 1) * groups // c - s * groups // c
                Rp = nb * ngs
                lo, hi = round_owner(jb * ngs, Rp, Tp), round_owner((jb + 1) * ngs - 1, Rp, Tp)
                n = min(hi - lo + 1, ngs)
                holes |= n < hi - lo + 1
                for t in range(Tp):                       # the members of slice s that own rounds of block jb
                    r0, r1 = t * Rp // Tp, (t + 1) * Rp // Tp
                    if max(r0, jb * ngs) < min(r1, (jb + 1) * ngs):
                        used.add(total + (max(r0, jb * ngs) - jb * ngs if n < hi - lo + 1 else t - lo))
                total += n
                bound += hi - lo + 1
            assert used == set(range(total)), (part, jb, sorted(used), total)
            assert total <= bound
    if (K, parts, c) == (1024, [256, 128], 3):
        assert holes, "this case must exercise a team with more members than rounds"
