"""Shapes of the fused rotate backward (paro_rotate_backward) that tests/test_gpu_rotate_backward.py runs, with the part of the
launch plan each is there for (a helper module: pytest does not collect it).  tests/test_reference_check.py asserts the property
of every case through paro_debug_rotate_backward_plan at 132 SMs (an H100 SXM), the GPU tests at the device's own SM count.

A warp of the backward owns one group and walks row blocks of 4 rows split, split + splits, ...; it sums its blocks' dL/dtheta and
dL/dscale partials and adds them to the fp32 outputs with one atomic per entry.  The kinds:

  multi    every warp walks at least 2 row blocks (its running sum adds several blocks, and reloads its tiles after a block's
           grad_x stores)
  uneven   multi, warps walk different numbers of blocks, and the last block is ragged (M % 4 != 0)
  smem     multi, and the dynamic shared memory is above 48 KB (the opt-in path) for every formula of the case
  few      one or two blocks per warp and about 1000 or more warp partials (atomics) per entry
  tiny     fewer rows than one block
"""
import torch

F32, F16, BF16 = torch.float32, torch.float16, torch.bfloat16
GRAD, REF, BOTH = (False,), (True,), (False, True)

# (x dtype, group, krot, M, K, theta formulas (reference_formula values), kind)
CASES = [
    (F32, 128, 8, 4096, 4096, GRAD, "multi"),
    (F32, 128, 8, 14333, 4096, GRAD, "uneven"),
    (BF16, 128, 8, 4093, 4096, BOTH, "multi"),
    (F16, 64, 16, 4097, 2048, GRAD, "multi"),
    (F32, 64, 8, 4096, 4096, GRAD, "multi"),
    (F32, 128, 13, 4095, 4096, GRAD, "smem"),
    (F32, 128, 16, 2049, 4096, BOTH, "smem"),
    (BF16, 128, 10, 4096, 4096, REF, "smem"),
    (F32, 64, 1, 8191, 192, GRAD, "few"),
    (F32, 128, 8, 16383, 128, GRAD, "few"),
    (F32, 64, 3, 1, 192, GRAD, "tiny"),
    (F16, 64, 3, 3, 192, GRAD, "tiny"),
]

STATIC_SMEM_LIMIT = 48 * 1024


def case_id(c) -> str:
    dt, G, krot, M, K, forms, kind = c
    f = "both" if len(forms) == 2 else ("ref" if forms[0] else "grad")
    return f"{str(dt).split('.')[-1]}-G{G}-krot{krot}-M{M}-K{K}-{f}-{kind}"


def assert_plan_reaches(plan: dict, kind: str, M: int, what: str = "") -> None:
    """The property `kind` of one plan (a dict of _cabi.debug_rotate_backward_plan)."""
    lo, hi = plan["min_blocks_per_warp"], plan["max_blocks_per_warp"]
    if kind in ("multi", "uneven", "smem"):
        assert lo >= 2, (what, plan)
    if kind == "uneven":
        assert hi > lo and M % 4 != 0, (what, plan)
    if kind == "smem":
        assert plan["dyn_smem"] > STATIC_SMEM_LIMIT, (what, plan)
    if kind == "few":
        assert hi == 2 and lo >= 1 and plan["splits"] >= 1000, (what, plan)
    if kind == "tiny":
        assert plan["row_blocks"] == 1 and plan["splits"] == 1 and M < 4, (what, plan)
