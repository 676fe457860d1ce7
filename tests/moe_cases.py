"""Shapes and routings that drive the MoE block (paro_moe_forward) through its launch plans (a helper module: pytest does not
collect it).  tests/test_moe_plan.py pins, without a GPU, that the default plans of these cases at 132 SMs cover every plan
feature below; tests/test_gpu_moe.py runs every case and routing and checks h and y element-wise, whatever plans the device
it runs on gets.

Plans at 132 SMs (cluster size c, K slices S; waves at U_max = min(E, T * k)):

  H, I, E          T, k   dtype, group, krot   gate_up                                  down
  256, 8192, 8     4, 1   bf16, 128, 8         c = 1, 4 waves                           c = 8, S = 2, 32 groups per item on 4 stages
  1024, 4096, 64   9, 1   bf16, 128, 8         c = 2, S = 2, 9 waves                    c = 8, S = 7 (an expert's slices cross a wave), 8 waves
  4096, 1536, 64   9, 1   fp16, 64, 3          c = 4, S = 2, 16 groups on 10 stages     c = 4, S = 3 (crosses waves), 7 waves
  4096, 14336, 8   1, 2   bf16, 128, 8         c = 4, S = 2                             c = 4, S = 4, 28 groups per item on 10 stages
  4096, 14336, 8   16, 2  fp16, 64, 5          c = 4, S = 2, 16 groups on 8 stages      c = 4, S = 7 (crosses waves), 14 waves, 16 groups on 8 stages
  4096, 128, 64    9, 1   bf16, 128, 8         c = 8, S = 7 of 32 groups (uneven)       c = 4, S = 1, 3 waves (the last partial)
  256, 128, 1      1, 1   bf16, 128, 8         c = 2, S = 2                             c = 1
  256, 128, 8      1, 2   fp16, 128, 8         c = 4, S = 2                             c = 2, S = 1
  2048, 768, 128   16, 8  bf16, 128, 8         c = 8, S = 2, 32 waves, 8 groups on 4    c = 8, 16 waves, 6 groups on 4 stages
  256, 384, 32     8, 16  bf16, 128, 8         c = 8, 4 waves                           c = 8, 4 waves

(the two Mixtral-shaped rows are Mixtral-8x7B's expert shapes, the 2048 / 768 / 128 row Qwen3-30B-A3B's)
"""
from __future__ import annotations

from dataclasses import dataclass

import torch


@dataclass(frozen=True)
class MoeCase:
    H: int
    I: int
    E: int
    T: int
    k: int
    dtype: torch.dtype = torch.bfloat16
    group: int = 128
    krot: int = 8

    @property
    def name(self) -> str:
        dt = "bf16" if self.dtype == torch.bfloat16 else "fp16"
        return f"H{self.H}-I{self.I}-E{self.E}-T{self.T}-k{self.k}-{dt}-g{self.group}-r{self.krot}"


CASES = [
    MoeCase(256, 8192, 8, 4, 1),
    MoeCase(1024, 4096, 64, 9, 1),
    MoeCase(4096, 1536, 64, 9, 1, torch.float16, 64, 3),
    MoeCase(4096, 14336, 8, 1, 2),
    MoeCase(4096, 14336, 8, 16, 2, torch.float16, 64, 5),
    MoeCase(4096, 128, 64, 9, 1),
    MoeCase(256, 128, 1, 1, 1),
    MoeCase(256, 128, 8, 1, 2, torch.float16),
    MoeCase(2048, 768, 128, 16, 8),
    MoeCase(256, 384, 32, 8, 16),
]

ROUTINGS = ("balanced", "skewed", "one_expert", "none_valid")


def routing(case: MoeCase, kind: str, seed: int = 0):
    """(ids [T, k] int32, weights [T, k] fp32) of one routing kind:
      balanced    distinct ids over the whole batch where T * k <= E, else every expert used: U = U_max
      skewed      every token's slot 0 on one hot expert (R = T tokens: two token tiles when T > 8), a duplicate id and a
                  dropped id (-1) elsewhere, the rest random
      one_expert  every slot on one expert (U = 1; duplicate ids in a token when k > 1)
      none_valid  ids -1 and E only (U = 0: on an expert-parallel rank none of the step's experts is local)
    Weights are softmax-like and distinct per slot, so a weight applied to the wrong slot changes the output."""
    T, k, E = case.T, case.k, case.E
    g = torch.Generator().manual_seed(1000 * seed + ROUTINGS.index(kind))
    w = torch.softmax(torch.randn(T, k, generator=g), -1)
    if kind == "balanced":
        ids = (torch.arange(T * k).reshape(T, k) + torch.randint(0, E, (1,), generator=g)) % E
    elif kind == "skewed":
        hot = int(torch.randint(0, E, (1,), generator=g))
        ids = torch.randint(0, E, (T, k), generator=g)
        ids[:, 0] = hot
        if k > 1:
            ids[0, 1] = ids[0, 0]                 # a duplicate id
            ids[T - 1, k - 1] = -1                # a dropped slot
    elif kind == "one_expert":
        ids = torch.full((T, k), int(torch.randint(0, E, (1,), generator=g)))
    elif kind == "none_valid":
        ids = torch.where(torch.rand(T, k, generator=g) < 0.5, -1, E)
    else:
        raise ValueError(kind)
    return ids.int(), w.float()
