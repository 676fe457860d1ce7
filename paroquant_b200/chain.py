"""Chains of fused ParoQuant linears: several quantised linears of a transformer block with the element-wise ops vLLM puts
between them folded in -- for decode (M <= 16) in ONE launch (include/paro_b200.h: paro_chain_forward), for any M as a
pre-pass + GEMM pair per linear (paro_prefill_chain_forward).

The reference runs each quantised linear on its own (`ParoQuantLinearMethod.apply`,
/root/reference/paroquant/inference/backends/vllm/plugin.py:281-311); what sits between two of them in a Llama / Qwen
block is vLLM's `fused_add_rms_norm` and `silu_and_mul`.  The attention itself is not ours, so a block is cut there:

    [attention output] -> o_proj -> (+ residual, RMSNorm) -> gate_up -> (SiLU * up) -> down -> (+ residual, RMSNorm)
                       -> next block's qkv -> [q | k | v for the next attention]

`ParoChain` / `ParoPrefillChain` hold fixed device buffers (CUDA-graph friendly); `decoder_tail()` builds the chain above
for the row count it is given.
"""
from __future__ import annotations

import ctypes
from dataclasses import dataclass

import torch

from . import _cabi
from .linear import ParoLinearKernel, shared_workspace

XOP = {"none": _cabi.XOP_NONE, "silu_mul": _cabi.XOP_SILU_MUL, "rmsnorm": _cabi.XOP_RMSNORM}
EPI = {"store": _cabi.EPI_STORE, "add_residual": _cabi.EPI_ADD_RESIDUAL}
_LINEAR_HEAD = 256   # include/paro_b200.h, paro_workspace_bytes: the head the M <= 16 kernels keep their counters in


@dataclass
class ChainStep:
    """One linear of a chain.  x=None takes the previous step's output."""
    kernel: ParoLinearKernel
    x: torch.Tensor | None = None
    y: torch.Tensor | None = None
    bias: torch.Tensor | None = None
    x_op: str = "none"
    epilogue: str = "store"
    residual_in: torch.Tensor | None = None
    residual_out: torch.Tensor | None = None
    norm_weight: torch.Tensor | None = None
    eps: float = 1e-5
    row_parallel: bool = False     # K is sharded over the tensor-parallel group: the kernel sums the ranks' outputs itself


def _descriptors(steps: list[ChainStep], m: int, tp_group=None):
    """Check the steps against the C ABI's descriptor for m rows and build it: (ctypes array of ParoChainStep, the
    (ParoTpInfo, PeerBuffer) pairs of the row-parallel steps, which must live as long as the array)."""
    if not 1 <= len(steps) <= _cabi.CHAIN_MAX_STEPS:
        raise RuntimeError(f"1..{_cabi.CHAIN_MAX_STEPS} steps per chain, got {len(steps)}")
    dev = steps[0].kernel.packed.device
    dt = _cabi._CODE_DTYPE[steps[0].kernel.shape.dtype]
    arr = (_cabi.ParoChainStep * len(steps))()
    tp = []
    for i, s in enumerate(steps):
        for name in ("x", "y", "bias", "residual_in", "residual_out", "norm_weight"):
            t = getattr(s, name)
            if t is None:
                continue
            if not t.is_cuda or t.device != dev or t.dtype != dt or not t.is_contiguous():
                raise RuntimeError(f"chain step {i}: {name} must be a contiguous {dt} tensor on {dev}")
        n, k = s.kernel.shape.out_features, s.kernel.shape.in_features
        kin = 2 * k if s.x_op == "silu_mul" else k
        if s.x is not None and tuple(s.x.shape) != (m, kin):
            raise RuntimeError(f"chain step {i}: x must be [{m}, {kin}], got {tuple(s.x.shape)}")
        for name in ("y", "residual_in", "residual_out"):
            t = getattr(s, name)
            if t is not None and tuple(t.shape) != (m, n):
                raise RuntimeError(f"chain step {i}: {name} must be [{m}, {n}], got {tuple(t.shape)}")
        c = arr[i]
        c.shape = ctypes.pointer(s.kernel.shape)
        c.packed = s.kernel.packed.data_ptr()
        c.bias = None if s.bias is None else s.bias.data_ptr()
        c.x = None if s.x is None else s.x.data_ptr()
        c.y = None if s.y is None else s.y.data_ptr()
        c.x_op, c.epilogue = XOP[s.x_op], EPI[s.epilogue]
        c.residual_in = None if s.residual_in is None else s.residual_in.data_ptr()
        c.residual_out = None if s.residual_out is None else s.residual_out.data_ptr()
        c.norm_weight = None if s.norm_weight is None else s.norm_weight.data_ptr()
        c.eps = float(s.eps)
        if s.row_parallel:
            import torch.distributed as dist

            from .peer import PeerBuffer

            world = dist.get_world_size(tp_group)
            if world > 1:
                nb = _cabi.lib().paro_tp_slot_bytes(ctypes.byref(s.kernel.shape), m, world)
                if nb == 0:
                    raise RuntimeError(f"chain step {i}: {_cabi.lib().paro_last_error().decode()}")
                pb = PeerBuffer(nb, dev, tp_group)
                info = _cabi.ParoTpInfo()
                info.world, info.rank = world, dist.get_rank(tp_group)
                for r, ptr in enumerate(pb.ptrs):
                    info.peer_slots[r] = ptr
                tp.append((info, pb))
                c.tp = ctypes.pointer(info)
    return arr, tp


class ParoChain:
    """A planned chain over fixed buffers: `chain()` launches it on the current stream (one kernel)."""

    def __init__(self, steps: list[ChainStep], m: int, tp_group=None):
        if not 1 <= m <= 16:
            raise RuntimeError(f"chains serve decode batches of 1..16 rows, got {m}")
        self.steps, self.m = steps, int(m)
        self._arr, self._tp = _descriptors(steps, self.m, tp_group)
        nbytes = _cabi.chain_workspace_bytes(self._arr, len(steps), self.m)
        # counters at the head must start at zero; every launch leaves them zeroed
        self.workspace = torch.zeros(nbytes, dtype=torch.uint8, device=steps[0].kernel.packed.device)

    def __call__(self) -> None:
        _cabi.chain_forward(self._arr, len(self.steps), self.m, self.workspace)


class ParoPrefillChain:
    """The same steps for any m >= 1 (include/paro_b200.h: paro_prefill_chain_forward): per step the rotation pre-pass with the
    step's x op and the INT4 wgmma GEMM with its epilogue, 2 launches per step on the current stream.  The workspace is pure
    scratch, so it is the per-device shared scratch of the single linears (linear.shared_workspace), sized here, outside any
    capture.  Row-parallel (tensor-parallel) steps run only in ParoChain (m <= 16)."""

    def __init__(self, steps: list[ChainStep], m: int):
        if m < 1:
            raise RuntimeError(f"prefill chains need at least one row, got {m}")
        for i, s in enumerate(steps):
            if s.row_parallel:
                raise RuntimeError(f"prefill chain step {i}: row_parallel steps are not supported above 16 rows "
                                   "(the all-reduce between the GEMM and the residual epilogue is not fused); use ParoChain for "
                                   "m <= 16 or RowParallelLinear")
        self.steps, self.m = steps, int(m)
        self._arr, _ = _descriptors(steps, self.m)
        nbytes = _cabi.prefill_chain_workspace_bytes(self._arr, len(steps), self.m)
        # behind the shared scratch's 256-byte head: the single linears' launch epoch and counters live there
        self.workspace = shared_workspace(steps[0].kernel.packed.device, _LINEAR_HEAD + nbytes)[_LINEAR_HEAD:_LINEAR_HEAD + nbytes]

    def __call__(self) -> None:
        _cabi.prefill_chain_forward(self._arr, len(self.steps), self.m, self.workspace)


def decoder_tail(o: ParoLinearKernel, gate_up: ParoLinearKernel, down: ParoLinearKernel, next_qkv: ParoLinearKernel | None, *,
                 attn_out: torch.Tensor, residual: torch.Tensor, post_attn_norm: torch.Tensor, next_input_norm: torch.Tensor | None,
                 eps: float = 1e-5, tp_group=None, tensor_parallel: bool = False) -> tuple[ParoChain | ParoPrefillChain, dict[str, torch.Tensor]]:
    """o_proj .. next block's qkv as one chain, for any number of rows m: a ParoChain (one launch) for m <= 16, a
    ParoPrefillChain (two launches per linear) above.  Returns the chain and its output buffers:
    `residual_mid` / `residual_out` (the residual stream after attention / after the MLP), `mlp_act` (gate_up output),
    `qkv` (None for the last block: then `residual_out` is what the final norm + LM head consume).
    `tensor_parallel`: the kernels are this rank's shards (o / down row-sharded, gate_up / qkv column-sharded as vLLM shards
    them); the two all-reduces of the block happen inside the launch, the residual stream stays replicated.  Only for m <= 16."""
    m, dev, dt = attn_out.shape[0], attn_out.device, attn_out.dtype
    if m > 16 and tensor_parallel:
        raise RuntimeError(f"decoder_tail: tensor-parallel chains serve 1..16 rows, got {m}; above that the row-parallel "
                           "linears need their own all-reduce (RowParallelLinear)")
    hidden = o.shape.out_features
    bufs = {
        "residual_mid": torch.empty(m, hidden, dtype=dt, device=dev),
        "mlp_act": torch.empty(m, gate_up.shape.out_features, dtype=dt, device=dev),
        "residual_out": torch.empty(m, hidden, dtype=dt, device=dev),
        "qkv": None if next_qkv is None else torch.empty(m, next_qkv.shape.out_features, dtype=dt, device=dev),
    }
    steps = [
        ChainStep(o, x=attn_out, epilogue="add_residual", residual_in=residual, residual_out=bufs["residual_mid"], row_parallel=tensor_parallel),
        ChainStep(gate_up, x_op="rmsnorm", norm_weight=post_attn_norm, eps=eps, y=bufs["mlp_act"]),
        ChainStep(down, x_op="silu_mul", epilogue="add_residual", residual_in=bufs["residual_mid"], residual_out=bufs["residual_out"],
                  row_parallel=tensor_parallel),
    ]
    if next_qkv is not None:
        steps.append(ChainStep(next_qkv, x_op="rmsnorm", norm_weight=next_input_norm, eps=eps, y=bufs["qkv"]))
    if m > 16:
        return ParoPrefillChain(steps, m), bufs
    return ParoChain(steps, m, tp_group), bufs
