"""MoE expert blocks on the fused kernels (SURVEY 8f rank 3).

The reference quantises a fused expert block with ONE rotation per projection shared by all experts
(`paroquant/cli/convert.py:281-381`: gate_up rotation on the hidden dim, down rotation on the intermediate dim; stored once as
`<base>.{gate_up,down}_weight_{theta,pairs,channel_scales}`) and serves it only through its MLX backend
(`inference/backends/mlx/modules.py:159-212`, `RotateSwitchGLU`: rotate x, per-expert gate / up, activation, rotate, per-expert
down).  Here every expert is two fused linears -- merged gate|up (two partitions carrying the same rotation) and down -- so an
expert costs two launches, or ONE for decode batches (a two-step chain with SiLU*up folded into the down step).  The rotation is
recomputed per selected expert inside the kernel (it is a prologue of a few microseconds).

`decode_step(T, top_k)` runs the whole block for a decode batch in two launches with the routing read on the device
(include/paro_b200.h: paro_moe_forward): no host synchronisation, CUDA-graph capturable with the routing changing between replays.
`prefill_step(T, top_k)` does the same for any T as grouped wgmma GEMMs in six launches (paro_moe_grouped_forward).
`ParoRouter` computes the routing itself (router logits, softmax, top-k) in one more launch; given to either step as `router=`,
the step runs from the hidden state to the block output with no torch op in between (3 and 7 launches).
"""
from __future__ import annotations

import ctypes

import torch

from . import _cabi
from .chain import ChainStep, ParoChain
from .checkpoint import ParoLayerBuffers, validate_pairs
from .linear import ParoLinearKernel


class ParoRouter:
    """The router of one MoE block: softmax over `weight [E, hidden] @ x`, the top_k experts (equal logits: the lower id first)
    and their probabilities, renormalised to sum to one when `renormalize` (Qwen3-MoE's norm_topk_prob; Mixtral), in one launch
    (include/paro_b200.h: paro_moe_route).  The weight is used as the checkpoint stores `mlp.gate.weight`, cast to the block's
    dtype.  A token's routing does not depend on the batch it is routed in."""

    def __init__(self, weight: torch.Tensor, top_k: int, renormalize: bool = True, dtype: torch.dtype = torch.bfloat16, device="cuda"):
        if weight.dim() != 2:
            raise RuntimeError(f"ParoRouter: weight must be [n_experts, hidden], got {tuple(weight.shape)}")
        if dtype not in (torch.float16, torch.bfloat16):
            raise RuntimeError(f"ParoRouter: dtype must be float16 or bfloat16, got {dtype}")
        self.n_experts, self.hidden = weight.shape
        self.top_k, self.renormalize, self.dtype = int(top_k), bool(renormalize), dtype
        if self.hidden % 128 or not 1 <= self.n_experts <= 256 or not 1 <= self.top_k <= min(self.n_experts, 16):
            raise RuntimeError(f"ParoRouter: hidden a multiple of 128, 1 <= n_experts <= 256 and 1 <= top_k <= min(n_experts, 16) supported, "
                               f"got weight {tuple(weight.shape)}, top_k = {top_k}")
        self.weight = weight.to(device=device, dtype=dtype).contiguous()

    @classmethod
    def from_checkpoint(cls, ck, experts_base: str, top_k: int, renormalize: bool = True, dtype: torch.dtype = torch.bfloat16,
                        device="cuda") -> "ParoRouter":
        """The router beside the expert block `experts_base` of a loaded checkpoint (`checkpoint_io.load_paro_checkpoint`): the
        dense tensor `<parent of experts_base>.gate.weight`."""
        name = experts_base.rsplit(".", 1)[0] + ".gate.weight"
        if name not in ck.dense:
            raise RuntimeError(f"ParoRouter: the checkpoint has no router weight {name!r} beside the expert block {experts_base!r}")
        return cls(ck.dense[name], top_k, renormalize, dtype, device)

    def __call__(self, x: torch.Tensor, ids_out: torch.Tensor, weights_out: torch.Tensor, logits_out: torch.Tensor | None = None) -> None:
        """x [T, hidden] -> ids_out [T, top_k] int32, weights_out [T, top_k] fp32 and, when given, logits_out [T, E] fp32."""
        _cabi.moe_route(x, self.weight, self.top_k, self.renormalize, ids_out, weights_out, logits_out)


class ParoExperts:
    """Experts of one MoE block.  `blocks[e] = {"gate_up": merged ParoLayerBuffers, "down": ParoLayerBuffers}` as
    `checkpoint_io.load_paro_checkpoint(...).experts[base]` returns them."""

    def __init__(self, blocks: list[dict[str, ParoLayerBuffers]], dtype: torch.dtype = torch.bfloat16, device="cuda", check_pairs: bool = False):
        self.dtype = dtype
        self.n_experts = len(blocks)
        if self.n_experts < 1:
            raise RuntimeError("ParoExperts needs at least one expert")
        # the decode kernels (decode_step) read one rotation per projection: every expert must carry the same one, and gate and up
        # the same as each other (convert.py:281-381 stores it once per block)
        for proj in ("gate_up", "down"):
            r0 = blocks[0][proj]
            for e, b in enumerate(blocks):
                r = b[proj]
                if not all(torch.equal(getattr(r, n).cpu(), getattr(r0, n).cpu()) for n in ("theta", "pairs", "channel_scales")):
                    raise RuntimeError(f"expert {e}: its {proj} rotation differs from expert 0's; an expert block shares one rotation per projection")
        gu0 = blocks[0]["gate_up"]
        if not all(torch.equal(getattr(gu0, n)[0].cpu(), getattr(gu0, n)[1].cpu()) for n in ("theta", "pairs", "channel_scales")):
            raise RuntimeError("gate and up carry different rotations; an expert block's merged gate_up shares one")
        # every expert prepacked into ONE stacked buffer per projection, [E, stride]; the per-expert kernels wrap row views of it
        self.gate_up, self.down = [], []
        self.packed, self.shapes, self.strides = {}, {}, {}
        for proj, kernels in (("gate_up", self.gate_up), ("down", self.down)):
            b0 = blocks[0][proj]
            shape = _cabi.make_shape(b0.qweight.shape[0], b0.part_sizes, b0.group_size, b0.theta.shape[-2], dtype)
            stride = (_cabi.packed_bytes(shape) + 255) // 256 * 256
            stack = torch.empty(self.n_experts, stride, dtype=torch.uint8, device=device)
            for e, b in enumerate(blocks):
                b = b[proj].to(device)
                theta, pairs, cs = b.theta, b.pairs, b.channel_scales
                if theta.dim() == 2:
                    theta, pairs, cs = theta[None], pairs[None], cs.reshape(1, -1)
                if check_pairs:
                    validate_pairs(pairs, b.group_size)
                _cabi.prepack(shape, b.qweight, b.qzeros, b.scales, pairs, theta, cs, out=stack[e])
                kernels.append(ParoLinearKernel(stack[e], shape))
            self.packed[proj], self.shapes[proj], self.strides[proj] = stack, shape, stride
        self.hidden = self.down[0].shape.out_features
        self.inter = self.down[0].shape.in_features
        self._chains: dict[tuple[int, int], tuple] = {}

    def _chain(self, e: int, m: int):
        """Two-step chain of expert e for m rows over its own fixed buffers (built once per (expert, m))."""
        key = (e, m)
        c = self._chains.get(key)
        if c is None:
            dev = self.gate_up[e].packed.device
            x = torch.empty(m, self.hidden, dtype=self.dtype, device=dev)
            y = torch.empty(m, self.hidden, dtype=self.dtype, device=dev)
            c = (ParoChain([ChainStep(self.gate_up[e], x=x), ChainStep(self.down[e], x_op="silu_mul", y=y)], m), x, y)
            self._chains[key] = c
        return c

    def expert_forward(self, e: int, x: torch.Tensor) -> torch.Tensor:
        """down_e(silu(gate_e(x)) * up_e(x)) for the rows x [m, hidden]."""
        m = x.shape[0]
        if m <= 16:
            ch, xin, y = self._chain(e, m)
            xin.copy_(x)
            ch()
            return y
        gu = self.gate_up[e](x)
        return self.down[e](torch.nn.functional.silu(gu[:, : self.inter]) * gu[:, self.inter:])

    def __call__(self, x: torch.Tensor, topk_ids: torch.Tensor, topk_weights: torch.Tensor) -> torch.Tensor:
        """x [T, hidden], topk_ids / topk_weights [T, k] -> sum_k w_k * expert_{id_k}(x) in fp32, rounded once.  A slot whose id
        lies outside [0, n_experts) contributes nothing, as in decode_step (expert parallelism marks non-local experts with -1)."""
        out = torch.zeros(x.shape[0], self.hidden, dtype=torch.float32, device=x.device)
        valid = (topk_ids >= 0) & (topk_ids < self.n_experts)
        for e in torch.unique(topk_ids[valid]).tolist():
            rows, slot = (topk_ids == e).nonzero(as_tuple=True)
            y = self.expert_forward(int(e), x[rows].contiguous())
            out.index_add_(0, rows, y.float() * topk_weights[rows, slot].float()[:, None])
        return out.to(x.dtype)

    def desc(self) -> _cabi.ParoMoEDesc:
        """The C descriptor of the stacked expert buffers (kept alive by this object)."""
        d = _cabi.ParoMoEDesc()
        d.gate_up, d.down = ctypes.pointer(self.shapes["gate_up"]), ctypes.pointer(self.shapes["down"])
        d.n_experts = self.n_experts
        d.gate_up_packed, d.gate_up_stride = self.packed["gate_up"].data_ptr(), self.strides["gate_up"]
        d.down_packed, d.down_stride = self.packed["down"].data_ptr(), self.strides["down"]
        return d

    def decode_step(self, T: int, top_k: int, router: ParoRouter | None = None) -> "ParoMoEStep":
        """The block for T <= 16 tokens with top_k slots each over fixed device buffers (see ParoMoEStep)."""
        return ParoMoEStep(self, T, top_k, router)

    def prefill_step(self, T: int, top_k: int, router: ParoRouter | None = None) -> "ParoMoEPrefill":
        """The block for any T >= 1 tokens with top_k slots each over fixed device buffers (see ParoMoEPrefill)."""
        return ParoMoEPrefill(self, T, top_k, router)


class ParoMoEStep:
    """The expert block of one decode step over fixed device buffers, like ParoChain: write the inputs into `x` [T, hidden],
    `topk_ids` [T, k] int32 and `topk_weights` [T, k] fp32 (int64 ids from torch.topk convert with a device `copy_`), call
    `step()`, read `y` [T, hidden].  `h` [T, k, 2I] holds every valid slot's gate|up output.  Construction allocates; a call
    never does, never synchronises the host, and launches two kernels on the current stream, so it can be captured in a CUDA
    graph whose replays see whatever routing the buffers hold.  With a `router`, `step()` first routes `x` on the device into
    `topk_ids` / `topk_weights` (and the router logits into `logits` [T, E] fp32), one more launch under the same rules: only
    `x` is an input then."""

    def __init__(self, experts: ParoExperts, T: int, top_k: int, router: ParoRouter | None = None):
        dev = experts.packed["gate_up"].device
        self.experts, self.T, self.top_k = experts, int(T), int(top_k)
        self._desc = experts.desc()
        nbytes = self._workspace_bytes(self._desc, self.T, self.top_k)
        dt = experts.dtype
        self.x = torch.zeros(self.T, experts.hidden, dtype=dt, device=dev)
        self.topk_ids = torch.zeros(self.T, self.top_k, dtype=torch.int32, device=dev)
        self.topk_weights = torch.zeros(self.T, self.top_k, dtype=torch.float32, device=dev)
        self.h = torch.zeros(self.T, self.top_k, 2 * experts.inter, dtype=dt, device=dev)
        self.y = torch.zeros(self.T, experts.hidden, dtype=dt, device=dev)
        self.workspace = torch.zeros(nbytes, dtype=torch.uint8, device=dev)
        self.router = router
        if router is not None:
            have = (router.n_experts, router.hidden, router.dtype, router.top_k, router.weight.device)
            want = (experts.n_experts, experts.hidden, dt, self.top_k, dev)
            if have != want:
                raise RuntimeError(f"router (n_experts, hidden, dtype, top_k, device) = {have} does not match the expert block's {want}")
            self.logits = torch.zeros(self.T, experts.n_experts, dtype=torch.float32, device=dev)

    def _route(self) -> None:
        if self.router is not None:
            self.router(self.x, self.topk_ids, self.topk_weights, self.logits)

    def step(self) -> torch.Tensor:
        self._route()
        _cabi.moe_forward(self._desc, self.x, self.topk_ids, self.topk_weights, self.h, self.y, self.workspace)
        return self.y

    __call__ = step

    _workspace_bytes = staticmethod(_cabi.moe_workspace_bytes)


class ParoMoEPrefill(ParoMoEStep):
    """The expert block for any number of tokens (prefill, or decode with more than 16 sequences), with ParoMoEStep's buffers and
    contract: the routed experts run as grouped INT4 wgmma GEMMs in six launches on the current stream (include/paro_b200.h:
    paro_moe_grouped_forward), with no host synchronisation and no allocation, so a CUDA graph of `step()` serves every routing.
    The workspace holds the routing table, the rotated operands and the per-slot expert outputs: about
    (T * k + n_experts * 128) * max(hidden, I) * 2 + T * k * hidden * 2 bytes at most."""

    _workspace_bytes = staticmethod(_cabi.moe_grouped_workspace_bytes)

    def step(self) -> torch.Tensor:
        self._route()
        _cabi.moe_grouped_forward(self._desc, self.x, self.topk_ids, self.topk_weights, self.h, self.y, self.workspace)
        return self.y

    __call__ = step
