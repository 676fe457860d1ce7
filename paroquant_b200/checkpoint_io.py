"""Checkpoint I/O for ParoQuant linears: the step either side of the hot path (SURVEY.md section 8(f), rank 1).

Writes and reads the reference's on-disk format so the kernels run on real ``z-lab/*-PARO`` checkpoints:

* export (reference ``paroquant/cli/convert.py``): optimiser state of one linear -> rotate the weight,
  round to INT4 with the learned scale / zero point (``convert.py:158-191``), AWQ-pack
  (``convert.py:149-155,194-203``), fp16 rotation buffers and ``1 / channel_scales`` (``convert.py:240-277``);
  the model directory gets ``quantization_config = {quant_method: "paroquant", bits, group_size, krot}``
  (``convert.py:450-455``).
* import (reference ``paroquant/inference/backends/transformers/quantizer.py:30-44,88-115`` and the vLLM plugin's
  ``plugin.py:123-151``): a module is quantised iff the checkpoint holds ``<module>.qweight``; everything else is left
  alone.  Merged projections (qkv, gate_up) are ONE weight spanning all partitions plus stacked rotation sets
  (``plugin.py:196-198``) -- ``merge_layers``.

The only arithmetic with a kernel in it is the weight rotation of ``export_layer`` (fp32, ``torch.ops.rotation.rotate``):
CUDA only, like the reference.  Packing / quantisation / file handling are plain torch and run anywhere.
"""
from __future__ import annotations

import json
from dataclasses import dataclass, field
from pathlib import Path

import torch

from .checkpoint import ParoLayerBuffers, pack_awq, validate_pairs

QUANT_KEYS = ("qweight", "qzeros", "scales", "theta", "pairs", "channel_scales")


# ------------------------------------------------------------------------------------------ export
def quantize_rotated(rotated: torch.Tensor, scales_flat: torch.Tensor, zp_flat: torch.Tensor, *, bits: int = 4,
                     group_size: int = 128) -> tuple[torch.Tensor, torch.Tensor, torch.Tensor]:
    """Rotated weight [N, K] fp32 + the optimiser's per-(row, group) scale / float zero point ->
    integer weight [N, K], scales [N, K/G] fp32, zero points [N, K/G] int32 (convert.py:176-191:
    z = clamp(-round(zp), 0, 2^b - 1);  q = clamp(round(w / s) + z, 0, 2^b - 1))."""
    n, k = rotated.shape
    if k % group_size:
        raise ValueError("in_features must be a multiple of group_size")
    qmax = (1 << bits) - 1
    s = scales_flat.reshape(-1, 1).to(torch.float32)
    z = torch.clamp(-torch.round(zp_flat.reshape(-1, 1).to(torch.float32)), 0, qmax)
    q = torch.clamp(torch.round(rotated.to(torch.float32).reshape(-1, group_size) / s) + z, 0, qmax)
    groups = k // group_size
    return q.to(torch.int32).reshape(n, k), s.reshape(n, groups), z.to(torch.int32).reshape(n, groups)


def to_awq_buffers(quantized: torch.Tensor, scales_2d: torch.Tensor, zeros_2d: torch.Tensor) -> dict[str, torch.Tensor]:
    """[N, K] integers + [N, K/G] scales / zeros -> the three AWQ tensors, K-major (convert.py:194-203)."""
    return {
        "qweight": pack_awq(quantized.T.contiguous()).cpu(),
        "qzeros": pack_awq(zeros_2d.T.contiguous()).cpu(),
        "scales": scales_2d.T.contiguous().to(torch.float16).cpu(),
    }


def _first(state: dict, *keys):
    for k in keys:
        if k in state:
            v = state[k]
            return v.item() if isinstance(v, torch.Tensor) else v
    raise KeyError(keys[0])


def _stacked(state: dict, key: str) -> torch.Tensor:
    """`key` as one tensor, or `key.0`, `key.1`, ... stacked (one entry per rotation; convert.py:133-146)."""
    if key in state:
        return state[key]
    parts = []
    while f"{key}.{len(parts)}" in state:
        parts.append(state[f"{key}.{len(parts)}"])
    if not parts:
        raise KeyError(key)
    return torch.stack(parts)


@torch.no_grad()
def export_layer(state: dict, device="cuda") -> tuple[dict[str, torch.Tensor], int, int, int]:
    """Optimiser state of one linear (keys of convert.py:240-252) -> checkpoint buffers, bits, group_size, krot.
    The weight is rotated in fp32 by this package's ``torch.ops.rotation.rotate`` (CUDA only)."""
    import paroquant_b200.kernels.cuda  # noqa: F401  registers the op
    dev = torch.device(device)
    if dev.type != "cuda":
        raise RuntimeError("export_layer: the weight rotation is CUDA-only (no CPU fallback)")
    weight = state["weight"].to(device=dev, dtype=torch.float32)
    bits = int(_first(state, "n_bits", "quantizer.n_bits"))
    group = int(_first(state, "group_size", "quantizer.group_size"))
    pairs = _stacked(state, "pairs_grouped").to(device=dev, dtype=torch.int16)
    theta = _stacked(state, "angles_grouped").to(device=dev, dtype=torch.float32)
    cs_opt = state["channel_scales"].to(device=dev, dtype=torch.float32).reshape(1, -1)
    validate_pairs(pairs, group)
    rotated = torch.ops.rotation.rotate(weight * cs_opt, pairs, theta, None, group)
    q, s2, z2 = quantize_rotated(rotated, state["quantizer.scale"].to(dev), state["quantizer.zero_point_float"].to(dev),
                                 bits=bits, group_size=group)
    buffers = {**to_awq_buffers(q, s2, z2), "theta": theta.to(torch.float16).cpu(), "pairs": pairs.cpu(),
               "channel_scales": (1.0 / cs_opt).to(torch.float16).cpu()}
    if state.get("bias") is not None:
        buffers["bias"] = state["bias"].to(torch.float16).cpu()
    return buffers, bits, group, int(theta.shape[0])


def export_moe(state: dict, device="cuda") -> tuple[dict[str, dict[str, torch.Tensor]], dict[str, torch.Tensor], int, int, int]:
    """Optimiser state of one fused MoE expert block (reference ``convert.py:281-381``, ``_quantize_moe``) -> per-projection expert
    stacks ``{gate_proj, up_proj, down_proj: {qweight [E, K, N/8], qzeros [E, K/G, N/8], scales [E, K/G, N]}}`` and the rotation
    buffers ALL experts share (one rotation of x before gate / up, one of the activation before down), bits, group_size, krot.
    ``gate_up_weight`` is [E, 2I, H] (gate rows first), ``down_weight`` [E, H, I]; quantiser scales / zero points are per
    (expert row, group), flattened in that order."""
    import paroquant_b200.kernels.cuda  # noqa: F401  registers the op
    dev = torch.device(device)
    if dev.type != "cuda":
        raise RuntimeError("export_moe: the weight rotation is CUDA-only (no CPU fallback)")
    bits = int(_first(state, "n_bits", "quantizer.n_bits"))
    group = int(_first(state, "group_size", "quantizer.group_size"))
    gate_up = state["gate_up_weight"].to(device=dev, dtype=torch.float32)
    down = state["down_weight"].to(device=dev, dtype=torch.float32)
    E, gu_out, gu_in = gate_up.shape
    _, d_out, d_in = down.shape
    if gu_in != d_out:
        raise ValueError(f"Unexpected MoE shapes: gate_up={tuple(gate_up.shape)} down={tuple(down.shape)}")   # convert.py:293-294
    rot, quant = {}, {}
    for tag, w, n_in in (("gate_up", gate_up, gu_in), ("down", down, d_in)):
        pairs = _stacked(state, f"{tag}_pairs_grouped").to(device=dev, dtype=torch.int16)
        theta = _stacked(state, f"{tag}_angles_grouped").to(device=dev, dtype=torch.float32)
        cs = state[f"{tag}_channel_scales"].to(device=dev, dtype=torch.float32).reshape(1, -1)
        validate_pairs(pairs, group)
        rotated = torch.ops.rotation.rotate(w.reshape(-1, n_in) * cs, pairs, theta, None, group)
        quant[tag] = quantize_rotated(rotated, state[f"{tag}_quantizer.scale"].to(dev), state[f"{tag}_quantizer.zero_point_float"].to(dev),
                                      bits=bits, group_size=group)
        rot[f"{tag}_weight_theta"] = theta.to(torch.float16).cpu()
        rot[f"{tag}_weight_pairs"] = pairs.cpu()
        rot[f"{tag}_weight_channel_scales"] = (1.0 / cs).to(torch.float16).cpu()
    return moe_expert_buffers(quant["gate_up"], quant["down"], E), rot, bits, group, int(rot["gate_up_weight_theta"].shape[0])


def moe_expert_buffers(gate_up_q, down_q, num_experts: int) -> dict[str, dict[str, torch.Tensor]]:
    """(q, scales, zeros) of the flattened expert rows -> AWQ buffers stacked per expert, gate rows / up rows split
    (convert.py:339-366).  Plain integer work: runs anywhere."""
    q, s, z = gate_up_q
    gu_out = q.shape[0] // num_experts
    half = gu_out // 2
    q, s, z = (t.reshape(num_experts, gu_out, -1) for t in (q, s, z))
    dq, ds, dz = (t.reshape(num_experts, down_q[0].shape[0] // num_experts, -1) for t in down_q)
    out: dict[str, dict[str, torch.Tensor]] = {}
    for proj, (qq, ss, zz) in (("gate_proj", (q[:, :half], s[:, :half], z[:, :half])), ("up_proj", (q[:, half:], s[:, half:], z[:, half:])),
                               ("down_proj", (dq, ds, dz))):
        per = [to_awq_buffers(qq[e], ss[e], zz[e]) for e in range(num_experts)]
        out[proj] = {k: torch.stack([b[k] for b in per]) for k in ("qweight", "qzeros", "scales")}
    return out


def moe_state_entries(base_prefix: str, proj_buffers: dict, rotation_buffers: dict) -> dict[str, torch.Tensor]:
    """Checkpoint names of one expert block (convert.py:384-406): ``<base>.<e>.<proj>.{qweight,qzeros,scales}`` per expert and
    ``<base>.{gate_up,down}_weight_{theta,pairs,channel_scales}`` once."""
    out = {}
    E = proj_buffers["gate_proj"]["qweight"].shape[0]
    for e in range(E):
        for proj in ("gate_proj", "up_proj", "down_proj"):
            for leaf in ("qweight", "qzeros", "scales"):
                out[f"{base_prefix}.{e}.{proj}.{leaf}"] = proj_buffers[proj][leaf][e]
    for name, t in rotation_buffers.items():
        out[f"{base_prefix}.{name}"] = t
    return out


def save_paro_checkpoint(out_dir, tensors: dict[str, torch.Tensor], *, bits: int = 4, group_size: int = 128, krot: int = 8,
                         base_config: dict | None = None) -> Path:
    """Write `tensors` (full state-dict names, e.g. ``model.layers.0.self_attn.q_proj.qweight``) as ``model.safetensors``
    and a ``config.json`` carrying the reference's quantization_config (convert.py:450-455)."""
    from safetensors.torch import save_file
    out = Path(out_dir)
    out.mkdir(parents=True, exist_ok=True)
    save_file({k: v.contiguous().cpu() for k, v in tensors.items()}, str(out / "model.safetensors"))
    cfg = dict(base_config or {})
    cfg["quantization_config"] = {"quant_method": "paroquant", "bits": bits, "group_size": group_size, "krot": krot}
    (out / "config.json").write_text(json.dumps(cfg, indent=2))
    return out


# ------------------------------------------------------------------------------------------ import
@dataclass
class ParoCheckpoint:
    quant_config: dict
    layers: dict[str, ParoLayerBuffers]                      # quantised modules, one partition each
    dense: dict[str, torch.Tensor] = field(default_factory=dict)   # every other tensor, untouched
    experts: dict[str, list[dict[str, ParoLayerBuffers]]] = field(default_factory=dict)
    # MoE blocks: <base> -> per expert {"gate_up": merged gate | up, "down": ...}; all experts of a block carry the SAME rotation

    @property
    def quantized_modules(self) -> set[str]:
        return set(self.layers)


def find_quantized_modules(model_dir) -> set[str]:
    """Modules with a ``.qweight`` key, from the index file when there is one (quantizer.py:30-44)."""
    from safetensors import safe_open
    d = Path(model_dir)
    index = d / "model.safetensors.index.json"
    if index.exists():
        keys = list(json.loads(index.read_text()).get("weight_map", {}))
    else:
        keys = []
        for sf in sorted(d.glob("*.safetensors")):
            with safe_open(str(sf), framework="pt") as st:
                keys.extend(st.keys())
    return {k.rsplit(".", 1)[0] for k in keys if k.endswith(".qweight")}


def load_paro_checkpoint(model_dir, *, modules_to_not_convert: list[str] | None = None, check_pairs: bool = True) -> ParoCheckpoint:
    """Read every ``*.safetensors`` of a converted model directory.  Raises on a config that is not ParoQuant INT4 with groups of 64 or 128
    (the formats the fused kernels implement) and on incomplete / inconsistent quantised modules."""
    from safetensors import safe_open
    d = Path(model_dir)
    cfg_file = d / "config.json"
    qcfg = json.loads(cfg_file.read_text()).get("quantization_config", {}) if cfg_file.exists() else {}
    if qcfg.get("quant_method") != "paroquant":
        raise ValueError(f"{d}: quantization_config.quant_method is {qcfg.get('quant_method')!r}, expected 'paroquant'")
    bits, group, krot = int(qcfg.get("bits", 4)), int(qcfg.get("group_size", 128)), int(qcfg.get("krot", 8))
    if bits != 4 or group not in (64, 128):
        raise ValueError(f"{d}: bits={bits}, group_size={group}: the kernels implement INT4 with group_size 64 or 128 only")
    quantized = find_quantized_modules(d)
    if modules_to_not_convert:
        quantized -= set(modules_to_not_convert)
    raw: dict[str, dict[str, torch.Tensor]] = {m: {} for m in quantized}
    dense: dict[str, torch.Tensor] = {}
    for sf in sorted(d.glob("*.safetensors")):
        with safe_open(str(sf), framework="pt") as st:
            for key in st.keys():
                mod, _, leaf = key.rpartition(".")
                if mod in raw and leaf in QUANT_KEYS + ("bias",):
                    raw[mod][leaf] = st.get_tensor(key)
                else:
                    dense[key] = st.get_tensor(key)
    layers = {}
    experts: dict[str, dict[int, dict[str, dict]]] = {}
    for mod in list(raw):
        # <base>.<e>.{gate,up,down}_proj without rotation buffers of its own + <base>.gate_up_weight_theta: an MoE expert
        head, _, proj = mod.rpartition(".")
        base, _, eid = head.rpartition(".")
        if proj in ("gate_proj", "up_proj", "down_proj") and eid.isdigit() and "theta" not in raw[mod] and f"{base}.gate_up_weight_theta" in dense:
            experts.setdefault(base, {}).setdefault(int(eid), {})[proj] = raw.pop(mod)
    moe: dict[str, list[dict[str, ParoLayerBuffers]]] = {}
    for base, by_id in experts.items():
        rot = {}
        for tag in ("gate_up", "down"):
            th, pr, cs = (dense.pop(f"{base}.{tag}_weight_{leaf}") for leaf in ("theta", "pairs", "channel_scales"))
            if check_pairs:
                validate_pairs(pr, group)
            rot[tag] = (th[None].contiguous(), pr[None].contiguous(), cs.reshape(1, 1, -1).contiguous())
        blocks = []
        for e in sorted(by_id):
            t = by_id[e]
            if set(t) != {"gate_proj", "up_proj", "down_proj"}:
                raise ValueError(f"{base}.{e}: expert without all of gate_proj / up_proj / down_proj")

            def part(p, tag):
                b = t[p]
                th, pr, cs = rot[tag]
                n = int(b["qweight"].shape[1]) * 8
                return ParoLayerBuffers(b["qweight"], b["qzeros"], b["scales"], th, pr, cs, [n], group, None)

            blocks.append({"gate_up": merge_layers([part("gate_proj", "gate_up"), part("up_proj", "gate_up")]), "down": part("down_proj", "down")})
        if sorted(by_id) != list(range(len(blocks))):
            raise ValueError(f"{base}: expert ids are not 0..{len(blocks) - 1}")
        moe[base] = blocks
    for mod, t in raw.items():
        missing = [k for k in QUANT_KEYS if k not in t]
        if missing:
            raise ValueError(f"{mod}: quantised module without {missing}")
        K, N = int(t["qweight"].shape[0]), int(t["qweight"].shape[1]) * 8
        shapes_ok = (tuple(t["qzeros"].shape) == (K // group, N // 8) and tuple(t["scales"].shape) == (K // group, N)
                     and tuple(t["theta"].shape) == (krot, K // 2) and tuple(t["pairs"].shape) == (krot, K)
                     and t["channel_scales"].numel() == K)
        if not shapes_ok:
            raise ValueError(f"{mod}: buffer shapes do not match in_features={K}, out_features={N}, krot={krot}, group_size={group}")
        if check_pairs:
            validate_pairs(t["pairs"], group)
        layers[mod] = ParoLayerBuffers(t["qweight"], t["qzeros"], t["scales"], t["theta"][None].contiguous(), t["pairs"][None].contiguous(),
                                       t["channel_scales"].reshape(1, 1, K).contiguous(), [N], group, t.get("bias"))
    return ParoCheckpoint({"quant_method": "paroquant", "bits": bits, "group_size": group, "krot": krot}, layers, dense, moe)


def merge_layers(parts: list[ParoLayerBuffers]) -> ParoLayerBuffers:
    """q/k/v (or gate/up) -> one merged projection: weights concatenated along N, rotation sets stacked (plugin.py:196-198).
    All partitions must share in_features, group size and krot; biases must be all present or all absent."""
    if not parts:
        raise ValueError("merge_layers: nothing to merge")
    K, g, r = parts[0].in_features, parts[0].group_size, parts[0].krot
    for p in parts:
        if p.in_features != K or p.group_size != g or p.krot != r:
            raise ValueError("merge_layers: partitions disagree on in_features / group_size / krot")
    has_bias = [p.bias is not None for p in parts]
    if any(has_bias) and not all(has_bias):
        raise ValueError("merge_layers: some partitions have a bias and some do not")
    cat = lambda name: torch.cat([getattr(p, name) for p in parts], dim=-1 if name != "bias" else 0)
    return ParoLayerBuffers(cat("qweight"), cat("qzeros"), cat("scales"), torch.cat([p.theta for p in parts], 0),
                            torch.cat([p.pairs for p in parts], 0), torch.cat([p.channel_scales for p in parts], 0),
                            [n for p in parts for n in p.part_sizes], g, cat("bias") if all(has_bias) else None)


DEFAULT_MERGES = {"qkv_proj": ("q_proj", "k_proj", "v_proj"), "gate_up_proj": ("gate_proj", "up_proj")}


def merged_view(ckpt: ParoCheckpoint, merges: dict[str, tuple[str, ...]] = DEFAULT_MERGES) -> dict[str, ParoLayerBuffers]:
    """The layers as a serving engine wants them: siblings listed in `merges` fused under the merged name (vLLM's
    stacked-parameter convention), everything else as is."""
    out: dict[str, ParoLayerBuffers] = {}
    done: set[str] = set()
    for mod in sorted(ckpt.layers):
        if mod in done:
            continue
        parent, _, leaf = mod.rpartition(".")
        target = next((m for m, members in merges.items() if leaf in members), None)
        if target is None:
            out[mod] = ckpt.layers[mod]
            continue
        names = [f"{parent}.{x}" if parent else x for x in merges[target]]
        if not all(n in ckpt.layers for n in names):
            out[mod] = ckpt.layers[mod]      # incomplete family: leave the members alone
            continue
        out[f"{parent}.{target}" if parent else target] = merge_layers([ckpt.layers[n] for n in names])
        done.update(names)
    return out
