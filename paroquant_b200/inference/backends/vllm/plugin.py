"""vLLM quantisation plugin: `ParoQuantConfig` / `ParoQuantLinearMethod` on sm_90a.

Drop-in for /root/reference/paroquant/inference/backends/vllm/plugin.py (same registration name
"paroquant", same parameter names / shapes / loaders, same TP input-dim sharding of the rotation
parameters), with a different engine underneath:

  reference                                   here
  ---------                                   ----
  subclass of AWQMarlinLinearMethod           plain LinearMethodBase, no Marlin anywhere
  AWQ -> Marlin repack per partition          one prepack into the streaming layout of csrc/
  apply(): n rotate + n Marlin + cat (+bias)  apply(): ONE fused launch for all partitions
  theta / scales cast to x.dtype per call     cast once at prepack
  min capability 75                            90 (sm_90a only, no fallback path)
"""
from __future__ import annotations

from typing import TYPE_CHECKING, Any

import torch
from torch.nn import Parameter
from vllm.logger import init_logger
from vllm.model_executor.layers.linear import LinearBase, LinearMethodBase, UnquantizedLinearMethod
from vllm.model_executor.layers.quantization import register_quantization_config
from vllm.model_executor.layers.quantization.base_config import QuantizationConfig
from vllm.model_executor.layers.quantization.utils.quant_utils import is_layer_skipped
from vllm.model_executor.parameter import GroupQuantScaleParameter, PackedvLLMParameter

import paroquant_b200.kernels.cuda  # noqa: F401  (registers torch.ops.rotation.rotate)
from paroquant_b200.linear import ParoLinearKernel

if TYPE_CHECKING:
    from vllm.model_executor.layers.quantization import QuantizationMethods

logger = init_logger(__name__)

_QKV_SLOT = {"q": 0, "k": 1, "v": 2}
_SUPPORTED_BITS = (4,)
_TILE_N = 16  # output partitions must be multiples of the fused kernel's column tile


def _maybe_shard_input(target: torch.Tensor, loaded_weight: torch.Tensor) -> torch.Tensor:
    """Row-parallel layers allocate rotation params for K / tp input channels while the checkpoint
    holds all K: take this rank's contiguous slice (rotations are 128-channel local, so any
    shard that is a multiple of 128 is self-contained)."""
    have, want = loaded_weight.shape[-1], target.shape[-1]
    if have == want:
        return loaded_weight
    if have % want:
        raise ValueError(f"ParoQuant rotation loader: incompatible shapes target={tuple(target.shape)} "
                         f"loaded={tuple(loaded_weight.shape)}")
    from vllm.distributed import get_tensor_model_parallel_rank

    return loaded_weight.narrow(-1, get_tensor_model_parallel_rank() * want, want)


def _rotation_weight_loader(param: Parameter, loaded_weight: torch.Tensor,
                            loaded_shard_id: int | str | tuple | None = None) -> None:
    """Route a per-projection rotation tensor into its slot of the stacked [n_parts, ...] param.
    shard id: None (single projection), "q"/"k"/"v", an int (gate/up), or a tuple of ints."""
    if loaded_shard_id is None:
        dst = param.data[0] if param.data.dim() > loaded_weight.dim() else param.data
        dst.copy_(_maybe_shard_input(dst, loaded_weight))
        return
    slots = loaded_shard_id if isinstance(loaded_shard_id, tuple) else (loaded_shard_id,)
    for slot in slots:
        dst = param.data[_QKV_SLOT.get(slot, slot)]
        dst.copy_(_maybe_shard_input(dst, loaded_weight))


@register_quantization_config("paroquant")
class ParoQuantConfig(QuantizationConfig):
    def __init__(self, bits: int, group_size: int, krot: int, zero_point: bool) -> None:
        super().__init__()
        if bits not in _SUPPORTED_BITS:
            raise ValueError(f"Unsupported bits={bits}. Supported: {list(_SUPPORTED_BITS)}")
        self.bits, self.group_size, self.krot, self.zero_point = bits, group_size, krot, zero_point
        self.pack_factor = 32 // bits
        self.modules_to_not_convert: list[str] | None = None  # discovered from the checkpoint

    def __repr__(self) -> str:
        return (f"ParoQuantConfig(bits={self.bits}, group_size={self.group_size}, krot={self.krot}, "
                f"zero_point={self.zero_point})")

    @classmethod
    def get_name(cls) -> "QuantizationMethods":
        return "paroquant"

    @classmethod
    def get_supported_act_dtypes(cls) -> list[torch.dtype]:
        return [torch.half, torch.bfloat16]

    @classmethod
    def get_min_capability(cls) -> int:
        return 90

    @classmethod
    def get_config_filenames(cls) -> list[str]:
        return ["config.json"]

    @classmethod
    def from_config(cls, config: dict[str, Any]) -> "ParoQuantConfig":
        get = cls.get_from_keys_or
        return cls(bits=get(config, ["bits"], 4), group_size=get(config, ["group_size"], 128),
                   krot=get(config, ["krot"], 8), zero_point=get(config, ["zero_point"], True))

    def maybe_update_config(self, model_name: str, revision: str | None = None):
        """Layers whose checkpoint entry is a plain fp weight (no integer tensors) stay unquantised."""
        if self.modules_to_not_convert:
            return
        from safetensors.torch import _TYPES as sf_types
        from vllm.transformers_utils.config import get_safetensors_params_metadata

        floats = {torch.float16, torch.bfloat16, torch.float32}
        meta = get_safetensors_params_metadata(model_name, revision=revision)
        with_weight, with_ints = set(), set()
        for key, info in meta.items():
            module, _, leaf = key.rpartition(".")
            if leaf == "weight":
                with_weight.add(module)
            if info.get("dtype") and sf_types[info["dtype"]] not in floats:
                with_ints.add(module)

        def suffix(name: str) -> str:  # "…layers.N.x" so vLLM's substring match is nesting-agnostic
            name = name.removeprefix("model.")
            at = name.find("layers.")
            return name[at:] if at >= 0 else name

        self.modules_to_not_convert = sorted(suffix(m) for m in with_weight - with_ints)

    def get_quant_method(self, layer: torch.nn.Module, prefix: str) -> LinearMethodBase | None:
        if not isinstance(layer, LinearBase):
            return None
        if is_layer_skipped(prefix, self.modules_to_not_convert or [], self.packed_modules_mapping,
                            skip_with_substr=True):
            return UnquantizedLinearMethod()
        return ParoQuantLinearMethod(self)


class ParoQuantLinearMethod(LinearMethodBase):
    """Per-projection pairwise rotation + INT4 GEMM, fused."""

    def __init__(self, quant_config: ParoQuantConfig) -> None:
        self.quant_config = quant_config

    def create_weights(self, layer: torch.nn.Module, input_size_per_partition: int,
                       output_partition_sizes: list[int], input_size: int, output_size: int,
                       params_dtype: torch.dtype, **extra_weight_attrs) -> None:
        cfg = self.quant_config
        if input_size_per_partition % cfg.group_size:
            raise ValueError("The input size is not aligned with the quantized weight shape. "
                             "This can be caused by too large tensor parallel size.")
        if any(n % _TILE_N for n in output_partition_sizes):
            raise ValueError(f"ParoQuant: output partitions must be multiples of {_TILE_N}, got {output_partition_sizes}")
        n_out = sum(output_partition_sizes)
        loader = extra_weight_attrs.get("weight_loader")
        groups = input_size_per_partition // cfg.group_size
        packed_kw = dict(input_dim=0, output_dim=1, packed_dim=1, packed_factor=cfg.pack_factor, weight_loader=loader)
        layer.register_parameter("qweight", PackedvLLMParameter(
            data=torch.empty(input_size_per_partition, n_out // cfg.pack_factor, dtype=torch.int32), **packed_kw))
        layer.register_parameter("qzeros", PackedvLLMParameter(
            data=torch.empty(groups, n_out // cfg.pack_factor, dtype=torch.int32), **packed_kw))
        layer.register_parameter("scales", GroupQuantScaleParameter(
            data=torch.empty(groups, n_out, dtype=params_dtype), input_dim=0, output_dim=1, weight_loader=loader))

        n_parts, K = len(output_partition_sizes), input_size_per_partition
        for name, shape, dtype, fill in (("theta", (n_parts, cfg.krot, K // 2), torch.float16, 0.0),
                                         ("pairs", (n_parts, cfg.krot, K), torch.int16, 0),
                                         ("channel_scales", (n_parts, 1, K), torch.float16, 1.0)):
            p = Parameter(torch.full(shape, fill, dtype=dtype), requires_grad=False)
            p.weight_loader = _rotation_weight_loader
            layer.register_parameter(name, p)
        layer.num_partitions = n_parts
        layer.output_partition_sizes = list(output_partition_sizes)
        layer.input_size_per_partition = input_size_per_partition
        layer.params_dtype = params_dtype

    def process_weights_after_loading(self, layer: torch.nn.Module) -> None:
        layer.paro_kernel = ParoLinearKernel.from_tensors(
            layer.qweight.data, layer.qzeros.data, layer.scales.data, layer.theta.data, layer.pairs.data,
            layer.channel_scales.data, layer.output_partition_sizes, group_size=self.quant_config.group_size,
            dtype=layer.params_dtype)
        # same post-load attribute names as the reference (plugin.py:276-279)
        layer.rot_theta, layer.rot_pairs, layer.rot_scales = layer.theta.data, layer.pairs.data, layer.channel_scales.data
        for name in ("qweight", "qzeros", "scales", "theta", "pairs", "channel_scales"):
            delattr(layer, name)

    def apply(self, layer: torch.nn.Module, x: torch.Tensor, bias: torch.Tensor | None = None) -> torch.Tensor:
        return layer.paro_kernel(x, bias)
