"""ctypes binding of libparo_b200.so (include/paro_b200.h) for PyTorch tensors.

PyTorch is plumbing here: it owns device memory and streams; every byte of arithmetic happens
inside the C-ABI library.  There is NO fallback: if the library is missing or a kernel fails the
call raises (the reference raises RuntimeError from TORCH_CHECK the same way).
"""
from __future__ import annotations

import ctypes
import os
from pathlib import Path

import torch

_LIB_PATH = Path(os.environ.get("PARO_B200_LIB") or Path(__file__).resolve().parent / "lib" / "libparo_b200.so")   # (override: A/B runs of kernel variants)
PARO_MAX_PARTS = 8
F32, F16, BF16 = 0, 1, 2
_DTYPE_CODE = {torch.float32: F32, torch.float16: F16, torch.bfloat16: BF16}
_CODE_DTYPE = {v: k for k, v in _DTYPE_CODE.items()}


class ParoLinearShape(ctypes.Structure):
    """struct paro_linear_shape"""

    _fields_ = [
        ("in_features", ctypes.c_int32), ("out_features", ctypes.c_int32), ("group_size", ctypes.c_int32),
        ("krot", ctypes.c_int32), ("n_parts", ctypes.c_int32), ("part_sizes", ctypes.c_int32 * PARO_MAX_PARTS),
        ("dtype", ctypes.c_int32),
    ]

    def key(self) -> tuple:
        return (self.in_features, self.out_features, self.group_size, self.krot, self.dtype,
                tuple(self.part_sizes[: self.n_parts]))


class ParoTpInfo(ctypes.Structure):
    """struct paro_tp_info"""

    _fields_ = [("world", ctypes.c_int32), ("rank", ctypes.c_int32), ("peer_slots", ctypes.c_void_p * 8)]


class ParoChainStep(ctypes.Structure):
    """struct paro_chain_step"""

    _fields_ = [
        ("shape", ctypes.POINTER(ParoLinearShape)), ("packed", ctypes.c_void_p), ("bias", ctypes.c_void_p),
        ("x", ctypes.c_void_p), ("y", ctypes.c_void_p), ("x_op", ctypes.c_int32), ("epilogue", ctypes.c_int32),
        ("residual_in", ctypes.c_void_p), ("residual_out", ctypes.c_void_p), ("norm_weight", ctypes.c_void_p),
        ("eps", ctypes.c_float), ("tp", ctypes.POINTER(ParoTpInfo)),
    ]


class ParoMoEDesc(ctypes.Structure):
    """struct paro_moe_desc"""

    _fields_ = [
        ("gate_up", ctypes.POINTER(ParoLinearShape)), ("down", ctypes.POINTER(ParoLinearShape)), ("n_experts", ctypes.c_int32),
        ("gate_up_packed", ctypes.c_void_p), ("gate_up_stride", ctypes.c_size_t), ("down_packed", ctypes.c_void_p),
        ("down_stride", ctypes.c_size_t),
    ]


ABI_VERSION = 5
CHAIN_MAX_STEPS = 6
XOP_NONE, XOP_SILU_MUL, XOP_RMSNORM = 0, 1, 2
EPI_STORE, EPI_ADD_RESIDUAL = 0, 1

_lib = None


def lib() -> ctypes.CDLL:
    """Load the library once; raise loudly when it has not been built."""
    global _lib
    if _lib is None:
        if not _LIB_PATH.exists():
            raise ImportError(
                f"{_LIB_PATH} is missing: build it with `python -m paroquant_b200.build` "
                "(paroquant_b200 has no CPU or PyTorch fallback for its kernels)")
        L = ctypes.CDLL(str(_LIB_PATH))
        vp, i32, i64, sz = ctypes.c_void_p, ctypes.c_int32, ctypes.c_int64, ctypes.c_size_t
        shp = ctypes.POINTER(ParoLinearShape)
        L.paro_abi_version.restype = ctypes.c_int
        L.paro_last_error.restype = ctypes.c_char_p
        L.paro_last_launch_count.restype = ctypes.c_int
        L.paro_rotate.restype = ctypes.c_int
        L.paro_rotate.argtypes = [vp, vp, vp, vp, i32, vp, i32, i64, i32, i32, i32, i32, vp]
        L.paro_rotate_backward.restype = ctypes.c_int
        L.paro_rotate_backward.argtypes = [vp, vp, vp, vp, vp, i32, vp, i32, vp, vp, vp, i64, i32, i32, i32, i32, i32, vp]
        L.paro_debug_rotate_backward_plan.restype = ctypes.c_int
        L.paro_debug_rotate_backward_plan.argtypes = [i64, i32, i32, i32, i32, i32, i32, ctypes.POINTER(ctypes.c_int64)]
        L.paro_packed_bytes.restype = sz
        L.paro_packed_bytes.argtypes = [shp]
        L.paro_prepack.restype = ctypes.c_int
        L.paro_prepack.argtypes = [shp, vp, vp, vp, i32, vp, vp, i32, vp, i32, vp, vp]
        L.paro_workspace_bytes.restype = sz
        L.paro_workspace_bytes.argtypes = [shp, i64]
        L.paro_linear_forward.restype = ctypes.c_int
        L.paro_linear_forward.argtypes = [shp, vp, vp, i64, vp, vp, vp, sz, vp]
        L.paro_unpack_dense.restype = ctypes.c_int
        L.paro_unpack_dense.argtypes = [shp, vp, vp, vp]
        L.paro_debug_silu_mul.restype = ctypes.c_int
        L.paro_debug_silu_mul.argtypes = [i32, vp, vp, i64, i32, vp]
        L.paro_debug_trace.restype = ctypes.c_int
        L.paro_debug_trace.argtypes = [vp, i32]
        L.paro_chain_workspace_bytes.restype = sz
        L.paro_chain_workspace_bytes.argtypes = [ctypes.POINTER(ParoChainStep), i32, i64]
        L.paro_chain_forward.restype = ctypes.c_int
        L.paro_chain_forward.argtypes = [ctypes.POINTER(ParoChainStep), i32, i64, vp, sz, vp]
        L.paro_prefill_chain_workspace_bytes.restype = sz
        L.paro_prefill_chain_workspace_bytes.argtypes = [ctypes.POINTER(ParoChainStep), i32, i64]
        L.paro_prefill_chain_forward.restype = ctypes.c_int
        L.paro_prefill_chain_forward.argtypes = [ctypes.POINTER(ParoChainStep), i32, i64, vp, sz, vp]
        L.paro_tp_slot_bytes.restype = sz
        L.paro_tp_slot_bytes.argtypes = [shp, i64, i32]
        L.paro_debug_stream_plan.restype = ctypes.c_int
        L.paro_debug_stream_plan.argtypes = [shp, i64, i32, i32, ctypes.POINTER(ctypes.c_int32)]
        L.paro_debug_gemm_plan.restype = ctypes.c_int
        L.paro_debug_gemm_plan.argtypes = [shp, i64, i32, ctypes.POINTER(ctypes.c_int32)]
        L.paro_debug_stream_trace.restype = ctypes.c_int
        L.paro_debug_stream_trace.argtypes = [vp, i32]
        moe = ctypes.POINTER(ParoMoEDesc)
        L.paro_moe_workspace_bytes.restype = sz
        L.paro_moe_workspace_bytes.argtypes = [moe, i64, i32]
        L.paro_moe_forward.restype = ctypes.c_int
        L.paro_moe_forward.argtypes = [moe, vp, vp, vp, i64, i32, vp, vp, vp, sz, vp]
        L.paro_debug_moe_plan.restype = ctypes.c_int
        L.paro_debug_moe_plan.argtypes = [moe, i64, i32, i32, ctypes.POINTER(ctypes.c_int32)]
        L.paro_moe_grouped_workspace_bytes.restype = sz
        L.paro_moe_grouped_workspace_bytes.argtypes = [moe, i64, i32]
        L.paro_moe_grouped_forward.restype = ctypes.c_int
        L.paro_moe_grouped_forward.argtypes = [moe, vp, vp, vp, i64, i32, vp, vp, vp, sz, vp]
        L.paro_debug_moe_grouped_plan.restype = ctypes.c_int
        L.paro_debug_moe_grouped_plan.argtypes = [moe, i64, i32, i32, ctypes.POINTER(ctypes.c_int32)]
        L.paro_moe_route.restype = ctypes.c_int
        L.paro_moe_route.argtypes = [vp, vp, i32, i64, i32, i32, i32, i32, vp, vp, vp, vp]
        L.paro_debug_moe_route_plan.restype = ctypes.c_int
        L.paro_debug_moe_route_plan.argtypes = [i64, i32, i32, i32, i32, ctypes.POINTER(ctypes.c_int32)]
        if L.paro_abi_version() != ABI_VERSION:
            raise ImportError("libparo_b200.so ABI version mismatch")
        _lib = L
    return _lib


EXPORTED_SYMBOLS = (
    "paro_abi_version", "paro_last_error", "paro_last_launch_count", "paro_rotate", "paro_rotate_backward", "paro_packed_bytes",
    "paro_prepack", "paro_workspace_bytes", "paro_linear_forward", "paro_unpack_dense", "paro_debug_trace", "paro_debug_decode_plan",
    "paro_chain_workspace_bytes", "paro_chain_forward", "paro_debug_stream_plan", "paro_debug_stream_trace", "paro_tp_slot_bytes",
    "paro_debug_gemm_plan", "paro_moe_workspace_bytes", "paro_moe_forward", "paro_debug_moe_plan", "paro_debug_silu_mul",
    "paro_moe_grouped_workspace_bytes", "paro_moe_grouped_forward", "paro_debug_moe_grouped_plan",
    "paro_prefill_chain_workspace_bytes", "paro_prefill_chain_forward", "paro_moe_route", "paro_debug_moe_route_plan",
    "paro_debug_rotate_backward_plan",
)


def _check(rc: int, what: str) -> None:
    if rc != 0:
        raise RuntimeError(f"{what}: {lib().paro_last_error().decode()} (code {rc})")


def dtype_code(dt: torch.dtype) -> int:
    try:
        return _DTYPE_CODE[dt]
    except KeyError:
        raise RuntimeError(f"rotate supports Float, Half, and BFloat16, got {dt}") from None


def _stream(dev: torch.device) -> int:
    return torch.cuda.current_stream(dev).cuda_stream


def _need_cuda(*tensors) -> torch.device:
    dev = None
    for t in tensors:
        if t is None:
            continue
        if not t.is_cuda:
            raise RuntimeError("paroquant_b200 kernels are CUDA-only (sm_90a); got a CPU tensor")
        if dev is not None and t.device != dev:
            raise RuntimeError("all tensors must be on the same CUDA device")
        dev = t.device
    return dev


def make_shape(in_features: int, part_sizes, group_size: int, krot: int, dtype: torch.dtype) -> ParoLinearShape:
    parts = [int(p) for p in part_sizes]
    if not 1 <= len(parts) <= PARO_MAX_PARTS:
        raise RuntimeError(f"1..{PARO_MAX_PARTS} output partitions supported, got {len(parts)}")
    s = ParoLinearShape()
    s.in_features, s.out_features, s.group_size, s.krot = int(in_features), sum(parts), int(group_size), int(krot)
    s.n_parts = len(parts)
    for i, p in enumerate(parts):
        s.part_sizes[i] = p
    s.dtype = dtype_code(dtype)
    return s


def rotate(x: torch.Tensor, idx_ij: torch.Tensor, theta: torch.Tensor, scales: torch.Tensor | None = None,
           group_size: int = 128) -> torch.Tensor:
    """torch.ops.rotation.rotate -- same contract as rotation.cu:111-124."""
    dev = _need_cuda(x, idx_ij, theta, scales)
    if theta.size(0) != idx_ij.size(0):
        raise RuntimeError("theta.size(0) must equal idx_ij.size(0)")
    if idx_ij.dtype != torch.int16:
        raise RuntimeError("idx_ij must be int16")
    x = x.contiguous()
    idx_ij, theta = idx_ij.contiguous(), theta.contiguous()
    has_scale = scales is not None and scales.numel() > 0
    if has_scale:
        scales = scales.contiguous()
    out = torch.empty_like(x)
    K = x.size(-1)
    M = x.numel() // K if K else 0
    if M == 0:
        dtype_code(x.dtype)
        return out
    with torch.cuda.device(dev):
        rc = lib().paro_rotate(x.data_ptr(), out.data_ptr(), idx_ij.data_ptr(), theta.data_ptr(), dtype_code(theta.dtype),
                               scales.data_ptr() if has_scale else None, dtype_code(scales.dtype) if has_scale else 0,
                               M, K, idx_ij.size(0), group_size, dtype_code(x.dtype), _stream(dev))
    _check(rc, "rotate")
    return out


def rotate_backward(y: torch.Tensor, grad_out: torch.Tensor, x: torch.Tensor, idx_ij: torch.Tensor, theta: torch.Tensor,
                    scales: torch.Tensor | None = None, group_size: int = 128, reference_formula: bool = False):
    """Backward of `rotate` in one launch: (grad_x, grad_theta fp32 [krot, K/2], grad_scale fp32 [K] | None).
    Replaces the per-rotation Python walk of kernels/cuda/autograd.py:20-61.  reference_formula: grad_theta takes the value of the
    reference's expression (cos * gradient - sin * sum_rows(g . t)) instead of the gradient."""
    dev = _need_cuda(y, grad_out, x, idx_ij, theta, scales)
    if idx_ij.dtype != torch.int16:
        raise RuntimeError("idx_ij must be int16")
    if grad_out.dtype != y.dtype or x.dtype != y.dtype:
        raise RuntimeError("rotate_backward: y, grad_out and x must share a dtype")
    y, grad_out, x = y.contiguous(), grad_out.contiguous(), x.contiguous()
    idx_ij, theta = idx_ij.contiguous(), theta.contiguous()
    has_scale = scales is not None and scales.numel() > 0
    if has_scale:
        scales = scales.contiguous()
    K = y.size(-1)
    M = y.numel() // K if K else 0
    grad_x = torch.empty_like(y)
    grad_theta = torch.zeros(idx_ij.size(0), K // 2, dtype=torch.float32, device=dev)
    grad_scale = torch.zeros(K, dtype=torch.float32, device=dev) if has_scale else None
    if M == 0:
        dtype_code(y.dtype)
        return grad_x, grad_theta, grad_scale
    with torch.cuda.device(dev):
        rc = lib().paro_rotate_backward(y.data_ptr(), grad_out.data_ptr(), x.data_ptr(), idx_ij.data_ptr(), theta.data_ptr(),
                                        dtype_code(theta.dtype), scales.data_ptr() if has_scale else None,
                                        dtype_code(scales.dtype) if has_scale else 0, grad_x.data_ptr(), grad_theta.data_ptr(),
                                        grad_scale.data_ptr() if has_scale else None, M, K, idx_ij.size(0), group_size,
                                        dtype_code(y.dtype), 1 if reference_formula else 0, _stream(dev))
    _check(rc, "rotate_backward")
    return grad_x, grad_theta, grad_scale


ROTATE_BACKWARD_PLAN_FIELDS = ("dyn_smem", "ctas_per_sm", "splits", "row_blocks", "max_blocks_per_warp", "min_blocks_per_warp", "grid")


def debug_rotate_backward_plan(M: int, K: int, krot: int, group_size: int, dtype: torch.dtype, reference_formula: bool = False,
                               sms: int | None = None) -> dict:
    """paro_debug_rotate_backward_plan: the launch plan `rotate_backward` uses, as a dict of ROTATE_BACKWARD_PLAN_FIELDS (host
    only; sms defaults to cuda:0's SM count)."""
    if sms is None:
        sms = torch.cuda.get_device_properties(0).multi_processor_count
    out = (ctypes.c_int64 * len(ROTATE_BACKWARD_PLAN_FIELDS))()
    _check(lib().paro_debug_rotate_backward_plan(M, K, krot, group_size, dtype_code(dtype), 1 if reference_formula else 0, sms, out),
           "debug_rotate_backward_plan")
    return dict(zip(ROTATE_BACKWARD_PLAN_FIELDS, out))


def packed_bytes(shape: ParoLinearShape) -> int:
    n = lib().paro_packed_bytes(ctypes.byref(shape))
    if n == 0:
        raise RuntimeError(f"prepack: {lib().paro_last_error().decode()}")
    return n


def prepack(shape: ParoLinearShape, qweight, qzeros, scales, pairs, theta, channel_scales, out: torch.Tensor | None = None) -> torch.Tensor:
    """AWQ + rotation buffers -> one uint8 tensor in the streaming layout (csrc/paro_layout.h).  `out`: a caller-owned
    uint8 buffer of at least packed_bytes(shape) bytes, 128-byte aligned (e.g. one expert's row of a stacked buffer)."""
    dev = _need_cuda(qweight, qzeros, scales, pairs, theta, channel_scales)
    K, N, P, R = shape.in_features, shape.out_features, shape.n_parts, shape.krot
    G = shape.group_size
    exp = {"qweight": ((K, N // 8), torch.int32, qweight), "qzeros": ((K // G, N // 8), torch.int32, qzeros),
           "scales": ((K // G, N), None, scales), "pairs": ((P, R, K), torch.int16, pairs),
           "theta": ((P, R, K // 2), None, theta), "channel_scales": ((P, K), None, channel_scales.reshape(P, -1))}
    for name, (shp, dt, t) in exp.items():
        if tuple(t.shape) != shp or (dt is not None and t.dtype != dt):
            raise RuntimeError(f"prepack: {name} must be {shp} {dt or 'float'}, got {tuple(t.shape)} {t.dtype}")
    qweight, qzeros, scales, pairs, theta = (t.contiguous() for t in (qweight, qzeros, scales, pairs, theta))
    cs = channel_scales.reshape(P, -1).contiguous()
    if out is None:
        packed = torch.empty(packed_bytes(shape), dtype=torch.uint8, device=dev)
    else:
        if out.device != dev or out.dtype != torch.uint8 or not out.is_contiguous() or out.numel() < packed_bytes(shape):
            raise RuntimeError(f"prepack: out must be a contiguous uint8 tensor of >= {packed_bytes(shape)} bytes on {dev}")
        packed = out
    with torch.cuda.device(dev):
        rc = lib().paro_prepack(ctypes.byref(shape), qweight.data_ptr(), qzeros.data_ptr(), scales.data_ptr(),
                                dtype_code(scales.dtype), pairs.data_ptr(), theta.data_ptr(), dtype_code(theta.dtype),
                                cs.data_ptr(), dtype_code(cs.dtype), packed.data_ptr(), _stream(dev))
    _check(rc, "prepack")
    return packed


def workspace_bytes(shape: ParoLinearShape, max_m: int) -> int:
    return lib().paro_workspace_bytes(ctypes.byref(shape), max_m)


def new_workspace(shape: ParoLinearShape, max_m: int, device) -> torch.Tensor:
    """Zero-filled scratch for paro_linear_forward (the kernels leave it zeroed)."""
    return torch.zeros(max(workspace_bytes(shape, max_m), 256), dtype=torch.uint8, device=device)


def linear_forward(shape: ParoLinearShape, packed: torch.Tensor, x: torch.Tensor, bias: torch.Tensor | None,
                   workspace: torch.Tensor, out: torch.Tensor | None = None) -> torch.Tensor:
    dev = _need_cuda(packed, x, bias, workspace)
    if dtype_code(x.dtype) != shape.dtype:
        raise RuntimeError(f"linear_forward: layer was prepacked for {_CODE_DTYPE[shape.dtype]}, got {x.dtype}")
    if x.size(-1) != shape.in_features:
        raise RuntimeError(f"linear_forward: last dim {x.size(-1)} != in_features {shape.in_features}")
    x = x.contiguous()
    M = x.numel() // shape.in_features
    if out is None:
        out = torch.empty(*x.shape[:-1], shape.out_features, dtype=x.dtype, device=dev)
    if bias is not None and (bias.dtype != x.dtype or not bias.is_contiguous()):
        raise RuntimeError(f"linear_forward: bias must be a contiguous {x.dtype} tensor (ParoLinearKernel casts it once)")
    if M == 0:
        return out
    need = workspace_bytes(shape, M)
    if workspace.numel() < need:
        raise RuntimeError(f"linear_forward: workspace has {workspace.numel()} bytes, {need} needed for M={M}")
    with torch.cuda.device(dev):
        rc = lib().paro_linear_forward(ctypes.byref(shape), packed.data_ptr(), x.data_ptr(), M,
                                       bias.data_ptr() if bias is not None else None, out.data_ptr(),
                                       workspace.data_ptr(), workspace.numel(), _stream(dev))
    _check(rc, "linear_forward")
    return out


def unpack_dense(shape: ParoLinearShape, packed: torch.Tensor) -> torch.Tensor:
    dev = _need_cuda(packed)
    W = torch.empty(shape.in_features, shape.out_features, dtype=_CODE_DTYPE[shape.dtype], device=dev)
    with torch.cuda.device(dev):
        rc = lib().paro_unpack_dense(ctypes.byref(shape), packed.data_ptr(), W.data_ptr(), _stream(dev))
    _check(rc, "unpack_dense")
    return W


def debug_silu_mul(gate_up: torch.Tensor) -> torch.Tensor:
    """gate_up [..., 2I] (gate | up) -> [..., I]: the library's SiLU * up, bit-identical to the operand the MoE down launch
    and a chain's silu_mul step rotate (tests)."""
    if gate_up.dtype not in (torch.float16, torch.bfloat16):
        raise RuntimeError(f"debug_silu_mul: gate_up must be float16 or bfloat16, got {gate_up.dtype}")
    if gate_up.dim() < 1 or gate_up.size(-1) < 4 or gate_up.size(-1) % 4:
        raise RuntimeError(f"debug_silu_mul: the last dimension must be 2I with I even and >= 2, got {tuple(gate_up.shape)}")
    dev = _need_cuda(gate_up)
    gate_up = gate_up.contiguous()
    I = gate_up.size(-1) // 2
    act = torch.empty(*gate_up.shape[:-1], I, dtype=gate_up.dtype, device=dev)
    with torch.cuda.device(dev):
        rc = lib().paro_debug_silu_mul(dtype_code(gate_up.dtype), gate_up.data_ptr(), act.data_ptr(), act.numel() // max(I, 1), I,
                                       _stream(dev))
    _check(rc, "debug_silu_mul")
    return act


def last_launch_count() -> int:
    return lib().paro_last_launch_count()


def chain_workspace_bytes(steps, n: int, M: int) -> int:
    nb = lib().paro_chain_workspace_bytes(steps, n, M)
    if nb == 0:
        raise RuntimeError(f"chain: {lib().paro_last_error().decode()}")
    return nb


def chain_forward(steps, n: int, M: int, workspace: torch.Tensor) -> None:
    """paro_chain_forward on the current stream of the workspace's device (steps: ctypes array of ParoChainStep)."""
    dev = workspace.device
    with torch.cuda.device(dev):
        rc = lib().paro_chain_forward(steps, n, M, workspace.data_ptr(), workspace.numel(), _stream(dev))
    _check(rc, "chain_forward")


def prefill_chain_workspace_bytes(steps, n: int, M: int) -> int:
    nb = lib().paro_prefill_chain_workspace_bytes(steps, n, M)
    if nb == 0:
        raise RuntimeError(f"prefill_chain: {lib().paro_last_error().decode()}")
    return nb


def prefill_chain_forward(steps, n: int, M: int, workspace: torch.Tensor) -> None:
    """paro_prefill_chain_forward on the current stream of the workspace's device (steps: ctypes array of ParoChainStep)."""
    dev = workspace.device
    with torch.cuda.device(dev):
        rc = lib().paro_prefill_chain_forward(steps, n, M, workspace.data_ptr(), workspace.numel(), _stream(dev))
    _check(rc, "prefill_chain_forward")


def moe_workspace_bytes(desc: ParoMoEDesc, T: int, top_k: int) -> int:
    nb = lib().paro_moe_workspace_bytes(ctypes.byref(desc), T, top_k)
    if nb == 0:
        raise RuntimeError(f"moe: {lib().paro_last_error().decode()}")
    return nb


def moe_forward(desc: ParoMoEDesc, x: torch.Tensor, topk_ids: torch.Tensor, topk_weights: torch.Tensor, h: torch.Tensor, y: torch.Tensor,
                workspace: torch.Tensor) -> None:
    """paro_moe_forward on the current stream of x's device: x [T, hidden], topk_ids [T, k] int32, topk_weights [T, k] fp32,
    h [T, k, 2I] and y [T, hidden] of the experts' dtype, all contiguous on one CUDA device."""
    _moe_call("moe_forward", lib().paro_moe_forward, desc, x, topk_ids, topk_weights, h, y, workspace)


def moe_grouped_forward(desc: ParoMoEDesc, x: torch.Tensor, topk_ids: torch.Tensor, topk_weights: torch.Tensor, h: torch.Tensor,
                        y: torch.Tensor, workspace: torch.Tensor) -> None:
    """paro_moe_grouped_forward (any T) with the arguments of moe_forward; the workspace holds moe_grouped_workspace_bytes."""
    _moe_call("moe_grouped_forward", lib().paro_moe_grouped_forward, desc, x, topk_ids, topk_weights, h, y, workspace)


def moe_grouped_workspace_bytes(desc: ParoMoEDesc, T: int, top_k: int) -> int:
    nb = lib().paro_moe_grouped_workspace_bytes(ctypes.byref(desc), T, top_k)
    if nb == 0:
        raise RuntimeError(f"moe_grouped: {lib().paro_last_error().decode()}")
    return nb


def debug_moe_grouped_plan(desc: ParoMoEDesc, T: int, top_k: int, sms: int) -> list[int]:
    """[NT, tiles_max, six launch grids, workspace regions / 256 (table, operand, y_s, total)] (include/paro_b200.h)."""
    out = (ctypes.c_int32 * 12)()
    _check(lib().paro_debug_moe_grouped_plan(ctypes.byref(desc), T, top_k, sms, out), "debug_moe_grouped_plan")
    return list(out)


def _moe_call(what: str, fn, desc: ParoMoEDesc, x, topk_ids, topk_weights, h, y, workspace) -> None:
    dt = _CODE_DTYPE[desc.gate_up.contents.dtype]
    H, I2 = desc.gate_up.contents.in_features, desc.gate_up.contents.out_features
    if topk_ids.dtype != torch.int32 or topk_weights.dtype != torch.float32:
        raise RuntimeError(f"{what}: topk_ids must be int32 and topk_weights float32, got {topk_ids.dtype} / {topk_weights.dtype}")
    for name, t in (("x", x), ("h", h), ("y", y)):
        if t.dtype != dt:
            raise RuntimeError(f"{what}: {name} must be {dt}, got {t.dtype}")
    dev = _need_cuda(x, topk_ids, topk_weights, h, y, workspace)
    if topk_ids.dim() != 2 or tuple(topk_weights.shape) != tuple(topk_ids.shape):
        raise RuntimeError(f"{what}: topk_ids and topk_weights must both be [T, k]")
    T, k = topk_ids.shape
    want = {"x": ((T, H), x), "h": ((T, k, I2), h), "y": ((T, H), y)}
    for name, (shp, t) in want.items():
        if tuple(t.shape) != shp:
            raise RuntimeError(f"{what}: {name} must be {shp}, got {tuple(t.shape)}")
    if not all(t.is_contiguous() for t in (x, topk_ids, topk_weights, h, y)):
        raise RuntimeError(f"{what}: all tensors must be contiguous")
    with torch.cuda.device(dev):
        rc = fn(ctypes.byref(desc), x.data_ptr(), topk_ids.data_ptr(), topk_weights.data_ptr(), T, k, h.data_ptr(), y.data_ptr(),
                workspace.data_ptr(), workspace.numel(), _stream(dev))
    _check(rc, what)


def debug_moe_plan(desc: ParoMoEDesc, T: int, top_k: int, sms: int) -> list[int]:
    out = (ctypes.c_int32 * 18)()
    _check(lib().paro_debug_moe_plan(ctypes.byref(desc), T, top_k, sms, out), "debug_moe_plan")
    return list(out)


def moe_route(x: torch.Tensor, w: torch.Tensor, top_k: int, renormalize: bool, ids_out: torch.Tensor, weights_out: torch.Tensor,
              logits_out: torch.Tensor | None = None) -> None:
    """paro_moe_route on the current stream of x's device: x [T, hidden] and the router weight w [E, hidden] of one dtype (float16
    or bfloat16) -> ids_out [T, top_k] int32, weights_out [T, top_k] fp32 and, when given, logits_out [T, E] fp32; all contiguous
    on one CUDA device.  One launch, nothing allocated."""
    if x.dtype not in (torch.float16, torch.bfloat16) or w.dtype != x.dtype:
        raise RuntimeError(f"moe_route: x and w must share float16 or bfloat16, got {x.dtype} / {w.dtype}")
    if ids_out.dtype != torch.int32 or weights_out.dtype != torch.float32 or (logits_out is not None and logits_out.dtype != torch.float32):
        raise RuntimeError("moe_route: ids_out must be int32, weights_out and logits_out float32")
    dev = _need_cuda(x, w, ids_out, weights_out, logits_out)
    if x.dim() != 2 or w.dim() != 2 or w.size(1) != x.size(1):
        raise RuntimeError(f"moe_route: x must be [T, hidden] and w [E, hidden], got {tuple(x.shape)} / {tuple(w.shape)}")
    (T, H), E, k = x.shape, w.size(0), int(top_k)
    want = {"ids_out": ((T, k), ids_out), "weights_out": ((T, k), weights_out), "logits_out": ((T, E), logits_out)}
    for name, (shp, t) in want.items():
        if t is not None and tuple(t.shape) != shp:
            raise RuntimeError(f"moe_route: {name} must be {shp}, got {tuple(t.shape)}")
    if not all(t is None or t.is_contiguous() for t in (x, w, ids_out, weights_out, logits_out)):
        raise RuntimeError("moe_route: all tensors must be contiguous")
    with torch.cuda.device(dev):
        rc = lib().paro_moe_route(x.data_ptr(), w.data_ptr(), dtype_code(x.dtype), T, H, E, k, 1 if renormalize else 0, ids_out.data_ptr(),
                                  weights_out.data_ptr(), logits_out.data_ptr() if logits_out is not None else None, _stream(dev))
    _check(rc, "moe_route")


def debug_moe_route_plan(T: int, hidden: int, n_experts: int, top_k: int, sms: int) -> list[int]:
    """[NT, cluster size, K slices, grid, shared-memory bytes, coverage violations, token tiles, threads] (include/paro_b200.h)."""
    out = (ctypes.c_int32 * 8)()
    _check(lib().paro_debug_moe_route_plan(T, hidden, n_experts, top_k, sms, out), "debug_moe_route_plan")
    return list(out)
