"""The C-ABI boundary without a GPU: the library loads, exports every symbol include/*.h
declares, and its host-side checks / size queries behave (no compute calls here)."""
import ctypes
import re
from pathlib import Path

import pytest
import torch

from paroquant_b200 import _cabi

ROOT = Path(__file__).resolve().parents[1]


def _declared_symbols():
    text = (ROOT / "include" / "paro_b200.h").read_text()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    return sorted(set(re.findall(r"\b(paro_[a-z_0-9]+)\s*\(", text)))


def test_library_exports_every_declared_symbol():
    lib = _cabi.lib()
    names = _declared_symbols()
    assert len(names) >= 9
    for n in names:
        assert hasattr(lib, n), f"{n} declared in include/paro_b200.h but not exported"
    assert set(names) == set(_cabi.EXPORTED_SYMBOLS)
    assert lib.paro_abi_version() == _cabi.ABI_VERSION == 5


def test_debug_silu_mul_argument_checks():
    """paro_debug_silu_mul's host-side checks (no launch): dtype, an even I, pointers and alignment; no rows is a no-op."""
    lib = _cabi.lib()
    buf = (ctypes.c_char * 4096)()
    p = (ctypes.addressof(buf) + 255) // 256 * 256
    for args, code, msg in (((0, p, p, 1, 8), 1, b"F16 or BF16"), ((2, p, p, 1, 7), 1, b"even I"), ((2, p, p, -1, 8), 1, b"M >= 0"),
                            ((2, None, p, 1, 8), 1, b"null pointer"), ((1, p + 2, p, 1, 8), 1, b"4-byte aligned"),
                            ((2, p, p, 0, 8), 0, None)):
        rc = lib.paro_debug_silu_mul(*args, None)
        assert rc == code and (msg is None or msg in lib.paro_last_error()), (args, rc, lib.paro_last_error())
    assert lib.paro_last_launch_count() == 0
    with pytest.raises(RuntimeError, match="CUDA-only"):
        _cabi.debug_silu_mul(torch.zeros(2, 16, dtype=torch.bfloat16))
    for last in (17, 18, 2):   # gate | up halves must each have an even width: an odd last dimension would shift the up half
        with pytest.raises(RuntimeError, match="last dimension must be 2I"):
            _cabi.debug_silu_mul(torch.zeros(2, last, dtype=torch.bfloat16))
    with pytest.raises(RuntimeError, match="float16 or bfloat16"):
        _cabi.debug_silu_mul(torch.zeros(2, 16))


def test_struct_layout_matches_header():
    assert ctypes.sizeof(_cabi.ParoLinearShape) == 4 * (5 + 8 + 1)


def test_size_queries_and_shape_errors():
    s = _cabi.make_shape(4096, [4096], 128, 8, torch.bfloat16)
    # 32 blocks of 128 columns x 32 groups x 8576-byte records + 32 groups x (8*256+256) bytes of rotation metadata
    assert _cabi.packed_bytes(s) == 32 * 32 * 8576 + 32 * 2304
    assert _cabi.workspace_bytes(s, 1) >= 256          # the small-M kernel reduces through distributed shared memory
    assert _cabi.workspace_bytes(s, 4096) >= 4096 * 4096 * 2   # M > 16: the rotated activations are staged once
    assert _cabi.workspace_bytes(s, 16) >= _cabi.workspace_bytes(s, 8)
    # a partition that is not a whole number of 128-column blocks is padded to one
    s2 = _cabi.make_shape(256, [272, 16], 128, 8, torch.float16)
    assert _cabi.packed_bytes(s2) == (3 + 1) * 2 * 8576 + 2 * 2 * 2304
    # group_size 64: a record still covers 128 channels and carries two scale / zero sets (8960 bytes)
    s64 = _cabi.make_shape(4096, [4096], 64, 8, torch.bfloat16)
    assert _cabi.packed_bytes(s64) == 32 * 32 * 8960 + 32 * 2304
    for bad, msg in ((dict(in_features=4000), "multiple of 128"), (dict(part_sizes=[100]), "multiple of 16"),
                     (dict(group_size=32), "group_size"), (dict(krot=17), "krot")):
        kw = dict(in_features=4096, part_sizes=[4096], group_size=128, krot=8, dtype=torch.bfloat16)
        kw.update(bad)
        with pytest.raises(RuntimeError, match=msg):
            _cabi.packed_bytes(_cabi.make_shape(**kw))
    with pytest.raises(RuntimeError, match="Float, Half, and BFloat16"):
        _cabi.make_shape(4096, [4096], 128, 8, torch.int8)


def test_merged_layout_is_partition_major():
    s = _cabi.make_shape(4096, [4096, 1024, 1024], 128, 8, torch.float16)
    assert _cabi.packed_bytes(s) == 32 * 48 * 8576 + ((3 * 32 * 2304 + 127) // 128) * 128


def test_cpu_tensors_are_rejected_loudly():
    x = torch.zeros(2, 128)
    with pytest.raises(RuntimeError, match="CUDA-only"):
        _cabi.rotate(x, torch.zeros(8, 128, dtype=torch.int16), torch.zeros(8, 64))
    import paroquant_b200.kernels.cuda  # noqa: F401
    with pytest.raises(NotImplementedError):
        torch.ops.rotation.rotate(x, torch.zeros(8, 128, dtype=torch.int16), torch.zeros(8, 64))


def test_null_and_bad_arguments_return_codes():
    lib = _cabi.lib()
    rc = lib.paro_rotate(None, None, None, None, 0, None, 0, 1, 128, 8, 128, 2, None)
    assert rc == 1 and b"null pointer" in lib.paro_last_error()
    buf = (ctypes.c_char * 4096)()
    p = ctypes.addressof(buf)
    p = (p + 255) // 256 * 256
    rc = lib.paro_rotate(p, p, p, p, 1, None, 0, 1, 128, 8, 32, 2, None)
    assert rc == 2 and b"Unsupported group_size: 32; expected 64 or 128" in lib.paro_last_error()
    rc = lib.paro_rotate(p, p, p, p, 1, None, 0, 1, 100, 8, 64, 2, None)
    assert rc == 1 and b"h must be divisible by GROUP_SIZE" in lib.paro_last_error()
    rc = lib.paro_rotate(p, p, p, p, 1, None, 0, 1, 128, 8, 128, 7, None)
    assert rc == 1 and b"Float, Half, and BFloat16" in lib.paro_last_error()
    rc = lib.paro_rotate(p, p, p, p, 1, None, 0, 0, 128, 8, 128, 2, None)   # empty input: no launch, success
    assert rc == 0 and lib.paro_last_launch_count() == 0


def test_rotate_backward_argument_checks():
    """paro_rotate_backward: same schema errors as the forward op, plus its own pointer rules (host side only)."""
    lib = _cabi.lib()
    buf = (ctypes.c_char * 8192)()
    p = (ctypes.addressof(buf) + 255) // 256 * 256
    q, g = p + 1024, p + 2048
    rc = lib.paro_rotate_backward(None, None, None, None, None, 0, None, 0, None, None, None, 1, 128, 8, 128, 0, 0, None)
    assert rc == 1 and b"null pointer" in lib.paro_last_error()
    rc = lib.paro_rotate_backward(p, p, p, p, p, 0, None, 0, q, g, g, 1, 128, 8, 128, 0, 0, None)        # grad_scale without scales
    assert rc == 1 and b"grad_scale needs x and scales" in lib.paro_last_error()
    rc = lib.paro_rotate_backward(p, p, p, p, p, 0, None, 0, p, g, None, 1, 128, 8, 128, 0, 0, None)     # grad_x aliases y
    assert rc == 1 and b"must not alias" in lib.paro_last_error()
    rc = lib.paro_rotate_backward(p, p, p, p, p, 0, None, 0, q, g, None, 1, 128, 8, 32, 0, 0, None)
    assert rc == 2 and b"Unsupported group_size: 32; expected 64 or 128" in lib.paro_last_error()
    rc = lib.paro_rotate_backward(p, p, p, p, p, 0, None, 0, q, g, None, 1, 100, 8, 64, 0, 0, None)
    assert rc == 1 and b"h must be divisible by GROUP_SIZE" in lib.paro_last_error()
    rc = lib.paro_rotate_backward(p, p, p, p, p, 0, None, 0, q, g, None, 1, 128, 17, 128, 0, 0, None)
    assert rc == 2 and b"Unsupported KROT" in lib.paro_last_error()
    rc = lib.paro_rotate_backward(p, p, p, p, p, 0, None, 0, q, g, None, 1, 128, 8, 128, 9, 0, None)
    assert rc == 1 and b"Float, Half, and BFloat16" in lib.paro_last_error()
    rc = lib.paro_rotate_backward(p, p, p, p, p, 0, None, 0, q, g, None, 1, 128, 8, 128, 0, 2, None)
    assert rc == 1 and b"unknown theta_formula" in lib.paro_last_error()
    rc = lib.paro_rotate_backward(p, p, p, p, p, 0, None, 0, q, g, None, 0, 128, 8, 128, 0, 1, None)     # no rows: no launch, success
    assert rc == 0 and lib.paro_last_launch_count() == 0


def _chain(steps):
    arr = (_cabi.ParoChainStep * len(steps))()
    keep = []
    for c, kw in zip(arr, steps):
        shape = kw.pop("shape")
        keep.append(shape)
        c.shape = ctypes.pointer(shape)
        c.packed = 0x10000 if kw.pop("packed", True) else None      # never dereferenced by the host-side checks
        for k, v in kw.items():
            setattr(c, k, v)
    return arr, keep


def test_chain_host_checks_and_sizes():
    """paro_chain_workspace_bytes / paro_tp_slot_bytes and the argument checks of a chain, host side only."""
    lib = _cabi.lib()
    o = _cabi.make_shape(4096, [4096], 128, 8, torch.bfloat16)
    gu = _cabi.make_shape(4096, [14336, 14336], 128, 8, torch.bfloat16)
    down = _cabi.make_shape(14336, [4096], 128, 8, torch.bfloat16)
    arr, keep = _chain([dict(shape=o, x=0x20000, epilogue=_cabi.EPI_ADD_RESIDUAL, residual_in=0x30000, residual_out=0x40000),
                        dict(shape=gu, x_op=_cabi.XOP_RMSNORM, norm_weight=0x50000, y=0x60000),
                        dict(shape=down, x_op=_cabi.XOP_SILU_MUL, y=0x70000)])
    one = lib.paro_chain_workspace_bytes(arr, 1, 1)
    three = lib.paro_chain_workspace_bytes(arr, 3, 1)
    assert 256 < one < three < 64 << 20
    assert lib.paro_chain_workspace_bytes(arr, 3, 16) > three          # slots and published words grow with the rows
    assert lib.paro_chain_workspace_bytes(arr, 3, 17) == 0 and b"M <= 16" in lib.paro_last_error()
    assert lib.paro_chain_workspace_bytes(arr, 7, 1) == 0 and b"steps" in lib.paro_last_error()
    bad, keep2 = _chain([dict(shape=o, x=0x20000, epilogue=_cabi.EPI_ADD_RESIDUAL, residual_in=0x30000, residual_out=0x30000)])
    assert lib.paro_chain_workspace_bytes(bad, 1, 1) == 0 and b"alias" in lib.paro_last_error()
    bad, keep3 = _chain([dict(shape=o, x=0x20000, x_op=7, y=0x30000)])
    assert lib.paro_chain_workspace_bytes(bad, 1, 1) == 0 and b"x_op" in lib.paro_last_error()
    # tensor parallel: 2 halves (launch parity) x blocks x ranks x rows x 128 columns x 8-byte {value, tag} words
    assert lib.paro_tp_slot_bytes(ctypes.byref(o), 1, 8) == 2 * 32 * 8 * 1 * 128 * 8
    assert lib.paro_tp_slot_bytes(ctypes.byref(o), 4, 2) == 2 * 32 * 2 * 4 * 128 * 8
    assert lib.paro_tp_slot_bytes(ctypes.byref(o), 1, 9) == 0
    info = _cabi.ParoTpInfo()
    info.world, info.rank = 2, 0
    info.peer_slots[0] = 0x100000                                     # rank 1's buffer missing
    tp, keep4 = _chain([dict(shape=o, x=0x20000, y=0x30000, tp=ctypes.pointer(info))])
    assert lib.paro_chain_workspace_bytes(tp, 1, 1) == 0 and b"peer_slots[1]" in lib.paro_last_error()
    info.rank = 2
    assert lib.paro_chain_workspace_bytes(tp, 1, 1) == 0 and b"rank < world" in lib.paro_last_error()
