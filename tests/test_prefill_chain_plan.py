"""Host-side checks of the prefill chain (paro_prefill_chain_workspace_bytes / paro_prefill_chain_forward): the workspace
regions, the row bounds of both chain entries, the rejection of tensor-parallel steps, and the step-to-step checks it shares
with the decode chain, message for message.  Descriptors carry made-up device addresses; nothing here touches a device."""
import ctypes

import pytest
import torch

from paroquant_b200 import _cabi

BASE = 1 << 32   # made-up, suitably aligned device addresses


def _addr(i):
    return BASE + i * (1 << 24)


def _steps(specs):
    """specs: dicts with K, parts and optionally x / y / x_op / epilogue / res / norm / tp (True: a 2-rank tp step)."""
    arr = (_cabi.ParoChainStep * len(specs))()
    keep = []
    for i, sp in enumerate(specs):
        shape = _cabi.make_shape(sp["K"], sp["parts"], sp.get("G", 128), sp.get("krot", 8), sp.get("dtype", torch.bfloat16))
        keep.append(shape)
        c = arr[i]
        c.shape = ctypes.pointer(shape)
        c.packed = _addr(10 * i + 1)
        c.x = _addr(10 * i + 2) if sp.get("x", i == 0) else None
        c.y = _addr(10 * i + 3) if sp.get("y", True) else None
        c.x_op = {"none": _cabi.XOP_NONE, "silu_mul": _cabi.XOP_SILU_MUL, "rmsnorm": _cabi.XOP_RMSNORM}[sp.get("x_op", "none")]
        c.epilogue = _cabi.EPI_ADD_RESIDUAL if sp.get("epilogue") == "add_residual" else _cabi.EPI_STORE
        if c.epilogue == _cabi.EPI_ADD_RESIDUAL:
            r = sp.get("res", (_addr(10 * i + 4), _addr(10 * i + 5)))
            c.residual_in, c.residual_out = r
        if c.x_op == _cabi.XOP_RMSNORM and sp.get("norm", True):
            c.norm_weight = _addr(10 * i + 6)
        c.eps = 1e-5
        if sp.get("tp"):
            info = _cabi.ParoTpInfo()
            info.world, info.rank = 2, 0
            info.peer_slots[0], info.peer_slots[1] = _addr(10 * i + 7), _addr(10 * i + 8)
            keep.append(info)
            c.tp = ctypes.pointer(info)
    arr._keep = keep
    return arr


def _tail(H=512, I=1024, qkv=(512, 128, 128), mlp_y=True):
    return [dict(K=H, parts=[H], x=True, y=False, epilogue="add_residual"),
            dict(K=H, parts=[I, I], x=False, x_op="rmsnorm", y=mlp_y),
            dict(K=I, parts=[H], x=False, x_op="silu_mul", y=False, epilogue="add_residual"),
            dict(K=H, parts=list(qkv), x=False, x_op="rmsnorm")]


def _ws(specs, M):
    return _cabi.lib().paro_prefill_chain_workspace_bytes(_steps(specs), len(specs), M)


def _err():
    return _cabi.lib().paro_last_error().decode()


def _up(b):
    return -(-b // 256) * 256


@pytest.mark.parametrize("M", [1, 17, 40, 100, 256, 1000, 4096])
def test_workspace_regions(M):
    """operand of the largest step (rows padded to 256, every partition) + fp32 [blocks][M] statistics of each ADD_RESIDUAL
    step an RMSNORM step reads + the outputs of consumed STORE steps without y."""
    H, I = 512, 1024
    m256 = -(-M // 256) * 256
    operand = max(1 * m256 * H * 2, 2 * m256 * H * 2, 1 * m256 * I * 2, 3 * m256 * H * 2)
    stats = 2 * _up(4 * M * 4)   # o and down: 4 blocks of 128 columns each
    assert _ws(_tail(H, I), M) == operand + stats
    assert _ws(_tail(H, I, mlp_y=False), M) == operand + stats + _up(M * 2 * I * 2)   # gate_up output kept in the workspace
    # no RMSNORM consumer, no statistics
    assert _ws(_tail(H, I)[:1] + [dict(K=H, parts=[H], x=False)], M) == _up(m256 * H * 2)


def test_workspace_grows_with_rows_and_the_largest_step():
    sizes = [_ws(_tail(), M) for M in (17, 256, 257, 1000, 4096)]
    assert all(a < b for a, b in zip(sizes, sizes[1:])), sizes
    small = _ws([dict(K=512, parts=[256])], 300)
    wide = _ws([dict(K=512, parts=[256]), dict(K=256, parts=[2048, 2048], x=True)], 300)
    deep = _ws([dict(K=512, parts=[256]), dict(K=2048, parts=[256], x=True)], 300)
    assert small == 512 * 512 * 2 and wide == 512 * 256 * 2 * 2 and deep == 512 * 2048 * 2


def test_row_bounds_of_both_entries():
    L = _cabi.lib()
    specs = [dict(K=512, parts=[256])]
    for M in (0, -1):
        assert _ws(specs, M) == 0 and "1 <= M" in _err()
        rc = L.paro_prefill_chain_forward(_steps(specs), 1, M, _addr(99), 1 << 30, None)
        assert rc == 2 and "1 <= M" in _err()
    assert _ws(specs, 17) > 0 and _ws(specs, 1) > 0
    assert L.paro_chain_workspace_bytes(_steps(specs), 1, 17) == 0 and "M <= 16" in _err()
    rc = L.paro_chain_forward(_steps(specs), 1, 17, _addr(99), 1 << 30, None)
    assert rc == 2 and "M <= 16" in _err()


def test_tensor_parallel_steps_are_unsupported():
    L = _cabi.lib()
    specs = _tail()
    specs[0]["tp"] = True
    assert _ws(specs, 64) == 0 and "tensor-parallel" in _err()
    rc = L.paro_prefill_chain_forward(_steps(specs), 4, 64, _addr(99), 1 << 30, None)
    assert rc == 2 and "tensor-parallel" in _err()


def test_a_short_workspace_is_named():
    need = _ws(_tail(), 300)
    rc = _cabi.lib().paro_prefill_chain_forward(_steps(_tail()), 4, 300, _addr(99), need - 1, None)
    assert rc == 4 and f"need {need}" in _err()


@pytest.mark.parametrize("case,code,msg", [
    ("no_input", 1, "chain: step 0 needs an input"),
    ("rmsnorm_with_x", 2, "chain: step 0: RMSNORM needs the statistics of the previous step (x must be NULL)"),
    ("rmsnorm_after_store", 1, "chain: step 1: RMSNORM follows an ADD_RESIDUAL epilogue"),
    ("columns", 1, "chain: step 0 produces 256 columns, step 1 consumes 512"),
    ("silu_columns", 1, "chain: step 0 produces 512 columns, step 1 consumes 1024"),
    ("no_residual", 1, "chain: step 0: ADD_RESIDUAL needs residual_in and residual_out"),
    ("no_norm_weight", 1, "chain: step 1: RMSNORM needs norm_weight"),
    ("no_output", 1, "chain: step 0 has no output"),
    ("dtypes", 1, "chain: every step must use the same activation dtype"),
    ("alias", 1, "chain: step 0: residual_out must not alias residual_in"),
])
def test_link_checks_match_the_decode_chain(case, code, msg):
    """Every rejection: the same code and message from both entries of the prefill chain and from the decode chain's forward."""
    specs = {
        "no_input": [dict(K=256, parts=[128], x=False)],
        "rmsnorm_with_x": [dict(K=256, parts=[128], x_op="rmsnorm")],
        "rmsnorm_after_store": [dict(K=256, parts=[256]), dict(K=256, parts=[128], x=False, x_op="rmsnorm")],
        "columns": [dict(K=256, parts=[256]), dict(K=512, parts=[128], x=False)],
        "silu_columns": [dict(K=256, parts=[256, 256]), dict(K=512, parts=[128], x=False, x_op="silu_mul")],
        "no_residual": [dict(K=256, parts=[128], epilogue="add_residual", res=(_addr(7), 0))],
        "no_norm_weight": [dict(K=256, parts=[256], epilogue="add_residual"), dict(K=256, parts=[128], x=False, x_op="rmsnorm", norm=False)],
        "no_output": [dict(K=256, parts=[128], y=False)],
        "dtypes": [dict(K=256, parts=[128]), dict(K=128, parts=[128], x=False, dtype=torch.float16)],
        "alias": [dict(K=256, parts=[128], epilogue="add_residual", res=(_addr(7), _addr(7)))],
    }[case]
    L = _cabi.lib()
    n = len(specs)
    assert _ws(specs, 40) == 0 and _err() == msg
    assert L.paro_prefill_chain_forward(_steps(specs), n, 40, _addr(99), 1 << 30, None) == code and _err() == msg
    assert L.paro_chain_forward(_steps(specs), n, 4, _addr(99), 1 << 30, None) == code and _err() == msg


def test_exported_and_abi_unchanged():
    assert {"paro_prefill_chain_workspace_bytes", "paro_prefill_chain_forward"} <= set(_cabi.EXPORTED_SYMBOLS)
    assert _cabi.lib().paro_abi_version() == 5


def test_wrapper_rejects_row_parallel_steps():
    from paroquant_b200 import chain

    class K:   # what ParoPrefillChain looks at before it builds a descriptor
        shape = _cabi.make_shape(256, [128], 128, 8, torch.bfloat16)
        packed = torch.zeros(1, dtype=torch.uint8)

    with pytest.raises(RuntimeError, match="row_parallel"):
        chain.ParoPrefillChain([chain.ChainStep(K(), row_parallel=True)], 40)
