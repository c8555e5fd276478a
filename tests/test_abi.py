"""CPU: the C-ABI library loads, exports every symbol include/fcsa_b200.h declares, its struct
layouts match the ctypes mirrors, and argument errors are reported through return codes.
No compute call is made (there is no GPU here)."""
import ctypes
import os
import re

import pytest

from flash_cosine_sim_attention_b200 import _abi

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "include", "fcsa_b200.h")


@pytest.fixture(scope="module")
def lib():
    if not os.path.exists(_abi.LIB_PATH):
        from flash_cosine_sim_attention_b200.build import build_library
        build_library()
    return _abi.load()


def header_functions():
    src = open(HEADER).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(fcsa_[a-z0-9_]+)\s*\(", src)))


def test_header_and_binding_agree():
    assert header_functions() == sorted(_abi.EXPORTED_SYMBOLS)


def test_library_exports_every_declared_symbol(lib):
    for name in header_functions():
        assert hasattr(lib, name), f"{name} declared in fcsa_b200.h but not exported"


def test_struct_layouts():
    # fcsa_tensor: void* + 3 x int64; fcsa_problem: 8 x int32, 2 x float, pointer, int64, 2 x int32
    assert ctypes.sizeof(_abi.FcsaTensor) == 32
    assert ctypes.sizeof(_abi.FcsaProblem) == 8 * 4 + 2 * 4 + 8 + 8 + 8
    assert _abi.FcsaProblem.out_f32.offset == 56
    assert _abi.FcsaProblem.key_mask.offset == 40


def test_version_and_launch_counter(lib):
    assert lib.fcsa_version() >= 100
    assert lib.fcsa_debug() == 0          # nothing launched in this process


def test_errors_are_returned_not_printed(lib):
    p = _abi.FcsaProblem()
    p.dtype, p.batch, p.heads, p.kv_heads, p.seq_q, p.seq_k, p.head_dim = _abi.FCSA_BF16, 1, 2, 2, 16, 16, 48
    t = _abi.FcsaTensor(None, 0, 0, 0)
    rc = lib.fcsa_forward(_abi.ref(p), _abi.ref(t), _abi.ref(t), _abi.ref(t), _abi.ref(t), None, None)
    assert rc == _abi.FCSA_ERR_UNSUPPORTED and b"head_dim" in lib.fcsa_last_error()
    p.head_dim = 64
    rc = lib.fcsa_forward(_abi.ref(p), _abi.ref(t), _abi.ref(t), _abi.ref(t), _abi.ref(t), None, None)
    assert rc == _abi.FCSA_ERR_INVALID and b"null" in lib.fcsa_last_error()
    p.kv_heads = 3
    rc = lib.fcsa_forward(_abi.ref(p), _abi.ref(t), _abi.ref(t), _abi.ref(t), _abi.ref(t), None, None)
    assert rc == _abi.FCSA_ERR_INVALID and b"kv_heads" in lib.fcsa_last_error()
    p.kv_heads, p.causal, p.key_mask = 2, 1, 1
    rc = lib.fcsa_forward(_abi.ref(p), _abi.ref(t), _abi.ref(t), _abi.ref(t), _abi.ref(t), None, None)
    assert rc == _abi.FCSA_ERR_INVALID and b"mask should not be supplied" in lib.fcsa_last_error()
    with pytest.raises(_abi.FcsaError):
        _abi.check(rc)


def test_misaligned_tensor_rejected(lib):
    p = _abi.FcsaProblem()
    p.dtype, p.batch, p.heads, p.kv_heads, p.seq_q, p.seq_k, p.head_dim = _abi.FCSA_F16, 1, 1, 1, 8, 8, 64
    good = _abi.FcsaTensor(4096, 512, 512, 64)
    bad_ptr = _abi.FcsaTensor(4098, 512, 512, 64)
    bad_stride = _abi.FcsaTensor(4096, 512, 512, 68)
    assert lib.fcsa_forward(_abi.ref(p), _abi.ref(bad_ptr), _abi.ref(good), _abi.ref(good), _abi.ref(good), None, None) == _abi.FCSA_ERR_INVALID
    assert lib.fcsa_forward(_abi.ref(p), _abi.ref(good), _abi.ref(bad_stride), _abi.ref(good), _abi.ref(good), None, None) == _abi.FCSA_ERR_INVALID


def test_workspace_size_formula(lib):
    p = _abi.FcsaProblem()
    p.dtype, p.batch, p.heads, p.kv_heads, p.seq_q, p.seq_k, p.head_dim = _abi.FCSA_BF16, 4, 8, 8, 4096, 4096, 64
    n = lib.fcsa_backward_workspace_bytes(_abi.ref(p))
    stats = 4 * 8 * 64 * 128 * 4            # 64 query tiles of 64 rows: {c3, -delta} per row
    dq = 4 * 8 * 4096 * 64 * 4
    assert n == stats                       # scratch: per-row constants only
    assert lib.fcsa_backward_zeroed_bytes(_abi.ref(p)) == dq            # self-cleaning fp32 dq accumulator
    p.kv_heads = 1
    assert lib.fcsa_backward_workspace_bytes(_abi.ref(p)) == stats + 2 * 4 * 4096 * 64 * 4
    assert lib.fcsa_backward_zeroed_bytes(_abi.ref(p)) == dq


def test_backward_rejects_missing_zeroed_workspace(lib):
    p = _abi.FcsaProblem()
    p.dtype, p.batch, p.heads, p.kv_heads, p.seq_q, p.seq_k, p.head_dim = _abi.FCSA_BF16, 1, 1, 1, 128, 128, 64
    p.scale, p.shift = 8.0, 8.0
    t = _abi.FcsaTensor(4096, 128 * 64, 128 * 64, 64)
    need = lib.fcsa_backward_workspace_bytes(_abi.ref(p))
    rc = lib.fcsa_backward(_abi.ref(p), *([_abi.ref(t)] * 5), 4096, *([_abi.ref(t)] * 3), 4096, need, None, 0, None)
    assert rc == _abi.FCSA_ERR_WORKSPACE and b"zeroed workspace" in lib.fcsa_last_error()
    assert lib.fcsa_zeroed_init(None, 0, None) == _abi.FCSA_ERR_INVALID


def test_row_pass_shape_checks(lib):
    """The 16-bit l2norm takes head dims 32 to 256 and groups > 0; the float32 cast takes 16 to 128 and groups >= 0
    (0: a plain scaled cast).  Shapes that pass reach the null-tensor check, so nothing here is launched."""
    t = _abi.FcsaTensor(None, 0, 0, 0)

    def l2(D, G, dtype=_abi.FCSA_BF16, B=1):
        rc = lib.fcsa_l2norm_forward(dtype, B, 1, 8, D, G, _abi.ref(t), _abi.ref(t), None, None)
        return rc, lib.fcsa_last_error()

    def f32(D, G, dtype=_abi.FCSA_BF16, B=1):
        rc = lib.fcsa_f32_cast(dtype, B, 1, 8, D, G, _abi.ref(t), _abi.ref(t), None, None, 0, None)
        return rc, lib.fcsa_last_error()

    accepted = (_abi.FCSA_ERR_INVALID, b"null")
    for fn, prefix in ((l2, b"l2norm: "), (f32, b"f32 cast: ")):
        assert fn(64, 1, dtype=7)[0] == _abi.FCSA_ERR_UNSUPPORTED
        assert fn(64, 1, B=0) == (_abi.FCSA_ERR_INVALID, prefix + b"empty tensor")
        for D in (8, 48, 96, 512):
            assert fn(D, 1) == (_abi.FCSA_ERR_UNSUPPORTED, prefix + b"head_dim %d not implemented" % D)
        for G in (-1, 3, 128):
            rc, msg = fn(64, G)
            assert rc == _abi.FCSA_ERR_INVALID and msg.startswith(prefix + b"groups")
        for G in (1, 2, 16, 64):
            assert fn(64, G)[0] == accepted[0] and accepted[1] in fn(64, G)[1]
    assert l2(16, 1)[0] == _abi.FCSA_ERR_UNSUPPORTED and accepted[1] in f32(16, 1)[1]
    assert accepted[1] in l2(256, 1)[1] and f32(256, 1)[0] == _abi.FCSA_ERR_UNSUPPORTED
    assert l2(64, 0)[1].startswith(b"l2norm: groups") and accepted[1] in f32(64, 0)[1]
