"""CPU: the `deterministic` keyword is checked before any device is touched, the deterministic entry points exist in
the library and its binding, their workspace is the per-row constants alone (a pure function of the problem, with no
dk / dv or dq accumulator), their arguments are checked before any launch, and the ABI structs keep their layout."""
import ctypes
import os

import pytest
import torch

from flash_cosine_sim_attention_b200 import _abi
from flash_cosine_sim_attention_b200.flash_cosine_sim_attention import (flash_cosine_sim_attention,
                                                                        flash_cosine_sim_attention_varlen)

NEW = ("fcsa_backward_fused_deterministic_workspace_bytes", "fcsa_backward_fused_deterministic",
       "fcsa_backward_fused_deterministic_varlen_workspace_bytes", "fcsa_backward_fused_deterministic_varlen")


@pytest.fixture(scope="module")
def lib():
    if not os.path.exists(_abi.LIB_PATH):
        from flash_cosine_sim_attention_b200.build import build_library
        build_library()
    return _abi.load()


def qkv(D=64, n=16):
    return tuple(torch.randn(1, 2, n, D) for _ in range(3))       # CPU tensors: any device check would raise


@pytest.mark.parametrize("bad", [1, 0, None, "yes", 1.0, torch.tensor(True)])
def test_non_bool_rejected_first(bad):
    with pytest.raises(TypeError, match="deterministic must be a bool"):
        flash_cosine_sim_attention(*qkv(), deterministic=bad)
    q, k, v = (t[0].transpose(0, 1) for t in qkv())
    cu = torch.tensor([0, 16], dtype=torch.int32)
    with pytest.raises(TypeError, match="deterministic must be a bool"):
        flash_cosine_sim_attention_varlen(q, k, v, cu, cu, 16, 16, deterministic=bad)


def test_bias_rejected_first():
    q, k, v = qkv()
    with pytest.raises(NotImplementedError, match="deterministic=True with attn_bias"):
        flash_cosine_sim_attention(q, k, v, attn_bias=torch.zeros(2, 16, 16), deterministic=True)
    # deterministic=False keeps the existing behaviour: the CPU tensors are refused by the device check
    with pytest.raises(RuntimeError, match="CUDA tensors required"):
        flash_cosine_sim_attention(q, k, v, attn_bias=torch.zeros(2, 16, 16), deterministic=False)
    with pytest.raises(RuntimeError, match="CUDA tensors required"):
        flash_cosine_sim_attention(q, k, v, deterministic=True)


def test_symbols(lib):
    for name in NEW:
        assert name in _abi.EXPORTED_SYMBOLS
        assert hasattr(lib, name)


def problem(B, H, Hk, Nq, Nk, D):
    p = _abi.FcsaProblem()
    p.dtype, p.batch, p.heads, p.kv_heads, p.seq_q, p.seq_k, p.head_dim = _abi.FCSA_BF16, B, H, Hk, Nq, Nk, D
    p.scale, p.shift = 8.0, 8.0
    return p


@pytest.mark.parametrize("B,H,Hk,Nq,Nk,D", [(4, 8, 8, 4096, 4096, 64), (4, 8, 1, 4096, 4096, 64),
                                            (1, 16, 2, 4096, 4096, 128), (2, 4, 2, 300, 700, 64),
                                            (3, 6, 3, 1, 129, 128)])
def test_workspace_is_the_stats_alone(lib, B, H, Hk, Nq, Nk, D):
    p = problem(B, H, Hk, Nq, Nk, D)
    n = lib.fcsa_backward_fused_deterministic_workspace_bytes(_abi.ref(p))
    stats = B * H * ((Nq + 63) // 64) * 128 * 4            # {c3, -delta} per row of every 64-row query tile
    assert n == (stats + 255) // 256 * 256
    assert lib.fcsa_backward_fused_deterministic_workspace_bytes(_abi.ref(p)) == n
    # the default backward's scratch adds the fp32 dk / dv accumulators of grouped problems
    assert lib.fcsa_backward_workspace_bytes(_abi.ref(p)) == n + (2 * B * Hk * Nk * D * 4 if Hk < H else 0)
    p.window, p.causal = 65, 1
    assert lib.fcsa_backward_fused_deterministic_workspace_bytes(_abi.ref(p)) == n
    p.head_dim = 96
    assert lib.fcsa_backward_fused_deterministic_workspace_bytes(_abi.ref(p)) == 0      # refused problem


def test_varlen_workspace_is_the_stats_alone(lib):
    p = problem(5, 8, 2, 1500, 1500, 64)
    vl = _abi.FcsaVarlen()
    vl.cu_seqlens_q = vl.cu_seqlens_k = 4096               # never read on the host
    vl.total_q, vl.total_k = 3000, 3000
    n = lib.fcsa_backward_fused_deterministic_varlen_workspace_bytes(_abi.ref(p), _abi.ref(vl))
    stats = 8 * (3000 // 64 + 5 + 1) * 128 * 4
    assert n == (stats + 255) // 256 * 256
    assert lib.fcsa_backward_fused_varlen_workspace_bytes(_abi.ref(p), _abi.ref(vl)) == n + 2 * 2 * 3000 * 64 * 4
    vl.cu_seqlens_q = None
    assert lib.fcsa_backward_fused_deterministic_varlen_workspace_bytes(_abi.ref(p), _abi.ref(vl)) == 0


def test_arguments_checked_before_any_launch(lib):
    p = problem(1, 1, 1, 128, 128, 64)
    t = _abi.FcsaTensor(4096, 128 * 64, 128 * 64, 64)
    n = _abi.FcsaL2Norm(0, t, t, None, None)
    need = lib.fcsa_backward_fused_deterministic_workspace_bytes(_abi.ref(p))
    T = _abi.ref(t)
    rc = lib.fcsa_backward_fused_deterministic(_abi.ref(p), None, T, T, T, 4096, T, T, T, 4096, need, None)
    assert rc == _abi.FCSA_ERR_INVALID and b"fcsa_l2norm" in lib.fcsa_last_error()
    rc = lib.fcsa_backward_fused_deterministic(_abi.ref(p), _abi.ref(n), T, T, T, 4096, T, T, T, 4096, need - 1, None)
    assert rc == _abi.FCSA_ERR_WORKSPACE and b"workspace too small" in lib.fcsa_last_error()
    n.groups = 1                                            # fused l2norm without the reciprocal norms
    rc = lib.fcsa_backward_fused_deterministic(_abi.ref(p), _abi.ref(n), T, T, T, 4096, T, T, T, 4096, need, None)
    assert rc == _abi.FCSA_ERR_INVALID and b"rnorm" in lib.fcsa_last_error()
    vl = _abi.FcsaVarlen(4096, 4096, 128, 128)
    p.out_f32 = 1
    rc = lib.fcsa_backward_fused_deterministic_varlen(_abi.ref(p), _abi.ref(vl), _abi.ref(n), T, T, T, 4096, T, T, T,
                                                      4096, need, None)
    assert rc == _abi.FCSA_ERR_UNSUPPORTED and b"out_f32" in lib.fcsa_last_error()


def test_abi_unchanged(lib):
    assert ctypes.sizeof(_abi.FcsaProblem) == 64
    assert _abi.FcsaProblem.out_f32.offset == 56 and _abi.FcsaProblem.window.offset == 60
    assert lib.fcsa_version() == 300
