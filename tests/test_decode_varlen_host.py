"""CPU: the argument checks of flash_cosine_sim_attention_with_kv_cache with packed new tokens (cu_seqlens_q,
max_seqlen_q) that need no device, and the rejections of fcsa_decode_varlen through the C ABI's return codes."""
import pytest
import torch


def _args(B=2, H=8, Hk=2, total=5, D=64, cap=128):
    q = torch.zeros(total, H, D, dtype=torch.bfloat16)
    kc = torch.zeros(B, Hk, cap, D, dtype=torch.bfloat16)
    sl = torch.zeros(B, dtype=torch.int32)
    cu = torch.tensor([0, 2, total], dtype=torch.int32)
    k = torch.zeros(total, Hk, D, dtype=torch.bfloat16)
    return q, kc, sl, cu, k


def test_packed_argument_checks():
    from flash_cosine_sim_attention_b200 import flash_cosine_sim_attention_with_kv_cache as f
    q, kc, sl, cu, k = _args()
    # q is 3-D exactly when cu_seqlens_q is given
    with pytest.raises(ValueError, match="with cu_seqlens_q, q must be packed"):
        f(q.unsqueeze(0), kc, kc, sl, cu_seqlens_q=cu, max_seqlen_q=3)
    with pytest.raises(ValueError, match="merged"):
        f(q, kc, kc, sl)
    with pytest.raises(ValueError, match="max_seqlen_q is for packed"):
        f(torch.zeros(2, 8, 1, 64, dtype=torch.bfloat16), kc, kc, sl, max_seqlen_q=1)
    # k, v packed like q
    with pytest.raises(ValueError, match="packed like q"):
        f(q, kc, kc, sl, k=k[:4], v=k[:4], cu_seqlens_q=cu, max_seqlen_q=3)
    with pytest.raises(ValueError, match="packed like q"):
        f(q, kc, kc, sl, k=k, v=k[:4], cu_seqlens_q=cu, max_seqlen_q=3)
    with pytest.raises(ValueError, match="packed like q"):
        f(q, kc, kc, sl, k=k.unsqueeze(0), v=k.unsqueeze(0), cu_seqlens_q=cu, max_seqlen_q=3)
    with pytest.raises(ValueError, match="both k and v"):
        f(q, kc, kc, sl, k=k, cu_seqlens_q=cu, max_seqlen_q=3)
    # cu_seqlens_q: dtype, length B + 1, contiguity, device
    with pytest.raises(TypeError, match="cu_seqlens_q must be an int32"):
        f(q, kc, kc, sl, cu_seqlens_q=cu.long(), max_seqlen_q=3)
    with pytest.raises(TypeError, match="cu_seqlens_q must be an int32"):
        f(q, kc, kc, sl, cu_seqlens_q=[0, 2, 5], max_seqlen_q=3)
    with pytest.raises(ValueError, match="needs 3"):
        f(q, kc, kc, sl, cu_seqlens_q=cu[:2], max_seqlen_q=3)
    with pytest.raises(ValueError, match="contiguous"):
        f(q, kc, kc, sl, cu_seqlens_q=torch.zeros(3, 2, dtype=torch.int32)[:, 0], max_seqlen_q=3)
    with pytest.raises(RuntimeError, match="on q's device"):
        f(q, kc, kc, sl, cu_seqlens_q=torch.zeros(3, dtype=torch.int32, device="meta"), max_seqlen_q=3)
    # max_seqlen_q: a non-negative Python int
    for bad in (None, -1, 3.0, True, torch.tensor(3)):
        with pytest.raises(TypeError, match="max_seqlen_q must be a non-negative Python int"):
            f(q, kc, kc, sl, cu_seqlens_q=cu, max_seqlen_q=bad)
    # the caches' batch sets B: cache_seqlens (B,)
    with pytest.raises(TypeError, match=r"cache_seqlens must be an int32 tensor of shape \(2,\)"):
        f(q, kc, kc, torch.zeros(5, dtype=torch.int32), cu_seqlens_q=cu, max_seqlen_q=3)
    # the rejections of the dense call hold as they were
    with pytest.raises(NotImplementedError, match="attn_bias"):
        f(q, kc, kc, sl, attn_bias=torch.zeros(8, 1, 128), cu_seqlens_q=cu, max_seqlen_q=3)
    with pytest.raises(NotImplementedError, match="mask"):
        f(q, kc, kc, sl, mask=torch.ones(2, 128, dtype=torch.bool), cu_seqlens_q=cu, max_seqlen_q=3)
    with pytest.raises(RuntimeError, match="no autograd"):
        f(q.clone().requires_grad_(), kc, kc, sl, cu_seqlens_q=cu, max_seqlen_q=3)
    with pytest.raises(TypeError, match="float32"):
        f(q.float(), kc.float(), kc.float(), sl, cu_seqlens_q=cu, max_seqlen_q=3)
    with pytest.raises(NotImplementedError, match="head_dim 96"):
        f(torch.zeros(5, 8, 96, dtype=torch.bfloat16), torch.zeros(2, 2, 8, 96, dtype=torch.bfloat16),
          torch.zeros(2, 2, 8, 96, dtype=torch.bfloat16), sl, cu_seqlens_q=cu, max_seqlen_q=3)
    with pytest.raises(ValueError, match="kv_heads"):
        f(q[:, :6], torch.zeros(2, 4, 8, 64, dtype=torch.bfloat16), torch.zeros(2, 4, 8, 64, dtype=torch.bfloat16), sl,
          cu_seqlens_q=cu, max_seqlen_q=3)
    with pytest.raises(ValueError, match="groups"):
        f(q, kc, kc, sl, groups=3, cu_seqlens_q=cu, max_seqlen_q=3)
    with pytest.raises(ValueError, match="window"):
        f(q, kc, kc, sl, window=0, cu_seqlens_q=cu, max_seqlen_q=3)
    with pytest.raises(RuntimeError, match="CUDA tensors required"):
        f(q, kc, kc, sl, cu_seqlens_q=cu, max_seqlen_q=3)          # CPU tensors: no CPU path
    with pytest.raises(RuntimeError, match="CUDA tensors required"):
        f(q, kc, kc, sl, k=k, v=k, cu_seqlens_q=cu, max_seqlen_q=0)


def _problem(_abi, **kw):
    p = _abi.FcsaProblem()
    p.dtype, p.batch, p.heads, p.kv_heads, p.seq_q, p.seq_k, p.head_dim = _abi.FCSA_BF16, 2, 8, 2, 4, 128, 64
    p.scale, p.shift = 8.0, 8.0
    for name, value in kw.items():
        setattr(p, name, value)
    return p


def test_abi_decode_varlen_rejects_bad_problems():
    """fcsa_decode_varlen validates through the library's own checks (no device needed to reject)."""
    from flash_cosine_sim_attention_b200 import _abi
    lib = _abi.load()
    t = _abi.FcsaTensor(16, 0, 0, 0)

    def call(p, cu=16, total=6, k=None, v=None):
        rc = lib.fcsa_decode_varlen(_abi.ref(p), cu, total, _abi.ref(t), _abi.ref(t), _abi.ref(t), 16, k, v, 1,
                                    _abi.ref(t), 16, 0, None)
        return rc, lib.fcsa_last_error()

    rc, msg = call(_problem(_abi, kv_heads=3))
    assert rc == _abi.FCSA_ERR_INVALID and b"kv_heads" in msg
    assert call(_problem(_abi, head_dim=96))[0] == _abi.FCSA_ERR_UNSUPPORTED
    rc, msg = call(_problem(_abi), cu=None)
    assert rc == _abi.FCSA_ERR_INVALID and b"null cu_seqlens_q" in msg
    rc, msg = call(_problem(_abi), cu=18)
    assert rc == _abi.FCSA_ERR_INVALID and b"4-byte aligned" in msg
    rc, msg = call(_problem(_abi), total=-1)
    assert rc == _abi.FCSA_ERR_INVALID and b"total_q -1 < 0" in msg
    rc, msg = call(_problem(_abi, seq_q=-1))
    assert rc == _abi.FCSA_ERR_INVALID and b"max_seqlen_q" in msg
    rc, msg = call(_problem(_abi, key_mask=16))
    assert rc == _abi.FCSA_ERR_UNSUPPORTED and b"key mask" in msg
    rc, msg = call(_problem(_abi, out_f32=1))
    assert rc == _abi.FCSA_ERR_UNSUPPORTED and b"out_f32" in msg
    rc, msg = call(_problem(_abi), k=_abi.ref(t))
    assert rc == _abi.FCSA_ERR_INVALID and b"both k_new and v_new" in msg
    # a problem that passes reaches the tensor checks: nothing is launched here
    null = _abi.FcsaTensor(None, 0, 0, 0)
    rc = lib.fcsa_decode_varlen(_abi.ref(_problem(_abi)), 16, 6, _abi.ref(null), _abi.ref(t), _abi.ref(t), 16, None,
                                None, 1, _abi.ref(t), 16, 0, None)
    assert rc == _abi.FCSA_ERR_INVALID and b"q: null tensor" in lib.fcsa_last_error()


def test_abi_decode_varlen_workspace_bytes():
    from flash_cosine_sim_attention_b200 import _abi
    lib = _abi.load()
    for bad in (_problem(_abi, kv_heads=3), _problem(_abi, seq_q=-1), _problem(_abi, head_dim=96),
                _problem(_abi, out_f32=1)):
        assert lib.fcsa_decode_varlen_workspace_bytes(_abi.ref(bad), 6) == 0
    assert lib.fcsa_decode_varlen_workspace_bytes(_abi.ref(_problem(_abi)), -1) == 0


def test_abi_symbols_exported_and_declared():
    from flash_cosine_sim_attention_b200 import _abi
    lib = _abi.load()
    for name in ("fcsa_decode_varlen", "fcsa_decode_varlen_workspace_bytes"):
        assert name in _abi.EXPORTED_SYMBOLS
        assert getattr(lib, name).argtypes is not None and getattr(lib, name).restype is not None
