"""CPU: the argument checks of flash_cosine_sim_attention_with_kv_cache(..., rolling=True) that need no device, the
rejections of fcsa_decode_rolling through the C ABI's return codes, and the transformer's rolling cache on the plain
(PyTorch) attention path."""
import pytest
import torch


def _dense(B=2, H=8, Hk=2, n=1, D=64, C=256):
    q = torch.zeros(B, H, n, D, dtype=torch.bfloat16)
    kc = torch.zeros(B, Hk, C, D, dtype=torch.bfloat16)
    sl = torch.zeros(B, dtype=torch.int32)
    k = torch.zeros(B, Hk, n, D, dtype=torch.bfloat16)
    return q, kc, sl, k


def _packed(B=2, H=8, Hk=2, total=5, D=64, C=256):
    q = torch.zeros(total, H, D, dtype=torch.bfloat16)
    kc = torch.zeros(B, Hk, C, D, dtype=torch.bfloat16)
    sl = torch.zeros(B, dtype=torch.int32)
    cu = torch.tensor([0, 2, total], dtype=torch.int32)
    k = torch.zeros(total, Hk, D, dtype=torch.bfloat16)
    return q, kc, sl, cu, k


def test_dense_rejections():
    from flash_cosine_sim_attention_b200 import flash_cosine_sim_attention_with_kv_cache as f
    q, kc, sl, k = _dense(n=4)
    with pytest.raises(ValueError, match="needs a window"):
        f(q, kc, kc, sl, k=k, v=k, rolling=True)
    with pytest.raises(ValueError, match="multiple of 128 rows, got 200"):
        f(q, kc[:, :, :200], kc[:, :, :200], sl, k=k, v=k, window=100, rolling=True)
    # C >= W + n - 1: 256 holds W = 253 with 4 new tokens, not W = 254
    with pytest.raises(ValueError, match="at least window \\+ n - 1 = 257 rows"):
        f(q, kc, kc, sl, k=k, v=k, window=254, rolling=True)
    with pytest.raises(ValueError, match="one row per query"):
        f(q, kc, kc, sl, k=k[:, :, :2], v=k[:, :, :2], window=100, rolling=True)
    with pytest.raises(TypeError, match="rolling must be a bool"):
        f(q, kc, kc, sl, window=100, rolling=1)
    # a problem that passes reaches the device check: no CPU path
    with pytest.raises(RuntimeError, match="CUDA tensors required"):
        f(q, kc, kc, sl, k=k, v=k, window=253, rolling=True)
    with pytest.raises(RuntimeError, match="CUDA tensors required"):
        f(q, kc, kc, sl, window=253, rolling=True)           # nothing appended: the same bound on the keys it sees


def test_packed_rejections():
    from flash_cosine_sim_attention_b200 import flash_cosine_sim_attention_with_kv_cache as f
    q, kc, sl, cu, k = _packed()
    with pytest.raises(ValueError, match="needs a window"):
        f(q, kc, kc, sl, k=k, v=k, cu_seqlens_q=cu, max_seqlen_q=3, rolling=True)
    with pytest.raises(ValueError, match="multiple of 128 rows, got 300"):
        f(q, kc.new_zeros(2, 2, 300, 64), kc.new_zeros(2, 2, 300, 64), sl, k=k, v=k, window=8, cu_seqlens_q=cu,
          max_seqlen_q=3, rolling=True)
    # n is max_seqlen_q in the packed form
    with pytest.raises(ValueError, match="at least window \\+ n - 1 = 265 rows"):
        f(q, kc, kc, sl, k=k, v=k, window=250, cu_seqlens_q=cu, max_seqlen_q=16, rolling=True)
    with pytest.raises(RuntimeError, match="CUDA tensors required"):
        f(q, kc, kc, sl, k=k, v=k, window=241, cu_seqlens_q=cu, max_seqlen_q=16, rolling=True)


def _problem(_abi, **kw):
    p = _abi.FcsaProblem()
    p.dtype, p.batch, p.heads, p.kv_heads, p.seq_q, p.seq_k, p.head_dim = _abi.FCSA_BF16, 2, 8, 2, 4, 256, 64
    p.scale, p.shift, p.causal, p.window = 8.0, 8.0, 1, 253
    for name, value in kw.items():
        setattr(p, name, value)
    return p


@pytest.mark.parametrize("packed", [False, True], ids=["dense", "packed"])
def test_abi_decode_rolling_rejects_bad_problems(packed):
    """fcsa_decode_rolling validates through the library's own checks (no device needed to reject)."""
    from flash_cosine_sim_attention_b200 import _abi
    lib = _abi.load()
    t = _abi.FcsaTensor(16, 0, 0, 0)

    def call(p, cu=16 if packed else None, total=6, k=None, v=None):
        rc = lib.fcsa_decode_rolling(_abi.ref(p), cu, total, _abi.ref(t), _abi.ref(t), _abi.ref(t), 16, k, v, 1,
                                     _abi.ref(t), 16, 0, None)
        return rc, lib.fcsa_last_error()

    rc, msg = call(_problem(_abi, window=0))
    assert rc == _abi.FCSA_ERR_INVALID and b"needs a window" in msg
    rc, msg = call(_problem(_abi, seq_k=200))
    assert rc == _abi.FCSA_ERR_INVALID and b"multiple of 128" in msg
    rc, msg = call(_problem(_abi, window=254))
    assert rc == _abi.FCSA_ERR_INVALID and b"cache rows 256 < window 254 + new queries 4 - 1" in msg
    rc, msg = call(_problem(_abi, kv_heads=3))
    assert rc == _abi.FCSA_ERR_INVALID and b"kv_heads" in msg
    assert call(_problem(_abi, head_dim=96))[0] == _abi.FCSA_ERR_UNSUPPORTED
    rc, msg = call(_problem(_abi, key_mask=16, causal=0))
    assert rc == _abi.FCSA_ERR_UNSUPPORTED and b"key mask" in msg
    rc, msg = call(_problem(_abi), k=_abi.ref(t))
    assert rc == _abi.FCSA_ERR_INVALID and b"both k_new and v_new" in msg
    if packed:
        rc, msg = call(_problem(_abi), cu=18)
        assert rc == _abi.FCSA_ERR_INVALID and b"4-byte aligned" in msg
        rc, msg = call(_problem(_abi), total=-1)
        assert rc == _abi.FCSA_ERR_INVALID and b"total_q -1 < 0" in msg
    # a problem that passes reaches the tensor checks: nothing is launched here
    null = _abi.FcsaTensor(None, 0, 0, 0)
    rc = lib.fcsa_decode_rolling(_abi.ref(_problem(_abi)), 16 if packed else None, 6, _abi.ref(null), _abi.ref(t),
                                 _abi.ref(t), 16, None, None, 1, _abi.ref(t), 16, 0, None)
    assert rc == _abi.FCSA_ERR_INVALID and b"q: null tensor" in lib.fcsa_last_error()


def test_abi_decode_rolling_workspace_bytes():
    from flash_cosine_sim_attention_b200 import _abi
    lib = _abi.load()
    for cu in (None, 16):
        for bad in (_problem(_abi, window=0), _problem(_abi, seq_k=200), _problem(_abi, window=254),
                    _problem(_abi, kv_heads=3), _problem(_abi, head_dim=96), _problem(_abi, out_f32=1)):
            assert lib.fcsa_decode_rolling_workspace_bytes(_abi.ref(bad), cu, 6) == 0
    assert lib.fcsa_decode_rolling_workspace_bytes(_abi.ref(_problem(_abi)), 16, -1) == 0
    assert lib.fcsa_decode_rolling_workspace_bytes(_abi.ref(_problem(_abi, seq_q=-1)), 16, 6) == 0


def test_abi_symbols_exported_and_declared():
    from flash_cosine_sim_attention_b200 import _abi
    lib = _abi.load()
    for name in ("fcsa_decode_rolling", "fcsa_decode_rolling_workspace_bytes"):
        assert name in _abi.EXPORTED_SYMBOLS
        assert getattr(lib, name).argtypes is not None and getattr(lib, name).restype is not None


# ---- the transformer's rolling cache on the plain attention path --------------------------------------------------
def _model(window, **kw):
    from flash_cosine_sim_attention_b200.transformer import CosineSimCausalTransformer
    torch.manual_seed(0)
    return CosineSimCausalTransformer(num_tokens=64, dim=32, max_seq_len=640, depth=2, heads=4, dim_head=8,
                                      kv_heads=2, pre_norm=True, window=window, **kw).eval()


def test_transformer_rolling_cache_plain_path():
    """Window 40: rings of round_up(39 + 128, 128) = 256 rows, prefill chunks of 256 - 40 + 1 = 217 tokens.  A 300-token
    prompt, then steps of 1 and 9 tokens past 2 C positions, give the full-length cache's and the full forward's
    logits."""
    from flash_cosine_sim_attention_b200.transformer import ROLLING_CHUNK, rolling_capacity
    assert ROLLING_CHUNK == 128 and rolling_capacity(40) == 256 and rolling_capacity(4096) == 4224
    m = _model(40)
    x = torch.randint(0, 64, (2, 550))
    with torch.no_grad():
        full = m(x)
        ring, flat = m.new_cache(rolling=True), m.new_cache()
        assert all(c.rolling and c.capacity == 256 for c in ring)
        steps_r, steps_f = [m(x[:, :300], cache=ring)], [m(x[:, :300], cache=flat)]
        i = 300
        while i < 550:
            n = 1 if i % 2 else 9
            steps_r.append(m(x[:, i:i + n], cache=ring))
            steps_f.append(m(x[:, i:i + n], cache=flat))
            i += n
    inc_r, inc_f = torch.cat(steps_r, 1), torch.cat(steps_f, 1)
    assert ring[0].k.shape[2] == 256 and ring[0].length == 550
    assert (inc_r - inc_f).abs().max() <= 1e-4 * inc_f.abs().max()
    assert (inc_r - full).abs().max() <= 1e-4 * full.abs().max()


def test_transformer_rolling_cache_needs_a_window():
    from flash_cosine_sim_attention_b200.transformer import KVCache
    m = _model(None)
    with pytest.raises(ValueError, match="windowed model"):
        m.new_cache(rolling=True)
    with pytest.raises(ValueError, match="windowed layer"), torch.no_grad():
        m(torch.zeros(1, 4, dtype=torch.long), cache=[KVCache(256, rolling=True) for _ in m.layers])
    with pytest.raises(ValueError, match="multiple of 128"):
        KVCache(200, rolling=True)
    with pytest.raises(ValueError, match="windowed model"), torch.no_grad():
        m.generate(torch.zeros(1, 4, dtype=torch.long), 2, kv_cache=True, rolling_cache=True)
    # the defaults are the full-length cache
    assert not any(c.rolling for c in m.new_cache()) and m.new_cache()[0].capacity == 640
