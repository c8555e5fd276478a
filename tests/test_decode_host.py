"""CPU: the key/value-cache logic of the transformer on the plain attention (float64), the split rule of the decode
kernel (a Python mirror that the GPU tests tie to the kernel through its launch count), and the argument checks of
flash_cosine_sim_attention_with_kv_cache that need no device."""
import math

import pytest
import torch


def decode_split(items, cap, sms):
    """Key splits per work item (mirror of decode_split in csrc/decode_kernel.cuh): 1 when the work items fill the
    SMs, otherwise the fewest that do, at most the key tiles of the capacity."""
    if items >= sms:
        return 1
    return min(math.ceil(sms / items), math.ceil(cap / 128))


@pytest.mark.parametrize("items,cap,sms,want", [
    (132, 4096, 132, 1),          # the items alone fill the SMs
    (500, 128, 132, 1),
    (64, 4096, 132, 3),           # B 8 x kv_heads 8, one row block: 3 x 64 = 192 >= 132
    (2, 32768, 132, 66),          # B 1 x kv_heads 2
    (8, 8192, 132, 17),
    (32, 8192, 132, 5),
    (1, 256, 132, 2),             # capped by the 2 key tiles of the capacity
    (1, 129, 132, 2),
    (1, 100, 132, 1),
    (131, 4096, 132, 2),
])
def test_split_rule(items, cap, sms, want):
    s = decode_split(items, cap, sms)
    assert s == want
    assert s == 1 or items * s >= sms or s == math.ceil(cap / 128)


def _model(**kw):
    from flash_cosine_sim_attention_b200.transformer import CosineSimCausalTransformer
    torch.manual_seed(0)
    return CosineSimCausalTransformer(num_tokens=256, dim=128, max_seq_len=48, depth=2, heads=4, dim_head=32,
                                      **kw).double().eval()


@pytest.mark.parametrize("kw", [dict(), dict(kv_heads=2, attn_l2norm_groups=8, attn_scale=1),
                                dict(pre_norm=True, kv_heads=1)])
def test_incremental_logits_equal_full_forward(kw):
    m = _model(**kw)
    x = torch.randint(0, 256, (2, 48))
    with torch.no_grad():
        full = m(x)
        cache = m.new_cache()
        parts = [m(x[:, :7], cache=cache), m(x[:, 7:9], cache=cache)]
        parts += [m(x[:, i:i + 1], cache=cache) for i in range(9, 48)]
    inc = torch.cat(parts, 1)
    assert cache[0].length == 48 and cache[1].seqlens.tolist() == [48, 48]
    assert (inc - full).abs().max().item() <= 1e-10
    with pytest.raises(ValueError, match="capacity"):
        m(x[:, :1], cache=cache)


def test_generate_with_cache_matches_without_past_max_seq_len():
    """Same sampling seed, with and without the cache: identical tokens, also after the window starts sliding."""
    m = _model(kv_heads=2, attn_l2norm_groups=8)
    start = torch.randint(0, 256, (2, 40))
    torch.manual_seed(5)
    a = m.generate(start, 20)
    torch.manual_seed(5)
    b = m.generate(start, 20, kv_cache=True)
    assert a.shape == (2, 20) and torch.equal(a, b)


def test_length_errors_name_their_cause():
    m = _model()
    with torch.no_grad(), pytest.raises(ValueError, match="exceed max_seq_len 48"):
        m(torch.randint(0, 256, (1, 49)))
    with torch.no_grad(), pytest.raises(ValueError, match="cache full"):
        m(torch.randint(0, 256, (1, 49)), cache=m.new_cache())


def test_cache_rejects_attention_keywords_it_would_drop():
    """A keyword the uncached CUDA path hands flash_cosine_sim_attention must not be dropped silently with a cache."""
    from flash_cosine_sim_attention_b200.transformer import CosineSimCausalTransformer
    m = CosineSimCausalTransformer(num_tokens=256, dim=64, max_seq_len=16, depth=1, heads=2, dim_head=32,
                                   use_cuda_kernel=True, attn_bias_batch_dim=True).eval()
    with torch.no_grad(), pytest.raises(NotImplementedError, match="attn_bias_batch_dim"):
        m(torch.randint(0, 256, (1, 3)), cache=m.new_cache())


def test_cache_rejects_non_cosine_sim_attention():
    m = _model(non_cosine_sim_attn=True)
    with torch.no_grad(), pytest.raises(NotImplementedError, match="cosine-sim"):
        m(torch.randint(0, 256, (1, 3)), cache=m.new_cache())


def test_with_kv_cache_argument_checks():
    from flash_cosine_sim_attention_b200 import flash_cosine_sim_attention_with_kv_cache as f
    q = torch.zeros(2, 8, 1, 64, dtype=torch.bfloat16)
    kc = torch.zeros(2, 2, 128, 64, dtype=torch.bfloat16)
    sl = torch.zeros(2, dtype=torch.int32)
    with pytest.raises(NotImplementedError, match="attn_bias"):
        f(q, kc, kc, sl, attn_bias=torch.zeros(8, 1, 128))
    with pytest.raises(NotImplementedError, match="mask"):
        f(q, kc, kc, sl, mask=torch.ones(2, 128, dtype=torch.bool))
    with pytest.raises(ValueError, match="merged"):
        f(q[:, 0], kc[:, 0], kc[:, 0], sl)
    with pytest.raises(ValueError, match="both k and v"):
        f(q, kc, kc, sl, k=kc[:, :, :1])
    with pytest.raises(RuntimeError, match="no autograd"):
        f(q.clone().requires_grad_(), kc, kc, sl)
    with pytest.raises(TypeError, match="float32"):
        f(q.float(), kc.float(), kc.float(), sl)
    with pytest.raises(NotImplementedError, match="head_dim 96"):
        f(torch.zeros(2, 8, 1, 96, dtype=torch.bfloat16), torch.zeros(2, 2, 8, 96, dtype=torch.bfloat16),
          torch.zeros(2, 2, 8, 96, dtype=torch.bfloat16), sl)
    with pytest.raises(ValueError, match="kv_heads"):
        f(q[:, :6], torch.zeros(2, 4, 8, 64, dtype=torch.bfloat16), torch.zeros(2, 4, 8, 64, dtype=torch.bfloat16), sl)
    with pytest.raises(TypeError, match="int32"):
        f(q, kc, kc, sl.long())
    with pytest.raises(ValueError, match="contiguous"):
        f(q, kc, kc, torch.tensor([3], dtype=torch.int32).expand(2))     # read as a dense array by the kernels
    with pytest.raises(ValueError, match="groups"):
        f(q, kc, kc, sl, groups=3)
    with pytest.raises(RuntimeError, match="CUDA"):
        f(q, kc, kc, sl)                         # CPU tensors: no CPU path


def test_abi_decode_rejects_bad_problems():
    """fcsa_decode validates through the library's own checks (no device needed to reject)."""
    from flash_cosine_sim_attention_b200 import _abi
    lib = _abi.load()
    p = _abi.FcsaProblem()
    p.dtype, p.batch, p.heads, p.kv_heads, p.seq_q, p.seq_k, p.head_dim = _abi.FCSA_BF16, 1, 8, 3, 1, 128, 64
    t = _abi.FcsaTensor(16, 0, 0, 0)
    r = lib.fcsa_decode(_abi.ref(p), _abi.ref(t), _abi.ref(t), _abi.ref(t), 16, None, None, 0, 1, _abi.ref(t), 16, 0,
                        None)
    assert r == _abi.FCSA_ERR_INVALID and b"kv_heads" in lib.fcsa_last_error()
    p.kv_heads, p.head_dim = 2, 96
    assert lib.fcsa_decode(_abi.ref(p), _abi.ref(t), _abi.ref(t), _abi.ref(t), 16, None, None, 0, 1, _abi.ref(t), 16,
                           0, None) == _abi.FCSA_ERR_UNSUPPORTED
    p.head_dim = 64
    assert lib.fcsa_decode(_abi.ref(p), _abi.ref(t), _abi.ref(t), _abi.ref(t), 16, None, None, -1, 1, _abi.ref(t), 16,
                           0, None) == _abi.FCSA_ERR_INVALID
    assert lib.fcsa_decode_workspace_bytes(_abi.ref(p), -1) == 0
