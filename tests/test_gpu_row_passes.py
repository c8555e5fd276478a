"""GPU parity of the row passes around the attention kernels - the grouped l2norm of `l2norm_tensors`, the float32
cast of q, k (and its plain scaled cast of v) with their backwards, and the in-place l2norm backward of dk when keys
are shared by several query heads - against the float64 oracle, with the tolerances of test_gpu_parity.py.  Row
counts are not multiples of the rows a block covers, so every block shape has a partial tail."""
import numpy as np
import pytest
import torch

from oracle import cosine_sim_attention_oracle as oracle
from test_gpu_parity import TOL_GRAD, TOL_OUT, check, fcsa, rel_err  # noqa: F401  (fcsa is a fixture)

pytestmark = pytest.mark.gpu

DTYPES = [torch.float16, torch.bfloat16]


def _l2norm_round_trip(fcsa, x, dy, groups):
    xd = x.cuda().requires_grad_()
    (y,) = fcsa.l2norm_tensors(xd, groups=groups)
    y.backward(dy.cuda())
    x64, dy64 = x.float().numpy(), dy.float().numpy()
    assert rel_err(y, oracle.l2norm(x64, groups)[0]) <= TOL_OUT[x.dtype]
    # the kernel differentiates through the ROUNDED y it stored, like autograd on 16-bit tensors
    assert rel_err(xd.grad, oracle.l2norm_backward(dy64, x64, groups)) <= TOL_GRAD[x.dtype]


@pytest.mark.parametrize("group_size", [1, 2, 4, 8, 16, None])
@pytest.mark.parametrize("dim_head", [32, 128, 256])
@pytest.mark.parametrize("dtype", DTYPES)
def test_l2norm_tensors_group_sizes(fcsa, dim_head, group_size, dtype):
    g = torch.Generator().manual_seed(dim_head + (group_size or 0))
    x, dy = (torch.randn(2, 3, 77, dim_head, generator=g).to(dtype) for _ in range(2))
    _l2norm_round_trip(fcsa, x, dy, dim_head // group_size if group_size else 1)


@pytest.mark.parametrize("dtype", DTYPES)
def test_l2norm_tensors_strided_input(fcsa, dtype):
    g = torch.Generator().manual_seed(5)
    x, dy = (torch.randn(2, 77, 3, 64, generator=g).to(dtype).transpose(1, 2) for _ in range(2))
    assert not x.is_contiguous()
    _l2norm_round_trip(fcsa, x, dy, 4)


@pytest.mark.parametrize("group_size", [1, 2, 4, None])
@pytest.mark.parametrize("dim_head", [16, 64])
@pytest.mark.parametrize("half", DTYPES)
def test_float32_cast_group_sizes(fcsa, dim_head, group_size, half):
    from flash_cosine_sim_attention_b200.flash_cosine_sim_attention import _ext
    groups = dim_head // group_size if group_size else 1
    g = torch.Generator().manual_seed(dim_head + (group_size or 0))
    x, dy = (torch.randn(2, 3, 77, dim_head, generator=g) for _ in range(2))
    y, rnorm = _ext().f32_cast(x.cuda(), half == torch.bfloat16, groups, None, False, dim_head)
    assert y.dtype == half
    assert rel_err(y, oracle.l2norm(x.numpy(), groups)[0]) <= TOL_OUT[half]
    dx = _ext().f32_cast_backward(dy.cuda(), y, rnorm, groups, None, False, dim_head)
    assert dx.dtype == torch.float32
    assert rel_err(dx, oracle.l2norm_backward(dy.numpy(), x.numpy(), groups)) <= TOL_GRAD[half]


@pytest.mark.parametrize("reciprocal", [False, True])
def test_float32_plain_scaled_cast(fcsa, reciprocal):
    """groups = 0: y = x * m and dx = dy * m, with m = *mul or 1 / *mul read on the device; padded features stay 0."""
    from flash_cosine_sim_attention_b200.flash_cosine_sim_attention import _ext
    g = torch.Generator().manual_seed(6)
    x, dy = (torch.randn(2, 3, 77, 32, generator=g) for _ in range(2))
    mul = torch.tensor([4.0], device="cuda")
    m = 0.25 if reciprocal else 4.0
    y, _ = _ext().f32_cast(x.cuda(), False, 0, mul, reciprocal, 64)
    assert y.shape[-1] == 64 and not y[..., 32:].any()
    assert rel_err(y[..., :32], x.double().numpy() * m) <= TOL_OUT[torch.float16]
    dx = _ext().f32_cast_backward(dy.cuda(), None, None, 0, mul, reciprocal, 32)
    assert np.array_equal(dx.cpu().numpy(), dy.numpy() * np.float32(m))


@pytest.mark.parametrize("groups", [2, 4])
@pytest.mark.parametrize("dtype", DTYPES)
def test_shared_keys_l2norm_backward_pass(fcsa, dtype, groups):
    """Keys/values shared by all heads: dk is summed over the heads first and its l2norm backward runs as a pass of
    its own, in place on dk."""
    check(fcsa, (2, 4, 77, 64), (2, 77, 64), dtype, seed=groups, groups=groups, scale=4, causal=True)
