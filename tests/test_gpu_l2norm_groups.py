"""GPU parity of the l2norm backward of dk that the backward kernel's epilogue applies (keys of their own per
head): group sizes of 1, 2 and 4 features, whose sums stay inside one lane or one lane pair of a key row's quad,
at both head dims.  The oracle and the tolerances are those of test_gpu_parity.py."""
import pytest
import torch

from test_gpu_parity import check, fcsa  # noqa: F401  (fcsa is a fixture)

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("dim_head,groups", [(64, 64), (64, 32), (128, 128), (128, 64), (128, 32)])
@pytest.mark.parametrize("causal", [False, True])
def test_narrow_l2norm_groups(fcsa, dim_head, groups, causal):
    # the shift is scale * groups; scale = 64 / groups holds it at 64, so exp(scale * q.k - shift) stays inside
    # the fp32 exponent range (q.k of `groups` unit groups has a spread of about sqrt(groups))
    check(fcsa, (1, 2, 200, dim_head), (1, 2, 200, dim_head), torch.bfloat16, seed=groups + dim_head,
          groups=groups, scale=64 / groups, causal=causal)
