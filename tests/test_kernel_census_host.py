"""CPU: the kernel instantiations libfcsa_b200.so contains, per family (tests/kernel_census.py reads them from the ELF
file).  The counts are a tripwire: an instantiation added or dropped must be accounted for here, and a new one must
get a row in tests/test_gpu_kernel_census.py, which launches and judges every kernel of the library."""
import collections
import os

import pytest

from flash_cosine_sim_attention_b200 import _abi
from kernel_census import FAMILIES, family, library_kernels, short_name

COUNTS = {"forward": 20, "backward": 68, "dQ": 16, "decode": 8, "combine": 4, "prep": 8, "dq finish": 8,
          "kv finish": 2, "varlen tail": 1, "row passes": 20}


@pytest.fixture(scope="module")
def kernels():
    if not os.path.exists(_abi.LIB_PATH):
        from flash_cosine_sim_attention_b200.build import build_library
        build_library()
    return library_kernels(_abi.LIB_PATH)


def test_short_names():
    assert short_name("void fcsa::k<__half, 64, true>(CUtensorMap_st, std::conditional<true, A, B>::type)") == \
        "fcsa::k<__half, 64, true>"
    assert short_name("fcsa::varlen_tail_kernel(fcsa::TailArgs)") == "fcsa::varlen_tail_kernel"
    assert family("fcsa::row_bwd_kernel<__half, float>") == "row passes"


def test_kernel_count_per_family(kernels):
    per = collections.Counter(family(k) for k in kernels)
    unknown = [k for k in kernels if family(k) is None]
    assert not unknown, f"kernels of no known family: {unknown}"
    print(f"{len(kernels)} kernels: " + ", ".join(f"{f} {per[f]}" for f in COUNTS))
    assert dict(per) == COUNTS
    assert len(kernels) == len(set(kernels)) == 155
    assert set(COUNTS) == set(FAMILIES.values())


def test_template_arguments_are_complete(kernels):
    """Each family is the full product of its template arguments (the dispatch's dtype x head-dim axes included)."""
    import itertools
    from kernel_census import bwd, combine, decode, dq, dq_finish, fwd, kv_finish, prep
    import torch
    TD = list(itertools.product((torch.bfloat16, torch.float16), (64, 128)))
    B = (False, True)
    want = {fwd(t, D, bias=True) for t, D in TD}
    want |= {fwd(t, D, varlen=vl, window=w) for t, D in TD for vl in B for w in B}
    want |= {bwd(t, D, bias=True) for t, D in TD}
    want |= {bwd(t, D, hl, vl, w, q) for t, D in TD for hl in B for vl in B for w in B for q in B}
    want |= {dq(t, D, vl, w) for t, D in TD for vl in B for w in B}
    want |= {decode(t, D, w) for t, D in TD for w in B} | {combine(t, D) for t, D in TD}
    want |= {prep(t, D, vl) for t, D in TD for vl in B} | {dq_finish(t, D, vl) for t, D in TD for vl in B}
    want |= {kv_finish(t) for t in (torch.bfloat16, torch.float16)}
    have = {k for k in kernels if family(k) not in ("row passes", "varlen tail")}
    assert have == want, (sorted(have - want), sorted(want - have))
