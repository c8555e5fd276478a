"""H100-native (sm_90a) fused cosine-similarity attention.

Same public names as the reference package's `__init__.py:1`
(flash_cosine_sim_attention, plain_cosine_sim_attention, l2norm_tensors, debug)."""
from .flash_cosine_sim_attention import (  # noqa: F401
    FlashCosineSimAttention,
    debug,
    flash_cosine_sim_attention,
    flash_cosine_sim_attention_cuda,
    flash_cosine_sim_attention_with_kv_cache,
    l2norm_tensors,
    plain_cosine_sim_attention,
    release_workspaces,
)
from .version import __version__  # noqa: F401
