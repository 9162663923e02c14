"""Python surface of the hand-written sm_90a kernels (+ PyTorch fallbacks for CPU runs)."""
from ._native import HAS_CUDA_EXT, USE_NATIVE, native, use_native  # noqa: F401
from .attention_ops import (  # noqa: F401
    PAGED_BLOCK_MULTIPLE,
    attention_reference,
    attention_varlen_reference,
    attention_with_kv_cache,
    attention_with_kv_cache_reference,
    attention_with_kv_cache_varlen,
    attention_with_kv_cache_varlen_reference,
    cache_capacity,
    fused_attention,
    fused_attention_qkvpacked,
    fused_attention_supported,
    fused_attention_varlen,
    fused_attention_varlen_qkvpacked,
    fused_attention_varlen_supported,
    fused_head_dim_supported,
    kv_blocks_release,
    kv_blocks_reserve,
    kv_cache_append,
    kv_group,
    varlen_positions,
)
from .fused_ops import (  # noqa: F401
    bias_dropout_add_layer_norm,
    bias_gelu,
    embedding,
    gaussian_basis,
    gaussian_basis_reference,
    linear,
    softmax_cross_entropy,
    vocab_projection,
)
from .norm_ops import layer_norm, rms_norm  # noqa: F401
from .optim_ops import (  # noqa: F401
    ema_update_,
    fp32_to_bf16_sr,
    fused_adam,
    multi_tensor_l2norm,
    multi_tensor_scale_,
)
from .layout_ops import heads_to_pair, merge_heads, pair_tail, pair_to_heads, split_heads  # noqa: F401
from .rotary_ops import rotary_embedding, rotary_embedding_reference, rotary_inv_freq  # noqa: F401
from .softmax_ops import softmax_dropout, softmax_dropout_with_logits  # noqa: F401
