"""H100-native SE(3)-Transformer attention hot path -- drop-in for `se3_transformer_pytorch.SE3Transformer`.

    from se3_transformer_pytorch_b200 import SE3Transformer

Same constructor / forward / state_dict as the reference; the hot path runs in hand-written sm_90a CUDA kernels
(libse3b200.so, C ABI in include/se3b200.h).  CUDA only, forward only.
"""
from .model import SE3Transformer, CausalDecoder, PackedCausalDecoder, PagedCausalDecoder, DecoderCacheFull, ConvSE3, AttentionSE3, OneHeadedKVAttentionSE3, LinearSE3, NormSE3, Fiber
from .ops import get_basis

__all__ = ['SE3Transformer', 'CausalDecoder', 'PackedCausalDecoder', 'PagedCausalDecoder', 'DecoderCacheFull', 'ConvSE3', 'AttentionSE3', 'OneHeadedKVAttentionSE3', 'LinearSE3', 'NormSE3', 'Fiber', 'get_basis']
__version__ = '0.1.0'
