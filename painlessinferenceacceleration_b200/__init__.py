# -*- coding: utf-8 -*-
"""H100-native (sm_90a) draft -> verify -> accept hot loop of PIA LOOKAHEAD behind the reference's Python surface.

    from painlessinferenceacceleration_b200.common.lookahead_cache import LookaheadCache, Tree
    from painlessinferenceacceleration_b200.models.llama.modeling_llama import LlamaForCausalLM

Everything that computes runs in hand-written CUDA (libpia_b200.so, C ABI in include/pia_b200.h) or cuBLAS
GEMMs; there is no CPU fallback."""
__version__ = '0.1.0'
