# -*- coding: utf-8 -*-
"""Qwen2 (HF model_type `qwen2`: Qwen1.5, Qwen2, Qwen2.5) with the lookahead patch (reference:
models/qwen2/modeling_qwen2.py, patch :997-1000 - the Llama one: position_ids = rowsum - 1, additive mask - q/k/v
with biases and o without :234-237).  The decoder is Llama's with biases on the fused QKV projection: fuse() stacks
them into one `qkv_bias` (the HF-named biases become views of it) and the projection is one addmm, the bias added in
fp32 before the single bf16 rounding as HF's F.linear does.  The weight-streaming GEMM has no bias epilogue, so the
QKV projection stays on cuBLAS (PIA_GEMM_SET=qkv is refused).  Query heads per KV head are often odd (28/4, 40/8):
the tree attention kernel packs them two per tile all the same, the last tile of each KV head holding one.
As on the reference's lookahead branch, the sliding window is ignored (:997-1000 builds the mask without one; the
window mask exists only on the non-lookahead branch, :1036-1043)."""
from ...common import ops
from ..llama.modeling_llama import LlamaDecoderLayer, LlamaForCausalLM, LlamaModel
from ..mistral.modeling_mistral import warn_sliding_window


class Qwen2DecoderLayer(LlamaDecoderLayer):
    qkv_bias = True


class Qwen2Model(LlamaModel):
    layer_cls = Qwen2DecoderLayer


class Qwen2ForCausalLM(LlamaForCausalLM):
    model_cls = Qwen2Model
    rmsnorm_rounding = ops.ROUND_TWICE   # weight * hidden_states.to(input_dtype) (qwen2/modeling_qwen2.py:96)

    def rope_tables(self, max_pos):
        # Qwen2 configs carry a `sliding_window` value even when the window is off: only use_sliding_window=True counts
        if getattr(self.config, 'use_sliding_window', False):
            warn_sliding_window(self.config, max_pos)
        return super().rope_tables(max_pos)
