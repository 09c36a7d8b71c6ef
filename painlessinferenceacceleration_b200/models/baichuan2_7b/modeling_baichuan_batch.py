# -*- coding: utf-8 -*-
"""Baichuan2-7B with the BATCHED lookahead loop (reference: models/baichuan2_7b/modeling_baichuan_batch.py); the
request-slot runtime of common/pretrained_model_batch.py over the model of modeling_baichuan.py, as
models/llama/modeling_llama_batch.py does for Llama."""
from ...common.pretrained_model_batch import LookaheadPreTrainedModel as _BatchLoop
from .modeling_baichuan import BaichuanForCausalLM as _BaichuanForCausalLM


class BaichuanForCausalLM(_BatchLoop, _BaichuanForCausalLM):
    pass


__all__ = ['BaichuanForCausalLM']
