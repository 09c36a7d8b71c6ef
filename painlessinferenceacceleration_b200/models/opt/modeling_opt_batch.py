# -*- coding: utf-8 -*-
"""OPT with the BATCHED lookahead loop (reference: models/opt/modeling_opt_batch.py); the request-slot runtime of
common/pretrained_model_batch.py over the model of modeling_opt.py, as models/llama/modeling_llama_batch.py does for
Llama."""
from ...common.pretrained_model_batch import LookaheadPreTrainedModel as _BatchLoop
from .modeling_opt import OPTForCausalLM as _OPTForCausalLM


class OPTForCausalLM(_BatchLoop, _OPTForCausalLM):
    def lookahead_generation(self, input_ids, *args, max_length=None, decoding_kwargs=None, **kwargs):
        """the batched loop, after refusing a max_length beyond max_position_embeddings (before any capture)"""
        self.check_max_length(max_length if max_length is not None
                              else int((decoding_kwargs or {}).get('max_length', 2048)))
        self.check_max_length(input_ids.shape[1])
        return super().lookahead_generation(input_ids, *args, max_length=max_length, decoding_kwargs=decoding_kwargs,
                                            **kwargs)


__all__ = ['OPTForCausalLM']
