# -*- coding: utf-8 -*-
"""Mistral with the lookahead patch (reference: models/mistral/modeling_mistral.py, patch :979-982, attention
:241-320, repeat_kv :183-192, rope :94-164).  Same decoder as Llama with grouped-query attention: the tree
attention kernel packs two query heads of one KV head into each UMMA M=128 tile (no repeat_kv copy), and - as on
the reference's lookahead branch - the sliding window is ignored (:979-982 vs :1016-1022)."""
import warnings

from ...common import ops
from ..llama.modeling_llama import LlamaForCausalLM


def warn_sliding_window(config, max_pos):
    """The reference's lookahead branch builds its rank-4 mask without the window (mistral/modeling_mistral.py:979-982;
    the sliding-window mask is only made on the non-lookahead branch, :1016-1022; SURVEY A.2-15), and so does the
    attention kernel here: say so instead of silently diverging from a sliding-window checkpoint once a context can
    outgrow the window."""
    window = getattr(config, 'sliding_window', None)
    if window is not None and max_pos > int(window) + 8:
        warnings.warn(f'sliding_window={window} is ignored on the lookahead path (as in the reference); contexts '
                      f'beyond it attend to the full prefix')


class MistralForCausalLM(LlamaForCausalLM):
    rmsnorm_rounding = ops.ROUND_TWICE   # weight * hidden_states.to(input_dtype) (mistral/modeling_mistral.py:90)

    def rope_tables(self, max_pos):
        warn_sliding_window(self.config, max_pos)
        return super().rope_tables(max_pos)
