# -*- coding: utf-8 -*-
"""Baichuan2-7B (reference: models/baichuan2_7b/modeling_baichuan.py): fp32 RoPE (:112-155) and the L2-normalised
lm_head (NormHead).  See models/baichuan/modeling_baichuan.py."""
from ..baichuan.modeling_baichuan import BaichuanBase


class BaichuanForCausalLM(BaichuanBase):
    norm_head = True
    rope_fp32 = True


__all__ = ['BaichuanForCausalLM']
