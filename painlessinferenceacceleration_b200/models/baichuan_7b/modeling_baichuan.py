# -*- coding: utf-8 -*-
"""Baichuan-7B (reference: models/baichuan_7b/modeling_baichuan.py): Llama with a fused W_pack projection and Llama's
bf16 RoPE (:94-141).  See models/baichuan/modeling_baichuan.py."""
from ..baichuan.modeling_baichuan import BaichuanBase


class BaiChuanForCausalLM(BaichuanBase):
    pass


__all__ = ['BaiChuanForCausalLM']
