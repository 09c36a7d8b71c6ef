# -*- coding: utf-8 -*-
"""Baichuan-13B (reference: models/baichuan_13b/modeling_baichuan.py): ALiBi instead of RoPE (slopes :25-36, attention
:146-157), taken at tree positions.  See models/baichuan/modeling_baichuan.py."""
from ..baichuan.modeling_baichuan import BaichuanBase


class BaichuanForCausalLM(BaichuanBase):
    alibi = True


__all__ = ['BaichuanForCausalLM']
