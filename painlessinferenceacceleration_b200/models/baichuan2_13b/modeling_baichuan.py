# -*- coding: utf-8 -*-
"""Baichuan2-13B (reference: models/baichuan2_13b/modeling_baichuan.py): ALiBi (:37-62, :398-402) at tree positions and
the L2-normalised lm_head (NormHead :504-521).  See models/baichuan/modeling_baichuan.py."""
from ..baichuan.modeling_baichuan import BaichuanBase


class BaichuanForCausalLM(BaichuanBase):
    alibi = True
    norm_head = True


__all__ = ['BaichuanForCausalLM']
