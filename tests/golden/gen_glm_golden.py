# -*- coding: utf-8 -*-
"""Generates tests/golden/loop_glm_bf16_rp11.npz: the reference's own loop code (tests/golden/ref_loop.py) around a
tiny Hugging Face GLM (model_type `glm`) in bf16 - 16 query heads over 2 KV heads, head dim 128, interleaved RoPE on
the first half of each head, non-zero q/k/v biases - with repetition_penalty=1.1, every request run twice so that the
second pass drafts the first pass's answer.  Records only this fixture.  Run in the build container only:

    python tests/golden/gen_glm_golden.py

tests/test_loop_golden.py and tests/test_gpu_loop_golden.py replay it like every other loop_*.npz."""
import os
import sys

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))

from tests.golden import gen_loop_golden  # noqa: E402
from tests.tiny_glm import glm_hf_model  # noqa: E402
from tests.tiny_models import prompts, tiny_hf_model  # noqa: E402


def _tiny_hf_model(family, **kw):
    """scenario() builds its model through tiny_models.tiny_hf_model, which knows the older families; glm comes from
    tests/tiny_glm.py"""
    return glm_hf_model('glm', 128, **kw) if family == 'glm' else tiny_hf_model(family, **kw)


def main():
    gen_loop_golden.tiny_hf_model = _tiny_hf_model
    V = 96
    gen_loop_golden.scenario('glm_bf16_rp11', 'glm', torch.bfloat16, 11, V,
                             [dict(prompt=p, max_new_tokens=36) for p in prompts(26, 3, 20, V)], repetition_penalty=1.1)


if __name__ == '__main__':
    main()
