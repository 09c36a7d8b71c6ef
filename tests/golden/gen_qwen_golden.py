# -*- coding: utf-8 -*-
"""Generates tests/golden/qwen_rope_logn.npz from the reference's own Qwen (v1) code.  The reference module does not
import under current transformers, so the `RotaryEmbedding` class and the `logn_list` expression are taken out of
lookahead/models/qwen/modeling_qwen.py with `ast` and executed as they stand (einops required).  Run in the build
container only:

    python tests/golden/gen_qwen_golden.py

Records, for head dim 128, base 10000 and 1e6, ntk_alpha 1, 3, 7, 31: selected rows of the fp32 cos / sin tables (the
first half of each row; the second half repeats it), built at two cache lengths to show rows do not depend on the
length; and, for seq_length 64, 2048, 8192, the bf16 log-n values around and past the boundary.
tests/test_qwen_host.py compares models/qwen's host tables with them bit for bit."""
import ast
import importlib
import math
import os

import numpy as np
import torch
from torch import nn

HERE = os.path.dirname(os.path.abspath(__file__))
REF = os.environ.get('PIA_REFERENCE', '/root/reference/lookahead')
SRC = os.path.join(REF, 'lookahead', 'models', 'qwen', 'modeling_qwen.py')

ROWS = np.array([0, 1, 2, 63, 64, 65, 1000, 2047, 2048, 2049, 4095, 8191, 8192, 12345, 20000, 32766], dtype=np.int64)
DIM = 128
BASES = (10000, 1000000)
ALPHAS = (1, 3, 7, 31)
SEQ_LENGTHS = (64, 2048, 8192)


def _reference_pieces():
    tree = ast.parse(open(SRC).read())
    cls = next(n for n in tree.body if isinstance(n, ast.ClassDef) and n.name == 'RotaryEmbedding')
    ns = {'torch': torch, 'nn': nn, 'importlib': importlib, 'math': math}
    exec(compile(ast.Module(body=[cls], type_ignores=[]), SRC, 'exec'), ns)
    logn = None
    for node in ast.walk(tree):
        if isinstance(node, ast.Assign) and any(isinstance(t, ast.Name) and t.id == 'logn_list' for t in node.targets):
            logn = node.value
    assert logn is not None
    return ns['RotaryEmbedding'], logn


def main():
    RotaryEmbedding, logn_expr = _reference_pieces()
    out = {'rows': ROWS}
    for base in BASES:
        for alpha in ALPHAS:
            tables = []
            for length in (ROWS.max() + 1, 40000):   # update_rotary_pos_emb_cache builds max(2 * length, 16) rows
                re = RotaryEmbedding(DIM, base=base)
                cos, sin = re(int(length), ntk_alpha=alpha)
                cos, sin = cos[0, :, 0, :DIM // 2], sin[0, :, 0, :DIM // 2]
                tables.append((cos[ROWS].numpy().copy(), sin[ROWS].numpy().copy()))
            assert all(np.array_equal(a, b) for a, b in zip(tables[0], tables[1]))
            out[f'cos_b{base}_a{alpha}'], out[f'sin_b{base}_a{alpha}'] = tables[0]
    for seq_length in SEQ_LENGTHS:
        holder = type('Attn', (), {'seq_length': seq_length})()
        vals = eval(compile(ast.Expression(body=logn_expr), SRC, 'eval'), {'math': math, 'self': holder})
        t = torch.tensor(vals)[None, :, None, None].type_as(torch.zeros(1, dtype=torch.bfloat16))
        pos = np.unique(np.clip(np.concatenate([np.arange(seq_length - 4, seq_length + 6),
                                                np.array([0, 2 * seq_length - 1, 2 * seq_length, 32766])]), 0, 32766))
        out[f'logn_pos_s{seq_length}'] = pos
        out[f'logn_s{seq_length}'] = t[0, pos, 0, 0].view(torch.int16).numpy()   # bf16 bit patterns
    np.savez_compressed(os.path.join(HERE, 'qwen_rope_logn.npz'), **out)


if __name__ == '__main__':
    main()
