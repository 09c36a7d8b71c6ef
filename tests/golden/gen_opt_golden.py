# -*- coding: utf-8 -*-
"""Generates tests/golden/opt_tree_positions.npz from the reference's own OPT position embedding.  The
`OPTLearnedPositionalEmbedding` class is taken out of lookahead/models/opt/modeling_opt.py with `ast` and executed as
it stands, with a one-column table whose row r holds r, so that its output is the embedding row it read
(position + offset).  Run in the build container only:

    python tests/golden/gen_opt_golden.py

Records, as position ids (row read - offset):
  * the rank-4 (lookahead) branch, `sum(attention_mask, dim=3) - 1`, for trees of 64 and 128 nodes after prefixes of
    P columns of which the first pad are left padding (mask [1, 1, n, P + n]);
  * the 2-D (prefill) branch, `cumsum(attention_mask) * attention_mask - 1`, for prompts with and without left
    padding.
tests/test_opt_host.py restates the tree-position rule of pia_learned_pos_embed against them."""
import ast
import os

import numpy as np
import torch
from torch import nn

HERE = os.path.dirname(os.path.abspath(__file__))
REF = os.environ.get('PIA_REFERENCE', '/root/reference/lookahead')
SRC = os.path.join(REF, 'lookahead', 'models', 'opt', 'modeling_opt.py')

TREES = [(64, 0, 0), (64, 37, 0), (64, 37, 5), (128, 100, 9), (128, 0, 0)]   # (n, P, pad)
PROMPTS = [(20, 0), (20, 6), (70, 13)]                                       # (T, pad)


def _reference_class():
    tree = ast.parse(open(SRC).read())
    cls = next(n for n in tree.body if isinstance(n, ast.ClassDef) and n.name == 'OPTLearnedPositionalEmbedding')
    ns = {'torch': torch, 'nn': nn}
    exec(compile(ast.Module(body=[cls], type_ignores=[]), SRC, 'exec'), ns)
    return ns['OPTLearnedPositionalEmbedding']


def _tree_rows(rng, n):
    """ancestor bit rows of a random tree of n nodes: node i's parent is a random earlier node"""
    parent = [-1] + [int(rng.integers(max(0, i - 8), i)) for i in range(1, n)]
    rows = []
    for i in range(n):
        r, j = 0, i
        while j >= 0:
            r |= 1 << j
            j = parent[j]
        rows.append(r)
    return rows


def main():
    Emb = _reference_class()
    emb = Emb(512, 1)
    with torch.no_grad():
        emb.weight.copy_(torch.arange(emb.weight.shape[0], dtype=torch.float32)[:, None])
    off = emb.offset
    out = {'offset': np.array(off)}
    rng = np.random.default_rng(0)
    for k, (n, P, pad) in enumerate(TREES):
        rows = _tree_rows(rng, n)
        m = torch.zeros((1, 1, n, P + n), dtype=torch.long)
        m[..., pad:P] = 1
        for i, r in enumerate(rows):
            for j in range(n):
                if (r >> j) & 1:
                    m[0, 0, i, P + j] = 1
        pos = emb(m, P)[0, :, 0].long() - off
        words = np.array([[(r >> (64 * w)) & 0xFFFFFFFFFFFFFFFF for w in range(n // 64)] for r in rows],
                         dtype=np.uint64)
        out[f'tree{k}_meta'] = np.array([n, P, pad])
        out[f'tree{k}_rows'] = words.view(np.int64)
        out[f'tree{k}_pos'] = pos.numpy()
    for k, (T, pad) in enumerate(PROMPTS):
        am = torch.ones((1, T), dtype=torch.long)
        am[:, :pad] = 0
        out[f'prompt{k}_meta'] = np.array([T, pad])
        out[f'prompt{k}_pos'] = (emb(am, 0)[0, :, 0].long() - off).numpy()
    np.savez_compressed(os.path.join(HERE, 'opt_tree_positions.npz'), **out)


if __name__ == '__main__':
    main()
