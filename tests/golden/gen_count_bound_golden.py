# -*- coding: utf-8 -*-
"""Generates tests/golden/count_bound_forests.npz: the forests the REFERENCE's own trie (lookahead_cache.py) holds after
the seeded put / stream_put streams of tests/test_reference_count_bound.py, sampled at every checkpoint of the stream.
Needs the reference checkout on the path:
    PYTHONPATH=<reference>/lookahead python tests/golden/gen_count_bound_golden.py
Each stored node keeps its parent (-1 for a tree's top level) and its counts for the slots (-1, 0, 1, 2)."""
import os

import numpy as np

from lookahead.common.lookahead_cache import LookaheadCache

OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'count_bound_forests.npz')
CASES = [(1, 12, False), (2, 3000, True), (3, 40, False)]
IDXS = (-1, 0, 1, 2)
MAX_TREES_PER_CHECKPOINT = 6   # a seeded sample of the trees keeps the file small


def flatten(tree, parents, freqs):
    stack = [(node, -1) for node in tree.nodes.values()]
    while stack:
        node, parent = stack.pop()
        parents.append(parent)
        freqs.append([node.freqs.get(k, 0.0) for k in IDXS])
        me = len(parents) - 1
        stack.extend((child, me) for child in node.children.values())


def run(seed, vocab, zipf):
    rng = np.random.default_rng(seed)
    pick = np.random.default_rng(1000 + seed)

    def toks(k):
        if zipf:
            return np.clip(rng.zipf(1.3, size=k), 3, vocab - 1).tolist()
        return rng.integers(3, vocab, size=k).tolist()

    c = LookaheadCache(eos_ids=[2])
    c.max_node, c.max_output_node = 64, 24
    parents, freqs, checkpoints = [], [], 0
    for req in range(1500 if zipf else 300):
        idx = req % 3
        prompt = toks(int(rng.integers(4, 80)))
        c.put(prompt[1:], branch_length=9, final=False, mode='input', idx=idx)
        for _ in range(int(rng.integers(1, 10))):
            c.stream_put(toks(int(rng.integers(1, 9))), branch_length=9, final=False, mode='output', idx=idx)
        c.stream_put([], branch_length=9, final=True, mode='output', idx=idx)
        if req % 50 == 49:
            keys = sorted(c.mem.keys())
            for k in pick.permutation(keys)[:MAX_TREES_PER_CHECKPOINT]:
                flatten(c.mem[int(k)], parents, freqs)   # parent indices are global within the case
            checkpoints += 1
    return np.asarray(parents, np.int32), np.asarray(freqs, np.float32), checkpoints


def main():
    out = {}
    for seed, vocab, zipf in CASES:
        parents, freqs, checkpoints = run(seed, vocab, zipf)
        out[f'parents_{seed}'], out[f'freqs_{seed}'] = parents, freqs
        out[f'checkpoints_{seed}'] = np.int32(checkpoints)
        print(seed, vocab, zipf, 'nodes', len(parents), 'checkpoints', checkpoints)
    np.savez_compressed(OUT, **out)
    print(OUT, os.path.getsize(OUT), 'bytes')


if __name__ == '__main__':
    main()
