# -*- coding: utf-8 -*-
"""The premise of the pruned query walk (csrc/trie.cu tree_get), checked on forests of the reference trie: whatever
sequence of put / stream_put / reset_input_freqs / squeeze the reference executes, every node's counts bound its
children's (`_put` adds along root paths, lookahead_cache.py:40-56; `_squeeze` halves top-down and pops whole subtrees,
:302-310; `_reset_input_freq` zeroes top-down, :326-333).  The forests are what the reference's own LookaheadCache held
at every checkpoint of three seeded streams (tests/golden/gen_count_bound_golden.py, a seeded sample of the trees);
the CUDA trie asserts the same on its own forests in tests/test_gpu_trie.py."""
import os

import numpy as np
import pytest

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'count_bound_forests.npz')


@pytest.mark.parametrize('seed,vocab,zipf', [(1, 12, False), (2, 3000, True), (3, 40, False)])
def test_reference_counts_bound_their_children(seed, vocab, zipf):
    g = np.load(GOLDEN)
    parents, freqs = g[f'parents_{seed}'], g[f'freqs_{seed}']
    assert int(g[f'checkpoints_{seed}']) == (30 if zipf else 6)
    assert len(parents) == len(freqs) and (parents < np.arange(len(parents))).all()   # parents come first
    child = parents >= 0
    assert child.sum() > 20 and (~child).sum() > 20
    # every (node, slot) count of the slots -1, 0, 1, 2 is at most its parent's
    assert int((freqs[child] > freqs[parents[child]]).sum()) == 0
