# -*- coding: utf-8 -*-
"""Drop-in for /root/reference/flood/flood/utils/speculative.py: `Spec` (:6-20) and `Lookahead(Spec)` (:23-124), the
hash-table lookahead draft FLOOD's batcher drives (flood/utils/batch.py:484 lookahead_batching).  Same constructor,
same four methods, same tensors in and out; the Triton kernels of flood/ops/draft.py are replaced by the sm_90a
kernels of csrc/flood_draft.cu through the C ABI (include/pia_b200.h, pia_flood_*).  No CPU fallback."""
import math
import os

import torch

from .. import _lib as L


def _s():
    return torch.cuda.current_stream().cuda_stream


class Spec:
    """reference :6-20"""

    def __init__(*args, **kwargs):
        pass

    def proposal_draft(self, input_ids, **kwargs):
        raise NotImplementedError

    def update_state(self, input_ids, **kwargs):
        raise NotImplementedError

    def verify_draft(self, input_ids, next_ids, **kwargs):
        raise NotImplementedError

    def update_cache(self, src_idx, dst_idx, caches, **kwargs):
        raise NotImplementedError


def update_draft_table(tokens, freq_table, draft_table, table_size=2 ** 16, branch_length=8, branch_count=8,
                       vocab=128256, eos=0):
    """draft.py:168-204 (tokens: python list of ids)"""
    token_count = len(tokens)
    if token_count <= 3:
        return
    t = torch.tensor(list(tokens), device=draft_table.device, dtype=torch.int32)
    with torch.cuda.device(draft_table.device):
        L.check(L.load().pia_flood_update_draft_table(t.data_ptr(), token_count, freq_table.data_ptr(),
                                                      draft_table.data_ptr(), table_size, branch_length, branch_count,
                                                      vocab, _s()))


def retrieve_draft_table(tokens, freq_table, draft_table, table_size=2 ** 16, vocab=128256, branch_length=8,
                         branch_count=8, retrieve_count=8):
    """draft.py:352-402 (tokens: list of [token_id_0, token_id_1]) -> (output_tokens [bs, l], output_masks [bs, l, l]
    int8) with l = retrieve_count * branch_length"""
    batch_size = len(tokens)
    device = draft_table.device
    q = torch.tensor(tokens, device=device, dtype=torch.int32).view(batch_size, 2).contiguous()
    assert retrieve_count <= branch_count
    ln = retrieve_count * branch_length
    output_tokens = torch.zeros((batch_size, ln + 1), device=device, dtype=draft_table.dtype)
    output_masks = torch.tril(torch.ones((batch_size, ln, ln), device=device, dtype=torch.int8), diagonal=0)
    for j in range(1, retrieve_count):  # independent branches below the root (:377-382)
        output_masks[:, j * branch_length + 1:(j + 1) * branch_length + 1, 1:j * branch_length + 1] = 0
    with torch.cuda.device(device):
        L.check(L.load().pia_flood_retrieve_draft_table(q.data_ptr(), batch_size, freq_table.data_ptr(),
                                                        draft_table.data_ptr(), table_size, vocab, branch_length,
                                                        branch_count, retrieve_count, output_tokens.data_ptr(), _s()))
    return output_tokens[:, :-1].contiguous(), output_masks


def verify_draft(input_ids, next_ids, cache_offsets, masks, batch_size, branch_count, branch_length):
    """draft.py:491-543"""
    assert input_ids.size(0) == batch_size * branch_count * branch_length
    device = input_ids.device
    i32 = dict(device=device, dtype=torch.int32)
    ii, nn_, co = (input_ids.to(torch.int32).contiguous(), next_ids.to(torch.int32).contiguous(),
                   cache_offsets.to(torch.int32).contiguous())
    output_ids = torch.full((batch_size, branch_length + 1), -1, **i32)
    cache_src = torch.full((batch_size * branch_length,), -1, **i32)
    cache_dst = torch.full((batch_size * branch_length,), -1, **i32)
    with torch.cuda.device(device):
        L.check(L.load().pia_flood_verify_draft(ii.data_ptr(), nn_.data_ptr(), co.data_ptr(), batch_size, branch_count,
                                                branch_length, output_ids.data_ptr(), cache_src.data_ptr(),
                                                cache_dst.data_ptr(), _s()))
    dt = input_ids.dtype
    return output_ids.to(dt), cache_src.to(dt), cache_dst.to(dt)


def update_draft_cache(cache, src_indices, dst_indices):
    """draft.py:562-570: cache [rows, dim] (any dtype), rows src -> dst where src >= 0 and src != dst"""
    assert cache.is_contiguous()
    s, d = src_indices.to(torch.int32).contiguous(), dst_indices.to(torch.int32).contiguous()
    with torch.cuda.device(cache.device):
        L.check(L.load().pia_flood_update_draft_cache(cache.data_ptr(), cache.size(1) * cache.element_size() *
                                                      (cache[0, 0].numel() if cache.dim() > 2 else 1), s.data_ptr(),
                                                      d.data_ptr(), s.numel(), _s()))


class Lookahead(Spec):
    """reference :23-124"""

    def __init__(self, table_size=2 ** 20, branch_length=8, branch_count=32, vocab_size=128256,
                 device=torch.device('cuda:0'), tokenizer=None):
        assert 2 ** (int(round(math.log2(branch_length)))) == branch_length
        assert 2 ** (int(round(math.log2(branch_count)))) == branch_count
        self.table_size = table_size
        self.branch_length = branch_length
        self.branch_count = branch_count
        self.vocab_size = vocab_size
        self.tokenizer = tokenizer  # used for debug
        self.rank = int(os.environ.get('FLOOD_RANK', '0'))
        if self.rank == 0:
            self.freq_table = torch.zeros((table_size,), dtype=torch.float32, device=device)
            self.draft_table = torch.zeros((table_size, branch_length), dtype=torch.int32, device=device)
        else:
            self.freq_table = None
            self.draft_table = None

    def proposal_draft(self, input_ids, retrieve_count=4, **kwargs):
        return retrieve_draft_table(input_ids, self.freq_table, self.draft_table, table_size=self.table_size,
                                    vocab=self.vocab_size, branch_length=self.branch_length,
                                    branch_count=self.branch_count, retrieve_count=retrieve_count)

    def update_state(self, input_ids, **kwargs):
        update_draft_table(input_ids, self.freq_table, self.draft_table, table_size=self.table_size,
                           vocab=self.vocab_size, branch_length=self.branch_length, branch_count=self.branch_count)

    def verify_draft(self, input_ids, next_ids, **kwargs):
        meta = kwargs['batch_meta_info']
        bs = meta.batch_size
        cache_offsets = meta.cache_indices.view(bs, -1)[:, 0].contiguous()
        masks = None  # the reference does not support arbitrary masks here either (:89)
        return verify_draft(input_ids, next_ids, cache_offsets, masks, bs, meta.retrieve_count, self.branch_length)

    def update_cache(self, src_idx, dst_idx, caches, **kwargs):
        device = caches.caches[0].device
        if src_idx.device != device:
            src_idx = src_idx.to(device)
        if getattr(caches, 'fix_size_indices', None):
            raise NotImplementedError('fixed-size (linear-attention) draft caches (draft.py:574-660) are outside the '
                                      'lookahead hot path')
        for i in range(caches.num_layers):
            update_draft_cache(caches.caches[i], src_idx, dst_idx)
