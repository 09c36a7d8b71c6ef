# -*- coding: utf-8 -*-
"""Batched LOOKAHEAD loop, H100-native: the reference's
/root/reference/lookahead/lookahead/common/pretrained_model_batch.py (lookahead_prepare_inputs_for_generation
:664-759 with LookaheadCache.bat_get lookahead_cache.py:519-561, _lookahead_update_model_kwargs_for_generation
:767-935, _early_stop :937-980, _update_cache :982-989, lookahead_generation :1002-1330) and the cursor-addressed
preallocated KV cache of models/llama/modeling_llama_batch.py:375-405.

Every request of the batch is a request SLOT of the runtime (include/pia_b200.h pia_slots_t): it owns a share of the
64 draft rows of the shared activation buffers, its own token sequence, cursor, left padding and KV cache.
The share: the reference loop hands bat_get `decoding_length // active` (:713) and bat_get divides by the batch size
AGAIN (lookahead_cache.py:534), so a request drafts decoding_length // active // active nodes (64 -> 16 at 2 requests,
4 at 4, 1 - i.e. no draft at all - at 8).  That is reproduced by default (drafts, dls and edls are parity-exact with
the reference); decoding_kwargs['batch_share'] = 'rows' gives every request decoding_length // active rows instead,
which is what :713 evidently intended and what fills the 64 rows of a verify step.  One decode step = ONE CUDA graph over all active slots:

    batched trie get (one query row per slot, request idx per row)            bat_get, lookahead_cache.py:519-561
    embed -> L x [norm, qkv GEMM, rope + KV append at each slot's cursor, tree attention per slot (gridDim.z), ...]
    lm_head -> per-slot arg-max + accept walk bounded by max_length (:862) -> per-slot in-place KV compaction (:986-989)
    -> per-slot stream_put (:1243-1248) -> one pinned record

so the weight stream (13.5 GB for Llama-2-7B) is read once for all requests of the step.  When requests finish they
leave the batch like the reference's _early_stop: the remaining slots are compacted to the front (state rows and KV
caches are copied on the device) and the step graph of the new active count is used."""
import time

import numpy as np
import torch

from . import ops
from .lookahead_cache import LookaheadCache
from .lookahead_generation_utils import GenerationMode, LookaheadDecoderOnlyOutput
from .pretrained_model import REC, warn_trie_errors
from .pretrained_model import LookaheadPreTrainedModel as _Base


class LookaheadPreTrainedModel(_Base):
    _batch_generation = True

    def _capture_batch_step(self, rt, trie, k, share, bl, mql, tmode, kind, accept, sample=False):
        """one decode step over the k active slots (dense: slots 0..k-1), `share` draft rows each"""
        W = rt.max_nodes // 64
        rows = k * share
        draft = dict(ids=rt.ids[:rows].view(k, share), mask=rt.mask[:rows].view(k, share, W), n=rt.n, sizes=rt.sizes,
                     nsizes=rt.nsizes, status=rt.status)
        slots = rt.decode_slots(k, share) if k > 1 else ops.Slots(rt.n, rt.prefix_len, rt.pad, share, 0, batch=1)
        n_rows = torch.full((1,), rows, dtype=torch.int32, device=rt.device)
        db = rt.decode_bufs
        min_out = max(share // 2, 1)  # bat_get, lookahead_cache.py:530

        def step():
            trie.get_device(rt.seq, rt.seq_len, share, bl, max_query_length=mql, min_input_size=0,
                            min_output_size=min_out, mode=tmode, idx=0, kind=kind, max_seq_length=0, out=draft,
                            batch=k, d_idx=rt.trie_idx)
            saved = db.slots, db.n_total
            db.slots, db.n_total = slots, n_rows
            try:
                self._verify_layers(rt)
            finally:
                db.slots, db.n_total = saved
            accept.run(rt.logits, rt.ids, rt.mask, rt.n, rt.seq, rt.seq_len, rt.acc_tokens, rt.acc_count, rt.acc_nodes,
                       rt.prefix_len, rt.finished, batch=k, rows_per_slot=share, max_length=rt.max_length,
                       rng=rt.rng if sample else None)
            ops.kv_compact(rt.k_cache, rt.v_cache, rt.acc_nodes, rt.acc_count, rt.prefix_len, batch=k)
            for s in range(k):  # :1243-1248; the request idx of a slot is read on the device
                trie.stream_put_device(rt.acc_tokens[s], rt.max_nodes, rt.acc_count[s:s + 1],
                                       branch_length=self._put_bl, final=False, idx=0, d_idx=rt.trie_idx[s:s + 1])
            trie.copy_error_flags_device(rt.trie_err)
            rt.record[:k, 0] = rt.acc_count[:k]
            rt.record[:k, 1] = rt.finished[:k]
            rt.record[:k, 2] = rt.n[:k]
            rt.record[:k, 3] = rt.status[:k]
            rt.record[:k, 4] = rt.trie_err
            rt.record[:k, REC:] = rt.acc_tokens[:k]
            rt.record_host[0].copy_(rt.record, non_blocking=True)

        g = torch.cuda.CUDAGraph()
        l0 = ops.launch_count()
        with torch.cuda.graph(g):
            step()
        rt.kernels_per_graph = ops.launch_count() - l0
        return dict(graphs=[g], keep=(trie, accept, slots, n_rows, draft))

    @torch.no_grad()
    def lookahead_generation(self, input_ids, logits_processor=None, stopping_criteria=None, max_length=None,
                             pad_token_id=None, eos_token_id=None, output_attentions=None, output_hidden_states=None,
                             output_scores=None, return_dict_in_generate=None, synced_gpus=False, streamer=None,
                             attention_mask=None, decoding_kwargs=None, repetition_penalty=1.0, **model_kwargs):
        dev = self.device
        torch.cuda.set_device(dev)
        bs, prompt_len = input_ids.shape
        decoding_kwargs = decoding_kwargs if decoding_kwargs is not None else {}
        if isinstance(eos_token_id, int):
            eos_token_id = [eos_token_id]
        assert decoding_kwargs.get('generation_mode', GenerationMode.LOOKAHEAD_GENERATION) == \
            GenerationMode.LOOKAHEAD_GENERATION and decoding_kwargs.get('use_lookahead', True), \
            'the batched loop is the lookahead loop (pretrained_model_batch.py:1002)'
        dl = int(decoding_kwargs.get('decoding_length', 64))
        bl = int(decoding_kwargs.get('branch_length', 8))
        dmode = decoding_kwargs.get('decoding_mode', 'hier')
        if dmode in ('hier', 'par', 'one'):
            dmode = dmode + '_mix'  # :710-711
        fmt, tmode = dmode.split('_')
        assert fmt in ('hier', 'one'), 'bat_get drafts are hier or one (lookahead_cache.py:521)'
        assert dl <= 64 and bl <= 32 and bs <= dl, 'decoding_length <= 64 rows shared by <= decoding_length requests'
        if max_length is None:
            max_length = int(decoding_kwargs.get('max_length', 2048))
        if pad_token_id is None:
            pad_token_id = int(decoding_kwargs.get('pad', 2))
        max_nodes = 64
        max_seq = max_length + dl + 1
        rt = self._runtime(max_seq, max_nodes, n_slots=bs)
        S = rt.n_slots

        if not hasattr(self, 'lookahead_cache') or self.lookahead_cache is None:
            self.lookahead_cache = LookaheadCache(device=dev, vocab_capacity=max(self.geometry()['vocab'], 1024),
                                                  n_input_slots=max(bs, 8))
        trie = self.lookahead_cache
        assert trie._t.cfg.n_input_slots >= bs, f'the LookaheadCache was built for {trie._t.cfg.n_input_slots} request slots'
        trie.eos_ids = eos_token_id
        trie.stop_words = decoding_kwargs.get('stop_words', {})
        decoding_kwargs.update({'eos': eos_token_id[0] if eos_token_id is not None else 2, 'edls': [], 'dls': [],
                                'fts': [], 'qts': [], 'pad': pad_token_id})
        decoding_kwargs['max_length'] = max_length
        decoding_kwargs['decoding_max_length'] = max_seq
        self._put_bl = bl + 1

        ts = time.time()
        ids32 = input_ids.to(device=dev, dtype=torch.int32)
        pads = [0] * bs
        if attention_mask is not None:
            assert attention_mask.dim() == 2, 'the batched loop takes a [bs, src_len] 0/1 mask (left padding)'
            am = attention_mask.to('cpu') != 0
            for b in range(bs):
                nz = torch.nonzero(am[b])
                pads[b] = int(nz[0]) if nz.numel() else 0
        rt.seq[:bs, :prompt_len] = ids32
        rt.finished.zero_()
        rt.max_length.fill_(max_length)
        rt.pad[:bs] = torch.tensor(pads, dtype=torch.int32).to(dev)
        rt.trie_idx.copy_(torch.arange(S, dtype=torch.int32))
        for i in range(bs):  # :1203-1206  (ids[1:-1])
            trie.put_device(rt.seq[i, 1:], max(prompt_len - 2, 0), None, branch_length=bl + 1, final=False, mode='input',
                            idx=i)
        akey = ('batch', float(repetition_penalty), tuple(eos_token_id or ()), max_nodes)
        accept = rt.accepts.get(akey)
        if accept is None:
            accept = ops.Accept(self.geometry()['vocab'], max_nodes, repetition_penalty, eos_token_id, max_length, dev,
                                bound_walk=True)
            rt.accepts[akey] = accept

        # prefill (:781-808): every request through the chain-chunk prefill into its own cache, then one batched
        # arg-max of the last prompt rows
        sample = bool(decoding_kwargs.get('do_sample', False))  # :796-798, :821-823, :871-873
        if sample:
            rt.rng.copy_(torch.tensor([torch.initial_seed() & 0x7FFFFFFF, rt.replays & 0x7FFFFFFF], dtype=torch.int32))
        share_mode = decoding_kwargs.get('batch_share', 'reference')
        assert share_mode in ('reference', 'rows')

        def rows_of(k):
            sub = max(dl // k, 1)                        # sub_decoding_length (:713)
            if share_mode == 'reference':
                sub = sub // k                           # bat_get divides once more (lookahead_cache.py:534)
            assert sub >= 1, f'decoding_length {dl} leaves no draft row for {k} requests'
            return sub

        share = rows_of(bs)
        for b in range(bs):
            rt.pad_host = pads[b]
            self._prefill_logits(rt, prompt_len, slot=b, row=b * share)
            rt.ids[b * share:b * share + 1] = rt.seq[b, prompt_len - 1:prompt_len]
            rt.mask[b * share:b * share + 1] = rt.chain[0:1]
        rt.n[:bs].fill_(1)
        rt.seq_len[:bs].fill_(prompt_len)
        rt.prefix_len[:bs].fill_(prompt_len)
        accept.run(rt.logits, rt.ids, rt.mask, rt.n, rt.seq, rt.seq_len, rt.acc_tokens, rt.acc_count, rt.acc_nodes,
                   rt.prefix_len, rt.finished, batch=bs, rows_per_slot=share, max_length=rt.max_length,
                   rng=rt.rng if sample else None)
        rt.prefix_len[:bs].fill_(prompt_len)
        first = rt.acc_tokens[:bs, 0].tolist()
        fin = rt.finished[:bs].tolist()
        seqs = [[t] for t in first]                     # generated tokens per request
        decoding_kwargs['dls'].extend([1] * bs)
        decoding_kwargs['edls'].extend([1] * bs)
        if streamer is not None:
            streamer.put(np.array([first[0]]))
        for b in range(bs):                              # :1243-1248 after the prefill step
            trie.stream_put_device(rt.seq[b, prompt_len:], 1, None, branch_length=bl + 1, final=False, idx=b)
        active = [b for b in range(bs) if not fin[b]]    # batch_indices (:1213), dense slot s <-> request active[s]
        if len(active) != bs:
            self._compact_slots(rt, list(range(bs)), active)
        te = time.time()
        decoding_kwargs['fts'].append(te - ts)
        ts = te

        kind = 'hier' if fmt == 'hier' else 'one'
        stream = torch.cuda.current_stream()
        while active:
            k = len(active)
            share = rows_of(k)
            key = ('batch', k, share, bl, tmode, kind, akey, id(trie._t), sample)
            ent = self._graph_entry(rt, key, lambda: self._capture_batch_step(rt, trie, k, share, bl, 2, tmode, kind,
                                                                             accept, sample))
            ent['graphs'][0].replay()
            rt.replays += 1
            stream.synchronize()
            rec = rt.record_host[0][:k].numpy()
            widest = int(rec[:, 2].max())                # rows are padded to the longest draft (bat_get :552-560)
            still = []
            for s in range(k):
                count, f, status = int(rec[s, 0]), int(rec[s, 1]), int(rec[s, 3])
                if status != 0:
                    from .. import _lib as L
                    L.check(status)
                if int(rec[s, 4]) != 0 and not getattr(trie, '_warned_pool', False):
                    trie._warned_pool = True
                    warn_trie_errors(int(rec[s, 4]))
                toks = rec[s, REC:REC + count].tolist()
                seqs[active[s]].extend(toks)
                decoding_kwargs['dls'].append(widest)
                decoding_kwargs['edls'].append(count)
                if not f:
                    still.append(s)
                if streamer is not None and s == 0:
                    streamer.put(np.array(toks))
            decoding_kwargs['qts'].append(0.0)
            if len(still) != k:                          # _early_stop (:937-980)
                new_active = [active[s] for s in still]
                if new_active:
                    self._compact_slots(rt, active, new_active)
                active = new_active
            te = time.time()
            decoding_kwargs['fts'].append(te - ts)
            ts = te
        for i in range(bs):                              # :1287-1289
            trie.stream_put([], branch_length=bl + 1, final=True, mode='output', idx=i)
        if rt.replays - rt.last_compact_check >= 2048:   # reclaim squeezed trie storage if a pool fills up
            rt.last_compact_check = rt.replays
            trie.maybe_compact()
        if streamer is not None:
            streamer.end()
        width = prompt_len + max(len(x) for x in seqs)
        out_ids = torch.full((bs, width), int(pad_token_id), dtype=input_ids.dtype, device=dev)
        out_ids[:, :prompt_len] = input_ids.to(dev)
        for b in range(bs):
            out_ids[b, prompt_len:prompt_len + len(seqs[b])] = torch.tensor(seqs[b], dtype=input_ids.dtype, device=dev)
        if return_dict_in_generate:
            kw = {k_: decoding_kwargs[k_] for k_ in ('dls', 'edls', 'fts', 'qts')}
            kw['lengths'] = [prompt_len + len(x) for x in seqs]
            return LookaheadDecoderOnlyOutput(sequences=out_ids, scores=() if output_scores else None, kwargs=kw)
        return out_ids

    @staticmethod
    def _compact_slots(rt, old_active, new_active):
        """_early_stop (:937-980): the unfinished requests move to the front slots, in order (input ids, cursors,
        batch_indices and the KV cache rows of the reference; here the slot state and caches, on the device)"""
        pos = {req: s for s, req in enumerate(old_active)}
        for s_new, req in enumerate(new_active):
            s_old = pos[req]
            if s_old == s_new:
                continue
            assert s_new < s_old
            for t in (rt.seq, rt.seq_len, rt.prefix_len, rt.pad, rt.trie_idx, rt.k_cache, rt.v_cache):
                t[s_new].copy_(t[s_old])
        rt.finished.zero_()
