# -*- coding: utf-8 -*-
"""LookaheadPreTrainedModel: the reference's generation surface
(/root/reference/lookahead/lookahead/common/pretrained_model.py: class :48, generate :108, lookahead_prepare_inputs
:666-756, _lookahead_update_model_kwargs :764-892, _update_cache :894-945, lookahead_generation :947-1268,
stream_generate :1323-1350) re-built H100-first.

The reference loop crosses the host/device boundary several times per step (draft ids + n x n mask H2D, one argmax
+ .tolist() sync per accepted token, kv_idx H2D, a torch.cat of the whole KV cache per layer).  Here one decode step

    trie get -> embed -> L x [rmsnorm, qkv GEMM, rope+kv-append, tree attention, o GEMM, rmsnorm, gate/up GEMM,
    silu*mul, down GEMM] -> norm -> lm_head GEMM -> accept walk -> KV compaction -> trie stream_put

runs entirely on the device from device-resident state (token sequences, lengths, KV caches, trie) and is replayed
as ONE CUDA graph; the host reads back a single small pinned record (count, finished flag, accepted tokens) per
step to drive streamers / stopping, one step late: step k+1 is already enqueued when record k is read (a step that
runs after its request finished is a no-op on the device).  Everything per-request that varies - prompt length,
left padding, max_length - lives in device scalars, so one captured graph serves every request of a configuration.
The runtime is organised in request SLOTS (include/pia_b200.h pia_slots_t): this per-request loop runs one slot,
the batched loop (pretrained_model_batch.py) one slot per request, a prefill pass one slot per 64-row prompt chunk.
There is no CPU fallback."""
import os
import time
from collections import OrderedDict
from threading import Thread

import numpy as np
import torch
from torch import nn

from . import ops
from .lookahead_cache import LookaheadCache
from .lookahead_generation_utils import GenerationMode, LookaheadDecoderOnlyOutput

MAX_GRAPHS = 8  # captured step graphs kept per runtime (LRU)
REC = 5         # header words of a step record: count, finished, n, status, trie error bits


def warn_trie_errors(bits):
    """the trie's sticky pool-exhaustion bits arrived with a step record: generation stays lossless, but inserts are
    being dropped, i.e. the draft cache has stopped learning (the reference's Python dicts cannot run out)"""
    import warnings
    warnings.warn(f'LookaheadCache pools exhausted (error bits {bits:#x}: 1 nodes, 2 edges, 4 frontier, 8 stream buffer, '
                  '16 histogram, 32 token id): new n-grams are no longer stored; call lookahead_cache.fresh() or build '
                  'the cache with a larger node_capacity', RuntimeWarning, stacklevel=3)


class _Bufs(object):
    """activation buffers of one forward pass over `rows` token rows; `slots` (ops.Slots) says which request slot
    owns which rows and `mask` holds the rows' ancestor bit sets"""

    def __init__(self, g, rows, dev, with_logits):
        bf = dict(dtype=torch.bfloat16, device=dev)
        hid, qkv_dim = g['hidden'], (g['n_q_heads'] + 2 * g['n_kv_heads']) * g['head_dim']
        self.rows = rows
        self.ids = torch.zeros((rows,), dtype=torch.int32, device=dev)
        self.n_total = torch.zeros((1,), dtype=torch.int32, device=dev)
        self.h = torch.zeros((rows, hid), **bf)
        self.resid = torch.zeros((rows, hid), **bf)
        self.y = torch.zeros((rows, hid), **bf)
        self.qkv = torch.zeros((rows, qkv_dim), **bf)
        self.q = torch.zeros((rows, g['n_q_heads'], g['head_dim']), **bf)
        self.attn = torch.zeros((rows, g['n_q_heads'] * g['head_dim']), **bf)
        self.logits = torch.zeros((rows, g['vocab']), **bf) if with_logits else None
        self.mask = None
        self.slots = None
        self.kv_slot = 0   # cache the pointer-addressed kernels (rope / KV append) start from


class _Runtime(object):
    """device-resident state of one model's draft-verify loop: `n_slots` request slots sharing max_nodes draft rows"""

    def __init__(self, model, max_seq, max_nodes, n_slots=1):
        dev = model.device
        self.device = dev
        self.max_seq, self.max_nodes, self.n_slots = int(max_seq), int(max_nodes), int(n_slots)
        g = model.geometry()
        self.g = g
        i32 = dict(dtype=torch.int32, device=dev)
        bf = dict(dtype=torch.bfloat16, device=dev)
        W, R, S = self.max_nodes // 64, self.max_nodes, self.n_slots
        self.k_cache = torch.zeros((S, g['n_layers'], g['n_kv_heads'], self.max_seq, g['head_dim']), **bf)
        self.v_cache = torch.zeros_like(self.k_cache)
        self.cache_elems = self.k_cache[0].numel()
        self.plan = ops.AttnPlan(self.k_cache, self.v_cache, g['n_q_heads'], g['n_kv_heads'], g['head_dim'], R)
        # drafts (filled by the trie kernel or, for prefill chunks, by the host): R rows shared by the slots
        self.ids = torch.zeros((R,), **i32)
        self.mask = torch.zeros((R, W), dtype=torch.int64, device=dev)
        self.n = torch.ones((S,), **i32)
        self.sizes = torch.zeros((S, 2), **i32)
        self.nsizes = torch.zeros((S,), **i32)
        self.status = torch.zeros((S,), **i32)
        # per-slot sequence state
        self.seq = torch.zeros((S, self.max_seq + 8), **i32)
        self.seq_len = torch.zeros((S,), **i32)
        self.prefix_len = torch.zeros((S,), **i32)
        self.finished = torch.zeros((S,), **i32)
        self.pad = torch.zeros((S,), **i32)            # left-pad columns (pretrained_model.py:1123-1131)
        self.trie_idx = torch.arange(S, **i32)         # slot -> request idx of the trie (batched loop)
        self.max_length = torch.zeros((1,), **i32)     # MaxLengthCriteria, read on the device
        self.rng = torch.zeros((2,), **i32)            # {seed, step counter} of the multinomial accept (do_sample)
        self.acc_tokens = torch.zeros((S, R), **i32)
        self.acc_count = torch.zeros((S,), **i32)
        self.acc_nodes = torch.zeros((S, R), **i32)
        # host-visible step record per slot: [count, finished, n, status, trie error bits, tokens...]; two pinned copies
        # so that the step launched ahead does not overwrite the record the host is still reading
        self.record = torch.zeros((S, REC + R), **i32)
        self.record_host = [torch.zeros((S, REC + R), dtype=torch.int32).pin_memory() for _ in range(2)]
        self.trie_err = torch.zeros((1,), **i32)
        # activations of a decode step
        db = _Bufs(g, R, dev, with_logits=True)
        db.ids = self.ids
        db.mask = self.mask
        db.slots = ops.Slots(self.n, self.prefix_len, self.pad, R, 0, batch=1)
        db.n_total = self.n  # one slot: live rows = n[0]
        self.decode_bufs = db
        self.h, self.resid, self.y, self.qkv, self.q, self.attn, self.logits = db.h, db.resid, db.y, db.qkv, db.q, \
            db.attn, db.logits
        # activations of a prefill pass: up to pf_chunks chain chunks of R rows through one set of GEMMs, one slot each
        C = max(1, 256 // R)
        self.pf_chunks = C
        pb = _Bufs(g, R * C, dev, with_logits=False)
        self.pf_meta = torch.zeros((3, C), **i32)       # rows: n, P, pad of every chunk
        self.pf_meta_host = torch.zeros((3, C), dtype=torch.int32).pin_memory()
        self.chain = self.chain_mask_rows()
        pb.mask = self.chain.repeat(C, 1).contiguous()
        self.pf_mask_dirty = False
        self.pf_slots = {}
        self.prefill_bufs = pb
        self.rope_cos, self.rope_sin = model.rope_tables(self.max_seq + 8)
        self.graphs = OrderedDict()
        self.replays = 0
        self.kernels_per_graph = 0
        self.prefill_graphs, self.prefill_kernels, self.prefill_warm = {}, {}, set()
        self.graph_launches = 0  # kernels of replayed prefill graphs
        self.last_compact_check = 0
        self.accepts = {}
        self.pad_host = 0

    def k_layer(self, layer, slot=0):
        return self.k_cache[slot, layer]

    def v_layer(self, layer, slot=0):
        return self.v_cache[slot, layer]

    def prefill_slots(self, slot):
        """slot table of a prefill pass into request slot `slot`'s cache: one table slot per 64-row chain chunk"""
        if slot not in self.pf_slots:
            self.pf_slots[slot] = ops.Slots(self.pf_meta[0], self.pf_meta[1], self.pf_meta[2], self.max_nodes, 0,
                                            batch=self.pf_chunks, kv_first_slot=slot)
        return self.pf_slots[slot]

    def decode_slots(self, batch, rows_per_slot):
        key = ('dec', batch, rows_per_slot)
        if key not in self.pf_slots:
            self.pf_slots[key] = ops.Slots(self.n, self.prefix_len, self.pad, rows_per_slot,
                                           self.cache_elems if batch > 1 else 0, batch=batch)
        return self.pf_slots[key]

    # -- prefill: the prompt is fed as chain drafts of <= max_nodes tokens through the same verify kernels
    def chain_mask_rows(self):
        R = self.max_nodes
        rows = np.zeros((R, R // 64), dtype=np.uint64)
        for i in range(R):
            for w in range(R // 64):
                lo = 64 * w
                if i >= lo + 63:
                    rows[i, w] = np.uint64(0xFFFFFFFFFFFFFFFF)
                elif i >= lo:
                    rows[i, w] = np.uint64((1 << (i - lo + 1)) - 1)
        return torch.from_numpy(rows.view(np.int64)).to(self.device)

    def chain_without_first(self, k):
        """chain mask whose first k columns (left-pad tokens of this chunk) are cleared"""
        cache = self.__dict__.setdefault('_chain_cut', {})
        if k not in cache:
            rows = self.chain.cpu().numpy().view(np.uint64).copy()
            R = self.max_nodes
            for w in range(R // 64):
                lo = 64 * w
                if k >= lo + 64:
                    rows[:, w] = 0
                elif k > lo:
                    rows[:, w] &= ~np.uint64((1 << (k - lo)) - 1)
            cache[k] = torch.from_numpy(rows.view(np.int64)).to(self.device)
        return cache[k]

    def set_request(self, slot, pad_len, max_length):
        """per-request scalars the captured graphs read on the device"""
        self.pad_host = int(pad_len)
        self.pad[slot:slot + 1].fill_(int(pad_len))
        self.max_length.fill_(int(max_length))


class LookaheadPreTrainedModel(nn.Module):
    """Base class of the patched models (reference :48). Subclasses implement geometry(), rope_tables() and
    _verify_layers(rt) (the per-model forward over the static draft buffers)."""
    _batch_generation = False
    _stream_generation = False

    def __init__(self, config):
        super().__init__()
        self.config = config
        self._rt = None

    # ------------------------------------------------------------------ plumbing
    @property
    def device(self):
        return next(self.parameters()).device

    def _runtime(self, max_seq, max_nodes, n_slots=1, keep_cache=False):
        rt = self._rt
        if rt is None or rt.max_seq < max_seq or rt.max_nodes != max_nodes or rt.n_slots < n_slots:
            assert not keep_cache or rt is None, \
                (f'the KV cache holds a context but the runtime has to be rebuilt ({max_seq=} {max_nodes=} '
                 f'vs {rt.max_seq=} {rt.max_nodes=}): past tokens would be dropped')
            self._rt = None
            rt = _Runtime(self, max(max_seq, 128), max_nodes, n_slots)
            self._rt = rt
            # one-time weight preparation must never end up inside a captured step graph
            if hasattr(self, 'fuse'):
                self.fuse()
            if hasattr(self, '_gemm_plans'):
                self._gemm_plans(rt)
        return rt

    def quantize_fp8(self):
        """fp8 weight-only mode; the Llama family implements it (GPT-2's linears run through torch)"""
        raise NotImplementedError(f'{type(self).__name__} has no fp8 weight mode')

    def _decoding_args(self):
        return ['decoding_kwargs']

    def _get_generation_mode(self, do_sample, use_cache, decoding_kwargs):
        """reference :55-106 (the branches reachable from this surface)"""
        if use_cache and decoding_kwargs.get('use_lookahead', False) and decoding_kwargs.get('decoding_length', 64) > 1 \
                and decoding_kwargs.get('branch_length', 12) > 0:
            return GenerationMode.LOOKAHEAD_GENERATION
        return GenerationMode.SAMPLE if do_sample else GenerationMode.GREEDY_SEARCH

    # ------------------------------------------------------------------ generate (reference :108-664)
    @torch.no_grad()
    def generate(self, inputs=None, generation_config=None, logits_processor=None, stopping_criteria=None,
                 prefix_allowed_tokens_fn=None, synced_gpus=None, assistant_model=None, streamer=None, **kwargs):
        allowed = {'input_ids', 'attention_mask', 'position_ids', 'max_new_tokens', 'max_length', 'pad_token_id',
                   'eos_token_id', 'use_cache', 'repetition_penalty', 'do_sample', 'return_dict_in_generate',
                   'output_scores', 'decoding_kwargs', 'num_beams', 'temperature', 'top_k', 'top_p'}
        unknown = [k for k in kwargs if k not in allowed]
        if unknown:  # reference :1309-1317
            raise ValueError(f'The following `model_kwargs` are not used by the model: {unknown} (note: typos in the'
                             ' generate arguments will also show up in this list)')
        if prefix_allowed_tokens_fn or assistant_model is not None:
            raise NotImplementedError('prefix_allowed_tokens_fn / assistant models are not on the lookahead path')
        if kwargs.get('num_beams', 1) != 1:
            raise NotImplementedError('beam search is not on the lookahead path')
        input_ids = kwargs.get('input_ids', inputs)
        assert input_ids is not None and input_ids.dim() == 2
        gc = generation_config if generation_config is not None else getattr(self, 'generation_config', None)

        def opt(name, default=None):
            if name in kwargs and kwargs[name] is not None:
                return kwargs[name]
            v = getattr(gc, name, None) if gc is not None else None
            return v if v is not None else default

        decoding_kwargs = kwargs.get('decoding_kwargs', None)
        if decoding_kwargs is None:
            decoding_kwargs = getattr(gc, 'decoding_kwargs', None) if gc is not None else None
        if decoding_kwargs is None:
            decoding_kwargs = {}
        do_sample = bool(opt('do_sample', False))
        use_cache = bool(opt('use_cache', True))
        max_new = opt('max_new_tokens')
        max_length = input_ids.shape[1] + int(max_new) if max_new is not None else int(opt('max_length', 20))
        eos = opt('eos_token_id', getattr(self.config, 'eos_token_id', None))
        pad = opt('pad_token_id', getattr(self.config, 'pad_token_id', None))
        mode = self._get_generation_mode(do_sample, use_cache, decoding_kwargs)
        if do_sample and mode != GenerationMode.LOOKAHEAD_GENERATION:
            decoding_kwargs = dict(decoding_kwargs, use_lookahead=False)  # plain sampling = a draft of the root alone
        # the reference mutates the caller's dict (:362-372)
        decoding_kwargs['generation_mode'] = mode
        decoding_kwargs['do_sample'] = do_sample
        decoding_kwargs['max_length'] = max_length
        dl = decoding_kwargs.get('decoding_length', 64) if mode == GenerationMode.LOOKAHEAD_GENERATION else 0
        decoding_kwargs['decoding_max_length'] = max_length + dl + (1 if dl else 0)
        crit_max = getattr(stopping_criteria, 'max_length', None) if stopping_criteria is not None else None
        if crit_max is not None:
            max_length = min(max_length, int(crit_max))
        # caller-supplied processors / criteria (reference :349-360): MaxLengthCriteria is the device-side max_length;
        # anything else runs on the host path of the loop, one processor call per accepted token like the reference
        extra_criteria = [c for c in (stopping_criteria or []) if type(c).__name__ != 'MaxLengthCriteria']
        return self.lookahead_generation(input_ids, logits_processor=list(logits_processor or []) or None,
                                         stopping_criteria=extra_criteria or None, max_length=max_length,
                                         pad_token_id=pad, eos_token_id=eos,
                                         output_scores=opt('output_scores', False),
                                         return_dict_in_generate=opt('return_dict_in_generate', False),
                                         streamer=streamer, attention_mask=kwargs.get('attention_mask'),
                                         decoding_kwargs=decoding_kwargs,
                                         repetition_penalty=float(opt('repetition_penalty', 1.0)))

    # ------------------------------------------------------------------ the loop (reference :947-1268)
    def _graph_entry(self, rt, key, build):
        """LRU cache of captured step graphs; an entry keeps alive what its graph points into (trie, accept config)"""
        ent = rt.graphs.get(key)
        if ent is None:
            ent = build()
            rt.graphs[key] = ent
            while len(rt.graphs) > MAX_GRAPHS:
                rt.graphs.popitem(last=False)
        else:
            rt.graphs.move_to_end(key)
        return ent

    def _capture_step(self, rt, trie, use_trie, dl, bl, mql, min_out, tmode, kind, accept, sample=False):
        """one decode step of the per-request loop as a CUDA graph over the static buffers (slot 0)"""
        draft = dict(ids=rt.ids, mask=rt.mask, n=rt.n, sizes=rt.sizes, nsizes=rt.nsizes, status=rt.status)

        def step():
            if use_trie:
                # lookahead_prepare_inputs_for_generation :708-723 (query = last tokens of the device sequence;
                # branch_length clamped by the device-resident max_length, :680)
                trie.get_device(rt.seq, rt.seq_len, dl, bl, max_query_length=mql, min_input_size=0,
                                min_output_size=min_out, mode=tmode, idx=0, kind=kind, max_seq_length=1,
                                d_max_seq_length=rt.max_length, out=draft)
            else:  # plain greedy: the draft is the last token alone
                rt.ids[0:1] = rt.seq[0].gather(0, (rt.seq_len - 1).long())
                rt.n.fill_(1)
                rt.mask[0, 0:1].fill_(1)
            self._verify_layers(rt)
            accept.run(rt.logits, rt.ids, rt.mask, rt.n, rt.seq, rt.seq_len, rt.acc_tokens, rt.acc_count, rt.acc_nodes,
                       rt.prefix_len, rt.finished, batch=1, rows_per_slot=rt.max_nodes, max_length=rt.max_length,
                       rng=rt.rng if sample else None)
            ops.kv_compact(rt.k_cache, rt.v_cache, rt.acc_nodes, rt.acc_count, rt.prefix_len, batch=1)
            if use_trie:  # :1203
                trie.stream_put_device(rt.acc_tokens, rt.max_nodes, rt.acc_count, branch_length=self._put_bl,
                                       final=False, idx=0)
                trie.copy_error_flags_device(rt.trie_err)
            rt.record[0, 0:1] = rt.acc_count
            rt.record[0, 1:2] = rt.finished
            rt.record[0, 2:3] = rt.n
            rt.record[0, 3:4] = rt.status
            rt.record[0, 4:5] = rt.trie_err
            rt.record[0, REC:] = rt.acc_tokens[0]

        graphs = []
        l0 = ops.launch_count()
        for host in rt.record_host:  # one graph per pinned record copy (the step launched ahead writes the other)
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g):
                step()
                host.copy_(rt.record, non_blocking=True)
            graphs.append(g)
        rt.kernels_per_graph = (ops.launch_count() - l0) // 2  # libpia_b200 kernels per replay (bench.py gpu_launches)
        return dict(graphs=graphs, keep=(trie, accept))

    @torch.no_grad()
    def lookahead_generation(self, input_ids, logits_processor=None, stopping_criteria=None, max_length=None,
                             pad_token_id=None, eos_token_id=None, output_attentions=None, output_hidden_states=None,
                             output_scores=None, return_dict_in_generate=None, synced_gpus=False, streamer=None,
                             attention_mask=None, decoding_kwargs=None, repetition_penalty=1.0, **model_kwargs):
        assert input_ids.size(0) == 1, 'the lookahead loop is per request (reference :1152)'
        dev = self.device
        torch.cuda.set_device(dev)
        decoding_kwargs = decoding_kwargs if decoding_kwargs is not None else {}
        if isinstance(eos_token_id, int):
            eos_token_id = [eos_token_id]
        use_trie = decoding_kwargs.get('generation_mode', GenerationMode.LOOKAHEAD_GENERATION) == \
            GenerationMode.LOOKAHEAD_GENERATION and decoding_kwargs.get('use_lookahead', True)
        dl = int(decoding_kwargs.get('decoding_length', 64)) if use_trie else 1
        bl = int(decoding_kwargs.get('branch_length', 12)) if use_trie else 1
        dmode = decoding_kwargs.get('decoding_mode', 'hier')
        mql = int(decoding_kwargs.get('max_query_length', 2))
        if dmode in ('hier', 'par', 'one'):
            dmode = dmode + '_mix'  # :712-713
        fmt, tmode = dmode.split('_')
        if fmt == 'par':
            # the reference dies here as well: par_get returns a float64 mask (lookahead_cache.py:481), and its accept
            # routine then slices a list with float indices (pretrained_model.py:817-819: TypeError on the first
            # non-empty draft; tests/golden/gen_loop_golden.py).  LookaheadCache.par_get itself is built (host API).
            raise TypeError('slice indices must be integers or None or have an __index__ method '
                            "(decoding_mode 'par' never worked inside the reference's loop, pretrained_model.py:819)")
        assert dl <= 128 and bl <= 32, 'decoding_length <= 128 and branch_length <= 32 are built'
        if max_length is None:
            max_length = int(decoding_kwargs.get('max_length', 2048))
        max_nodes = 64 if dl <= 64 else 128
        prompt_len = input_ids.shape[1]
        max_seq = max_length + dl + 1  # decoding_max_length (:1115)
        rt = self._runtime(max_seq, max_nodes)

        # init lookahead cache (:1086-1089)
        if not hasattr(self, 'lookahead_cache') or self.lookahead_cache is None:
            self.lookahead_cache = LookaheadCache(device=dev, vocab_capacity=max(self.geometry()['vocab'], 1024))
        trie = self.lookahead_cache
        trie.eos_ids = eos_token_id
        trie.stop_words = decoding_kwargs.get('stop_words', {})
        decoding_kwargs.update({'eos': eos_token_id[0] if eos_token_id is not None else 2, 'edls': [], 'dls': [],
                                'fts': [], 'qts': []})
        decoding_kwargs['max_length'] = max_length
        decoding_kwargs['decoding_max_length'] = max_seq
        self._put_bl = bl + 1

        # left padding (:1123-1131): bs == 1, so a 2-D mask can only mark a padded prefix
        pad_len = 0
        if attention_mask is not None:
            am = attention_mask.reshape(-1)[:prompt_len] if attention_mask.dim() == 2 else None
            if am is not None:
                nz = torch.nonzero(am.to('cpu') != 0)
                pad_len = int(nz[0]) if nz.numel() else 0
        rt.set_request(0, pad_len, max_length)
        # multinomial accept (:787-789, :835-837): softmax of the processed scores, no warpers on this path (:430-441)
        sample = bool(decoding_kwargs.get('do_sample', False))
        if sample:
            rt.rng.copy_(torch.tensor([torch.initial_seed() & 0x7FFFFFFF, rt.replays & 0x7FFFFFFF], dtype=torch.int32))

        ts = time.time()
        prompt = input_ids[0].to(device=dev, dtype=torch.int32)
        rt.seq[0, :prompt_len] = prompt
        rt.finished.zero_()
        if use_trie:  # (:1153-1156)
            trie.put_device(rt.seq[0, 1:], max(prompt_len - 1, 0), None, branch_length=bl + 1, final=False, mode='input',
                            idx=0)
        akey = (float(repetition_penalty), tuple(eos_token_id or ()), max_nodes)
        accept = rt.accepts.get(akey)
        if accept is None:  # referenced by captured graphs: lives as long as the runtime
            accept = ops.Accept(self.geometry()['vocab'], max_nodes, repetition_penalty, eos_token_id, max_length, dev)
            rt.accepts[akey] = accept
        host_path = bool(logits_processor or stopping_criteria)
        if host_path:          # built-in penalty + the caller's processors, in generate()'s order (:349-355)
            logits_processor = list(logits_processor or [])
            if float(repetition_penalty) != 1.0:
                from transformers import RepetitionPenaltyLogitsProcessor
                logits_processor.insert(0, RepetitionPenaltyLogitsProcessor(penalty=float(repetition_penalty)))
        if host_path:          # the processors also see the prefill logits (:786)
            self._prefill_logits(rt, prompt_len)
            first = self._host_pick(logits_processor, input_ids.to(dev), rt.logits[0:1], sample)
            rt.seq[0, prompt_len] = first
            rt.seq_len.fill_(prompt_len + 1)
            rt.prefix_len.fill_(prompt_len)
        else:
            first = self._prefill(rt, prompt_len, accept, sample)
        new_tokens = [first]
        decoding_kwargs['dls'].append(1)  # the prefill step counts as one fed token (:797-798)
        decoding_kwargs['edls'].append(1)
        if streamer is not None:
            streamer.put(input_ids.cpu())
            streamer.put(np.array([[first]]))
        if use_trie:
            trie.stream_put_device(rt.seq[0, prompt_len:], 1, None, branch_length=bl + 1, final=False, idx=0)
        finished = (eos_token_id is not None and first in eos_token_id) or prompt_len + 1 >= max_length
        te = time.time()
        decoding_kwargs['fts'].append(te - ts)
        ts = te

        min_out = max(dl // 2, 1)  # :710
        key = (use_trie, dl, bl, mql, tmode, fmt, akey, id(trie._t), sample)
        stream = torch.cuda.current_stream()
        if host_path and not finished:
            finished = self._host_accept_loop(rt, trie, use_trie, dl, bl, mql, min_out, tmode,
                                              'hier' if fmt == 'hier' else 'one', logits_processor or [],
                                              stopping_criteria or [], sample, eos_token_id, max_length, new_tokens,
                                              decoding_kwargs, streamer, input_ids)
        if not finished:
            ent = self._graph_entry(rt, key, lambda: self._capture_step(
                rt, trie, use_trie, dl, bl, mql, min_out, tmode, 'hier' if fmt == 'hier' else 'one', accept, sample))
            graphs = ent['graphs']
            # step k+1 is enqueued before the host reads record k: the ~0.25 ms of host work per step (record read,
            # python bookkeeping, streamer) overlaps the next verify forward; a step that runs after `finished` was
            # raised changes nothing on the device (pia_accept no-op, zero-length stream_put)
            # A step launched ahead of the one that ends the request is a whole wasted forward (3.5 ms at 7B): near the end
            # of the length budget - when the step in flight could already exhaust it (a step accepts at most
            # branch_length + 1 tokens) - the next step is only launched once the record has been read.  An EOS / stop
            # still costs the one step that was in flight.
            events = [torch.cuda.Event(), torch.cuda.Event()]
            k = 0
            launched = 1
            graphs[0].replay()
            events[0].record(stream)
            rt.replays += 1
            while True:
                if launched == k + 1 and max_length - (prompt_len + len(new_tokens)) > bl + 1:
                    graphs[launched & 1].replay()
                    events[launched & 1].record(stream)
                    rt.replays += 1
                    launched += 1
                events[k & 1].synchronize()
                rec = rt.record_host[k & 1][0]
                count, fin, n, status = int(rec[0]), int(rec[1]), int(rec[2]), int(rec[3])
                if status != 0:
                    from .. import _lib as L
                    L.check(status)
                if int(rec[4]) != 0 and not getattr(trie, '_warned_pool', False):
                    trie._warned_pool = True
                    warn_trie_errors(int(rec[4]))
                toks = rec[REC:REC + count].tolist()
                new_tokens.extend(toks)
                decoding_kwargs['dls'].append(n)
                decoding_kwargs['edls'].append(count)
                decoding_kwargs['qts'].append(0.0)
                if streamer is not None:
                    streamer.put(np.array([toks]))
                if decoding_kwargs.get('debug_lookahead', False):
                    tok = decoding_kwargs.get('tokenizer', None)
                    words = '' if tok is None else tok.decode(toks)
                    print(f'decoding_length:{n} accept_length:{count} accept_token:{toks} accept_word:{words}')
                te = time.time()
                decoding_kwargs['fts'].append(te - ts)
                ts = te
                k += 1
                if fin:
                    break
                if launched == k:  # near the end of the budget: launch only now that the request is known to go on
                    graphs[launched & 1].replay()
                    events[launched & 1].record(stream)
                    rt.replays += 1
                    launched += 1
            if launched > k:
                events[k & 1].synchronize()  # a step launched ahead (a no-op on the device) has drained
        if use_trie:  # :1237-1238
            trie.stream_put([], branch_length=bl + 1, final=True, mode='output', idx=0)
            if rt.replays - rt.last_compact_check >= 2048:   # every few thousand steps: reclaim squeezed storage if a pool fills up
                rt.last_compact_check = rt.replays
                trie.maybe_compact()
        if streamer is not None:
            streamer.end()
        out_ids = torch.cat([input_ids.to(dev), torch.tensor([new_tokens], dtype=input_ids.dtype, device=dev)], dim=1)
        if return_dict_in_generate:
            kw = {k_: decoding_kwargs[k_] for k_ in ('dls', 'edls', 'fts', 'qts')}
            return LookaheadDecoderOnlyOutput(sequences=out_ids, scores=() if output_scores else None, kwargs=kw)
        return out_ids

    # ------------------------------------------------------------------ host accept path (custom processors / criteria)
    @staticmethod
    def _host_pick(processors, ids, logits_row, sample):
        """next_tokens_scores = logits_processor(update_input_ids, next_token_logits); arg-max / multinomial (:834-839)"""
        scores = logits_row
        for proc in processors:
            scores = proc(ids, scores)
        if sample:
            return int(torch.multinomial(torch.softmax(scores, dim=-1), num_samples=1)[0, 0])
        return int(torch.argmax(scores, dim=-1)[0])

    def _host_accept_loop(self, rt, trie, use_trie, dl, bl, mql, min_out, tmode, kind, processors, criteria, sample,
                          eos_token_id, max_length, new_tokens, decoding_kwargs, streamer, input_ids):
        """The loop for caller-supplied logits processors / stopping criteria (reference :349-360, :786, :834, :1225):
        arbitrary Python callables cannot run inside the captured step, so the accept walk runs on the host exactly like
        the reference's (:827-860: one processor call + one device->host sync per accepted token) while draft, verify
        forward, KV compaction and trie update stay the device kernels.  Returns True (the request finished here)."""
        dev = rt.device
        draft = dict(ids=rt.ids, mask=rt.mask, n=rt.n, sizes=rt.sizes, nsizes=rt.nsizes, status=rt.status)
        seq = input_ids[0].tolist() + list(new_tokens)
        ts = time.time()
        while True:
            if use_trie:
                trie.get_device(rt.seq, rt.seq_len, dl, bl, max_query_length=mql, min_input_size=0,
                                min_output_size=min_out, mode=tmode, idx=0, kind=kind, max_seq_length=1,
                                d_max_seq_length=rt.max_length, out=draft)
            else:
                rt.ids[0:1] = rt.seq[0].gather(0, (rt.seq_len - 1).long())
                rt.n.fill_(1)
                rt.mask[0, 0:1].fill_(1)
            self._verify_layers(rt)
            n = int(rt.n[0])
            ids = rt.ids[:n].tolist()
            rows = rt.mask[:n].cpu().numpy().view(np.uint64)
            parent = [-1] * n
            for j in range(1, n):   # nearest ancestor = highest set bit below j (DFS pre-order)
                below = [k for k in range(j) if (int(rows[j, k >> 6]) >> (k & 63)) & 1]
                parent[j] = below[-1] if below else -1
            cur, toks, nodes = 0, [], []
            ctx = torch.tensor([seq], dtype=torch.long, device=dev)
            while True:
                t = self._host_pick(processors, ctx, rt.logits[cur:cur + 1], sample)
                toks.append(t)
                nodes.append(cur)
                ctx = torch.cat([ctx, torch.tensor([[t]], dtype=torch.long, device=dev)], dim=1)
                nxt = [j for j in range(1, n) if parent[j] == cur and ids[j] == t]
                if not nxt or len(toks) >= n:
                    break
                cur = nxt[0]
            count = len(toks)
            L0 = len(seq)
            seq.extend(toks)
            rt.seq[0, L0:L0 + count] = torch.tensor(toks, dtype=torch.int32, device=dev)
            rt.seq_len.fill_(L0 + count)
            rt.acc_tokens[0, :count] = torch.tensor(toks, dtype=torch.int32, device=dev)
            rt.acc_nodes[0, :count] = torch.tensor(nodes, dtype=torch.int32, device=dev)
            rt.acc_count.fill_(count)
            rt.prefix_len.fill_(L0 - 1 + count)
            ops.kv_compact(rt.k_cache, rt.v_cache, rt.acc_nodes, rt.acc_count, rt.prefix_len, batch=1)
            if use_trie:
                trie.stream_put_device(rt.acc_tokens, rt.max_nodes, rt.acc_count, branch_length=self._put_bl,
                                       final=False, idx=0)
            new_tokens.extend(toks)
            decoding_kwargs['dls'].append(n)
            decoding_kwargs['edls'].append(count)
            decoding_kwargs['qts'].append(0.0)
            if streamer is not None:
                streamer.put(np.array([toks]))
            fin = len(seq) >= max_length or (eos_token_id is not None and any(e in toks for e in eos_token_id))
            full = torch.tensor([seq], dtype=torch.long, device=dev)
            for crit in criteria:   # StoppingCriteriaList semantics: any criterion may stop (:1225)
                fin = fin or bool(torch.as_tensor(crit(full, None)).any())
            te = time.time()
            decoding_kwargs['fts'].append(te - ts)
            ts = te
            if fin:
                return True

    def _prefill_kv(self, rt, prompt_len, slot=0):
        """prompt tokens rt.seq[slot, :prompt_len] -> KV rows [0, prompt_len) of that slot's cache; leaves the last
        prompt row's hidden state in the prefill buffers and its logits in rt.logits[0].  The prompt goes through
        the verify kernels as chain drafts (row i attends rows <= i): per pass the GEMMs see up to 256 rows at once,
        RoPE/KV-append and tree attention run once over all 64-row chunks (one table slot per chunk)."""
        R, C = rt.max_nodes, rt.pf_chunks
        pb = rt.prefill_bufs
        pb.slots = rt.prefill_slots(slot)
        pb.kv_slot = slot
        pad = rt.pad_host
        pos = 0
        while pos < prompt_len:
            m = min(R * C, prompt_len - pos)
            pb.ids[:m] = rt.seq[slot, pos:pos + m]
            pb.n_total.fill_(m)
            ns = [max(0, min(R, m - R * c)) for c in range(C)]
            rt.pf_meta_host.copy_(torch.tensor([ns, [pos + R * c for c in range(C)], [pad] * C], dtype=torch.int32))
            rt.pf_meta.copy_(rt.pf_meta_host, non_blocking=True)
            if pad > pos:  # left padding (:1123-1131): pad columns are invisible, also inside a chain chunk
                for c in range(C):
                    k = min(max(pad - (pos + R * c), 0), R)
                    pb.mask[R * c:R * (c + 1)] = rt.chain if k == 0 else rt.chain_without_first(k)
                rt.pf_mask_dirty = True
            elif rt.pf_mask_dirty:
                pb.mask.copy_(rt.chain.repeat(C, 1))
                rt.pf_mask_dirty = False
            last = pos + m >= prompt_len
            self._prefill_pass(rt, pb, slot, last)
            torch.cuda.current_stream().synchronize()  # pf_meta_host is rewritten by the next pass
            pos += m
        last_row = (prompt_len - 1) % (R * C)
        return pb.y[last_row:last_row + 1]

    def _prefill_pass(self, rt, pb, slot, last):
        """one pass of the prompt through the layers.  Everything a pass depends on (ids, chunk table, masks, cursors)
        lives in device buffers, so the ~350 launches are captured once per (slot, last) - the first pass of a runtime
        runs eagerly (library handles / workspaces come into being outside a capture), the second is captured, later
        ones replay: an eager pass is bound by the host's launch rate, not by the GPU."""
        key = (slot, last)
        g = rt.prefill_graphs.get(key)
        if g is None:
            if key not in rt.prefill_warm or os.environ.get('PIA_PREFILL_GRAPH', '1') == '0':
                rt.prefill_warm.add(key)
                self._verify_layers(rt, bufs=pb, last_only=not last)
                return
            torch.cuda.current_stream().synchronize()
            l0 = ops.launch_count()
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g):
                self._verify_layers(rt, bufs=pb, last_only=not last)
            rt.prefill_graphs[key] = g
            rt.prefill_kernels[key] = ops.launch_count() - l0
        g.replay()
        rt.graph_launches += rt.prefill_kernels[key]   # libpia_b200 kernels replayed (bench.py gpu_launches)

    def _prefill_logits(self, rt, prompt_len, slot=0, row=0):
        """prefill of slot `slot` + the last prompt row's logits into rt.logits[row]"""
        y = self._prefill_kv(rt, prompt_len, slot)
        torch.mm(y, self.lm_head.weight.t(), out=rt.logits[row:row + 1])

    def _prefill(self, rt, prompt_len, accept, sample=False):
        """prefill + the first generated token: (penalised) arg-max / draw of the last prompt row's logits (:783-798)"""
        self._prefill_logits(rt, prompt_len)
        return self._first_token(rt, prompt_len, accept, sample)

    def _first_token(self, rt, prompt_len, accept, sample=False):
        rt.ids[0:1] = rt.seq[0, prompt_len - 1:prompt_len]
        rt.mask.copy_(rt.chain)
        rt.n.fill_(1)
        rt.seq_len.fill_(prompt_len)
        rt.prefix_len.fill_(prompt_len)
        accept.run(rt.logits, rt.ids, rt.mask, rt.n, rt.seq, rt.seq_len, rt.acc_tokens, rt.acc_count, rt.acc_nodes,
                   rt.prefix_len, rt.finished, batch=1, rows_per_slot=rt.max_nodes, max_length=rt.max_length,
                   rng=rt.rng if sample else None)
        rt.prefix_len.fill_(prompt_len)
        return int(rt.acc_tokens[0, 0].item())

    # ------------------------------------------------------------------ reference-shaped forward (API parity)
    @torch.no_grad()
    def forward(self, input_ids=None, attention_mask=None, position_ids=None, past_key_values=None, use_cache=True,
                return_dict=True, **kwargs):
        """The patched forward of the reference (:544-677, :710-790) for rank-4 lookahead masks
        `[1, 1, n, P + n]` (visible prefix || tree).  `past_key_values` is the integer P returned by the previous
        call (the KV cache itself is the model's preallocated device cache).  Returns (logits [1, n, V], P + n)."""
        assert input_ids is not None and input_ids.shape[0] == 1
        n = input_ids.shape[1]
        P = int(past_key_values) if past_key_values is not None else 0
        am = attention_mask
        assert am is not None and am.dim() == 4 and am.shape[2] == n and am.shape[3] == P + n, \
            'forward expects the lookahead mask [1,1,n,P+n] (modeling_llama.py:585-588)'
        am = am[0, 0].to('cpu').long().numpy()
        pad_len = 0
        if P > 0:
            nz = am[0, :P].nonzero()[0]
            pad_len = int(nz[0]) if len(nz) else P
        tree = am[:, P:]
        need = P + n + 1
        have = self._rt
        rt = self._runtime(need if have is not None and have.max_seq >= need else max(need, 256),
                           64 if n <= 64 else 128, keep_cache=P > 0)
        assert n <= rt.max_nodes, 'at most 128 tree nodes per forward; prefill goes through generate()'
        packed = np.packbits(np.pad(tree.astype(np.uint8), ((0, rt.max_nodes - n), (0, rt.max_nodes - n))), axis=1,
                             bitorder='little')
        rows = torch.from_numpy(packed.view(np.int64).reshape(rt.max_nodes, rt.max_nodes // 64))
        rt.mask.copy_(rows.to(rt.device))
        rt.ids[:n] = input_ids[0].to(device=rt.device, dtype=torch.int32)
        rt.n.fill_(n)
        rt.prefix_len.fill_(P)
        rt.set_request(0, pad_len, 1 << 30)
        self._verify_layers(rt)
        logits = rt.logits[:n].clone()[None]
        return logits, P + n

    # ------------------------------------------------------------------ streaming (reference :1323-1350)
    @torch.no_grad()
    def stream_generate(self, inputs=None, generation_config=None, logits_processor=None, stopping_criteria=None,
                        prefix_allowed_tokens_fn=None, synced_gpus=None, assistant_model=None, streamer=None,
                        **kwargs):
        generation_kwargs = dict(inputs=inputs, generation_config=generation_config, logits_processor=logits_processor,
                                 stopping_criteria=stopping_criteria,
                                 prefix_allowed_tokens_fn=prefix_allowed_tokens_fn, synced_gpus=synced_gpus,
                                 assistant_model=assistant_model, streamer=streamer)
        generation_kwargs.update(kwargs)
        thread = Thread(target=self.generate, kwargs=generation_kwargs)
        thread.start()
        for words in streamer:
            yield words
