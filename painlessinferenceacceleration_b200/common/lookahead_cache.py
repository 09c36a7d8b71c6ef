# -*- coding: utf-8 -*-
"""LookaheadCache / Tree with the reference's method surface
(/root/reference/lookahead/lookahead/common/lookahead_cache.py: Tree :24, LookaheadCache :336), backed by the
GPU-resident trie of libpia_b200.so (csrc/trie.cu).  put/stream_put/hier_get/one_get run as CUDA kernels;
par_get (:441-488) and bat_get (:519-561) are thin host compositions over the batched get kernel.

Host-facing calls take Python lists and return ``(ids: list, mask: np.int64[n, n], sizes: list)`` exactly like
the reference.  The generation loop does not use them: it calls the ``*_device`` methods, which read the query
from the device-resident token sequence and leave the draft in HBM (no host round trip per step)."""
import ctypes as C

import numpy as np
import torch

from .. import _lib as L


def _bits_to_mask(rows, n):
    """uint64 bit rows [n, W] -> np.int64 [n, n]"""
    rows = np.ascontiguousarray(rows[:n]).astype('<u8')
    bits = np.unpackbits(rows.view(np.uint8).reshape(n, -1), axis=1, bitorder='little')
    return bits[:, :n].astype(np.int64)


class _DeviceTrie(object):
    """owner of one pia_trie_t handle plus its small staging buffers"""

    def __init__(self, device, eos_ids, stop_words, max_node, max_output_node, vocab_capacity, node_capacity,
                 edge_capacity, n_input_slots, max_put_tokens, frontier_capacity, max_resident_queries):
        if not torch.cuda.is_available():
            raise RuntimeError('LookaheadCache needs a CUDA device (H100); there is no CPU fallback')
        self.lib = L.load()
        self.device = torch.device(device if device is not None else f'cuda:{torch.cuda.current_device()}')
        cfg = L.TrieConfig(vocab_capacity, node_capacity, edge_capacity, n_input_slots, max_node, max_output_node,
                           max_put_tokens, frontier_capacity, max_resident_queries)
        self.cfg = cfg
        h = L.vp()
        with torch.cuda.device(self.device):
            L.check(self.lib.pia_trie_create(C.byref(cfg), C.byref(h)))
        self.h = h
        self._out = {}

    def close(self):
        if getattr(self, 'h', None):
            with torch.cuda.device(self.device):
                self.lib.pia_trie_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def stream(self):
        return torch.cuda.current_stream(self.device).cuda_stream

    def out_buffers(self, batch, dl):
        key = (batch, dl)
        if key not in self._out:
            W = (dl + 63) // 64
            dev = self.device
            self._out[key] = dict(ids=torch.empty((batch, dl), dtype=torch.int32, device=dev),
                                  mask=torch.empty((batch, dl, W), dtype=torch.int64, device=dev),
                                  n=torch.empty((batch,), dtype=torch.int32, device=dev),
                                  sizes=torch.empty((batch, 2), dtype=torch.int32, device=dev),
                                  nsizes=torch.empty((batch,), dtype=torch.int32, device=dev),
                                  status=torch.empty((batch,), dtype=torch.int32, device=dev))
        return self._out[key]


class LookaheadCache(object):
    """Drop-in for lookahead.common.lookahead_cache.LookaheadCache (reference :336-587)."""

    def __init__(self, debug=False, eos_ids=(2,), stop_words=None, max_node=65536, max_output_node=512, device=None,
                 vocab_capacity=262144, node_capacity=1 << 24, edge_capacity=None, n_input_slots=8,
                 max_put_tokens=16384, frontier_capacity=1 << 18, max_resident_queries=296):
        self.debug = debug
        self._node_capacity = node_capacity
        self._edge_capacity = edge_capacity if edge_capacity is not None else node_capacity
        self._t = _DeviceTrie(device, eos_ids, stop_words, max_node, max_output_node, vocab_capacity, node_capacity,
                              edge_capacity if edge_capacity is not None else node_capacity, n_input_slots,
                              max_put_tokens, frontier_capacity, max_resident_queries)
        self._max_node, self._max_output_node = max_node, max_output_node
        self._eos_ids = None
        self._stop_words = None
        self.eos_ids = eos_ids if eos_ids is not None else [None]
        self.stop_words = stop_words if stop_words is not None else {}
        self.default_mask = np.ones((1, 1), dtype=np.int64)

    # ---- attributes the callers read/write (benchmark.py:270-273, pretrained_model.py:1088-1089)
    @property
    def device(self):
        return self._t.device

    @property
    def eos_ids(self):
        return self._eos_ids

    @eos_ids.setter
    def eos_ids(self, v):
        v = list(v) if v is not None else [None]
        if v == self._eos_ids:
            return
        ids = [int(e) for e in v if e is not None]
        arr = (C.c_int32 * max(len(ids), 1))(*ids)
        with torch.cuda.device(self._t.device):
            L.check(self._t.lib.pia_trie_set_eos(self._t.h, arr, len(ids)))
        self._eos_ids = v

    @property
    def stop_words(self):
        return self._stop_words

    @stop_words.setter
    def stop_words(self, v):
        v = v if v is not None else {}
        if self._stop_words is not None and set(v) == set(self._stop_words):
            self._stop_words = v
            return
        ids = sorted(int(x) for x in v)
        arr = (C.c_int32 * max(len(ids), 1))(*ids)
        with torch.cuda.device(self._t.device):
            L.check(self._t.lib.pia_trie_set_stop_words(self._t.h, arr, len(ids)))
        self._stop_words = v

    @property
    def max_node(self):
        return self._max_node

    @max_node.setter
    def max_node(self, v):
        self._max_node = int(v)
        with torch.cuda.device(self._t.device):
            L.check(self._t.lib.pia_trie_set_limits(self._t.h, self._max_node, self._max_output_node))

    @property
    def max_output_node(self):
        return self._max_output_node

    @max_output_node.setter
    def max_output_node(self, v):
        self._max_output_node = int(v)
        with torch.cuda.device(self._t.device):
            L.check(self._t.lib.pia_trie_set_limits(self._t.h, self._max_node, self._max_output_node))

    # ---- helpers
    def _tokens(self, token_ids):
        n = len(token_ids)
        t = torch.tensor(list(token_ids) if n else [0], dtype=torch.int32).pin_memory() if n > 64 else \
            torch.tensor(list(token_ids) if n else [0], dtype=torch.int32)
        return t.to(self._t.device, non_blocking=True), n

    # ---- writes
    def put(self, token_ids, branch_length=8, final=False, mode='output', idx=0):
        """reference :349-373"""
        assert mode in ('input', 'output')
        d, n = self._tokens(token_ids)
        with torch.cuda.device(self._t.device):
            L.check(self._t.lib.pia_trie_put(self._t.h, d.data_ptr(), n, None, branch_length, L.MODE[mode], idx,
                                             int(final), self._t.stream()))

    def stream_put(self, token_ids, branch_length=8, final=False, mode='output', idx=0):
        """reference :375-406"""
        assert mode == 'output' and idx >= 0
        d, n = self._tokens(token_ids)
        with torch.cuda.device(self._t.device):
            L.check(self._t.lib.pia_trie_stream_put(self._t.h, d.data_ptr(), n, None, branch_length, idx, None,
                                                    int(final), self._t.stream()))

    def put_device(self, d_tokens, n_max, d_n=None, branch_length=8, final=False, mode='output', idx=0):
        """put() on tokens already in HBM (int32 tensor); the live length may itself be a device scalar"""
        L.check(self._t.lib.pia_trie_put(self._t.h, d_tokens.data_ptr(), n_max,
                                         d_n.data_ptr() if d_n is not None else None, branch_length, L.MODE[mode],
                                         idx, int(final), self._t.stream()))

    def stream_put_device(self, d_tokens, n_max, d_n=None, branch_length=8, final=False, idx=0, d_idx=None):
        """stream_put() on tokens in HBM; `d_idx` (int32 device scalar) overrides idx on the device: the batched
        loop's slot -> request map changes as requests finish (pretrained_model_batch.py:937-980)"""
        L.check(self._t.lib.pia_trie_stream_put(self._t.h, d_tokens.data_ptr(), n_max,
                                                d_n.data_ptr() if d_n is not None else None, branch_length, idx,
                                                d_idx.data_ptr() if d_idx is not None else None, int(final),
                                                self._t.stream()))

    # ---- reads
    def _get_batch(self, queries, decoding_length, branch_length, min_input_size, min_output_size, mode, indices,
                   kind, flags=0):
        bs = len(queries)
        stride = max(max(len(q) for q in queries), 1)
        assert stride <= 16, 'query longer than 16 tokens'
        host = np.zeros((bs, stride), dtype=np.int32)
        qlen = np.zeros((bs,), dtype=np.int32)
        for b, q in enumerate(queries):
            host[b, :len(q)] = q
            qlen[b] = len(q)
        dev = self._t.device
        dq = torch.from_numpy(host).to(dev)
        dl = torch.from_numpy(qlen).to(dev)
        didx = torch.tensor(list(indices), dtype=torch.int32, device=dev)
        cap = max(decoding_length, 1)
        o = self._t.out_buffers(bs, cap)
        with torch.cuda.device(dev):
            L.check(self._t.lib.pia_trie_get(self._t.h, dq.data_ptr(), dl.data_ptr(), bs, stride, stride,
                                             didx.data_ptr(), 0, cap, branch_length, min_input_size, min_output_size,
                                             L.MODE[mode], kind, flags, 0, None, o['ids'].data_ptr(), o['mask'].data_ptr(),
                                             o['n'].data_ptr(), o['sizes'].data_ptr(), o['nsizes'].data_ptr(),
                                             o['status'].data_ptr(), self._t.stream()))
        ids = o['ids'].cpu().numpy()
        mask = o['mask'].cpu().numpy().view(np.uint64)
        ns = o['n'].cpu().numpy()
        sizes = o['sizes'].cpu().numpy()
        nsizes = o['nsizes'].cpu().numpy()
        status = o['status'].cpu().numpy()
        out = []
        for b in range(bs):
            if status[b] != 0:
                L.check(int(status[b]))
            n = int(ns[b])
            m = _bits_to_mask(mask[b], n) if n > 0 else self.default_mask
            out.append((ids[b, :n].tolist(), m, sizes[b, :int(nsizes[b])].tolist()))
        return out

    def hier_get(self, token_ids, decoding_length=64, branch_length=8, min_input_size=0, min_output_size=0,
                 mode='mix', idx=0):
        """reference :408-439"""
        assert mode in ('input', 'output', 'mix')
        return self._get_batch([list(token_ids)], decoding_length, branch_length, min_input_size, min_output_size,
                               mode, [idx], L.GET_HIER)[0]

    def one_get(self, token_ids, decoding_length=64, branch_length=8, min_input_size=0, min_output_size=0,
                mode='mix', idx=0):
        """reference :490-517"""
        assert mode in ('input', 'output', 'mix')
        return self._get_batch([list(token_ids)], decoding_length, branch_length, min_input_size, min_output_size,
                               mode, [idx], L.GET_ONE)[0]

    def par_get(self, token_ids, decoding_length=16, branch_length=8, min_input_size=0, min_output_size=0,
                mode='mix', idx=0):
        """reference :441-488: re-express hier_get's tree as independent root-to-leaf branches"""
        tree_ids, tree_mask, _ = self.hier_get(token_ids, decoding_length=decoding_length,
                                               branch_length=branch_length, min_input_size=min_input_size,
                                               min_output_size=min_output_size, mode=mode, idx=idx)
        n_draft = len(tree_ids) - 1
        paths = []
        for row in range(n_draft, 0, -1):
            anc = frozenset(np.flatnonzero(tree_mask[row, 1:]).tolist())
            if not any(anc <= seen for seen in paths):
                paths.append(anc)
        paths.reverse()
        used, ids, spans = 0, [tree_ids[0]], []
        for anc in paths:
            cols = sorted(anc)[:n_draft - used]
            ids.extend(tree_ids[c + 1] for c in cols)
            spans.append(len(cols))
            used += len(cols)
            if used >= n_draft:
                break
        masks = np.tril(np.ones((used + 1, used + 1)), 0)
        at = 1
        for span in spans:
            masks[at:at + span, 1:at] = 0
            at += span
        return ids, masks, [at - 1]

    def bat_get(self, token_id_list, decoding_length=64, branch_length=8, decoding_cursors=None, mode='output',
                indices=None, decoding_mode='hier'):
        """reference :519-561 -- all rows go to the GPU in ONE batched get launch"""
        assert mode in ('input', 'output', 'mix')
        assert decoding_mode in ('hier', 'one')
        bs = len(token_id_list)
        assert bs == len(decoding_cursors) and bs == len(indices), \
            f'{bs=} {len(decoding_cursors)=} {len(indices)=}'
        share = decoding_length // bs
        rows = self._get_batch([list(q) for q in token_id_list], share, branch_length, 0, max(share // 2, 1), mode,
                               indices, L.GET_HIER if decoding_mode == 'hier' else L.GET_ONE)
        lo, hi = min(decoding_cursors), max(decoding_cursors)
        widest = max(len(r[0]) for r in rows)
        masks = np.zeros((bs, widest, hi - lo + widest), dtype=np.int64)
        id_list, size_list = [], []
        for b, (ids, m, sizes) in enumerate(rows):
            k = len(ids)
            shift = decoding_cursors[b] - lo
            masks[b, :k, shift:shift + k] = m
            masks[b, :, :shift + 1] = 1
            id_list.append(ids + [0] * (widest - k))
            size_list.append(sizes)
        return id_list, masks, size_list

    def get_device(self, d_seq, d_seq_len, decoding_length, branch_length, max_query_length=2, min_input_size=0,
                   min_output_size=0, mode='mix', idx=0, kind='hier', max_seq_length=0, out=None, batch=1,
                   d_idx=None, d_max_seq_length=None):
        """hier_get/one_get for the generation loops: the query of row b is the tail of the device token sequence
        d_seq[b, :d_seq_len[b]] (pretrained_model.py:708; batched :705-707) and the drafts stay in HBM.  `out` is a
        dict like out_buffers(batch, dl).  d_idx [batch]: request idx per row (bat_get's `indices`);
        d_max_seq_length: int32 device scalar replacing max_seq_length (the :680 clamp of branch_length)."""
        o = out if out is not None else self._t.out_buffers(batch, max(decoding_length, 1))
        stride = d_seq.shape[-1] if d_seq.dim() == 2 else d_seq.numel()
        L.check(self._t.lib.pia_trie_get(self._t.h, d_seq.data_ptr(), d_seq_len.data_ptr(), int(batch), int(stride),
                                         max_query_length, d_idx.data_ptr() if d_idx is not None else None, idx,
                                         decoding_length, branch_length, min_input_size,
                                         min_output_size, L.MODE[mode], L.GET_HIER if kind == 'hier' else L.GET_ONE,
                                         L.GET_TAIL, max_seq_length,
                                         d_max_seq_length.data_ptr() if d_max_seq_length is not None else None,
                                         o['ids'].data_ptr(), o['mask'].data_ptr(),
                                         o['n'].data_ptr(), o['sizes'].data_ptr(), o['nsizes'].data_ptr(),
                                         o['status'].data_ptr(), self._t.stream()))
        return o

    # ---- maintenance
    def fresh(self):
        """reference :563-564"""
        with torch.cuda.device(self._t.device):
            L.check(self._t.lib.pia_trie_fresh(self._t.h, self._t.stream()))

    def reset_input_freqs(self, idx):
        """reference :566-570"""
        with torch.cuda.device(self._t.device):
            L.check(self._t.lib.pia_trie_reset_input_freqs(self._t.h, idx, self._t.stream()))

    def squeeze_branch_counts(self):
        """reference :572-576"""
        with torch.cuda.device(self._t.device):
            L.check(self._t.lib.pia_trie_squeeze_branch_counts(self._t.h, self._t.stream()))

    def copy_error_flags_device(self, d_out):
        """sticky pool-exhaustion bits -> int32 device scalar, on the current stream (capturable)"""
        L.check(self._t.lib.pia_trie_copy_error_flags(self._t.h, d_out.data_ptr(), self._t.stream()))

    def stats(self):
        s = L.TrieStats()
        with torch.cuda.device(self._t.device):
            L.check(self._t.lib.pia_trie_stats(self._t.h, C.byref(s), self._t.stream()))
        return {k: getattr(s, k) for k, _ in s._fields_}

    def compact(self):
        """reclaims the storage of squeezed / abandoned nodes and child blocks (pia_trie_compact): the reachable forest
        is copied to the front of the pools; nothing a get / put can observe changes.  Returns (nodes before, after).
        The reference gets this from Python's garbage collector (Tree._squeeze pops nodes, lookahead_cache.py:302-310)."""
        a, b = C.c_int64(0), C.c_int64(0)
        with torch.cuda.device(self._t.device):
            L.check(self._t.lib.pia_trie_compact(self._t.h, C.byref(a), C.byref(b), self._t.stream()))
        return a.value, b.value

    def maybe_compact(self, threshold=0.75):
        """compact() once a pool is more than `threshold` full; the generation loops call this between requests.  If
        the forest itself (not garbage) fills the pools the warning of warn_trie_errors() still applies."""
        s = self.stats()
        if s['nodes_used'] > threshold * self._node_capacity or s['edges_used'] > threshold * self._edge_capacity:
            return self.compact()
        return None

    def tree_counters(self, token_id):
        a, b = C.c_int64(0), C.c_int64(0)
        with torch.cuda.device(self._t.device):
            L.check(self._t.lib.pia_trie_tree_counters(self._t.h, int(token_id), C.byref(a), C.byref(b),
                                                       self._t.stream()))
        return a.value, b.value

    # ---- persistence (reference :578-587): the file is json(json(pickle(mem).decode('latin-1'))) with
    #      mem = {token: Tree}, Tree/Node being the reference's classes; they are re-created here by name so that
    #      files written by either implementation load in the other
    def _export_arrays(self):
        t = self._t
        nn, ne = C.c_int64(0), C.c_int64(0)
        with torch.cuda.device(t.device):
            L.check(t.lib.pia_trie_export_sizes(t.h, C.byref(nn), C.byref(ne), t.stream()))
        nodes = np.zeros((max(nn.value, 1),), dtype=_NODE_DTYPE)
        edges = np.zeros((max(ne.value, 1), 2), dtype=np.int32)
        V = t.cfg.vocab_capacity
        root_of = np.zeros((V,), dtype=np.int32)
        n_node = np.zeros((V,), dtype=np.int32)
        n_out = np.zeros((V,), dtype=np.int32)
        with torch.cuda.device(t.device):
            L.check(t.lib.pia_trie_export(t.h, nodes.ctypes.data, nn.value, edges.ctypes.data, ne.value,
                                          root_of.ctypes.data, n_node.ctypes.data, n_out.ctypes.data, t.stream()))
        return nodes[:nn.value], edges[:ne.value], root_of, n_node, n_out

    def snapshot(self):
        """the forest as raw host arrays (pia_trie_export); restore() puts it back.  Pending stream_put carries and
        the touched-tree lists are not part of it: take it between requests."""
        return self._export_arrays()

    def restore(self, snap):
        nodes, edges, root_of, n_node, n_out = snap
        nodes = np.ascontiguousarray(nodes) if len(nodes) else np.zeros((1,), dtype=_NODE_DTYPE)
        edges = np.ascontiguousarray(edges) if len(edges) else np.zeros((1, 2), dtype=np.int32)
        t = self._t
        with torch.cuda.device(t.device):
            L.check(t.lib.pia_trie_import(t.h, nodes.ctypes.data, len(snap[0]), edges.ctypes.data, len(snap[1]),
                                          root_of.ctypes.data, n_node.ctypes.data, n_out.ctypes.data, t.stream()))

    def to_reference_mem(self):
        """the forest as the reference's `mem` structure: {token: Tree} of nested Node dicts"""
        nodes, edges, root_of, n_node, n_out = self._export_arrays()
        tok, nch, child, cap = nodes['token'], nodes['n_child'], nodes['child'], nodes['cap']
        fo, fi = nodes['fo'], nodes['fi']

        def kids(i):
            if nch[i] == 0:
                return []
            if cap[i] == 0:
                return [int(child[i])]
            return edges[child[i]:child[i] + nch[i], 1].tolist()

        def build(i):
            # iterative post-order (tries are at most branch_length+1 deep, but fan-out can be large)
            freqs = {}
            if fo[i] != 0.0 or fi[i] == 0.0:
                freqs[-1] = float(fo[i])
            if fi[i] != 0.0:
                freqs[0] = float(fi[i])
            return _RefNode({int(tok[c]): build(c) for c in kids(i)}, freqs)

        mem = {}
        for token in np.flatnonzero(root_of >= 0).tolist():
            r = int(root_of[token])
            tree = _RefTree.__new__(_RefTree)
            tree.token_id = token
            tree.max_node, tree.max_output_node = self._max_node, self._max_output_node
            tree.n_node, tree.n_output_node = int(n_node[token]), int(n_out[token])
            tree.nodes = {int(tok[c]): build(c) for c in kids(r)}
            mem[token] = tree
        return mem

    def from_reference_mem(self, mem):
        """replace the forest by a reference-format `mem` ({token: Tree}); freqs[-1] -> fo, freqs[0] -> fi"""
        recs, edges = [], []
        V = self._t.cfg.vocab_capacity
        root_of = np.full((V,), -1, dtype=np.int32)
        n_node = np.zeros((V,), dtype=np.int32)
        n_out = np.zeros((V,), dtype=np.int32)

        def add(token, node):
            i = len(recs)
            fr = getattr(node, 'freqs', {}) if node is not None else {}
            recs.append([token, 0, -1, 0, float(fr.get(-1, 0.0)), float(fr.get(0, 0.0))])
            return i

        def link(i, children):  # children: dict token -> Node, in insertion order
            ids = [add(int(tk), nd) for tk, nd in children.items()]
            recs[i][1] = len(ids)
            if len(ids) == 1:
                recs[i][2] = ids[0]
            elif len(ids) > 1:
                cap_ = 4
                while cap_ < len(ids):
                    cap_ *= 2
                recs[i][2], recs[i][3] = len(edges), cap_
                edges.extend([[int(tk), c] for tk, c in zip(children.keys(), ids)])
                edges.extend([[0, 0]] * (cap_ - len(ids)))
            for c, nd in zip(ids, children.values()):
                link(c, nd.children)

        for token, tree in mem.items():
            token = int(token)
            assert 0 <= token < V
            r = add(token, None)
            root_of[token] = r
            n_node[token], n_out[token] = int(tree.n_node), int(tree.n_output_node)
            link(r, tree.nodes)
        nodes = np.zeros((max(len(recs), 1),), dtype=_NODE_DTYPE)
        for i, (tk, nc, ch, cp, fo_, fi_) in enumerate(recs):
            nodes[i] = (tk, nc, ch, cp, fo_, fi_, 0)
        ed = np.asarray(edges if edges else [[0, 0]], dtype=np.int32)
        t = self._t
        with torch.cuda.device(t.device):
            L.check(t.lib.pia_trie_import(t.h, nodes.ctypes.data, len(recs), ed.ctypes.data, len(edges),
                                          root_of.ctypes.data, n_node.ctypes.data, n_out.ctypes.data, t.stream()))

    def save_mem(self, save_dir):
        """reference :578-582"""
        import json
        import pickle
        import io

        class _P(pickle._Pickler):  # writes the reference's class names without needing that package installed
            def save_global(self, obj, name=None):
                if obj is _RefTree or obj is _RefNode:
                    self.write(pickle.GLOBAL + b'lookahead.common.lookahead_cache\n' + obj.__name__.encode() + b'\n')
                    self.memoize(obj)
                    return
                super().save_global(obj, name)

        buf = io.BytesIO()
        _P(buf, protocol=4).dump(self.to_reference_mem())
        serialized_object = buf.getvalue()
        json_string = json.dumps(serialized_object.decode('latin-1'))
        with open(save_dir, 'w') as f:
            json.dump(json_string, f)

    def load_mem(self, load_dir):
        """reference :584-587"""
        import io
        import json
        import pickle
        with open(load_dir, 'r') as f:
            json_string = json.load(f)

        class _U(pickle.Unpickler):
            def find_class(self, module, name):
                if module.endswith('lookahead_cache') and name == 'Tree':
                    return _RefTree
                if module.endswith('lookahead_cache') and name == 'Node':
                    return _RefNode
                return super().find_class(module, name)

        self.from_reference_mem(_U(io.BytesIO(json.loads(json_string).encode('latin-1'))).load())


_NODE_DTYPE = np.dtype([('token', '<i4'), ('n_child', '<i4'), ('child', '<i4'), ('cap', '<i4'), ('fo', '<f8'),
                        ('fi', '<f4'), ('aux', '<i4')])


class _RefNode(object):
    """pickles as the reference's lookahead.common.lookahead_cache.Node (:13-21)"""
    __slots__ = ['freqs', 'children']

    def __init__(self, children, freqs):
        self.children = children
        self.freqs = freqs


class _RefTree(object):
    """pickles as the reference's lookahead.common.lookahead_cache.Tree (:24-31); data only"""
    pass


_RefNode.__module__ = _RefTree.__module__ = 'lookahead.common.lookahead_cache'
_RefNode.__qualname__ = _RefNode.__name__ = 'Node'
_RefTree.__qualname__ = _RefTree.__name__ = 'Tree'


class Tree(object):
    """Drop-in for the reference's Tree (:24-333) for callers/tests that build a single tree by hand.
    Backed by a private one-tree device trie."""

    def __init__(self, token_id, max_node=65536, max_output_node=512, device=None):
        self.token_id = token_id
        self.max_node = max_node
        self.max_output_node = max_output_node
        self._c = LookaheadCache(eos_ids=None, max_node=max_node, max_output_node=max_output_node, device=device,
                                 node_capacity=1 << 20, max_resident_queries=4, frontier_capacity=1 << 16)

    def put(self, token_ids, mode='output', idx=0, freq=1.0):
        """reference :33-37"""
        assert mode in ('input', 'output')
        assert freq == 1.0, 'only unit increments exist on the reference path'
        d, n = self._c._tokens(token_ids)
        t = self._c._t
        with torch.cuda.device(t.device):
            L.check(t.lib.pia_trie_tree_put(t.h, int(self.token_id), d.data_ptr(), n, L.MODE[mode],
                                            max(idx, 0), t.stream()))

    def get(self, token_ids, max_size=64, max_length=8, min_input_size=0, min_output_size=0, output_weight=1e-4,
            mode='mix', idx=0):
        """reference :65-144"""
        assert mode in ('input', 'output', 'mix')
        assert output_weight == 1e-4, 'the kernels implement the reference default output_weight=1e-4'
        return self._c._get_batch([[self.token_id] + list(token_ids)], max_size, max_length, min_input_size,
                                  min_output_size, mode, [idx], L.GET_HIER, flags=L.GET_FIRST_ONLY)[0]

    def get_one_branch(self, token_ids, max_length=8, mode='mix', idx=0):
        """reference :171-222"""
        return self._c._get_batch([[self.token_id] + list(token_ids)], 64, max_length, 0, 0, mode, [idx],
                                  L.GET_ONE, flags=L.GET_FIRST_ONLY)[0]

    def squeeze(self):
        """reference :295-301"""
        t = self._c._t
        with torch.cuda.device(t.device):
            L.check(t.lib.pia_trie_set_limits(t.h, int(self.max_node), int(self.max_output_node)))
            L.check(t.lib.pia_trie_tree_squeeze(t.h, int(self.token_id), t.stream()))

    def reset_input_freq(self, idx):
        """reference :320-333"""
        t = self._c._t
        with torch.cuda.device(t.device):
            L.check(t.lib.pia_trie_tree_reset_input_freq(t.h, int(self.token_id), int(idx), t.stream()))

    @property
    def n_node(self):
        return max(self._c.tree_counters(self.token_id)[0], 0)   # an empty Tree counts 0 nodes (reference :29)

    @property
    def n_output_node(self):
        return max(self._c.tree_counters(self.token_id)[1], 0)
