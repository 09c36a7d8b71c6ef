# -*- coding: utf-8 -*-
"""Warm, graph-replayed device timings of the individual pieces of one verify step (Llama-2-7B shape by default).
CUDA events around `reps` replays of a graph that holds `per` launches of one piece; no profiler attached."""
import argparse
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import bench  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument('--model', default='llama2-7b')
ap.add_argument('--P', type=int, default=384)
ap.add_argument('--n', type=int, default=64)
ap.add_argument('--max-seq', type=int, default=577)
ap.add_argument('--forward-only', action='store_true')
a = ap.parse_args()
from painlessinferenceacceleration_b200.common import ops  # noqa: E402
from painlessinferenceacceleration_b200.common.lookahead_cache import LookaheadCache  # noqa: E402
from painlessinferenceacceleration_b200.models.llama.modeling_llama import LlamaForCausalLM  # noqa: E402

dev = torch.device('cuda:0')
cfg, _ = bench.make_config(a.model)
model = LlamaForCausalLM(cfg, device=dev).init_weights(seed=0).requires_grad_(False)
model.fuse()
rt = model._runtime(a.max_seq, 64)
rt.mask.copy_(rt.chain)
rt.n.fill_(a.n)
draft = dict(ids=rt.ids, mask=rt.mask, n=rt.n, sizes=rt.sizes, nsizes=rt.nsizes, status=rt.status)
rt.prefix_len.fill_(a.P)
g = rt.g
L0 = model.model.layers[0]


def timeit(name, fn, per, reps=20, bytes_per=None):
    fn()
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        fn()
    graph.replay()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    for _ in range(reps):
        graph.replay()
    e1.record()
    torch.cuda.synchronize()
    us = e0.elapsed_time(e1) * 1e3 / (reps * per)
    extra = f'  {bytes_per / us / 1e3:8.1f} GB/s' if bytes_per else ''
    print(f'{name:34s} {us:9.2f} us/launch{extra}', flush=True)
    return us


NL = g['n_layers']
layers = model.model.layers
if a.forward_only:
    timeit('verify layers (whole forward)', lambda: model._verify_layers(rt), 1,
           bytes_per=sum(p.numel() for p in model.parameters()) * 2)
    sys.exit(0)
L = a.P + a.n
kv_bytes = 2 * L * g['n_kv_heads'] * g['head_dim'] * 2 + 2 * a.n * g['n_q_heads'] * g['head_dim'] * 2
timeit('tree_attn+combine (32 layers)', lambda: [rt.plan.forward(li, rt.q, rt.mask, rt.decode_bufs.slots, rt.attn) for li in range(NL)], NL, bytes_per=kv_bytes)
timeit('rmsnorm', lambda: [ops.rmsnorm(rt.h, rt.resid, layers[li].input_layernorm.weight, 1e-5, rt.resid, rt.y) for li in range(NL)], NL)
timeit('rope_kv_append', lambda: [ops.rope_kv_append(rt.qkv, rt.mask, rt.decode_bufs.slots, g['n_q_heads'], g['n_kv_heads'], g['head_dim'], rt.rope_cos, rt.rope_sin, rt.q, rt.k_layer(li), rt.v_layer(li), rt.max_seq) for li in range(NL)], NL)
gu = torch.zeros((64, 2 * g['inter']), dtype=torch.bfloat16, device=dev)
act = torch.zeros((64, g['inter']), dtype=torch.bfloat16, device=dev)
timeit('silu_mul', lambda: [ops.silu_mul(gu, act) for _ in range(NL)], NL)
hid = g['hidden']
qkv_w = [l.self_attn.qkv_weight for l in layers]
timeit('gemm qkv', lambda: [torch.mm(rt.y, w.t(), out=rt.qkv) for w in qkv_w], NL, bytes_per=qkv_w[0].numel() * 2)
timeit('gemm o', lambda: [torch.mm(rt.attn, l.self_attn.o_proj.weight.t()) for l in layers], NL, bytes_per=hid * hid * 2)
timeit('gemm gate_up', lambda: [torch.mm(rt.y, l.mlp.gate_up_weight.t(), out=gu) for l in layers], NL, bytes_per=2 * g['inter'] * hid * 2)
timeit('gemm down', lambda: [torch.mm(act, l.mlp.down_proj.weight.t()) for l in layers], NL, bytes_per=g['inter'] * hid * 2)
timeit('gemm lm_head', lambda: torch.mm(rt.y, model.lm_head.weight.t()), 1, bytes_per=g['vocab'] * hid * 2)
timeit('verify layers (whole forward)', lambda: model._verify_layers(rt), 1, bytes_per=sum(p.numel() for p in model.parameters()) * 2)
# single-request trie get on a warmed trie
trie = LookaheadCache(eos_ids=[2], device=dev, vocab_capacity=cfg.vocab_size)
docs = bench.phrase_bank_prompts(64, cfg.vocab_size, seed=3)
for d in docs:
    trie.put(d, branch_length=9, mode='output', idx=-1)
rt.seq[0, :256] = torch.tensor(docs[0], dtype=torch.int32, device=dev)
rt.seq_len.fill_(200)
timeit('trie get (1 query, tail mode)', lambda: trie.get_device(rt.seq, rt.seq_len, 64, 8, min_output_size=32, out=draft), 1)
print('draft n =', int(rt.n))

import sys; sys.exit(0) if __import__("os").environ.get("PIA_ATTN_TILES_PER_CTA") else None
# single-request trie get on a large forest (1 M nodes), hot and cold queries
big = LookaheadCache(eos_ids=[2], device=dev, vocab_capacity=cfg.vocab_size, node_capacity=1 << 23)
docs = bench.phrase_bank_prompts(1500, cfg.vocab_size, seed=7)
for d in docs:
    big.put(d, branch_length=9, mode='output', idx=-1)
st0 = big.stats()
for name, q in (('hot (3,3)', [3, 3]), ('doc pair', docs[5][100:102]), ('rare', docs[7][40:42])):
    rt.seq[0, :2] = torch.tensor(q, dtype=torch.int32, device=dev)
    rt.seq_len.fill_(2)
    s0 = big.stats()
    us = timeit(f'trie get 1M-node forest, {name}', lambda: big.get_device(rt.seq, rt.seq_len, 64, 8, min_output_size=32, out=draft), 1)
    s1 = big.stats()
    print('   draft n =', int(rt.n), ' nodes visited per call ~', (s1['nodes_visited'] - s0['nodes_visited']) // 22)
