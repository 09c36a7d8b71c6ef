# -*- coding: utf-8 -*-
"""Qwen (v1) on one H100: k_rope_kv_append's fp32 instance with and without log-n query scaling, and bench.py's
workload on the Qwen-7B shape in bf16 and fp8 with dynamic NTK and log-n live.

    python scripts/bench_qwen.py [--steps K] [--warmup W] [--skip-loop]

Kernel: pia_rope_f32_logn_kv_append against pia_rope_f32_kv_append at Qwen-7B heads (32 / 32, head dim 128), 64 draft
rows of a chain at P = 3968 (every row past seq_length 2048), one launch per layer over 32 layers' caches, CUDA-graph
replay timed with CUDA events, the two entries alternating in one process, median of 7.
Loop: bench.py's workload (256-token phrase-bank prompts -> 256 new tokens, 64-token / 8-branch drafts, bench.synth_fill
weights) on a Qwen-7B-shaped model (32 layers, 4096 hidden, 32 x 128 MHA, 11008 per MLP branch, V = 151936, c_attn
bias) with seq_length 128, below the prompt length: every request runs at NTK alpha 3 and every position past 127 has
its queries scaled.  A trie warmed on other prompts, then a first and a second pass over the timed prompts; the fp8 run
quantises the same bf16 weights in place.  The card's name and power limit are read in the same run.  One JSON line
on stdout."""
import argparse
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bench  # noqa: E402
from scripts.bench_glm import loop_numbers  # noqa: E402


def qwen_7b_shape(seq_length=128):
    from painlessinferenceacceleration_b200.models.qwen.modeling_qwen import QWenLMHeadModel, qwen_config
    return QWenLMHeadModel, qwen_config(dict(
        model_type='qwen', vocab_size=151936, hidden_size=4096, intermediate_size=22016, num_hidden_layers=32,
        num_attention_heads=32, kv_channels=128, layer_norm_epsilon=1e-6, rotary_emb_base=10000, rotary_pct=1.0,
        seq_length=seq_length, max_position_embeddings=32768, use_dynamic_ntk=True, use_logn_attn=True, no_bias=True,
        tie_word_embeddings=False, eos_token_id=2, pad_token_id=0, bos_token_id=1))


def rope_numbers(dev, reps=7, layers=32, H=32, D=128, R=64, P=3968, seq_length=2048):
    """us per k_rope_kv_append launch (64 rows), log-n instance vs the plain fp32 instance"""
    from painlessinferenceacceleration_b200.common import ops
    from painlessinferenceacceleration_b200.models.qwen.modeling_qwen import logn_table, ntk_alpha, rope_tables_f32
    max_seq = P + R + 64
    alpha = ntk_alpha(P, seq_length)
    cos, sin = (t.to(dev) for t in rope_tables_f32(D, 10000, alpha, max_seq + 8))
    scale = logn_table(seq_length, max_seq + 8).to(dev)
    rows = np.array([(1 << (i + 1)) - 1 if i < 63 else 0xFFFFFFFFFFFFFFFF for i in range(R)], dtype=np.uint64)
    mask = torch.from_numpy(rows.view(np.int64)).to(dev).view(R, 1)
    qkv = (torch.randn((R, 3 * H * D), device=dev)).to(torch.bfloat16)
    q = torch.zeros((R, H, D), dtype=torch.bfloat16, device=dev)
    kc = torch.zeros((layers, H, max_seq, D), dtype=torch.bfloat16, device=dev)
    vc = torch.zeros_like(kc)
    slots = ops.Slots(torch.tensor([R], dtype=torch.int32, device=dev), torch.tensor([P], dtype=torch.int32, device=dev),
                      None, R)

    def sweep(logn):
        for li in range(layers):
            ops.rope_kv_append(qkv, mask, slots, H, H, D, cos, sin, q, kc[li], vc[li], max_seq,
                               q_scale=scale if logn else None)

    us = {'logn': [], 'plain': []}
    for _ in range(reps):
        for kind in ('logn', 'plain'):
            us[kind].append(bench._graph_time(lambda: sweep(kind == 'logn'), reps=50) / layers)
    med = {k: float(np.median(v)) for k, v in us.items()}
    return {'rows': R, 'P': P, 'heads': H, 'layers': layers, 'us_per_launch': med, 'us_all': us,
            'logn_over_plain': med['logn'] / med['plain'] - 1.0}


def loop_shape_numbers(dev, K, W):
    cls, cfg = qwen_7b_shape()
    model = bench.synth_fill(cls(cfg, device=dev), cfg)
    out = {'seq_length': cfg.seq_length, 'bf16': loop_numbers(model, cfg, dev, K, W)}
    out['ntk_alpha'] = model._rt.ntk_alpha
    model.quantize_fp8()
    out['fp8'] = loop_numbers(model, cfg, dev, K, W)
    del model
    torch.cuda.empty_cache()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=8)
    ap.add_argument('--warmup', type=int, default=3)
    ap.add_argument('--skip-loop', action='store_true')
    a = ap.parse_args()
    assert torch.cuda.is_available(), 'needs an H100'
    dev = torch.device('cuda', 0)
    torch.cuda.set_device(dev)
    sampler = bench.ClockSampler(0)
    sampler.start()
    line = {'workload': f'Qwen-7B shape, seq_length 128, {bench.DL}-token/{bench.BL}-branch drafts, '
                        f'{bench.PROMPT_LEN}-token prompts -> {bench.NEW_TOKENS} new tokens, {a.steps} timed requests, '
                        f'{a.warmup} warm-up requests'}
    line['rope_kv_append'] = rope_numbers(dev)
    if not a.skip_loop:
        line['qwen-7b'] = loop_shape_numbers(dev, a.steps, a.warmup)
    sampler.stop_flag = True
    sampler.join(timeout=2)
    line['clocks'] = sampler.summary()   # gpu name, power limit (W), SM clock during the run
    line['gpu'] = torch.cuda.get_device_name(0)
    print(json.dumps(line))


if __name__ == '__main__':
    main()
