# -*- coding: utf-8 -*-
"""Baichuan family on one H100: bench.py's workload on the Baichuan-13B and Baichuan2-7B shapes in bf16 and fp8, and
k_tree_attn's ALiBi instance against the plain one.

    python scripts/bench_baichuan.py [--steps K] [--warmup W] [--skip-loop]

Loop: bench.py's workload (256-token phrase-bank prompts -> 256 new tokens, 64-token / 8-branch drafts, bench.synth_fill
weights, untied lm_head; Baichuan2's NormHead applied), a trie warmed on other prompts, then a first and a second pass
over the timed prompts.  The fp8 run quantises the same bf16 weights in place (quantize_fp8()).  Shapes: Baichuan-13B
(40 layers, 5120 / 13696, 40 heads, V = 64000, ALiBi) and Baichuan2-7B (32 layers, 4096 / 11008, 32 heads,
V = 125696, fp32 RoPE, NormHead).  The weight bytes per step are computed from the shapes.
Attention: Baichuan-13B heads (40 / 40, head dim 128, 64 draft rows), P = 384 and 3968, one launch per layer over
enough layers that K / V exceed the 50 MB L2, CUDA-graph replay (CUDA events), the two instances alternating in one
process, median of 5.  The card's name and power limit are read in the same run.  One JSON line on stdout."""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bench  # noqa: E402
from scripts.bench_glm import HBM_PEAK_GBS, loop_numbers  # noqa: E402

L2_BYTES = 50 * 2 ** 20


def baichuan_13b_shape():
    from painlessinferenceacceleration_b200.models.baichuan.modeling_baichuan import baichuan_config
    from painlessinferenceacceleration_b200.models.baichuan_13b.modeling_baichuan import BaichuanForCausalLM
    return BaichuanForCausalLM, baichuan_config(dict(
        model_type='baichuan', vocab_size=64000, hidden_size=5120, intermediate_size=13696, num_hidden_layers=40,
        num_attention_heads=40, hidden_act='silu', model_max_length=4096, rms_norm_eps=1e-6, bos_token_id=1,
        eos_token_id=2, pad_token_id=0, tie_word_embeddings=False))


def baichuan2_7b_shape():
    from painlessinferenceacceleration_b200.models.baichuan.modeling_baichuan import baichuan_config
    from painlessinferenceacceleration_b200.models.baichuan2_7b.modeling_baichuan import BaichuanForCausalLM
    return BaichuanForCausalLM, baichuan_config(dict(
        model_type='baichuan', vocab_size=125696, hidden_size=4096, intermediate_size=11008, num_hidden_layers=32,
        num_attention_heads=32, hidden_act='silu', max_position_embeddings=4096, model_max_length=4096,
        rms_norm_eps=1e-6, bos_token_id=1, eos_token_id=2, pad_token_id=0, tie_word_embeddings=False))


def shape_bytes(cfg):
    """bf16 bytes of every decoder / lm_head weight (the embedding is gathered, not streamed)"""
    h, i, L, V = cfg.hidden_size, cfg.intermediate_size, cfg.num_hidden_layers, cfg.vocab_size
    return 2 * (L * (4 * h * h + 3 * h * i + 2 * h) + h + V * h)


def shape_numbers(name, dev, K, W):
    cls, cfg = baichuan_13b_shape() if name == 'baichuan-13b' else baichuan2_7b_shape()
    model = bench.synth_fill(cls(cfg, device=dev), cfg).normalize_lm_head()
    wb = shape_bytes(cfg)
    out = {'weight_bytes_from_shape': wb, 'floor_ms_at_3.35TBs': wb / (HBM_PEAK_GBS * 1e9) * 1e3,
           'bf16': loop_numbers(model, cfg, dev, K, W)}
    model.quantize_fp8()
    out['fp8'] = loop_numbers(model, cfg, dev, K, W)
    del model
    torch.cuda.empty_cache()
    return out


def attn_numbers(dev, reps=5, n=64, R=64, H=40, D=128):
    """k_tree_attn per launch at Baichuan-13B heads: ALiBi instance vs the plain instance, one launch per layer"""
    from painlessinferenceacceleration_b200.common import ops
    rows = np.array([(1 << (i + 1)) - 1 if i < 63 else 0xFFFFFFFFFFFFFFFF for i in range(R)], dtype=np.uint64)
    mask = torch.from_numpy(rows.view(np.int64)).to(dev).view(R, 1)
    q = (torch.randn((R, H, D), device=dev) * 0.7).to(torch.bfloat16)
    out = torch.zeros_like(q)
    slopes = ops.alibi_slopes(H).to(dev)
    res = {}
    for P in (384, 3968):
        max_seq = P + n + 64
        layers = max(4, -(-3 * L2_BYTES // (2 * H * max_seq * D * 2)))   # K + V of all layers >= 3 x L2
        kc = (torch.randn((layers, H, max_seq, D), device=dev) * 0.7).to(torch.bfloat16)
        vc = (torch.randn((layers, H, max_seq, D), device=dev) * 0.7).to(torch.bfloat16)
        plan = ops.AttnPlan(kc, vc, H, H, D, R)
        slots = ops.Slots(torch.tensor([n], dtype=torch.int32, device=dev),
                          torch.tensor([P], dtype=torch.int32, device=dev), None, R)

        def sweep(alibi):
            for li in range(layers):
                plan.forward(li, q, mask, slots, out, alibi_slopes=slopes if alibi else None)

        us = {'alibi': [], 'plain': []}
        for _ in range(reps):
            for kind in ('alibi', 'plain'):
                us[kind].append(bench._graph_time(lambda: sweep(kind == 'alibi')) / layers)
        med = {k: float(np.median(v)) for k, v in us.items()}
        res[f'P={P}'] = {'layers': layers, 'us_per_launch': med, 'us_all': us,
                         'alibi_over_plain': med['alibi'] / med['plain'] - 1.0}
        del plan, kc, vc
        torch.cuda.empty_cache()
    return res


def power_limit():
    try:
        return subprocess.run(['nvidia-smi', '--query-gpu=power.limit', '--format=csv,noheader', '-i', '0'],
                              capture_output=True, text=True, timeout=20).stdout.strip()
    except Exception as e:   # noqa: BLE001
        return f'unavailable: {e}'


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
    line = {'workload': f'{bench.DL}-token/{bench.BL}-branch drafts, {bench.PROMPT_LEN}-token prompts -> '
                        f'{bench.NEW_TOKENS} new tokens, {a.steps} timed requests, {a.warmup} warm-up requests'}
    line['tree_attn'] = attn_numbers(dev)
    if not a.skip_loop:
        for name in ('baichuan-13b', 'baichuan2-7b'):
            line[name] = shape_numbers(name, dev, a.steps, a.warmup)
    sampler.stop_flag = True
    sampler.join(timeout=2)
    line['clocks'] = sampler.summary()
    line['gpu'] = torch.cuda.get_device_name(0)
    line['power_limit'] = power_limit()
    print(json.dumps(line))


if __name__ == '__main__':
    main()
