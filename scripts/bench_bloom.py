# -*- coding: utf-8 -*-
"""BLOOM on one H100: bench.py's workload on the BLOOM-7b1 and BLOOM-560m shapes, and pia_layernorm / pia_bloom_gelu
against their eager torch equivalents.

    python scripts/bench_bloom.py [--steps K] [--warmup W] [--skip-loop]

Loop: bench.py's workload (256-token phrase-bank prompts -> 256 new tokens, 64-token / 8-branch drafts), a trie warmed
on other prompts, then a first and a second pass over the timed prompts.  Weights: synth_fill_bloom (bench.py's
hashed fill under BLOOM's parameter names, untied lm_head, LayerNorm weights 1, biases 0).  Shapes: BLOOM-7b1 (30
layers, 4096, 32 heads of 128, V = 250 880) and BLOOM-560m (24 layers, 1024, 16 heads of 64, run zero-padded to 128).
The weight bytes per step are computed from the shapes.
Kernels: pia_layernorm with a residual vs `F.layer_norm(x + r)` and pia_bloom_gelu vs transformers'
bloom_gelu_forward, at 64 and 256 rows (hidden 4096, 4h = 16384), CUDA-graph replays timed with CUDA events, median
of 5; GB/s of the algorithmic bytes (every input read once, every output written once).  The card's name and power
limit are read in the same run.  One JSON line on stdout."""
import argparse
import json
import os
import sys
import zlib

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bench  # noqa: E402
from scripts.bench_baichuan import power_limit  # noqa: E402
from scripts.bench_glm import HBM_PEAK_GBS, loop_numbers  # noqa: E402


def bloom_7b1_config():
    from transformers import BloomConfig
    return BloomConfig(vocab_size=250880, hidden_size=4096, n_layer=30, n_head=32, layer_norm_epsilon=1e-5,
                       bos_token_id=1, eos_token_id=2, pad_token_id=3, tie_word_embeddings=False)


def bloom_560m_config():
    from transformers import BloomConfig
    return BloomConfig(vocab_size=250880, hidden_size=1024, n_layer=24, n_head=16, layer_norm_epsilon=1e-5,
                       bos_token_id=1, eos_token_id=2, pad_token_id=3, tie_word_embeddings=False)


def synth_fill_bloom(model, seed=0):
    """bench.synth_fill for BLOOM's parameter names: LayerNorm weights 1, biases 0, decoder weights hashed std 0.02,
    word embeddings hashed std bench.EMBED_STD, and the untied lm_head row v = bench.LM_SCALE * the sum of the unit
    embeddings of the tokens t with succ(t) = v (hashed std 0.02 for tokens without a predecessor)"""
    assert model.lm_head.weight is not model.transformer.word_embeddings.weight, 'the fill needs an untied lm_head'
    emb = lm = None
    with torch.no_grad():
        for name, p in model.named_parameters():
            pseed = zlib.crc32(name.encode()) ^ (seed * 7919)
            if 'layernorm' in name or '.ln_f.' in name:
                p.fill_(1.0 if name.endswith('weight') else 0.0)
            elif name.endswith('bias'):
                p.zero_()
            elif name.endswith('word_embeddings.weight'):
                bench.hashed_normal_(p.data, pseed, bench.EMBED_STD)
                emb = p
            else:
                bench.hashed_normal_(p.data, pseed, 0.02)
                if name == 'lm_head.weight':
                    lm = p
        V = emb.shape[0]
        succ = bench.successor_map(V).to(emb.device)
        unit = emb.data.double()
        unit = unit / unit.norm(dim=1, keepdim=True).clamp_min(1e-30)
        acc = torch.zeros_like(unit)
        acc.index_add_(0, succ[3:], unit[3:])
        has = torch.zeros((V,), dtype=torch.bool, device=emb.device)
        has[succ[3:]] = True
        lm.data[has] = (acc[has] * bench.LM_SCALE).to(lm.dtype)
    return model


def shape_bytes(cfg):
    """bf16 bytes of every streamed weight: per layer QKV / dense / h_to_4h / 4h_to_h with their biases and two
    LayerNorms (12 E^2 + 13 E), the embedding LayerNorm and ln_f, and lm_head (the embedding is gathered)"""
    E, L, V = cfg.hidden_size, cfg.n_layer, cfg.vocab_size
    return 2 * (L * (12 * E * E + 13 * E) + 4 * E + V * E)


def shape_numbers(cfg, dev, K, W):
    from painlessinferenceacceleration_b200.models.bloom.modeling_bloom import BloomForCausalLM
    model = synth_fill_bloom(BloomForCausalLM(cfg, device=dev))
    out = loop_numbers(model, cfg, dev, K, W)
    wb = shape_bytes(cfg)
    out['weight_bytes_per_step'] = wb   # bench.weight_bytes_per_step would count word_embeddings as streamed
    out['floor_ms_at_3.35TBs'] = wb / (HBM_PEAK_GBS * 1e9) * 1e3
    for r in (out['first_pass'], out['second_pass']):
        r['weight_stream_frac_of_3.35TBs'] = wb / (r['ms_per_verify_step'] * 1e-3) / 1e9 / HBM_PEAK_GBS
    del model
    torch.cuda.empty_cache()
    return out


def kernel_numbers(dev, reps=5, hidden=4096):
    from transformers.models.bloom.modeling_bloom import bloom_gelu_forward
    from torch.nn import functional as F
    from painlessinferenceacceleration_b200.common import ops
    res = {}
    bf = dict(dtype=torch.bfloat16, device=dev)
    for rows in (64, 256):
        x, r = torch.randn((rows, hidden), **bf), torch.randn((rows, hidden), **bf)
        w, b = torch.ones((hidden,), **bf), torch.zeros((hidden,), **bf)
        ro, y = torch.empty_like(x), torch.empty_like(x)
        a = torch.randn((rows, 4 * hidden), **bf)
        g = torch.empty_like(a)
        arms = {
            'layernorm': (lambda: ops.layernorm(x, r, w, b, 1e-5, ro, y),
                          lambda: F.layer_norm(x + r, (hidden,), w, b, 1e-5), (4 * rows + 2) * hidden * 2),
            'bloom_gelu': (lambda: ops.bloom_gelu(a, out=g), lambda: bloom_gelu_forward(a), 2 * a.numel() * 2),
        }
        for name, (ours, eager, nbytes) in arms.items():
            us = {'ours': [], 'torch_eager': []}
            for _ in range(reps):
                us['ours'].append(bench._graph_time(ours))
                us['torch_eager'].append(bench._graph_time(eager))
            med = {k: float(np.median(v)) for k, v in us.items()}
            res[f'{name}_rows={rows}'] = {'us': med, 'GBps': {k: nbytes / (v * 1e-6) / 1e9 for k, v in med.items()},
                                          'algorithmic_bytes': nbytes, 'us_all': us}
    return res


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
    line['kernels'] = kernel_numbers(dev)
    if not a.skip_loop:
        for name, cfg in (('bloom-7b1', bloom_7b1_config()), ('bloom-560m', bloom_560m_config())):
            line[name] = shape_numbers(cfg, dev, a.steps, a.warmup)
    sampler.stop_flag = True
    sampler.join(timeout=2)
    line['clocks'] = sampler.summary()
    line['gpu'] = torch.cuda.get_device_name(0)
    line['power_limit'] = power_limit()
    print(json.dumps(line))


if __name__ == '__main__':
    main()
