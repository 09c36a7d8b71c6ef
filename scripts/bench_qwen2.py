# -*- coding: utf-8 -*-
"""Qwen2-7B-shaped lookahead loop and tree attention at an odd GQA group, on one H100.

    python scripts/bench_qwen2.py [--steps K] [--warmup W] [--layers N]

Loop: bench.py's workload (256-token phrase-bank prompts -> 256 new tokens, 64-token / 8-branch drafts, synthetic
weights of bench.synth_fill) on a Qwen2-7B-shaped model: 3584 hidden, 18944 inter, 28 layers, 28 query heads over 4
KV heads (G = 7), V = 152064, rope_theta 1e6, q/k/v biases.  First pass over prompts the trie has never seen (after
a warm-up on other prompts), then a second pass that has seen every answer once.
Attention: k_tree_attn alone, 64 draft rows, one launch per layer over `--layers` layers in turn (CUDA-graph replay,
CUDA events), G = 7 (28 / 4) against G = 8 (32 / 4) at the same Hkv and P, the two shapes alternating in one process.
One JSON line on stdout."""
import argparse
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bench  # noqa: E402

HBM_PEAK_GBS = 3350.0   # H100 SXM data sheet (700 W); a reference point, not a reached rate


def qwen2_7b_config():
    from transformers import Qwen2Config
    return Qwen2Config(vocab_size=152064, hidden_size=3584, intermediate_size=18944, num_hidden_layers=28,
                       num_attention_heads=28, num_key_value_heads=4, max_position_embeddings=4096, rms_norm_eps=1e-6,
                       rope_theta=1000000.0, use_sliding_window=False, tie_word_embeddings=False,
                       bos_token_id=1, eos_token_id=2, pad_token_id=0)


def loop_numbers(dev, K, W):
    from painlessinferenceacceleration_b200.common.lookahead_cache import LookaheadCache
    from painlessinferenceacceleration_b200.models.qwen2.modeling_qwen2 import Qwen2ForCausalLM
    cfg = qwen2_7b_config()
    model = bench.synth_fill(Qwen2ForCausalLM(cfg, device=dev), cfg)
    model.lookahead_cache = LookaheadCache(eos_ids=[2], device=dev, vocab_capacity=cfg.vocab_size)
    allp = bench.phrase_bank_prompts(64 + 8 * max(W, 1), cfg.vocab_size)
    timed = [allp[j] for j in bench.timed_requests(K)]
    warm = [allp[64 + i % (8 * max(W, 1))] for i in range(W)]
    gen = dict(max_new_tokens=bench.NEW_TOKENS, eos_token_id=2, return_dict_in_generate=True,
               decoding_kwargs={'use_lookahead': True, 'decoding_length': bench.DL, 'branch_length': bench.BL})
    for p in warm:
        model.generate(input_ids=torch.tensor([p], device=dev), **gen)

    def timed_pass():
        ins = [torch.tensor([p], device=dev) for p in timed]
        toks, edls = 0, []
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        e0.record()
        for x in ins:
            o = model.generate(input_ids=x, **gen)
            toks += o.sequences.shape[1] - bench.PROMPT_LEN
            edls += o.kwargs['edls'][1:]
        e1.record()
        torch.cuda.synchronize()
        ms = e0.elapsed_time(e1)
        return {'tokens_per_s': toks / (ms / 1e3), 'mean_accepted_len_per_step': float(np.mean(edls)),
                'verify_steps': len(edls), 'ms_per_verify_step': ms / len(edls)}

    first = timed_pass()
    second = timed_pass()
    wbytes = bench.weight_bytes_per_step(model)
    for r in (first, second):
        r['weight_stream_frac_of_3.35TBs'] = wbytes / (r['ms_per_verify_step'] * 1e-3) / 1e9 / HBM_PEAK_GBS
    del model
    torch.cuda.empty_cache()
    return {'first_pass': first, 'second_pass': second, 'weight_bytes_per_step': wbytes}


def attention_numbers(dev, layers, reps=5):
    """k_tree_attn per launch at G = 7 and G = 8 (Hkv = 4), P = 384 and 3968, alternating"""
    from painlessinferenceacceleration_b200.common import ops
    D, R, n, hkv = 128, 64, 64, 4
    rows = np.array([(1 << (i + 1)) - 1 if i < 63 else 0xFFFFFFFFFFFFFFFF for i in range(R)], dtype=np.uint64)
    mask = torch.from_numpy(rows.view(np.int64)).to(dev).view(R, 1)
    out = {}
    for P in (384, 3968):
        max_seq = P + n + 64
        kc = (torch.randn((layers, hkv, max_seq, D), device=dev) * 0.5).to(torch.bfloat16)
        vc = (torch.randn((layers, hkv, max_seq, D), device=dev) * 0.5).to(torch.bfloat16)
        slots = ops.Slots(torch.tensor([n], dtype=torch.int32, device=dev),
                          torch.tensor([P], dtype=torch.int32, device=dev), None, R)
        runs = {}
        for hq in (28, 32):
            q = (torch.randn((R, hq, D), device=dev) * 0.5).to(torch.bfloat16)
            o = torch.zeros_like(q)
            plan = ops.AttnPlan(kc, vc, hq, hkv, D, R)

            def sweep(plan=plan, q=q, o=o):
                for li in range(layers):
                    plan.forward(li, q, mask, slots, o)
            runs[hq] = (sweep, [])
        for _ in range(reps):
            for hq in (28, 32):
                sweep, us = runs[hq]
                us.append(bench._graph_time(sweep) / layers)
        L = P + n
        kv_bytes = 2 * L * hkv * D * 2
        for hq in (28, 32):
            us = float(np.median(runs[hq][1]))
            out[f'G{hq // hkv}_P{P}'] = {'us_per_launch': us, 'us_all': runs[hq][1], 'kv_bytes': kv_bytes,
                                         'kv_gbs': kv_bytes / (us * 1e-6) / 1e9,
                                         'kv_set_mb': layers * kv_bytes / 2 ** 20}
        del kc, vc
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=8)
    ap.add_argument('--warmup', type=int, default=3)
    ap.add_argument('--layers', type=int, default=28)
    ap.add_argument('--skip-loop', action='store_true')
    a = ap.parse_args()
    assert torch.cuda.is_available(), 'needs an H100'
    dev = torch.device('cuda', 0)
    torch.cuda.set_device(dev)
    sampler = bench.ClockSampler(0)
    sampler.start()
    line = {'workload': f'Qwen2-7B shape (28 layers, 28/4 heads, V=152064) bf16, greedy, {bench.DL}-token/{bench.BL}-'
                        f'branch drafts, {bench.PROMPT_LEN}-token prompts -> {bench.NEW_TOKENS} new tokens, '
                        f'{a.steps} timed requests, {a.warmup} warm-up requests'}
    if not a.skip_loop:
        line['loop'] = loop_numbers(dev, a.steps, a.warmup)
    line['attention'] = attention_numbers(dev, a.layers)
    sampler.stop_flag = True
    sampler.join(timeout=2)
    line['clocks'] = sampler.summary()
    line['gpu'] = torch.cuda.get_device_name(0)
    print(json.dumps(line))


if __name__ == '__main__':
    main()
