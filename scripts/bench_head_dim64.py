# -*- coding: utf-8 -*-
"""Head dim 64 on one H100: k_tree_attn<64> against k_tree_attn<128>, and bench.py's workload on the Llama-3.2-1B and
Qwen2.5-0.5B shapes in bf16 and fp8.

    python scripts/bench_head_dim64.py [--steps K] [--warmup W] [--skip-loop]

Attention: k_tree_attn alone, 32 query heads over 8 KV heads, 64 draft rows, P in {384, 3968}; one launch per layer
over enough layers that the K/V planes of the sweep exceed the 50 MB L2 (CUDA-graph replay, CUDA events), head dim 64
and 128 alternating in one process, median of 5.  Bytes = the algorithmic K/V + Q/O traffic,
2 L Hkv HD 2 + 2 n Hq HD 2.
Loop: bench.py's workload (256-token phrase-bank prompts -> 256 new tokens, 64-token / 8-branch drafts, bench.synth_fill
weights, untied lm_head), a trie warmed on other prompts, then a first and a second pass over the timed prompts.  The
fp8 run quantises the same bf16 weights in place (quantize_fp8()).
The card's name and power limit are read in the same run.  One JSON line on stdout."""
import argparse
import json
import math
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bench  # noqa: E402

HBM_PEAK_GBS = 3350.0   # H100 SXM data sheet (700 W); a reference point, not a reached rate
L2_BYTES = 50 * 2 ** 20


def llama32_1b_shape():
    from transformers import LlamaConfig
    return LlamaConfig(vocab_size=128256, hidden_size=2048, intermediate_size=8192, num_hidden_layers=16,
                       num_attention_heads=32, num_key_value_heads=8, max_position_embeddings=4096, rms_norm_eps=1e-5,
                       rope_theta=500000.0, tie_word_embeddings=False, bos_token_id=1, eos_token_id=2, pad_token_id=0,
                       rope_scaling={'rope_type': 'llama3', 'factor': 32.0, 'low_freq_factor': 1.0,
                                     'high_freq_factor': 4.0, 'original_max_position_embeddings': 8192})


def qwen25_05b_shape():
    from transformers import Qwen2Config
    return Qwen2Config(vocab_size=151936, hidden_size=896, intermediate_size=4864, num_hidden_layers=24,
                       num_attention_heads=14, num_key_value_heads=2, max_position_embeddings=4096, rms_norm_eps=1e-6,
                       rope_theta=1000000.0, use_sliding_window=False, tie_word_embeddings=False,
                       bos_token_id=1, eos_token_id=2, pad_token_id=0)


def loop_numbers(model, cfg, dev, K, W):
    from painlessinferenceacceleration_b200.common.lookahead_cache import LookaheadCache
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
    return {'first_pass': first, 'second_pass': second, 'weight_bytes_per_step': wbytes}


def shape_numbers(name, dev, K, W):
    from painlessinferenceacceleration_b200.models.llama.modeling_llama import LlamaForCausalLM
    from painlessinferenceacceleration_b200.models.qwen2.modeling_qwen2 import Qwen2ForCausalLM
    cfg, cls = (llama32_1b_shape(), LlamaForCausalLM) if name == 'llama3.2-1b' else (qwen25_05b_shape(), Qwen2ForCausalLM)
    model = bench.synth_fill(cls(cfg, device=dev), cfg)
    out = {'bf16': loop_numbers(model, cfg, dev, K, W)}
    model.quantize_fp8()
    out['fp8'] = loop_numbers(model, cfg, dev, K, W)
    del model
    torch.cuda.empty_cache()
    return out


def attention_numbers(dev, reps=5):
    """k_tree_attn per launch at head dim 64 and 128 (Hq 32, Hkv 8, 64 draft rows), P = 384 and 3968, alternating"""
    from painlessinferenceacceleration_b200.common import ops
    R, n, hq, hkv = 64, 64, 32, 8
    rows = np.array([(1 << (i + 1)) - 1 if i < 63 else 0xFFFFFFFFFFFFFFFF for i in range(R)], dtype=np.uint64)
    mask = torch.from_numpy(rows.view(np.int64)).to(dev).view(R, 1)
    out = {}
    for P in (384, 3968):
        L = P + n
        max_seq = L + 64
        layers = max(16, math.ceil(2 * L2_BYTES / (2 * L * hkv * 64 * 2)))   # the head-dim-64 set is 2x the L2
        slots = ops.Slots(torch.tensor([n], dtype=torch.int32, device=dev),
                          torch.tensor([P], dtype=torch.int32, device=dev), None, R)
        runs = {}
        for hd in (64, 128):
            kc = (torch.randn((layers, hkv, max_seq, hd), device=dev) * 0.5).to(torch.bfloat16)
            vc = (torch.randn((layers, hkv, max_seq, hd), device=dev) * 0.5).to(torch.bfloat16)
            q = (torch.randn((R, hq, hd), device=dev) * 0.5).to(torch.bfloat16)
            o = torch.zeros_like(q)
            plan = ops.AttnPlan(kc, vc, hq, hkv, hd, R)

            def sweep(plan=plan, q=q, o=o):
                for li in range(layers):
                    plan.forward(li, q, mask, slots, o)
            runs[hd] = (sweep, [], (kc, vc, q, o, plan))
        for _ in range(reps):
            for hd in (64, 128):
                sweep, us, _ = runs[hd]
                us.append(bench._graph_time(sweep) / layers)
        for hd in (64, 128):
            us = float(np.median(runs[hd][1]))
            nbytes = 2 * L * hkv * hd * 2 + 2 * n * hq * hd * 2
            out[f'HD{hd}_P{P}'] = {'us_per_launch': us, 'us_all': runs[hd][1], 'bytes': nbytes,
                                   'gbs': nbytes / (us * 1e-6) / 1e9, 'layers': layers,
                                   'kv_set_mb': layers * 2 * L * hkv * hd * 2 / 2 ** 20}
        del runs
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
    line = {'workload': f'{bench.DL}-token/{bench.BL}-branch drafts, {bench.PROMPT_LEN}-token prompts -> '
                        f'{bench.NEW_TOKENS} new tokens, {a.steps} timed requests, {a.warmup} warm-up requests'}
    line['attention'] = attention_numbers(dev)
    if not a.skip_loop:
        for name in ('llama3.2-1b', 'qwen2.5-0.5b'):
            line[name] = shape_numbers(name, dev, a.steps, a.warmup)
    sampler.stop_flag = True
    sampler.join(timeout=2)
    line['clocks'] = sampler.summary()
    line['gpu'] = torch.cuda.get_device_name(0)
    print(json.dumps(line))


if __name__ == '__main__':
    main()
