# -*- coding: utf-8 -*-
"""GLM-family models on one H100: bench.py's workload on the GLM-4-9B and ChatGLM3-6B shapes in bf16 and fp8, and
k_rope_kv_append's interleaved (GLM) instance against the half-split (Llama) one.

    python scripts/bench_glm.py [--steps K] [--warmup W] [--skip-loop]

Loop: bench.py's workload (256-token phrase-bank prompts -> 256 new tokens, 64-token / 8-branch drafts, bench.synth_fill
weights, untied lm_head), a trie warmed on other prompts, then a first and a second pass over the timed prompts.  The
fp8 run quantises the same bf16 weights in place (quantize_fp8()).  Shapes: GLM-4-9B (40 layers, 4096 / 13696,
32 / 2 heads, V = 151552, GlmForCausalLM) and ChatGLM3-6B (28 layers, V = 65024, ChatGLMForConditionalGeneration).
RoPE / KV append: 64 draft rows, GLM-4-9B heads (32 / 2, head dim 128, rotary_dim 64), one launch per layer over 40
layers (CUDA-graph replay, CUDA events), the two instances alternating in one process, median of 5.
The card's name and power limit are read in the same run.  One JSON line on stdout."""
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


def glm4_9b_shape():
    from transformers import GlmConfig
    from painlessinferenceacceleration_b200.models.glm4.modeling_glm4 import GlmForCausalLM
    return GlmForCausalLM, GlmConfig(vocab_size=151552, hidden_size=4096, intermediate_size=13696, num_hidden_layers=40,
                                     num_attention_heads=32, num_key_value_heads=2, head_dim=128,
                                     max_position_embeddings=8192, rms_norm_eps=1.5625e-07, attention_bias=True,
                                     tie_word_embeddings=False, bos_token_id=1, eos_token_id=2, pad_token_id=0)


def chatglm3_6b_shape():
    from painlessinferenceacceleration_b200.models.chatglm.modeling_chatglm import ChatGLMForConditionalGeneration
    return ChatGLMForConditionalGeneration, ChatGLMForConditionalGeneration.chatglm_config(dict(
        model_type='chatglm', add_bias_linear=False, add_qkv_bias=True, apply_query_key_layer_scaling=True,
        apply_residual_connection_post_layernorm=False, ffn_hidden_size=13696, hidden_size=4096, kv_channels=128,
        layernorm_epsilon=1e-05, multi_query_attention=True, multi_query_group_num=2, num_attention_heads=32,
        num_layers=28, original_rope=True, padded_vocab_size=65024, post_layer_norm=True, rmsnorm=True,
        seq_length=8192, eos_token_id=2, pad_token_id=0))


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
    cls, cfg = glm4_9b_shape() if name == 'glm-4-9b' else chatglm3_6b_shape()
    model = bench.synth_fill(cls(cfg, device=dev), cfg)
    out = {'bf16': loop_numbers(model, cfg, dev, K, W)}
    model.quantize_fp8()
    out['fp8'] = loop_numbers(model, cfg, dev, K, W)
    del model
    torch.cuda.empty_cache()
    return out


def rope_numbers(dev, reps=5, layers=40, P=384):
    """k_rope_kv_append per launch, interleaved (rotary_dim 64) against half-split, GLM-4-9B heads, 64 draft rows"""
    from painlessinferenceacceleration_b200.common import ops
    R, n, hq, hkv, D, rd = 64, 64, 32, 2, 128, 64
    rows = np.array([(1 << (i + 1)) - 1 if i < 63 else 0xFFFFFFFFFFFFFFFF for i in range(R)], dtype=np.uint64)
    mask = torch.from_numpy(rows.view(np.int64)).to(dev).view(R, 1)
    max_seq = P + n + 64
    kc = torch.zeros((layers, hkv, max_seq, D), dtype=torch.bfloat16, device=dev)
    vc = torch.zeros_like(kc)
    qkv = (torch.randn((R, (hq + 2 * hkv) * D), device=dev)).to(torch.bfloat16)
    q = torch.zeros((R, hq, D), dtype=torch.bfloat16, device=dev)
    slots = ops.Slots(torch.tensor([n], dtype=torch.int32, device=dev), torch.tensor([P], dtype=torch.int32, device=dev),
                      None, R)
    runs = {}
    for kind, dim in (('interleaved', rd), ('half_split', D)):
        inv = 1.0 / (10000.0 ** (torch.arange(0, dim, 2, device=dev).float() / dim))
        ang = torch.arange(max_seq + 8, device=dev).float()[:, None] * inv[None]
        cos, sin = ang.cos().to(torch.bfloat16).contiguous(), ang.sin().to(torch.bfloat16).contiguous()
        rdim = rd if kind == 'interleaved' else None

        def sweep(cos=cos, sin=sin, rdim=rdim):
            for li in range(layers):
                ops.rope_kv_append(qkv, mask, slots, hq, hkv, D, cos, sin, q, kc[li], vc[li], max_seq, rotary_dim=rdim)
        runs[kind] = (sweep, [], (cos, sin))
    for _ in range(reps):
        for kind in ('interleaved', 'half_split'):
            sweep, us, _ = runs[kind]
            us.append(bench._graph_time(sweep) / layers)
    nbytes = R * (hq + 2 * hkv) * D * 2 * 2   # qkv read once, q + K + V written once
    return {kind: {'us_per_launch': float(np.median(us)), 'us_all': us, 'bytes': nbytes,
                   'gbs': nbytes / (float(np.median(us)) * 1e-6) / 1e9} for kind, (_, us, _) in runs.items()}


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
    line['rope_kv_append'] = rope_numbers(dev)
    if not a.skip_loop:
        for name in ('glm-4-9b', 'chatglm3-6b'):
            line[name] = shape_numbers(name, dev, a.steps, a.warmup)
    sampler.stop_flag = True
    sampler.join(timeout=2)
    line['clocks'] = sampler.summary()
    line['gpu'] = torch.cuda.get_device_name(0)
    print(json.dumps(line))


if __name__ == '__main__':
    main()
