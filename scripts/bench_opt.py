# -*- coding: utf-8 -*-
"""OPT on one H100: the new kernels against today's way of doing the same work, the per-layer LayerNorm / ReLU path,
and bench.py's workload at the OPT-125m, OPT-2.7B (head dim 80, run zero-padded to 128) and OPT-6.7B shapes in bf16
and fp8 and at the OPT-66B shape in fp8.

    python scripts/bench_opt.py [--steps K] [--warmup W] [--skip-loop] [--shapes 125m,2.7b,6.7b,66b]

Kernels (CUDA-graph replays timed with CUDA events, median of 5), 64 draft rows:
  * pia_kv_append_qscale vs the BLOOM-style path it replaces: a torch copy into the zero-padded [rows, 3H, 128]
    layout (head dim 80 only), a torch `q *= scaling`, and k_rope_kv_append with identity tables;
  * pia_learned_pos_embed vs GPT-2's chain of torch ops (models/gpt2 `_positions` + `wte[ids] + wpe[pos]`);
  * the per-layer LayerNorm / ReLU path: two pia_layernorm with the residual add and the ReLU over fc1's output.
Loop: bench.py's workload (256-token phrase-bank prompts -> 256 new tokens, 64-token / 8-branch drafts), a trie
warmed on other prompts, then a first and a second pass over the timed prompts.  Weights: synth_opt (bench.py's hashed
fill under OPT's parameter names, untied lm_head so that the fill's successor structure makes drafts acceptable,
LayerNorm weights 1, biases 0); fp8 = the same weights quantised (quantize_fp8, or build_fp8 for OPT-66B, whose bf16
decoder does not fit on one card).  The weight bytes per step are computed from the shapes.  The card's name and
power limit are read in the same run.  One JSON line on stdout."""
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

SHAPES = {  # name: (layers, hidden, heads, ffn)
    '125m': (12, 768, 12, 3072),
    '2.7b': (32, 2560, 32, 10240),
    '6.7b': (32, 4096, 32, 16384),
    '66b': (64, 9216, 72, 36864),
}


def opt_config(name, tie=False):
    from transformers import OPTConfig
    L, E, H, F = SHAPES[name]
    return OPTConfig(vocab_size=50272, hidden_size=E, num_hidden_layers=L, ffn_dim=F, num_attention_heads=H,
                     max_position_embeddings=2048, do_layer_norm_before=True, word_embed_proj_dim=E,
                     pad_token_id=1, bos_token_id=2, eos_token_id=2, tie_word_embeddings=tie)


def _fill(model, seed=0):
    """bench.synth_fill under OPT's names on every parameter that is not a meta tensor: LayerNorm weights 1, biases
    0, embed_tokens hashed std bench.EMBED_STD, the other weights hashed std 0.02, and the untied lm_head row v =
    bench.LM_SCALE * the sum of the unit embeddings of the tokens t with succ(t) = v"""
    dec = model.model.decoder
    assert model.lm_head.weight is not dec.embed_tokens.weight, 'the fill needs an untied lm_head'
    with torch.no_grad():
        for name, p in model.named_parameters():
            if p.is_meta:
                continue
            pseed = zlib.crc32(name.encode()) ^ (seed * 7919)
            if 'layer_norm' in name:
                p.fill_(1.0 if name.endswith('weight') else 0.0)
            elif name.endswith('bias'):
                p.zero_()
            elif name.endswith('embed_tokens.weight'):
                bench.hashed_normal_(p.data, pseed, bench.EMBED_STD)
            else:
                bench.hashed_normal_(p.data, pseed, 0.02)
        emb, lm = dec.embed_tokens.weight, model.lm_head.weight
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


def synth_opt(cfg, fp8=False, dev=None, seed=0):
    """the benchmark's OPT weights; fp8=True builds the quantised model layer by layer (build_fp8), never holding the
    bf16 decoder"""
    from painlessinferenceacceleration_b200.models.opt.modeling_opt import OPTForCausalLM
    dev = dev if dev is not None else torch.device('cuda', torch.cuda.current_device())
    if not fp8:
        return _fill(OPTForCausalLM(cfg, device=dev), seed)
    return OPTForCausalLM.build_fp8(
        cfg, lambda m: _fill(m, seed),
        lambda name, t: bench.hashed_normal_(t, zlib.crc32(name.encode()) ^ (seed * 7919), 0.02), device=dev)


def weight_bytes(cfg, fp8):
    """bytes streamed per verify step: the decoder projections (bf16, or e4m3 + fp32 row scales and fp32 biases), the
    bf16 biases and LayerNorms, the final LayerNorm and lm_head (token and position embeddings are gathered)"""
    L, E, F, V = cfg.num_hidden_layers, cfg.hidden_size, cfg.ffn_dim, cfg.vocab_size
    w = L * (4 * E * E + 2 * E * F)
    rows = L * (3 * E + E + F + E)          # output rows = bias entries = fp8 scales
    ln = L * 4 * E + 2 * E
    dec = w + 8 * rows if fp8 else 2 * w + 2 * rows
    return dec + 2 * ln + 2 * V * cfg.word_embed_proj_dim


def shape_numbers(name, dev, K, W, modes):
    cfg = opt_config(name)
    out = {}
    model = None
    for mode in modes:
        torch.cuda.reset_peak_memory_stats(dev)
        try:
            if mode == 'bf16':
                model = synth_opt(cfg, False, dev)
            elif model is not None:
                model.quantize_fp8()
            else:
                model = synth_opt(cfg, True, dev)
            r = loop_numbers(model, cfg, dev, K, W)
        except torch.cuda.OutOfMemoryError as e:
            out[mode] = {'fits_on_one_card': False, 'error': str(e).splitlines()[0]}
            model = None
            torch.cuda.empty_cache()
            continue
        wb = weight_bytes(cfg, mode == 'fp8')
        r['weight_bytes_per_step'] = wb
        r['floor_ms_at_3.35TBs'] = wb / (HBM_PEAK_GBS * 1e9) * 1e3
        for p in (r['first_pass'], r['second_pass']):
            p['weight_stream_frac_of_3.35TBs'] = wb / (p['ms_per_verify_step'] * 1e-3) / 1e9 / HBM_PEAK_GBS
        r['fits_on_one_card'] = True
        r['gpu_mem_peak_GB'] = torch.cuda.max_memory_allocated(dev) / 1e9
        r['gpu_mem_total_GB'] = torch.cuda.get_device_properties(dev).total_memory / 1e9
        r['kv_cache_GB'] = (model._rt.k_cache.numel() * 4 / 1e9) if model._rt is not None else None
        out[mode] = r
    del model
    torch.cuda.empty_cache()
    return out


def _median_us(fn, reps=5):
    v = [bench._graph_time(fn) for _ in range(reps)]
    return float(np.median(v)), v


def kernel_numbers(dev):
    from painlessinferenceacceleration_b200.common import ops
    bf = dict(dtype=torch.bfloat16, device=dev)
    rows, P, max_seq = 64, 300, 512
    chain = np.array([(1 << (i + 1)) - 1 if i < 63 else 0xFFFFFFFFFFFFFFFF for i in range(rows)], dtype=np.uint64)
    mask = torch.from_numpy(chain.view(np.int64).reshape(rows, 1)).to(dev)
    i32 = dict(dtype=torch.int32, device=dev)
    sl = ops.Slots(torch.full((1,), rows, **i32), torch.full((1,), P, **i32), torch.zeros((1,), **i32), rows, 0)
    res = {}
    for shape in ('2.7b', '6.7b'):
        _, E, H, _ = SHAPES[shape]
        d, D = E // H, 128
        src = torch.randn((rows, 3 * E), **bf)
        padded = torch.zeros((rows, 3 * H * D), **bf)
        kc, vc = torch.zeros((H, max_seq, D), **bf), torch.zeros((H, max_seq, D), **bf)
        q = torch.zeros((rows, H, D), **bf)
        cos, sin = torch.ones((max_seq, D // 2), **bf), torch.zeros((max_seq, D // 2), **bf)
        scaling = d ** -0.5

        def ours():
            ops.kv_append(src, mask, sl, H, H, d, D, scaling, q, kc, vc, max_seq)

        def today():
            if d != D:   # BLOOM's padding copy; at head dim 128 the QKV GEMM writes the kernel's layout directly
                padded.view(rows, 3 * H, D)[:, :, :d].copy_(src.view(rows, 3 * H, d))
            x = padded if d != D else src
            x.view(rows, 3 * H, D)[:, :H].mul_(scaling)
            ops.rope_kv_append(x, mask, sl, H, H, D, cos, sin, q, kc, vc, max_seq)

        a, av = _median_us(ours)
        b, bv = _median_us(today)
        res[f'kv_append_{shape}'] = {'us': {'kv_append_qscale': a, 'copy_scale_identity_rope': b},
                                     'us_all': {'kv_append_qscale': av, 'copy_scale_identity_rope': bv}}
    for shape in ('125m', '6.7b', '66b'):
        E = SHAPES[shape][1]
        wte, wpe = torch.randn((50272, E), **bf), torch.randn((2050, E), **bf)
        ids = torch.randint(3, 50272, (rows,), **i32)
        out = torch.zeros((rows, E), **bf)
        shifts = torch.arange(64, device=dev)

        def ours():
            ops.learned_pos_embed(wte, ids, wpe, 2, mask, sl, out)

        def torch_ops():   # models/gpt2/modeling_gpt2.py _positions + the embedding sum, with OPT's offset
            depth = ((mask.unsqueeze(-1) >> shifts) & 1).sum(dim=(1, 2)) - 1
            pos = ((sl.prefix_len.long() - sl.pad_len.long()).clamp(min=0) + depth).clamp(min=0, max=2047)
            out.copy_(wte[ids.long()] + wpe[pos + 2])

        a, av = _median_us(ours)
        b, bv = _median_us(torch_ops)
        res[f'pos_embed_{shape}'] = {'us': {'learned_pos_embed': a, 'gpt2_torch_ops': b},
                                     'us_all': {'learned_pos_embed': av, 'gpt2_torch_ops': bv}}
    for shape in ('125m', '6.7b', '66b'):
        _, E, _, F = SHAPES[shape]
        x, resid, y = torch.randn((rows, E), **bf), torch.randn((rows, E), **bf), torch.zeros((rows, E), **bf)
        w, b = torch.ones((E,), **bf), torch.zeros((E,), **bf)
        act = torch.randn((rows, F), **bf)

        def ln_relu():
            ops.layernorm(x, resid, w, b, 1e-5, resid, y)
            ops.layernorm(x, resid, w, b, 1e-5, resid, y)
            torch.relu_(act)

        a, av = _median_us(ln_relu)
        res[f'layernorm_x2_relu_{shape}'] = {'us': a, 'us_all': av}
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=8)
    ap.add_argument('--warmup', type=int, default=3)
    ap.add_argument('--skip-loop', action='store_true')
    ap.add_argument('--shapes', default='125m,2.7b,6.7b,66b')
    a = ap.parse_args()
    assert torch.cuda.is_available(), 'needs an H100'
    dev = torch.device('cuda', 0)
    torch.cuda.set_device(dev)
    sampler = bench.ClockSampler(0)
    sampler.start()
    line = {'workload': f'{bench.DL}-token/{bench.BL}-branch drafts, {bench.PROMPT_LEN}-token prompts -> '
                        f'{bench.NEW_TOKENS} new tokens, {a.steps} timed requests, {a.warmup} warm-up requests',
            'gpu': torch.cuda.get_device_name(0), 'power_limit': power_limit()}
    line['kernels'] = kernel_numbers(dev)
    if not a.skip_loop:
        for name in a.shapes.split(','):
            line[f'opt-{name}'] = shape_numbers(name, dev, a.steps, a.warmup,
                                                ('fp8',) if name == '66b' else ('bf16', 'fp8'))
    sampler.stop_flag = True
    sampler.join(timeout=2)
    line['clocks'] = sampler.summary()
    print(json.dumps(line))


if __name__ == '__main__':
    main()
