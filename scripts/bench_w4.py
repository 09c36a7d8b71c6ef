# -*- coding: utf-8 -*-
"""Int4 (GPTQ / compressed-tensors W4A16, group 128) weights against fp8 and bf16 on one GPU; prints one JSON line.

  projections: k_gemm_w4 against k_gemm_fp8, k_gemm_ws (HBM-tiled bf16) and cuBLAS at 64 rows, us and GB/s of
               algorithmic weight bytes (int4: codes + scales + zero points), at the Llama-2-7B and Qwen2-7B shapes;
               plus k_gemm_w4 at 256 rows.  Each timing rotates through enough weight copies (>= 200 MB, 4x the 50 MB
               L2) that every launch streams from HBM
  forward:     the 32-layer Llama-2-7B verify forward (64 draft rows, 256 cached tokens) as one CUDA graph, bf16 / fp8 /
               int4 alternating in one process, median of 5; the weight bytes' share of 3.35 TB/s (H100 SXM data sheet)
  loop:        bench.py's workload (256-token phrase-bank prompts, 256 new tokens, 64/8 drafts): accepted tokens/s, mean
               accepted length, ms per verify step and the weight bytes' share of 3.35 TB/s at that step time, for the
               Llama-2-7B and Qwen2-7B shapes in the three modes
  70b:         the Llama-2-70B shape in int4 on one card (built layer by layer): the loop numbers and
               max_memory_allocated

Weights: bench.synth_fill; fp8 = quantize_fp8() of them; int4 = the same weights rounded to symmetric group-128 int4
(s = amax / 7 per group, bf16), built with LlamaForCausalLM.build_w4 so that the bf16 decoder never exists.  The card
name, power limit and SM clock are read in the same run.
Usage: python scripts/bench_w4.py [--iters N] [--steps K] [--warmup W] [--sections projections,7b,70b]"""
import argparse
import json
import os
import subprocess
import sys
import zlib

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'scripts'))

HBM = 3.35e12
L2_ROTATE_BYTES = 200 << 20
GS = 128


def card():
    try:
        out = subprocess.check_output(['nvidia-smi', '--query-gpu=name,power.limit,clocks.sm,clocks.max.sm',
                                       '--format=csv,noheader'], text=True).strip().split('\n')[0]
        return dict(zip(('gpu', 'power_limit', 'sm_clock', 'max_sm_clock'), [s.strip() for s in out.split(',')]))
    except Exception:
        return dict(gpu=torch.cuda.get_device_name(0))


def quantize_w4(w, gs=GS):
    """symmetric min-max int4 of a bf16 weight [N, K] per group of gs: s = bf16(amax / 7) (1 for a zero group),
    u = clamp(round(w / s), -8, 7) + 8, z = 8 -> ops' internal (u, s, z, gs)"""
    N, K = w.shape
    wg = w.float().view(N, K // gs, gs)
    s = (wg.abs().amax(-1) / 7).to(torch.bfloat16)
    s = torch.where(s == 0, torch.ones_like(s), s)
    u = (torch.round(wg / s.float()[..., None]).clamp_(-8, 7) + 8).to(torch.uint8).view(N, K)
    return u, s, torch.full_like(s, 8, dtype=torch.uint8), gs


def synth_w4(cls, cfg, dev, seed=0):
    """bench.synth_fill's weights in int4 without the bf16 model: each projection is filled in a bf16 buffer as
    synth_fill fills it, rounded to int4 and freed"""
    import bench

    def fill(name, shape):
        w = torch.empty(shape, dtype=torch.bfloat16, device=dev)
        bench.hashed_normal_(w, zlib.crc32(name.encode()) ^ (seed * 7919), 0.02)
        return quantize_w4(w)
    return cls.build_w4(cfg, lambda m: bench.synth_fill(m, cfg, seed), fill, device=dev)


def qwen2_7b_config():
    from transformers import Qwen2Config
    return Qwen2Config(vocab_size=32000, hidden_size=3584, intermediate_size=18944, num_hidden_layers=28,
                       num_attention_heads=28, num_key_value_heads=4, max_position_embeddings=4096, rms_norm_eps=1e-6,
                       rope_theta=1000000.0, use_sliding_window=False, tie_word_embeddings=False, bos_token_id=1,
                       eos_token_id=2, pad_token_id=0)


def llama2_70b_config():
    from transformers import LlamaConfig
    return LlamaConfig(vocab_size=32000, hidden_size=8192, intermediate_size=28672, num_hidden_layers=80,
                       num_attention_heads=64, num_key_value_heads=8, max_position_embeddings=4096, rms_norm_eps=1e-5,
                       bos_token_id=1, eos_token_id=2, pad_token_id=0)


def with_share(loop, wbytes):
    for p in loop.values():
        p['hbm_share_at_step'] = round(wbytes / (p['ms_per_verify_step'] * 1e-3) / HBM, 3)
    return loop


def main():
    import bench
    import bench_fp8 as B
    from painlessinferenceacceleration_b200.common import ops
    from painlessinferenceacceleration_b200.models.llama.modeling_llama import LlamaForCausalLM
    from painlessinferenceacceleration_b200.models.qwen2.modeling_qwen2 import Qwen2ForCausalLM
    ap = argparse.ArgumentParser()
    ap.add_argument('--iters', type=int, default=20)
    ap.add_argument('--steps', type=int, default=8)
    ap.add_argument('--warmup', type=int, default=2)
    ap.add_argument('--sections', default='projections,7b,70b')
    args = ap.parse_args()
    sections = args.sections.split(',')
    dev = torch.device('cuda:0')
    torch.cuda.set_device(dev)
    res = card()
    n_sm = torch.cuda.get_device_properties(dev).multi_processor_count

    # ---------------------------------------------------------------- projections
    proj = {}
    shapes = [('llama_qkv', 12288, 4096), ('llama_o', 4096, 4096), ('llama_gate_up', 22016, 4096),
              ('llama_down', 4096, 11008), ('qwen2_qkv', 4608, 3584), ('qwen2_down', 3584, 18944)]
    for pname, N, K in shapes if 'projections' in sections else []:
        w = (torch.randn((N, K), device=dev) * 0.02).to(torch.bfloat16)
        x = torch.randn((256, K), device=dev).to(torch.bfloat16)
        xs = x[:64].contiguous()
        u, s, z, gs = quantize_w4(w)
        codes, st, zt = ops.tile_weight_w4(u), s.t().contiguous(), z.t().contiguous()
        w4_bytes = codes.numel() + st.numel() * 2 + zt.numel()
        q, s8 = ops.quantize_fp8(w)
        qw = ops.tile_weight_fp8(q)
        split8 = LlamaForCausalLM._fp8_split(w, n_sm)
        split4 = LlamaForCausalLM._fp8_split(torch.empty((N, -(-K // 256) * 128), device='meta'), n_sm)
        out = torch.empty((64, N), dtype=torch.bfloat16, device=dev)
        c4 = -(-L2_ROTATE_BYTES // w4_bytes)
        c8 = -(-L2_ROTATE_BYTES // (N * K))
        c16 = -(-L2_ROTATE_BYTES // (2 * N * K))
        g4 = [ops.Gemm.w4(codes if i == 0 else codes.clone(), st if i == 0 else st.clone(),
                          zt if i == 0 else zt.clone(), gs, x, split_k=split4) for i in range(c4)]
        g8 = [ops.Gemm.fp8(qw if i == 0 else qw.clone(), s8, x, split_k=split8) for i in range(c8)]
        tw = ops.tile_weight(w)
        tws = [tw] + [tw.clone() for _ in range(c16 - 1)]
        for t_ in tws:
            t_.pia_shape = (N, K)
        g16 = [ops.Gemm(t_, xs, tiled=True) for t_ in tws]
        ws = [w if i == 0 else w.clone() for i in range(c16)]

        def rot(fns):
            it = [0]

            def f():
                fns[it[0] % len(fns)]()
                it[0] += 1
            return f
        r = {'weight_copies': {'int4': c4, 'fp8': c8, 'bf16': c16}, 'int4_split': split4}
        for k, fn, nbytes in (('int4', rot([lambda g=g: g.run(64) for g in g4]), w4_bytes),
                              ('fp8', rot([lambda g=g: g.run(64) for g in g8]), N * K),
                              ('bf16_gemm_ws', rot([lambda g=g: g.run(64) for g in g16]), 2 * N * K),
                              ('cublas', rot([lambda ww=ww: torch.mm(xs, ww.t(), out=out) for ww in ws]), 2 * N * K)):
            us = B.time_us(fn, args.iters * 5)
            r[k] = dict(us=round(us, 1), gbps=round(nbytes / (us * 1e-6) / 1e9, 1))
        us = B.time_us(rot([lambda g=g: g.run(256) for g in g4]), args.iters * 2)
        r['int4_256rows'] = dict(us=round(us, 1), gbps=round(w4_bytes / (us * 1e-6) / 1e9, 1))
        proj[pname] = r
        del g4, g8, g16, ws, tws, tw, qw, q, s8, codes, st, zt, u, s, z, w, x
        torch.cuda.empty_cache()
    if proj:
        res['projections_64rows'] = proj

    # ---------------------------------------------------------------- forward + loops
    for label, cls, cfg in (('llama2_7b', LlamaForCausalLM, bench.make_config('llama2-7b')[0]),
                            ('qwen2_7b_shape', Qwen2ForCausalLM, qwen2_7b_config())) if '7b' in sections else ():
        models = {}
        bf = cls(cfg, device=dev)
        bench.synth_fill(bf, cfg)
        models['bf16'] = bf
        f8 = cls(cfg, device=dev)
        f8.load_state_dict(bf.state_dict())
        models['fp8'] = f8.quantize_fp8()
        models['int4'] = synth_w4(cls, cfg, dev)
        torch.cuda.empty_cache()
        wb = {k: bench.weight_bytes_per_step(m) for k, m in models.items()}
        if label == 'llama2_7b':
            graphs = {k: B.forward_graph(m) for k, m in models.items()}
            t = {k: [] for k in graphs}
            for _ in range(5):
                for k, g in graphs.items():
                    t[k].append(B.time_us(g.replay, args.iters))
            fwd = {}
            for k in graphs:
                us = sorted(t[k])[len(t[k]) // 2]
                fwd[k] = dict(us=round(us, 1), weight_gb=round(wb[k] / 1e9, 3),
                              hbm_share=round(wb[k] / (us * 1e-6) / HBM, 3))
            res['forward_llama2_7b_64rows'] = fwd
            del graphs
            for m in models.values():
                m._rt = None
            torch.cuda.empty_cache()
        res['loop_' + label] = {k: with_share(B.loop_numbers(m, cfg, dev, args.steps, args.warmup), wb[k])
                                for k, m in models.items()}
        del models, bf, f8
        torch.cuda.empty_cache()

    if '70b' in sections:
        cfg = llama2_70b_config()
        torch.cuda.reset_peak_memory_stats()
        m = synth_w4(LlamaForCausalLM, cfg, dev)
        built = torch.cuda.max_memory_allocated()
        wb = bench.weight_bytes_per_step(m)
        loop = with_share(B.loop_numbers(m, cfg, dev, max(2, args.steps // 2), 1), wb)
        res['llama2_70b_int4'] = dict(loop, weight_gb=round(wb / 1e9, 2),
                                      max_memory_allocated_gb_build=round(built / 1e9, 2),
                                      max_memory_allocated_gb=round(torch.cuda.max_memory_allocated() / 1e9, 2))
    print(json.dumps(res))


if __name__ == '__main__':
    with torch.no_grad():
        main()
