# -*- coding: utf-8 -*-
"""Int4 (GPTQ / compressed-tensors W4A16, group 128) Mixtral experts against fp8 on one GPU; prints one JSON line.

  projections: at the Mixtral-8x7B shape (8 experts, H 4096, I 14336), for 64 and 128 rows: the grouped int4 down launch
               (k_gemm_w4, one expert per group) against the grouped fp8 launch (k_gemm_fp8), and the stacked int4
               gate_up launch with the SiLU*up epilogue against the fp8 one; us per launch (CUDA events over many
               launches) and GB/s of algorithmic weight bytes (int4: codes + scales + zero points; fp8: codes + scales).
               Each weight is larger than the 50 MB L2, so every launch streams it from HBM
  8x7b:        the 32-layer Mixtral-8x7B verify forward (64 draft rows, 256 cached tokens) as one CUDA graph, median of 5,
               and bench.py's loop workload (256-token phrase-bank prompts, 256 new tokens, 64/8 drafts), in fp8 and then
               in int4 (one model at a time: both together do not fit beside other work on a shared card); weight GB,
               resident GB after the build, peak GB of build and loop
  8x22b:       (--mixtral-8x22b) the Mixtral-8x22B shape (56 layers, H 6144, I 16384) in int4, built only if
               torch.cuda.mem_get_info() shows the memory it needs free; otherwise "not run: X GB free, Y GB needed"

Weights: bench.synth_fill for the bf16 parameters; int4 = seeded uniform codes with group-128 bf16 scales and zero point
8 (MixtralForCausalLM.build_w4, the bf16 experts never exist); fp8 = build_fp8 of synth_fill's weights.  The card name
and power limit are read in the same run.
Usage: python scripts/bench_w4_moe.py [--iters N] [--steps K] [--warmup W] [--sections projections,8x7b] [--mixtral-8x22b]"""
import argparse
import json
import os
import sys
import zlib

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'scripts'))

HBM = 3.35e12
GS = 128


def synth_w4_mixtral(cfg, dev, seed=0):
    """seeded random int4 codes for every projection and expert, built layer by layer"""
    import bench
    from painlessinferenceacceleration_b200.models.mixtral.modeling_mixtral import MixtralForCausalLM

    def fill(name, shape):
        g = torch.Generator(device=dev).manual_seed(zlib.crc32(name.encode()) ^ (seed * 7919))
        N, K = shape
        u = torch.randint(0, 16, (N, K), generator=g, device=dev, dtype=torch.uint8)
        s = ((0.5 + torch.rand((N, K // GS), generator=g, device=dev)) * 0.02 / 8).to(torch.bfloat16)
        return u, s, torch.full((N, K // GS), 8, dtype=torch.uint8, device=dev), GS
    return MixtralForCausalLM.build_w4(cfg, lambda m: bench.synth_fill(m, cfg, seed), fill, device=dev)


def mixtral_8x22b_config():
    from transformers import MixtralConfig
    return MixtralConfig(vocab_size=32768, hidden_size=6144, intermediate_size=16384, num_hidden_layers=56,
                         num_attention_heads=48, num_key_value_heads=8, max_position_embeddings=65536,
                         num_local_experts=8, num_experts_per_tok=2, rms_norm_eps=1e-5, rope_theta=1e6,
                         sliding_window=None, bos_token_id=1, eos_token_id=2, pad_token_id=0)


def w4_model_bytes(cfg, gs=GS):
    """(resident weight bytes of an int4 Mixtral, the most one layer's build adds on top) computed from the shapes:
    codes N K / 2, bf16 scales and uint8 zero points per group of gs, bf16 embedding, lm_head and router.  The build
    holds a layer's unpacked experts (one byte per code), their stacked copy and the tiling's intermediates."""
    H, I, E, L, V = cfg.hidden_size, cfg.intermediate_size, cfg.num_local_experts, cfg.num_hidden_layers, cfg.vocab_size
    kv = cfg.num_key_value_heads * (H // cfg.num_attention_heads)
    q4 = lambda N, K: N * K // 2 + 3 * N * (K // gs)
    layer = q4(H + 2 * kv, H) + q4(H, H) + E * (q4(2 * I, H) + q4(H, I)) + 2 * E * H + 4 * H
    return L * layer + 2 * V * H * 2 + 2 * H, 4 * E * 3 * I * H


def model_numbers(label, build, cfg, dev, args, B, bench):
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    m = build()
    out = dict(resident_gb=round((torch.cuda.memory_allocated() - base) / 1e9, 2),
               build_peak_gb=round((torch.cuda.max_memory_allocated() - base) / 1e9, 2),
               weight_gb=round(bench.weight_bytes_per_step(m) / 1e9, 3))
    g = B.forward_graph(m)
    t = sorted(B.time_us(g.replay, args.iters) for _ in range(5))
    us = t[len(t) // 2]
    out['forward_64rows'] = dict(us=round(us, 1), us_min=round(t[0], 1), us_max=round(t[-1], 1),
                                 hbm_share=round(bench.weight_bytes_per_step(m) / (us * 1e-6) / HBM, 3))
    del g
    m._rt = None
    torch.cuda.empty_cache()
    out['loop'] = B.loop_numbers(m, cfg, dev, args.steps, args.warmup)
    out['peak_gb'] = round((torch.cuda.max_memory_allocated() - base) / 1e9, 2)
    print(label, json.dumps(out), file=sys.stderr)
    del m
    torch.cuda.empty_cache()
    return out


def main():
    import bench
    import bench_fp8 as B
    from painlessinferenceacceleration_b200.common import ops
    from painlessinferenceacceleration_b200.models.llama.modeling_llama import _gate_up_order
    from painlessinferenceacceleration_b200.models.mixtral.modeling_mixtral import Int4Stack, MixtralForCausalLM
    ap = argparse.ArgumentParser()
    ap.add_argument('--iters', type=int, default=20)
    ap.add_argument('--steps', type=int, default=8)
    ap.add_argument('--warmup', type=int, default=2)
    ap.add_argument('--sections', default='projections,8x7b')
    ap.add_argument('--mixtral-8x22b', action='store_true')
    args = ap.parse_args()
    sections = args.sections.split(',')
    dev = torch.device('cuda:0')
    torch.cuda.set_device(dev)
    name, limit = B.card()
    res = dict(gpu=name, power_limit=limit)

    # ---------------------------------------------------------------- projections (Mixtral-8x7B shape)
    if 'projections' in sections:
        E, H, I = 8, 4096, 14336
        gen = torch.Generator(device=dev).manual_seed(0)
        proj = {}
        for pname, N, K in (('down', H, I), ('gate_up_silu', 2 * I, H)):
            u = torch.randint(0, 16, (E, N, K), generator=gen, device=dev, dtype=torch.uint8)
            s = (0.002 + 0.001 * torch.rand((E, N, K // GS), generator=gen, device=dev)).to(torch.bfloat16)
            z = torch.full((E, N, K // GS), 8, dtype=torch.uint8, device=dev)
            st = Int4Stack(u, s, z, GS, interleaved=pname != 'down')
            del u, s, z
            w4_bytes = st.qweight.numel() + st.scale.numel() * 2 + st.zero.numel()
            w = torch.empty((E, N, K), dtype=torch.bfloat16, device=dev)
            for e in range(E):
                w[e].normal_(0.0, 0.02, generator=gen)
            if pname != 'down':
                w = _gate_up_order(w)
            q, s8 = ops.quantize_fp8(w)
            del w
            qw = ops.tile_weight_fp8(q)
            del q
            f8_bytes = qw.numel() + s8.numel() * 4
            x = torch.randn((256, E * K if pname == 'down' else K), device=dev).to(torch.bfloat16)
            act = torch.empty((256, E * I), dtype=torch.bfloat16, device=dev)
            if pname == 'down':
                g4 = ops.Gemm.grouped_w4(st.qweight, st.scale, st.zero, GS, E, x)
                g8 = ops.Gemm.grouped_fp8(qw, s8, x)
                run4, run8 = (lambda r: g4.run(r)), (lambda r: g8.run(r))
            else:
                g4 = st.gemm(x, out=act).set_silu()
                g8 = ops.Gemm.fp8(qw.view(-1, *qw.shape[2:]), s8.view(-1), x, out=act).set_silu()
                run4, run8 = (lambda r: g4.run(r, out=act)), (lambda r: g8.run(r, out=act))
            r = dict(int4_weight_mb=round(w4_bytes / 1e6, 1), fp8_weight_mb=round(f8_bytes / 1e6, 1))
            for rows in (64, 128):
                for k, fn, nb in (('int4', run4, w4_bytes), ('fp8', run8, f8_bytes)):
                    us = B.time_us(lambda: fn(rows), args.iters * 5)
                    r[f'{k}_{rows}rows'] = dict(us=round(us, 1), gbps=round(nb / (us * 1e-6) / 1e9, 1))
            proj[pname] = r
            del g4, g8, st, qw, s8, x, act
            torch.cuda.empty_cache()
        res['projections_mixtral_8x7b'] = proj

    # ---------------------------------------------------------------- the whole 8x7B model, fp8 then int4
    if '8x7b' in sections:
        cfg, _ = bench.make_config('mixtral-8x7b-16l')
        cfg.num_hidden_layers = 32
        res['mixtral_8x7b_32l'] = {
            'fp8': model_numbers('fp8', lambda: B.synth_fp8(MixtralForCausalLM, cfg, dev), cfg, dev, args, B, bench),
            'int4': model_numbers('int4', lambda: synth_w4_mixtral(cfg, dev), cfg, dev, args, B, bench)}

    # ---------------------------------------------------------------- 8x22B in int4, only if it fits in free memory
    if args.mixtral_8x22b:
        cfg = mixtral_8x22b_config()
        weights, build_extra = w4_model_bytes(cfg)
        need = weights + build_extra + (4 << 30)   # + the runtime's buffers, KV cache and plans
        torch.cuda.empty_cache()
        free, total = torch.cuda.mem_get_info()
        if free < need:
            res['mixtral_8x22b_int4'] = (f'not run: {free / 1e9:.1f} GB free, {need / 1e9:.1f} GB needed '
                                         f'({weights / 1e9:.1f} GB of weights, computed from the shapes)')
        else:
            torch.cuda.reset_peak_memory_stats()
            m = synth_w4_mixtral(cfg, dev)
            built = torch.cuda.max_memory_allocated()
            loop = B.loop_numbers(m, cfg, dev, max(2, args.steps // 2), 1)
            res['mixtral_8x22b_int4'] = dict(loop, weight_gb=round(bench.weight_bytes_per_step(m) / 1e9, 2),
                                             max_memory_allocated_gb_build=round(built / 1e9, 2),
                                             max_memory_allocated_gb=round(torch.cuda.max_memory_allocated() / 1e9, 2))
            del m
    print(json.dumps(res))


if __name__ == '__main__':
    with torch.no_grad():
        main()
