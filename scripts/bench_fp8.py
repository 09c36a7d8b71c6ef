# -*- coding: utf-8 -*-
"""FP8 (e4m3) weight-only mode against bf16 on one GPU; prints one JSON line.

  forward:     the whole 32-layer Llama-2-7B verify forward (64 draft rows, 256 cached tokens) as one CUDA graph, bf16
               default plans against fp8, alternating in one process; us per forward and the weight bytes' share of
               the card's HBM bandwidth (3.35 TB/s, H100 SXM data sheet)
  projections: the fp8 GEMM against bf16 k_gemm_ws (HBM-tiled) and cuBLAS at 64 rows, GB/s of algorithmic weight
               bytes, at the Llama-2-7B, Qwen2-7B and Mixtral-8x7B shapes; plus the fp8 GEMM at 256 rows (prefill).
               Each timing rotates through enough copies of the weight (>= 4 x the 50 MB L2) that every launch
               streams from HBM
  loop:        bench.py's workload (256-token phrase-bank prompts, 256 new tokens, 64/8 drafts, the trie warmed on
               disjoint prompts): accepted tokens/s, mean accepted length and ms per verify step on the first pass
               and on the second (every answer seen once), Llama-2-7B bf16 against fp8
  mixtral:     the same loop numbers for Mixtral-8x7B with all 32 layers in fp8, built layer by layer (each weight
               filled in a bf16 buffer and quantised, so the bf16 model never exists), and max_memory_allocated

Weights: bench.synth_fill; fp8 = the same weights quantised (quantize_fp8(), or LlamaForCausalLM.build_fp8 with the
same fills).  The card name and power limit are read in the same run.
Usage: python scripts/bench_fp8.py [--iters N] [--steps K] [--warmup W] [--skip-mixtral]"""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

HBM = 3.35e12
L2_ROTATE_BYTES = 200 << 20


def card():
    try:
        out = subprocess.check_output(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'],
                                      text=True).strip().split('\n')[0]
        name, limit = [s.strip() for s in out.split(',')]
        return name, limit
    except Exception:
        return torch.cuda.get_device_name(0), 'unknown'


def time_us(fn, iters, warm=3):
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) * 1000.0 / iters


def synth_fp8(cls, cfg, dev, seed=0):
    """bench.synth_fill's weights, quantised, without the bf16 model: synth_fill runs on the skeleton whose quantised
    projections are still meta tensors (it initialises everything that stays bf16 and leaves those alone), then each
    projection gets synth_fill's own per-name fill in a bf16 buffer and is quantised"""
    import zlib
    import bench
    return cls.build_fp8(cfg, lambda m: bench.synth_fill(m, cfg, seed),
                         lambda name, t: bench.hashed_normal_(t, zlib.crc32(name.encode()) ^ (seed * 7919), 0.02),
                         device=dev)


def loop_numbers(model, cfg, dev, K, Wm, penalty=1.0):
    """bench.py's timed passes (device-resident prompts): first pass over unseen prompts, then the second pass"""
    import bench
    from painlessinferenceacceleration_b200.common.lookahead_cache import LookaheadCache
    model.lookahead_cache = LookaheadCache(eos_ids=[2], device=dev, vocab_capacity=cfg.vocab_size)
    allp = bench.phrase_bank_prompts(64 + 8 * max(Wm, 1), cfg.vocab_size)
    timed = [allp[j] for j in bench.timed_requests(K)]
    warm = [allp[64 + i % (8 * max(Wm, 1))] for i in range(Wm)]
    gen = dict(max_new_tokens=bench.NEW_TOKENS, eos_token_id=2, return_dict_in_generate=True,
               repetition_penalty=penalty,
               decoding_kwargs={'use_lookahead': True, 'decoding_length': bench.DL, 'branch_length': bench.BL})
    for p in warm:
        model.generate(input_ids=torch.tensor([p], device=dev), **gen)

    def one_pass():
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
        return dict(tokens_per_s=round(toks / (ms / 1000.0), 1), mean_accepted_len=round(sum(edls) / max(len(edls), 1), 3),
                    ms_per_verify_step=round(ms / max(len(edls), 1), 3))

    first = one_pass()
    second = one_pass()
    return dict(first_pass=first, second_pass=second)


def forward_graph(model):
    rt = model._runtime(1024, 64)
    rt.n.fill_(64)
    rt.prefix_len.fill_(256)
    rt.ids.copy_(torch.randint(3, 1000, (64,), device=rt.device, dtype=torch.int32))
    rt.mask.copy_(rt.chain)
    model._verify_layers(rt)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        model._verify_layers(rt)
    return g


def main():
    import bench
    from painlessinferenceacceleration_b200.common import ops
    from painlessinferenceacceleration_b200.models.llama.modeling_llama import LlamaForCausalLM
    ap = argparse.ArgumentParser()
    ap.add_argument('--iters', type=int, default=20)
    ap.add_argument('--steps', type=int, default=8, help='timed requests per pass of the loop sections')
    ap.add_argument('--warmup', type=int, default=2)
    ap.add_argument('--skip-mixtral', action='store_true')
    args = ap.parse_args()
    dev = torch.device('cuda:0')
    torch.cuda.set_device(dev)
    name, limit = card()
    res = dict(gpu=name, power_limit=limit)

    cfg, _ = bench.make_config('llama2-7b')
    bf = LlamaForCausalLM(cfg, device=dev)
    bench.synth_fill(bf, cfg)
    f8 = LlamaForCausalLM(cfg, device=dev)
    f8.load_state_dict(bf.state_dict())
    f8.quantize_fp8()
    torch.cuda.empty_cache()
    wb = {'bf16': bench.weight_bytes_per_step(bf), 'fp8': bench.weight_bytes_per_step(f8)}
    graphs = {'bf16': forward_graph(bf), 'fp8': forward_graph(f8)}
    t = {k: [] for k in graphs}
    for _ in range(5):   # alternate the two forwards
        for k, g in graphs.items():
            t[k].append(time_us(g.replay, args.iters))
    fwd = {}
    for k in graphs:
        us = sorted(t[k])[len(t[k]) // 2]
        fwd[k] = dict(us=round(us, 1), weight_gb=round(wb[k] / 1e9, 3), hbm_share=round(wb[k] / (us * 1e-6) / HBM, 3))
    fwd['speedup'] = round(fwd['bf16']['us'] / fwd['fp8']['us'], 3)
    res['forward_llama2_7b_64rows'] = fwd
    del graphs
    bf._rt = f8._rt = None
    torch.cuda.empty_cache()
    res['loop_llama2_7b'] = {'bf16': loop_numbers(bf, cfg, dev, args.steps, args.warmup),
                             'fp8': loop_numbers(f8, cfg, dev, args.steps, args.warmup)}
    del bf, f8
    torch.cuda.empty_cache()

    shapes = [('llama_qkv', 12288, 4096), ('llama_o', 4096, 4096), ('llama_gate_up', 22016, 4096),
              ('llama_down', 4096, 11008), ('qwen2_qkv', 4608, 3584), ('qwen2_down', 3584, 18944),
              ('mixtral_expert_gate_up', 28672, 4096), ('mixtral_expert_down', 4096, 14336)]
    proj = {}
    for pname, N, K in shapes:
        w = (torch.randn((N, K), device=dev) * 0.02).to(torch.bfloat16)
        x = torch.randn((256, K), device=dev).to(torch.bfloat16)
        q, s = ops.quantize_fp8(w)
        qw = ops.tile_weight_fp8(q)
        split = LlamaForCausalLM._fp8_split(w, torch.cuda.get_device_properties(dev).multi_processor_count)
        xs = x[:64].contiguous()
        out = torch.empty((64, N), dtype=torch.bfloat16, device=dev)
        c8 = -(-L2_ROTATE_BYTES // (N * K))        # weight copies per arm: each launch reads a weight not in L2
        c16 = -(-L2_ROTATE_BYTES // (2 * N * K))
        g8 = [ops.Gemm.fp8(qw if i == 0 else qw.clone(), s, x, split_k=split) for i in range(c8)]
        tw = ops.tile_weight(w)
        tws = [tw] + [tw.clone() for _ in range(c16 - 1)]
        for t_ in tws:
            t_.pia_shape = (N, K)
        g16 = [ops.Gemm(t_, xs, tiled=True) for t_ in tws]
        ws = [w if i == 0 else w.clone() for i in range(c16)]
        r = {'weight_copies': {'fp8': c8, 'bf16': c16}}

        def rot(fns):
            it = [0]

            def f():
                fns[it[0] % len(fns)]()
                it[0] += 1
            return f
        for k, fn, nbytes in (('fp8', rot([lambda g=g: g.run(64) for g in g8]), N * K),
                              ('bf16_gemm_ws', rot([lambda g=g: g.run(64) for g in g16]), 2 * N * K),
                              ('cublas', rot([lambda ww=ww: torch.mm(xs, ww.t(), out=out) for ww in ws]), 2 * N * K)):
            us = time_us(fn, args.iters * 5)
            r[k] = dict(us=round(us, 1), gbps=round(nbytes / (us * 1e-6) / 1e9, 1))
        r['fp8_256rows_us'] = round(time_us(rot([lambda g=g: g.run(256) for g in g8]), args.iters * 2), 1)
        r['fp8_split'] = split
        proj[pname] = r
        del g8, g16, ws, tws, tw, qw, q, s, w, x
        torch.cuda.empty_cache()
    res['projections_64rows'] = proj

    if not args.skip_mixtral:
        from painlessinferenceacceleration_b200.models.mixtral.modeling_mixtral import MixtralForCausalLM
        mcfg, _ = bench.make_config('mixtral-8x7b-16l')
        mcfg.num_hidden_layers = 32                  # the whole model: Mixtral-8x7B's 32 layers
        torch.cuda.empty_cache()
        torch.cuda.reset_peak_memory_stats()
        mx = synth_fp8(MixtralForCausalLM, mcfg, dev)
        built = torch.cuda.max_memory_allocated()
        loop = loop_numbers(mx, mcfg, dev, args.steps, args.warmup)
        res['mixtral_8x7b_32l_fp8'] = dict(loop, weight_gb=round(bench.weight_bytes_per_step(mx) / 1e9, 3),
                                           max_memory_allocated_gb_build=round(built / 1e9, 2),
                                           max_memory_allocated_gb=round(torch.cuda.max_memory_allocated() / 1e9, 2))
        del mx
    print(json.dumps(res))


if __name__ == '__main__':
    with torch.no_grad():
        main()
