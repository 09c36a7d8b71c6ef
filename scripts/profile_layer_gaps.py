# -*- coding: utf-8 -*-
"""Where each verify layer's time goes on the GPU (GPU only; without one it fails).

1. The bench-shape verify forward (Llama-2-7B shape, bench.synth_fill weights, 64 draft rows, P = 384 cached tokens) as
   one CUDA graph, replayed under torch.profiler with CUDA activities: every kernel of the main stream is labelled by
   its phase, and the script prints the time each phase adds per layer, the mean gap (negative: overlap under programmatic
   dependent launch) between a phase and the next, and each phase's algorithmic bytes over its time.
2. Without the profiler, each of the five projections alone with its weights cold in L2 (32 distinct weights per
   shape, 8 for the large ones), CUDA events around graph replays as in scripts/gemm_bench.py.

The card's name, power limit and SM clock are printed with the numbers.  The trace is written to --trace-dir (default:
a new temporary directory).
"""
import argparse
import collections
import json
import os
import sys
import tempfile

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import bench  # noqa: E402

PHASES = ('norm1', 'qkv', 'rope', 'attn', 'o', 'norm2', 'gate_up', 'silu', 'down')


def card():
    s = bench.ClockSampler(0)
    s.start()
    return s


def label_kernels(kernels, n_layers):
    """main-stream kernels in time order -> (phase, kernel); the layer's order is fixed by _verify_layers"""
    out, state, norms = [], 'embed', 0
    for k in kernels:
        n = k['name']
        if 'embed' in n:
            ph = 'embed'
        elif 'rmsnorm' in n:
            norms += 1
            ph = 'final_norm' if norms == 2 * n_layers + 1 else ('norm1' if norms % 2 == 1 else 'norm2')
        elif 'rope' in n:
            ph = 'rope'
        elif 'tree_attn' in n or 'attn' in n:
            ph = 'attn'
        elif 'silu' in n:
            ph = 'silu'
        else:   # a GEMM: which one follows from the phase before it
            ph = {'norm1': 'qkv', 'attn': 'o', 'norm2': 'gate_up', 'silu': 'down', 'final_norm': 'lm_head'}.get(state, state)
        out.append((ph, k))
        state = ph
    return out


def phase_bytes(g, P, n=64):
    hid, inter, hq, hkv, hd = g['hidden'], g['inter'], g['n_q_heads'], g['n_kv_heads'], g['head_dim']
    row = n * hid * 2
    qkv_n = (hq + 2 * hkv) * hd
    return {'norm1': 4 * row, 'norm2': 4 * row, 'qkv': qkv_n * hid * 2 + row + n * qkv_n * 2,
            'rope': 2 * n * qkv_n * 2, 'attn': 2 * (P + n) * hkv * hd * 2 + 2 * n * hq * hd * 2,
            'o': hid * hid * 2 + 2 * row, 'gate_up': 2 * inter * hid * 2 + row + n * 2 * inter * 2,
            'silu': n * 3 * inter * 2, 'down': inter * hid * 2 + n * inter * 2 + row,
            'lm_head': g['vocab'] * hid * 2 + row + n * g['vocab'] * 2}


def graph_of(fn):
    fn()
    torch.cuda.synchronize()
    gr = torch.cuda.CUDAGraph()
    with torch.cuda.graph(gr):
        fn()
    gr.replay()
    torch.cuda.synchronize()
    return gr


def event_time(gr, reps=20):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    gr.replay()
    torch.cuda.synchronize()
    e0.record()
    for _ in range(reps):
        gr.replay()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) * 1e3 / reps


def trace_forward(model, rt, out_dir, reps=5):
    from torch.profiler import ProfilerActivity, profile
    gr = graph_of(lambda: model._verify_layers(rt))
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            gr.replay()
        torch.cuda.synchronize()
    path = os.path.join(out_dir, 'profile_layer_gaps.pt.trace.json')
    prof.export_chrome_trace(path)
    ev = [e for e in json.load(open(path))['traceEvents'] if e.get('cat') == 'kernel']
    ev.sort(key=lambda e: e['ts'])
    main = collections.Counter(e['tid'] for e in ev).most_common(1)[0][0]
    side = [e for e in ev if e['tid'] != main]
    ev = [e for e in ev if e['tid'] == main]
    per = len(ev) // reps
    return [ev[i * per:(i + 1) * per] for i in range(reps)], side, event_time(gr)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--P', type=int, default=384)
    ap.add_argument('--trace-dir', default=None, help='where the chrome trace goes (default: a new temporary directory)')
    a = ap.parse_args()
    assert torch.cuda.is_available(), 'profile_layer_gaps.py measures on the GPU; there is no CPU fallback'
    from painlessinferenceacceleration_b200.common import ops
    from painlessinferenceacceleration_b200.models.llama.modeling_llama import LlamaForCausalLM
    out_dir = a.trace_dir or tempfile.mkdtemp()
    os.makedirs(out_dir, exist_ok=True)
    clk = card()
    dev = torch.device('cuda:0')
    cfg, _ = bench.make_config('llama2-7b')
    model = LlamaForCausalLM(cfg, device=dev).requires_grad_(False)
    bench.synth_fill(model, cfg)
    model.fuse()
    rt = model._runtime(a.P + 193, 64)
    rt.mask.copy_(rt.chain)
    rt.n.fill_(64)
    rt.prefix_len.fill_(a.P)
    g, NL = rt.g, rt.g['n_layers']

    passes, side, fwd_us = trace_forward(model, rt, out_dir)
    dur, excl, gap, names = collections.defaultdict(list), collections.defaultdict(list), collections.defaultdict(list), {}
    for kernels in passes:
        lab = label_kernels(kernels, NL)
        prev_end = kernels[0]['ts']
        for i, (ph, k) in enumerate(lab):
            dur[ph].append(k['dur'])
            # the time this kernel adds to the stream: under programmatic dependent launch a kernel starts (and its
            # recorded duration begins) while its predecessor still runs, so its span is not its cost
            end = k['ts'] + k['dur']
            excl[ph].append(max(0.0, end - prev_end))
            prev_end = max(prev_end, end)
            names.setdefault(ph, k['name'][:60])
            if i + 1 < len(lab):
                nxt_ph, nxt = lab[i + 1]
                gap[(ph, nxt_ph)].append(nxt['ts'] - (k['ts'] + k['dur']))
        span = kernels[-1]['ts'] + kernels[-1]['dur'] - kernels[0]['ts']
    by = phase_bytes(g, a.P)
    reps = len(passes)
    print(f'verify forward, 64 rows, P = {a.P}: {fwd_us:.1f} us per graph replay (CUDA events, no profiler); '
          f'{span:.1f} us first-to-last kernel under the profiler')
    print(f'{"phase":10s} {"added us":>9s} {"span us":>8s} {"launches":>8s} {"GB/s":>8s}  kernel   (per layer; added = '
          f'end minus the previous kernel\'s end; GB/s = algorithmic bytes / added time)')
    tot = 0.0
    for ph in PHASES + ('embed', 'final_norm', 'lm_head'):
        if ph not in dur:
            continue
        n_per = len(dur[ph]) / reps
        div = NL if ph in PHASES else 1
        span_l, add_l = sum(dur[ph]) / reps / div, sum(excl[ph]) / reps / div
        tot += sum(excl[ph]) / reps
        gbs = by[ph] / add_l / 1e3 if ph in by and add_l > 0 else float('nan')
        print(f'{ph:10s} {add_l:9.2f} {span_l:8.2f} {n_per:8.0f} {gbs:8.0f}  {names[ph]}')
    gsum = sum(sum(v) for v in gap.values()) / reps
    print(f'added time {tot:.1f} us per forward; summed gaps between kernels {gsum:+.1f} us (main stream)')
    for (p0, p1), v in sorted(gap.items(), key=lambda kv: -sum(kv[1])):
        print(f'gap {p0:>10s} -> {p1:<10s} {sum(v) / len(v):+7.2f} us mean, {sum(v) / reps:+8.1f} us per forward')
    if side:
        print(f'side stream: {len(side) // reps} kernels per forward, {sum(e["dur"] for e in side) / reps:.1f} us')
    del rt
    model._rt = None
    torch.cuda.empty_cache()

    # ---- the five projections alone, weights cold in L2
    print('projection alone, weights cold in L2 (CUDA events, graph replay):')
    hid, inter = g['hidden'], g['inter']
    x = torch.randn((64, 11008), device=dev).to(torch.bfloat16)
    for name, N, K, ours in (('qkv', 3 * hid, hid, False), ('o', hid, hid, False), ('gate_up', 2 * inter, hid, True),
                             ('down', hid, inter, False), ('lm_head', g['vocab'], hid, True)):
        nl = 32 if N * K < 1.5e8 else 8
        ws = [bench.hashed_normal_(torch.empty((N, K), dtype=torch.bfloat16, device=dev), 100 + i, 0.02) for i in range(nl)]
        xk = x[:, :K].contiguous()
        fn = (lambda gs=[ops.Gemm(ops.tile_weight(w), xk, tiled=True) for w in ws]: [gg.run(64) for gg in gs]) if ours \
            else (lambda: [torch.mm(xk, w.t()) for w in ws])
        us = event_time(graph_of(fn)) / nl
        print(f'{name:8s} {"k_gemm" if ours else "cuBLAS":7s} {us:8.2f} us  {N * K * 2 / us / 1e3:7.0f} GB/s')
        if ours:
            us = event_time(graph_of(lambda: [torch.mm(xk, w.t()) for w in ws])) / nl
            print(f'{name:8s} {"cuBLAS":7s} {us:8.2f} us  {N * K * 2 / us / 1e3:7.0f} GB/s')
        del ws, fn
        torch.cuda.empty_cache()
    clk.stop_flag = True
    clk.join(timeout=2)
    print('card:', json.dumps(clk.summary()))


if __name__ == '__main__':
    main()
