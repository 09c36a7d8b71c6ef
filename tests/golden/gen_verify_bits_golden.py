# -*- coding: utf-8 -*-
"""SHA-256 digests of the bf16 verify path's outputs at the benchmark's shapes, recorded on an H100:

  * the gate_up (N = 22016) and lm_head (N = 32000) weight-streaming GEMM plans, K = 4096, tiled weights, seeded
    hashed-normal operands (bench.hashed_normal_), at 64, 1, 17 and 63 rows;
  * b.logits of the full 32-layer Llama-2-7B-shape verify forward (bench.synth_fill weights, a 64-node chain draft of
    seeded tokens, a seeded KV cache) at cached prefix lengths P = 384 and P = 3968.

Digests rather than tensors: the logits alone are 4 MB per case.  Any change of the GEMMs' fp32 summation order
moves some outputs by an ulp and changes the digest.  Run once on the GPU:

    python tests/golden/gen_verify_bits_golden.py      # writes tests/golden/verify_bits.json
"""
import hashlib
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'verify_bits.json')

GEMM_SHAPES = {'gate_up': (22016, 4096), 'lm_head': (32000, 4096)}
GEMM_ROWS = (64, 1, 17, 63)
FORWARD_P = (384, 3968)


def digest(t):
    import torch
    return hashlib.sha256(t.contiguous().view(torch.int16).cpu().numpy().tobytes()).hexdigest()


def gemm_digests(split_k=1):
    """{'gate_up/64': sha, ...}: each plan's bf16 output for `rows` rows (the rows past `rows` are not written)"""
    import torch
    import bench
    from painlessinferenceacceleration_b200.common import ops
    out = {}
    for name, (N, K) in GEMM_SHAPES.items():
        w = bench.hashed_normal_(torch.empty((N, K), dtype=torch.bfloat16, device='cuda'), 11 + N, 0.02)
        x = bench.hashed_normal_(torch.empty((64, K), dtype=torch.bfloat16, device='cuda'), 13 + N, 1.0)
        g = ops.Gemm(ops.tile_weight(w), x, split_k=split_k, tiled=True)
        for rows in GEMM_ROWS:
            y = torch.zeros((64, N), dtype=torch.bfloat16, device='cuda')
            g.run(rows, out=y)
            torch.cuda.synchronize()
            out[f'{name}/{rows}'] = digest(y[:rows])
        del g, w
    return out


def forward_digests():
    """{'logits/P384': sha, ...}: b.logits of one decode-buffer verify forward, eager launches"""
    import torch
    import bench
    from painlessinferenceacceleration_b200.models.llama.modeling_llama import LlamaForCausalLM
    cfg, _ = bench.make_config('llama2-7b')
    model = LlamaForCausalLM(cfg, device=torch.device('cuda')).requires_grad_(False)
    bench.synth_fill(model, cfg)
    model.fuse()
    out = {}
    for P in FORWARD_P:
        rt = model._runtime(P + 96, 64)
        rt.mask.copy_(rt.chain)
        rt.n.fill_(64)
        rt.prefix_len.fill_(P)
        ids = bench.hashed_normal_(torch.empty((64,), dtype=torch.float32, device='cuda'), 17, 1.0)
        rt.ids.copy_((ids.abs() * 1e4).to(torch.int32) % (cfg.vocab_size - 3) + 3)
        bench.hashed_normal_(rt.k_cache, 19, 1.0)
        bench.hashed_normal_(rt.v_cache, 23, 1.0)
        model._verify_layers(rt)
        torch.cuda.synchronize()
        out[f'logits/P{P}'] = digest(rt.decode_bufs.logits)
        del rt
        model._rt = None
        torch.cuda.empty_cache()
    return out


if __name__ == '__main__':
    import torch
    assert torch.cuda.is_available(), 'the digests are recorded on the GPU'
    d = dict(gemm_digests(), **forward_digests())
    d['device'] = torch.cuda.get_device_name(0)
    with open(OUT, 'w') as f:
        json.dump(d, f, indent=1, sort_keys=True)
    print(json.dumps(d, indent=1, sort_keys=True))
