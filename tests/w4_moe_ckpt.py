# -*- coding: utf-8 -*-
"""Seeded tiny int4 Mixtral checkpoints, written with torch alone (tests/w4_ckpt.py's codes and packers) in the
published per-expert layout: `block_sparse_moe.experts.{e}.{w1,w3,w2}` and the attention projections packed as
compressed-tensors `pack-quantized` or GPTQ v1, the router `block_sparse_moe.gate.weight`, embeddings, lm_head and norms
unquantised.  tests/golden/gen_w4_mixtral_golden.py records the eager transformers model of each checkpoint;
tests/test_w4_mixtral_host.py and tests/test_gpu_w4_mixtral.py load them."""
import json
import os
import zlib

import torch

from tests import w4_ckpt

VOCAB = w4_ckpt.VOCAB
PROMPT_LEN = w4_ckpt.PROMPT_LEN
ATTN = ('self_attn.q_proj', 'self_attn.k_proj', 'self_attn.v_proj', 'self_attn.o_proj')

# name -> (format, symmetric, group size (None: channel-wise), scale dtype, seed, config overrides)
FIXTURES = {
    'mixtral_ct_sym_g128_bf16': ('compressed-tensors', True, 128, torch.bfloat16, 1, {}),
    'mixtral_ct_asym_g128_fp16': ('compressed-tensors', False, 128, torch.float16, 2, {}),
    'mixtral_gptq_asym_g128_fp16': ('gptq', False, 128, torch.float16, 2, {}),   # the codes of the one above
    'mixtral_ct_asym_channel_bf16': ('compressed-tensors', False, None, torch.bfloat16, 3, {}),
    # the down projection's K = 384 is an odd multiple of 128: its last k chunk is a half chunk
    'mixtral_ct_sym_g128_i384': ('compressed-tensors', True, 128, torch.bfloat16, 4, {'intermediate_size': 384}),
    'mixtral_ct_asym_g128_e8': ('compressed-tensors', False, 128, torch.bfloat16, 5, {'num_local_experts': 8}),
}


def hf_config(name):
    from tests.tiny_models import tiny_config
    return tiny_config('mixtral', vocab=VOCAB, **FIXTURES[name][5])


def experts(cfg):
    """the per-expert projection names of a layer, relative to it"""
    return [f'block_sparse_moe.experts.{e}.{x}' for e in range(cfg.num_local_experts) for x in ('w1', 'w3', 'w2')]


def quantization_config(fmt, sym, group_size):
    q = w4_ckpt.quantization_config(fmt, sym, group_size)
    if fmt != 'gptq':   # the router stays unquantised, as in published compressed-tensors Mixtral checkpoints
        q['ignore'] = ['lm_head', 're:.*block_sparse_moe.gate']
    return q


def build(name):
    """-> (config, {tensor name: tensor} of the checkpoint, {projection name: (u, s, z)})"""
    fmt, sym, gs, sdt, seed, _ = FIXTURES[name]
    cfg = hf_config(name)
    gen = torch.Generator().manual_seed(2000 + seed)
    H, I, V, E = cfg.hidden_size, cfg.intermediate_size, cfg.vocab_size, cfg.num_local_experts
    kv = cfg.num_key_value_heads * (H // cfg.num_attention_heads)
    shapes = {'self_attn.q_proj': (H, H), 'self_attn.k_proj': (kv, H), 'self_attn.v_proj': (kv, H),
              'self_attn.o_proj': (H, H)}
    for p in experts(cfg):
        shapes[p] = (H, I) if p.endswith('w2') else (I, H)
    sd, codes = {}, {}
    bf = lambda *shape: (0.08 * torch.randn(shape, generator=gen)).to(torch.bfloat16)
    sd['model.embed_tokens.weight'] = bf(V, H)
    sd['lm_head.weight'] = bf(V, H)
    sd['model.norm.weight'] = (1 + 0.1 * torch.randn(H, generator=gen)).to(torch.bfloat16)
    for li in range(cfg.num_hidden_layers):
        pre = f'model.layers.{li}.'
        for n in ('input_layernorm', 'post_attention_layernorm'):
            sd[pre + n + '.weight'] = (1 + 0.1 * torch.randn(H, generator=gen)).to(torch.bfloat16)
        sd[pre + 'block_sparse_moe.gate.weight'] = (0.3 * torch.randn((E, H), generator=gen)).to(torch.bfloat16)
        for p in ATTN + tuple(experts(cfg)):
            u, s, z = w4_ckpt.random_codes(*shapes[p], gs, sym, sdt, gen)
            codes[pre + p] = (u, s, z)
            packed = w4_ckpt.pack_gptq(u, s, z, gs) if fmt == 'gptq' else w4_ckpt.pack_compressed_tensors(u, s, z, sym)
            for k, v in packed.items():
                sd[f'{pre}{p}.{k}'] = v
    cfg.quantization_config = quantization_config(fmt, sym, gs)
    return cfg, sd, codes


def shard_of(key, shards):
    return zlib.crc32(key.encode()) % shards


def write(name, path, shards=1, edit=None):
    """the checkpoint directory (config.json + model*.safetensors, split over `shards` files by a hash of the tensor
    name, so that a layer's experts and router land in different files); edit(sd) may change the tensors first.
    Returns the projections' (u, s, z)."""
    from safetensors.torch import save_file
    cfg, sd, codes = build(name)
    if edit is not None:
        edit(sd)
    os.makedirs(path, exist_ok=True)
    cfg.torch_dtype = 'bfloat16'
    d = cfg.to_dict()
    d['quantization_config'] = cfg.quantization_config
    d.pop('_attn_implementation', None)
    with open(os.path.join(path, 'config.json'), 'w') as f:
        json.dump(d, f, indent=1)
    for i in range(shards):
        part = {k: v.contiguous() for k, v in sd.items() if shards == 1 or shard_of(k, shards) == i}
        fn = 'model.safetensors' if shards == 1 else f'model-{i + 1:05d}-of-{shards:05d}.safetensors'
        save_file(part, os.path.join(path, fn), metadata={'format': 'pt'})
    return codes


def prompt(name):
    seed = FIXTURES[name][4]
    return torch.randint(3, VOCAB, (1, PROMPT_LEN), generator=torch.Generator().manual_seed(177 + seed))
