# -*- coding: utf-8 -*-
"""Seeded tiny int4 checkpoints (no checkpoints exist offline), written with torch alone so that the GPU machine can
rebuild them bit for bit: random 4-bit codes, scales and zero points for every decoder projection of the tiny Llama /
Mistral / Qwen2 models of tests/tiny_models.py and tests/tiny_qwen2.py, packed as compressed-tensors `pack-quantized`
or as GPTQ v1.  tests/golden/gen_w4_golden.py checks the packing against compressed_tensors' own packer and records the
eager transformers model of each checkpoint; tests/test_w4_host.py checks the unpackers against the library."""
import json
import os

import torch

PROJ = ('self_attn.q_proj', 'self_attn.k_proj', 'self_attn.v_proj', 'self_attn.o_proj', 'mlp.gate_proj',
        'mlp.up_proj', 'mlp.down_proj')
VOCAB = 200
PROMPT_LEN = 32

# name -> (family, format, symmetric, group size (None: channel-wise), scale dtype, seed)
FIXTURES = {
    'llama_ct_sym_g128_bf16': ('llama', 'compressed-tensors', True, 128, torch.bfloat16, 1),
    'llama_ct_asym_channel_bf16': ('llama', 'compressed-tensors', False, None, torch.bfloat16, 2),
    'llama_ct_asym_g128_fp16': ('llama', 'compressed-tensors', False, 128, torch.float16, 3),
    'llama_gptq_asym_g128_fp16': ('llama', 'gptq', False, 128, torch.float16, 3),   # the codes of the one above
    'mistral_ct_sym_g256_bf16': ('mistral', 'compressed-tensors', True, 256, torch.bfloat16, 4),
    'mistral_ct_asym_g128_bf16': ('mistral', 'compressed-tensors', False, 128, torch.bfloat16, 5),
    'qwen2_ct_sym_g128_bf16': ('qwen2', 'compressed-tensors', True, 128, torch.bfloat16, 6),
    'qwen2_ct_asym_g128_fp16': ('qwen2', 'compressed-tensors', False, 128, torch.float16, 7),
}


def hf_config(family):
    from tests.tiny_models import tiny_config
    from tests.tiny_qwen2 import qwen2_config
    return qwen2_config(vocab=VOCAB) if family == 'qwen2' else tiny_config(family, vocab=VOCAB)


def random_codes(N, K, group_size, sym, scale_dtype, gen):
    """(u uint8 [N, K], s [N, G] scale_dtype, z uint8 [N, G]): uniform codes, scales around 0.02 (the dequantised
    weights then have a std near tests/tiny_models.py's 0.08), zero points 8 (symmetric) or uniform in 6..10, as a
    min-max quantiser gives for roughly zero-mean weights (zero points far from the middle give every row a large mean
    and a model whose bf16 logits are dominated by cancellation)"""
    G = K // (group_size or K)
    u = torch.randint(0, 16, (N, K), generator=gen).to(torch.uint8)
    s = (0.01 + 0.02 * torch.rand((N, G), generator=gen)).to(scale_dtype)
    z = torch.full((N, G), 8, dtype=torch.uint8) if sym else torch.randint(6, 11, (N, G), generator=gen).to(torch.uint8)
    return u, s, z


def pack_nibbles(codes, dim):
    """uint8 codes 0..15 -> int32, 8 consecutive codes along `dim` per element, code i at bits 4i"""
    c = codes.to(torch.int32)
    if dim == 0:
        c = c.t()
    R, C = c.shape
    c = c.reshape(R, C // 8, 8)
    packed = torch.zeros((R, C // 8), dtype=torch.int64)
    for i in range(8):
        packed |= c[..., i].to(torch.int64) << (4 * i)
    packed = torch.where(packed >= 1 << 31, packed - (1 << 32), packed).to(torch.int32)
    return packed.t().contiguous() if dim == 0 else packed.contiguous()


def pack_compressed_tensors(u, s, z, sym):
    """compressed-tensors pack-quantized tensors of one projection (compressors/pack_quantized): weight_packed int32
    [N, K/8] along K, weight_scale [N, G], weight_shape, and (asymmetric) weight_zero_point int32 [ceil(N/8), G] packed
    along N.  Both store the signed value + 8, i.e. u and z themselves."""
    out = {'weight_packed': pack_nibbles(u, 1), 'weight_scale': s.clone(),
           'weight_shape': torch.tensor(list(u.shape), dtype=torch.int64)}
    if not sym:
        out['weight_zero_point'] = pack_nibbles(z, 0)
    return out


def pack_gptq(u, s, z, group_size):
    """GPTQ v1 tensors of one projection: qweight int32 [K/8, N] packed along K, qzeros int32 [G, N/8] packed along N
    holding z - 1, scales [G, N], g_idx = k // group_size"""
    N, K = u.shape
    return {'qweight': pack_nibbles(u.t().contiguous(), 0), 'qzeros': pack_nibbles((z - 1).t().contiguous(), 1),
            'scales': s.t().contiguous(), 'g_idx': (torch.arange(K) // (group_size or K)).to(torch.int32)}


def quantization_config(fmt, sym, group_size):
    if fmt == 'gptq':
        return {'quant_method': 'gptq', 'bits': 4, 'group_size': group_size or -1, 'desc_act': False, 'sym': sym,
                'checkpoint_format': 'gptq', 'true_sequential': True, 'damp_percent': 0.01}
    weights = {'num_bits': 4, 'type': 'int', 'symmetric': sym, 'strategy': 'group' if group_size else 'channel',
               'group_size': group_size, 'actorder': None, 'dynamic': False, 'observer': 'minmax',
               'block_structure': None, 'observer_kwargs': {}}
    return {'quant_method': 'compressed-tensors', 'format': 'pack-quantized', 'quantization_status': 'compressed',
            'config_groups': {'group_0': {'targets': ['Linear'], 'weights': weights, 'input_activations': None,
                                          'output_activations': None, 'format': 'pack-quantized'}},
            'ignore': ['lm_head'], 'kv_cache_scheme': None, 'global_compression_ratio': None}


def build(name):
    """-> (config, {tensor name: tensor} of the checkpoint, {projection name: (u, s, z)})"""
    family, fmt, sym, gs, sdt, seed = FIXTURES[name]
    cfg = hf_config(family)
    gen = torch.Generator().manual_seed(1000 + seed)
    H, I, V = cfg.hidden_size, cfg.intermediate_size, cfg.vocab_size
    hd = H // cfg.num_attention_heads
    kv = cfg.num_key_value_heads * hd
    shapes = {'self_attn.q_proj': (H, H), 'self_attn.k_proj': (kv, H), 'self_attn.v_proj': (kv, H),
              'self_attn.o_proj': (H, H), 'mlp.gate_proj': (I, H), 'mlp.up_proj': (I, H), 'mlp.down_proj': (H, I)}
    sd, codes = {}, {}
    bf = lambda *shape: (0.08 * torch.randn(shape, generator=gen)).to(torch.bfloat16)
    sd['model.embed_tokens.weight'] = bf(V, H)
    sd['lm_head.weight'] = bf(V, H)
    sd['model.norm.weight'] = (1 + 0.1 * torch.randn(H, generator=gen)).to(torch.bfloat16)
    for li in range(cfg.num_hidden_layers):
        pre = f'model.layers.{li}.'
        for n in ('input_layernorm', 'post_attention_layernorm'):
            sd[pre + n + '.weight'] = (1 + 0.1 * torch.randn(H, generator=gen)).to(torch.bfloat16)
        if family == 'qwen2':
            for n, std in (('q_proj', 1.0), ('k_proj', 3.0), ('v_proj', 1.0)):
                sd[pre + f'self_attn.{n}.bias'] = (std * torch.randn(shapes[f'self_attn.{n}'][0], generator=gen)).to(torch.bfloat16)
        for p in PROJ:
            u, s, z = random_codes(*shapes[p], gs, sym, sdt, gen)
            codes[pre + p] = (u, s, z)
            packed = pack_gptq(u, s, z, gs) if fmt == 'gptq' else pack_compressed_tensors(u, s, z, sym)
            for k, v in packed.items():
                sd[f'{pre}{p}.{k}'] = v
    cfg.quantization_config = quantization_config(fmt, sym, gs)
    return cfg, sd, codes


def write(name, path):
    """the checkpoint directory (config.json + model.safetensors); returns the projections' (u, s, z)"""
    from safetensors.torch import save_file
    cfg, sd, codes = build(name)
    os.makedirs(path, exist_ok=True)
    cfg.torch_dtype = 'bfloat16'
    d = cfg.to_dict()
    d['quantization_config'] = cfg.quantization_config
    d.pop('_attn_implementation', None)
    with open(os.path.join(path, 'config.json'), 'w') as f:
        json.dump(d, f, indent=1)
    save_file(sd, os.path.join(path, 'model.safetensors'), metadata={'format': 'pt'})
    return codes


def prompt(name):
    seed = FIXTURES[name][5]
    return torch.randint(3, VOCAB, (1, PROMPT_LEN), generator=torch.Generator().manual_seed(77 + seed))
