# -*- coding: utf-8 -*-
"""Records tests/golden/w4_mixtral_logits.npz: for every compressed-tensors checkpoint of tests/w4_moe_ckpt.py (tiny
Mixtral, symmetric and asymmetric, group 128 and channel-wise, bf16 and fp16 scales, I = 384, 8 experts), the logits of
the eager transformers model of that checkpoint on its prompt, in bf16 and in fp32.  The GPTQ checkpoint's logits are
those of the compressed-tensors checkpoint with the same codes (the GPU test checks the two load to identical weights).

transformers' quantised loader is not used: it does not map a compressed-tensors Mixtral's per-expert tensors onto its
stacked expert parameters (they are reported missing and left randomly initialised).  Instead every tensor is
decompressed here with compressed_tensors' own unpack_from_int32 and dequantize, in the scale's dtype and then rounded
to bf16, checked bit for bit against ops.dequantize_w4, stacked into transformers' [E, 2I, H] / [E, H, I] expert
parameters and loaded with load_state_dict(strict=True).

Needs transformers and compressed_tensors (this is why the GPU tests read the recorded logits):
    python tests/golden/gen_w4_mixtral_golden.py"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)


def decompress(sd, base, sym, group_size, scale_dtype):
    """one projection's weight: compressed_tensors' unpacking and dequantisation in the scale's dtype, then bf16"""
    from compressed_tensors.compressors.pack_quantized.helpers import unpack_from_int32
    from compressed_tensors.quantization import QuantizationArgs
    from compressed_tensors.quantization.lifecycle.forward import dequantize
    shape = torch.Size(sd[base + '.weight_shape'].tolist())
    s = sd[base + '.weight_scale']
    x_q = unpack_from_int32(sd[base + '.weight_packed'], 4, shape, packed_dim=1)
    zp = None if sym else unpack_from_int32(sd[base + '.weight_zero_point'], 4, torch.Size([shape[0], s.shape[1]]),
                                            packed_dim=0)
    args = QuantizationArgs(num_bits=4, type='int', symmetric=sym, strategy='group' if group_size else 'channel',
                            group_size=group_size)
    return dequantize(x_q, s, zp, args=args, dtype=scale_dtype).to(torch.bfloat16)


def main():
    from transformers import AutoModelForCausalLM
    from painlessinferenceacceleration_b200.common import ops
    from tests import w4_moe_ckpt
    out = {}
    for name, (fmt, sym, gs, sdt, seed, _) in w4_moe_ckpt.FIXTURES.items():
        if fmt == 'gptq':
            continue
        cfg, sd, codes = w4_moe_ckpt.build(name)
        w = {}
        for base, (u, s, z) in codes.items():
            w[base] = decompress(sd, base, sym, gs, sdt)
            assert torch.equal(w[base], ops.dequantize_w4(u, s, z, gs or u.shape[1])), (name, base)
        state = {k: v for k, v in sd.items() if k.endswith('norm.weight') or k in ('model.embed_tokens.weight',
                                                                                   'lm_head.weight')}
        E = cfg.num_local_experts
        for li in range(cfg.num_hidden_layers):
            pre = f'model.layers.{li}.'
            for p in w4_moe_ckpt.ATTN:
                state[f'{pre}{p}.weight'] = w[pre + p]
            state[pre + 'mlp.gate.weight'] = sd[pre + 'block_sparse_moe.gate.weight']
            ex = pre + 'block_sparse_moe.experts.'
            state[pre + 'mlp.experts.gate_up_proj'] = torch.stack(
                [torch.cat([w[f'{ex}{e}.w1'], w[f'{ex}{e}.w3']]) for e in range(E)])
            state[pre + 'mlp.experts.down_proj'] = torch.stack([w[f'{ex}{e}.w2'] for e in range(E)])
        del cfg.quantization_config
        ids = w4_moe_ckpt.prompt(name)
        for dt, tag in ((torch.bfloat16, 'bf16'), (torch.float32, 'fp32')):
            m = AutoModelForCausalLM.from_config(cfg, attn_implementation='eager', dtype=dt).eval()
            m.load_state_dict({k: v.to(dt) for k, v in state.items()}, strict=True)
            with torch.no_grad():
                out[f'{name}/{tag}'] = m(input_ids=ids).logits[0].float().numpy()
        print(name, out[name + '/bf16'].shape, float(np.abs(out[name + '/bf16'] - out[name + '/fp32']).max()))
    np.savez_compressed(os.path.join(ROOT, 'tests', 'golden', 'w4_mixtral_logits.npz'), **out)


if __name__ == '__main__':
    main()
