# -*- coding: utf-8 -*-
"""Records tests/golden/w4_logits.npz: for every int4 checkpoint of tests/w4_ckpt.py (tiny Llama, Mistral and Qwen2 in
compressed-tensors pack-quantized format, symmetric and asymmetric, and one GPTQ v1 checkpoint with the codes of one of
them), the logits of the eager transformers model of that checkpoint on its prompt, in bf16 and in fp32.  The
compressed-tensors checkpoints are loaded by transformers, which decompresses them with compressed_tensors; the packed
tensors are first checked against compressed_tensors' own packer.  The GPTQ checkpoint's logits are those of the
compressed-tensors checkpoint with the same codes (the GPU test checks the two load to identical weights).

Needs transformers and compressed_tensors (this is why the GPU tests read the recorded logits):
    python tests/golden/gen_w4_golden.py"""
import os
import sys
import tempfile

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)


def check_packing(name, sd, codes):
    from compressed_tensors.compressors.pack_quantized.helpers import pack_to_int32
    for base, (u, s, z) in codes.items():
        got = sd[base + '.weight_packed']
        assert torch.equal(got, pack_to_int32((u.to(torch.int16) - 8).to(torch.int8), 4, packed_dim=1)), (name, base)
        if base + '.weight_zero_point' in sd:
            assert torch.equal(sd[base + '.weight_zero_point'],
                               pack_to_int32((z.to(torch.int16) - 8).to(torch.int8), 4, packed_dim=0)), (name, base)


def eager_logits(path, ids, scale_dtype):
    """the checkpoint decompressed by compressed_tensors (run_compressed=False) in the scale's dtype, so that each weight
    is dtype_s(s * (u - z)) as the checkpoint defines it (loaded into a bf16 model, transformers would cast fp16 scales
    to bf16 first), then rounded to bf16: the eager bf16 model and its fp32 twin run those weights"""
    from transformers import AutoModelForCausalLM, CompressedTensorsConfig
    m = AutoModelForCausalLM.from_pretrained(path, dtype=scale_dtype, attn_implementation='eager',
                                             quantization_config=CompressedTensorsConfig(run_compressed=False))
    for mod in m.modules():
        assert 'Quantized' not in type(mod).__name__ and not hasattr(mod, 'weight_packed'), type(mod)
    sd = {k: v for k, v in m.state_dict().items() if not k.endswith(('_scale', '_shape', '_zero_point'))}
    cfg = m.config
    del cfg.quantization_config
    out = []
    for dt in (torch.bfloat16, torch.float32):
        e = AutoModelForCausalLM.from_config(cfg, attn_implementation='eager', dtype=dt).eval()
        e.load_state_dict({k: v.to(torch.bfloat16).to(dt) for k, v in sd.items()})
        with torch.no_grad():
            out.append(e(input_ids=ids).logits[0].float().numpy())
    return sd, out[0], out[1]


def main():
    from tests import w4_ckpt
    out = {}
    for name, (family, fmt, sym, gs, sdt, seed) in w4_ckpt.FIXTURES.items():
        if fmt == 'gptq':
            continue
        cfg, sd, codes = w4_ckpt.build(name)
        check_packing(name, sd, codes)
        with tempfile.TemporaryDirectory() as d:
            w4_ckpt.write(name, d)
            sd, bf, f32 = eager_logits(d, w4_ckpt.prompt(name), sdt)
        from painlessinferenceacceleration_b200.common import ops   # the library's dequantisation is the formula's
        for base, (u, s, z) in codes.items():
            w = sd[base + '.weight'].to(torch.bfloat16)
            assert torch.equal(w, ops.dequantize_w4(u, s, z, gs or u.shape[1])), (name, base)
        out[name + '/bf16'] = bf
        out[name + '/fp32'] = f32
        print(name, bf.shape, float(np.abs(bf - f32).max()))
    np.savez_compressed(os.path.join(ROOT, 'tests', 'golden', 'w4_logits.npz'), **out)


if __name__ == '__main__':
    main()
