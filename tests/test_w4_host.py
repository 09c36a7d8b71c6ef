# -*- coding: utf-8 -*-
"""Host checks of the int4 (GPTQ / compressed-tensors W4A16) weight mode: the two unpackers against compressed_tensors'
own compressor and decompressor, the GPTQ v1 layout, the tiled layout the int4 GEMM reads, the gate/up interleave of
codes, scales and zero points, loading a checkpoint on the CPU, and every refusal - none of which touches a GPU."""
import json

import pytest
import torch

from tests import w4_ckpt

ct = pytest.importorskip('compressed_tensors')


def _ops():
    from painlessinferenceacceleration_b200.common import ops
    return ops


CASES = [(128, True, torch.bfloat16), (256, False, torch.bfloat16), (None, False, torch.float16),
         (128, False, torch.float16)]


@pytest.mark.parametrize('group_size,sym,sdt', CASES)
def test_compressed_tensors_unpacker_matches_the_library(group_size, sym, sdt):
    """random u / s / z packed by the library's pack_to_int32 and dequantised by its _dequantize: our unpacker returns
    (u, s, z) and ops.dequantize_w4 of them equals the library's weight .to(bf16) bit for bit"""
    from compressed_tensors.compressors.pack_quantized.helpers import pack_to_int32, unpack_from_int32
    from compressed_tensors.quantization import QuantizationArgs
    from compressed_tensors.quantization.lifecycle.forward import dequantize
    ops = _ops()
    N, K = 384, 512
    u, s, z = w4_ckpt.random_codes(N, K, group_size, sym, sdt, torch.Generator().manual_seed(N + K))
    if not sym:   # the whole zero-point range the library can store
        z[:16, 0] = torch.arange(16, dtype=torch.uint8)
    packed = pack_to_int32((u.to(torch.int16) - 8).to(torch.int8), 4, packed_dim=1)
    assert torch.equal(packed, w4_ckpt.pack_compressed_tensors(u, s, z, sym)['weight_packed'])
    zp_signed = (z.to(torch.int16) - 8).to(torch.int8)
    zp_packed = pack_to_int32(zp_signed, 4, packed_dim=0) if not sym else None
    got_u, got_s, got_z, gs = ops.unpack_compressed_tensors_w4(packed, s, torch.tensor([N, K]), zp_packed)
    assert torch.equal(got_u, u) and torch.equal(got_s, s) and torch.equal(got_z, z) and gs == (group_size or K)
    args = QuantizationArgs(num_bits=4, type='int', symmetric=sym, strategy='group' if group_size else 'channel',
                            group_size=group_size)
    x_q = unpack_from_int32(packed, 4, torch.Size([N, K]), packed_dim=1)
    lib = dequantize(x_q, s, zp_signed if not sym else None, args=args, dtype=sdt).to(torch.bfloat16)
    assert torch.equal(ops.dequantize_w4(got_u, got_s, got_z, gs), lib)


@pytest.mark.parametrize('group_size,sym,sdt', CASES)
def test_gptq_unpacker_gives_the_same_codes(group_size, sym, sdt):
    """the same codes in GPTQ v1 layout (K-packed qweight, zeros stored - 1, [G, N] scales, trivial g_idx) unpack to the
    identical (u, s, z)"""
    ops = _ops()
    N, K = 256, 768
    u, s, z = w4_ckpt.random_codes(N, K, group_size, sym, sdt, torch.Generator().manual_seed(7))
    g = w4_ckpt.pack_gptq(u, s, z, group_size)
    assert g['qweight'].shape == (K // 8, N) and g['qzeros'].shape == (K // (group_size or K), N // 8)
    got = ops.unpack_gptq_w4(g['qweight'], g['qzeros'], g['scales'], g['g_idx'])
    ct_got = ops.unpack_compressed_tensors_w4(**w4_ckpt.pack_compressed_tensors(u, s, z, sym))
    for a, b in zip(got, ct_got):
        assert (a == b) if isinstance(a, int) else torch.equal(a, b)
    if group_size:   # an act-order permutation of the groups
        with pytest.raises(ValueError, match='g_idx'):
            ops.unpack_gptq_w4(g['qweight'], g['qzeros'], g['scales'], g['g_idx'].flip(0))


def test_tiled_layout_and_its_inverse():
    ops = _ops()
    gen = torch.Generator().manual_seed(1)
    for K in (512, 384):
        u = torch.randint(0, 16, (256, K), generator=gen).to(torch.uint8)
        t = ops.tile_weight_w4(u)
        assert t.shape == (2, -(-K // 256), 128, 128) and t.dtype == torch.uint8
        # block (tile, chunk), row r, byte b: nibble positions p = 2b (low) and 2b + 1 (high) of 16-byte group b // 16
        perm = ops._W4_KPERM
        for (nt, kc, r, b) in [(0, 0, 0, 0), (1, 0, 127, 127), (0, 1, 5, 18), (1, 1, 64, 37)]:
            if kc * 256 + (b // 16) * 32 >= K:
                continue
            for half in (0, 1):
                p = (2 * b + half) % 32
                k = kc * 256 + (b // 16) * 32 + perm[p]
                assert (t[nt, kc, r, b] >> (4 * half)) & 15 == u[nt * 128 + r, k]
        assert torch.equal(ops.untile_weight_w4(t, K), u)
    with pytest.raises(ValueError):
        ops.tile_weight_w4(u[:, :320])
    # word c of a 16-byte group: nibble j holds k 2c + (0, 8, 16, 24)[j % 4] + j // 4 (the kernel's fragment pairs)
    assert sorted(ops._W4_KPERM) == list(range(32))
    assert ops._W4_KPERM[8 * 3 + 0] == 6 and ops._W4_KPERM[8 * 3 + 4] == 7 and ops._W4_KPERM[8 * 3 + 3] == 30


def test_gate_up_interleave_carries_scales_and_zeros():
    from painlessinferenceacceleration_b200.models.llama.modeling_llama import Int4Linear
    ops = _ops()
    u, s, z = w4_ckpt.random_codes(512, 256, 128, False, torch.bfloat16, torch.Generator().manual_seed(3))
    lin = Int4Linear(u, s, z, 128, interleaved=True)
    got = lin.codes()
    assert torch.equal(got[0], u) and torch.equal(got[1], s) and torch.equal(got[2], z)
    assert torch.equal(lin.dequantize(), ops.dequantize_w4(u, s, z, 128))
    # stored rows: 64 gate rows then the 64 up rows of the same columns, scales / zero points alike
    assert torch.equal(lin.scale[:, 64:128].t(), s[256:320]) and torch.equal(lin.zero[:, 64:128].t(), z[256:320])
    assert torch.equal(ops.untile_weight_w4(lin.qweight, 256)[64:128], u[256:320])


@pytest.mark.parametrize('name', ['llama_ct_sym_g128_bf16', 'qwen2_ct_asym_g128_fp16', 'llama_gptq_asym_g128_fp16'])
def test_checkpoint_loads_its_codes_on_the_cpu(name, tmp_path):
    """from_pretrained reads the checkpoint's quantization_config and loads its codes, scales and zero points as they
    are (q|k|v fused, the HF names view their rows)"""
    from painlessinferenceacceleration_b200.models.llama.modeling_llama import LlamaForCausalLM
    from painlessinferenceacceleration_b200.models.qwen2.modeling_qwen2 import Qwen2ForCausalLM
    cls = Qwen2ForCausalLM if name.startswith('qwen2') else LlamaForCausalLM
    codes = w4_ckpt.write(name, str(tmp_path))
    m = cls.from_pretrained(str(tmp_path), device='cpu')
    assert m._w4 and not m._fp8
    for li, layer in enumerate(m.model.layers):
        for p in w4_ckpt.PROJ:
            mod = layer.get_submodule(p)
            u, s, z = codes[f'model.layers.{li}.{p}']
            got = mod.codes()
            assert torch.equal(got[0], u) and torch.equal(got[1], s) and torch.equal(got[2], z), (li, p)
    if name.startswith('qwen2'):
        a = m.model.layers[0].self_attn
        assert a.qkv_bias is not None and a.qkv_bias.dtype == torch.bfloat16


def _cfg_dir(tmp_path, name, edit):
    w4_ckpt.write(name, str(tmp_path))
    f = tmp_path / 'config.json'
    d = json.loads(f.read_text())
    edit(d['quantization_config'], d)
    f.write_text(json.dumps(d))
    return str(tmp_path)


def _set(path, value):
    def edit(q, d):
        o = q
        for k in path[:-1]:
            o = o[k]
        o[path[-1]] = value
    return edit


WG = ('config_groups', 'group_0', 'weights')
REFUSALS = [
    ('llama_ct_sym_g128_bf16', _set(WG + ('num_bits',), 8), 'num_bits'),
    ('llama_ct_sym_g128_bf16', _set(WG + ('group_size',), 64), 'group_size'),
    ('llama_ct_sym_g128_bf16', _set(WG + ('group_size',), 32), 'group_size'),
    ('llama_ct_sym_g128_bf16', _set(WG + ('actorder',), 'group'), 'actorder'),
    ('llama_ct_sym_g128_bf16', _set(WG + ('type',), 'float'), 'type'),
    ('llama_ct_sym_g128_bf16', _set(('ignore',), []), 'lm_head'),
    ('llama_ct_sym_g128_bf16', _set(('format',), 'int-quantized'), 'format'),
    ('llama_ct_sym_g128_bf16', _set(('config_groups', 'group_0', 'input_activations'), {'num_bits': 8}),
     'input_activations'),
    ('llama_gptq_asym_g128_fp16', _set(('bits',), 8), 'bits'),
    ('llama_gptq_asym_g128_fp16', _set(('group_size',), 64), 'group_size'),
    ('llama_gptq_asym_g128_fp16', _set(('desc_act',), True), 'desc_act'),
    ('llama_gptq_asym_g128_fp16', _set(('checkpoint_format',), 'gptq_v2'), 'checkpoint_format'),
    ('llama_gptq_asym_g128_fp16', _set(('lm_head',), True), 'lm_head'),
    ('llama_gptq_asym_g128_fp16', _set(('quant_method',), 'awq'), 'quant_method'),
    ('llama_gptq_asym_g128_fp16', lambda q, d: d.update(intermediate_size=576), 'intermediate_size'),
]


@pytest.mark.parametrize('name,edit,field', REFUSALS, ids=[f'{r[2]}-{i}' for i, r in enumerate(REFUSALS)])
def test_refusals_name_their_field_before_any_gpu_memory(name, edit, field, tmp_path, monkeypatch):
    from painlessinferenceacceleration_b200.models.llama.modeling_llama import LlamaForCausalLM
    path = _cfg_dir(tmp_path, name, edit)
    touched = []
    monkeypatch.setattr(LlamaForCausalLM, '_fp8_skeleton', classmethod(lambda *a, **k: touched.append(1)))
    with pytest.raises(ValueError, match=field):
        LlamaForCausalLM.from_pretrained(path)
    assert not touched


def test_quantised_lm_head_tensor_and_act_order_tensor_are_refused(tmp_path):
    from safetensors.torch import load_file, save_file
    from painlessinferenceacceleration_b200.models.llama.modeling_llama import LlamaForCausalLM
    w4_ckpt.write('llama_ct_sym_g128_bf16', str(tmp_path))
    f = tmp_path / 'model.safetensors'
    sd = load_file(str(f))
    sd['lm_head.weight_packed'] = torch.zeros((200, 32), dtype=torch.int32)
    save_file(sd, str(f), metadata={'format': 'pt'})
    with pytest.raises(ValueError, match='lm_head'):
        LlamaForCausalLM.from_pretrained(str(tmp_path), device='cpu')
    del sd['lm_head.weight_packed']
    sd['model.layers.0.self_attn.q_proj.weight_g_idx'] = torch.zeros(256, dtype=torch.int32)
    save_file(sd, str(f), metadata={'format': 'pt'})
    with pytest.raises(ValueError, match='g_idx'):
        LlamaForCausalLM.from_pretrained(str(tmp_path), device='cpu')


def test_fp8_requests_on_an_int4_checkpoint_are_refused(tmp_path):
    from painlessinferenceacceleration_b200.models.llama.modeling_llama import LlamaForCausalLM
    w4_ckpt.write('llama_ct_sym_g128_bf16', str(tmp_path))
    with pytest.raises(ValueError, match='already quantised'):
        LlamaForCausalLM.from_pretrained(str(tmp_path), quantization='fp8')
    with pytest.raises(ValueError, match='int4'):
        LlamaForCausalLM.from_pretrained(str(tmp_path), quantization='int4')
    m = LlamaForCausalLM.from_pretrained(str(tmp_path), device='cpu')
    with pytest.raises(ValueError, match='int4'):
        m.quantize_fp8()


def test_other_families_keep_their_refusal(tmp_path):
    """Mixtral / GLM / Baichuan / Qwen (v1) do not read int4 checkpoints through the Llama loader"""
    from painlessinferenceacceleration_b200.models.baichuan.modeling_baichuan import BaichuanBase
    from painlessinferenceacceleration_b200.models.glm4.modeling_glm4 import GlmForCausalLM
    from painlessinferenceacceleration_b200.models.mixtral.modeling_mixtral import MixtralForCausalLM
    from painlessinferenceacceleration_b200.models.qwen.modeling_qwen import QWenLMHeadModel
    assert not any(c.int4_checkpoints for c in (BaichuanBase, GlmForCausalLM, MixtralForCausalLM, QWenLMHeadModel))


def test_new_symbol_is_declared_and_typed():
    from painlessinferenceacceleration_b200 import _lib
    assert 'pia_gemm_plan_create_w4' in _lib.SYMBOLS
    assert hasattr(_lib.load(), 'pia_gemm_plan_create_w4')
