# -*- coding: utf-8 -*-
"""Host checks of the fp8 (e4m3) weight mode: the quantiser against an independent restatement of its recipe (per-row
scale amax / 448, round to nearest even on the e4m3 grid, ties to the even code), the tiled layout the fp8 GEMM reads,
and the refusals that happen before anything is converted.  torch's CPU float8 is enough; no GPU needed."""
import numpy as np
import pytest
import torch


def _e4m3_grid():
    """value of every non-negative finite e4m3fn code 0x00..0x7E (ascending with the code)"""
    c = np.arange(0x7F)
    e, m = (c >> 3) & 0xF, c & 7
    return np.where(e == 0, m / 8.0 * 2.0 ** -6, (1 + m / 8.0) * 2.0 ** (e - 7.0))


def _reference_quantize(w):
    """the recipe, written out with numpy: s = amax / 448 (1 for a zero row), x = W / s in fp32, clamp to +-448, nearest
    grid value with ties to the even code; the sign bit follows x (so -0 and tiny negatives give 0x80)"""
    w32 = w.float().numpy().astype(np.float32)
    amax = np.abs(w32).max(axis=1)
    s = np.where(amax > 0, amax / np.float32(448.0), np.float32(1.0)).astype(np.float32)
    x = np.clip(w32 / s[:, None], np.float32(-448.0), np.float32(448.0))
    grid = _e4m3_grid()
    a = np.abs(x).astype(np.float64)
    hi = np.clip(np.searchsorted(grid, a), 0, len(grid) - 1)
    lo = np.clip(hi - 1, 0, None)
    dlo, dhi = a - grid[lo], grid[hi] - a
    code = np.where(dlo < dhi, lo, np.where(dhi < dlo, hi, np.where(lo % 2 == 0, lo, hi)))
    code = np.where(a == grid[hi], hi, code)
    return (code | (np.signbit(x) << 7)).astype(np.uint8), s


def _weights():
    g = torch.Generator().manual_seed(0)
    w = (torch.randn((6, 384), generator=g) * 0.02).to(torch.bfloat16)
    w[1] = 0                                               # all-zero row: s = 1, codes 0
    w[2, :] = -w[2, :].abs()                               # negative row
    w[3, :7] = torch.tensor([1e-9, -1e-9, 3e-4, -3e-4, 0.0, -0.0, 5.0])   # underflow to +-0, subnormal codes
    # a row whose amax is 448 (s = 1 exactly) holding every midpoint between neighbouring grid values that bf16 holds:
    # exercises ties-to-even on the whole range, both signs
    grid = _e4m3_grid()
    mids = torch.tensor((grid[:-1] + grid[1:]) / 2, dtype=torch.float32)
    mids = mids[mids.to(torch.bfloat16).float() == mids]
    row = torch.zeros(384)
    row[0] = 448.0
    row[1:1 + len(mids)] = mids
    row[1 + len(mids):1 + 2 * len(mids)] = -mids
    w[4] = row.to(torch.bfloat16)
    w[5] = (torch.randn(384, generator=g) * 300).to(torch.bfloat16)
    return w


def test_quantiser_matches_the_recipe_bit_for_bit():
    from painlessinferenceacceleration_b200.common import ops
    w = _weights()
    q, s = ops.quantize_fp8(w)
    want_q, want_s = _reference_quantize(w)
    assert q.dtype == torch.float8_e4m3fn and s.dtype == torch.float32
    assert np.array_equal(s.numpy(), want_s)
    assert np.array_equal(q.view(torch.uint8).numpy(), want_q)
    assert (q.view(torch.uint8)[1] == 0).all() and s[1].item() == 1.0
    # the dequantised weight is float(q) * s and never leaves the grid's range
    deq = q.float() * s[:, None]
    assert deq.abs().max(dim=1).values.le(s * 448 + 1e-6).all()


def test_quantiser_handles_stacked_weights_row_by_row():
    from painlessinferenceacceleration_b200.common import ops
    w = torch.stack([_weights(), _weights().flip(0)])
    q, s = ops.quantize_fp8(w)
    for e in range(2):
        qe, se = ops.quantize_fp8(w[e])
        assert torch.equal(q[e].view(torch.uint8), qe.view(torch.uint8)) and torch.equal(s[e], se)


def test_tiled_layout_and_its_inverse():
    from painlessinferenceacceleration_b200.common import ops
    g = torch.Generator().manual_seed(1)
    codes = torch.randint(0, 256, (2, 256, 384), generator=g, dtype=torch.uint8)
    codes[codes == 0x7F] = 0
    codes[codes == 0xFF] = 0
    q = codes.view(torch.float8_e4m3fn)
    t = ops.tile_weight_fp8(q)
    assert t.shape == (2, 2, 3, 128, 128) and t.dtype == torch.uint8 and t.is_contiguous()
    # block (e, tile, chunk) holds rows tile*128.., k chunk*128..; inside a 16-byte group position p holds k PERM[p]
    perm = ops._FP8_KPERM
    for (e, nt, kt, r, p) in [(0, 0, 0, 0, 0), (1, 1, 2, 127, 127), (0, 1, 1, 5, 18), (1, 0, 2, 64, 37)]:
        k = kt * 128 + (p // 16) * 16 + perm[p % 16]
        assert t[e, nt, kt, r, p] == codes[e, nt * 128 + r, k]
    assert torch.equal(ops.untile_weight_fp8(t).view(torch.uint8), codes)
    with pytest.raises(ValueError):
        ops.tile_weight_fp8(q[:, :, :320])


def test_gate_up_order_matches_interleave_and_inverts():
    from painlessinferenceacceleration_b200.common import ops
    from painlessinferenceacceleration_b200.models.llama.modeling_llama import _gate_up_order
    w = torch.randn((512, 128))
    assert torch.equal(_gate_up_order(w), ops.interleave_gate_up(w))
    assert torch.equal(_gate_up_order(_gate_up_order(w), inverse=True), w)
    s = torch.randn((3, 512))
    assert torch.equal(_gate_up_order(s, vec=True)[1], ops.interleave_gate_up(s[1][:, None])[:, 0])
    assert torch.equal(_gate_up_order(_gate_up_order(s, vec=True), inverse=True, vec=True), s)


def test_misaligned_model_raises_before_converting():
    from transformers import LlamaConfig
    from painlessinferenceacceleration_b200.models.llama.modeling_llama import LlamaForCausalLM
    cfg = LlamaConfig(vocab_size=64, hidden_size=256, intermediate_size=320, num_hidden_layers=2,
                      num_attention_heads=2, num_key_value_heads=2, rms_norm_eps=1e-6)
    m = LlamaForCausalLM(cfg, device='cpu')
    with pytest.raises(ValueError, match='divisible by 128'):
        m.quantize_fp8()
    assert not m._fp8
    assert all(isinstance(layer.self_attn.q_proj, torch.nn.Linear) for layer in m.model.layers)
    assert all(p.dtype == torch.bfloat16 for p in m.parameters())


def test_gpt2_has_no_fp8_mode():
    from transformers import GPT2Config
    from painlessinferenceacceleration_b200.models.gpt2.modeling_gpt2 import GPT2LMHeadModel
    m = GPT2LMHeadModel(GPT2Config(vocab_size=64, n_positions=128, n_embd=64, n_layer=1, n_head=4), device='meta')
    with pytest.raises(NotImplementedError):
        m.quantize_fp8()


def test_unknown_quantization_is_refused(tmp_path):
    from painlessinferenceacceleration_b200.models.llama.modeling_llama import LlamaForCausalLM
    with pytest.raises(ValueError):
        LlamaForCausalLM.from_pretrained(str(tmp_path), quantization='int4')


def test_build_fp8_equals_quantize_fp8_of_the_filled_bf16_model():
    """LlamaForCausalLM.build_fp8 (one layer in bf16 at a time) gives the bytes of filling the whole bf16 model the same
    way and calling quantize_fp8(); bench.synth_fill on the skeleton leaves the meta projections alone"""
    import zlib
    import bench
    from transformers import LlamaConfig
    from painlessinferenceacceleration_b200.models.llama.modeling_llama import LlamaForCausalLM
    cfg = LlamaConfig(vocab_size=512, hidden_size=256, intermediate_size=512, num_hidden_layers=2,
                      num_attention_heads=2, num_key_value_heads=2, rms_norm_eps=1e-6)
    a = LlamaForCausalLM(cfg, device='cpu')
    bench.synth_fill(a, cfg)
    a.quantize_fp8()
    b = LlamaForCausalLM.build_fp8(cfg, lambda m: bench.synth_fill(m, cfg),
                                   lambda n, t: bench.hashed_normal_(t, zlib.crc32(n.encode()), 0.02), device='cpu')
    pa, pb = dict(a.named_parameters()), dict(b.named_parameters())
    assert sorted(pa) == sorted(pb)
    for k in pa:
        assert torch.equal(pa[k].view(-1).view(torch.uint8), pb[k].view(-1).view(torch.uint8)), k
