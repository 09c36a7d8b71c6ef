# -*- coding: utf-8 -*-
"""Seeded tiny BLOOM models (no checkpoints exist offline): transformers' own BloomForCausalLM (the oracle) with
non-zero biases and non-unit LayerNorm weights and biases, and our BloomForCausalLM holding the same weights.
Head dims 64 (bloom-560m), 80 (bloom-3b), 96 (bloom-1b1) and 128 (bloom-1b7 / 7b1), with head counts that are not
all powers of two (ALiBi's second slope series)."""
import torch

HEADS = {64: 4, 80: 3, 96: 5, 128: 3}


def tiny_config(head_dim, vocab=200, layers=2, tie=True):
    from transformers import BloomConfig
    H = HEADS[head_dim]
    return BloomConfig(vocab_size=vocab, hidden_size=H * head_dim, n_layer=layers, n_head=H, layer_norm_epsilon=1e-5,
                       initializer_range=0.06, bos_token_id=1, eos_token_id=2, pad_token_id=3,
                       tie_word_embeddings=tie)


@torch.no_grad()
def hf_model(head_dim, seed=0, device='cuda:0', tie=True):
    """transformers' BloomForCausalLM in fp32 (bf16-representable values), eval mode, with perturbed biases and
    LayerNorms"""
    from transformers import BloomForCausalLM
    torch.manual_seed(seed)
    m = BloomForCausalLM(tiny_config(head_dim, tie=tie)).float().eval()
    g = torch.Generator().manual_seed(seed + 1000)
    for name, p in m.named_parameters():
        if 'layernorm' in name or 'ln_f' in name:
            if name.endswith('weight'):
                p.copy_(1.0 + 0.2 * torch.randn(p.shape, generator=g))
            else:
                p.copy_(0.05 * torch.randn(p.shape, generator=g))
        elif name.endswith('bias'):
            p.copy_(0.03 * torch.randn(p.shape, generator=g))
        elif name.endswith('word_embeddings.weight'):
            p.copy_(0.5 * torch.randn(p.shape, generator=g))
    for p in m.parameters():   # the oracle holds exactly the bf16 weights our model runs
        p.copy_(p.to(torch.bfloat16).float())
    return m.to(device)


def tiny_model(head_dim, seed=0, device='cuda:0', tie=True):
    """(ours, hf): our model holding the bf16-rounded weights of the fp32 HF oracle"""
    from painlessinferenceacceleration_b200.models.bloom.modeling_bloom import BloomForCausalLM
    hf = hf_model(head_dim, seed, device, tie)
    ours = BloomForCausalLM(hf.config, device=torch.device(device)).load_hf_state_dict(hf.state_dict())
    return ours, hf


@torch.no_grad()
def hf_logits(hf, ids, dtype=torch.float32):
    """causal forward of the HF model over ids [T] in `dtype` (float32: the truth; bfloat16: eager bf16 with the
    bf16-rounded weights); fp32 logits [T, V]"""
    m = hf
    if dtype != torch.float32:
        import copy
        m = copy.deepcopy(hf).to(dtype)
    return m(input_ids=ids[None].to(next(hf.parameters()).device)).logits[0].float()
