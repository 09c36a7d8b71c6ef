# -*- coding: utf-8 -*-
"""Seeded tiny OPT models (no checkpoints exist offline): transformers' own OPTForCausalLM (the oracle) in fp32 with
bf16-representable weights, non-zero biases, perturbed LayerNorms and position embeddings, and our OPTForCausalLM
holding the same weights.  Four shapes: pre-LN at head dims 64 (OPT-125m / 350m / 1.3b), 80 (OPT-2.7b, zero-padded to
128) and 128 (OPT-6.7b and up), and an OPT-350m-like post-LN model with word_embed_proj_dim != hidden_size
(project_in / project_out, no final LayerNorm)."""
import torch

SHAPES = {  # name: (head_dim, heads, do_layer_norm_before, word_embed_proj_dim or None)
    64: (64, 4, True, None),
    80: (80, 3, True, None),
    128: (128, 2, True, None),
    '350m': (64, 4, False, 128),
}
MAX_POS = 512


def tiny_config(shape, vocab=200, layers=2, tie=True):
    from transformers import OPTConfig
    d, H, pre, wp = SHAPES[shape]
    E = d * H
    return OPTConfig(vocab_size=vocab, hidden_size=E, num_hidden_layers=layers, ffn_dim=2 * E,
                     num_attention_heads=H, max_position_embeddings=MAX_POS, do_layer_norm_before=pre,
                     word_embed_proj_dim=wp if wp is not None else E, init_std=0.06, pad_token_id=1, bos_token_id=2,
                     eos_token_id=2, tie_word_embeddings=tie, dropout=0.0, attention_dropout=0.0,
                     activation_dropout=0.0)


@torch.no_grad()
def hf_model(shape, seed=0, device='cuda:0', tie=True):
    """transformers' OPTForCausalLM in fp32 (bf16-representable values), eval mode, with perturbed biases, LayerNorms
    and position embeddings"""
    from transformers import OPTForCausalLM
    torch.manual_seed(seed)
    m = OPTForCausalLM(tiny_config(shape, tie=tie)).float().eval()
    g = torch.Generator().manual_seed(seed + 1000)
    for name, p in m.named_parameters():
        if 'layer_norm' in name:
            if name.endswith('weight'):
                p.copy_(1.0 + 0.2 * torch.randn(p.shape, generator=g))
            else:
                p.copy_(0.05 * torch.randn(p.shape, generator=g))
        elif name.endswith('bias'):
            p.copy_(0.03 * torch.randn(p.shape, generator=g))
        elif name.endswith('embed_tokens.weight'):
            p.copy_(0.5 * torch.randn(p.shape, generator=g))
        elif name.endswith('embed_positions.weight'):
            p.copy_(0.3 * torch.randn(p.shape, generator=g))
    for p in m.parameters():   # the oracle holds exactly the bf16 weights our model runs
        p.copy_(p.to(torch.bfloat16).float())
    return m.to(device)


def tiny_model(shape, seed=0, device='cuda:0', tie=True, batch=False):
    """(ours, hf): our model (the batched-loop class with batch=True) holding the bf16-rounded weights of the fp32 HF
    oracle"""
    if batch:
        from painlessinferenceacceleration_b200.models.opt.modeling_opt_batch import OPTForCausalLM
    else:
        from painlessinferenceacceleration_b200.models.opt.modeling_opt import OPTForCausalLM
    hf = hf_model(shape, seed, device, tie)
    ours = OPTForCausalLM(hf.config, device=torch.device(device)).load_hf_state_dict(hf.state_dict())
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
