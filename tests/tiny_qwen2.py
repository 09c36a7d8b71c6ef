# -*- coding: utf-8 -*-
"""a seeded tiny random-init HF Qwen2 (no checkpoints exist offline): 7 query heads over 1 KV head - an odd GQA group,
like Qwen2-7B's 28 / 4 - head dim 128 and non-zero q/k/v biases.  Built the way tests/tiny_models.py builds the other
families (same seeding and weight init), plus the biases."""
import torch


def qwen2_config(vocab=64, **over):
    from transformers import Qwen2Config
    cfg = Qwen2Config(vocab_size=vocab, hidden_size=896, intermediate_size=512, num_hidden_layers=2,
                      num_attention_heads=7, num_key_value_heads=1, max_position_embeddings=1024, rms_norm_eps=1e-6,
                      rope_theta=1000000.0, use_sliding_window=False, tie_word_embeddings=False, bos_token_id=1,
                      eos_token_id=2, pad_token_id=0)
    for k, v in over.items():
        setattr(cfg, k, v)
    cfg._attn_implementation = 'eager'
    return cfg


def qwen2_hf_model(seed=0, dtype=torch.float32, device='cpu', vocab=64, **over):
    from transformers import AutoModelForCausalLM
    torch.manual_seed(seed)
    model = AutoModelForCausalLM.from_config(qwen2_config(vocab=vocab, **over), attn_implementation='eager')
    with torch.no_grad():
        for n, p in model.named_parameters():
            if p.dim() >= 2:
                p.normal_(0.0, 0.08)
        for layer in model.model.layers:
            a = layer.self_attn
            a.q_proj.bias.normal_(0.0, 1.0)
            a.k_proj.bias.normal_(0.0, 3.0)   # trained Qwen2 checkpoints carry large k biases
            a.v_proj.bias.normal_(0.0, 1.0)
    return model.to(device=device, dtype=dtype).eval()
