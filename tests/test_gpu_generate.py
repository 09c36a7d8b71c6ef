# -*- coding: utf-8 -*-
"""End-to-end parity of the H100 loop (generate -> lookahead_generation, one CUDA graph per step) with the CPU
restatement of the reference loop (oracle/loop.py) on seeded tiny models that share their weights.

bf16 caveat (lookahead/README.md:45, SURVEY A.2-16): identical text is only guaranteed in fp32; in bf16 the two
implementations round differently (fused fp32 scores vs bf16 scores), so a token may flip where the oracle's
top-2 logit margin is within bf16 noise.  The test therefore requires exact equality up to the first position
whose oracle margin is below MARGIN, and requires that the great majority of sequences match entirely."""
import pytest
import torch

from tests.tiny_models import prompts, tiny_config, tiny_hf_model

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'
EPS = 0.35  # fp32 logit margin below which a bf16 implementation may legitimately pick the other candidate


def _diag(name, **kw):
    import json
    import os
    d = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), 'gpurun_out')
    if os.path.isdir(d):
        with open(os.path.join(d, 'diag_generate.jsonl'), 'a') as f:
            f.write(json.dumps(dict(test=name, **kw)) + '\n')


def _pair(family, seed):
    """HF oracle model (bf16, on the GPU so that it is fast) and our model with the same weights"""
    from painlessinferenceacceleration_b200.models.llama.modeling_llama import LlamaForCausalLM
    from painlessinferenceacceleration_b200.models.mixtral.modeling_mixtral import MixtralForCausalLM
    hf = tiny_hf_model(family, seed=seed, dtype=torch.bfloat16, device=DEV, vocab=200)
    hf.fp32_twin = None
    ours = (MixtralForCausalLM if family == 'mixtral' else LlamaForCausalLM)(hf.config, device=torch.device(DEV))
    missing = ours.load_state_dict(hf.state_dict(), strict=False)
    assert not missing.missing_keys, missing
    return hf, ours


def _legit_divergence(family, hf, prefix, tok_a, tok_b, penalty=1.0):
    """a bf16 flip is legitimate iff, under an fp32 evaluation of the same weights on the common prefix, BOTH
    candidate tokens lie within the bf16 noise of the optimum; noise = the reference-style eager bf16 forward's own
    max logit error on that prefix (x4, +0.05)."""
    if hf.fp32_twin is None:
        twin = tiny_hf_model(family, seed=0, dtype=torch.float32, device=DEV, vocab=200)
        twin.load_state_dict({k: v.float() for k, v in hf.state_dict().items()})
        hf.fp32_twin = twin
    with torch.no_grad():
        truth = hf.fp32_twin(input_ids=prefix).logits[0, -1].float()
        noisy = hf(input_ids=prefix).logits[0, -1].float()
    noise = (noisy - truth).abs().max().item()
    if penalty != 1.0:  # the arg-max is taken over the penalised scores (pretrained_model.py:834)
        from transformers import RepetitionPenaltyLogitsProcessor
        truth = RepetitionPenaltyLogitsProcessor(penalty)(prefix, truth[None])[0]
    gap = max((truth.max() - truth[tok_a]).item(), (truth.max() - truth[tok_b]).item())
    return gap <= 4 * noise + 0.05, gap, noise


@pytest.mark.parametrize('family,penalty', [('llama', 1.0), ('mistral', 1.0), ('mistral', 1.1), ('mixtral', 1.0)])
def test_generate_matches_oracle(family, penalty):
    from oracle.loop import lookahead_generate
    from oracle.trie import OracleLookaheadCache
    from painlessinferenceacceleration_b200.common.lookahead_cache import LookaheadCache
    hf, ours = _pair(family, seed=2)
    ours.lookahead_cache = LookaheadCache(eos_ids=[2], device=DEV, vocab_capacity=1024, node_capacity=1 << 20)
    otrie = OracleLookaheadCache(eos_ids=[2])
    exact, total, edl_pairs, agree_tok, all_tok = 0, 0, [], 0, 0
    for rep in range(2):
        for p in prompts(21, 4, 24, 200):
            p = p.to(DEV)
            dk = {'use_lookahead': True, 'decoding_length': 64, 'branch_length': 8}
            out = ours.generate(input_ids=p, max_new_tokens=48, eos_token_id=2, repetition_penalty=penalty,
                                decoding_kwargs=dk, return_dict_in_generate=True)
            ref = lookahead_generate(hf, otrie, p, max_new_tokens=48, eos_token_id=[2], repetition_penalty=penalty)
            a, b = out.sequences[0].tolist(), ref['sequences'][0].tolist()
            total += 1
            all_tok += len(b) - p.shape[1]
            if a == b:
                exact += 1
                agree_tok += len(b) - p.shape[1]
                # identical tokens + parity-exact trie => identical drafts => identical accepted lengths
                assert out.kwargs['edls'] == ref['edls'], (out.kwargs['edls'], ref['edls'])
                assert out.kwargs['dls'] == ref['dls']
                edl_pairs.append(sum(ref['edls'][1:]) / max(len(ref['edls']) - 1, 1))
            else:
                k = next(i for i in range(min(len(a), len(b))) if a[i] != b[i])
                agree_tok += k - p.shape[1]
                ok, gap, noise = _legit_divergence(family, hf, ref['sequences'][:, :k], a[k], b[k], penalty)
                _diag('generate_matches_oracle', family=family, pos=k, gap=gap, noise=noise)
                assert ok, f'diverged at {k}: fp32 gap {gap:.3f} vs bf16 noise {noise:.3f}'
                # stated tolerance: both candidates within EPS of the fp32 optimum (logit std of these models ~1.3-1.8,
                # the eager bf16 model's own max logit error 0.07-0.3)
                assert gap < EPS, f'diverged at {k} although the fp32 top-2 margin is {gap:.3f} >= {EPS}'
                # the tries have diverged with the text: resync both from scratch
                ours.lookahead_cache.fresh()
                otrie.fresh()
    # random tiny models have near-tied logits every few dozen tokens, so most 48-token continuations contain at
    # least one bf16 near-tie; what must hold is that EVERY divergence sits on such a tie (asserted above) and
    # that equal text implies equal drafts (dls) and accepted lengths (edls).  The exact-loop-logic statement is
    # test_loop_is_exact_given_the_same_logits below.
    _diag('generate_matches_oracle_summary', family=family, penalty=penalty, exact=exact, total=total,
          agree_tok=agree_tok, all_tok=all_tok)
    # measured on these seeds (round 2): the fp32 top-2 margin of a random 2-layer model is below the eager bf16
    # model's own logit error at ~3-8 % of the positions, so a free-running 48-token continuation meets such a tie
    # more often than not; every divergence must sit on one (asserted above, EPS stated), a quarter of the sequences
    # and 40 % of the tokens must come before any tie
    assert 4 * exact >= total, f'only {exact}/{total} sequences identical'
    assert agree_tok >= 0.4 * all_tok, f'only {agree_tok}/{all_tok} tokens precede the first bf16 near-tie'


def test_lookahead_equals_own_greedy_and_respects_limits():
    """lossless property on our own kernels: drafts never change the output (up to bf16 near-ties), max_length
    is never overshot, eos stops the loop, and dls/edls/fts/qts are reported like the reference (README :217-233)"""
    from painlessinferenceacceleration_b200.common.lookahead_cache import LookaheadCache
    hf, ours = _pair('llama', seed=4)
    ours.lookahead_cache = LookaheadCache(eos_ids=[2], device=DEV, vocab_capacity=1024, node_capacity=1 << 20)
    same = 0
    ps = prompts(33, 6, 16, 200)
    for p in ps:
        p = p.to(DEV)
        g = ours.generate(input_ids=p, max_new_tokens=40, eos_token_id=2, decoding_kwargs={'use_lookahead': False})
        for _ in range(2):
            o = ours.generate(input_ids=p, max_new_tokens=40, eos_token_id=2,
                              decoding_kwargs={'use_lookahead': True, 'decoding_length': 64, 'branch_length': 8},
                              return_dict_in_generate=True)
        assert o.sequences.shape[1] <= 16 + 40
        assert sum(o.kwargs['edls']) == o.sequences.shape[1] - 16
        assert len(o.kwargs['fts']) == len(o.kwargs['edls'])
        same += int(o.sequences[0].tolist() == g[0].tolist())
        if o.sequences[0].tolist() == g[0].tolist():
            assert max(o.kwargs['edls']) > 1  # the second pass drafts the first pass's answer
    assert same >= len(ps) - 2


class OursBackend(object):
    """adapter for oracle.loop: the verify forward / KV cache of OUR model behind the oracle's backend interface, so
    that the oracle loop (reference semantics on the host) and our fused device loop consume the same logits"""

    def __init__(self, ours, prefill_like_generate=False, max_seq=512):
        self.m, self.P = ours, 0
        self.prefill_like_generate, self.max_seq = prefill_like_generate, max_seq

    def rows(self):
        return self.P

    def forward(self, ids_in, m01, pos):
        n = ids_in.shape[1]
        if self.P == 0 and self.prefill_like_generate:  # prompt: exactly the prefill generate() runs (last row only)
            rt = self.m._runtime(self.max_seq, 64)
            rt.set_request(0, 0, 1 << 30)
            rt.seq[0, :n] = ids_in[0].to(device=rt.device, dtype=torch.int32)
            self.m._prefill_logits(rt, n)
            self.P = n
            return rt.logits[0:1].clone()[None]
        if self.P == 0 and n > 64:  # prompt: chain chunks of 64 through forward()
            outs = []
            for c0 in range(0, n, 64):
                m = min(64, n - c0)
                lg, self.P = self.m.forward(ids_in[:, c0:c0 + m], m01[:, :, c0:c0 + m, :c0 + m], past_key_values=c0)
                outs.append(lg)
            return torch.cat(outs, dim=1)
        lg, self.P = self.m.forward(ids_in, m01, past_key_values=self.P)
        return lg

    def compact(self, keep_idx):
        rt = self.m._rt
        L = keep_idx.numel()
        rt.k_cache[0][:, :, :L] = rt.k_cache[0][:, :, keep_idx.to(rt.device)]
        rt.v_cache[0][:, :, :L] = rt.v_cache[0][:, :, keep_idx.to(rt.device)]
        self.P = L


@pytest.mark.parametrize('family,penalty', [('llama', 1.0), ('mistral', 1.1)])
def test_loop_is_exact_given_the_same_logits(family, penalty):
    """Loop logic parity, free of floating-point noise: the oracle loop (reference draft/accept/compaction semantics
    + C oracle trie, on the host) drives one copy of our model through the oracle's backend interface while our fused
    device loop (GPU trie, accept/compaction kernels, CUDA graph) drives another copy with the same weights.  The
    kernels are deterministic, so both see bit-identical logits and every request must agree exactly in tokens,
    drafts (dls) and accepted lengths (edls) - with the tries carried across requests."""
    from oracle.loop import lookahead_generate
    from oracle.trie import OracleLookaheadCache
    from painlessinferenceacceleration_b200.common.lookahead_cache import LookaheadCache
    from painlessinferenceacceleration_b200.models.llama.modeling_llama import LlamaForCausalLM
    hf, a = _pair(family, seed=6)
    b = LlamaForCausalLM(hf.config, device=torch.device(DEV))
    b.load_state_dict(hf.state_dict(), strict=False)
    a.lookahead_cache = LookaheadCache(eos_ids=[2], device=DEV, vocab_capacity=1024, node_capacity=1 << 20)
    otrie = OracleLookaheadCache(eos_ids=[2])
    edl_all = []
    for rep in range(2):
        for p in prompts(55, 4, 90, 200):
            p = p.to(DEV)
            out = a.generate(input_ids=p, max_new_tokens=56, eos_token_id=2, repetition_penalty=penalty,
                             decoding_kwargs={'use_lookahead': True, 'decoding_length': 64, 'branch_length': 8},
                             return_dict_in_generate=True)
            ref = lookahead_generate(None, otrie, p, max_new_tokens=56, eos_token_id=[2], repetition_penalty=penalty,
                                     backend=OursBackend(b, prefill_like_generate=True, max_seq=90 + 56 + 65))
            assert out.sequences[0].tolist() == ref['sequences'][0].tolist()
            assert out.kwargs['edls'] == ref['edls'] and out.kwargs['dls'] == ref['dls']
            edl_all += ref['edls'][1:]
    assert max(edl_all) > 2


@pytest.mark.parametrize('family', ['llama', 'mistral', 'mixtral'])
def test_verify_logits_within_tolerance(family):
    """"verify logits within a stated fp tolerance" (BASELINE north_star): our bf16 forward vs an fp32 evaluation of
    the same weights (the truth, SURVEY A.2-16), next to the reference-style bf16 eager forward's own error.
    Tolerance: max |logit error| <= 2 x the eager bf16 model's error (+0.02 absolute)."""
    hf, ours = _pair(family, seed=8)
    hf32 = tiny_hf_model(family, seed=8, dtype=torch.float32, device=DEV, vocab=200)
    hf32.load_state_dict({k: v.float() for k, v in hf.state_dict().items()})
    p = prompts(77, 1, 100, 200)[0].to(DEV)
    with torch.no_grad():
        truth = hf32(input_ids=p).logits[0].float()
        eager = hf(input_ids=p).logits[0].float()
    be = OursBackend(ours)
    m01 = torch.tril(torch.ones((1, 1, 100, 100), dtype=torch.long, device=DEV))
    got = be.forward(p, m01, None)[0].float()
    e_ours, e_eager = (got - truth).abs().max().item(), (eager - truth).abs().max().item()
    top = torch.topk(truth, 2, dim=-1).values
    margin = top[:, 0] - top[:, 1]
    _diag('verify_logits', family=family, e_ours=e_ours, e_eager=e_eager, rms_ours=(got - truth).pow(2).mean().sqrt().item(),
          rms_eager=(eager - truth).pow(2).mean().sqrt().item(), logit_std=truth.std().item(),
          median_margin=margin.median().item())
    assert e_ours <= 2 * e_eager + 0.02, (e_ours, e_eager)
    # greedy tokens agree wherever the fp32 margin exceeds twice the error
    sure = margin > 2 * e_ours
    assert torch.equal(got.argmax(-1)[sure], truth.argmax(-1)[sure])


def test_left_padding_eos_and_streamer():
    """2-D attention_mask with a left-padded prompt (pretrained_model.py:1123-1131), eos stopping (:1228-1231) and the
    streamer protocol (:1199-1201: the whole accepted list per step) against the oracle loop"""
    from oracle.loop import lookahead_generate
    from oracle.trie import OracleLookaheadCache
    from painlessinferenceacceleration_b200.common.lookahead_cache import LookaheadCache
    hf, ours = _pair('llama', seed=12)
    ours.lookahead_cache = LookaheadCache(eos_ids=[2], device=DEV, vocab_capacity=1024, node_capacity=1 << 20)
    otrie = OracleLookaheadCache(eos_ids=[2])
    p = prompts(91, 1, 70, 200)[0].to(DEV)
    pad = 5
    padded = torch.cat([torch.zeros((1, pad), dtype=torch.long, device=DEV), p], dim=1)
    am = torch.cat([torch.zeros((1, pad), dtype=torch.long, device=DEV), torch.ones_like(p)], dim=1)
    ref = lookahead_generate(hf, otrie, padded, max_new_tokens=24, eos_token_id=[2], attention_mask=am)
    eos = ref['sequences'][0, min(padded.shape[1] + 6, ref['sequences'].shape[1] - 1)].item()  # an early token as eos

    class Collect(object):
        def __init__(self):
            self.chunks, self.ended = [], False

        def put(self, x):
            self.chunks.append(x)

        def end(self):
            self.ended = True

    for rep in range(2):
        otrie2 = OracleLookaheadCache(eos_ids=[eos])
        ours.lookahead_cache.fresh()
        ref = lookahead_generate(hf, otrie2, padded, max_new_tokens=24, eos_token_id=[eos], attention_mask=am)
        st = Collect()
        out = ours.generate(input_ids=padded, attention_mask=am, max_new_tokens=24, eos_token_id=eos, streamer=st,
                            decoding_kwargs={'use_lookahead': True, 'decoding_length': 64, 'branch_length': 8},
                            return_dict_in_generate=True)
        a, b = out.sequences[0].tolist(), ref['sequences'][0].tolist()
        if a != b:
            k = next(i for i in range(min(len(a), len(b))) if a[i] != b[i])
            # the pad columns are invisible and positions are mask row sums, so the unpadded prefix is equivalent
            ok, gap, noise = _legit_divergence('llama', hf, ref['sequences'][:, pad:k], a[k], b[k])
            assert ok, f'diverged at {k}: gap {gap:.3f} noise {noise:.3f}'
        else:
            assert a[-1] == eos and len(a) < padded.shape[1] + 24
        assert st.ended
        streamed = [int(t) for c in st.chunks[1:] for t in (c.reshape(-1).tolist())]
        assert streamed == a[padded.shape[1]:]


# ---------------------------------------------------------------------------------------------------------------
# Parity at the BASELINE shapes (BASELINE.json configs 2-4): the same exact-loop statement as above, at full size.
# Random-init weights of the named shapes (no checkpoints offline), phrase-bank prompts of bench.py; every request
# runs twice so that the second pass drafts the first pass's answer from the trie (multi-token accepts, non-contiguous
# KV compaction at the real head counts / cache strides / vocabulary).
# ---------------------------------------------------------------------------------------------------------------
def _shape_model(name, layers=None):
    import bench
    from painlessinferenceacceleration_b200.models.llama.modeling_llama import LlamaForCausalLM
    from painlessinferenceacceleration_b200.models.mixtral.modeling_mixtral import MixtralForCausalLM
    cfg, fam = bench.make_config(name)
    if layers is not None:
        cfg.num_hidden_layers = layers
    cls = MixtralForCausalLM if fam == 'mixtral' else LlamaForCausalLM
    a = cls(cfg, device=torch.device(DEV)).init_weights(seed=0)
    b = cls(cfg, device=torch.device(DEV))
    b.load_state_dict(a.state_dict(), strict=True)
    return cfg, a, b


@pytest.mark.big
@pytest.mark.parametrize('name,layers,penalty,n_prompts,new', [('llama2-7b', None, 1.0, 4, 128),
                                                               ('mistral-7b', None, 1.1, 3, 96),
                                                               ('mixtral-8x7b-16l', 3, 1.0, 3, 64)])
def test_loop_is_exact_at_baseline_shapes(name, layers, penalty, n_prompts, new):
    """Llama-2-7B (32 layers, 4096, MHA-32, V=32000; config 2), Mistral-7B (GQA-4) with repetition_penalty=1.1
    (config 3) and an 8-expert Mixtral-8x7B-shaped slice (3 of the 32 layers; config 4): the oracle loop (reference
    semantics + C oracle trie on the host) drives one copy of the model through the backend interface, the fused device
    loop drives the other; 64-token / 8-branch drafts, 256-token phrase-bank prompts.  Tokens, dls and edls must be
    identical for every request, with the tries carried across requests."""
    import bench
    from oracle.loop import lookahead_generate
    from oracle.trie import OracleLookaheadCache
    from painlessinferenceacceleration_b200.common.lookahead_cache import LookaheadCache
    cfg, a, b = _shape_model(name, layers)
    a.lookahead_cache = LookaheadCache(eos_ids=[2], device=DEV, vocab_capacity=cfg.vocab_size)
    otrie = OracleLookaheadCache(eos_ids=[2])
    ps = bench.phrase_bank_prompts(n_prompts, cfg.vocab_size)
    edl_all, moved = [], 0
    for rep in range(2):
        for p in ps:
            p = torch.tensor([p], device=DEV)
            out = a.generate(input_ids=p, max_new_tokens=new, eos_token_id=2, repetition_penalty=penalty,
                             decoding_kwargs={'use_lookahead': True, 'decoding_length': 64, 'branch_length': 8},
                             return_dict_in_generate=True)
            ref = lookahead_generate(None, otrie, p, max_new_tokens=new, eos_token_id=[2], repetition_penalty=penalty,
                                     backend=OursBackend(b, prefill_like_generate=True, max_seq=256 + new + 65),
                                     trace=True)
            assert out.sequences[0].tolist() == ref['sequences'][0].tolist(), (name, rep)
            assert out.kwargs['edls'] == ref['edls'] and out.kwargs['dls'] == ref['dls'], (name, rep)
            if rep == 1:
                edl_all += ref['edls'][1:]
                moved += sum(1 for st in ref['steps'] if len(st['tokens']) > 1 and
                             st['logit_indices'] != list(range(len(st['tokens']))))
    _diag('baseline_shape_parity', model=name, mean_edl_second_pass=sum(edl_all) / len(edl_all), max_edl=max(edl_all),
          non_contiguous_steps=moved)
    assert max(edl_all) > 2, 'the second pass never accepted a draft: the test did not exercise the accept path'


def test_caller_supplied_logits_processor_and_stopping_criteria():
    """generate(logits_processor=..., stopping_criteria=...) (reference :349-360, :786, :834, :1225): the processors
    run on the host path of the loop.  An explicit RepetitionPenaltyLogitsProcessor must reproduce the built-in
    repetition_penalty run token for token (same kernels, same logits; dls / edls too), and a custom criterion stops the
    request at the step where it first fires."""
    from transformers import RepetitionPenaltyLogitsProcessor, StoppingCriteria
    from painlessinferenceacceleration_b200.common.lookahead_cache import LookaheadCache
    hf, ours = _pair('mistral', seed=14)
    ps = [p.to(DEV) for p in prompts(93, 2, 40, 200)]
    dk = {'use_lookahead': True, 'decoding_length': 64, 'branch_length': 8}
    runs = {}
    for mode in ('builtin', 'processor'):
        ours.lookahead_cache = LookaheadCache(eos_ids=[2], device=DEV, vocab_capacity=1024, node_capacity=1 << 20)
        outs = []
        for rep in range(2):
            for p in ps:
                kw = dict(repetition_penalty=1.1) if mode == 'builtin' else \
                    dict(logits_processor=[RepetitionPenaltyLogitsProcessor(1.1)])
                o = ours.generate(input_ids=p, max_new_tokens=40, eos_token_id=2, decoding_kwargs=dict(dk),
                                  return_dict_in_generate=True, **kw)
                outs.append((o.sequences[0].tolist(), o.kwargs['dls'], o.kwargs['edls']))
        runs[mode] = outs
    assert runs['builtin'] == runs['processor']
    assert max(e for _, _, ed in runs['processor'] for e in ed) > 1

    class StopOnToken(StoppingCriteria):
        def __init__(self, tok):
            self.tok = tok

        def __call__(self, input_ids, scores, **kw):
            return torch.tensor([bool((input_ids[0, 40:] == self.tok).any())])

    full = runs['builtin'][0][0]
    tok = full[40 + 9]
    ours.lookahead_cache = LookaheadCache(eos_ids=[2], device=DEV, vocab_capacity=1024, node_capacity=1 << 20)
    o = ours.generate(input_ids=ps[0], max_new_tokens=40, eos_token_id=2, repetition_penalty=1.1,
                      stopping_criteria=[StopOnToken(tok)], decoding_kwargs=dict(dk), return_dict_in_generate=True)
    got = o.sequences[0].tolist()
    assert got == full[:len(got)] and tok in got[40:] and len(got) < len(full)
    first = 40 + full[40:].index(tok)
    assert len(got) > first and sum(o.kwargs['edls']) == len(got) - 40


# ---------------------------------------------------------------------------------------------------------------
# GPT-2 patch surface on the GPU (reference models/gpt2/modeling_gpt2.py:805-809, 183-221; BASELINE config 1's family)
# ---------------------------------------------------------------------------------------------------------------
def _gpt2_pair(seed):
    from painlessinferenceacceleration_b200.models.gpt2.modeling_gpt2 import GPT2LMHeadModel
    hf = tiny_hf_model('gpt2', seed=seed, dtype=torch.bfloat16, device=DEV, vocab=200)
    ours = GPT2LMHeadModel(hf.config, device=torch.device(DEV))
    missing = ours.load_state_dict(hf.state_dict(), strict=False)
    assert not missing.missing_keys, missing
    return hf, ours


def test_gpt2_verify_logits_and_loop():
    """GPT-2 (64-wide or narrower heads, learned positions, LayerNorm, gelu_new, Conv1D + bias, tied head) through the
    shared kernels: heads zero-padded to the 128-wide attention tile.  (i) logits vs an fp32 evaluation of the
    same weights within 2 x the eager bf16 model's own error + 0.02; (ii) the oracle loop (reference semantics, 16-token
    / 4-branch drafts = BASELINE config 1) driving one copy == our fused device loop on the other copy: tokens, dls,
    edls identical; (iii) lookahead == plain greedy on the same kernels."""
    from oracle.loop import lookahead_generate
    from oracle.trie import OracleLookaheadCache
    from painlessinferenceacceleration_b200.common.lookahead_cache import LookaheadCache
    from painlessinferenceacceleration_b200.models.gpt2.modeling_gpt2 import GPT2LMHeadModel
    hf, ours = _gpt2_pair(seed=16)
    hf32 = tiny_hf_model('gpt2', seed=16, dtype=torch.float32, device=DEV, vocab=200)
    hf32.load_state_dict({k: v.float() for k, v in hf.state_dict().items()})
    p = prompts(78, 1, 100, 200)[0].to(DEV)
    with torch.no_grad():
        truth = hf32(input_ids=p).logits[0].float()
        eager = hf(input_ids=p).logits[0].float()
    m01 = torch.tril(torch.ones((1, 1, 100, 100), dtype=torch.long, device=DEV))
    got = OursBackend(ours).forward(p, m01, None)[0].float()
    e_ours, e_eager = (got - truth).abs().max().item(), (eager - truth).abs().max().item()
    _diag('verify_logits', family='gpt2', e_ours=e_ours, e_eager=e_eager)
    assert e_ours <= 2 * e_eager + 0.02, (e_ours, e_eager)
    b = GPT2LMHeadModel(hf.config, device=torch.device(DEV))
    b.load_state_dict(hf.state_dict(), strict=False)
    ours.lookahead_cache = LookaheadCache(eos_ids=[2], device=DEV, vocab_capacity=1024, node_capacity=1 << 20)
    otrie = OracleLookaheadCache(eos_ids=[2])
    edl_all, same = [], 0
    for rep in range(2):
        for q in prompts(56, 3, 70, 200):
            q = q.to(DEV)
            dk = {'use_lookahead': True, 'decoding_length': 16, 'branch_length': 4}
            out = ours.generate(input_ids=q, max_new_tokens=48, eos_token_id=2, decoding_kwargs=dk,
                                return_dict_in_generate=True)
            ref = lookahead_generate(None, otrie, q, max_new_tokens=48, eos_token_id=[2], decoding_length=16,
                                     branch_length=4, backend=OursBackend(b, prefill_like_generate=True, max_seq=70 + 48 + 17))
            assert out.sequences[0].tolist() == ref['sequences'][0].tolist()
            assert out.kwargs['edls'] == ref['edls'] and out.kwargs['dls'] == ref['dls']
            edl_all += ref['edls'][1:]
            plain = ours.generate(input_ids=q, max_new_tokens=48, eos_token_id=2, decoding_kwargs={'use_lookahead': False})
            same += int(plain[0].tolist() == out.sequences[0].tolist())
    assert max(edl_all) > 2
    assert same >= 4   # a draft of 1 vs 16 nodes changes the KV split count, i.e. the fp32 summation order (bf16 near-ties)


@pytest.mark.parametrize('family', ['mistral', 'mixtral'])
def test_sliding_window_checkpoints_warn_instead_of_diverging_silently(family):
    """the reference's lookahead branch ignores the window (mistral/modeling_mistral.py:979-982), so does the kernel:
    a config that sets one gets a warning as soon as a context can outgrow it, and the same tokens as without it"""
    from painlessinferenceacceleration_b200.models.mistral.modeling_mistral import MistralForCausalLM
    from painlessinferenceacceleration_b200.models.mixtral.modeling_mixtral import MixtralForCausalLM
    hf = tiny_hf_model(family, seed=3, dtype=torch.bfloat16, device=DEV, vocab=200)
    cls = MixtralForCausalLM if family == 'mixtral' else MistralForCausalLM
    outs = []
    for window in (None, 16):
        cfg = tiny_config(family, vocab=200, sliding_window=window)
        ours = cls(cfg, device=torch.device(DEV))
        assert not ours.load_state_dict(hf.state_dict(), strict=False).missing_keys
        ids = prompts(5, 1, 24, 200)[0].to(DEV)
        kw = dict(input_ids=ids, max_new_tokens=12, eos_token_id=2,
                  decoding_kwargs={'use_lookahead': True, 'decoding_length': 64, 'branch_length': 8})
        if window is None:
            outs.append(ours.generate(**kw))
        else:
            with pytest.warns(UserWarning, match='sliding_window=16 is ignored'):
                outs.append(ours.generate(**kw))
    assert torch.equal(outs[0], outs[1])
