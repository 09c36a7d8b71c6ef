# -*- coding: utf-8 -*-
"""Tests of k_rmsnorm, k_silu_mul and k_embed_gather (csrc/fused_ops.cu) that can fail: RMSNorm in each family's own
rounding against an fp64 reference whose comparator tolerates only real ties (tests/norm_ref.py), the residual sum and
the split-K slice sum bit for bit, the in-place residual update at every width up to 16384, the families' own norm
modules, the rounding every model passes on every norm call, and SiLU*up over every bf16 gate value.

The first half runs without a GPU: the comparators accept an emulation of the kernels' fp32 arithmetic and reject every
wrong kernel of norm_ref's mutation lists on the inputs the GPU half uses, those inputs make the two rounding modes
differ, and every model class carries its family's rounding."""
import pytest
import torch

from tests import norm_ref as R

DEV = 'cuda:0'
HIDDEN = (8, 256, 896, 1536, 2048, 3584, 4096, 5120, 6144, 8192, 8200, 12288, 16384)
ROWS = (1, 5, 64, 320)
EPS = (1e-5, 1e-6, 1.5625e-7)
RESIDUAL = ('none', 'separate', 'inplace', 'in_only')
SENT = 0x7FA5               # a NaN bit pattern no kernel writes
MAX_AMBIGUOUS = 0.005       # share of elements the comparator may leave open, over all rows of a test
MAX_AMBIGUOUS_CASE = 0.05   # ... and in any one call (a few rows: the ties come in clumps, see norm_ref.rms_check)


class Ambiguity(object):
    """the comparator's ambiguous elements, counted per call and over a whole test"""

    def __init__(self):
        self.n_amb, self.n = 0, 0

    def add(self, n_amb, n, small=False):
        assert small or n_amb <= MAX_AMBIGUOUS_CASE * n, (n_amb, n)
        self.n_amb += n_amb
        self.n += n

    def check(self):
        assert self.n > 0 and self.n_amb <= MAX_AMBIGUOUS * self.n, (self.n_amb, self.n)


def _bits(t):
    return t.view(torch.int16)


def _sentinel(shape, device):
    return torch.full(shape, SENT, dtype=torch.int16, device=device).view(torch.bfloat16)


def norm_inputs(rows, hidden, seed, weights='normal', device='cpu'):
    """(x, r, w) bf16: x, r ~ N(0, 1) with a few outlier channels x 64; with rows >= 3, row 1 is all zero (x and r) and
    row 2 is dominated by eps (|x| ~ 1e-4, r = 0).  weights: 'normal' N(1, 0.3) with some zero and negative entries,
    'spread' |w| in [1e-3, 20] log-uniform with random signs"""
    g = torch.Generator().manual_seed(seed)
    x = torch.randn((rows, hidden), generator=g)
    r = torch.randn((rows, hidden), generator=g)
    out = torch.randint(0, hidden, (max(1, hidden // 512),), generator=g)
    x[:, out] *= 64
    if rows >= 3:
        x[1], r[1] = 0, 0
        x[2], r[2] = x[2] * 1e-4, 0
    if weights == 'normal':
        w = 1 + 0.3 * torch.randn((hidden,), generator=g)
        w[torch.randint(0, hidden, (max(1, hidden // 64),), generator=g)] = 0
        w[torch.randint(0, hidden, (max(1, hidden // 16),), generator=g)] *= -1
    else:
        w = torch.exp(torch.empty((hidden,)).uniform_(-6.9, 3.0, generator=g))
        w = w * (torch.randint(0, 2, (hidden,), generator=g) * 2 - 1)
    bf = torch.bfloat16
    return x.to(bf).to(device), r.to(bf).to(device), w.to(bf).to(device)


def part_inputs(n_parts, rows, hidden, seed, device='cpu'):
    """fp32 split-K slices [n_parts, 64, hidden] of very different magnitudes (1, 1e3, 1e-2, 3e2, ...) so that the
    summation order shows in the rounded sum"""
    g = torch.Generator().manual_seed(seed)
    scale = torch.tensor([1.0, 1e3, 1e-2, 3e2, 7.0, 1e-3, 50.0, 2e3])[:n_parts]
    parts = torch.randn((n_parts, 64, hidden), generator=g) * scale[:, None, None]
    if n_parts > 2:   # cancellation of the big slice: the order of the terms decides the low bits
        parts[-1, :, ::3] = -parts[1, :, ::3]
    return parts.to(device)


# ---------------------------------------------------------------------------------------------------------------
# the CPU half
# ---------------------------------------------------------------------------------------------------------------
CPU_CASES = [(5, 896, 1e-6, 'normal'), (5, 4096, 1e-5, 'spread'), (3, 12288, 1.5625e-7, 'normal'),
             (3, 16384, 1e-6, 'spread'), (5, 8, 1e-5, 'normal'), (5, 8200, 1e-6, 'normal')]


def _cpu_rms_cases():
    for i, (rows, hidden, eps, wk) in enumerate(CPU_CASES):
        x, r, w = norm_inputs(rows, hidden, seed=100 + i, weights=wk)
        yield dict(rows=rows, hidden=hidden, eps=eps, x=x, r=r, w=w, parts=None)
    for i, n in enumerate((1, 2, 4, 7, 8)):
        parts = part_inputs(n, 5, 4096, seed=200 + i)
        _, r, w = norm_inputs(5, 4096, seed=300 + i)
        yield dict(rows=5, hidden=4096, eps=1e-6, x=None, r=r, w=w, parts=parts[:, :5])


def _rejects(c, rounding, mut, amb=None):
    """whether the checks reject the emulation under mutation `mut` (None: the emulated kernel itself)"""
    ro, y = R.emulate_rmsnorm(c['x'], c['w'], c['eps'], rounding, r=c['r'], parts=c['parts'], mut=mut)
    s, xh = R.rmsnorm_ref(c['x'], c['w'], c['eps'], r=c['r'], parts=c['parts'])
    bad, n_amb = R.rms_check(y, xh, c['w'], rounding, c['hidden'])
    if amb is not None:
        amb.add(n_amb, y.numel(), small=c['hidden'] < 256)
    return bad > 0 or not torch.equal(_bits(ro), _bits(s))


def test_rms_mutation_list_is_complete():
    assert set(R.RMS_MUTATIONS) == {'other_rounding', 'residual_unrounded', 'no_eps', 'eps_after_sqrt',
                                    'mean_over_hidden_minus_1', 'slices_reversed', 'inplace_reread'}
    assert set(R.SILU_MUTATIONS) == {'silu_unrounded', 'gate_up_swapped'}


@pytest.mark.parametrize('rounding', [R.ONCE, R.TWICE])
def test_rms_comparator_accepts_the_kernel_and_rejects_every_mutation(rounding):
    cases = list(_cpu_rms_cases())
    amb = Ambiguity()
    for c in cases:
        assert not _rejects(c, rounding, None, amb), (c['hidden'], c['parts'] is not None)
    amb.check()
    for mut in R.RMS_MUTATIONS:
        assert any(_rejects(c, rounding, mut) for c in cases), mut


def test_inputs_make_the_two_roundings_differ():
    """on the test inputs bf16(w * x_hat) and bf16(w * bf16(x_hat)) differ on > 10 % of the elements, so a test of
    either mode tells them apart"""
    for i, (rows, hidden, eps, wk) in enumerate(CPU_CASES):
        if hidden < 256:
            continue
        x, r, w = norm_inputs(rows, hidden, seed=100 + i, weights=wk)
        _, xh = R.rmsnorm_ref(x, w, eps, r=r)
        once = R.bf16_rne(w.double() * xh)
        twice = R.bf16_rne(w.double() * R.bf16_rne(xh))
        live = xh[0] != 0
        assert (once[0][live] != twice[0][live]).double().mean().item() > 0.10, (hidden, wk)


def _silu_all_gates(u_kind):
    g = torch.arange(-32768, 32768, dtype=torch.int32).to(torch.int16).view(torch.bfloat16)
    if u_kind == 'plus':
        u = torch.ones_like(g)
    elif u_kind == 'minus':
        u = -torch.ones_like(g)
    else:
        u = torch.randn(g.shape, generator=torch.Generator().manual_seed(9)).to(torch.bfloat16)
    return g, u


@pytest.mark.parametrize('u_kind', ['plus', 'minus', 'random'])
def test_silu_comparator_accepts_the_kernel(u_kind):
    g, u = _silu_all_gates(u_kind)
    bad, n_amb = R.silu_check(R.emulate_silu(torch.cat([g, u])[None])[0], g, u)
    assert bad == 0 and n_amb <= MAX_AMBIGUOUS * g.numel(), (bad, n_amb)


def test_silu_comparator_rejects_every_mutation():
    """with up = +-1 an unrounded SiLU output is invisible (one rounding either way); the random up row shows it"""
    for mut in R.SILU_MUTATIONS:
        hits = []
        for u_kind in ('plus', 'minus', 'random'):
            g, u = _silu_all_gates(u_kind)
            hits.append(R.silu_check(R.emulate_silu(torch.cat([g, u])[None], mut=mut)[0], g, u)[0] > 0)
        assert any(hits), mut


def _family_classes():
    """(class, expected rounding) for every RMSNorm model class"""
    from painlessinferenceacceleration_b200.models.baichuan2_13b.modeling_baichuan import BaichuanForCausalLM as B2_13
    from painlessinferenceacceleration_b200.models.baichuan2_7b.modeling_baichuan import BaichuanForCausalLM as B2_7
    from painlessinferenceacceleration_b200.models.baichuan2_7b.modeling_baichuan_batch import \
        BaichuanForCausalLM as B2_7_batch
    from painlessinferenceacceleration_b200.models.baichuan_13b.modeling_baichuan import BaichuanForCausalLM as B13
    from painlessinferenceacceleration_b200.models.baichuan_7b.modeling_baichuan import BaiChuanForCausalLM as B7
    from painlessinferenceacceleration_b200.models.chatglm.modeling_chatglm import ChatGLMForConditionalGeneration
    from painlessinferenceacceleration_b200.models.chatglm3 import modeling_chatglm as chatglm3
    from painlessinferenceacceleration_b200.models.glm4.modeling_glm4 import Glm4ForCausalLM, GlmForCausalLM
    from painlessinferenceacceleration_b200.models.llama.modeling_llama import LlamaForCausalLM
    from painlessinferenceacceleration_b200.models.llama.modeling_llama_batch import LlamaForCausalLM as LlamaBatch
    from painlessinferenceacceleration_b200.models.mistral.modeling_mistral import MistralForCausalLM
    from painlessinferenceacceleration_b200.models.mixtral.modeling_mixtral import MixtralForCausalLM
    from painlessinferenceacceleration_b200.models.qwen2.modeling_qwen2 import Qwen2ForCausalLM
    out = [(LlamaForCausalLM, R.ONCE), (LlamaBatch, R.ONCE), (ChatGLMForConditionalGeneration, R.ONCE),
           (MistralForCausalLM, R.TWICE), (MixtralForCausalLM, R.TWICE), (Qwen2ForCausalLM, R.TWICE),
           (B7, R.TWICE), (B13, R.TWICE), (B2_7, R.TWICE), (B2_13, R.TWICE), (B2_7_batch, R.TWICE),
           (GlmForCausalLM, R.TWICE), (Glm4ForCausalLM, R.TWICE)]
    for name in dir(chatglm3):
        cls = getattr(chatglm3, name)
        if isinstance(cls, type) and issubclass(cls, LlamaForCausalLM):
            out.append((cls, R.ONCE))
    return out


def test_every_model_class_carries_its_familys_rounding():
    from painlessinferenceacceleration_b200.common import ops
    assert (ops.ROUND_ONCE, ops.ROUND_TWICE) == (R.ONCE, R.TWICE)
    for cls, want in _family_classes():
        assert cls.rmsnorm_rounding == want, cls


# ---------------------------------------------------------------------------------------------------------------
# the GPU half
# ---------------------------------------------------------------------------------------------------------------
def _ops():
    from painlessinferenceacceleration_b200.common import ops
    return ops


def _run_rmsnorm(x, r, w, eps, mode, rounding):
    """one pia_rmsnorm call in residual mode `mode` -> (residual buffer after the call or None, y); y and the residual
    output carry a sentinel row after `rows` that must stay untouched"""
    ops = _ops()
    rows, hidden = x.shape
    y = _sentinel((rows + 1, hidden), x.device)
    if mode == 'none':
        ro = _sentinel((rows + 1, hidden), x.device)
        ops.rmsnorm(x, None, w, eps, ro[:rows], y[:rows], rounding=rounding)
    elif mode == 'separate':
        ro = _sentinel((rows + 1, hidden), x.device)
        r_in = r.clone()
        ops.rmsnorm(x, r_in, w, eps, ro[:rows], y[:rows], rounding=rounding)
        assert torch.equal(_bits(r_in), _bits(r))
    elif mode == 'inplace':
        ro = torch.cat([r, _sentinel((1, hidden), x.device)])
        ops.rmsnorm(x, ro[:rows], w, eps, ro[:rows], y[:rows], rounding=rounding)
    else:
        ro = None
        ops.rmsnorm(x, r, w, eps, None, y[:rows], rounding=rounding)
    torch.cuda.synchronize()
    assert (_bits(y[rows]) == SENT).all()
    if ro is not None:
        assert (_bits(ro[rows]) == SENT).all()
        ro = ro[:rows]
    return ro, y[:rows]


@pytest.mark.gpu
@pytest.mark.parametrize('rounding', [R.ONCE, R.TWICE], ids=['once', 'twice'])
@pytest.mark.parametrize('hidden', HIDDEN)
def test_rmsnorm_against_fp64(hidden, rounding):
    """every row count and residual mode; eps and the weight kind vary with the row count.  residual_out is bit exact,
    y is the fp64 reference up to real ties, the zero row is exactly 0"""
    amb = Ambiguity()
    for ri, rows in enumerate(ROWS):
        eps = EPS[(ri + hidden) % len(EPS)]
        x, r, w = norm_inputs(rows, hidden, seed=hidden * 7 + ri, weights=('normal', 'spread')[ri % 2], device=DEV)
        for mode in RESIDUAL:
            ro, y = _run_rmsnorm(x, r, w, eps, mode, rounding)
            res = r if mode != 'none' else None
            s, xh = R.rmsnorm_ref(x, w, eps, r=res)
            if ro is not None:
                assert torch.equal(_bits(ro), _bits(s)), (rows, mode)
            bad, n_amb = R.rms_check(y, xh, w, rounding, hidden)
            assert bad == 0, (rows, mode, eps, bad)
            amb.add(n_amb, y.numel(), small=hidden < 256)
            if rows >= 3:
                assert float(y[1].float().abs().max()) == 0.0
    amb.check()


@pytest.mark.gpu
@pytest.mark.parametrize('n_parts', [1, 2, 4, 7, 8])
@pytest.mark.parametrize('rows', [5, 64])
@pytest.mark.parametrize('hidden', [4096, 12288])
def test_rmsnorm_partials_against_fp64(hidden, rows, n_parts):
    """residual_out = bf16(bf16(((p0 + p1) + p2) + ...) + r) bit for bit, in place; rows past `rows` untouched"""
    ops = _ops()
    parts = part_inputs(n_parts, rows, hidden, seed=n_parts * 31 + rows, device=DEV)
    _, r, w = norm_inputs(64, hidden, seed=n_parts + rows, device=DEV)
    amb = Ambiguity()
    for rounding in (R.ONCE, R.TWICE):
        for mode in ('inplace', 'none'):
            y = _sentinel((64, hidden), DEV)
            if mode == 'inplace':
                resid = r.clone()
                resid[rows:] = _sentinel((64 - rows, hidden), DEV)
                ops.rmsnorm_partials(parts, resid, w, 1e-6, resid, y[:rows], rounding=rounding)
            else:
                resid = None
                ops.rmsnorm_partials(parts, None, w, 1e-6, None, y[:rows], rounding=rounding)
            torch.cuda.synchronize()
            p = parts[:, :rows]
            s, xh = R.rmsnorm_ref(None, w, 1e-6, r=r[:rows] if resid is not None else None, parts=p)
            if resid is not None:
                assert torch.equal(_bits(resid[:rows]), _bits(s))
                assert (_bits(resid[rows:]) == SENT).all()
            assert (_bits(y[rows:]) == SENT).all()
            bad, n_amb = R.rms_check(y[:rows], xh, w, rounding, hidden)
            assert bad == 0, (rounding, mode, bad)
            amb.add(n_amb, y[:rows].numel())
    amb.check()
    if n_parts > 2:   # the inputs make the order observable (two slices commute)
        flipped = R.slice_sum(parts[:, :rows].flip(0))
        assert not torch.equal(_bits(flipped), _bits(R.slice_sum(parts[:, :rows])))


def _hf_norm(cls_path, hidden, w, eps):
    mod, name = cls_path.rsplit('.', 1)
    import importlib
    cls = getattr(importlib.import_module(mod), name)
    m = cls(hidden, eps=eps).to(device=DEV, dtype=torch.bfloat16)
    with torch.no_grad():
        m.weight.copy_(w)
    return m


def _restated(kind, x, w, eps):
    """the lookahead reference modules' formulas in eager bf16 torch (the reference tree itself is not available here)"""
    variance = x.to(torch.float32).pow(2).mean(-1, keepdim=True)
    h = x * torch.rsqrt(variance + eps)                 # bf16 * fp32 -> fp32
    if kind in ('llama', 'chatglm'):                    # llama/modeling_llama.py:90, chatglm/modeling_chatglm.py:187
        return (w * h).to(x.dtype)
    return w * h.to(w.dtype)                            # baichuan_7b/modeling_baichuan.py:84-91 (and its siblings)


MODULES = [('transformers.models.mistral.modeling_mistral.MistralRMSNorm', R.TWICE),
           ('transformers.models.mixtral.modeling_mixtral.MixtralRMSNorm', R.TWICE),
           ('transformers.models.qwen2.modeling_qwen2.Qwen2RMSNorm', R.TWICE),
           ('transformers.models.glm.modeling_glm.GlmRMSNorm', R.TWICE),
           ('transformers.models.glm4.modeling_glm4.Glm4RMSNorm', R.TWICE),
           ('llama', R.ONCE), ('chatglm', R.ONCE), ('baichuan', R.TWICE)]


@pytest.mark.gpu
@pytest.mark.parametrize('module,rounding', MODULES, ids=[m[0].rsplit('.', 1)[-1] for m in MODULES])
def test_rmsnorm_matches_the_familys_own_module(module, rounding):
    """with non-unit weights the kernel in the family's mode equals the family's norm run eagerly in bf16 on this GPU,
    except where the fp64 comparator reports a tie; the other mode differs from it on > 10 % of the elements"""
    ops = _ops()
    n_amb = n = 0
    for hidden, eps in ((896, 1e-6), (4096, 1e-5), (5120, 1.5625e-7)):
        x, _, w = norm_inputs(64, hidden, seed=hidden, device=DEV)
        with torch.no_grad():
            want = _hf_norm(module, hidden, w, eps)(x) if '.' in module else _restated(module, x, w, eps)
        assert want.dtype == torch.bfloat16
        y, y_other = torch.empty_like(x), torch.empty_like(x)
        ops.rmsnorm(x, None, w, eps, None, y, rounding=rounding)
        ops.rmsnorm(x, None, w, eps, None, y_other, rounding=1 - rounding)
        torch.cuda.synchronize()
        _, xh = R.rmsnorm_ref(x, w, eps)
        _, _, amb = R.rms_accept(xh, w, rounding, hidden)
        differ = y != want
        assert not (differ & ~amb).any(), (hidden, int((differ & ~amb).sum()))
        n_amb, n = n_amb + int(amb.sum()), n + amb.numel()
        live = x != 0
        assert (y_other != want)[live].double().mean().item() > 0.10
    assert n_amb <= MAX_AMBIGUOUS * n, (n_amb, n)


def _tiny(family):
    """(our model with non-unit norm weights, expected rounding)"""
    dev = torch.device(DEV)
    if family in ('llama', 'mistral', 'mixtral'):
        from tests.tiny_models import tiny_config
        from painlessinferenceacceleration_b200.models.llama.modeling_llama import LlamaForCausalLM
        from painlessinferenceacceleration_b200.models.mistral.modeling_mistral import MistralForCausalLM
        from painlessinferenceacceleration_b200.models.mixtral.modeling_mixtral import MixtralForCausalLM
        cls = dict(llama=LlamaForCausalLM, mistral=MistralForCausalLM, mixtral=MixtralForCausalLM)[family]
        m = cls(tiny_config(family, vocab=200), device=dev)
    elif family == 'qwen2':
        from tests.tiny_qwen2 import qwen2_config
        from painlessinferenceacceleration_b200.models.qwen2.modeling_qwen2 import Qwen2ForCausalLM
        m = Qwen2ForCausalLM(qwen2_config(vocab=200), device=dev)
    elif family == 'baichuan':
        from tests.tiny_baichuan import tiny_model
        return tiny_model('7b'), R.TWICE
    else:
        from tests.tiny_glm import glm_config, glm_model_class
        if family == 'chatglm':
            from painlessinferenceacceleration_b200.models.chatglm.modeling_chatglm import \
                ChatGLMForConditionalGeneration as cls
        else:
            cls = glm_model_class(family)
        m = cls(glm_config('glm4' if family == 'glm4' else 'glm', hd=64, vocab=200), device=dev)
    m.init_weights(seed=3, std=0.08)
    want = R.ONCE if family in ('llama', 'chatglm') else R.TWICE
    return m, want


FAMILIES = ('llama', 'mistral', 'mixtral', 'qwen2', 'baichuan', 'glm', 'glm4', 'chatglm')


@pytest.mark.gpu
@pytest.mark.parametrize('split', [False, True], ids=['bf16', 'split_k_slices'])
@pytest.mark.parametrize('family', FAMILIES)
def test_every_norm_call_carries_the_familys_rounding(family, split, monkeypatch):
    """the ops.rmsnorm / ops.rmsnorm_partials calls of a prompt forward and a verify forward: input, post-attention,
    glm4's sandwich and the final norms, all in the family's mode; split: the o / down projections return fp32 split-K
    slices, which the norms then read"""
    ops = _ops()
    if split:
        monkeypatch.setenv('PIA_GEMM_SET', 'gate_up,o,down')
        monkeypatch.setenv('PIA_GEMM_SPLIT', '2')
    m, want = _tiny(family)
    calls = []

    def spy(name, fn):
        def wrapped(*a, **kw):
            calls.append((name, kw.get('rounding', ops.ROUND_ONCE)))
            return fn(*a, **kw)
        monkeypatch.setattr(ops, name, wrapped)

    spy('rmsnorm', ops.rmsnorm)
    spy('rmsnorm_partials', ops.rmsnorm_partials)
    g = torch.Generator().manual_seed(5)
    p = torch.randint(3, 200, (1, 16), generator=g).to(DEV)
    m01 = torch.tril(torch.ones((1, 1, 16, 16), dtype=torch.long, device=DEV))
    _, P = m.forward(p, m01, past_key_values=0)
    d = torch.randint(3, 200, (1, 8), generator=g).to(DEV)
    m01 = torch.cat([torch.ones((1, 1, 8, P), dtype=torch.long, device=DEV),
                     torch.tril(torch.ones((1, 1, 8, 8), dtype=torch.long, device=DEV))], -1)
    m.forward(d, m01, past_key_values=P)
    torch.cuda.synchronize()
    L = m.config.num_hidden_layers
    per_forward = 2 * L + 1 + (2 * L if m.sandwich_norms else 0)
    assert len(calls) == 2 * per_forward, calls
    assert all(rnd == want for _, rnd in calls), calls
    if split and family != 'mixtral':   # Mixtral's decode plans (router, grouped experts) return no fp32 slices
        assert any(name == 'rmsnorm_partials' for name, _ in calls), calls


@pytest.mark.gpu
def test_rmsnorm_refuses_rows_wider_than_16384_and_bad_roundings():
    ops = _ops()
    from painlessinferenceacceleration_b200 import _lib
    for hidden, rounding in ((16392, R.ONCE), (32768, R.TWICE), (4096, 2), (4096, -1)):
        x = torch.ones((2, hidden), dtype=torch.bfloat16, device=DEV)
        w = torch.ones((hidden,), dtype=torch.bfloat16, device=DEV)
        y = _sentinel((2, hidden), DEV)
        n0 = _lib.load().pia_launch_count()
        with pytest.raises(AssertionError):
            ops.rmsnorm(x, None, w, 1e-6, None, y, rounding=rounding)
        with pytest.raises(AssertionError):
            ops.rmsnorm_partials(x.float()[None], None, w, 1e-6, None, y, rounding=rounding)
        torch.cuda.synchronize()
        assert _lib.load().pia_launch_count() == n0
        assert (_bits(y) == SENT).all()


@pytest.mark.gpu
def test_rmsnorm_cuda_graph_replays_the_eager_bits():
    ops = _ops()
    x, r, w = norm_inputs(64, 4096, seed=77, device=DEV)
    parts = part_inputs(4, 64, 4096, seed=78, device=DEV)
    want = {}
    for rounding in (R.ONCE, R.TWICE):
        resid, y, y2 = r.clone(), torch.empty_like(x), torch.empty_like(x)
        ops.rmsnorm(x, resid, w, 1e-5, resid, y, rounding=rounding)
        ops.rmsnorm_partials(parts, resid, w, 1e-5, resid, y2, rounding=rounding)
        want[rounding] = (resid, y, y2)
    torch.cuda.synchronize()
    bufs = {k: (r.clone(), torch.empty_like(x), torch.empty_like(x)) for k in want}
    graph = torch.cuda.CUDAGraph()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        with torch.cuda.graph(graph, stream=s):
            for rounding, (resid, y, y2) in bufs.items():
                ops.rmsnorm(x, resid, w, 1e-5, resid, y, rounding=rounding)
                ops.rmsnorm_partials(parts, resid, w, 1e-5, resid, y2, rounding=rounding)
    torch.cuda.current_stream().wait_stream(s)
    for _ in range(2):
        for k in bufs:
            bufs[k][0].copy_(r)
        graph.replay()
        torch.cuda.synchronize()
        for k in bufs:
            for a, b in zip(bufs[k], want[k]):
                assert torch.equal(_bits(a), _bits(b))
    assert not torch.equal(_bits(want[R.ONCE][1]), _bits(want[R.TWICE][1]))


@pytest.mark.gpu
@pytest.mark.parametrize('u_kind', ['plus', 'minus', 'random'])
def test_silu_mul_every_bf16_gate(u_kind):
    """all 65 536 bf16 gate values, bit for bit against eager F.silu(g) * u on this GPU (NaN where it is NaN), and
    through the fp64 comparator"""
    ops = _ops()
    g, u = _silu_all_gates(u_kind)
    rows = 8
    gu = torch.cat([g.view(rows, -1), u.view(rows, -1)], 1).to(DEV)
    inter = g.numel() // rows
    out = torch.empty((rows, inter), dtype=torch.bfloat16, device=DEV)
    ops.silu_mul(gu, out)
    want = torch.nn.functional.silu(gu[:, :inter]) * gu[:, inter:]
    torch.cuda.synchronize()
    nan_o, nan_w = torch.isnan(out), torch.isnan(want)
    assert torch.equal(nan_o, nan_w)
    assert torch.equal(_bits(out)[~nan_o], _bits(want)[~nan_w])
    bad, n_amb = R.silu_check(out.reshape(-1).cpu(), g, u)
    assert bad == 0 and n_amb <= MAX_AMBIGUOUS * g.numel(), (bad, n_amb)


@pytest.mark.gpu
@pytest.mark.parametrize('rows,inter', [(1, 8), (5, 2056), (64, 4864), (64, 8960), (5, 13696), (64, 18944),
                                        (64 * 8, 256), (320 * 8, 14336)])
def test_silu_mul_widths_and_guard(rows, inter):
    """the width tails of real models and Mixtral's [rows * E, inter] shape; a sentinel guard after the output stays"""
    ops = _ops()
    g = torch.Generator().manual_seed(rows + inter)
    gu = (torch.randn((rows, 2 * inter), generator=g) * 4).to(torch.bfloat16).to(DEV)
    buf = _sentinel((rows * inter + 1024,), DEV)
    out = buf[:rows * inter].view(rows, inter)
    ops.silu_mul(gu, out)
    want = torch.nn.functional.silu(gu[:, :inter]) * gu[:, inter:]
    torch.cuda.synchronize()
    assert torch.equal(_bits(out), _bits(want))
    assert (_bits(buf[rows * inter:]) == SENT).all()
    assert torch.equal(_bits(out.cpu()), _bits(R.emulate_silu(gu.cpu())))


@pytest.mark.gpu
@pytest.mark.parametrize('hidden', [896, 4096, 8200])
def test_embed_gather_exact_and_zero_filled(hidden):
    """ids 0 and V - 1, n in {0, 1, rows - 1, rows}: copied rows bit exact, rows >= n exactly zero (hidden 896: fewer
    vectors than threads)"""
    ops = _ops()
    V, rows = 1000, 64
    g = torch.Generator().manual_seed(hidden)
    table = torch.randn((V, hidden), generator=g).to(torch.bfloat16).to(DEV)
    ids = torch.randint(0, V, (rows,), generator=g, dtype=torch.int32)
    ids[0], ids[1], ids[-1] = 0, V - 1, V - 1
    ids = ids.to(DEV)
    for n in (0, 1, rows - 1, rows):
        out = _sentinel((rows + 1, hidden), DEV)
        ops.embed_gather(table, ids, torch.tensor([n], dtype=torch.int32, device=DEV), out[:rows])
        torch.cuda.synchronize()
        assert torch.equal(_bits(out[:n]), _bits(table[ids[:n].long()]))
        assert (_bits(out[n:rows]) == 0).all()
        assert (_bits(out[rows]) == SENT).all()
