# -*- coding: utf-8 -*-
"""Tests of k_layernorm (csrc/fused_ops.cu, pia_layernorm) that can fail: BLOOM's and OPT's LayerNorm against an fp64
reference whose comparator tolerates only real ties (tests/norm_ref.py), at every BLOOM and OPT width and the edge
widths of the kernel's thread layout, on rows whose variance is dominated by eps, rows with a large mean next to a
small spread, outliers, constant and zero rows; the residual sum bit for bit; every aliasing of the verify forwards'
calls; torch's own nn.LayerNorm; and every LayerNorm call of the BLOOM and OPT verify forwards.

The first half runs without a GPU: the comparator accepts an emulation of the kernel's fp32 arithmetic and rejects
every wrong kernel of norm_ref.LN_MUTATIONS on the inputs the GPU half uses, and each row class and call form makes
its target mutation visible on its own."""
import pytest
import torch

from tests import norm_ref as R

DEV = 'cuda:0'
MODEL_WIDTHS = (768, 1024, 1536, 2048, 2560, 4096, 5120, 7168, 9216, 12288, 14336)
# one warp (8), a partly idle warp (264: 33 vectors on 64 threads), one thread with a second vector (4104: 513 vectors
# on 512 threads), the maximum
EDGE_WIDTHS = (8, 256, 264, 4104, 16384)
WIDTHS = EDGE_WIDTHS[:2] + MODEL_WIDTHS[:1] + EDGE_WIDTHS[2:3] + MODEL_WIDTHS[1:6] + EDGE_WIDTHS[3:4] + \
    MODEL_WIDTHS[6:] + EDGE_WIDTHS[4:]
ROWS = (1, 5, 64, 256)
EPS = (1e-5, 1e-3)
CLASSES = ('random', 'offset', 'offset_steps', 'eps_dominated', 'var_eps', 'outliers', 'constant', 'zero')
SENT = 0x7FA5               # a NaN bit pattern no kernel writes
# the share of elements the comparator may leave open.  Offset rows are the widest: the fp32 mean's error, an absolute
# (d + 1) u |mu| in every f - mean, is many ulps of x_hat where |mu| is 16 (offset) or ~115 (offset_steps) times the
# spread.  Measured with pia_layernorm on an H100 (80 GB HBM3, 700 W) over the model widths: 6.6 % of offset rows,
# 22.6 % of offset_steps rows, 0.3-0.7 % of the other classes, 0 for zero and constant rows; 3.1 % (hidden 8) to
# 8.3 % (hidden 14336 and 16384) over test_layernorm_against_fp64's calls, which include a cancelling row per call
MAX_AMBIGUOUS = 0.10        # over all calls of a test
MAX_AMBIGUOUS_CASE = 0.12   # in any one call of 64 rows or more (the ties come in clumps)
MAX_AMBIGUOUS_CLASS = dict(offset=0.20, offset_steps=0.60, default=0.03)   # per row class over the model widths
CONSTANT = 3.5              # the value of a constant row; the residual part is a multiple of 1/4 so both are exact


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


def row_classes(rows, rot=0, classes=CLASSES):
    return [classes[(i + rot) % len(classes)] for i in range(rows)]


def ln_inputs(rows, hidden, seed, eps=1e-5, classes=None, weights='normal', bias='normal', device='cpu'):
    """(x, r, w, b) bf16 and the class of each row.  The rows of s = x + r by class:
      random         x, r ~ N(0, 1)
      offset         mean 8, spread 0.5 (x ~ 8 + 0.4 N, r ~ 0.3 N): a bf16 ulp of 1/16 leaves ~8 steps per sigma
      offset_steps   x = 64 + 0.5 k, k uniform in 0..3, r = 0: two-ulp steps, |mean| ~115 x the spread, where a one-pass
                     variance E[s^2] - mean^2 cancels (the Gaussian offset row cannot get there: bf16 flattens it)
      eps_dominated  |x| ~ 1e-4, r = 0: the variance is ~1e-8, far below eps
      var_eps        x ~ sqrt(eps) N, r = 0: the variance is eps
      outliers       random, plus a few elements x 64 (as in OPT's and BLOOM's activations)
      constant       s = 3.5 exactly (r a multiple of 1/4 in [-1, 1], x = 3.5 - r)
      zero           x = r = 0
    weights: 'normal' N(1, 0.3) with some zero and negative entries, 'spread' |w| in [1e-3, 20] log-uniform with random
    signs.  bias: 'normal' 0.1 N, 'cancel' b = -bf16(x_hat * w) of row 0, so that row's x_hat * w and b cancel"""
    classes = classes or row_classes(rows)
    g = torch.Generator().manual_seed(seed)
    x = torch.randn((rows, hidden), generator=g)
    r = torch.randn((rows, hidden), generator=g)
    for i, c in enumerate(classes):
        if c == 'offset':
            x[i], r[i] = 8 + 0.4 * x[i], 0.3 * r[i]
        elif c == 'offset_steps':
            x[i], r[i] = 64 + 0.5 * torch.randint(0, 4, (hidden,), generator=g), 0
        elif c == 'eps_dominated':
            x[i], r[i] = 1e-4 * x[i], 0
        elif c == 'var_eps':
            x[i], r[i] = eps ** 0.5 * x[i], 0
        elif c == 'outliers':
            out = torch.randint(0, hidden, (max(1, hidden // 512),), generator=g)
            x[i, out] *= 64
        elif c == 'constant':
            r[i] = torch.randint(-4, 5, (hidden,), generator=g) * 0.25
            x[i] = CONSTANT - r[i]
        elif c == 'zero':
            x[i], r[i] = 0, 0
    if weights == 'normal':
        w = 1 + 0.3 * torch.randn((hidden,), generator=g)
        w[torch.randint(0, hidden, (max(1, hidden // 64),), generator=g)] = 0
        w[torch.randint(0, hidden, (max(1, hidden // 16),), generator=g)] *= -1
    else:
        w = torch.exp(torch.empty((hidden,)).uniform_(-6.9, 3.0, generator=g))
        w = w * (torch.randint(0, 2, (hidden,), generator=g) * 2 - 1)
    bf = torch.bfloat16
    x, r, w = x.to(bf), r.to(bf), w.to(bf)
    if bias == 'cancel':
        _, _, z, _, _ = R.layernorm_ref(x[:1], w, torch.zeros_like(w), eps, r[:1])
        b = -R.bf16_rne(z[0]).to(bf)
    else:
        b = (0.1 * torch.randn((hidden,), generator=g)).to(bf)
    return x.to(device), r.to(device), w.to(device), b.to(device), classes


# the call forms of the verify forwards: (residual_in, residual_out, y) given x
#   'none'      (x, None -> None, y)   the layers' x without a residual (tests; the prefill's last row)
#   'res_out'   (x, None -> ro, y)     the first layer's input norm: the residual stream starts as x
#   'inplace'   (x, r -> r, y)         every later BLOOM / pre-LN OPT norm: the residual updated in place
#   'separate'  (x, r -> None, y)      OPT-350m's post-LN norms
#   'y_is_x'    (x, None -> None, x)   BLOOM's word_embeddings_layernorm
#   'y_is_r'    (x, r -> None, r)      OPT-350m's last post-LN norm
FORMS = ('none', 'res_out', 'inplace', 'separate', 'y_is_x', 'y_is_r')


def _uses_r(form):
    return form in ('inplace', 'separate', 'y_is_r')


# ---------------------------------------------------------------------------------------------------------------
# the CPU half
# ---------------------------------------------------------------------------------------------------------------
def _emulate(c, form, mut=None):
    r = c['r'] if _uses_r(form) else None
    return R.emulate_layernorm(c['x'], c['w'], c['b'], c['eps'], r=r, mut=mut, inplace=form == 'inplace',
                               y_is_residual=form == 'y_is_r')


def _rejects(c, form, mut, amb=None):
    """whether the checks reject the emulation under mutation `mut` (None: the emulated kernel itself) in call form
    `form`: the comparator on y, residual_out bit for bit"""
    r = c['r'] if _uses_r(form) else None
    ro, y = _emulate(c, form, mut)
    s = R.residual_sum(c['x'], r)
    bad, n_amb = R.ln_check(y, c['x'], c['w'], c['b'], c['eps'], r)
    if amb is not None:
        amb.add(n_amb, y.numel(), small=c['x'].shape[0] < 64 or c['x'].shape[1] < 256)
    return bad > 0 or not torch.equal(_bits(ro), _bits(s))


def _gpu_case(hidden, ri):
    """the inputs test_layernorm_against_fp64 gives pia_layernorm at this width and row-count index"""
    rows = ROWS[ri]
    eps = EPS[(ri + hidden) % len(EPS)]
    x, r, w, b, cls = ln_inputs(rows, hidden, seed=hidden * 7 + ri, eps=eps, classes=row_classes(rows, hidden + ri),
                                weights=('normal', 'spread')[ri % 2], bias='cancel' if rows >= 64 else 'normal')
    return dict(x=x, r=r, w=w, b=b, eps=eps, classes=cls)


CPU_CASES = [(8, 2), (264, 2), (768, 3), (4104, 2), (9216, 2), (14336, 2), (16384, 1), (1024, 0)]


def test_ln_mutation_list_is_complete():
    assert set(R.LN_MUTATIONS) == {'no_eps', 'eps_after_sqrt', 'unbiased_variance', 'one_pass_variance',
                                   'xhat_rounded', 'two_roundings', 'bias_dropped', 'residual_unrounded',
                                   'stats_without_residual', 'mean_over_padded_width', 'inplace_reread',
                                   'y_before_residual_read'}


def test_ln_thread_layout():
    """blockDim and the summation depth at the edge widths, as pia_layernorm launches k_layernorm"""
    assert [R.ln_threads(h) for h in (8, 256, 264, 768, 4096, 4104, 16384)] == [32, 32, 64, 96, 512, 512, 512]
    assert [R.ln_depth(h) for h in (8, 264, 4096, 4104, 16384)] == [7 + 5, 7 + 5 + 1, 7 + 5 + 15, 15 + 5 + 15,
                                                                    31 + 5 + 15]


def test_ln_comparator_accepts_the_kernel_and_rejects_every_mutation():
    cases = [_gpu_case(h, ri) for h, ri in CPU_CASES]
    amb = Ambiguity()
    for c in cases:
        for form in FORMS:
            assert not _rejects(c, form, None, amb), (c['x'].shape, form)
    amb.check()
    for mut in R.LN_MUTATIONS:
        assert any(_rejects(c, form, mut) for c in cases for form in FORMS), mut


# (row class, width, call form, the mutations the class must expose on its own)
CLASS_TARGETS = [
    ('eps_dominated', 1024, 'separate', ('no_eps', 'eps_after_sqrt')),
    ('var_eps', 1024, 'separate', ('no_eps', 'eps_after_sqrt')),
    ('offset_steps', 768, 'separate', ('one_pass_variance',)),
    ('offset_steps', 4096, 'separate', ('one_pass_variance',)),
    ('random', 14336, 'separate', ('unbiased_variance',)),
    ('random', 9216, 'inplace', ('inplace_reread',)),
    ('random', 16384, 'inplace', ('inplace_reread',)),
    ('random', 768, 'y_is_r', ('y_before_residual_read',)),
    ('random', 14336, 'y_is_r', ('y_before_residual_read',)),
    ('random', 8, 'none', ('mean_over_padded_width',)),
    ('random', 264, 'none', ('mean_over_padded_width',)),
    ('random', 4104, 'none', ('mean_over_padded_width',)),
]


@pytest.mark.parametrize('cls,hidden,form,muts', CLASS_TARGETS,
                         ids=[f'{c}-{h}-{f}' for c, h, f, _ in CLASS_TARGETS])
def test_each_input_class_exposes_its_mutation(cls, hidden, form, muts):
    """64 rows of one class alone, eps 1e-5: the comparator accepts the kernel and rejects each target mutation"""
    x, r, w, b, _ = ln_inputs(64, hidden, seed=hidden + 1, classes=[cls] * 64)
    c = dict(x=x, r=r, w=w, b=b, eps=1e-5)
    assert not _rejects(c, form, None)
    for mut in muts:
        assert _rejects(c, form, mut), mut


def test_the_row_classes_are_needed():
    """on random rows of variance ~1 (the inputs an fp32 tolerance test uses) eps and the variance formula are
    invisible: the classes above are what exposes them"""
    x, r, w, b, _ = ln_inputs(64, 4096, seed=5, classes=['random'] * 64)
    c = dict(x=x, r=r, w=w, b=b, eps=1e-5)
    for mut in ('no_eps', 'eps_after_sqrt', 'one_pass_variance'):
        assert not _rejects(c, 'separate', mut), mut


def test_constant_and_zero_rows_give_the_bias():
    x, r, w, b, cls = ln_inputs(14, 4104, seed=3, classes=row_classes(14))
    for form in ('separate', 'none'):
        ro, y = _emulate(dict(x=x, r=r, w=w, b=b, eps=1e-5), form)
        for i, c in enumerate(cls):
            if c in ('constant', 'zero') and (c == 'zero' or _uses_r(form)):
                assert torch.equal(y[i].float(), b.float()), (form, c)


# ---------------------------------------------------------------------------------------------------------------
# the GPU half
# ---------------------------------------------------------------------------------------------------------------
def _ops():
    from painlessinferenceacceleration_b200.common import ops
    return ops


def _run(x, r, w, b, eps, form):
    """one pia_layernorm call in call form `form` on copies of the inputs -> (residual sum written or None, y, the
    untouched residual input or None).  Outputs carry a sentinel row after `rows` that must stay"""
    ops = _ops()
    rows, hidden = x.shape
    xb = torch.cat([x, _sentinel((1, hidden), x.device)])
    rb = torch.cat([r, _sentinel((1, hidden), x.device)])
    yb = _sentinel((rows + 1, hidden), x.device)
    rob = _sentinel((rows + 1, hidden), x.device)
    xi, ri, y, ro = xb[:rows], rb[:rows], yb[:rows], rob[:rows]
    if form == 'none':
        ops.layernorm(xi, None, w, b, eps, None, y)
        ro = None
    elif form == 'res_out':
        ops.layernorm(xi, None, w, b, eps, ro, y)
    elif form == 'inplace':
        ops.layernorm(xi, ri, w, b, eps, ri, y)
        ro = ri
    elif form == 'separate':
        ops.layernorm(xi, ri, w, b, eps, None, y)
        ro = None
    elif form == 'y_is_x':
        ops.layernorm(xi, None, w, b, eps, None, xi)
        y, ro = xi, None
    else:
        ops.layernorm(xi, ri, w, b, eps, None, ri)
        y, ro = ri, None
    torch.cuda.synchronize()
    for t in (xb, rb, yb, rob):
        assert (_bits(t[rows]) == SENT).all(), form
    if form not in ('y_is_x',):
        assert torch.equal(_bits(xi), _bits(x)), form
    if form in ('separate',):
        assert torch.equal(_bits(ri), _bits(r)), form
    if form not in ('res_out',):
        assert (_bits(rob) == SENT).all(), form
    if form not in ('none', 'res_out', 'inplace', 'separate'):
        assert (_bits(yb) == SENT).all(), form
    return ro, y


@pytest.mark.gpu
@pytest.mark.parametrize('hidden', WIDTHS)
def test_layernorm_against_fp64(hidden):
    """every row count, with and without a residual; eps, weights and the row classes vary with the row count.
    residual_out is bf16(x + r) bit for bit, y is the fp64 reference up to real ties, zero and constant rows give
    exactly b"""
    amb = Ambiguity()
    for ri in range(len(ROWS)):
        c = _gpu_case(hidden, ri)
        x, r, w, b = (c[k].to(DEV) for k in 'xrwb')
        for form in ('res_out', 'separate'):
            res = r if _uses_r(form) else None
            ro, y = _run(x, r, w, b, c['eps'], form)
            if ro is not None:
                assert torch.equal(_bits(ro), _bits(x)), (ROWS[ri], form)
            bad, n_amb = R.ln_check(y, x, w, b, c['eps'], res)
            assert bad == 0, (ROWS[ri], form, c['eps'], bad)
            amb.add(n_amb, y.numel(), small=ROWS[ri] < 64 or hidden < 256)
            for i, k in enumerate(c['classes']):
                if k == 'zero' or (k == 'constant' and res is not None):
                    assert torch.equal(y[i].float(), b.float()), (ROWS[ri], form, i, k)
    print(f'hidden={hidden}: {amb.n_amb} of {amb.n} elements ambiguous ({100.0 * amb.n_amb / amb.n:.4f} %)')
    amb.check()


@pytest.mark.gpu
def test_ambiguous_share_per_row_class():
    """the comparator's open share per row class over the model widths (printed) stays within MAX_AMBIGUOUS_CLASS; the
    zero and constant rows leave nothing open"""
    per = {}
    for hidden in MODEL_WIDTHS:
        x, r, w, b, cls = ln_inputs(len(CLASSES) * 16, hidden, seed=hidden + 11, weights='spread', device=DEV)
        _, y = _run(x, r, w, b, 1e-5, 'separate')
        lo, hi, amb = R.ln_accept(x, w, b, 1e-5, r)
        g = y.double()
        assert bool(((g >= lo) & (g <= hi)).all()), hidden
        for k in CLASSES:
            sel = torch.tensor([c == k for c in cls], device=DEV)
            a, n = per.get(k, (0, 0))
            per[k] = (a + int(amb[sel].sum()), n + int(sel.sum()) * hidden)
    for k, (a, n) in per.items():
        print(f'{k}: {a} of {n} elements ambiguous ({100.0 * a / n:.4f} %)')
        assert a <= MAX_AMBIGUOUS_CLASS.get(k, MAX_AMBIGUOUS_CLASS['default']) * n, k
    assert per['zero'][0] == 0 and per['constant'][0] == 0


@pytest.mark.gpu
@pytest.mark.parametrize('hidden', WIDTHS)
def test_every_aliasing_gives_the_separate_buffers_bits(hidden):
    """each call form of the verify forwards, with its outputs on top of its inputs, gives the bits of the call with
    separate buffers; the residual sum where it is written is bf16(x + r)"""
    x, r, w, b, _ = ln_inputs(64, hidden, seed=hidden + 3, device=DEV)
    want = {res: _run(x, r, w, b, 1e-5, 'separate' if res else 'none')[1] for res in (False, True)}
    s = R.residual_sum(x, r)
    bad, _ = R.ln_check(want[True], x, w, b, 1e-5, r)
    assert bad == 0
    for form in FORMS:
        ro, y = _run(x, r, w, b, 1e-5, form)
        assert torch.equal(_bits(y), _bits(want[_uses_r(form)])), form
        if ro is not None:
            assert torch.equal(_bits(ro), _bits(s if _uses_r(form) else x)), form


@pytest.mark.gpu
@pytest.mark.parametrize('hidden', (768, 1024, 4096, 5120, 9216, 14336, 16384))
def test_torch_layernorm_module(hidden):
    """torch.nn.LayerNorm in bf16 on this GPU, as transformers' BloomModel and OPTDecoderLayer apply it, differs from
    the kernel only where the comparator leaves the rounding open, and itself passes the comparator"""
    x, r, w, b, cls = ln_inputs(256, hidden, seed=hidden + 5, device=DEV, classes=row_classes(256, 0, CLASSES[:6]))
    s = R.residual_sum(x, r)
    m = torch.nn.LayerNorm(hidden, eps=1e-5).to(device=DEV, dtype=torch.bfloat16)
    with torch.no_grad():
        m.weight.copy_(w)
        m.bias.copy_(b)
        want = m(s)
    _, y = _run(x, r, w, b, 1e-5, 'separate')
    lo, hi, amb = R.ln_accept(x, w, b, 1e-5, r)
    t = want.double()
    assert bool(((t >= lo) & (t <= hi)).all()), int((~((t >= lo) & (t <= hi))).sum())
    differ = y != want
    print(f'hidden={hidden}: {int(differ.sum())} of {y.numel()} elements differ from torch.nn.LayerNorm, '
          f'{int((differ & amb).sum())} of them ambiguous; {int(amb.sum())} ambiguous in all')
    assert not (differ & ~amb).any()


def _tiny(name):
    if name.startswith('bloom'):
        from tests.tiny_bloom import tiny_model
        return tiny_model(int(name[5:]), seed=3)
    from tests.tiny_opt import tiny_model
    return tiny_model(64 if name == 'opt64' else '350m', seed=3)


def _hf_ln_order(hf, ids):
    """(module name, eps) of every nn.LayerNorm transformers' model applies in one forward, in order"""
    order, hooks = [], []
    for name, mod in hf.named_modules():
        if isinstance(mod, torch.nn.LayerNorm):
            hooks.append(mod.register_forward_hook(lambda m, a, o, n=name: order.append((n, m.eps))))
    try:
        with torch.no_grad():
            hf(input_ids=ids)
    finally:
        for h in hooks:
            h.remove()
    return order


@pytest.mark.gpu
@pytest.mark.parametrize('name', ['bloom64', 'bloom80', 'opt64', 'opt350m'])
def test_every_layernorm_call_of_the_verify_forward(name, monkeypatch):
    """ops.layernorm wrapped in a prompt forward and a tree verify forward: the calls follow transformers' module
    order with each module's eps (identified by its weight and bias storage), and each call's outputs, taken right
    after it, pass the checks against its inputs, taken right before it"""
    ops = _ops()
    model, hf = _tiny(name)
    by_ptr = {}
    for mname, mod in model.named_modules():
        if isinstance(mod, torch.nn.LayerNorm):
            by_ptr[(mod.weight.data_ptr(), mod.bias.data_ptr())] = mname
    g = torch.Generator().manual_seed(5)
    want = _hf_ln_order(hf, torch.randint(3, 200, (1, 8), generator=g).to(DEV))
    assert len(want) > 0
    calls = []
    real = ops.layernorm

    def spy(x, residual_in, weight, bias, eps, residual_out, y):
        torch.cuda.synchronize()
        snap = (x.clone(), None if residual_in is None else residual_in.clone())
        real(x, residual_in, weight, bias, eps, residual_out, y)
        torch.cuda.synchronize()
        calls.append(dict(module=by_ptr.get((weight.data_ptr(), bias.data_ptr())), eps=eps, x=snap[0], r=snap[1],
                          w=weight, b=bias, ro=None if residual_out is None else residual_out.clone(), y=y.clone(),
                          aliases=(y.data_ptr() == x.data_ptr(),
                                   residual_in is not None and y.data_ptr() == residual_in.data_ptr(),
                                   residual_in is not None and residual_out is not None and
                                   residual_out.data_ptr() == residual_in.data_ptr())))

    monkeypatch.setattr(ops, 'layernorm', spy)
    p = torch.randint(3, 200, (1, 16), generator=g).to(DEV)
    m01 = torch.tril(torch.ones((1, 1, 16, 16), dtype=torch.long, device=DEV))
    _, P = model.forward(p, m01, past_key_values=0)
    d = torch.randint(3, 200, (1, 8), generator=g).to(DEV)
    m01 = torch.cat([torch.ones((1, 1, 8, P), dtype=torch.long, device=DEV),
                     torch.tril(torch.ones((1, 1, 8, 8), dtype=torch.long, device=DEV))], -1)
    model.forward(d, m01, past_key_values=P)
    torch.cuda.synchronize()
    got = [(c['module'], c['eps']) for c in calls]
    assert got == 2 * want, (got, want)
    amb = Ambiguity()
    for c in calls:
        s = R.residual_sum(c['x'], c['r'])
        if c['ro'] is not None:
            assert torch.equal(_bits(c['ro']), _bits(s)), c['module']
        bad, n_amb = R.ln_check(c['y'], c['x'], c['w'], c['b'], c['eps'], c['r'])
        assert bad == 0, (c['module'], bad)
        amb.add(n_amb, c['y'].numel(), small=True)
    amb.check()
    forms = {c['aliases'] for c in calls}
    if name == 'opt350m':
        assert (False, True, False) in forms     # the last post-LN norm writes y over its residual input
    else:
        assert (False, False, True) in forms     # the residual updated in place
    if name.startswith('bloom'):
        assert (True, False, False) in forms     # the embedding norm in place


@pytest.mark.gpu
def test_layernorm_cuda_graph_replays_the_eager_bits():
    """every call form captured at hidden 14336 and 768: replay gives the eager bits"""
    ops = _ops()
    cases = []
    for hidden in (768, 14336):
        x, r, w, b, _ = ln_inputs(64, hidden, seed=hidden + 9, device=DEV)
        cases.append((x, r, w, b, {form: _run(x, r, w, b, 1e-5, form) for form in FORMS}))
    bufs = []
    graph = torch.cuda.CUDAGraph()
    st = torch.cuda.Stream()
    st.wait_stream(torch.cuda.current_stream())
    for x, r, w, b, _ in cases:
        for form in FORMS:
            bufs.append(dict(x=x.clone(), r=r.clone(), ro=torch.empty_like(x), y=torch.empty_like(x)))
    with torch.cuda.stream(st):
        with torch.cuda.graph(graph, stream=st):
            i = 0
            for x, r, w, b, _ in cases:
                for form in FORMS:
                    t = bufs[i]
                    i += 1
                    args = dict(none=(t['x'], None, None, t['y']), res_out=(t['x'], None, t['ro'], t['y']),
                                inplace=(t['x'], t['r'], t['r'], t['y']), separate=(t['x'], t['r'], None, t['y']),
                                y_is_x=(t['x'], None, None, t['x']), y_is_r=(t['x'], t['r'], None, t['r']))[form]
                    ops.layernorm(args[0], args[1], w, b, 1e-5, args[2], args[3])
    torch.cuda.current_stream().wait_stream(st)
    for _ in range(2):
        i = 0
        for x, r, _, _, _ in cases:
            for _ in FORMS:
                bufs[i]['x'].copy_(x)
                bufs[i]['r'].copy_(r)
                i += 1
        graph.replay()
        torch.cuda.synchronize()
        i = 0
        for _, _, _, _, want in cases:
            for form in FORMS:
                t = bufs[i]
                i += 1
                y = dict(y_is_x=t['x'], y_is_r=t['r']).get(form, t['y'])
                assert torch.equal(_bits(y), _bits(want[form][1])), form
                if want[form][0] is not None:
                    ro = t['r'] if form == 'inplace' else t['ro']
                    assert torch.equal(_bits(ro), _bits(want[form][0])), form


@pytest.mark.gpu
def test_layernorm_refuses_invalid_calls():
    """hidden off a multiple of 8 or above 16384, a null weight, bias or output: an AssertionError naming layernorm,
    nothing launched, the output untouched"""
    ops = _ops()
    bad = []
    for hidden in (12, 16392, 32768):
        z = torch.ones((4, hidden), dtype=torch.bfloat16, device=DEV)
        wz = torch.ones((hidden,), dtype=torch.bfloat16, device=DEV)
        bad.append((z, None, wz, wz, None, _sentinel((4, hidden), DEV)))
    z = torch.ones((4, 1024), dtype=torch.bfloat16, device=DEV)
    wz = torch.ones((1024,), dtype=torch.bfloat16, device=DEV)
    y = _sentinel((4, 1024), DEV)
    bad += [(z, None, None, wz, None, y), (z, None, wz, None, None, y), (z, None, wz, wz, y, None)]
    n0 = ops.launch_count()
    for x, r, w, b, ro, y in bad:
        with pytest.raises(AssertionError, match='layernorm'):
            ops.layernorm(x, r, w, b, 1e-5, ro, y)
    torch.cuda.synchronize()
    assert ops.launch_count() == n0
    for *_, ro, y in bad:
        for t in (ro, y):
            if t is not None:
                assert (_bits(t) == SENT).all()
