"""The per-step decoder ops (location attention, forward attention, LSTM cell; forward and backward) through the module-level C ABI
in fp32 mode, every element against the fp64 oracle of tests/step_ops_check.py with its own bound.

Every call also asserts: NaN-poisoned outputs and workspace come back finite, the sentinel guard bands around every buffer the call
writes are untouched, the += outputs accumulate onto random prefills, a second identical call is bitwise equal, and each utterance's
outputs equal that utterance run alone (inference_batch relies on it).  Run with -s to see the worst err / bound ratio of every
output of every case."""
import ctypes

import pytest
import torch

import step_check as S
import step_ops_check as O
from multilingual_text_to_speech_b200 import _lib

pytestmark = pytest.mark.gpu

GUARD = 64
SENTINEL = 1.2345678e30
NAN = float('nan')


@pytest.fixture(scope='module', autouse=True)
def fp32_mode():
    import __graft_entry__ as entry
    entry.build()
    _lib.set_precision('fp32')
    assert _lib.get_precision() == 'fp32'


class Buf:
    """a float32 device buffer inside GUARD sentinel elements either side"""

    def __init__(self, init):
        n = init.numel()
        self.full = torch.full((n + 2 * GUARD,), SENTINEL, dtype=torch.float32, device='cuda')
        self.t = self.full[GUARD:GUARD + n].view(init.shape)
        self.t.copy_(init)

    def guards_ok(self):
        return bool((self.full[:GUARD] == SENTINEL).all()) and bool((self.full[-GUARD:] == SENTINEL).all())


def _nan(*shape):
    return torch.full(shape, NAN, dtype=torch.float32, device='cuda')


def _call(fn, args, bufs, what):
    """args: ABI arguments, where a str names a buffer of bufs (built fresh from the {name: initial content} dict).  Asserts status,
    untouched guard bands and finite results; -> {name: result}"""
    b = {k: Buf(v) for k, v in bufs.items()}
    stream = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    call = [_lib.ptr(b[a].t) if isinstance(a, str) else a for a in args]
    _lib.check(fn(*call, stream), what)
    torch.cuda.synchronize()
    for k, x in b.items():
        assert x.guards_ok(), (what, k, 'guard band written')
        assert torch.isfinite(x.t).all(), (what, k, 'non-finite result')
    return {k: x.t.clone() for k, x in b.items()}


def _same(a, b, what):
    for k in a:
        assert torch.equal(a[k], b[k]), (what, k, 'not bitwise reproducible')


def _report(title, out, refs, lines):
    worst = 0.0
    for name, (ref, bound) in refs.items():
        r, i = O.ratio(out[name], ref, bound)
        lines.append(f'{title} {name:>8s}: worst err/bound {r:.3e}')
        assert r <= 1.0, (title, name, r, i, float(out[name].reshape(-1)[i]), float(ref.reshape(-1)[i]), float(bound.reshape(-1)[i]))
        worst = max(worst, r)
    return worst


def _lengths(B, L, g, extra=()):
    lens = torch.randint(1, L + 1, (B,), generator=g)
    lens[0] = L
    if B > 1:
        lens[-1] = 1
    for j, x in enumerate(extra):
        lens[1 + j] = x
    return lens.to(torch.int32)


def _cum_from_softmax_rows(lens, L, g, rows=3):
    """cumulative weights of `rows` earlier steps: sums of softmax rows over each utterance's length"""
    B = lens.numel()
    valid = torch.arange(L)[None, :] < lens[:, None].long()
    cum = torch.zeros(B, L, dtype=torch.float64)
    for _ in range(rows):
        e = (torch.randn(B, L, generator=g, dtype=torch.float64) * 3).masked_fill(~valid, -float('inf'))
        cum += torch.softmax(e, -1).masked_fill(~valid, 0.0)
    return cum.float()


# ------------------------------------------------------------------------------------------------------------------------
# location-sensitive attention
# ------------------------------------------------------------------------------------------------------------------------
def _loc_inputs(B, L, M, A, C, K, D, seed, lens_extra=(), v_scale=1.0):
    g = torch.Generator().manual_seed(seed)
    r = lambda *s, scale=1.0: (torch.randn(*s, generator=g) * scale)    # noqa: E731
    lens = _lengths(B, L, g, lens_extra)
    x = {'query': r(B, D), 'Wq': r(A, D, scale=D ** -0.5), 'memory': r(B, L, M), 'memT': r(B, L, A, scale=0.5),
         'Wloc': r(A, C, scale=C ** -0.5), 'Wc': r(C, 1, K, scale=K ** -0.5), 'bias': r(1, A, scale=0.1),
         'v': r(1, A, scale=6 * A ** -0.5) * v_scale, 'cum': _cum_from_softmax_rows(lens, L, g),
         'd_ctx': r(B, M, scale=0.1), 'd_w': r(B, L, scale=0.1), 'd_cum': r(B, L, scale=0.1),
         'p_memT': r(B, L, A, scale=0.1), 'p_Wloc': r(A, C, scale=0.1), 'p_Wc': r(C, 1, K, scale=0.1), 'p_v': r(1, A, scale=0.1)}
    x = {k: t.cuda() for k, t in x.items()}
    x['lens'] = lens.cuda()
    return x


def _loc_run(x, sel=None):
    """forward then backward of the batch (or of the utterances `sel`) -> (forward outputs, backward outputs)"""
    lib = _lib.load()
    if sel is not None:
        x = {k: (t[sel] if k in ('query', 'memory', 'memT', 'cum', 'd_ctx', 'd_w', 'd_cum', 'p_memT', 'lens') else t) for k, t in x.items()}
    B, L, M = x['memory'].shape
    A, D = x['Wq'].shape
    C, _, K = x['Wc'].shape
    fwd = _call(lib.b200tts_attention_step,
                [B, L, M, D, A, C, K, _lib.ptr(x['query']), _lib.ptr(x['memory']), _lib.ptr(x['memT']), _lib.ptr(x['lens']),
                 _lib.ptr(x['Wq']), _lib.ptr(x['Wloc']), _lib.ptr(x['Wc']), _lib.ptr(x['bias']), _lib.ptr(x['v']),
                 'cum', 'context', 'weights', 'ws'],
                {'cum': x['cum'], 'context': _nan(B, M), 'weights': _nan(B, L),
                 'ws': _nan(lib.b200tts_attention_step_workspace_elems(B, L, A))}, 'attention_step')
    fwd['q'] = fwd['ws'][:B * A].view(B, A).clone()
    bwd = _call(lib.b200tts_attention_step_backward,
                [B, L, M, A, C, K, _lib.ptr(fwd['q']), _lib.ptr(x['memory']), _lib.ptr(x['memT']), _lib.ptr(x['lens']),
                 _lib.ptr(x['Wloc']), _lib.ptr(x['Wc']), _lib.ptr(x['bias']), _lib.ptr(x['v']), _lib.ptr(x['cum']),
                 _lib.ptr(fwd['weights']), _lib.ptr(x['d_ctx']), _lib.ptr(x['d_w']),
                 'd_cum', 'd_q', 'd_memT', 'd_Wloc', 'd_Wc', 'd_v', 'ws'],
                {'d_cum': x['d_cum'], 'd_q': _nan(B, A), 'd_memT': x['p_memT'], 'd_Wloc': x['p_Wloc'], 'd_Wc': x['p_Wc'],
                 'd_v': x['p_v'], 'ws': _nan(lib.b200tts_attention_step_backward_workspace_elems(B, M, A, C, K))},
                'attention_step_backward')
    return fwd, bwd


LOC_CASES = [dict(B=4, L=L) for L in (1, 5, 31, 33, 216, 217, 220, 300, 400, 644)] + [
    dict(B=60, L=180),
    dict(B=3, L=640, M=512),
    dict(B=6, L=300, lens_extra=(171, 172, 173)),        # LC = 172: one below, at and above the chunk boundary
    dict(B=6, L=400, lens_extra=(119, 120, 121)),        # LC = 120
    dict(B=1, L=220), dict(B=7, L=217), dict(B=65, L=300),
    dict(B=5, L=33, A=64, C=16, K=5), dict(B=5, L=17, A=4, C=4, K=1),
    dict(B=4, L=60, v_scale=20.0, name='saturating'), dict(B=4, L=60, v_scale=0.0, name='equal energies'),
]


def _loc_id(c):
    return c.get('name', '').replace(' ', '_') or '-'.join(f'{k}{v}' for k, v in c.items() if k != 'lens_extra') + \
        ('-boundary' if 'lens_extra' in c else '')


@pytest.mark.parametrize('case', LOC_CASES, ids=[_loc_id(c) for c in LOC_CASES])
def test_location_attention_step_within_bounds(case):
    case = dict(case)
    title = f'[location {_loc_id(case)}]'
    case.pop('name', None)
    B, L = case['B'], case['L']
    M, A, C, K = case.get('M', 288), case.get('A', 128), case.get('C', 32), case.get('K', 31)
    x = _loc_inputs(B, L, M, A, C, K, 1024, seed=L + B, lens_extra=case.get('lens_extra', ()), v_scale=case.get('v_scale', 1.0))
    LC = _lib.load().b200tts_debug_attention_backward_chunk(L, M, A, C, K)
    assert LC > 0 and LC % 4 == 0
    chunks = -(-int(x['lens'].max()) // LC)
    fwd, bwd = _loc_run(x)
    lines = [f'{title} backward chunk LC = {LC}: {chunks} chunk(s)']
    prm = {'attn_location': x['Wloc'], 'attn_loc_features': x['Wc'], 'attn_bias': x['bias'], 'attn_energy': x['v']}
    lens = x['lens'].long()
    valid = torch.arange(L, device='cuda')[None, :] < lens[:, None]
    # exact properties
    assert torch.equal(fwd['cum'], x['cum'] + fwd['weights']), 'cum_next is not fl(cum_prev + w)'
    assert (fwd['weights'].masked_fill(valid, 0.0) == 0).all(), 'weights beyond the length'
    refs = {'q': O.query_product(x['query'], x['Wq'])}
    refs.update(O.location_forward(fwd['q'], x['cum'], x['memT'], x['memory'], x['lens'], prm, fwd['weights']))
    _report(title, fwd, refs, lines)
    ob = O.location_backward(fwd['q'], x['cum'], x['memT'], x['memory'], x['lens'], prm, fwd['weights'], x['d_ctx'], x['d_w'], x['d_cum'])
    refs = {'d_cum': ob['d_cum'], 'd_q': ob['d_q'], 'd_memT': O.accumulate(x['p_memT'], *ob['d_memT']),
            'd_Wloc': O.accumulate(x['p_Wloc'], *ob['d_Wloc']), 'd_Wc': O.accumulate(x['p_Wc'].reshape(C, K), *ob['d_Wc']),
            'd_v': O.accumulate(x['p_v'].reshape(-1), *ob['d_v'])}
    got = dict(bwd, d_Wc=bwd['d_Wc'].reshape(C, K), d_v=bwd['d_v'].reshape(-1))
    _report(title, got, refs, lines)
    # reproducible, and each utterance equal to itself run alone
    fwd2, bwd2 = _loc_run(x)
    _same({k: fwd[k] for k in ('cum', 'context', 'weights', 'q')}, fwd2, title)
    _same({k: bwd[k] for k in bwd if k != 'ws'}, bwd2, title)
    for b in range(B):
        f1, b1 = _loc_run(x, [b])
        for k in ('cum', 'context', 'weights', 'q'):
            assert torch.equal(f1[k][0], fwd[k][b]), (title, 'alone', b, k)
        for k in ('d_cum', 'd_q', 'd_memT'):
            assert torch.equal(b1[k][0], bwd[k][b]), (title, 'alone', b, k)
    print('\n' + '\n'.join(lines))


def test_location_attention_chunk_counts():
    """the L = 300 / 400 / 644 cases above run 2 / 4 / 161 backward chunks (LC = 172 / 120 / 4)"""
    lib = _lib.load()
    for L, n in ((300, 2), (400, 4), (644, 161)):
        LC = lib.b200tts_debug_attention_backward_chunk(L, 288, 128, 32, 31)
        assert -(-L // LC) == n, (L, LC)


# ------------------------------------------------------------------------------------------------------------------------
# forward attention
# ------------------------------------------------------------------------------------------------------------------------
def _fwd_inputs(B, L, M, A, D, seed):
    g = torch.Generator().manual_seed(seed)
    r = lambda *s, scale=1.0: (torch.randn(*s, generator=g) * scale)    # noqa: E731
    x = {'query': r(B, D), 'Wq': r(A, D, scale=D ** -0.5), 'memory': r(B, L, M), 'memT': r(B, L, A, scale=0.5),
         'bias': r(1, A, scale=0.1), 'v': r(1, A, scale=6 * A ** -0.5), 'd_ctx': r(B, M, scale=0.1), 'd_w': r(B, L, scale=0.1),
         'd_alpha': r(B, L, scale=0.1), 'p_memT': r(B, L, A, scale=0.1), 'p_v': r(1, A, scale=0.1)}
    x = {k: t.cuda() for k, t in x.items()}
    x['lens'] = _lengths(B, L, g).cuda()
    return x


def _fwd_step(x, alpha):
    lib = _lib.load()
    B, L, M = x['memory'].shape
    A, D = x['Wq'].shape
    out = _call(lib.b200tts_forward_attention_step,
                [B, L, M, D, A, _lib.ptr(x['query']), _lib.ptr(x['memory']), _lib.ptr(x['memT']), _lib.ptr(x['lens']),
                 _lib.ptr(x['Wq']), _lib.ptr(x['bias']), _lib.ptr(x['v']), 'alpha', 'context', 'weights', 'ws'],
                {'alpha': alpha, 'context': _nan(B, M), 'weights': _nan(B, L),
                 'ws': _nan(lib.b200tts_forward_attention_step_workspace_elems(B, L, A))}, 'forward_attention_step')
    out['q'] = out['ws'][:B * A].view(B, A).clone()
    return out


def _fwd_run(x, alpha, sel=None):
    lib = _lib.load()
    if sel is not None:
        x = {k: (t[sel] if k in ('query', 'memory', 'memT', 'd_ctx', 'd_w', 'd_alpha', 'p_memT', 'lens') else t) for k, t in x.items()}
        alpha = alpha[sel]
    B, L, M = x['memory'].shape
    A = x['Wq'].shape[0]
    fwd = _fwd_step(x, alpha)
    bwd = _call(lib.b200tts_forward_attention_step_backward,
                [B, L, M, A, _lib.ptr(fwd['q']), _lib.ptr(x['memory']), _lib.ptr(x['memT']), _lib.ptr(x['lens']), _lib.ptr(x['bias']),
                 _lib.ptr(x['v']), _lib.ptr(alpha), _lib.ptr(fwd['weights']), _lib.ptr(x['d_ctx']), _lib.ptr(x['d_w']),
                 'd_alpha', 'd_q', 'd_memT', 'd_v', 'ws'],
                {'d_alpha': x['d_alpha'], 'd_q': _nan(B, A), 'd_memT': x['p_memT'], 'd_v': x['p_v'],
                 'ws': _nan(lib.b200tts_forward_attention_step_backward_workspace_elems(B, M, A))}, 'forward_attention_step_backward')
    return fwd, bwd


@pytest.mark.parametrize('alpha_kind', ('reset', 'peaked', 'uniform'))
@pytest.mark.parametrize('L', (1, 2, 33, 180, 257, 300, 1000))
def test_forward_attention_step_within_bounds(L, alpha_kind):
    B, M, A, D = 4, 288, 128, 1024
    title = f'[forward L{L} {alpha_kind}]'
    x = _fwd_inputs(B, L, M, A, D, seed=L)
    alpha = torch.zeros(B, L, device='cuda')
    alpha[:, 0] = 1.0
    if alpha_kind == 'uniform':
        alpha.fill_(1.0 / L)
    elif alpha_kind == 'peaked':
        for _ in range(4):          # a few steps from the reset: everything past the first few positions sits on the floor
            alpha = _fwd_step(x, alpha)['alpha']
    fwd, bwd = _fwd_run(x, alpha)
    lines = []
    assert torch.equal(fwd['alpha'], fwd['weights']), 'alpha_next is not the weights'
    prm = {'attn_bias': x['bias'], 'attn_energy': x['v']}
    refs = {'q': O.query_product(x['query'], x['Wq'])}
    refs.update(O.forward_forward(fwd['q'], alpha, x['memT'], x['memory'], x['lens'], prm, fwd['weights']))
    _report(title, fwd, refs, lines)
    ob = O.forward_backward(fwd['q'], alpha, x['memT'], x['memory'], x['lens'], prm, fwd['weights'], x['d_ctx'], x['d_w'], x['d_alpha'])
    refs = {'d_alpha': ob['d_alpha'], 'd_q': ob['d_q'], 'd_memT': O.accumulate(x['p_memT'], *ob['d_memT']),
            'd_v': O.accumulate(x['p_v'].reshape(-1), *ob['d_v'])}
    _report(title, dict(bwd, d_v=bwd['d_v'].reshape(-1)), refs, lines)
    fwd2, bwd2 = _fwd_run(x, alpha)
    _same({k: fwd[k] for k in ('alpha', 'context', 'weights', 'q')}, fwd2, title)
    _same({k: bwd[k] for k in bwd if k != 'ws'}, bwd2, title)
    for b in range(B):
        f1, b1 = _fwd_run(x, alpha, [b])
        for k in ('alpha', 'context', 'weights', 'q'):
            assert torch.equal(f1[k][0], fwd[k][b]), (title, 'alone', b, k)
        for k in ('d_alpha', 'd_q', 'd_memT'):
            assert torch.equal(b1[k][0], bwd[k][b]), (title, 'alone', b, k)
    print('\n' + '\n'.join(lines))


# ------------------------------------------------------------------------------------------------------------------------
# LSTM cell
# ------------------------------------------------------------------------------------------------------------------------
CELL_VARIANTS = [(kind, training, masks, rate) for kind in (_lib.CELL_DROPOUT, _lib.CELL_ZONEOUT) for training in (True, False)
                 for masks in (True, False) for rate in (0.0, 0.1, 0.5)]
CELL_SHAPES = [(B, D) for B in (1, 5, 8, 9, 65, 130) for D in (1, 31, 33, 1024, 1280)]


def _cell_run(B, D, kind, training, rate, z, hp, cp, mh, mc, dh, dc):
    lib = _lib.load()
    fwd = _call(lib.b200tts_lstm_cell_forward,
                [B, D, kind, int(training), rate, rate, 'gates', _lib.ptr(hp), _lib.ptr(cp), _lib.ptr(mh), _lib.ptr(mc), 'h', 'c'],
                {'gates': z, 'h': _nan(B, D), 'c': _nan(B, D)}, 'lstm_cell_forward')
    bwd = _call(lib.b200tts_lstm_cell_backward,
                [B, D, kind, int(training), rate, rate, _lib.ptr(fwd['gates']), _lib.ptr(cp), _lib.ptr(mh), _lib.ptr(mc), _lib.ptr(dh),
                 'd_c', 'd_h_prev', 'd_gates'],
                {'d_c': dc, 'd_h_prev': _nan(B, D), 'd_gates': _nan(B, 4 * D)}, 'lstm_cell_backward')
    return fwd, bwd


@pytest.mark.parametrize('shape', CELL_SHAPES, ids=lambda s: 'B{}_D{}'.format(*s))
def test_lstm_cell_step_within_bounds(shape):
    B, D = shape
    i = CELL_SHAPES.index(shape)
    lines = []
    for j in (i, i + len(CELL_SHAPES)):          # two variants per shape: together the shapes run every variant
        kind, training, masks, rate = CELL_VARIANTS[j % len(CELL_VARIANTS)]
        title = f'[cell B{B} D{D} {"zoneout" if kind else "dropout"} {"train" if training else "eval"} ' \
                f'{"masks" if masks else "no masks"} rate {rate}]'
        g = torch.Generator().manual_seed(B * 10000 + D + j)
        z = torch.randn(B, 4 * D, generator=g) * 4
        z.view(-1)[::7] = 20.0 * torch.sign(torch.randn(z.view(-1)[::7].shape, generator=g))   # saturated gates
        hp, cp = torch.randn(B, D, generator=g), torch.randn(B, D, generator=g) * 2
        dh, dc = torch.randn(B, D, generator=g), torch.randn(B, D, generator=g)
        mh = mc = None
        if masks:
            mh = (torch.rand(B, D, generator=g) >= rate).to(torch.uint8).cuda()
            mc = (torch.rand(B, D, generator=g) >= rate).to(torch.uint8).cuda() if kind == _lib.CELL_ZONEOUT else None
        z, hp, cp, dh, dc = (t.cuda() for t in (z, hp, cp, dh, dc))
        fwd, bwd = _cell_run(B, D, kind, training, rate, z, hp, cp, mh, mc, dh, dc)
        cfg = S.Config(kind, training, rate, rate if kind == _lib.CELL_ZONEOUT else 0.0)
        _report(title, fwd, O.cell_fwd(z, hp, cp, mh, mc, cfg, fwd['gates']), lines)
        _report(title, bwd, O.cell_bwd(fwd['gates'], cp, mh, mc, dh, dc, cfg), lines)
        if kind == _lib.CELL_DROPOUT:
            assert (bwd['d_h_prev'] == 0).all(), 'the dropout cell has no direct h gradient'
        fwd2, bwd2 = _cell_run(B, D, kind, training, rate, z, hp, cp, mh, mc, dh, dc)
        _same(fwd, fwd2, title)
        _same(bwd, bwd2, title)
        for b in sorted({0, B // 2, B - 1}):
            sel = slice(b, b + 1)
            f1, b1 = _cell_run(1, D, kind, training, rate, z[sel], hp[sel], cp[sel], None if mh is None else mh[sel],
                               None if mc is None else mc[sel], dh[sel], dc[sel])
            for k in f1:
                assert torch.equal(f1[k][0], fwd[k][b]), (title, 'alone', b, k)
            for k in b1:
                assert torch.equal(b1[k][0], bwd[k][b]), (title, 'alone', b, k)
    print('\n' + '\n'.join(lines))
