"""The training-step reduction kernels through the C ABI, every element against the fp64 oracle of tests/train_ops_check.py with its own
bound: the Tacotron loss (forward and backward), the WaveRNN losses (RAW and MOL), the upsampling-layer and aux-stretch adjoints, the
fixed-order column sums, and the fused clip + Adam step.

Every call also asserts: NaN-poisoned outputs and workspaces come back finite (except the NaN rows the ABI documents), the sentinel guard
bands around every buffer the call writes are untouched, the += outputs accumulate onto random prefills, the inputs come back unchanged,
and a second identical call is bitwise equal.  Run with -s to see the worst err / bound ratio of every output of every case."""
import ctypes
import math

import numpy as np
import pytest
import torch

import train_ops_check as O
from multilingual_text_to_speech_b200 import _lib

pytestmark = pytest.mark.gpu

GUARD = 64
SENTINEL = 1.2345678e30
NAN = float('nan')


@pytest.fixture(scope='module', autouse=True)
def built():
    import __graft_entry__ as entry
    entry.build()
    _lib.set_precision('fp32')


class Buf:
    """a float32 device buffer inside GUARD sentinel elements either side (GUARD floats keep the start 16-byte aligned)"""

    def __init__(self, init):
        n = init.numel()
        self.full = torch.full((n + 2 * GUARD,), SENTINEL, dtype=torch.float32, device='cuda')
        self.t = self.full[GUARD:GUARD + n].view(init.shape)
        self.t.copy_(init)

    def guards_ok(self):
        return bool((self.full[:GUARD] == SENTINEL).all()) and bool((self.full[-GUARD:] == SENTINEL).all())


def _nan(*shape):
    return torch.full(shape, NAN, dtype=torch.float32, device='cuda')


def _call(fn, args, bufs, what, inputs=(), written=None):
    """args: ABI arguments, where a str names a buffer of bufs (built fresh from the {name: initial content} dict).  Asserts status,
    untouched guard bands, unchanged inputs and finite results (written: {name: the part of the buffer the call writes, or None for a
    buffer checked by the caller}); -> {name: result}"""
    saved = [x.clone() for x in inputs]
    b = {k: Buf(v) for k, v in bufs.items()}
    stream = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    call = [_lib.ptr(b[a].t) if isinstance(a, str) else a for a in args]
    _lib.check(fn(*call, stream), what)
    torch.cuda.synchronize()
    for k, x in b.items():
        assert x.guards_ok(), (what, k, 'guard band written')
        part = (written or {}).get(k, slice(None))
        if part is not None:
            assert torch.isfinite(x.t.reshape(-1)[part]).all(), (what, k, 'non-finite result')
    for x, s in zip(inputs, saved):
        assert torch.equal(x, s), (what, 'an input changed')
    return {k: x.t.clone() for k, x in b.items()}


def _same(a, b, what):
    for k in a:
        assert torch.equal(a[k], b[k]) or (torch.isnan(a[k]).any() and torch.equal(torch.nan_to_num(a[k], 7.0), torch.nan_to_num(b[k], 7.0))), \
            (what, k, 'not bitwise reproducible')


def _report(title, out, refs, lines):
    for name, (ref, bound) in refs.items():
        r, i = O.ratio(out[name], ref, bound)
        lines.append(f'{title} {name:>8s}: worst err/bound {r:.3e}')
        assert r <= 1.0, (title, name, r, i, float(out[name].reshape(-1)[i]), float(ref.reshape(-1)[i]), float(bound.reshape(-1)[i]))


def _gen(seed):
    return torch.Generator(device='cuda').manual_seed(seed)


# ------------------------------------------------------------------------------------------------------------------------
# Tacotron loss
# ------------------------------------------------------------------------------------------------------------------------
def _loss_inputs(B, N, T, L, R, seed):
    g = torch.Generator().manual_seed(seed)
    S = -(-T // R)
    x = {k: torch.randn(B, N, T, generator=g) for k in ('pre', 'pre_t', 'post')}
    x['post_t'] = x['pre_t'] + 0.1 * torch.randn(B, N, T, generator=g)
    tlen = torch.randint(1, L + 1, (B,), generator=g)
    mlen = torch.randint(1, T + 1, (B,), generator=g)
    tlen[0], mlen[0] = L, T
    if B > 1:
        tlen[-1], mlen[-1] = 1, 1                                   # text_len = 1 and target_len = 1
    if B > 2:
        mlen[1] = max(1, T - R - 1)                                 # target_len < T, not on the step grid
    if B > 3:
        tlen[2] = L + 3                                             # longer than the alignment: Lb = min(text_len, L)
    stop = torch.randn(B, T, generator=g) * 3
    stop_t = torch.zeros(B, T)
    for b in range(B):
        stop_t[b, max(int(mlen[b]) - 2, 0):] = 1.0
        stop[b, int(mlen[b]):] = 1000.0                             # the padding Tacotron.forward writes
    stop[0, 0] = -1000.0                                            # confident and right: exactly 0 in the limit
    x['stop'], x['stop_t'] = stop, stop_t
    x['align'] = torch.softmax(torch.randn(B, S, L, generator=g) * 2, dim=2)
    x = {k: v.cuda() for k, v in x.items()}
    x['tlen'], x['mlen'] = tlen.to(torch.int32).cuda(), mlen.to(torch.int32).cuda()
    return x


def _loss_fwd(x, shape, views=None):
    lib = _lib.load()
    v = views or x
    ws = lib.b200tts_loss_workspace_bytes() // 4
    ins = [x[k] for k in ('pre', 'pre_t', 'post', 'post_t', 'stop', 'stop_t', 'align', 'tlen', 'mlen')]
    return _call(lib.b200tts_tacotron_loss_forward,
                 [ctypes.byref(shape)] + [_lib.ptr(v[k]) for k in ('pre', 'pre_t', 'post', 'post_t')] +
                 [_lib.ptr(x[k]) for k in ('stop', 'stop_t', 'align', 'tlen', 'mlen')] + ['losses', 'ws'],
                 {'losses': _nan(4), 'ws': _nan(ws)}, 'tacotron_loss_forward', inputs=ins)


def _loss_bwd(x, shape, gl, outs=('d_pre', 'd_post', 'd_stop', 'd_align')):
    lib = _lib.load()
    B, N, T = x['pre'].shape
    _, S, L = x['align'].shape
    full = {'d_pre': _nan(B, N, T), 'd_post': _nan(B, N, T), 'd_stop': _nan(B, T), 'd_align': _nan(B, S, L)}
    bufs = {k: full[k] for k in outs}
    ins = [x[k] for k in ('pre', 'pre_t', 'post', 'post_t', 'stop', 'stop_t', 'tlen', 'mlen')] + [gl]
    return _call(lib.b200tts_tacotron_loss_backward,
                 [ctypes.byref(shape)] + [_lib.ptr(x[k]) for k in ('pre', 'pre_t', 'post', 'post_t', 'stop', 'stop_t', 'tlen', 'mlen')] +
                 [_lib.ptr(gl)] + [(k if k in outs else None) for k in ('d_pre', 'd_post', 'd_stop', 'd_align')],
                 bufs, 'tacotron_loss_backward', inputs=ins)


LOSS_CASES = [
    dict(B=60, N=80, T=900, L=180, name='bench'),
    dict(B=3, N=12, T=17, L=11), dict(B=10, N=80, T=301, L=77), dict(B=4, N=80, T=64, L=180, g=0.05), dict(B=2, N=5, T=9, L=4, guided=0),
    dict(B=2, N=2, T=5, L=3, pw=1.0), dict(B=3, N=5, T=7, L=9, pw=7.5), dict(B=2, N=3, T=7, L=5, g=0.05), dict(B=1, N=3, T=5, L=4),
    dict(B=4, N=80, T=37, L=50, R=2), dict(B=3, N=16, T=41, L=20, R=3, g=0.05), dict(B=5, N=7, T=23, L=13, R=3, pw=7.5),
    dict(B=6, N=80, T=301, L=77, R=2, guided=0),
]


def _loss_id(c):
    return c.get('name') or '-'.join(f'{k}{v}' for k, v in c.items())


@pytest.mark.parametrize('case', LOSS_CASES, ids=[_loss_id(c) for c in LOSS_CASES])
def test_tacotron_loss_within_bounds(case):
    c = dict(dict(R=1, g=0.2, pw=100.0, guided=1), **case)
    B, N, T, L, R = c['B'], c['N'], c['T'], c['L'], c['R']
    title = f'[loss {_loss_id(case)}] B*N*T % 4 = {B * N * T % 4}'
    x = _loss_inputs(B, N, T, L, R, seed=B * 1000 + T + R)
    shape = _lib.LossShape(B, N, T, L, c['guided'], c['g'], c['pw'], R)
    lines = []
    fwd = _loss_fwd(x, shape)
    refs = O.tacotron_loss_forward(x['pre'], x['pre_t'], x['post'], x['post_t'], x['stop'], x['stop_t'], x['align'], x['tlen'].cpu(),
                                   x['mlen'].cpu(), R, c['g'], c['pw'], c['guided'])
    _report(title, fwd, refs, lines)
    if not c['guided']:
        assert fwd['losses'][3] == 0
    gl = torch.tensor([0.7, 1.3, 2.0, 0.5], device='cuda')
    bwd = _loss_bwd(x, shape, gl)
    refs = O.tacotron_loss_backward(x['pre'], x['pre_t'], x['post'], x['post_t'], x['stop'], x['stop_t'], x['tlen'].cpu(), x['mlen'].cpu(),
                                    -(-T // R), L, R, c['g'], c['pw'], c['guided'], gl.cpu())
    _report(title, bwd, refs, lines)
    # outside each utterance's step / text grid, or with the guided term off, d_align is exactly 0 (the bound there is 0)
    _same(fwd, _loss_fwd(x, shape), title)
    _same(bwd, _loss_bwd(x, shape, gl), title)
    print('\n' + '\n'.join(lines))


def test_tacotron_loss_backward_null_outputs():
    """every subset of d_pre / d_post / d_stop / d_align: the outputs passed are the full call's, bit for bit"""
    B, N, T, L, R = 4, 80, 37, 50, 2
    x = _loss_inputs(B, N, T, L, R, seed=5)
    shape = _lib.LossShape(B, N, T, L, 1, 0.2, 100.0, R)
    gl = torch.tensor([0.7, 1.3, 2.0, 0.5], device='cuda')
    full = _loss_bwd(x, shape, gl)
    names = ('d_pre', 'd_post', 'd_stop', 'd_align')
    for mask in range(1, 16):
        outs = tuple(n for j, n in enumerate(names) if mask >> j & 1)
        got = _loss_bwd(x, shape, gl, outs)
        for k in outs:
            assert torch.equal(got[k], full[k]), (outs, k)


@pytest.mark.parametrize('shape', ((3, 80, 41, 20), (3, 7, 41, 20), (2, 7, 41, 20), (1, 7, 41, 20)), ids=lambda s: f'BNT%4={s[0] * s[1] * s[2] % 4}')
@pytest.mark.parametrize('shift', (1, 2, 3))
def test_tacotron_loss_forward_any_float_alignment(shift, shape):
    """pre / pre_target / post / post_target at 1, 2 and 3 floats past a 16-byte boundary (each its own shift), with and without an
    nmel % 4 tail: the forward takes its scalar loads there and equals the aligned call bit for bit"""
    B, N, T, L = shape
    x = _loss_inputs(B, N, T, L, 1, seed=11)
    shape = _lib.LossShape(B, N, T, L, 1, 0.2, 100.0, 1)
    views = {}
    for j, k in enumerate(('pre', 'pre_t', 'post', 'post_t')):
        s = (shift + j) % 4 if j else shift
        store = torch.empty(x[k].numel() + 4, device='cuda')
        assert store.data_ptr() % 16 == 0
        views[k] = store[s:s + x[k].numel()].view_as(x[k])
        views[k].copy_(x[k])
    got = _loss_fwd(x, shape, views)
    want = _loss_fwd(x, shape)
    assert torch.equal(got['losses'], want['losses']), (got['losses'], want['losses'])


# ------------------------------------------------------------------------------------------------------------------------
# WaveRNN losses
# ------------------------------------------------------------------------------------------------------------------------
def _wloss(mode, logits, target):
    lib = _lib.load()
    N, n_out = logits.shape
    ws = lib.b200tts_wavernn_loss_workspace_bytes(N) // 4
    bad = None
    if mode == _RAW:
        bad = ((target < 0) | (target >= n_out)).nonzero().reshape(-1).cpu()
    written = {'loss': (slice(None) if bad is None or bad.numel() == 0 else None),
               'ws': (slice(None) if bad is None or bad.numel() == 0 else None)}
    out = _call(lib.b200tts_wavernn_loss, [mode, N, n_out, _lib.ptr(logits), _lib.ptr(target), 'loss', 'dlogits', 'ws', ws * 4],
                {'loss': _nan(1), 'dlogits': _nan(N, n_out), 'ws': _nan(ws)}, 'wavernn_loss', inputs=[logits, target], written=written)
    return out


_RAW, _MOL = 0, 1
ROW_COUNTS = (1, 7, 8, 9, 4096, 64 * 2750)


def _raw_inputs(N, n, seed):
    g = _gen(seed)
    logits = torch.randn(N, n, device='cuda', generator=g) * 3
    lab = torch.randint(0, n, (N,), device='cuda', generator=g, dtype=torch.int32)
    lab[0] = 0
    if N > 1:
        lab[-1] = n - 1
    return logits, lab


def _check_raw(N, n, seed, lines):
    title = f'[raw N{N} n{n}]'
    logits, lab = _raw_inputs(N, n, seed)
    out = _wloss(_RAW, logits, lab)
    refs = O.raw_loss(logits, lab)
    _report(title, {'loss': out['loss'], 'rows': out['ws'], 'dlogits': out['dlogits']}, refs, lines)
    _same(out, _wloss(_RAW, logits, lab), title)
    # a row with a label outside [0, n): its row loss (and so the mean) is NaN, its d logits the softmax / N; the other rows unchanged
    r = N // 2
    for badlab in (n, -1):
        lab2 = lab.clone()
        lab2[r] = badlab
        bad = _wloss(_RAW, logits, lab2)
        assert torch.isnan(bad['loss']).all() and torch.isnan(bad['ws'][r])
        keep = torch.arange(N, device='cuda') != r
        assert torch.isfinite(bad['ws'][keep]).all() and torch.equal(bad['ws'][keep], out['ws'][keep])
        assert torch.isfinite(bad['dlogits']).all() and torch.equal(bad['dlogits'][keep], out['dlogits'][keep])
        ref, bnd = O.raw_loss(logits, lab2)['dlogits']
        rr, _ = O.ratio(bad['dlogits'][r], ref[r], bnd[r])
        lines.append(f'{title} label {badlab}: d logits of the row worst err/bound {rr:.3e}')
        assert rr <= 1.0


@pytest.mark.parametrize('n', (2, 31, 33, 512, 65536))
def test_raw_loss_within_bounds(n):
    lines = []
    _check_raw(9 if n == 65536 else 4096 if n == 512 else 300, n, n, lines)
    print('\n' + '\n'.join(lines))


@pytest.mark.parametrize('N', ROW_COUNTS)
def test_raw_loss_row_counts(N):
    lines = []
    _check_raw(N, 33, N + 1, lines)
    print('\n' + '\n'.join(lines))


def _threshold_mid(inv):
    """mid = inv (y - mu) where the fp64 cdf_delta = sigmoid(mid + inv hb) - sigmoid(mid - inv hb) equals 1e-5 (bisection, mid >= 0)"""
    lo, hi = 0.0, 60.0
    f = lambda m: 1 / (1 + math.exp(-(m + inv * O.HALF_BIN))) - 1 / (1 + math.exp(-(m - inv * O.HALF_BIN))) - O.CDF_FLOOR   # noqa: E731
    if f(lo) < 0:
        return None
    for _ in range(200):
        mid = 0.5 * (lo + hi)
        lo, hi = (mid, hi) if f(mid) > 0 else (lo, mid)
    return lo


def _mol_inputs(N, nr, seed):
    g = _gen(seed)
    lp = torch.randn(N, nr, device='cuda', generator=g) * 2
    mu = torch.rand(N, nr, device='cuda', generator=g) * 2 - 1
    ls = torch.rand(N, nr, device='cuda', generator=g) * 6 - 5.5
    y = torch.rand(N, device='cuda', generator=g) * 2 - 1
    f32 = lambda v: float(np.float32(v))                             # noqa: E731
    edge = f32(0.999)
    special = [-1.0, 1.0, edge, -edge, float(np.nextafter(np.float32(edge), np.float32(2))), float(np.nextafter(np.float32(edge), np.float32(0))),
               -float(np.nextafter(np.float32(edge), np.float32(2))), -float(np.nextafter(np.float32(edge), np.float32(0)))]
    for j, v in enumerate(special[:N]):
        y[j] = v
    if N > 10:
        ls[8, :] = O.LOG_SCALE_MIN                                   # the clamp edge: gradient passes
        ls[9, :] = O.LOG_SCALE_MIN - 1.0                             # below it: clamped, no gradient
        ls[10, :] = -20.0                                            # a tiny scale far from y: the pdf branch
        mu[10, :] = y[10] + 0.25 + 0.01 * torch.arange(nr, device='cuda')    # one mixture leads by far: finite bounds
    if N > 12:                                                       # on the cdf_delta threshold in fp64
        for r in (11, 12):
            inv = math.exp(1.0)
            ls[r, :] = -1.0
            m = _threshold_mid(inv)
            mu[r, :] = float(y[r]) - (m if r == 11 else -m) / inv
    return torch.cat([lp, mu, ls], 1).contiguous(), y


def _check_mol(N, nr, seed, lines):
    title = f'[mol N{N} nr{nr}]'
    logits, y = _mol_inputs(N, nr, seed)
    out = _wloss(_MOL, logits, y)
    refs = O.mol_loss(logits, y)
    _report(title, {'loss': out['loss'], 'rows': out['ws'], 'dlogits': out['dlogits']}, refs, lines)
    lo, hi = O.mol_branches(y)
    lines.append(f'{title} rows on the left / right edge: {int(lo.sum())} / {int(hi.sum())}')
    if N > 10:
        assert (out['dlogits'][9, 2 * nr:] == 0).all(), 'a clamped log scale passes gradient'
    _same(out, _wloss(_MOL, logits, y), title)


@pytest.mark.parametrize('nr', (1, 10, 31, 32))
def test_mol_loss_within_bounds(nr):
    lines = []
    _check_mol(777, nr, nr, lines)
    print('\n' + '\n'.join(lines))


@pytest.mark.parametrize('N', ROW_COUNTS)
def test_mol_loss_row_counts(N):
    lines = []
    _check_mol(N, 10, N, lines)
    print('\n' + '\n'.join(lines))


# ------------------------------------------------------------------------------------------------------------------------
# upsampling layer adjoint
# ------------------------------------------------------------------------------------------------------------------------
def _ups(C, ln, s, fir, x, dout, prefill, mode):
    lib = _lib.load()
    wsb = lib.b200tts_wavernn_upsample_layer_backward_workspace_bytes(C, ln, s)
    bufs = {'ws': _nan(wsb // 4)}
    if mode in ('din', 'both'):
        bufs['din'] = _nan(C, ln)
    if mode in ('dfir', 'both'):
        bufs['dfir'] = prefill
    return _call(lib.b200tts_wavernn_upsample_layer_backward,
                 [C, ln, s, _lib.ptr(fir), _lib.ptr(x), _lib.ptr(dout), 'din' if 'din' in bufs else None, 'dfir' if 'dfir' in bufs else None,
                  'ws', wsb], bufs, 'upsample_layer_backward', inputs=[fir, x, dout],
                 written={'ws': (slice(None) if 'dfir' in bufs else None)})


UPS_CASES = [(B, T, j) for B in (1, 7, 64) for T in (275, 2750) for j in range(3)]


@pytest.mark.parametrize('case', UPS_CASES + [(0, 0, 0)], ids=[f'B{b}-T{t}-layer{j}' for b, t, j in UPS_CASES] + ['tiny'])
def test_upsample_backward_within_bounds(case):
    B, T, j = case
    if B == 0:
        C, ln, s = 1, 3, 5                                           # C len s = 15 < 64: most chunks are empty
    else:
        W = T // 275 + 4
        C, ln, s = 80 * B, (W, 5 * W, 25 * W)[j], (5, 5, 11)[j]
    title = f'[upsample C{C} len{ln} s{s}]'
    g = _gen(C * 7 + ln + s)
    fir = torch.randn(2 * s + 1, device='cuda', generator=g) / (2 * s + 1)
    x = torch.randn(C, ln, device='cuda', generator=g)
    dout = torch.randn(C, ln * s, device='cuda', generator=g)
    prefill = torch.randn(2 * s + 1, device='cuda', generator=g)
    lines = []
    both = _ups(C, ln, s, fir, x, dout, prefill, 'both')
    refs = O.upsample_backward(fir, x, dout, s)
    _report(title, both, {'din': refs['din'], 'dfir': O.accumulate(prefill, *refs['dfir'])}, lines)
    _same(both, _ups(C, ln, s, fir, x, dout, prefill, 'both'), title)
    assert torch.equal(_ups(C, ln, s, fir, x, dout, prefill, 'din')['din'], both['din'])
    assert torch.equal(_ups(C, ln, s, fir, x, dout, prefill, 'dfir')['dfir'], both['dfir'])
    print('\n' + '\n'.join(lines))


# ------------------------------------------------------------------------------------------------------------------------
# aux stretch adjoint and column sums
# ------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('hop', (1, 275))
@pytest.mark.parametrize('BFC', ((1, 1, 1), (3, 14, 32), (7, 5, 33), (64, 14, 128)))
def test_stretch_backward_within_bounds(hop, BFC):
    B, F, C = BFC
    lib = _lib.load()
    dup = torch.randn(B, F * hop, C, device='cuda', generator=_gen(hop + C))
    run = lambda: _call(lib.b200tts_wavernn_stretch_backward, [B, F, C, hop, _lib.ptr(dup), 'daux'],      # noqa: E731
                        {'daux': _nan(B, F, C)}, 'stretch_backward', inputs=[dup])
    out = run()
    lines = []
    _report(f'[stretch B{B} F{F} C{C} hop{hop}]', out, O.stretch_backward(dup, F, hop), lines)
    _same(out, run(), 'stretch')
    print('\n' + '\n'.join(lines))


@pytest.mark.parametrize('cols', (1, 255, 257, 1536))
@pytest.mark.parametrize('rows', (1, 63, 64, 65, 64 * 2750))
def test_column_sum_within_bounds(rows, cols):
    lib = _lib.load()
    g = _gen(rows + cols)
    x = torch.randn(rows, cols, device='cuda', generator=g) + 0.5
    prefill = torch.randn(cols, device='cuda', generator=g)
    wsb = lib.b200tts_column_sum_workspace_bytes(cols)
    run = lambda: _call(lib.b200tts_column_sum, [rows, cols, _lib.ptr(x), 'out', 'ws', wsb],      # noqa: E731
                        {'out': prefill, 'ws': _nan(wsb // 4)}, 'column_sum', inputs=[x])
    out = run()
    lines = []
    ref, b = O.column_sum(x)['out']
    _report(f'[column_sum rows{rows} cols{cols}]', out, {'out': O.accumulate(prefill, ref, b)}, lines)
    _same(out, run(), 'column_sum')
    print('\n' + '\n'.join(lines))


# ------------------------------------------------------------------------------------------------------------------------
# fused clip + Adam
# ------------------------------------------------------------------------------------------------------------------------
BIG_N = 30_000_003


def _adam_inputs(n, seed):
    g = _gen(seed)
    p = torch.randn(n, device='cuda', generator=g)
    gr = torch.randn(n, device='cuda', generator=g) * 1e-3
    m = torch.randn(n, device='cuda', generator=g) * 1e-4
    v = torch.rand(n, device='cuda', generator=g) * 1e-7
    if n > 1:
        zero = torch.arange(n, device='cuda') % 3 == 1                # gradient elements that stay exactly zero: v = 0, denominator eps
        gr[zero], m[zero], v[zero] = 0.0, 0.0, 0.0
    gr[n // 2] = 1e3                                                  # one element 10^6 times the rest
    return p, gr, m, v


def _adam(p, gr, m, v, hp):
    lib = _lib.load()
    n = p.numel()
    nblk = O.norm_blocks(n)
    sf = lib.b200tts_adam_clip_scratch_floats()
    written = {'scratch': torch.cat([torch.arange(2), 8 + torch.arange(nblk)]).cuda()}
    return _call(lib.b200tts_adam_clip_step,
                 ['p', 'g', 'm', 'v', n, hp['lr'], 0.9, 0.999, 1e-8, hp['wd'], hp['max_norm'], hp['step'], 'scratch'],
                 {'p': p, 'g': gr, 'm': m, 'v': v, 'scratch': _nan(sf)}, 'adam_clip_step', written=written)


def _check_adam(n, hp, seed, lines):
    title = f'[adam n{n} wd{hp["wd"]} max_norm{hp["max_norm"]} step{hp["step"]}]'
    p, gr, m, v = _adam_inputs(n, seed)
    out = _adam(p, gr, m, v, hp)
    refs = O.adam_clip(p, gr, m, v, hp['lr'], 0.9, 0.999, 1e-8, hp['wd'], hp['max_norm'], hp['step'])
    got = dict(out, norm=out['scratch'][0:1], coef=out['scratch'][1:2])
    _report(title, got, refs, lines)
    coef, b_coef = refs['coef']
    if hp['max_norm'] <= 0 or float(coef[0]) == 1.0 and float(b_coef[0]) == 0.0:     # no clip, or the clip safely does not bind
        assert float(out['scratch'][1]) == 1.0
    _same(out, _adam(p, gr, m, v, hp), title)


ADAM_HP = [dict(lr=1e-3, wd=wd, max_norm=mx, step=st) for wd in (0.0, 1e-6) for mx in (-1.0, 0.0, 1e-3, 1e9) for st in (1, 2, 100000)]


@pytest.mark.parametrize('n', (1, 3, 4, 5, 1023))
def test_adam_clip_within_bounds(n):
    lines = []
    for j, hp in enumerate(ADAM_HP):
        _check_adam(n, hp, n * 100 + j, lines)
    print('\n' + '\n'.join(lines))


@pytest.mark.parametrize('hp', [ADAM_HP[7], ADAM_HP[12 + 9 + 2]], ids=('clip', 'decay-noclip-late'))
def test_adam_clip_large_within_bounds(hp):
    lines = []
    _check_adam(BIG_N, hp, 1, lines)
    print('\n' + '\n'.join(lines))


def test_adam_clip_refuses_unaligned_gradient():
    """the float4 norm pass needs a 16-byte aligned gradient: refused on the host, nothing launched"""
    lib = _lib.load()
    buf = torch.zeros(64, device='cuda')
    n0 = _lib.launch_count()
    st = lib.b200tts_adam_clip_step(_lib.ptr(buf), ctypes.c_void_p(buf.data_ptr() + 4), _lib.ptr(buf), _lib.ptr(buf), 8, 1e-3, 0.9, 0.999,
                                    1e-8, 0.0, 1.0, 1, _lib.ptr(buf), None)
    assert st != 0 and b'16-byte' in lib.b200tts_last_error()
    assert _lib.launch_count() == n0
