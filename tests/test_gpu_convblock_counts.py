"""The conv block with per-language row counts (b200tts_convblock_forward_counts / _backward_counts) against fp64, through the C ABI.

Channel block g holds counts[g] utterances in rows 0 .. counts[g] - 1 and its other rows are vacant.  Every occupied block is checked
on its own: the rows and channels of language g form a G = 1 block of counts[g] rows, whose fp64 epilogue and per-element bounds are
tests/convblock_check.py's, computed from the kernel's own convolution product.  Vacant rows of out and d x must be exact zeros
although the test fills the vacant rows of x and d out with random values.  An absent language (count 0) must keep its running
statistics bit for bit and get exactly zero d gamma / d beta / d w.  Every buffer the library writes sits inside a NaN-sentinel guard
band, a repeat call is bit-identical, and with every count equal to NB the results are bitwise those of the plain entry points.
"""
import ctypes

import pytest
import torch

import convblock_check as CC
from test_gpu_convblock import Guarded, _case, _intact, _operands, _run, _with_precision

pytestmark = pytest.mark.gpu


@pytest.fixture(scope='module', autouse=True)
def _built():
    import __graft_entry__ as entry
    entry.build()
    assert torch.cuda.is_available()


def _run_counts(c, T, counts):
    """Forward + backward through the counts ABI on guarded buffers -> (results, {buffer: sentinel intact})."""
    from multilingual_text_to_speech_b200 import _lib, functional as F
    NB, G, Cin, Cout, L = (c[n] for n in ('NB', 'G', 'Cin', 'Cout', 'L'))
    Ct = G * Cout
    Cf = Cout // 2 if c['highway'] else Cout
    n = NB * Ct * L
    tail = CC.a64(n) - n + 2 * CC.a64(Ct) + 64
    shape = _lib.ConvBlockShape(NB, G, Cin, Cout, L, c['k'], c['dil'], CC.ACTS[c['act']], c['highway'], c['training'], c['eps'],
                                c['momentum'], c['p'], c['stage'])
    lib, sh, st = _lib.load(), ctypes.byref(shape), F._stream()
    saved = F._bytes(lib.b200tts_convblock_saved_bytes(sh), 'cuda')
    ws = F._bytes(lib.b200tts_convblock_workspace_bytes(sh), 'cuda')
    cnt = Guarded(G, 16, 0, torch.tensor(counts, dtype=torch.int32).view(torch.float32))
    cnt_ptr = F.ptr(cnt.t)
    b = dict(x=Guarded(T['x'].numel(), tail, 0, T['x']), out=Guarded(NB * G * (Cf if c['stage'] != 1 else Cout) * L, tail),
             rm=Guarded(Ct, tail, 0, T['rm']), rv=Guarded(Ct, tail, 0, T['rv']))
    gamma = beta = None
    gs = Cout
    if c['stage'] != 1:
        if c['gen']:
            b['aff'] = Guarded(2 * Ct, tail, 0, torch.cat([T['gamma'].view(G, Cout), T['beta'].view(G, Cout)], 1))
            gamma, beta, gs = b['aff'].t, b['aff'].t[Cout:], 2 * Cout
        else:
            b['gamma'], b['beta'] = Guarded(Ct, tail, 0, T['gamma']), Guarded(Ct, tail, 0, T['beta'])
            gamma, beta = b['gamma'].t, b['beta'].t
    w = T['w'] if c['stage'] != 2 else None
    keep = T['keep'] if c['stage'] != 1 else None
    F.check(lib.b200tts_convblock_forward_counts(sh, cnt_ptr, G, NB, F.ptr(b['x'].t), F.ptr(w), F.ptr(gamma), F.ptr(beta), gs,
                                                 F.ptr(b['rm'].t), F.ptr(b['rv'].t), F.ptr(keep), F.ptr(b['out'].t), F.ptr(saved),
                                                 F.ptr(ws), st), 'b200tts_convblock_forward_counts')
    dout = T['dout']
    b['dout'] = Guarded(dout.numel(), tail, 0, dout)
    b['dx'] = Guarded(T['x'].numel(), tail)
    if w is not None:
        b['dw'] = Guarded(w.numel(), tail, 0, torch.zeros_like(w))
    dg = db = None
    if c['stage'] != 1:
        if c['gen']:
            b['dgb'] = Guarded(2 * Ct, tail, 0, torch.zeros(2 * Ct))
            dg, db = b['dgb'].t, b['dgb'].t[Cout:]
        else:
            b['dgamma'], b['dbeta'] = Guarded(Ct, tail, 0, torch.zeros(Ct)), Guarded(Ct, tail, 0, torch.zeros(Ct))
            dg, db = b['dgamma'].t, b['dbeta'].t
    F.check(lib.b200tts_convblock_backward_counts(sh, cnt_ptr, G, NB, F.ptr(b['x'].t), F.ptr(w), F.ptr(gamma), F.ptr(beta), gs,
                                                  F.ptr(keep), F.ptr(saved), F.ptr(b['dout'].t), F.ptr(b['dx'].t),
                                                  F.ptr(b.get('dw') and b['dw'].t), F.ptr(dg), F.ptr(db), F.ptr(ws), st),
            'b200tts_convblock_backward_counts')
    torch.cuda.synchronize()
    assert cnt.intact()
    sv = saved.view(torch.float32)
    m0, i0 = CC.a64(n), CC.a64(n) + CC.a64(Ct)
    res = dict(out=b['out'].t.view(NB, -1, L).clone(), dx=b['dx'].t.view_as(T['x']).clone())
    if c['stage'] != 1:
        res.update(mean=sv[m0:m0 + Ct].clone(), invstd=sv[i0:i0 + Ct].clone(),
                   conv=sv[:n].view(NB, Ct, L).clone() if c['stage'] == 0 else T['x'])
        res['rm'], res['rv'] = b['rm'].t.clone(), b['rv'].t.clone()
        if c['gen']:
            full = b['dgb'].t.view(G, 2 * Cout)
            res['dgamma'], res['dbeta'] = full[:, :Cout].reshape(-1).clone(), full[:, Cout:].reshape(-1).clone()
        else:
            res['dgamma'], res['dbeta'] = b['dgamma'].t.clone(), b['dbeta'].t.clone()
    if w is not None:
        res['dw'] = b['dw'].t.view_as(w).clone()
    return res, {name: g.intact() for name, g in b.items()}


def _block(t, g, C, rows):
    """Rows 0 .. rows-1 and channels g*C .. (g+1)*C - 1 of a [NB, G*C, L] tensor."""
    return t[:rows, g * C:(g + 1) * C]


def _check_language(c, T, res, g, n, mode):
    """Language g's n occupied rows against the fp64 epilogue of a G = 1 block of n rows; returns the worst err / bound per quantity."""
    G, Cin, Cout = c['G'], c['Cin'], c['Cout']
    Cf = Cout // 2 if c['highway'] else Cout
    cg = dict(c, G=1, NB=n)
    d = {k: v.double() for k, v in T.items()}
    sl = slice(g * Cout, (g + 1) * Cout)
    x, w = _block(d['x'], g, Cin, n), d['w'][sl]
    gamma, beta, rm, rv = d['gamma'][sl], d['beta'][sl], d['rm'][sl], d['rv'][sl]
    keep = _block(d['keep'], g, Cout, n) if c['training'] and c['p'] > 0 else None
    dout = _block(d['dout'], g, Cf, n)
    conv = _block(res['conv'].double(), g, Cout, n)
    R = CC.epilogue(cg, conv, gamma, beta, keep=keep, xin=x, rm=rm, rv=rv, dout=dout)
    K = dict(mean=res['mean'][sl].double(), invstd=res['invstd'][sl].double())
    B = CC.bounds(cg, R, K, conv, gamma, beta, keep=keep, xin=x, rm=rm, rv=rv, dout=dout, x=x, w=w, mode=mode)
    got = dict(out=_block(res['out'], g, Cf, n), mean=res['mean'][sl], invstd=res['invstd'][sl], dgamma=res['dgamma'][sl],
               dbeta=res['dbeta'][sl], dx=_block(res['dx'], g, Cin, n))
    ref = dict(out=R['out'], mean=R['mean'], invstd=1.0 / torch.sqrt(R['var'] + c['eps']), dgamma=R['dgamma'], dbeta=R['dbeta'])
    if c['training']:
        got['rm'], got['rv'] = res['rm'][sl], res['rv'][sl]
        ref['rm'], ref['rv'] = R['rm'], R['rv']
    if c['stage'] == 0:
        dx, ref['dw'] = CC.conv_transposes(x, w, 1, c['dil'], R['dconv'])
        ref['dx'] = dx + R['dskip'] if c['highway'] else dx
        got['dw'] = res['dw'][sl]
    else:
        ref['dx'] = R['dconv']
    rep = CC.report(got, ref, B)
    assert not CC.failures(rep), (g, n, CC.failures(rep))
    return rep


def _check_conv_only(c, T, res, g, n, mode):
    """Stage 1 (the product alone): out = conv, d x / d w = its transposes of d out, within the GEMM accumulation bound."""
    Cin, Cout, k, dil = c['Cin'], c['Cout'], c['k'], c['dil']
    d = {kk: v.double() for kk, v in T.items()}
    sl = slice(g * Cout, (g + 1) * Cout)
    x, w, dconv = _block(d['x'], g, Cin, n), d['w'][sl], _block(d['dout'], g, Cout, n)
    ref_out = CC.conv_groups(x, w, 1, dil)
    bnd_out = CC.conv_rel(Cin * k, mode) * CC.conv_groups(x.abs(), w.abs(), 1, dil) * CC.SLACK
    ref_dx, ref_dw = CC.conv_transposes(x, w, 1, dil, dconv)
    tx, tw = CC.conv_transposes(x.abs(), w.abs(), 1, dil, dconv.abs())
    B = dict(out=bnd_out, dx=CC.conv_rel(Cout * k, mode) * tx * CC.SLACK, dw=CC.conv_rel(n * c['L'], mode) * tw * CC.SLACK)
    got = dict(out=_block(res['out'], g, Cout, n), dx=_block(res['dx'], g, Cin, n), dw=res['dw'][sl])
    rep = CC.report(got, dict(out=ref_out, dx=ref_dx, dw=ref_dw), B)
    assert not CC.failures(rep), (g, n, CC.failures(rep))
    return rep


def _check_counts(c, T, res, counts, mode):
    G, Cin, Cout, NB = c['G'], c['Cin'], c['Cout'], c['NB']
    Cf = Cout // 2 if c['highway'] else Cout
    Co = Cout if c['stage'] == 1 else Cf
    worst = {}
    for g, n in enumerate(counts):
        # vacant rows: exact zeros of every output and of d x
        assert bool((res['out'][n:, g * Co:(g + 1) * Co] == 0).all()), f'vacant out rows of language {g} are not 0'
        assert bool((res['dx'][n:, g * Cin:(g + 1) * Cin] == 0).all()), f'vacant dx rows of language {g} are not 0'
        sl = slice(g * Cout, (g + 1) * Cout)
        if n == 0:                      # absent: statistics untouched, exactly zero parameter gradients
            if c['stage'] != 1:
                assert torch.equal(res['rm'][sl], T['rm'][sl]) and torch.equal(res['rv'][sl], T['rv'][sl]), f'language {g}: stats moved'
                assert bool((res['dgamma'][sl] == 0).all()) and bool((res['dbeta'][sl] == 0).all()), f'language {g}: d affine'
            if 'dw' in res:
                assert bool((res['dw'][sl] == 0).all()), f'language {g}: d w is not 0'
            continue
        rep = (_check_conv_only if c['stage'] == 1 else _check_language)(c, T, res, g, n, mode)
        for q, v in rep.items():
            worst[q] = max(worst.get(q, 0.0), v[0])
        if not c['training'] and c['stage'] != 1:
            assert torch.equal(res['rm'][sl], T['rm'][sl]) and torch.equal(res['rv'][sl], T['rv'][sl])
    return worst


ENC = dict(G=4, eps=1e-8, gen=True)
CASES = {
    'stage0_plain_k1_relu': _case(NB=5, G=4, Cin=64, Cout=48, L=36, act='relu', eps=1e-5),
    'stage0_gen_highway_k3_dil9': _case(NB=5, **ENC, Cin=32, Cout=64, L=40, k=3, dil=9, act='identity', highway=1),
    'stage0_gen_highway_k1_oddL': _case(NB=5, **ENC, Cin=32, Cout=64, L=37, act='identity', highway=1),
    'stage0_plain_k5_tanh': _case(NB=5, G=4, Cin=24, Cout=40, L=44, k=5, act='tanh', eps=1e-5),
    'stage1_conv_k3': _case(NB=5, G=4, Cin=24, Cout=40, L=44, k=3, dil=3, act='identity', stage=1),
    'stage2_gen_bn': _case(NB=5, **ENC, Cout=48, L=36, act='relu', stage=2),
}
COUNTS = {'full': [5, 5, 5, 5], 'uneven': [5, 2, 4, 1], 'absent': [3, 0, 5, 2]}


def _operands_counts(c, seed, mode):
    return _operands(c, seed, mode)        # d out of the convolution-only stage is [NB, G*Cout, L]: Cf == Cout without highway


@pytest.mark.parametrize('training', [1, 0], ids=['train', 'eval'])
@pytest.mark.parametrize('counts', list(COUNTS))
@pytest.mark.parametrize('name', list(CASES))
def test_counts_against_fp64(name, counts, training):
    c = dict(CASES[name], training=training)
    cn = COUNTS[counts]
    T = _operands_counts(c, sum(map(ord, name)) + training, 'fp32')
    (r1, g1), (r2, g2) = (_run_counts(c, T, cn) for _ in range(2))
    _intact(g1, name)
    _intact(g2, name)
    for q in r1:
        assert torch.equal(r1[q], r2[q]), f'{name}: {q} differs between two identical calls'
    worst = _check_counts(c, T, r1, cn, 'fp32')
    print(name, counts, 'train' if training else 'eval', {q: f'{v:.3f}' for q, v in worst.items()})
    if counts == 'full':           # every count == NB: bitwise the plain entry points (stage 1 writes no statistics)
        ref, _ = _run(c, T)
        for q in (('out', 'dx', 'dw') if c['stage'] == 1 else ('out', 'mean', 'invstd', 'rm', 'rv', 'dx', 'dw', 'dgamma', 'dbeta')):
            if q in ref:
                assert torch.equal(r1[q], ref[q]), f'{name}: {q} differs from b200tts_convblock_forward / _backward'


@pytest.mark.parametrize('name', ['stage0_gen_highway_k3_dil9', 'stage0_plain_k5_tanh'])
def test_counts_bf16_mode(name):
    """bf16 mode: the implicit wgmma convolutions and the bf16 weight gradient see zeros in the vacant rows."""
    c = dict(CASES[name], training=1)
    cn = COUNTS['absent']
    T = _operands_counts(c, 7, 'bf16')
    (r1, g1), (r2, _) = (_with_precision('bf16', lambda: _run_counts(c, T, cn)) for _ in range(2))
    _intact(g1, name)
    for q in r1:
        assert torch.equal(r1[q], r2[q]), q
    _check_counts(c, T, r1, cn, 'bf16')


@pytest.mark.parametrize('training', [1, 0], ids=['train', 'eval'])
def test_counts_single_row_at_length_one(training):
    """One language with a single row at L = 1: n = 1, so the running variance takes the biased variance (the n > 1 rule)."""
    c = _case(NB=3, G=3, Cin=16, Cout=32, L=1, act='identity', highway=1, gen=True, eps=1e-8, training=training)
    cn = [3, 1, 0]
    T = _operands_counts(c, 11, 'fp32')
    res, guards = _run_counts(c, T, cn)
    _intact(guards, 'L=1')
    _check_counts(c, T, res, cn, 'fp32')


def test_counts_out_of_range_are_clamped():
    """A count above NB reads as NB and a negative one as 0: the results equal those of the clamped counts, nothing outside is touched."""
    c = dict(CASES['stage0_gen_highway_k1_oddL'], training=1)
    T = _operands_counts(c, 3, 'fp32')
    a, ga = _run_counts(c, T, [9, -4, 5, 2])
    b, _ = _run_counts(c, T, [5, 0, 5, 2])
    _intact(ga, 'clamped')
    for q in a:
        assert torch.equal(a[q], b[q]), q
