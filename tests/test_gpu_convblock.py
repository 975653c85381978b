"""The conv block's batch-norm epilogue (csrc/encoder.cu: bn_stats / block_fwd / block_bwd_prep / bn_bwd_reduce / bn_bwd_apply, scalar
and float4) against fp64 at the real shapes, through the C ABI with every buffer owned by the test.

The reference and the per-element bounds are tests/convblock_check.py: the epilogue is recomputed in fp64 from the kernel's own
convolution product (the first conv_elems floats of `saved`, with mean / invstd after it, include/b200tts.h), so the bounds are those
of the fp32 epilogue alone; d x and d w add the GEMM's accumulation bound.  No blanket tolerance.

Every buffer the library writes (out, the running statistics, d x, d w, d gamma / d beta including the [G, 2C] generated gradient) is
carved from a larger one filled with a sentinel NaN pattern, with a tail longer than the per-channel sums a stage 2 backward once
wrote past d x; the sentinel must be intact after forward and backward.

Paths: L % 4 == 0 with 16-byte aligned tensors takes the float4 kernels; an odd L, or x / out / d out one float off alignment, the
scalar ones (the choice is vec4_ok and the alignment tests of channel_sum / bn_bwd_reduce / the backward launcher).
"""
import ctypes

import pytest
import torch

import convblock_check as CC

pytestmark = pytest.mark.gpu

SENT = 0x7fa1b2c3          # a NaN bit pattern no kernel writes
HEAD = 64


@pytest.fixture(scope='module', autouse=True)
def _built():
    import __graft_entry__ as entry
    entry.build()
    assert torch.cuda.is_available()


class Guarded:
    """n floats at float offset HEAD + off of a sentinel-filled buffer with `tail` floats after them."""

    def __init__(self, n, tail, off=0, init=None):
        self.buf = torch.full((HEAD + off + n + tail,), SENT, dtype=torch.int32, device='cuda')
        self.lo, self.hi = HEAD + off, HEAD + off + n
        self.t = self.buf[self.lo:self.hi].view(torch.float32)
        if init is not None:
            self.t.copy_(init.reshape(-1))

    def intact(self):
        return bool((self.buf[:self.lo] == SENT).all()) and bool((self.buf[self.hi:] == SENT).all())


def _case(**kw):
    c = dict(G=1, k=1, dil=1, highway=0, eps=1e-5, momentum=0.1, p=0.5, stage=0, gen=False, training=1)
    c.update(kw)
    if c['stage'] == 2:
        c['Cin'] = c['Cout']
    return c


def _operands(c, seed, mode='fp32'):
    g = torch.Generator().manual_seed(seed)
    NB, G, Cin, Cout, L, k = (c[n] for n in ('NB', 'G', 'Cin', 'Cout', 'L', 'k'))
    Ct, Cf = G * Cout, (Cout // 2 if c['highway'] else Cout)
    T = dict(x=torch.randn(NB, G * Cin, L, generator=g), w=torch.randn(Ct, Cin, k, generator=g) / (Cin * k) ** 0.5,
             gamma=1 + 0.3 * torch.randn(Ct, generator=g), beta=0.3 * torch.randn(Ct, generator=g),
             keep=(torch.rand(NB, Ct, L, generator=g) >= c['p']).to(torch.uint8), rm=0.2 * torch.randn(Ct, generator=g),
             rv=0.5 + torch.rand(Ct, generator=g), dout=torch.randn(NB, G * Cf, L, generator=g))
    if mode == 'bf16':        # what the bf16 GEMMs multiply
        T['x'], T['w'] = T['x'].bfloat16().float(), T['w'].bfloat16().float()
    return {n: t.cuda() for n, t in T.items()}


def _run(c, T, off=0, lengths=None, backward=True):
    """Forward (+ backward) through the C ABI on guarded buffers -> (results, {buffer: sentinel intact})."""
    from multilingual_text_to_speech_b200 import _lib, functional as F
    NB, G, Cin, Cout, L = (c[n] for n in ('NB', 'G', 'Cin', 'Cout', 'L'))
    Ct, Cf = G * Cout, (Cout // 2 if c['highway'] else Cout)
    n = NB * Ct * L
    tail = CC.a64(n) - n + 2 * CC.a64(Ct) + 64
    shape = _lib.ConvBlockShape(NB, G, Cin, Cout, L, c['k'], c['dil'], CC.ACTS[c['act']], c['highway'], c['training'], c['eps'],
                                c['momentum'], c['p'], c['stage'])
    lib, sh, st = _lib.load(), ctypes.byref(shape), F._stream()
    saved = F._bytes(lib.b200tts_convblock_saved_bytes(sh), 'cuda')
    ws = F._bytes(lib.b200tts_convblock_workspace_bytes(sh), 'cuda')
    b = dict(x=Guarded(T['x'].numel(), tail, off, T['x']), out=Guarded(NB * G * Cf * L, tail, off),
             rm=Guarded(Ct, tail, 0, T['rm']), rv=Guarded(Ct, tail, 0, T['rv']))
    if c['gen']:            # generated affine [G, 2C]: gamma = aff, beta = aff + C, stride 2C
        b['aff'] = Guarded(2 * Ct, tail, 0, torch.cat([T['gamma'].view(G, Cout), T['beta'].view(G, Cout)], 1))
        gamma, beta, gs = b['aff'].t, b['aff'].t[Cout:], 2 * Cout
    else:
        b['gamma'], b['beta'] = Guarded(Ct, tail, 0, T['gamma']), Guarded(Ct, tail, 0, T['beta'])
        gamma, beta, gs = b['gamma'].t, b['beta'].t, Cout
    w = T['w'] if c['stage'] != 2 else None
    args = (F.ptr(b['x'].t), F.ptr(w), F.ptr(gamma), F.ptr(beta), gs, F.ptr(b['rm'].t), F.ptr(b['rv'].t), F.ptr(T['keep']),
            F.ptr(b['out'].t), F.ptr(saved), F.ptr(ws), st)
    if lengths is None:
        F.check(lib.b200tts_convblock_forward(sh, *args), 'b200tts_convblock_forward')
    else:
        lens = torch.tensor(lengths, dtype=torch.int32, device='cuda')
        F.check(lib.b200tts_convblock_forward_masked(sh, F.ptr(lens), *args), 'b200tts_convblock_forward_masked')
    if backward:
        b['dout'] = Guarded(T['dout'].numel(), tail, off, T['dout'])
        b['dx'] = Guarded(T['x'].numel(), tail, off)
        if w is not None:
            b['dw'] = Guarded(w.numel(), tail, 0, torch.zeros_like(w))
        if c['gen']:
            b['dgb'] = Guarded(2 * Ct, tail, 0, torch.zeros(2 * Ct))
            dg, db = b['dgb'].t, b['dgb'].t[Cout:]
        else:
            b['dgamma'], b['dbeta'] = Guarded(Ct, tail, 0, torch.zeros(Ct)), Guarded(Ct, tail, 0, torch.zeros(Ct))
            dg, db = b['dgamma'].t, b['dbeta'].t
        F.check(lib.b200tts_convblock_backward(sh, F.ptr(b['x'].t), F.ptr(w), F.ptr(gamma), F.ptr(beta), gs, F.ptr(T['keep']),
                                               F.ptr(saved), F.ptr(b['dout'].t), F.ptr(b['dx'].t), F.ptr(b.get('dw') and b['dw'].t),
                                               F.ptr(dg), F.ptr(db), F.ptr(ws), st), 'b200tts_convblock_backward')
    torch.cuda.synchronize()
    sv = saved.view(torch.float32)
    m0, i0 = CC.a64(n), CC.a64(n) + CC.a64(Ct)
    res = dict(out=b['out'].t.view(NB, G * Cf, L).clone(), mean=sv[m0:m0 + Ct].clone(), invstd=sv[i0:i0 + Ct].clone(),
               conv=sv[:n].view(NB, Ct, L).clone() if c['stage'] == 0 else T['x'])
    if c['training']:
        res['rm'], res['rv'] = b['rm'].t.clone(), b['rv'].t.clone()
    if backward:
        res['dx'] = b['dx'].t.view_as(T['x']).clone()
        if w is not None:
            res['dw'] = b['dw'].t.view_as(w).clone()
        if c['gen']:
            full = b['dgb'].t.view(G, 2 * Cout)
            res['dgamma'], res['dbeta'] = full[:, :Cout].reshape(-1).clone(), full[:, Cout:].reshape(-1).clone()
        else:
            res['dgamma'], res['dbeta'] = b['dgamma'].t.clone(), b['dbeta'].t.clone()
    return res, {name: g.intact() for name, g in b.items()}


def _check(c, T, res, mode, title):
    """res against the fp64 epilogue of its own product; returns the worst err / bound per quantity."""
    d = {n: t.double() for n, t in T.items()}
    keep = d['keep'] if c['training'] and c['p'] > 0 else None
    conv = res['conv'].double()
    R = CC.epilogue(c, conv, d['gamma'], d['beta'], keep=keep, xin=d['x'], rm=d['rm'], rv=d['rv'], dout=d['dout'])
    K = dict(mean=res['mean'].double(), invstd=res['invstd'].double())
    B = CC.bounds(c, R, K, conv, d['gamma'], d['beta'], keep=keep, xin=d['x'], rm=d['rm'], rv=d['rv'], dout=d['dout'], x=d['x'],
                  w=d['w'], mode=mode)
    ref = dict(out=R['out'], mean=R['mean'], invstd=1.0 / torch.sqrt(R['var'] + c['eps']), dgamma=R['dgamma'], dbeta=R['dbeta'])
    if c['training']:
        ref['rm'], ref['rv'] = R['rm'], R['rv']
    if c['stage'] == 0:
        dx, ref['dw'] = CC.conv_transposes(d['x'], d['w'], c['G'], c['dil'], R['dconv'])
        ref['dx'] = dx + R['dskip'] if c['highway'] else dx
    else:
        ref['dx'] = R['dconv']
    rep = CC.report(res, ref, B)
    print('\n'.join(CC.worst_lines(title, rep)))
    assert not CC.failures(rep), (title, CC.failures(rep))
    return rep


def _intact(guards, what):
    broken = [name for name, ok in guards.items() if not ok]
    assert not broken, f'{what}: sentinel overwritten around {broken}'


def _same(a, b, what):
    for q in a:
        if torch.is_tensor(a[q]):
            assert torch.equal(a[q], b[q]), f'{what}: {q} differs'


def _with_precision(mode, fn):
    from multilingual_text_to_speech_b200 import _lib
    _lib.set_precision(mode)
    try:
        return fn()
    finally:
        _lib.set_precision('fp32')


ENC = dict(NB=6, G=10, L=180, eps=1e-8, gen=True)
POST = dict(NB=60, G=1, L=900, k=5)
REAL = {
    'enc_vanilla': _case(NB=64, Cin=512, Cout=512, L=180, k=5, act='relu'),
    'gen_in_k1': _case(**ENC, Cin=512, Cout=256, act='relu'),
    'gen_k1': _case(**ENC, Cin=256, Cout=256, act='identity'),
    'gen_highway_k3_dil27': _case(**ENC, Cin=256, Cout=512, k=3, dil=27, act='identity', highway=1),
    'gen_highway_k1': _case(**ENC, Cin=256, Cout=512, act='identity', highway=1),
    'post_in': _case(**POST, Cin=80, Cout=512, act='tanh'),
    'post_mid': _case(**POST, Cin=512, Cout=512, act='tanh'),
    'post_out': _case(**POST, Cin=512, Cout=80, act='identity'),
}


@pytest.mark.parametrize('training', [1, 0], ids=['train', 'eval'])
@pytest.mark.parametrize('mode', ['fp32', 'bf16'])
@pytest.mark.parametrize('name', list(REAL))
def test_block_real_shapes(name, mode, training):
    c = dict(REAL[name], training=training)
    T = _operands(c, sum(map(ord, name)) + training, mode)
    (r1, g1), (r2, g2) = (_with_precision(mode, lambda: _run(c, T)) for _ in range(2))
    _intact(g1, name)
    _intact(g2, name)
    _same(r1, r2, f'{name} {mode} run-to-run')
    _check(c, T, r1, mode, f'{name} {mode} {"train" if training else "eval"}')


@pytest.mark.parametrize('gen', [False, True], ids=['gstride_C', 'gstride_2C'])
@pytest.mark.parametrize('keep', [False, True], ids=['no_keep', 'keep'])
@pytest.mark.parametrize('act', list(CC.ACTS))
@pytest.mark.parametrize('training', [1, 0], ids=['train', 'eval'])
def test_stage2_batch_norm_only(training, act, keep, gen):
    """BatchNorm1dGenerated: the input is the pre-batch-norm tensor; d x is d conv."""
    c = _case(stage=2, NB=6, G=10, Cout=64, L=180, act=act, training=training, gen=gen, eps=1e-8 if gen else 1e-5,
              p=0.5 if keep else 0.0)
    T = _operands(c, 100 + 8 * training + 2 * keep + gen)
    res, guards = _run(c, T)
    _intact(guards, 'stage 2')
    _check(c, T, res, 'fp32', f'stage2 {act} keep={keep} gen={gen} {"train" if training else "eval"}')


PATH_CASES = {
    'plain': dict(NB=5, G=2, Cin=32, Cout=48, k=3, dil=2, act='relu'),
    'highway': dict(NB=5, G=2, Cin=32, Cout=64, k=3, dil=1, act='identity', highway=1, gen=True, eps=1e-8),
    'stage2': dict(NB=5, G=3, Cout=40, act='tanh', stage=2, gen=True, eps=1e-8),
}
VARIANTS = {'float4': (64, 0), 'L_odd': (63, 0), 'offset_by_one': (64, 1)}


@pytest.mark.parametrize('variant', list(VARIANTS))
@pytest.mark.parametrize('kind', list(PATH_CASES))
def test_paths(kind, variant):
    """Train and eval on the float4 and on the scalar kernels; eval forward of the two paths bitwise equal on the same data."""
    L, off = VARIANTS[variant]
    for training in (1, 0):
        c = _case(**PATH_CASES[kind], L=L, training=training)
        T = _operands(c, 7 + training)
        res, guards = _run(c, T, off=off)
        _intact(guards, f'{kind} {variant} training={training}')
        _check(c, T, res, 'fp32', f'{kind} {variant} {"train" if training else "eval"}')
        if variant == 'offset_by_one' and not training:
            vec, _ = _run(c, T, off=0, backward=False)
            assert torch.equal(vec['out'], res['out']), 'eval forward: the float4 and scalar epilogues differ'


MASKED = {
    'plain': _case(NB=6, Cin=64, Cout=64, L=180, k=5, act='relu', training=0),
    'highway': _case(NB=6, Cin=32, Cout=64, L=180, k=3, dil=3, act='identity', highway=1, training=0),
    'generated': _case(NB=6, G=2, Cin=64, Cout=64, L=180, k=3, act='relu', gen=True, eps=1e-8, training=0),
}


@pytest.mark.parametrize('mode', ['fp32', 'bf16'])
@pytest.mark.parametrize('name', list(MASKED))
def test_masked_eval(name, mode):
    """b200tts_convblock_forward_masked on a zero-padded batch with lengths L, 1, 4q + 1 / 2 / 3 and 4q: each sample against the fp64
    block run on its own prefix, exact zeros past the length, and bitwise equal to the unmasked forward inside the lengths (and
    everywhere when every length is L)."""
    c = MASKED[name]
    lengths = [180, 1, 97, 98, 99, 100]
    T = _operands(c, 31, mode)
    T['x'] = T['x'] * (torch.arange(c['L'], device='cuda')[None, :] < torch.tensor(lengths, device='cuda')[:, None])[:, None, :]
    masked, g1 = _with_precision(mode, lambda: _run(c, T, lengths=lengths, backward=False))
    plain, g2 = _with_precision(mode, lambda: _run(c, T, backward=False))
    full, g3 = _with_precision(mode, lambda: _run(c, T, lengths=[c['L']] * c['NB'], backward=False))
    for g in (g1, g2, g3):
        _intact(g, f'masked {name}')
    assert torch.equal(full['out'], plain['out']), 'every length L: not bit-identical to the unmasked forward'
    inside = (torch.arange(c['L'], device='cuda')[None, :] < torch.tensor(lengths, device='cuda')[:, None])[:, None, :]
    assert torch.equal(torch.where(inside, plain['out'], torch.zeros_like(plain['out'])), masked['out'])
    d = {n: t.double() for n, t in T.items()}
    K = dict(mean=masked['mean'].double(), invstd=masked['invstd'].double())
    ref, bnd = CC.masked_reference(c, d['x'], d['w'], d['gamma'], d['beta'], d['rm'], d['rv'], K, lengths, mode)
    rep = CC.report(dict(out=masked['out']), dict(out=ref), dict(out=bnd))
    print('\n'.join(CC.worst_lines(f'masked {name} {mode}', rep)))
    assert not CC.failures(rep)


@pytest.mark.parametrize('training', [1, 0], ids=['train', 'eval'])
@pytest.mark.parametrize('NB,G,L', [(6, 10, 180), (60, 1, 900)])
def test_ill_conditioned_channels(NB, G, L, training):
    """Stage 2, generated affine (eps 1e-8), ReLU, keep mask: channel 0 has mean 1e3 x its spread (a one-pass variance fails it),
    channel 1 is constant (variance 0 at eps 1e-8: out = relu(beta) exactly), channel 2's ReLU is dead everywhere (out and
    d conv exactly 0)."""
    c = _case(stage=2, NB=NB, G=G, Cout=8, L=L, act='relu', gen=True, eps=1e-8, training=training)
    T = _operands(c, 55 + training)
    x = T['x'].view(NB, G, 8, L)
    x[:, :, 0] += 1000.0
    x[:, :, 1] = 0.75
    T['beta'].view(G, 8)[:, 1] = 0.25
    T['beta'].view(G, 8)[:, 2] = -50.0
    T['gamma'].view(G, 8)[:, 2] = 1.0
    if not training:       # running statistics of the same data
        T['rm'].copy_(x.mean((0, 3)).reshape(-1))
        T['rv'].copy_(x.var((0, 3)).reshape(-1))
    res, guards = _run(c, T)
    _intact(guards, 'ill-conditioned')
    _check(c, T, res, 'fp32', f'ill-conditioned NB={NB} G={G} L={L} {"train" if training else "eval"}')
    out, dx = res['out'].view(NB, G, 8, L), res['dx'].view(NB, G, 8, L)
    keep = T['keep'].view(NB, G, 8, L).float() * 2.0 if training else torch.ones_like(out)
    if training:
        assert torch.equal(out[:, :, 1], 0.25 * keep[:, :, 1]), 'constant channel'
    assert torch.equal(out[:, :, 2], torch.zeros_like(out[:, :, 2])), 'dead ReLU channel: output'
    assert torch.equal(dx[:, :, 2], torch.zeros_like(dx[:, :, 2])), 'dead ReLU channel: d conv'
