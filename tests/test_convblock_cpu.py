"""The conv block's fp64 reference and bound checker (tests/convblock_check.py) without a GPU.

1. The reference composed from the oracle's pieces equals torch.nn.Conv1d + BatchNorm1d (+ activation, dropout mask, highway gate)
   modules in fp64: outputs, running statistics and every gradient.  This pins it to torch as well as to the oracle.
2. A result that is the fp32 rounding of the reference passes the bounds, and each kernel-style mutation of it is flagged.
"""
import pytest
import torch

import convblock_check as CC
from oracle import tacotron_oracle as O

D = torch.float64

PLAIN = dict(NB=3, G=1, Cin=6, Cout=8, L=13, k=5, dil=1, highway=0, eps=1e-5, momentum=0.1, p=0.5, stage=0)
GEN_HW = dict(NB=4, G=2, Cin=4, Cout=8, L=12, k=3, dil=2, highway=1, eps=1e-8, momentum=0.1, p=0.5, stage=0, act='identity')


def _operands(c, seed):
    g = torch.Generator().manual_seed(seed)
    NB, G, Cin, Cout, L, k = (c[n] for n in ('NB', 'G', 'Cin', 'Cout', 'L', 'k'))
    Ct = G * Cout
    return dict(x=torch.randn(NB, G * Cin, L, generator=g, dtype=D), w=torch.randn(Ct, Cin, k, generator=g, dtype=D) / (Cin * k) ** 0.5,
                gamma=1 + 0.3 * torch.randn(Ct, generator=g, dtype=D), beta=0.3 * torch.randn(Ct, generator=g, dtype=D),
                keep=(torch.rand(NB, Ct, L, generator=g, dtype=D) > c['p']).double(), rm=(0.2 * torch.randn(Ct, generator=g, dtype=D)).float().double(),
                rv=(0.5 + torch.rand(Ct, generator=g, dtype=D)).float().double(),
                dout=torch.randn(NB, G * (Cout // 2 if c['highway'] else Cout), L, generator=g, dtype=D))


def _torch_modules(c, T):
    """The same block from torch.nn modules: (out, running mean, running var, dx, dw, dgamma, dbeta)."""
    G, Cin, Cout, k, dil = (c[n] for n in ('G', 'Cin', 'Cout', 'k', 'dil'))
    conv = torch.nn.Conv1d(G * Cin, G * Cout, k, padding=(k - 1) * dil // 2, dilation=dil, groups=G, bias=False).double()
    bn = torch.nn.BatchNorm1d(G * Cout, eps=c['eps'], momentum=c['momentum']).double()
    with torch.no_grad():
        conv.weight.copy_(T['w'])
        bn.weight.copy_(T['gamma'])
        bn.bias.copy_(T['beta'])
        bn.running_mean.copy_(T['rm'])
        bn.running_var.copy_(T['rv'])
    bn.train(bool(c['training']))
    x = T['x'].clone().requires_grad_(True)
    act = {'identity': torch.nn.Identity(), 'relu': torch.nn.ReLU(), 'tanh': torch.nn.Tanh()}[c['act']]
    y = act(bn(conv(x)))
    if c['training']:
        y = y * T['keep'] / (1 - c['p'])
    if c['highway']:
        v = y.view(y.shape[0], G, 2, Cout // 2, -1)
        s = torch.sigmoid(v[:, :, 0]).flatten(1, 2)
        y = v[:, :, 1].flatten(1, 2) * s + x * (1 - s)
    y.backward(T['dout'])
    return dict(out=y.detach(), rm=bn.running_mean, rv=bn.running_var, dx=x.grad, dw=conv.weight.grad, dgamma=bn.weight.grad,
                dbeta=bn.bias.grad)


def _reference(c, T, **kw):
    conv = CC.conv_groups(T['x'], T['w'], c['G'], c['dil'])
    R = CC.epilogue(c, conv, T['gamma'], T['beta'], keep=T['keep'], xin=T['x'], rm=T['rm'], rv=T['rv'], dout=T['dout'], **kw)
    dx, dw = CC.conv_transposes(T['x'], T['w'], c['G'], c['dil'], R['dconv'])
    R['dx'] = dx + R['dskip'] if c['highway'] else dx
    R['dw'] = dw
    return conv, R


@pytest.mark.parametrize('training', [1, 0])
@pytest.mark.parametrize('base,act', [(PLAIN, 'relu'), (PLAIN, 'tanh'), (PLAIN, 'identity'), (GEN_HW, 'identity')])
def test_reference_equals_torch_modules(base, act, training):
    c = dict(base, act=act, training=training)
    T = _operands(c, 7 + training)
    _, R = _reference(c, T)
    M = _torch_modules(c, T)
    if not training:
        R['rm'], R['rv'] = T['rm'], T['rv']
    for q in ('out', 'rm', 'rv', 'dx', 'dw', 'dgamma', 'dbeta'):
        torch.testing.assert_close(R[q], M[q], rtol=1e-12, atol=1e-12, msg=q)


def _kernel_like(c, T, K=None):
    """The reference, the bounds and a result that is the reference rounded to fp32 (what a correct kernel could return)."""
    conv, R = _reference(c, T)
    f32 = lambda t: t.float().double()          # noqa: E731
    K = K or dict(mean=f32(R['mean']), invstd=f32(1.0 / torch.sqrt(R['var'] + c['eps'])))
    B = CC.bounds(c, R, K, conv, T['gamma'], T['beta'], keep=T['keep'], xin=T['x'], rm=T['rm'], rv=T['rv'], dout=T['dout'],
                  x=T['x'], w=T['w'])
    got = {q: f32(R[q]) for q in ('out', 'dx', 'dw', 'dgamma', 'dbeta') + (('rm', 'rv') if c['training'] else ())}
    got.update(K)
    ref = dict(R, invstd=1.0 / torch.sqrt(R['var'] + c['eps']))
    return conv, R, B, got, ref


def _flagged(got, ref, B, what):
    rep = CC.report(got, ref, B)
    print('\n'.join(CC.worst_lines(what, rep)))
    return set(CC.failures(rep))


@pytest.mark.parametrize('training', [1, 0])
@pytest.mark.parametrize('base,act', [(PLAIN, 'relu'), (PLAIN, 'tanh'), (GEN_HW, 'identity')])
def test_fp32_rounded_reference_passes(base, act, training):
    c = dict(base, act=act, training=training)
    T = _operands(c, 11)
    _, _, B, got, ref = _kernel_like(c, T)
    assert _flagged(got, ref, B, 'fp32(reference)') == set()


def test_flags_biased_running_var():
    c = dict(PLAIN, act='relu', training=1)
    T = _operands(c, 1)
    _, R, B, got, ref = _kernel_like(c, T)
    got['rv'] = ((1 - c['momentum']) * T['rv'] + c['momentum'] * R['var']).float().double()
    assert 'rv' in _flagged(got, ref, B, 'biased running_var')


def test_flags_missing_dropout_scale():
    c = dict(PLAIN, act='relu', training=1)
    T = _operands(c, 2)
    conv, R, B, got, ref = _kernel_like(c, T)
    got['out'] = CC.epilogue(c, conv, T['gamma'], T['beta'], keep=T['keep'], rm=T['rm'], rv=T['rv'], scale=1.0)['out'].float().double()
    assert 'out' in _flagged(got, ref, B, 'no 1/(1-p)')


def test_flags_swapped_highway_halves():
    c = dict(GEN_HW, training=1)
    T = _operands(c, 3)
    conv, R, B, got, ref = _kernel_like(c, T)
    got['out'] = CC.epilogue(c, conv, T['gamma'], T['beta'], keep=T['keep'], xin=T['x'], rm=T['rm'], rv=T['rv'],
                             swap_highway=True)['out'].float().double()
    assert 'out' in _flagged(got, ref, B, 'highway halves swapped')


def test_flags_gamma_read_at_stride_c():
    """Generated affine [G, 2C]: gamma (g, o) is aff[g, o] at stride 2C.  Read at stride C, groups past the first get beta / the
    wrong group's gamma."""
    c = dict(GEN_HW, training=1)
    T = _operands(c, 4)
    G, C = c['G'], c['Cout']
    aff = torch.cat([T['gamma'].view(G, C), T['beta'].view(G, C)], 1)
    conv, R, B, got, ref = _kernel_like(c, T)
    wrong = aff.reshape(-1)[:G * C]
    got['out'] = CC.epilogue(c, conv, wrong, T['beta'], keep=T['keep'], xin=T['x'], rm=T['rm'], rv=T['rv'])['out'].float().double()
    assert 'out' in _flagged(got, ref, B, 'gamma at stride C')


def test_flags_eval_backward_with_batch_statistics():
    c = dict(PLAIN, act='tanh', training=0)
    T = _operands(c, 5)
    conv, R, B, got, ref = _kernel_like(c, T)
    ct = dict(c, training=1, p=0.0)          # the train-mode gradient formula (batch statistics), no dropout as in eval
    Rt = CC.epilogue(ct, conv, T['gamma'], T['beta'], rm=T['rm'], rv=T['rv'], dout=T['dout'])
    dx, dw = CC.conv_transposes(T['x'], T['w'], c['G'], c['dil'], Rt['dconv'])
    got.update(dx=dx.float().double(), dw=dw.float().double(), dgamma=Rt['dgamma'].float().double(), dbeta=Rt['dbeta'].float().double())
    assert {'dx', 'dw', 'dgamma'} <= _flagged(got, ref, B, 'eval backward with batch stats')


@pytest.mark.parametrize('base', [PLAIN, GEN_HW])
def test_flags_float4_lane_past_length(base):
    """Masked eval: the lane just past a length 4q + 1 left with the unmasked value (a float4 group straddling the length)."""
    c = dict(base, act=base.get('act', 'relu'), training=0, L=16)
    T = _operands(c, 6)
    lengths = torch.tensor([16, 1, 9, 10, 11][:c['NB']])
    x = T['x'] * (torch.arange(c['L'])[None, :] < lengths[:, None])[:, None, :]
    K = dict(mean=T['rm'], invstd=(1.0 / torch.sqrt(T['rv'] + c['eps'])).float().double())
    ref, bnd = CC.masked_reference(c, x, T['w'], T['gamma'], T['beta'], T['rm'], T['rv'], K, lengths, 'fp32')
    ok = CC.report(dict(out=ref.float().double()), dict(out=ref), dict(out=bnd))
    assert CC.failures(ok) == {}
    full = CC.epilogue(c, CC.conv_groups(x, T['w'], c['G'], c['dil']), T['gamma'], T['beta'], xin=x, rm=T['rm'], rv=T['rv'])['out']
    got = ref.clone()
    got[2, :, 9] = full[2, :, 9]            # length 9 = 4 * 2 + 1: lane 1 of the group at 8
    assert float(got[2, :, 9].abs().max()) > 0
    assert 'out' in _flagged(dict(out=got.float().double()), dict(out=ref), dict(out=bnd), 'float4 lane past the length')


def test_sum_bound_covers_a_shifted_channel_but_not_one_pass_variance():
    """A channel of mean 1e3 x its spread: the two-pass variance of fp32 values stays inside the bound; the one-pass
    E[x^2] - E[x]^2 in fp32 does not."""
    g = torch.Generator().manual_seed(9)
    NB, L = 6, 180
    x32 = (1000.0 + torch.randn(NB, 1, L, generator=g)).float()
    x = x32.double()
    c = dict(NB=NB, G=1, Cin=1, Cout=1, L=L, k=1, dil=1, act='identity', highway=0, training=1, eps=1e-8, momentum=0.1, p=0.0,
             stage=2)
    R = CC.epilogue(c, x, torch.ones(1, dtype=D), torch.zeros(1, dtype=D), rm=torch.zeros(1, dtype=D), rv=torch.ones(1, dtype=D))
    is_ = 1.0 / torch.sqrt(R['var'] + c['eps'])
    mu1 = x32.sum() / (NB * L)
    one_pass = (x32 * x32).sum() / (NB * L) - mu1 * mu1
    mu2 = x32.mean()
    two_pass = ((x32 - mu2) ** 2).mean()
    for var, expect in ((two_pass, set()), (one_pass, {'invstd'})):
        K = dict(mean=mu2.double().view(1), invstd=(1.0 / torch.sqrt(var.double().clamp(min=0) + c['eps'])).view(1))
        B = CC.bounds(c, R, K, x, torch.ones(1, dtype=D), torch.zeros(1, dtype=D), rm=torch.zeros(1, dtype=D), rv=torch.ones(1, dtype=D))
        rep = CC.report(dict(mean=K['mean'], invstd=K['invstd']), dict(mean=R['mean'], invstd=is_), B)
        assert set(CC.failures(rep)) == expect, rep

