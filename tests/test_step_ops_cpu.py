"""The fp64 oracle of the per-step ops (tests/step_ops_check.py) without a GPU.

- It matches fp64 torch autograd of the reference formulas (location-sensitive and forward attention, zoneout / dropout LSTM cell)
  to 1e-12.
- Its bounds have power: an fp64 simulation laid out like each kernel (position chunks, the dF / accW tiles, the clamp gate),
  rounded to fp32, passes them, and each of a set of kernel-style mistakes falls outside them on at least one element.
- The attention backward's chunk size export, and the host-side argument checks of the step ABIs.
"""
import ctypes
import math

import pytest
import torch
import torch.nn.functional as Fn

import step_check as S
import step_ops_check as O

D64 = torch.float64


# ------------------------------------------------------------------------------------------------------------------------
# inputs
# ------------------------------------------------------------------------------------------------------------------------
def _loc_inputs(B=3, L=40, M=24, A=16, C=8, K=5, seed=0, lens=None):
    g = torch.Generator().manual_seed(seed)
    r = lambda *s, scale=1.0: (torch.randn(*s, generator=g, dtype=D64) * scale).float()    # noqa: E731
    if lens is None:
        lens = torch.randint(1, L + 1, (B,), generator=g)
        lens[0], lens[-1] = L, 1
    lens = torch.as_tensor(lens, dtype=torch.int32)
    valid = torch.arange(L)[None, :] < lens[:, None].long()
    cum = torch.zeros(B, L, dtype=D64)
    for _ in range(3):
        cum += torch.softmax((torch.randn(B, L, generator=g, dtype=D64) * 3).masked_fill(~valid, -math.inf), -1).masked_fill(~valid, 0)
    return {'q': r(B, A), 'memT': r(B, L, A, scale=0.5), 'memory': r(B, L, M), 'Wloc': r(A, C, scale=C ** -0.5),
            'Wc': r(C, 1, K, scale=K ** -0.5), 'bias': r(1, A, scale=0.1), 'v': r(1, A, scale=6 * A ** -0.5), 'cum': cum.float(),
            'd_ctx': r(B, M, scale=0.1), 'd_w': r(B, L, scale=0.1), 'd_cum': r(B, L, scale=0.1), 'lens': lens}


def _loc_prm(x):
    return {'attn_location': x['Wloc'], 'attn_loc_features': x['Wc'], 'attn_bias': x['bias'], 'attn_energy': x['v']}


def _fwd_inputs(B=3, L=30, M=24, A=16, seed=0, alpha='peaked'):
    g = torch.Generator().manual_seed(seed)
    r = lambda *s, scale=1.0: (torch.randn(*s, generator=g, dtype=D64) * scale).float()    # noqa: E731
    lens = torch.randint(1, L + 1, (B,), generator=g)
    lens[0], lens[-1] = L, 1
    al = torch.zeros(B, L)
    al[:, 0] = 1
    if alpha == 'peaked':       # mass on the first few positions: most products sit on the floor
        al[:, :4] = torch.tensor([0.5, 0.3, 0.15, 0.05])[:min(4, L)]
    elif alpha == 'uniform':
        al.fill_(1.0 / L)
    return {'q': r(B, A), 'memT': r(B, L, A, scale=0.5), 'memory': r(B, L, M), 'bias': r(1, A, scale=0.1),
            'v': r(1, A, scale=6 * A ** -0.5), 'alpha': al, 'd_ctx': r(B, M, scale=0.1), 'd_w': r(B, L, scale=0.1),
            'd_alpha': r(B, L, scale=0.1), 'lens': lens.to(torch.int32)}


def _cell_inputs(B=5, D=33, kind=1, training=True, rate=0.1, seed=0):
    g = torch.Generator().manual_seed(seed)
    z = (torch.randn(B, 4 * D, generator=g, dtype=D64) * 4).float()
    z.view(-1)[::7] = 20.0
    mh = (torch.rand(B, D, generator=g) >= rate).to(torch.uint8)
    mc = (torch.rand(B, D, generator=g) >= rate).to(torch.uint8) if kind == 1 else None
    return {'z': z, 'hp': torch.randn(B, D, generator=g), 'cp': torch.randn(B, D, generator=g) * 2, 'mh': mh, 'mc': mc,
            'dh': torch.randn(B, D, generator=g), 'dc': torch.randn(B, D, generator=g),
            'cfg': S.Config(kind, training, rate, rate if kind == 1 else 0.0)}


def _close(got, want, what):
    scale = max(float(want.abs().max()), 1e-300)
    assert float((got - want).abs().max()) <= 1e-12 * scale, (what, float((got - want).abs().max()), scale)


# ------------------------------------------------------------------------------------------------------------------------
# the oracle against torch autograd of the reference formulas
# ------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('dims', [dict(L=40, K=5), dict(L=3, K=7), dict(L=17, A=4, C=4, K=1)], ids=('L40', 'L_below_K', 'K1'))
def test_location_oracle_matches_autograd(dims):
    x = _loc_inputs(**dims)
    B, L = x['cum'].shape
    C, _, K = x['Wc'].shape
    leaves = {k: x[k].double().clone().requires_grad_(True) for k in ('q', 'memT', 'Wloc', 'Wc', 'v', 'cum')}
    mask = torch.arange(L)[None, :] < x['lens'][:, None].long()
    loc = Fn.conv1d(leaves['cum'][:, None, :], leaves['Wc'], padding=(K - 1) // 2).transpose(1, 2) @ leaves['Wloc'].t()
    energy = torch.tanh(leaves['q'][:, None, :] + leaves['memT'] + loc + x['bias'].double()) @ leaves['v'].reshape(-1)
    w = torch.softmax(energy.masked_fill(~mask, -math.inf), 1)
    ctx = torch.bmm(w[:, None, :], x['memory'].double()).squeeze(1)
    cum_next = leaves['cum'] + w
    (ctx * x['d_ctx'].double()).sum().add((w * x['d_w'].double()).sum()).add((cum_next * x['d_cum'].double()).sum()).backward()
    prm = _loc_prm(x)
    f = O.location_forward(x['q'].double(), x['cum'].double(), x['memT'], x['memory'], x['lens'], prm, w.detach())
    _close(f['weights'][0], w.detach(), 'weights')
    _close(f['context'][0], ctx.detach(), 'context')
    b = O.location_backward(x['q'], x['cum'], x['memT'], x['memory'], x['lens'], prm, w.detach(), x['d_ctx'], x['d_w'], x['d_cum'])
    for name, leaf in (('d_q', 'q'), ('d_memT', 'memT'), ('d_Wloc', 'Wloc'), ('d_Wc', 'Wc'), ('d_v', 'v'), ('d_cum', 'cum')):
        _close(b[name][0].reshape(leaves[leaf].grad.shape), leaves[leaf].grad, name)


@pytest.mark.parametrize('alpha', ('reset', 'peaked', 'uniform'))
def test_forward_attention_oracle_matches_autograd(alpha):
    x = _fwd_inputs(alpha=alpha)
    B, L = x['alpha'].shape
    leaves = {k: x[k].double().clone().requires_grad_(True) for k in ('q', 'memT', 'v', 'alpha')}
    mask = torch.arange(L)[None, :] < x['lens'][:, None].long()
    e = torch.tanh(leaves['q'][:, None, :] + leaves['memT'] + x['bias'].double()) @ leaves['v'].reshape(-1)
    s = torch.softmax(e, 1)
    a = (leaves['alpha'] + Fn.pad(leaves['alpha'], (1, 0))[:, :-1]) * s
    a = a.masked_fill(~mask, 0.0)
    w = Fn.normalize(torch.clamp(a, O.FLOOR), p=1)
    ctx = torch.bmm(w[:, None, :], x['memory'].double()).squeeze(1)
    (ctx * x['d_ctx'].double()).sum().add((w * (x['d_w'].double() + x['d_alpha'].double())).sum()).backward()
    prm = {'attn_bias': x['bias'], 'attn_energy': x['v']}
    f = O.forward_forward(x['q'], x['alpha'], x['memT'], x['memory'], x['lens'], prm, w.detach())
    _close(f['weights'][0], w.detach(), 'weights')
    _close(f['context'][0], ctx.detach(), 'context')
    b = O.forward_backward(x['q'], x['alpha'], x['memT'], x['memory'], x['lens'], prm, w.detach(), x['d_ctx'], x['d_w'], x['d_alpha'])
    for name, leaf in (('d_q', 'q'), ('d_memT', 'memT'), ('d_v', 'v'), ('d_alpha', 'alpha')):
        _close(b[name][0].reshape(leaves[leaf].grad.shape), leaves[leaf].grad, name)


@pytest.mark.parametrize('kind', (0, 1))
@pytest.mark.parametrize('training', (True, False))
def test_cell_oracle_matches_autograd(kind, training):
    x = _cell_inputs(kind=kind, training=training)
    cfg = x['cfg']
    D = x['hp'].shape[1]
    z, hp, cp = (x[k].double().clone().requires_grad_(True) for k in ('z', 'hp', 'cp'))
    gi, gf, gg, go = torch.sigmoid(z[:, :D]), torch.sigmoid(z[:, D:2 * D]), torch.tanh(z[:, 2 * D:3 * D]), torch.sigmoid(z[:, 3 * D:])
    cn = gf * cp + gi * gg
    hn = go * torch.tanh(cn)
    if kind == 1 and training:
        h = (1 - cfg.rate_h) * ((hn - hp) * x['mh'].double() / (1 - cfg.rate_h)) + hp
        c = (1 - cfg.rate_c) * ((cn - cp) * x['mc'].double() / (1 - cfg.rate_c)) + cp
    elif kind == 1:
        h, c = cfg.rate_h * hp + (1 - cfg.rate_h) * hn, cfg.rate_c * cp + (1 - cfg.rate_c) * cn
    else:
        h, c = (hn * x['mh'].double() / (1 - cfg.rate_h) if training else hn), cn
    (h * x['dh'].double()).sum().add((c * x['dc'].double()).sum()).backward()
    gates = torch.cat([gi, gf, gg, go], 1).detach()
    f = O.cell_fwd(x['z'], x['hp'], x['cp'], x['mh'], x['mc'], cfg, gates)
    _close(f['gates'][0], gates, 'gates')
    _close(f['h'][0], h.detach(), 'h')
    _close(f['c'][0], c.detach(), 'c')
    b = O.cell_bwd(gates, x['cp'], x['mh'], x['mc'], x['dh'], x['dc'], cfg)
    _close(b['d_gates'][0], z.grad, 'd_gates')
    _close(b['d_c'][0], cp.grad, 'd_c')
    if kind == 1:
        _close(b['d_h_prev'][0], hp.grad, 'd_h_prev')
    else:
        assert hp.grad is None or float(hp.grad.abs().max()) == 0 and float(b['d_h_prev'][0].abs().max()) == 0


# ------------------------------------------------------------------------------------------------------------------------
# fp64 simulations laid out like the kernels, with switchable mistakes
# ------------------------------------------------------------------------------------------------------------------------
def sim_location(x, LC, mut=()):
    """attn_fwd_kernel, then attn_bwd_kernel (position chunks of LC rows, dF / accW / dWc / d cum as the kernel forms them) and the
    batch sums, in fp64.  The backward reads the forward's weights rounded to fp32, as the ABI passes them."""
    q, memT, mem, cum = (x[k].double() for k in ('q', 'memT', 'memory', 'cum'))
    Wl, v, bias = x['Wloc'].double(), x['v'].double().reshape(-1), x['bias'].double().reshape(-1)
    C, _, K = x['Wc'].shape
    Wc = x['Wc'].double().reshape(C, K)
    B, L = cum.shape
    A = Wl.shape[0]
    half = (K - 1) // 2
    Lp = (L + 3) // 4 * 4
    cp2 = Fn.pad(cum, (half + 1, K - half + Lp - L))               # cp2[j] = cum[j - half - 1]

    def window(shift):                                           # [B, Lp, K]: cum[l + k - half + shift], zero padded
        return cp2.unfold(-1, K, 1)[:, 1 + shift:1 + shift + Lp]
    lens = x['lens'].long()
    out = {k: [] for k in ('weights', 'context', 'cum', 'd_q', 'd_memT', 'd_cum', 'd_Wloc', 'd_Wc', 'd_v')}
    for b in range(B):
        n = int(lens[b])
        f = window(1 if 'conv tap' in mut else 0)[b] @ Wc.t()               # [Lp, C]
        th = torch.tanh(f @ Wl.t() + q[b] + bias + Fn.pad(memT[b], (0, 0, 0, Lp - L)))   # [Lp, A]
        e = th @ v
        ns = min(L, max(1, n + (1 if 'softmax len+1' in mut else -1 if 'softmax len-1' in mut else 0)))
        w = torch.zeros(Lp, dtype=D64)
        w[:ns] = torch.softmax(e[:ns], 0)
        out['weights'].append(w[:L])
        out['cum'].append(cum[b] + w[:L])
        out['context'].append(w[:L] @ mem[b])
        # backward, from the fp32 weights of the correct forward
        wk = torch.zeros(Lp, dtype=D64)
        wk[:L] = (x['w32'][b] if 'w32' in x else w[:L].float()).double()
        f = window(0)[b] @ Wc.t()
        th = torch.tanh(f @ Wl.t() + q[b] + bias + Fn.pad(memT[b], (0, 0, 0, Lp - L)))
        dw = torch.zeros(Lp, dtype=D64)
        dw[:n] = mem[b, :n] @ x['d_ctx'][b].double() + x['d_cum'][b, :n].double()
        if 'd_weights ignored' not in mut:
            dw[:n] += x['d_w'][b, :n].double()
        de = wk * (dw - (wk * dw).sum())
        de[n:] = 0
        ds = de[:, None] * v * (1 - th * th)
        ds[n:] = 0
        out['d_q'].append(ds.sum(0))
        out['d_memT'].append(ds[:L])
        out['d_v'].append(de @ th)
        dF = torch.zeros(C, Lp, dtype=D64)
        accW = torch.zeros(A, C, dtype=D64)
        for lc0 in range(0, n, LC):
            rows = min(LC, (n - lc0 + 3) // 4 * 4)
            chunk = ds[lc0:lc0 + rows]
            at = 0 if 'dF without lc0' in mut else lc0
            dF[:, at:at + rows] = (chunk @ Wl).t()
            if 'accW reset per chunk' in mut:
                accW = torch.zeros_like(accW)
            accW = accW + chunk.t() @ f[lc0:lc0 + rows]
        out['d_Wloc'].append(accW)
        win = window(1 if 'dWc tap' in mut else 0)[b]
        out['d_Wc'].append(dF[:, :n] @ win[:n])
        conv = torch.zeros(L, dtype=D64)
        dFp = Fn.pad(dF, (K, K))
        for j in range(L):
            for k in range(K):
                conv[j] += dFp[:, K + j + half - k] @ Wc[:, k]
        out['d_cum'].append(conv + (0 if 'd_cum carry lost' in mut else x['d_cum'][b].double()))
    res = {k: torch.stack(t) for k, t in out.items()}
    for k in ('d_Wloc', 'd_Wc', 'd_v'):
        res[k] = res[k].sum(0)
    return {k: t.float() for k, t in res.items()}


def sim_forward_attention(x, mut=()):
    """fwd_attn_fwd_kernel then fwd_attn_bwd_kernel in fp64 (the backward reads the fp32 weights of the correct forward)"""
    q, memT, mem, al = (x[k].double() for k in ('q', 'memT', 'memory', 'alpha'))
    v, bias = x['v'].double().reshape(-1), x['bias'].double().reshape(-1)
    B, L = al.shape
    lens = x['lens'].long()
    th = torch.tanh(q[:, None, :] + bias + memT)
    s = torch.softmax(th @ v, 1)
    valid = torch.arange(L)[None, :] < lens[:, None]
    p = al + (0 if 'alpha[l-1] dropped' in mut else Fn.pad(al, (1, 0))[:, :-1])
    a = (p * s).masked_fill(~valid, 0.0)
    c = a.clamp(min=O.FLOOR)
    den = c.sum(1, keepdim=True)
    w = c / den
    res = {'weights': w, 'context': torch.einsum('bl,blm->bm', w, mem)}
    wk = (x['w32'] if 'w32' in x else w.float()).double()
    g = torch.einsum('blm,bm->bl', mem, x['d_ctx'].double()) + x['d_alpha'].double() + x['d_w'].double()
    gate = valid & ((a >= O.FLOOR) | ('floor gate ignored' in mut))
    da = torch.where(gate, (g - (g * wk).sum(1, keepdim=True)) / den, torch.zeros_like(g))
    res['d_alpha'] = da * s + Fn.pad(da * s, (0, 1))[:, 1:]
    ds = da * p
    de = s * (ds - (s * ds).sum(1, keepdim=True))
    dpre = de[..., None] * v * (1 - th * th)
    res.update(d_q=dpre.sum(1), d_memT=dpre, d_v=torch.einsum('bl,bla->a', de, th))
    return {k: t.float() for k, t in res.items()}


def sim_cell(x, mut=()):
    """lstm_cell_fwd_kernel then lstm_cell_bwd_kernel in fp64 (the backward reads the fp32 gates of the correct forward)"""
    cfg = x['cfg']
    z, hp, cp, dh, dc = (x[k].double() for k in ('z', 'hp', 'cp', 'dh', 'dc'))
    D = hp.shape[1]
    mh = x['mh'].double()
    mc = x['mc'].double() if x['mc'] is not None else None
    gi, gf, gg, go = torch.sigmoid(z[:, :D]), torch.sigmoid(z[:, D:2 * D]), torch.tanh(z[:, 2 * D:3 * D]), torch.sigmoid(z[:, 3 * D:])
    cn = gi * cp + gf * gg if 'i and f swapped' in mut else gf * cp + gi * gg
    hn = go * torch.tanh(cn)
    if cfg.kind == 1:
        if cfg.training:
            h = (1 - cfg.rate_h) * ((hn - hp) * (mc if 'mask_c on h' in mut else mh) / (1 - cfg.rate_h)) + hp
            c = (1 - cfg.rate_c) * ((cn - cp) * mc / (1 - cfg.rate_c)) + cp
        else:
            h, c = cfg.rate_h * hp + (1 - cfg.rate_h) * hn, cfg.rate_c * cp + (1 - cfg.rate_c) * cn
    else:
        h, c = (hn * mh / (1 - cfg.rate_h) if cfg.training else hn), cn
    res = {'gates': torch.cat([gi, gf, gg, go], 1), 'h': h, 'c': c}
    G = (x['g32'] if 'g32' in x else res['gates'].float()).double()
    gi, gf, gg, go = G[:, :D], G[:, D:2 * D], G[:, 2 * D:3 * D], G[:, 3 * D:]
    tc = torch.tanh(gf * cp + gi * gg)
    if cfg.kind == 1:
        kh = (1 - cfg.rate_h) * (mh / (1 - cfg.rate_h)) if cfg.training else 1 - cfg.rate_h
        kc = (1 - cfg.rate_c) * (mc / (1 - cfg.rate_c)) if cfg.training else 1 - cfg.rate_c
        dhn = dh * kh
        dcn = dc * kc + dhn * go * (1 - tc * tc)
        direct = 'zoneout direct terms dropped' not in mut
        dcp, dhp = dcn * gf + (dc - dc * kc) * direct, (dh - dhn) * direct
    else:
        dhn = dh * mh / (1 - cfg.rate_h) if cfg.training else dh
        dcn = dc + dhn * go * (1 - tc * tc)
        dcp, dhp = dcn * gf, torch.zeros_like(dh)
    res['d_gates'] = torch.cat([dcn * gg * gi * (1 - gi), dcn * cp * gf * (1 - gf), dcn * gi * (1 - gg * gg), dhn * tc * go * (1 - go)], 1)
    res.update(d_c=dcp, d_h_prev=dhp)
    return {k: t.float() for k, t in res.items()}


# ------------------------------------------------------------------------------------------------------------------------
# bound power
# ------------------------------------------------------------------------------------------------------------------------
def _ratios(got, refs):
    return {k: O.ratio(got[k], ref, bound)[0] for k, (ref, bound) in refs.items()}


def _location_ratios(x, LC, mut=()):
    prm = _loc_prm(x)
    if 'w32' not in x:
        x['w32'] = sim_location(x, LC)['weights']
    got = sim_location(x, LC, mut)
    refs = O.location_forward(x['q'], x['cum'], x['memT'], x['memory'], x['lens'], prm, got['weights'])
    refs.update(O.location_backward(x['q'], x['cum'], x['memT'], x['memory'], x['lens'], prm, x['w32'], x['d_ctx'], x['d_w'],
                                    x['d_cum']))
    got['d_Wc'] = got['d_Wc'].reshape(refs['d_Wc'][0].shape)
    return _ratios(got, refs)


def _real_dims_case(L, lens):
    """the real attention dims (A = 128, C = 32, K = 31) at M = 16: B = len(lens)"""
    return _loc_inputs(B=len(lens), L=L, M=16, A=128, C=32, K=31, lens=lens, seed=L)


def test_location_simulation_is_within_the_bounds():
    for x, LC in ((_loc_inputs(), 8), (_loc_inputs(L=3, K=7), 4), (_real_dims_case(300, [300, 173, 1]), 172)):
        r = _location_ratios(x, LC)
        assert max(r.values()) <= 1.0, r


LOC_MUTATIONS = [
    ('accW reset per chunk', 'd_Wloc'), ('dF without lc0', 'd_Wc'), ('dF without lc0', 'd_cum'), ('d_cum carry lost', 'd_cum'),
    ('d_weights ignored', 'd_q'), ('conv tap', 'weights'), ('dWc tap', 'd_Wc'), ('softmax len+1', 'weights'),
    ('softmax len-1', 'weights'),
]


@pytest.mark.parametrize('mut, output', LOC_MUTATIONS, ids=[f'{m}->{o}'.replace(' ', '_') for m, o in LOC_MUTATIONS])
def test_location_mutation_is_flagged(mut, output):
    """on the real dims at L = 300, the two-chunk case of the GPU suite (LC = 172), lengths on and across the boundary"""
    x = _real_dims_case(300, [300, 173, 172, 1])
    r = _location_ratios(x, 172, (mut,))
    assert r[output] > 1.0, (mut, output, r)


def _forward_ratios(x, mut=()):
    prm = {'attn_bias': x['bias'], 'attn_energy': x['v']}
    if 'w32' not in x:
        x['w32'] = sim_forward_attention(x)['weights']
    got = sim_forward_attention(x, mut)
    refs = O.forward_forward(x['q'], x['alpha'], x['memT'], x['memory'], x['lens'], prm, got['weights'])
    refs.update(O.forward_backward(x['q'], x['alpha'], x['memT'], x['memory'], x['lens'], prm, x['w32'], x['d_ctx'], x['d_w'],
                                   x['d_alpha']))
    return _ratios(got, refs)


@pytest.mark.parametrize('alpha', ('reset', 'peaked', 'uniform'))
def test_forward_attention_simulation_is_within_the_bounds(alpha):
    r = _forward_ratios(_fwd_inputs(alpha=alpha))
    assert max(r.values()) <= 1.0, r


@pytest.mark.parametrize('mut, output', [('alpha[l-1] dropped', 'weights'), ('floor gate ignored', 'd_alpha')])
def test_forward_attention_mutation_is_flagged(mut, output):
    r = _forward_ratios(_fwd_inputs(alpha='peaked'), (mut,))
    assert r[output] > 1.0, (mut, output, r)


def _cell_ratios(x, mut=()):
    if 'g32' not in x:
        x['g32'] = sim_cell(x)['gates']
    got = sim_cell(x, mut)
    refs = O.cell_fwd(x['z'], x['hp'], x['cp'], x['mh'], x['mc'], x['cfg'], got['gates'])
    refs.update(O.cell_bwd(x['g32'], x['cp'], x['mh'], x['mc'], x['dh'], x['dc'], x['cfg']))
    return _ratios(got, refs)


@pytest.mark.parametrize('kind', (0, 1))
@pytest.mark.parametrize('training', (True, False))
@pytest.mark.parametrize('rate', (0.0, 0.1, 0.5))
def test_cell_simulation_is_within_the_bounds(kind, training, rate):
    r = _cell_ratios(_cell_inputs(kind=kind, training=training, rate=rate))
    assert max(r.values()) <= 1.0, r


@pytest.mark.parametrize('mut, output', [('i and f swapped', 'c'), ('zoneout direct terms dropped', 'd_c'),
                                         ('zoneout direct terms dropped', 'd_h_prev'), ('mask_c on h', 'h')])
def test_cell_mutation_is_flagged(mut, output):
    r = _cell_ratios(_cell_inputs(kind=1, training=True, rate=0.5), (mut,))
    assert r[output] > 1.0, (mut, output, r)


# ------------------------------------------------------------------------------------------------------------------------
# the library's host side
# ------------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope='module')
def lib():
    import __graft_entry__ as entry
    from multilingual_text_to_speech_b200 import _lib
    entry.build()
    return _lib.load()


def test_attention_backward_chunk_export(lib):
    """LC and the chunk count of the attention backward at the real dims (A = 128, C = 32, K = 31, M = 288): one chunk up to
    L = 216, then chunks shrink until L = 644, the largest L it accepts (640 at M = 512)"""
    table = {1: (4, 1), 5: (8, 1), 31: (32, 1), 33: (36, 1), 180: (180, 1), 216: (216, 1), 217: (216, 2), 220: (216, 2),
             300: (172, 2), 400: (120, 4), 600: (12, 50), 644: (4, 161)}
    for L, (LC, n) in table.items():
        got = lib.b200tts_debug_attention_backward_chunk(L, 288, 128, 32, 31)
        assert (got, -(-L // got)) == (LC, n), (L, got)
    assert lib.b200tts_debug_attention_backward_chunk(645, 288, 128, 32, 31) == 0
    assert lib.b200tts_debug_attention_backward_chunk(640, 512, 128, 32, 31) == 4
    assert lib.b200tts_debug_attention_backward_chunk(641, 512, 128, 32, 31) == 0
    for bad in ((0, 288, 128, 32, 31), (300, 288, 132, 32, 31), (300, 288, 128, 30, 31), (300, 288, 128, 32, 30),
                (300, 513, 128, 32, 31), (300, 288, 128, 32, 0), (300, 288, 128, 0, 31)):
        assert lib.b200tts_debug_attention_backward_chunk(*bad) == 0, bad


def test_bad_step_arguments_fail_before_any_launch(lib):
    """each bad argument of the step ABIs returns an error from the host-side checks, with no kernel launched"""
    from multilingual_text_to_speech_b200 import _lib
    p = ctypes.c_void_p(16)          # never dereferenced: every call below must fail its argument checks first

    def att(B=2, L=8, M=8, D=8, A=8, C=4, K=3, null=None):
        ptrs = [p] * 13
        if null is not None:
            ptrs[null] = None
        return lib.b200tts_attention_step(B, L, M, D, A, C, K, *ptrs, None)

    def att_bwd(B=2, L=8, M=8, A=8, C=4, K=3):
        return lib.b200tts_attention_step_backward(B, L, M, A, C, K, *([p] * 19), None)

    def cell_bwd(rate_h=0.1, rate_c=0.1, kind=1):
        return lib.b200tts_lstm_cell_backward(2, 8, kind, 1, rate_h, rate_c, *([p] * 8), None)
    calls = [(lambda i=i: att(null=i), 'null argument') for i in range(4, 9)]            # the five weight pointers
    calls += [(lambda k=k: att(**{k: 0}), 'non-positive') for k in ('B', 'L', 'C', 'K')]
    calls += [(lambda: att(A=6), 'multiple of 4')]
    calls += [(lambda k=k: att_bwd(**{k: 0}), 'non-positive') for k in ('B', 'L', 'C', 'K')]
    calls += [(lambda: att_bwd(K=-1), 'non-positive'), (lambda: att_bwd(C=-4), 'non-positive')]
    calls += [(lambda: cell_bwd(rate_h=1.0), 'rates'), (lambda: cell_bwd(rate_c=1.0), 'rates'), (lambda: cell_bwd(rate_h=-0.1), 'rates'),
              (lambda: cell_bwd(kind=2), 'cell kind')]
    for call, msg in calls:
        n0 = _lib.launch_count()
        st = call()
        assert st != 0 and msg.encode() in lib.b200tts_last_error(), (msg, st, lib.b200tts_last_error())
        assert _lib.launch_count() == n0
