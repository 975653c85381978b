"""The fp64 oracle of the training-step reduction kernels (tests/train_ops_check.py) without a GPU.

- It matches fp64 torch autograd of the reference formulas (oracle.tacotron_oracle.tacotron_loss, tests/wavernn_train_oracle.py,
  torch.optim.Adam with clip_grad_norm_) and central finite differences of its own forward.
- Its bounds have power: an fp32 emulation of each kernel in the kernel's own order passes them at ratio <= 1, and each of a set of
  planted kernel mistakes fails them at ratio > 1.
- The host-side argument checks that need no device.
"""
import ctypes
import math
import types

import numpy as np
import pytest
import torch
import torch.nn.functional as Fn

import train_ops_check as O
import wavernn_train_oracle as W
from oracle import tacotron_oracle as TO

D64, F32 = torch.float64, torch.float32


def _close(got, want, what, tol=1e-12):
    scale = max(float(want.abs().max()), 1e-300)
    assert float((got - want).abs().max()) <= tol * scale, (what, float((got - want).abs().max()), scale)


# ------------------------------------------------------------------------------------------------------------------------
# inputs
# ------------------------------------------------------------------------------------------------------------------------
def _loss_inputs(B=3, N=5, T=11, L=7, R=1, seed=0, long_text=False):
    g = torch.Generator().manual_seed(seed)
    S = -(-T // R)
    x = {k: torch.randn(B, N, T, generator=g) for k in ('pre', 'pre_t', 'post', 'post_t')}
    tlen = torch.randint(1, L + 1, (B,), generator=g)
    mlen = torch.randint(1, T + 1, (B,), generator=g)
    tlen[0], mlen[0] = L, T
    tlen[-1], mlen[-1] = 1, 1
    if B > 2:
        mlen[1] = T - 1
    if long_text and B > 3:
        tlen[2] = L + 3                                             # longer than the alignment: Lb = min(text_len, L)
    stop = torch.randn(B, T, generator=g) * 3
    stop_t = torch.zeros(B, T)
    for b in range(B):
        stop_t[b, max(int(mlen[b]) - 2, 0):] = 1.0
        stop[b, int(mlen[b]):] = 1000.0
    stop[0, 0] = -1000.0
    x.update(stop=stop, stop_t=stop_t, align=torch.softmax(torch.randn(B, S, L, generator=g) * 2, 2), tlen=tlen.int(), mlen=mlen.int())
    return x


def _mol_inputs(N=40, nr=4, seed=0, edges=True):
    g = torch.Generator().manual_seed(seed)
    lp = torch.randn(N, nr, generator=g) * 2
    mu = torch.rand(N, nr, generator=g) * 2 - 1
    ls = torch.rand(N, nr, generator=g) * 6 - 5.5
    y = torch.rand(N, generator=g) * 2 - 1
    if edges:
        e = float(np.float32(0.999))
        y[:6] = torch.tensor([-1.0, 1.0, e, -e, float(np.nextafter(np.float32(e), np.float32(2))), -float(np.nextafter(np.float32(e), np.float32(2)))])
        ls[6] = O.LOG_SCALE_MIN
        ls[7] = O.LOG_SCALE_MIN - 1
        ls[8], mu[8] = -20.0, y[8] + 0.25 + 0.01 * torch.arange(nr)    # tiny scales far from y: the pdf branch, one mixture leading
    return torch.cat([lp, mu, ls], 1), y


# ------------------------------------------------------------------------------------------------------------------------
# the oracle against torch autograd and finite differences
# ------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('R, g, pw', [(1, 0.2, 100.0), (2, 0.05, 7.5), (3, 0.2, 1.0)])
def test_tacotron_loss_oracle_matches_autograd(R, g, pw):
    x = _loss_inputs(R=R, T=11)
    B, N, T = x['pre'].shape
    L = x['align'].shape[2]
    gf = float(np.float32(g))
    leaves = {k: x[k].double().clone().requires_grad_(True) for k in ('pre', 'post', 'stop', 'align')}
    Tb = O.loss_steps(x['mlen'], R)
    hp = types.SimpleNamespace(num_mels=N, reversal_classifier=False, guided_attention_loss=True)
    _, parts = TO.tacotron_loss(hp, gf, x['tlen'].long(), Tb, leaves['pre'], x['pre_t'].double(), leaves['post'], x['post_t'].double(),
                                leaves['stop'], x['stop_t'].double(), leaves['align'])
    # the oracle's stop term has pos_weight 100 built in; the ABI takes any: BCE-with-logits with pos_weight pw in its place
    parts['stop_token'] = Fn.binary_cross_entropy_with_logits(leaves['stop'], x['stop_t'].double(),
                                                              pos_weight=torch.tensor(float(np.float32(pw)), dtype=D64)) / (N + 2)
    if pw == 100.0:
        _, p100 = TO.tacotron_loss(hp, gf, x['tlen'].long(), Tb, x['pre'].double(), x['pre_t'].double(), x['post'].double(),
                                   x['post_t'].double(), x['stop'].double(), x['stop_t'].double(), x['align'].double())
        _close(parts['stop_token'].detach(), p100['stop_token'], 'stop, pos_weight 100')
    names = ('mel_pre', 'mel_pos', 'stop_token', 'guided_att')
    gl = torch.tensor([0.7, 1.3, 2.0, 0.5])
    sum(float(gl[k]) * parts[n] for k, n in enumerate(names)).backward()
    f = O.tacotron_loss_forward(*(x[k] for k in ('pre', 'pre_t', 'post', 'post_t', 'stop', 'stop_t', 'align', 'tlen', 'mlen')), R, g, pw, 1)
    _close(f['losses'][0], torch.stack([parts[n].detach() for n in names]), 'losses')
    b = O.tacotron_loss_backward(*(x[k] for k in ('pre', 'pre_t', 'post', 'post_t', 'stop', 'stop_t', 'tlen', 'mlen')), -(-T // R), L, R, g,
                                 pw, 1, gl)
    for name, leaf in (('d_pre', 'pre'), ('d_post', 'post'), ('d_stop', 'stop'), ('d_align', 'align')):
        _close(b[name][0], leaves[leaf].grad, name)
    # with stop logits at +-1000 (padding, confident and right) the terms are exactly 0 and finite
    assert torch.isfinite(b['d_stop'][0]).all() and torch.isfinite(f['losses'][0]).all()
    Tbx = Tb[:, None, None]
    t = torch.arange(-(-T // R))[None, :, None]
    l = torch.arange(L)[None, None, :]
    outside = (t >= Tbx) | (l >= x['tlen'].long()[:, None, None])
    assert (b['d_align'][0][outside] == 0).all() and (b['d_align'][1][outside] == 0).all()


def _fd(f, x, d, h):
    return (f(x + h * d) - f(x - h * d)) / (2 * h)


def test_tacotron_loss_oracle_matches_finite_differences():
    x = _loss_inputs(B=2, N=3, T=7, L=5, R=2, seed=3)
    T, L = 7, 5
    gl = torch.tensor([0.7, 1.3, 2.0, 0.5], dtype=D64)
    args = ('pre', 'pre_t', 'post', 'post_t', 'stop', 'stop_t', 'align', 'tlen', 'mlen')
    b = O.tacotron_loss_backward(*(x[k] for k in ('pre', 'pre_t', 'post', 'post_t', 'stop', 'stop_t', 'tlen', 'mlen')), 4, L, 2, 0.2, 7.5, 1, gl)
    for name, key in (('d_pre', 'pre'), ('d_post', 'post'), ('d_stop', 'stop'), ('d_align', 'align')):
        d = torch.randn(x[key].shape, generator=torch.Generator().manual_seed(1), dtype=D64)

        def loss(v):
            y = dict(x, **{key: v})
            return float((O.tacotron_loss_forward(*(y[k] if k != key else v for k in args), 2, 0.2, 7.5, 1)['losses'][0] * gl).sum())
        fd = _fd(loss, x[key].double(), d, 1e-6)
        an = float((b[name][0] * d).sum())
        assert abs(fd - an) <= 1e-7 * max(1.0, abs(an)), (name, fd, an)


def test_upsample_and_stretch_oracle_match_autograd_and_finite_differences():
    g = torch.Generator().manual_seed(0)
    for C, ln, s in ((3, 4, 5), (2, 7, 11), (1, 1, 1)):
        fir = torch.randn(2 * s + 1, generator=g, dtype=D64).requires_grad_(True)
        x = torch.randn(C, ln, generator=g, dtype=D64).requires_grad_(True)
        dout = torch.randn(C, ln * s, generator=g, dtype=D64)
        fwd = lambda w, xx: Fn.conv1d(xx.repeat_interleave(s, 1)[:, None, :], w[None, None, :], padding=s)[:, 0]    # noqa: E731
        (fwd(fir, x) * dout).sum().backward()
        r = O.upsample_backward(fir.detach(), x.detach(), dout, s)
        _close(r['din'][0], x.grad, 'din')
        _close(r['dfir'][0], fir.grad, 'dfir')
        d = torch.randn(C, ln, generator=g, dtype=D64)
        fd = _fd(lambda v: float((fwd(fir.detach(), v) * dout).sum()), x.detach(), d, 1e-6)
        assert abs(fd - float((r['din'][0] * d).sum())) <= 1e-8 * max(1.0, abs(fd))
    dup = torch.randn(2, 3 * 4, 5, dtype=D64)
    aux = torch.randn(2, 3, 5, dtype=D64, requires_grad=True)
    (aux.repeat_interleave(4, 1) * dup).sum().backward()
    _close(O.stretch_backward(dup, 3, 4)['daux'][0], aux.grad, 'daux')
    xs = torch.randn(70, 9, dtype=D64)
    _close(O.column_sum(xs)['out'][0], xs.sum(0), 'column_sum')


def test_raw_loss_oracle_matches_autograd():
    g = torch.Generator().manual_seed(0)
    for N, n in ((5, 2), (9, 33), (4, 512)):
        logits = torch.randn(N, n, generator=g) * 3
        lab = torch.randint(0, n, (N,), generator=g)
        leaf = logits.double().requires_grad_(True)
        lo = W.raw_loss(leaf[None], lab[None])
        lo.backward()
        r = O.raw_loss(logits, lab)
        _close(r['loss'][0][0], lo.detach(), 'loss')
        _close(r['dlogits'][0], leaf.grad, 'dlogits')
        d = torch.randn(N, n, generator=g, dtype=D64)
        fd = _fd(lambda v: float(O.raw_loss(v, lab)['loss'][0][0]), logits.double(), d, 1e-6)
        assert abs(fd - float((r['dlogits'][0] * d).sum())) <= 1e-7 * max(1.0, abs(fd))
    # a label outside [0, n): NaN row loss (and mean), d logits = softmax / N for the row
    lab[1] = n
    r = O.raw_loss(logits, lab)
    assert math.isnan(float(r['rows'][0][1])) and math.isnan(float(r['loss'][0][0]))
    _close(r['dlogits'][0][1], torch.softmax(logits[1].double(), 0) / N, 'bad row')


def test_mol_loss_oracle_matches_autograd():
    """rows away from y = +-0.999f (where the fp64 and fp32 branch choices differ by design) and away from the cdf_delta threshold"""
    logits, y = _mol_inputs(N=50, nr=5, seed=1, edges=False)
    y[:2] = torch.tensor([-1.0, 1.0])
    logits[3, 10:] = O.LOG_SCALE_MIN - 1.0
    leaf = logits.double().requires_grad_(True)
    lo = W.mol_loss(leaf[None], y.double()[None], log_scale_min=O.LOG_SCALE_MIN)
    lo.backward()
    r = O.mol_loss(logits, y)
    _close(r['loss'][0][0], lo.detach(), 'loss', 1e-10)
    _close(r['dlogits'][0], leaf.grad, 'dlogits', 1e-10)
    d = torch.randn(logits.shape, generator=torch.Generator().manual_seed(2), dtype=D64)
    fd = _fd(lambda v: float(O.mol_loss(v, y)['loss'][0][0]), logits.double(), d, 1e-7)
    assert abs(fd - float((r['dlogits'][0] * d).sum())) <= 1e-6 * max(1.0, abs(fd))


@pytest.mark.parametrize('max_norm, wd, step', [(-1.0, 0.0, 1), (1e-3, 1e-6, 2), (1e9, 1e-6, 100000), (0.5, 0.0, 3)])
def test_adam_oracle_matches_torch(max_norm, wd, step):
    g = torch.Generator().manual_seed(step)
    n = 37
    p, gr = torch.randn(n, generator=g), torch.randn(n, generator=g) * 0.1
    gr[::4] = 0.0
    m, v = torch.randn(n, generator=g) * 1e-2, torch.rand(n, generator=g) * 1e-3
    f = lambda z: float(np.float32(z))                                    # noqa: E731
    prm = torch.nn.Parameter(p.double().clone())
    opt = torch.optim.Adam([prm], lr=f(1e-3), betas=(f(0.9), f(0.999)), eps=f(1e-8), weight_decay=f(wd))
    opt.state[prm] = {'step': torch.tensor(float(step - 1), dtype=D64), 'exp_avg': m.double().clone(), 'exp_avg_sq': v.double().clone()}
    prm.grad = gr.double().clone()
    nrm = torch.linalg.vector_norm(prm.grad)
    if max_norm > 0:
        torch.nn.utils.clip_grad_norm_([prm], f(max_norm))
    opt.step()
    r = O.adam_clip(p, gr, m, v, 1e-3, 0.9, 0.999, 1e-8, wd, max_norm, step)
    _close(r['norm'][0][0], nrm, 'norm')
    _close(r['g'][0], prm.grad, 'clipped g')
    _close(r['m'][0], opt.state[prm]['exp_avg'], 'm')
    _close(r['v'][0], opt.state[prm]['exp_avg_sq'], 'v')
    _close(r['p'][0], prm.detach(), 'p', 1e-10)


# ------------------------------------------------------------------------------------------------------------------------
# fp32 emulations in each kernel's order, with switchable mistakes
# ------------------------------------------------------------------------------------------------------------------------
def _f(x):
    return x.to(F32)


def _warp_sum(v):
    """warp_sum over the last dimension (32 lanes, xor butterfly, fp32)"""
    for o in (16, 8, 4, 2, 1):
        v = v + v[..., torch.arange(32) ^ o]
    return v


def _block_sum(v):
    """block_sum of [..., 256] thread values: warp butterflies, then warp 0's butterfly over the 8 partials and 24 zeros"""
    w = _warp_sum(v.reshape(*v.shape[:-1], 8, 32))[..., 0]
    return _warp_sum(torch.cat([w, torch.zeros(*w.shape[:-1], 24, dtype=F32)], -1))[..., 0]


def _threads_chain(vals, idx, nthreads):
    """per-thread serial fp32 sums of the values assigned to thread idx, in index order"""
    acc = torch.zeros(nthreads, dtype=F32)
    order = torch.argsort(idx, stable=True)
    for v, i in zip(vals[order], idx[order]):
        acc[i] = acc[i] + v
    return acc


def _loss_blocks(thread_vals):
    """loss_partial_kernel's reduction of per-thread values: warp sums, 8 warp partials in order, block partials in double"""
    t = thread_vals.reshape(O.LOSS_BLOCKS, 8, 32)
    w = _warp_sum(t)[..., 0]
    blk = torch.zeros(O.LOSS_BLOCKS, dtype=F32)
    for k in range(8):
        blk = blk + w[:, k]
    return blk.double().sum()


def sim_tacotron_loss(x, R, g, pw, guided, gl, mut=()):
    """loss_partial_kernel + loss_final_kernel and loss_backward_kernel in fp32"""
    pre, pre_t, post, post_t, stop, stop_t, al = (_f(x[k]) for k in ('pre', 'pre_t', 'post', 'post_t', 'stop', 'stop_t', 'align'))
    B, N, T = pre.shape
    S, L = al.shape[1], al.shape[2]
    nth = O.LOSS_BLOCKS * O.LT
    nmel, nstop = B * N * T, B * T
    out = []
    for a, at in ((pre, pre_t), (post, post_t)):
        d = (a - at).reshape(-1)
        sq = d * d
        nfull = nmel // 4
        grp = ((sq[0:4 * nfull:4] + sq[1:4 * nfull:4]) + sq[2:4 * nfull:4]) + sq[3:4 * nfull:4]
        vals, idx = [grp], [torch.arange(nfull) % nth]
        if nmel % 4 and 'tail dropped' not in mut:
            vals.append(sq[4 * nfull:])
            idx.append(torch.full((nmel - 4 * nfull,), nfull % nth))
        out.append(_loss_blocks(_threads_chain(torch.cat(vals), torch.cat(idx), nth)))
    xs, ys = stop.reshape(-1), stop_t.reshape(-1)
    pwf = torch.tensor(pw, dtype=F32)
    sp = torch.log1p(torch.exp(-xs.abs())) + torch.clamp(-xs, min=0)
    bce = (1 - ys) * xs + (1 + (pwf - 1) * ys) * sp
    out.append(_loss_blocks(_threads_chain(bce, torch.arange(nstop) % nth, nth)))
    inv2g2 = torch.tensor(1.0, dtype=F32) / (2 * torch.tensor(g, dtype=F32) * torch.tensor(g, dtype=F32))
    tlen, mlen = x['tlen'].long(), x['mlen'].long()
    Tb = mlen if 'Tb from frames' in mut else (mlen + R - 1) // R
    Lb = torch.clamp(tlen, max=L)
    lane_acc = torch.zeros(nth, dtype=F32)
    wfull = torch.zeros(B, S, L, dtype=F32)
    for row in range(B * S):
        b, t = divmod(row, S)
        if t >= Tb[b]:
            continue
        lv = torch.arange(int(Lb[b]))
        dd = lv.to(F32) / torch.tensor(float(Lb[b]), dtype=F32) - torch.tensor(float(t), dtype=F32) / torch.tensor(float(Tb[b]), dtype=F32)
        w = 1 - torch.exp(-dd * dd * inv2g2)
        wfull[b, t, :int(Lb[b])] = w
        acc = torch.zeros(32, dtype=F32)
        for l0 in range(0, int(Lb[b]), 32):
            n = min(32, int(Lb[b]) - l0)
            acc[:n] = acc[:n] + w[l0:l0 + n] * al[b, t, l0:l0 + n]
        base = (row % (nth // 32)) * 32
        lane_acc[base:base + 32] = lane_acc[base:base + 32] + acc / torch.tensor(float(Tb[b]), dtype=F32)
    out.append(_loss_blocks(lane_acc) if guided else torch.zeros((), dtype=D64))
    scales = (2.0 / nmel, 1.0 / nmel, 1.0 / (nstop * (N + 2)), 1.0 / B)
    losses = torch.stack([(o * float(np.float32(s))).float() for o, s in zip(out, scales)])
    # backward
    glf = _f(gl)
    cs = [float(np.float32(c)) for c in (4.0 / nmel, 2.0 / nmel, 1.0 / (nstop * (N + 2)), 1.0 / B)]
    gk = [glf[k] * torch.tensor(cs[k], dtype=F32) for k in range(4)]
    res = {'losses': losses, 'd_pre': gk[0] * (pre - pre_t), 'd_post': gk[1] * (post - post_t)}
    sneg = 1 / (1 + torch.exp(stop))
    res['d_stop'] = gk[2] * ((1 - stop_t) - (1 + (pwf - 1) * stop_t) * sneg)
    Tbf = Tb.to(F32)[:, None, None]
    res['d_align'] = gk[3] * wfull / Tbf if guided else torch.zeros(B, S, L)
    return res


def sim_upsample(fir, x, dout, s, mut=()):
    """wavernn_upsample_bwd_in_kernel and the two-pass d fir in fp32"""
    C, ln = x.shape
    lo = ln * s
    w, d, xf = _f(fir), _f(dout), _f(x)
    hi = lo - 1 if 'edge tap' in mut else lo
    din = torch.zeros(C, ln, dtype=F32)
    j = torch.arange(ln)
    for q in range(s):
        p = j * s + q
        for k in range(-s, s + 1):
            i = p - k
            ok = (i >= 0) & (i < hi)
            din = din + torch.where(ok, w[k + s] * d[:, i.clamp(0, lo - 1)], torch.zeros(()))
    xs = xf.repeat_interleave(s, 1).reshape(-1)
    n = C * lo
    per = -(-n // O.UPS_CHUNKS)
    e = torch.arange(n)
    dfir = torch.zeros(2 * s + 1, dtype=F32)
    for k in range(-s, s + 1):
        i = e % lo
        ok = (i + k >= 0) & (i + k < hi)
        terms = torch.where(ok, d.reshape(-1) * xs[(e + k).clamp(0, n - 1)], torch.zeros(()))
        total = torch.zeros((), dtype=F32)
        for c in range(O.UPS_CHUNKS):
            chunk = terms[c * per:min(n, (c + 1) * per)]
            m = -(-chunk.numel() // 256) if chunk.numel() else 0
            th = torch.zeros(256, dtype=F32)
            for r in range(m):
                part = chunk[r * 256:(r + 1) * 256]
                th[:part.numel()] = th[:part.numel()] + part
            total = total + _block_sum(th)
        dfir[k + s] = total
    return {'din': din, 'dfir': dfir}


def sim_column_sum(x, mut=()):
    rows, cols = x.shape
    per = -(-rows // O.COLSUM_CHUNKS)
    xf = _f(x)
    out = torch.zeros(cols, dtype=F32)
    for c in range(O.COLSUM_CHUNKS):
        acc = torch.zeros(cols, dtype=F32)
        for r in range(c * per, min(rows, (c + 1) * per)):
            acc = acc + xf[r]
        if not ('chunk skipped' in mut and c == 1):
            out = out + acc
    return out


def sim_stretch(dup, F, hop):
    B, _, C = dup.shape
    d = _f(dup).reshape(B, F, hop, C)
    acc = torch.zeros(B, F, C, dtype=F32)
    for q in range(hop):
        acc = acc + d[:, :, q]
    return acc


def _rows_mean(rows):
    N = rows.numel()
    th = torch.zeros(O.LOSS_SUM_THREADS, dtype=F32)
    for i0 in range(0, N, O.LOSS_SUM_THREADS):
        part = rows[i0:i0 + O.LOSS_SUM_THREADS]
        th[:part.numel()] = th[:part.numel()] + part
    w = _warp_sum(th.reshape(32, 32))[:, 0]
    return (float(_warp_sum(w)[0]) / N)


def sim_raw(logits, lab):
    N, n = logits.shape
    lf = _f(logits)
    mx = lf.max(1, keepdim=True).values
    e = torch.exp(lf - mx)
    lanes = torch.zeros(N, 32, dtype=F32)
    for k0 in range(0, n, 32):
        m = min(32, n - k0)
        lanes[:, :m] = lanes[:, :m] + e[:, k0:k0 + m]
    s = _warp_sum(lanes)[:, :1]
    onehot = torch.zeros(N, n, dtype=F32)
    ok = (lab >= 0) & (lab < n)
    onehot[ok, lab[ok].long()] = 1
    d = (e * (1 / s) - onehot) * torch.tensor(1.0 / N, dtype=F32)
    row = torch.log(s[:, 0]) + mx[:, 0] - lf.gather(1, lab.long().clamp(0, n - 1)[:, None])[:, 0]
    row = torch.where(ok, row, torch.full_like(row, math.nan))
    return {'loss': torch.tensor([_rows_mean(row)], dtype=F32), 'rows': row, 'dlogits': d}


def sim_mol(logits, y, mut=()):
    """wavernn_loss_mol_kernel in fp32 (mixture sums as a warp butterfly over nr lanes padded to 32)"""
    N, n3 = logits.shape
    nr = n3 // 3
    lf = _f(logits)
    lp, mu, lsr = lf[:, :nr], lf[:, nr:2 * nr], lf[:, 2 * nr:]
    LSM = torch.tensor(O.LOG_SCALE_MIN, dtype=F32)
    ls = torch.maximum(lsr, LSM)
    yv = _f(y)[:, None].expand_as(mu)
    cy, inv = yv - mu, torch.exp(-ls)
    hb = torch.tensor(1.0 / 65535.0, dtype=F32)
    plus, mn, mid = inv * (cy + hb), inv * (cy - hb), inv * cy
    sp = lambda v: torch.where(v > 20, v, torch.log1p(torch.exp(v)))                 # noqa: E731
    dsp = lambda v: torch.where(v > 20, torch.ones_like(v), 1 / (1 + torch.exp(-v)))   # noqa: E731
    if 'threshold in fp64' in mut:
        lo_e, hi_e = yv.double() < -0.999, yv.double() > 0.999
    else:
        lo_e, hi_e = yv < np.float32(-0.999), yv > np.float32(0.999)
    cp, cm = 1 / (1 + torch.exp(-plus)), 1 / (1 + torch.exp(-mn))
    cd = cp - cm
    use = cd > np.float32(1e-5)
    z = torch.zeros_like(mu)
    logprob = torch.where(lo_e, plus - sp(plus), torch.where(hi_e, -sp(mn), torch.where(
        use, torch.log(torch.clamp(cd, min=1e-12)), mid - ls - 2 * sp(mid) - np.float32(math.log(32767.5)))))
    dplus = torch.where(lo_e, 1 - dsp(plus), torch.where(hi_e | ~use, z, cp * (1 - cp) / cd))
    dmin = torch.where(lo_e, z, torch.where(hi_e, -dsp(mn), torch.where(use, -cm * (1 - cm) / cd, z)))
    dmid = torch.where(lo_e | hi_e | use, z, 1 - 2 * dsp(mid))
    dls_d = torch.where(lo_e | hi_e | use, z, -torch.ones_like(z))
    dmu_l = -inv * (dplus + dmin + dmid)
    gate = lsr > LSM if 'clamp edge blocks gradient' in mut else lsr >= LSM
    dls_l = torch.where(gate, dls_d - (plus * dplus + mn * dmin + mid * dmid), z)
    pad = lambda v, fill: torch.cat([v, torch.full((N, 32 - nr), fill, dtype=F32)], 1)   # noqa: E731
    m = lp.max(1, keepdim=True).values
    e = torch.exp(lp - m)
    s = _warp_sum(pad(e, 0.0))[:, :1]
    a = logprob + (lp - m - torch.log(s))
    M = a.max(1, keepdim=True).values
    ea = torch.exp(a - M)
    S = _warp_sum(pad(ea, 0.0))[:, :1]
    invN = torch.tensor(1.0 / N, dtype=F32)
    w, sm = ea / S, e / s
    gmix = -w * invN
    row = -(M[:, 0] + torch.log(S[:, 0]))
    return {'loss': torch.tensor([_rows_mean(row)], dtype=F32), 'rows': row,
            'dlogits': torch.cat([(sm - w) * invN, gmix * dmu_l, gmix * dls_l], 1)}


def sim_adam(p, g, m, v, lr, b1, b2, eps, wd, max_norm, step, mut=()):
    """sqnorm_partial_kernel, sqnorm_finish_kernel and adam_clip_kernel in fp32"""
    n = g.numel()
    gf = _f(g)
    nblk = O.norm_blocks(n)
    n4 = n // 4
    acc = torch.zeros(nblk * 256, 4, dtype=F32)
    g4 = gf[:4 * n4].reshape(n4, 4)
    for i0 in range(0, n4, nblk * 256):
        part = g4[i0:i0 + nblk * 256]
        acc[:part.shape[0]] = acc[:part.shape[0]] + part * part
    for i in range(4 * n4, n):
        t = i - 4 * n4
        acc[t, 0] = acc[t, 0] + gf[i] * gf[i]
    th = ((acc[:, 0] + acc[:, 1]) + (acc[:, 2] + acc[:, 3])).reshape(nblk, 256)
    partial = _block_sum(th)
    fin = torch.zeros(256, dtype=F32)
    for i0 in range(0, nblk, 256):
        part = partial[i0:i0 + 256]
        fin[:part.numel()] = fin[:part.numel()] + part
    nrm = torch.sqrt(_block_sum(fin))
    f = lambda z: torch.tensor(float(np.float32(z)), dtype=F32)                            # noqa: E731
    coef = torch.minimum(f(max_norm) / (nrm + f(1e-6)), torch.ones(())) if max_norm > 0 else torch.ones((), dtype=F32)
    if 'coefficient doubled' in mut:
        coef = coef * 2
    gc = gf * coef
    gsrc = gf if 'clip after the moments' in mut else gc
    gi = f(wd) * _f(p) + gsrc
    mi = f(b1) * _f(m) + (1 - f(b1)) * gi
    vi = f(b2) * _f(v) + (1 - f(b2)) * gi * gi
    bc1 = f(1.0 - float(np.float32(b1)) ** step)
    bc2s = f(math.sqrt(1.0 - float(np.float32(b2)) ** step))
    pn = _f(p) - (f(lr) / bc1) * (mi / (torch.sqrt(vi) / bc2s + f(eps)))
    return {'norm': nrm.reshape(1), 'coef': coef.reshape(1), 'g': gc, 'm': mi, 'v': vi, 'p': pn}


# ------------------------------------------------------------------------------------------------------------------------
# bound power
# ------------------------------------------------------------------------------------------------------------------------
def _ratios(got, refs):
    return {k: O.ratio(got[k], ref, bound)[0] for k, (ref, bound) in refs.items()}


def _loss_ratios(x, R, g, pw, guided, mut=()):
    T = x['pre'].shape[2]
    L = x['align'].shape[2]
    gl = torch.tensor([0.7, 1.3, 2.0, 0.5])
    got = sim_tacotron_loss(x, R, g, pw, guided, gl, mut)
    refs = O.tacotron_loss_forward(*(x[k] for k in ('pre', 'pre_t', 'post', 'post_t', 'stop', 'stop_t', 'align', 'tlen', 'mlen')), R, g, pw,
                                   guided)
    refs.update(O.tacotron_loss_backward(*(x[k] for k in ('pre', 'pre_t', 'post', 'post_t', 'stop', 'stop_t', 'tlen', 'mlen')), -(-T // R), L,
                                         R, g, pw, guided, gl))
    r = _ratios(got, refs)
    r.update({f'loss{k}': O.ratio(got['losses'][k], refs['losses'][0][k], refs['losses'][1][k])[0] for k in range(4)})
    return r


LOSS_SIM = [dict(B=3, N=5, T=11, L=7, R=1, g=0.2, pw=100.0), dict(B=2, N=3, T=7, L=5, R=2, g=0.05, pw=7.5),
            dict(B=4, N=7, T=13, L=30, R=3, g=0.05, pw=1.0), dict(B=1, N=3, T=5, L=4, R=1, g=0.2, pw=100.0)]


@pytest.mark.parametrize('c', LOSS_SIM, ids=lambda c: '-'.join(f'{k}{v}' for k, v in c.items()))
def test_tacotron_loss_simulation_is_within_the_bounds(c):
    x = _loss_inputs(c['B'], c['N'], c['T'], c['L'], c['R'], seed=c['T'], long_text=True)
    for guided in (1, 0):
        r = _loss_ratios(x, c['R'], c['g'], c['pw'], guided)
        assert max(r.values()) <= 1.0, r


@pytest.mark.parametrize('mut, output', [('tail dropped', 'loss0'), ('tail dropped', 'loss1'), ('Tb from frames', 'loss3'),
                                         ('Tb from frames', 'd_align')])
def test_tacotron_loss_mutation_is_flagged(mut, output):
    x = _loss_inputs(3, 5, 11, 7, 2, seed=4)                      # B N T = 165: a tail of 1; R = 2
    r = _loss_ratios(x, 2, 0.2, 100.0, 1, (mut,))
    assert r[output] > 1.0, (mut, output, r)


def _ups_case(C, ln, s, seed=0):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(2 * s + 1, generator=g) / (2 * s + 1), torch.randn(C, ln, generator=g), torch.randn(C, ln * s, generator=g))


def _ups_ratios(C, ln, s, mut=()):
    fir, x, dout = _ups_case(C, ln, s)
    got = sim_upsample(fir, x, dout, s, mut)
    return _ratios(got, O.upsample_backward(fir, x, dout, s))


@pytest.mark.parametrize('C, ln, s', [(3, 4, 5), (2, 7, 11), (1, 3, 5), (40, 9, 5)])
def test_upsample_simulation_is_within_the_bounds(C, ln, s):
    r = _ups_ratios(C, ln, s)
    assert max(r.values()) <= 1.0, r


@pytest.mark.parametrize('output', ('din', 'dfir'))
def test_upsample_mutation_is_flagged(output):
    r = _ups_ratios(3, 4, 5, ('edge tap',))
    assert r[output] > 1.0, r


def test_stretch_and_column_sum_simulations():
    g = torch.Generator().manual_seed(0)
    dup = torch.randn(2, 3 * 275, 4, generator=g)
    assert O.ratio(sim_stretch(dup, 3, 275), *O.stretch_backward(dup, 3, 275)['daux'])[0] <= 1.0
    for rows in (1, 63, 65, 1000):
        x = torch.randn(rows, 7, generator=g) + 0.5
        ref, b = O.column_sum(x)['out']
        assert O.ratio(sim_column_sum(x), ref, b)[0] <= 1.0
        if rows > 64:
            assert O.ratio(sim_column_sum(x, ('chunk skipped',)), ref, b)[0] > 1.0, rows


@pytest.mark.parametrize('N, n', [(7, 2), (9, 33), (5, 512), (1030, 31)])
def test_raw_simulation_is_within_the_bounds(N, n):
    g = torch.Generator().manual_seed(n)
    logits = torch.randn(N, n, generator=g) * 3
    lab = torch.randint(0, n, (N,), generator=g)
    lab[0], lab[-1] = 0, n - 1
    r = _ratios(sim_raw(logits, lab), O.raw_loss(logits, lab))
    assert max(r.values()) <= 1.0, r


@pytest.mark.parametrize('nr', (1, 4, 10, 32))
def test_mol_simulation_is_within_the_bounds(nr):
    logits, y = _mol_inputs(N=60, nr=nr, seed=nr)
    r = _ratios(sim_mol(logits, y), O.mol_loss(logits, y))
    assert max(r.values()) <= 1.0, r
    assert (sim_mol(logits, y)['dlogits'][7, 2 * nr:] == 0).all()


def test_mol_clamp_edge_blocking_gradient_is_flagged():
    """lsr > log(1e-14)f in place of >=: the row with every log scale exactly on the clamp edge loses its d log-scale"""
    logits, y = _mol_inputs(N=60, nr=4, seed=3)
    ref, bnd = O.mol_loss(logits, y)['dlogits']
    assert torch.isfinite(bnd[6]).all() and (ref[6, 8:] != 0).any()
    r = O.ratio(sim_mol(logits, y, ('clamp edge blocks gradient',))['dlogits'][6], ref[6], bnd[6])[0]
    assert r > 1.0, r


def test_mol_threshold_in_fp64_is_flagged():
    logits, y = _mol_inputs(N=60, nr=4, seed=3)
    r = _ratios(sim_mol(logits, y, ('threshold in fp64',)), O.mol_loss(logits, y))
    assert r['dlogits'] > 1.0 and r['rows'] > 1.0, r


ADAM_SIM = [(n, mx, wd, st) for n in (1, 3, 5, 1023, 4099) for mx, wd, st in ((-1.0, 0.0, 1), (1e-3, 1e-6, 2), (1e9, 1e-6, 100000))]


def _adam_case(n, seed=0):
    g = torch.Generator().manual_seed(seed + n)
    p, gr = torch.randn(n, generator=g), torch.randn(n, generator=g) * 1e-3
    m, v = torch.randn(n, generator=g) * 1e-4, torch.rand(n, generator=g) * 1e-7
    if n > 1:
        gr[1::3], m[1::3], v[1::3] = 0.0, 0.0, 0.0
    gr[n // 2] = 1e3
    return p, gr, m, v


@pytest.mark.parametrize('n, max_norm, wd, step', ADAM_SIM)
def test_adam_simulation_is_within_the_bounds(n, max_norm, wd, step):
    p, gr, m, v = _adam_case(n)
    got = sim_adam(p, gr, m, v, 1e-3, 0.9, 0.999, 1e-8, wd, max_norm, step)
    r = _ratios(got, O.adam_clip(p, gr, m, v, 1e-3, 0.9, 0.999, 1e-8, wd, max_norm, step))
    assert max(r.values()) <= 1.0, r


@pytest.mark.parametrize('max_norm', (-1.0, 1e9))
def test_adam_doubled_coefficient_is_flagged(max_norm):
    """a coefficient of 2 where the clip does not bind (max_norm off, or far above the norm): there the kernel's min(1, .) is exactly 1
    and so is the reference's, with a bound of 0"""
    p, gr, m, v = _adam_case(1023)
    refs = O.adam_clip(p, gr, m, v, 1e-3, 0.9, 0.999, 1e-8, 1e-6, max_norm, 2)
    assert float(refs['coef'][0]) == 1.0 and float(refs['coef'][1]) == 0.0
    got = sim_adam(p, gr, m, v, 1e-3, 0.9, 0.999, 1e-8, 1e-6, max_norm, 2, ('coefficient doubled',))
    r = _ratios(got, refs)
    assert min(r['g'], r['m'], r['v'], r['p']) > 1.0, r


def test_adam_clip_after_the_moments_is_flagged():
    p, gr, m, v = _adam_case(1023)
    got = sim_adam(p, gr, m, v, 1e-3, 0.9, 0.999, 1e-8, 0.0, 1e-3, 2, ('clip after the moments',))
    r = _ratios(got, O.adam_clip(p, gr, m, v, 1e-3, 0.9, 0.999, 1e-8, 0.0, 1e-3, 2))
    assert r['m'] > 1.0 and r['v'] > 1.0 and r['p'] > 1.0, r


def test_mol_constants_are_the_kernels():
    """the fp32 literals of wavernn_loss_mol_kernel round the values the oracle uses"""
    assert np.float32(O.LOG_HALF_CLASSES) == np.float32(10.3971924)
    assert np.float32(math.log(1e-14)) == np.float32(O.LOG_SCALE_MIN)


# ------------------------------------------------------------------------------------------------------------------------
# the library's host side
# ------------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope='module')
def lib():
    import __graft_entry__ as entry
    from multilingual_text_to_speech_b200 import _lib
    entry.build()
    return _lib.load()


def test_bad_train_op_arguments_fail_before_any_launch(lib):
    """each bad argument returns an error from the host-side checks, with no kernel launched"""
    from multilingual_text_to_speech_b200 import _lib
    p = ctypes.c_void_p(16)             # never dereferenced: every call below must fail its argument checks first
    shape = _lib.LossShape(2, 3, 4, 5, 1, 0.2, 100.0, 1)
    calls = [
        (lambda: lib.b200tts_wavernn_loss(2, 4, 10, p, p, p, p, p, 64, None), 'unknown mode'),
        (lambda: lib.b200tts_wavernn_loss(0, 4, 1, p, p, p, p, p, 64, None), 'RAW needs'),
        (lambda: lib.b200tts_wavernn_loss(0, 4, 65537, p, p, p, p, p, 64, None), 'RAW needs'),
        (lambda: lib.b200tts_wavernn_loss(1, 4, 99, p, p, p, p, p, 64, None), 'MOL needs'),
        (lambda: lib.b200tts_wavernn_loss(1, 4, 10, p, p, p, p, p, 64, None), 'MOL needs'),
        (lambda: lib.b200tts_wavernn_loss(1, 0, 30, p, p, p, p, p, 64, None), 'rows'),
        (lambda: lib.b200tts_wavernn_loss(1, 4, 30, p, None, p, p, p, 64, None), 'null argument'),
        (lambda: lib.b200tts_column_sum(0, 4, p, p, p, 1 << 20, None), 'bad dimensions'),
        (lambda: lib.b200tts_column_sum(4, 0, p, p, p, 1 << 20, None), 'bad dimensions'),
        (lambda: lib.b200tts_column_sum(4, 4, None, p, p, 1 << 20, None), 'null argument'),
        (lambda: lib.b200tts_wavernn_stretch_backward(1, 2, 3, 0, p, p, None), 'bad dimensions'),
        (lambda: lib.b200tts_wavernn_stretch_backward(0, 2, 3, 4, p, p, None), 'bad dimensions'),
        (lambda: lib.b200tts_wavernn_upsample_layer_backward(4, 0, 5, p, p, p, p, p, p, 1 << 20, None), 'bad dimensions'),
        (lambda: lib.b200tts_wavernn_upsample_layer_backward(4, 3, 0, p, p, p, p, p, p, 1 << 20, None), 'bad dimensions'),
        (lambda: lib.b200tts_wavernn_upsample_layer_backward(4, 3, 5, p, p, p, None, None, p, 1 << 20, None), 'null argument'),
        (lambda: lib.b200tts_tacotron_loss_forward(ctypes.byref(shape), *([p] * 6), None, p, p, p, p, None), 'needs the alignments'),
        (lambda: lib.b200tts_tacotron_loss_forward(ctypes.byref(shape), p, None, *([p] * 8), p, None), 'null argument'),
        (lambda: lib.b200tts_tacotron_loss_backward(ctypes.byref(shape), *([p] * 8), None, p, p, p, p, None), 'null argument'),
    ]
    for call, msg in calls:
        n0 = _lib.launch_count()
        st = call()
        assert st != 0 and msg.encode() in lib.b200tts_last_error(), (msg, st, lib.b200tts_last_error())
        assert _lib.launch_count() == n0
