"""fp64 reference of the conv block epilogue (csrc/encoder.cu) and a per-element error bound for every value the library returns.

The reference is composed from the oracle's own pieces (oracle/tacotron_oracle.py): `conv1d_same` per group, `batch_norm_train` /
`batch_norm_eval`, `running_stats_update`, `_act`, `apply_dropout` with the kernel's keep mask, and the highway gate as
`generated_conv_block` writes it; autograd gives the gradients.  It starts from the kernel's OWN convolution product (the first
conv_elems floats of `saved`), so the convolution's error, bounded by tests/test_gpu_conv_exact.py, does not enter the epilogue
checks.  d x and d w are the fp64 conv transposes of the fp64 d conv.

Each element gets its own bound from the fp32 operations the kernels do (U = 2^-24), in the style of tests/step_check.py:
- batch statistics: `channel_sum` walks at most n / 256 + NB + 1 terms serially per accumulator, then 2 lane adds, the 5 + 5 levels
  of `block_sum` and a division: (m + 14) U of the sum of |terms|.  The variance is two-pass: the kernel's mean error enters only
  squared, which a one-pass E[x^2] - E[x]^2 would not do.
- the element-wise epilogue: a few roundings of the magnitude of each operation's operands, `tanhf` within 2 ulp, `sigmoidf_acc`
  as bounded in step_check.sigmoid_err, the keep scale 1 / (1 - p) rounded once.
- the deviation of the kernel's mean / invstd from the exact statistics is measured (and checked on its own against its bound)
  and carried into every element that uses them; a ReLU within its input bound of the kink may take either branch.
- the batch-norm backward (dz - s1/n - xhat s2/n) is bounded by the magnitude of its terms, not of its result.
- d x / d w: the d conv bound pushed through |W| / |x| plus the accumulation bound (K + 2) U |W| |d conv| of the GEMM (doubled,
  plus one bf16 rounding 2^-8 of d conv, in bf16 mode, where x and W are bf16 values by construction).
Everything is first order in the deviations; the 1 % slack (SLACK) covers the products of two of them.
"""
import torch

from oracle import tacotron_oracle as O
from step_check import U, ULP1, sigmoid_err

ACTS = {'identity': 0, 'relu': 1, 'tanh': 2}
BF16_U = 2.0 ** -8
SLACK = 1.01


def a64(m):
    return (m + 63) // 64 * 64


def sum_rel(NB, L):
    """Relative bound of channel_sum + block_sum over the n = NB L values of one channel (encoder.cu:56-86, common.cuh:68-81)."""
    m = (NB * L) // 256 + NB + 1
    return (m + 14) * U


def conv_groups(x, w, G, dil):
    """Grouped same-padded convolution: O.conv1d_same per group.  x [NB, G Cin, L], w [G Cout, Cin, k]."""
    Cin, Cout = x.shape[1] // G, w.shape[0] // G
    return torch.cat([O.conv1d_same(x[:, g * Cin:(g + 1) * Cin], w[g * Cout:(g + 1) * Cout], dil) for g in range(G)], 1)


def conv_transposes(x, w, G, dil, dconv):
    """(d x, d w) of conv_groups for the output gradient dconv (autograd through O.conv1d_same)."""
    xl, wl = x.detach().clone().requires_grad_(True), w.detach().clone().requires_grad_(True)
    conv_groups(xl, wl, G, dil).backward(dconv)
    return xl.grad, wl.grad


def _halves(t, G):
    """[NB, G*2C, L] -> the gate (first C of each group) and value (second C) halves, each [NB, G*C, L]."""
    NB, Ct, L = t.shape
    v = t.view(NB, G, 2, Ct // (2 * G), L)
    return v[:, :, 0].reshape(NB, -1, L), v[:, :, 1].reshape(NB, -1, L)


def _merge(t1, t2, G):
    NB, GC, L = t1.shape
    return torch.stack([t1.view(NB, G, GC // G, L), t2.view(NB, G, GC // G, L)], 2).reshape(NB, 2 * GC, L)


def epilogue(c, conv, gamma, beta, keep=None, xin=None, rm=None, rv=None, dout=None, scale=None, swap_highway=False):
    """The block after the convolution, in the precision of `conv`.  gamma / beta [G*Cout]; keep [NB, G*Cout, L] 0/1 or None.
    Returns the outputs, the batch statistics, the intermediates the bounds need and, given dout, every gradient.
    `scale` / `swap_highway` exist only to build the mutated results of tests/test_convblock_cpu.py."""
    conv = conv.detach().clone().requires_grad_(True)
    gamma, beta = (t.detach().clone().requires_grad_(True) for t in (gamma, beta))
    xin = xin.detach().clone().requires_grad_(True) if c['highway'] else None
    NB, Ct, L = conv.shape
    if c['training']:
        z, mean, var = O.batch_norm_train(conv, gamma, beta, c['eps'])
    else:
        z, mean, var = O.batch_norm_eval(conv, gamma, beta, rm, rv, c['eps']), rm, rv
    z.retain_grad()
    a = O._act(c['act'], z)
    a.retain_grad()
    if c['training'] and keep is not None and c['p'] > 0:
        h = O.apply_dropout(a, keep, c['p']) if scale is None else a * keep * scale
    else:
        h = a
    if c['highway']:                    # generated_conv_block: gate = sigmoid(first half), value = second half, per group
        gate, val = _halves(h, c['G'])
        if swap_highway:
            gate, val = val, gate
        s = O._sigmoid(gate)
        out = val * s + xin * (1.0 - s)
    else:
        out = h
    R = dict(out=out.detach(), z=z.detach(), a=a.detach(), h=h.detach(), mean=mean.detach().reshape(-1),
             var=var.detach().reshape(-1))
    if c['training']:
        R['rm'], R['rv'] = O.running_stats_update(rm, rv, R['mean'], R['var'], NB * L, c['momentum'])
    if dout is not None:
        out.backward(dout)
        R.update(dconv=conv.grad, dgamma=gamma.grad, dbeta=beta.grad, gz=z.grad, ga=a.grad,
                 dskip=xin.grad if c['highway'] else None)
    return R


def bounds(c, R, K, conv, gamma, beta, keep=None, xin=None, rm=None, rv=None, dout=None, x=None, w=None, mode='fp32', conv_dev=None):
    """Per-element bounds of the kernel's results around the reference R = epilogue(...) of the kernel's own product `conv`.
    K: the kernel's saved 'mean' and 'invstd' [Ct].  rm / rv: the running statistics before the call.  conv_dev: a bound on how far
    the product the kernel used may be from `conv` (masked eval against a per-sample fp64 block), else None."""
    NB, Ct, L = conv.shape
    n = NB * L
    gs = sum_rel(NB, L)
    v1 = lambda t: t.view(1, -1, 1)       # noqa: E731
    chan = lambda t: t.sum((0, 2))        # noqa: E731
    mu, var, eps, mo = R['mean'], R['var'], c['eps'], c['momentum']
    is_ = 1.0 / torch.sqrt(var + eps)
    B = {}
    if c['training']:
        B['mean'] = gs * chan(conv.abs()) / n + U * mu.abs()
        dvar = B['mean'] ** 2 + (gs + 3 * U) * (var + B['mean'] ** 2)      # (x - mean~)^2 = (x - mean)^2 + n dmean^2, then the sum
        f = n / max(n - 1, 1)
        B['rm'] = mo * B['mean'] + 4 * U * ((1 - mo) * rm.abs() + mo * mu.abs())
        B['rv'] = mo * f * dvar + 5 * U * ((1 - mo) * rv.abs() + mo * f * var)
    else:
        B['mean'] = torch.zeros_like(mu)                                       # the running mean itself
        dvar = torch.zeros_like(var)
    t = dvar / (var + eps)
    # 1 / sqrtf(var + eps): a relative error t of var + eps moves it by at most (1 - t)^-1/2 - 1; add, sqrt and divide round once each
    B['invstd'] = torch.where(t < 0.5, is_ * ((1 - t.clamp(max=0.5)) ** -0.5 - 1 + 4 * U), torch.full_like(t, float('inf')))

    dmu, r_is = v1((K['mean'] - mu).abs()), v1((K['invstd'] - is_).abs())
    isk, g, b = v1(K['invstd']), v1(gamma), v1(beta)
    xh = (conv - v1(mu)) * v1(is_)
    # |xhat~ - xhat| of the kernel's (x - mean~) * invstd~ (two roundings)
    xh_dev = dmu * isk + (conv - v1(mu)).abs() * r_is + 2 * U * xh.abs()
    if conv_dev is not None:
        xh_dev = xh_dev + conv_dev * isk
    A = (conv - v1(K['mean'])).abs() * isk * g.abs()
    zb = g.abs() * xh_dev + 2 * U * (A + b.abs())                              # * gamma, + beta
    z, a = R['z'], R['a']
    ab = zb + 2 * ULP1 * a.abs() if c['act'] == 'tanh' else zb                # tanhf: 2 ulp; relu / identity exact
    drop = c['training'] and keep is not None and c['p'] > 0
    ks = keep / (1.0 - c['p']) if drop else torch.ones_like(a)
    hb = ks * (ab + 3 * U * a.abs()) if drop else ab                           # the scale rounded once, the product once
    if c['highway']:
        G = c['G']
        h1, h2 = _halves(R['h'], G)
        hb1, hb2 = _halves(hb, G)
        s = torch.sigmoid(h1)
        sb = 0.25 * hb1 + sigmoid_err(h1, 'fp32')
        B['out'] = s * hb2 + (h2 - xin).abs() * sb + hb2 * sb + 4 * U * (h2.abs() * s + xin.abs() * (1 - s))
    else:
        B['out'] = hb
    if dout is None:
        return {k: v * SLACK for k, v in B.items()}

    ga, gz = R['ga'], R['gz']
    if c['highway']:
        ks1, ks2 = _halves(ks, G)
        ga1, ga2 = _halves(ga, G)
        q, qb = s * (1 - s), (1 - 2 * s).abs() * sb + sb * sb
        ga1_b = dout.abs() * ks1 * (hb2 * q + (h2 - xin).abs() * qb + hb2 * qb) + 6 * U * ga1.abs()
        ga2_b = dout.abs() * ks2 * sb + 3 * U * ga2.abs()
        ga_b = _merge(ga1_b, ga2_b, G)
        dskip_b = dout.abs() * sb + 2 * U * R['dskip'].abs()
    else:
        ga_b = 2 * U * ga.abs()
    if c['act'] == 'relu':              # within zb of the kink the kernel may take either branch
        gz_b = torch.where(z.abs() <= zb, ga.abs() + ga_b, torch.where(z > 0, ga_b, torch.zeros_like(ga_b)))
    elif c['act'] == 'tanh':            # 1 - a~^2
        gz_b = ga_b * (1 - a * a) + ga.abs() * (2 * a.abs() * ab + ab * ab + 3 * U)
    else:
        gz_b = ga_b
    S1, S2 = v1(chan(gz)), v1(chan(gz * xh))
    if c['training']:
        T = gz.abs() + S1.abs() / n + xh.abs() * S2.abs() / n                  # the terms of dz - s1/n - xhat s2/n
        e = (gz_b + v1(chan(gz_b)) / n + xh.abs() * v1(chan(gz_b * xh.abs())) / n             # from dz~
             + xh_dev * S2.abs() / n + xh.abs() * v1(chan(gz.abs() * xh_dev)) / n             # from xhat~ (apply and s2)
             + gs * v1(chan(gz.abs())) / n + xh.abs() * (gs + 3 * U) * v1(chan((gz * xh).abs())) / n   # s1, s2 sums
             + 6 * U * T)
        B['dconv'] = g.abs() * isk * e + g.abs() * r_is * (gz - S1 / n - xh * S2 / n).abs()
    else:
        B['dconv'] = g.abs() * isk * (gz_b + 2 * U * gz.abs()) + g.abs() * r_is * gz.abs()
    B['dgamma'] = chan(gz_b * xh.abs() + gz.abs() * xh_dev + gz_b * xh_dev) + (gs + 3 * U) * chan((gz * xh).abs())
    B['dbeta'] = chan(gz_b) + gs * chan(gz.abs())
    if c['stage'] == 2:
        B['dx'] = B['dconv']
    else:
        def rel(Kr):
            return (Kr + 2) * U if mode == 'fp32' else BF16_U * SLACK + 2 * (Kr + 2) * U
        dcb, dca = B['dconv'], R['dconv'].abs()
        tx1, tw1 = conv_transposes(x.abs(), w.abs(), c['G'], c['dil'], dcb)
        tx2, tw2 = conv_transposes(x.abs(), w.abs(), c['G'], c['dil'], dca)
        B['dx'] = tx1 + rel(c['Cout'] * c['k']) * tx2
        B['dw'] = tw1 + rel(NB * L) * tw2
        if c['highway']:
            B['dx'] = B['dx'] + dskip_b + U * (tx2 + R['dskip'].abs())     # the GEMM adds its product to the skip gradient
    return {k: v * SLACK for k, v in B.items()}


def conv_rel(K, mode):
    """Accumulation bound of a K-term product, relative to the sum of |terms| (with one bf16 rounding of an operand in bf16 mode)."""
    return (K + 2) * U if mode == 'fp32' else BF16_U * SLACK + 2 * (K + 2) * U


def masked_reference(c, x, w, gamma, beta, rm, rv, K, lengths, mode):
    """Eval-mode whole block of each sample on its own prefix x[n, :, :lengths[n]] in fp64, and the bound of the masked forward's
    output around it: the convolution's accumulation bound carried through the epilogue.  Positions past a length: reference 0,
    bound 0 (only an exact zero passes)."""
    NB, _, L = x.shape
    Cf = c['Cout'] // 2 if c['highway'] else c['Cout']
    ref = torch.zeros(NB, c['G'] * Cf, L, dtype=torch.float64, device=x.device)
    bnd = torch.zeros_like(ref)
    for q, ln in enumerate(int(v) for v in lengths):
        xq = x[q:q + 1, :, :ln]
        conv = conv_groups(xq, w, c['G'], c['dil'])
        dev = conv_rel(c['Cin'] * c['k'], mode) * conv_groups(xq.abs(), w.abs(), c['G'], c['dil'])
        R = epilogue(c, conv, gamma, beta, xin=xq, rm=rm, rv=rv)
        ref[q, :, :ln] = R['out'][0]
        bnd[q, :, :ln] = bounds(c, R, K, conv, gamma, beta, xin=xq, rm=rm, rv=rv, conv_dev=dev)['out'][0]
    return ref, bnd


def report(got, ref, bnd):
    """{quantity: (worst err / bound, err, bound at the worst)} over the quantities in all three dicts.  A zero bound admits only a
    zero error; a NaN counts as an infinite error."""
    out = {}
    for q in bnd:
        if q not in got or q not in ref:
            continue
        gq, rq, bq = got[q].double().reshape(-1), ref[q].double().reshape(-1), bnd[q].double().reshape(-1).to(got[q].device)
        rq = rq.to(gq.device)
        err = (gq - rq).abs()
        ratio = torch.where(err == 0, torch.zeros_like(err), err / bq)
        ratio = torch.nan_to_num(ratio, nan=float('inf'))
        j = int(ratio.argmax())
        out[q] = (float(ratio[j]), float(err[j]), float(bq[j]))
    return out


def worst_lines(title, rep):
    return [f'{title} {q:>7s}: worst err/bound {r:.3e} (err {e:.3e}, bound {b:.3e})' for q, (r, e, b) in rep.items()]


def failures(rep):
    return {q: v for q, v in rep.items() if not v[0] <= 1.0}
