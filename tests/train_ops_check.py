"""fp64 oracle and per-element bounds of the reduction kernels at the ends of both training steps, as the C ABI runs them:

    b200tts_tacotron_loss_forward / _backward          loss_partial_kernel + loss_final_kernel, loss_backward_kernel (csrc/loss.cu)
    b200tts_wavernn_upsample_layer_backward            wavernn_upsample_bwd_in_kernel, _fir_part_kernel + _fir_sum_kernel
    b200tts_wavernn_stretch_backward                   wavernn_stretch_bwd_kernel
    b200tts_column_sum                                 column_sum_part_kernel + column_sum_add_kernel
    b200tts_wavernn_loss (RAW, MOL)                    wavernn_loss_{raw,mol}_kernel + wavernn_loss_sum_kernel (csrc/wavernn_train.cu)
    b200tts_adam_clip_step                             sqnorm_partial_kernel, sqnorm_finish_kernel, adam_clip_kernel (csrc/optim.cu)

Each output is recomputed in fp64 from the inputs of the call, and gets its own bound, derived from the kernel's order of arithmetic:

    a sum of m fp32 terms added serially, then tree-reduced to depth d:   (m + d + c) 2^-24 sum |terms|  (+ the terms' own bounds)
    an element-wise formula:                                              a few ulps of the magnitudes it combines (class V below)

No bound is a blanket tolerance.  Every function returns {output name: (reference, bound)}; the bounds of the += outputs are those of
the increment (accumulate adds the final add onto the caller's buffer).
"""
import math

import numpy as np
import torch

U = 2.0 ** -24                   # fp32 unit roundoff: a correctly rounded op errs by at most U |result|
TINY = 2.0 ** -148               # absolute floor of one op's error: rounding into the subnormal range
NUM_SMS = 132                    # csrc/common.cuh:48
LOSS_BLOCKS = 4 * NUM_SMS        # csrc/loss.cu:12, the grid of loss_partial_kernel
LT = 256                         # csrc/loss.cu:11, its threads per block (LT / 32 = 8 warps)
UPS_CHUNKS = 64                  # csrc/wavernn_train.cu:217, chunks of the flat (c, i) range per FIR tap
COLSUM_CHUNKS = 64               # csrc/wavernn_train.cu:255, row chunks of column_sum
LOSS_SUM_THREADS = 1024          # csrc/wavernn_train.cu:360, the one block of wavernn_loss_sum_kernel
NORM_BLOCKS = 8 * NUM_SMS        # csrc/optim.cu:10, the most blocks of sqnorm_partial_kernel
BLOCK_SUM_DEPTH = 10             # common.cuh block_sum: a 5-level warp butterfly, then one over the warp partials
WARP_DEPTH = 5                   # warp_sum: a 5-level butterfly

# the literals of wavernn_loss_mol_kernel (csrc/wavernn_train.cu:302-304), as the fp32 values the kernel uses
LOG_SCALE_MIN = float(np.float32(-32.23619130191664))
HALF_BIN = 1.0 / 65535.0
LOG_HALF_CLASSES = math.log(65535.0 / 2.0)
CDF_FLOOR = float(np.float32(1e-5))


def ratio(got, ref, bound):
    """worst err / bound over all elements (0 / 0 = 0, err / 0 = inf, NaN = inf) and the flat index where it sits.  A bound that is
    not finite where the reference is counts as inf: such a bound accepts any value, so it checks nothing."""
    ref, bound = ref.double(), bound.double()
    err = (got.double() - ref).abs()
    r = torch.where(err == 0, torch.zeros_like(err), err / bound)
    r = torch.where(torch.isfinite(ref) & ~torch.isfinite(bound), torch.full_like(r, math.inf), r)
    r = torch.nan_to_num(r, nan=math.inf).reshape(-1)
    if r.numel() == 0:
        return 0.0, -1
    i = int(r.argmax())
    return float(r[i]), i


def accumulate(prefill, inc, b_inc):
    """out = prefill + increment, one fp32 add onto the caller's buffer -> (reference, bound)"""
    out = prefill.double() + inc
    return out, b_inc + U * (out.abs() + b_inc)


def sum_bound(terms, b_terms, depth, dim=None):
    """sum of fp32 terms (each within b_terms) by a chain / tree of the given depth -> (sum, bound)"""
    if dim is None:
        s, a, b = terms.sum(), terms.abs().sum(), b_terms.sum()
    else:
        s, a, b = terms.sum(dim), terms.abs().sum(dim), b_terms.sum(dim)
    return s, b + depth * U * (a + b)


# ------------------------------------------------------------------------------------------------------------------------
# running error bounds of element-wise fp32 formulas
# ------------------------------------------------------------------------------------------------------------------------
def _rnd(v, b, k=1):
    """k roundings of a result v already off by b: each errs by at most U |computed| <= U (|v| + b)"""
    return b + k * (U * (v.abs() + b) + TINY)


class V:
    """one fp32 kernel value: its fp64 reference v and a bound b on |kernel value - v|, carried through the kernel's own operations
    (first-order terms plus the cross terms of products).  libm errors are those of the CUDA maths library without fast maths:
    expf 2 ulp, logf / log1pf 1 ulp, division and sqrtf correctly rounded; one ulp is at most 2U relative."""

    def __init__(self, v, b=None):
        self.v = v
        self.b = torch.zeros_like(v) if b is None else (b if torch.is_tensor(b) else torch.full_like(v, b))

    @staticmethod
    def const(x, like, exact=False):
        """an fp32 literal or host-rounded argument standing for the real number x"""
        v = torch.full_like(like, x)
        return V(v, torch.zeros_like(v) if exact else U * v.abs())

    def __add__(self, o):
        v = self.v + o.v
        return V(v, _rnd(v, self.b + o.b))

    def __sub__(self, o):
        v = self.v - o.v
        return V(v, _rnd(v, self.b + o.b))

    def __mul__(self, o):
        v = self.v * o.v
        return V(v, _rnd(v, self.v.abs() * o.b + o.v.abs() * self.b + self.b * o.b))

    def __truediv__(self, o):
        v = self.v / o.v
        den = o.v.abs() - o.b
        prop = torch.where(den > 0, (self.b + v.abs() * o.b) / den.clamp(min=1e-300), torch.full_like(v, math.inf))
        return V(v, _rnd(v, prop))

    def __neg__(self):
        return V(-self.v, self.b)

    def where(self, cond, other):
        return V(torch.where(cond, self.v, other.v), torch.where(cond, self.b, other.b))

    def exp(self, cap=math.inf):
        """expf; cap: a bound on |kernel value - v| known beforehand (exp of a difference from a maximum lies in [0, 1])"""
        v = torch.exp(self.v)
        g = torch.exp(torch.clamp(self.b, max=700.0))
        return V(v, torch.clamp(v * torch.expm1(torch.clamp(self.b, max=700.0)) + 4 * U * v * g + TINY, max=cap))

    def log(self, ulps=1, floor=0.0):
        """logf; floor: a lower bound of both the kernel's argument and v (a sum of exps that includes exp(0) = 1 is >= 1)"""
        v = torch.log(self.v)
        den = torch.clamp(self.v - self.b, min=floor)
        prop = torch.where(den > 0, self.b / den.clamp(min=1e-300), torch.full_like(v, math.inf))
        return V(v, prop + 2 * ulps * U * (v.abs() + prop) + TINY)

    def sqrt(self):
        v = torch.sqrt(self.v)
        prop = torch.minimum(torch.sqrt(self.b), self.b / v.clamp(min=1e-300))
        return V(v, _rnd(v, prop))

    def sigmoid(self):
        """sigmoidf_acc: 1 / (1 + expf(-x)), 6U relative; sigmoid is monotone, so the input's error moves it at most to its value at
        x -+ b"""
        s = torch.sigmoid(self.v)
        hi, lo = torch.sigmoid(self.v + self.b), torch.sigmoid(self.v - self.b)
        prop = torch.maximum(hi - s, s - lo)
        return V(s, prop + 6 * U * hi + TINY)

    def softplus_t(self):
        """x > 20 ? x : log1pf(expf(x)): 6U relative; monotone like sigmoid.  The threshold switch at 20 moves the value by
        log1p(e^-20) < 3e-9, inside 6U |sp| there."""
        sp = lambda z: torch.where(z > 20, z, torch.nn.functional.softplus(z))      # noqa: E731
        v, hi, lo = sp(self.v), sp(self.v + self.b), sp(self.v - self.b)
        prop = torch.maximum(hi - v, v - lo)
        return V(v, prop + 6 * U * (v.abs() + prop) + TINY)

    def dsoftplus_t(self):
        """x > 20 ? 1 : sigmoidf_acc(x) (the switch moves it by 1 - sigmoid(20) < 3e-9 < 6U)"""
        s = self.sigmoid()
        big = self.v > 20
        return V(torch.where(big, torch.ones_like(s.v), s.v), torch.where(big, 6 * U + s.b, s.b + 6 * U))


def pick(cond, either, a, b):
    """a where cond, b elsewhere, and where `either` (the reference cannot tell which side the kernel took) their midpoint with half the
    difference added to the bound"""
    out = a.where(cond, b)
    mid = 0.5 * (a.v + b.v)
    half = 0.5 * (a.v - b.v).abs() + torch.maximum(a.b, b.b)
    return V(torch.where(either, mid, out.v), torch.where(either, half, out.b))


# ------------------------------------------------------------------------------------------------------------------------
# Tacotron loss (csrc/loss.cu)
# ------------------------------------------------------------------------------------------------------------------------
def loss_steps(target_len, R):
    """Tb = ceil(target_len / R): the steps of each utterance on the alignment's step grid"""
    return torch.div(target_len.long() + R - 1, R, rounding_mode='floor')


def guided_weight(B, S, L, text_len, target_len, R, g, device):
    """w[b, t, l] = 1 - exp(-(l / Lb - t / Tb)^2 / (2 g^2)) for t < Tb, l < Lb (else 0), as guided_weight() forms it in fp32 from
    inv2g2 = 1 / (2 g g) rounded on the host -> (V, valid).  The bound is absolute: 1 - e cancels for small d, and the error of d is
    carried through inv2g2 (200 at g = 0.05)."""
    Tb = loss_steps(target_len, R).to(device).double()[:, None, None]
    Lb = torch.clamp(text_len.long().to(device), max=L).double()[:, None, None]
    t = torch.arange(S, dtype=torch.float64, device=device)[None, :, None]
    l = torch.arange(L, dtype=torch.float64, device=device)[None, None, :]
    valid = (t < Tb) & (l < Lb)
    lf, tf = l / Lb, t / Tb
    d = V(lf, U * lf) - V(tf.expand_as(lf + tf), U * tf.expand_as(lf + tf))
    gf = float(np.float32(g))
    inv2g2 = 1.0 / (2.0 * gf * gf)
    arg = (-d) * d * V(torch.full_like(d.v, inv2g2), torch.full_like(d.v, 3 * U * inv2g2))       # -d d inv2g2, as the kernel orders it
    w = V.const(1.0, arg.v, exact=True) - arg.exp()
    return w, valid


def _stop_terms(stop, stop_t, pos_weight):
    """per-element stop BCE and its bound: (1 - y) x + (1 + (pw - 1) y) softplus(-x), softplus(-x) = log1pf(expf(-|x|)) + max(-x, 0)
    (the log1p part within 6U, +1 rounding); exact in the limit |x| -> inf"""
    x, y = stop.double(), stop_t.double()
    pw = float(np.float32(pos_weight))
    sp1 = torch.log1p(torch.exp(-x.abs()))
    sp = sp1 + torch.clamp(-x, min=0)
    a1 = (1 - y) * x
    wabs = 1 + abs(pw - 1) * y.abs()
    w = 1 + (pw - 1) * y
    bce = a1 + w * sp
    b = 2 * U * a1.abs() + 3 * U * wabs * sp + wabs * (6 * U * sp1 + U * sp) + U * (w * sp).abs() + U * bce.abs() + 4 * TINY
    return bce, b, x, y, pw, wabs


def tacotron_loss_forward(pre, pre_t, post, post_t, stop, stop_t, align, text_len, target_len, R, g, pos_weight, guided):
    """losses[4] = {2 MSE(pre), MSE(post), stop BCE / (N + 2), guided} as loss_partial_kernel + loss_final_kernel sum them: per thread
    float4 groups of the flat [B, N, T] range (3 adds a group, the nmel % 4 tail serially on one thread), the stop elements and the
    (b, t) rows of the guided term grid-strided over LOSS_BLOCKS x LT threads, a warp butterfly, 8 warp partials in order, the block
    partials in double, times the fp32-rounded scale -> {'losses': (ref [4], bound [4])}"""
    B, N, T = pre.shape
    dev = pre.device
    nthreads = LOSS_BLOCKS * LT
    nmel, nstop = B * N * T, B * T
    m_mel = -(-(-(-nmel // 4)) // nthreads)
    m_stop = -(-nstop // nthreads)
    ref, bnd = [], []
    for k, (a, at) in enumerate(((pre, pre_t), (post, post_t))):
        s = ((a.double() - at.double()) ** 2).sum()
        scale = (2.0 if k == 0 else 1.0) / nmel
        v = s * scale
        ref.append(v)
        bnd.append((m_mel + 3 + 3 + 3 + WARP_DEPTH + 8 + 1 + 2) * U * v.abs())      # square 3, group 3, tail 3, final scale + round 2
    bce, b_bce, *_ = _stop_terms(stop, stop_t, pos_weight)
    scale = 1.0 / (nstop * (N + 2))
    s, b_s = sum_bound(bce, b_bce, m_stop + WARP_DEPTH + 8 + 1)
    ref.append(s * scale)
    bnd.append(b_s * scale + 2 * U * (s * scale).abs())
    if guided:
        S, L = align.shape[1], align.shape[2]
        w, valid = guided_weight(B, S, L, text_len, target_len, R, g, dev)
        al = align.double()
        wv = torch.where(valid, w.v, torch.zeros_like(w.v))
        wb = torch.where(valid, w.b, torch.zeros_like(w.b))
        Tb = loss_steps(target_len, R).to(dev).double()
        Lb = torch.clamp(text_len.long().to(dev), max=L)
        rows_per_warp = -(-(B * S) // (nthreads // 32))
        lane_terms = (-(-Lb // 32)).double()                                  # each lane's chain over l = lane, lane + 32, ...
        per_row = (wv * al).sum(-1) / Tb[:, None]                             # [B, S]
        a_row = (wv * al).abs().sum(-1) / Tb[:, None]
        e_row = (wb * al.abs()).sum(-1) / Tb[:, None]
        depth = lane_terms[:, None] + 1 + 1 + rows_per_warp + WARP_DEPTH + 8 + 1
        v = per_row.sum() / B
        ref.append(v)
        bnd.append((e_row.sum() + (depth * U * (a_row + e_row)).sum()) / B + 2 * U * v.abs())
    else:
        ref.append(torch.zeros((), dtype=torch.float64, device=dev))
        bnd.append(torch.zeros((), dtype=torch.float64, device=dev))
    return {'losses': (torch.stack(ref), torch.stack(bnd))}


def tacotron_loss_backward(pre, pre_t, post, post_t, stop, stop_t, text_len, target_len, S, L, R, g, pos_weight, guided, grad_losses):
    """d_pre, d_post, d_stop, d_align of loss_backward_kernel: each element one formula times gl[k] c_k, c_k rounded on the host.
    d_align is exactly 0 where t >= Tb, l >= Lb or the guided term is off."""
    B, N, T = pre.shape
    dev = pre.device
    gl = [float(x) for x in grad_losses]
    nmel, nstop = B * N * T, B * T
    out = {}
    for name, (a, at), c in (('d_pre', (pre, pre_t), 4.0 / nmel), ('d_post', (post, post_t), 2.0 / nmel)):
        ref = gl[0 if name == 'd_pre' else 1] * c * (a.double() - at.double())
        out[name] = (ref, 4 * U * ref.abs() + 4 * TINY)
    x, y = stop.double(), stop_t.double()
    pw = float(np.float32(pos_weight))
    sneg = torch.sigmoid(-x)
    w = 1 + (pw - 1) * y
    wabs = 1 + abs(pw - 1) * y.abs()
    inner = (1 - y) - w * sneg
    G = gl[2] / (nstop * (N + 2))
    ref = G * inner
    out['d_stop'] = (ref, abs(G) * (U * (1 - y).abs() + 10 * U * wabs * sneg + U * inner.abs()) + 3 * U * ref.abs() + 4 * TINY)
    if guided:
        wv, valid = guided_weight(B, S, L, text_len, target_len, R, g, dev)
        Tb = loss_steps(target_len, R).to(dev).double()[:, None, None]
        Ga = gl[3] / B
        ref = torch.where(valid, Ga * wv.v / Tb, torch.zeros_like(wv.v))
        b = torch.where(valid, abs(Ga) * wv.b / Tb + 4 * U * ref.abs() + 4 * TINY, torch.zeros_like(wv.v))
    else:
        ref = b = torch.zeros(B, S, L, dtype=torch.float64, device=dev)
    out['d_align'] = (ref, b)
    return out


# ------------------------------------------------------------------------------------------------------------------------
# WaveRNN upsampling layer and aux stretch adjoints, column sums
# ------------------------------------------------------------------------------------------------------------------------
def upsample_backward(fir, x, dout, scale):
    """din [C, len] and the increment of dfir [2 s + 1] of one upsampling layer (nearest stretch x s, FIR of 2 s + 1 taps, zero padding s).
    din: one fmaf chain over the s (2 s + 1) (p, k) pairs of each input position.  dfir: per tap, UPS_CHUNKS slices of the flat (c, i)
    range, 256 strided fmaf chains each and a block sum, then the chunks in order."""
    C, ln = x.shape
    s = scale
    lo = ln * s
    w, d = fir.double().reshape(-1), dout.double()
    wt = w.flip(0)[None, None, :]
    # dx[c, q] = sum_k w[k + s] dout[c, q - k] over 0 <= q - k < lo  (the adjoint of conv1d(x, w, padding s))
    dx = torch.nn.functional.conv1d(d[:, None, :], wt, padding=s)[:, 0]
    ax = torch.nn.functional.conv1d(d.abs()[:, None, :], wt.abs(), padding=s)[:, 0]
    din = dx.reshape(C, ln, s).sum(-1)
    a_din = ax.reshape(C, ln, s).sum(-1)
    out = {'din': (din, s * (2 * s + 1) * U * a_din + TINY)}
    xs = x.double().repeat_interleave(s, dim=1)                     # [C, lo]
    per = -(-(C * lo) // UPS_CHUNKS)
    depth = -(-per // 256) + BLOCK_SUM_DEPTH + UPS_CHUNKS
    ref, bnd = [], []
    for k in range(-s, s + 1):
        i0, i1 = max(0, -k), lo - max(0, k)
        prod = d[:, i0:i1] * xs[:, i0 + k:i1 + k]
        ref.append(prod.sum())
        bnd.append(depth * U * prod.abs().sum() + TINY)
    out['dfir'] = (torch.stack(ref), torch.stack(bnd))
    return out


def stretch_backward(dup, F, hop):
    """daux[b, f, c] = sum_{q < hop} dup[b, f hop + q, c], one chain per element"""
    B, _, C = dup.shape
    d = dup.double().reshape(B, F, hop, C)
    return {'daux': (d.sum(2), hop * U * d.abs().sum(2) + TINY)}


def column_sum(x):
    """the increment of out[col]: COLSUM_CHUNKS chains of ceil(rows / 64) rows, then the chunks in order"""
    rows = x.shape[0]
    per = -(-rows // COLSUM_CHUNKS)
    xd = x.double()
    return {'out': (xd.sum(0), (per + COLSUM_CHUNKS) * U * xd.abs().sum(0) + TINY)}


# ------------------------------------------------------------------------------------------------------------------------
# WaveRNN losses
# ------------------------------------------------------------------------------------------------------------------------
def _mean_of_rows(row, b_row):
    """wavernn_loss_sum_kernel: thread i chains rows i, i + 1024, ..., a block sum, then / N in double, rounded"""
    N = row.numel()
    depth = -(-N // LOSS_SUM_THREADS) + BLOCK_SUM_DEPTH
    s, b = sum_bound(row, b_row, depth)
    return s / N, b / N + U * (s / N).abs() + TINY


def raw_loss(logits, labels):
    """cross entropy per row (one warp: lanes over the classes, warp max and butterfly sum), d logits = (softmax - onehot) / N.  A label
    outside [0, n) gives the row a NaN loss (and so a NaN mean) and d logits = softmax / N.
    -> {'loss': ([1]), 'rows': ([N]), 'dlogits': ([N, n])}"""
    N, n = logits.shape
    l = logits.double()
    lab = labels.long()
    ok = (lab >= 0) & (lab < n)
    mx = l.max(1, keepdim=True).values
    e = (V(l) - V(mx.expand_as(l))).exp(cap=1.0)                    # exp(l - max) lies in [0, 1] in both
    s, b_s = sum_bound(e.v, e.b, -(-n // 32) + WARP_DEPTH, dim=1)
    sv = V(s[:, None], b_s[:, None])
    inv = V.const(1.0, sv.v, exact=True) / sv
    sm = e * inv
    onehot = torch.zeros_like(l)
    onehot[ok, lab[ok]] = 1.0
    d = (sm - V(onehot)) * V.const(1.0 / N, l)
    row = sv.log(floor=1.0) + V(mx) - V(l.gather(1, lab.clamp(0, n - 1)[:, None]))
    rv = torch.where(ok, row.v[:, 0], torch.full_like(row.v[:, 0], math.nan))
    rb = torch.where(ok, row.b[:, 0], torch.zeros_like(row.b[:, 0]))
    loss, b_loss = _mean_of_rows(rv, rb)
    return {'loss': (loss.reshape(1), b_loss.reshape(1)), 'rows': (rv, rb), 'dlogits': (d.v, d.b)}


def max_offsets(a):
    """a - max(a) over the last dimension, as the kernel forms it from its own a (a warp_max, then one subtraction per lane).  Where
    one lane k leads every other by more than their two bounds, the kernel's maximum is its own a_k: a_k - M is exactly 0 and lane j's
    offset is off by at most b_j + b_k.  Elsewhere the kernel's maximum is within max b of the fp64 one."""
    v, b = a.v, a.b
    M, k = v.max(-1, keepdim=True)
    bk = b.gather(-1, k)
    lane = torch.arange(v.shape[-1], device=v.device)
    is_k = lane == k
    others = torch.where(is_k, torch.full_like(v, -math.inf), v + b)
    lead = (M - bk > others.max(-1, keepdim=True).values) if v.shape[-1] > 1 else torch.ones_like(M, dtype=torch.bool)
    off = v - M
    b_lead = torch.where(is_k, torch.zeros_like(b), _rnd(off, b + bk))
    b_any = _rnd(off, b + b.max(-1, keepdim=True).values)
    return V(off, torch.where(lead, b_lead, b_any))


def mol_branches(y):
    """the kernel's fp32 branch of each row: y < -0.999f (left edge), y > 0.999f (right edge), else the middle"""
    y32 = y.float()
    return y32 < np.float32(-0.999), y32 > np.float32(0.999)


def mol_loss(logits, y):
    """fatchord's discretized_mix_logistic_loss as wavernn_loss_mol_kernel forms it: lane j the mixture j of the row, the row's edge
    branch picked in fp32; in the middle the cdf_delta > 1e-5 branch, where the fp64 cdf_delta within its own bound of 1e-5 accepts
    either branch.  The log-scale clamp passes gradient where lsr >= log(1e-14)f.  -> {'loss', 'rows', 'dlogits'}"""
    N, n3 = logits.shape
    nr = n3 // 3
    l = logits.double()
    lp, mu, lsr = l[:, :nr], l[:, nr:2 * nr], l[:, 2 * nr:]
    yv = y.double()[:, None].expand_as(mu)
    a, b = mol_branches(y)
    lo_e, hi_e = a[:, None].expand_as(mu), b[:, None].expand_as(mu)
    ls = torch.clamp(lsr, min=LOG_SCALE_MIN)
    cy = V(yv) - V(mu)
    inv = (-V(ls)).exp()
    hb = V.const(HALF_BIN, mu)
    plus, mn, mid = inv * (cy + hb), inv * (cy - hb), inv * cy
    zero = V(torch.zeros_like(mu))
    one = V.const(1.0, mu, exact=True)
    # left edge
    lp_lo = plus - plus.softplus_t()
    dplus_lo = one - plus.dsoftplus_t()
    # right edge
    sp_mn = mn.softplus_t()
    lp_hi = V(-sp_mn.v, sp_mn.b)
    dmin_hi = -mn.dsoftplus_t()
    # middle, cdf_delta branch
    cp, cm = plus.sigmoid(), mn.sigmoid()
    cd = cp - cm
    lp_cd = cd.log()
    dplus_cd = cp * (one - cp) / cd
    dmin_cd = -(cm * (one - cm) / cd)
    # middle, pdf branch
    lp_pdf = mid - V(ls) - V.const(2.0, mu, exact=True) * mid.softplus_t() - V.const(LOG_HALF_CLASSES, mu)
    dmid_pdf = one - V.const(2.0, mu, exact=True) * mid.dsoftplus_t()
    use_cd = cd.v > CDF_FLOOR
    either = (cd.v - CDF_FLOOR).abs() <= cd.b
    middle = ~(lo_e | hi_e)
    edge_either = either & middle

    def choose(v_lo, v_hi, v_cd, v_pdf):
        mid_v = pick(use_cd, edge_either, v_cd, v_pdf)
        return v_lo.where(lo_e, v_hi.where(hi_e, mid_v))
    logprob = choose(lp_lo, lp_hi, lp_cd, lp_pdf)
    dplus = choose(dplus_lo, zero, dplus_cd, zero)
    dmin = choose(zero, dmin_hi, dmin_cd, zero)
    dmid = choose(zero, zero, zero, dmid_pdf)
    dls_direct = choose(zero, zero, zero, V.const(-1.0, mu, exact=True))
    dmu_l = -(inv * (dplus + dmin + dmid))
    dls_l = dls_direct - (plus * dplus + mn * dmin + mid * dmid)
    gate = lsr >= LOG_SCALE_MIN
    dls_l = dls_l.where(gate, zero)
    # logsumexp over the mixtures (warp max / butterfly sums over nr <= 32 lanes)
    m = lp.max(1, keepdim=True).values.expand_as(lp)
    e = (V(lp) - V(m)).exp(cap=1.0)
    s, b_s = sum_bound(e.v, e.b, WARP_DEPTH, dim=1)
    sv = V(s[:, None].expand_as(lp), b_s[:, None].expand_as(lp))
    a = logprob + ((V(lp) - V(m)) - sv.log(floor=1.0))
    am = max_offsets(a)
    M, bM = a.v.max(1, keepdim=True).values.expand_as(lp), a.b.max(1, keepdim=True).values.expand_as(lp)
    ea = am.exp(cap=1.0)
    S, b_S = sum_bound(ea.v, ea.b, WARP_DEPTH, dim=1)
    Sv = V(S[:, None].expand_as(lp), b_S[:, None].expand_as(lp))
    w, sm = ea / Sv, e / sv
    invN = V.const(1.0 / N, lp)
    gmix = -(w * invN)
    d_lp = (sm - w) * invN
    d_mu, d_ls = gmix * dmu_l, gmix * dls_l
    row = V(M, bM) + Sv.log(floor=1.0)
    loss, b_loss = _mean_of_rows(row.v[:, 0], row.b[:, 0])
    return {'loss': ((-loss).reshape(1), b_loss.reshape(1)), 'rows': (-row.v[:, 0], row.b[:, 0]),
            'dlogits': (torch.cat([d_lp.v, d_mu.v, d_ls.v], 1), torch.cat([d_lp.b, d_mu.b, d_ls.b], 1))}


# ------------------------------------------------------------------------------------------------------------------------
# fused clip + Adam (csrc/optim.cu)
# ------------------------------------------------------------------------------------------------------------------------
def norm_blocks(n):
    """blocks of sqnorm_partial_kernel: one per 256 float4 groups, 1 to NORM_BLOCKS"""
    return min(max((n // 4 + 255) // 256, 1), NORM_BLOCKS)


def clip_min1(c):
    """min(1, c) of a kernel value within c.b of c.v: the kernel's value lies in [c.v - c.b, c.v + c.b] clamped to at most 1.  Where
    c.v - c.b > 1 it is exactly 1; where c.v >= 1 it is off by at most 1 - (c.v - c.b); below 1 by at most c.b."""
    lo = c.v - c.b
    b = torch.where(lo > 1, torch.zeros_like(c.b), torch.where(c.v >= 1, torch.clamp(1 - lo, min=0), c.b))
    return V(torch.clamp(c.v, max=1.0), b)


def adam_clip(p, g, m, v, lr, beta1, beta2, eps, weight_decay, max_norm, step):
    """one b200tts_adam_clip_step in fp64 from the same inputs: the gradient norm (4 fmaf chains of float4 lanes per thread, block 0
    adds the n % 4 tail to lane 0, a block sum, then the partials strided over 256 threads and a block sum, sqrtf), the clip
    coefficient min(1, max_norm / (norm + 1e-6)), and the element-wise update.  Scalars are the fp32 values the kernel receives.
    -> {'norm', 'coef', 'p', 'g', 'm', 'v'}"""
    f = lambda x: float(np.float32(x))                               # noqa: E731
    lr, beta1, beta2, eps, weight_decay, max_norm = map(f, (lr, beta1, beta2, eps, weight_decay, max_norm))
    n = g.numel()
    gd = g.double()
    nblk = norm_blocks(n)
    m_thr = -(-(n // 4) // (nblk * 256))
    depth = m_thr + 1 + 2 + BLOCK_SUM_DEPTH + -(-nblk // 256) + BLOCK_SUM_DEPTH
    sq = (gd * gd).sum()
    nrm = V(sq.reshape(1), (depth * U * sq).reshape(1)).sqrt()
    out = {'norm': (nrm.v, nrm.b)}
    one = V.const(1.0, nrm.v, exact=True)
    if max_norm > 0:
        c = clip_min1(V.const(max_norm, nrm.v, exact=True) / (nrm + V.const(1e-6, nrm.v)))
    else:
        c = one
    out['coef'] = (c.v, c.b)
    coef = V(c.v.expand_as(gd), c.b.expand_as(gd))
    gc = V(gd) * coef
    out['g'] = (gc.v, gc.b)
    gi = V.const(weight_decay, gd, exact=True) * V(p.double()) + gc if weight_decay != 0 else gc
    b1, b2 = V.const(beta1, gd, exact=True), V.const(beta2, gd, exact=True)
    omb1, omb2 = V.const(1.0, gd, exact=True) - b1, V.const(1.0, gd, exact=True) - b2
    mi = b1 * V(m.double()) + omb1 * gi
    vi = b2 * V(v.double()) + omb2 * gi * gi
    out['m'], out['v'] = (mi.v, mi.b), (vi.v, vi.b)
    bc1 = 1.0 - beta1 ** step
    bc2s = math.sqrt(1.0 - beta2 ** step)
    denom = vi.sqrt() / V.const(bc2s, gd) + V.const(eps, gd, exact=True)
    step_size = V.const(lr, gd, exact=True) / V.const(bc1, gd)
    pn = V(p.double()) - step_size * (mi / denom)
    out['p'] = (pn.v, pn.b)
    return out
