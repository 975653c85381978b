"""Step-local fp64 check of the decoder recurrences, from the state the kernels saved.

Step i of every recurrence is recomputed in fp64 from the kernel's OWN saved state of step i-1 (decoder_workspace.py views), so
the reference never drifts off the kernel's trajectory and every element of every step gets its own bound:

    err   = |kernel value - fp64 reference|
    bound = fp32 accumulation bound K * 2^-24 * (|A| . |B|) of each product (computed in the same fp64 pass)
            + the documented maximum error of the approximate nonlinearities, propagated through Lipschitz constants

The reference rounds exactly the operands the kernel rounds (`mode`):
    'persist'     bf16 mode on the persistent TMA + wgmma loops (decoder_persist_tc.cu, decoder_persist_bwd_tc.cu,
                  decoder_persist_bwd.cu): bf16 weights and operand rows, ex2-based gate math, tanh.approx energies
    'chain_bf16'  bf16 mode on the per-step kernel chains: bf16 operands in every GEMM (gemm_bf16.cu), accurate math elsewhere
    'fp32'        fp32 mode (per-step chains): no rounding model at all
Every rounding point is named with the source line it models.  There is no blanket relative tolerance anywhere.

Each check_* function fills a Report: per stage, the worst err / bound ratio of every step and where the overall worst sits.
"""
import math

import torch
import torch.nn.functional as Fn

U = 2.0 ** -24                 # fp32 unit roundoff
ULP1 = 2.0 ** -23              # one fp32 ulp, relative (upper bound)
# a bf16 hi + lo split of an fp32 value x (hi = RN(x), lo = RN(x - hi)) leaves |x - hi - lo| <= 2^-9 |x - hi| <= 2^-18 |x|; a product
# hi.hi + lo.hi + hi.lo then misses at most lo.lo + the two residuals: < 2^-16 of |a| |b|
SPLIT_REL = 2.0 ** -16
# tanh.approx.f32: maximum relative error 2^-10.987 (PTX ISA, tanh); the absolute floor covers the subnormal-range behaviour
TANH_APPROX_REL, TANH_APPROX_ABS = 2.0 ** -10.987, 2.0 ** -22
MODES = ('persist', 'chain_bf16', 'fp32')


# ------------------------------------------------------------------------------------------------------------------------
# report
# ------------------------------------------------------------------------------------------------------------------------
class Report:
    """Per stage: worst err / bound ratio per step ([T] float64) and the overall worst (ratio, step, index, err, bound)."""

    def __init__(self, T):
        self.T = T
        self.per_step = {}
        self.worst = {}

    def add(self, stage, step0, err, bound):
        """err / bound: [S, ...] for steps step0 .. step0 + S - 1.  A zero bound admits only a zero error."""
        err, bound = err.double(), bound.double()
        ratio = torch.where(err == 0, torch.zeros_like(err), err / bound)
        ratio = torch.nan_to_num(ratio, nan=math.inf)
        S = ratio.shape[0]
        flat = ratio.reshape(S, -1)
        per, arg = flat.max(1) if flat.shape[1] else (torch.zeros(S, dtype=torch.float64), torch.zeros(S, dtype=torch.long))
        ps = self.per_step.setdefault(stage, torch.zeros(self.T, dtype=torch.float64))
        ps[step0:step0 + S] = torch.maximum(ps[step0:step0 + S], per.cpu())
        j = int(per.argmax())
        r = float(per[j])
        if stage not in self.worst or r > self.worst[stage]['ratio']:
            idx = tuple(int(x) for x in torch.unravel_index(arg[j].cpu(), ratio.shape[1:])) if flat.shape[1] else ()
            e = float(err.reshape(S, -1)[j, arg[j]]) if flat.shape[1] else 0.0
            b = float(bound.reshape(S, -1)[j, arg[j]]) if flat.shape[1] else 0.0
            self.worst[stage] = {'ratio': r, 'step': step0 + j, 'index': idx, 'err': e, 'bound': b}

    def failures(self):
        """{stage: [steps with ratio > 1]}"""
        out = {}
        for stage, ps in self.per_step.items():
            bad = torch.nonzero(ps > 1.0).flatten().tolist()
            if bad:
                out[stage] = bad
        return out

    def max_ratio(self):
        return max((w['ratio'] for w in self.worst.values()), default=0.0)

    def lines(self, title=''):
        out = []
        for stage in sorted(self.worst):
            w = self.worst[stage]
            out.append(f'{title}{stage:>10s}: worst err/bound {w["ratio"]:.3e} at step {w["step"]} index {w["index"]} '
                       f'(err {w["err"]:.3e}, bound {w["bound"]:.3e})')
        return out


# ------------------------------------------------------------------------------------------------------------------------
# rounding model and nonlinearities
# ------------------------------------------------------------------------------------------------------------------------
def rn(x):
    """fp32 -> bf16 round-to-nearest-even (__float2bfloat16_rn), back in fp64."""
    return x.float().to(torch.bfloat16).double()


def rw(w, mode):
    """A weight as the products read it: bf16 RN in both bf16 modes (decoder_persist_tc.cu:281, decoder_persist_bwd_tc.cu:114,
    decoder_persist_bwd.cu:191 pack the resident slices that way; gemm_bf16.cu:83-91 packs every GEMM operand the same way)."""
    return w.double() if mode == 'fp32' else rn(w)


def ra(x, mode):
    """An fp32 activation operand of a bf16-mode GEMM (gemm_bf16.cu:83-91); unrounded in fp32 mode."""
    return x.double() if mode == 'fp32' else rn(x)


def product(a, w):
    """a [..., K] . w[N, K]^T and its worst-case fp32 accumulation bound (K + 2) 2^-24 (|a| . |w|^T)."""
    y = a @ w.t()
    return y, (a.shape[-1] + 2) * U * (a.abs() @ w.abs().t())


def sigmoid_err(z, mode):
    """Maximum error of the gate sigmoid.  persist: sigmoid_fast = __fdividef(1, 1 + __expf(-x)) (decoder_persist_tc.cu:164):
    __expf is within 2 + floor(|1.173 x|) ulp and __fdividef within 2 ulp (CUDA C++ Programming Guide, intrinsic functions);
    an error e of exp(-x) moves 1 / (1 + exp(-x)) by s (1 - s) e.  Otherwise sigmoidf_acc = 1 / (1 + expf(-x)) (common.cuh:97):
    expf within 2 ulp, IEEE division."""
    s = torch.sigmoid(z)
    if mode == 'persist':
        return s * (1 - s) * ((2 + 1.173 * z.abs()) * ULP1 + U) + 2 * ULP1 * s
    return s * (1 - s) * (2 * ULP1 + U) + U * s


def tanh_gate_err(x, mode):
    """persist: tanh_exp(x) = 2 sigmoid_fast(2x) - 1 (decoder_persist_tc.cu:165); otherwise tanhf (2 ulp)."""
    if mode == 'persist':
        return 2 * sigmoid_err(2 * x, mode) + 2 * U
    return 2 * ULP1 * torch.tanh(x).abs() + U * 2.0 ** -100


def activate(z, mode):
    """LSTM gate activations (i, f, g, o; torch LSTMCell order) of pre-activations z [..., 4D] -> (gates, lipschitz, approx err)."""
    D = z.shape[-1] // 4
    g = torch.sigmoid(z)
    g[..., 2 * D:3 * D] = torch.tanh(z[..., 2 * D:3 * D])
    lip = torch.full_like(z, 0.25)
    lip[..., 2 * D:3 * D] = 1.0
    err = sigmoid_err(z, mode)
    err[..., 2 * D:3 * D] = tanh_gate_err(z[..., 2 * D:3 * D], mode)
    return g, lip, err


def wcomb_fp32(w_loc, w_c):
    """Wcomb[a, k] = sum_c Wloc[a, c] Wc[c, k] in fp32 with one fmaf per c, as wcomb_kernel (decoder_persist.cu:72-79) forms it:
    the bf16 copy the energies read (decoder_persist.cu:32) is the RN of exactly this fp32 value.  -> [A, K]"""
    A, C = w_loc.shape
    wc = w_c.reshape(C, -1)
    s = torch.zeros(A, wc.shape[1], dtype=torch.float32, device=w_loc.device)
    for c in range(C):
        s = (w_loc[:, c:c + 1].double() * wc[c:c + 1].double() + s.double()).float()
    return s


# ------------------------------------------------------------------------------------------------------------------------
# one step of each recurrence (shared by the checker and the synthetic workspace of the CPU tests)
# ------------------------------------------------------------------------------------------------------------------------
def cell_forward(gates, cp, hp, mh, mc, cfg, mode):
    """LSTM cell + regulariser from the kernel's activated gates (decoder_persist_tc.cu:503-520, decoder_fwd.cu:100-117).
    -> (c, h, bound c, bound h)"""
    D = cp.shape[-1]
    gi, gf, gg, go = gates[..., :D], gates[..., D:2 * D], gates[..., 2 * D:3 * D], gates[..., 3 * D:]
    cn = gf * cp + gi * gg
    b_cn = 2 * U * ((gf * cp).abs() + (gi * gg).abs())
    tc = torch.tanh(cn)
    b_tc = b_cn + tanh_gate_err(cn, mode)
    hn = go * tc
    b_hn = go.abs() * b_tc + U * hn.abs()
    if cfg.kind == 1:       # zoneout
        if cfg.training:
            kh = (1 - cfg.rate_h) * (mh.double() / (1 - cfg.rate_h) if mh is not None else 1.0)
            kc = (1 - cfg.rate_c) * (mc.double() / (1 - cfg.rate_c) if mc is not None else 1.0)
        else:
            kh, kc = 1 - cfg.rate_h, 1 - cfg.rate_c
        h = kh * (hn - hp) + hp
        c = kc * (cn - cp) + cp
        b_h = abs_(kh) * b_hn + 6 * U * (hn.abs() + hp.abs()) * (1 + abs_(kh))
        b_c = abs_(kc) * b_cn + 6 * U * (cn.abs() + cp.abs()) * (1 + abs_(kc))
        return c, h, b_c, b_h
    if cfg.training and mh is not None:
        k = mh.double() / (1 - cfg.rate_h)
        return cn, hn * k, b_cn, k * b_hn + 3 * U * (hn * k).abs()
    return cn, hn, b_cn, b_hn


def abs_(k):
    return k.abs() if torch.is_tensor(k) else abs(k)


def cell_backward(dh, b_dh, dc, b_dc, gates, cp, mh, mc, cfg, mode):
    """LSTM cell backward (decoder_persist_bwd_tc.cu:190-213, decoder_persist_bwd.cu:625-649, decoder_bwd.cu:221-245).
    dh / dc: total incoming gradients of h_out / c_out.  -> (dgates, bound, dc_prev, bound, dhz_prev, bound)"""
    D = cp.shape[-1]
    gi, gf, gg, go = gates[..., :D], gates[..., D:2 * D], gates[..., 2 * D:3 * D], gates[..., 3 * D:]
    cr = gf * cp + gi * gg
    tc = torch.tanh(cr)
    b_tc = tanh_gate_err(cr, mode) + 2 * U * ((gf * cp).abs() + (gi * gg).abs())
    dtc = go * (1 - tc * tc)
    b_dtc = go.abs() * 2 * tc.abs() * b_tc + 3 * U * dtc.abs()
    if cfg.kind == 1:
        if cfg.training:
            kh = (1 - cfg.rate_h) * (mh.double() / (1 - cfg.rate_h) if mh is not None else 1.0)
            kc = (1 - cfg.rate_c) * (mc.double() / (1 - cfg.rate_c) if mc is not None else 1.0)
        else:
            kh, kc = 1 - cfg.rate_h, 1 - cfg.rate_c
        dhn = dh * kh
        b_dhn = abs_(kh) * b_dh + 3 * U * dhn.abs()
        dhz = dh - dhn
        b_dhz = abs_(1 - kh) * b_dh + U * (dh.abs() + dhn.abs())
        dcn = dc * kc + dhn * dtc
        b_dcn = abs_(kc) * b_dc + dtc.abs() * b_dhn + dhn.abs() * b_dtc + 3 * U * ((dc * kc).abs() + (dhn * dtc).abs())
        dcp_direct = dc - dc * kc
        b_direct = abs_(1 - kc) * b_dc + 2 * U * (dc.abs() + (dc * kc).abs())
    else:
        k = mh.double() / (1 - cfg.rate_h) if (cfg.training and mh is not None) else 1.0
        dhn = dh * k
        b_dhn = abs_(k) * b_dh + 3 * U * dhn.abs()
        dhz, b_dhz = torch.zeros_like(dh), torch.zeros_like(dh)
        dcn = dc + dhn * dtc
        b_dcn = b_dc + dtc.abs() * b_dhn + dhn.abs() * b_dtc + 2 * U * (dc.abs() + (dhn * dtc).abs())
        dcp_direct, b_direct = torch.zeros_like(dc), torch.zeros_like(dc)
    fac = torch.cat([gg * gi * (1 - gi), cp * gf * (1 - gf), gi * (1 - gg * gg)], -1)
    d3 = dcn.repeat(*([1] * (dcn.dim() - 1)), 3) * fac
    b3 = b_dcn.repeat(*([1] * (dcn.dim() - 1)), 3) * fac.abs() + 5 * U * d3.abs()
    fo = go * (1 - go)
    dO = dhn * tc * fo
    b_dO = (tc * fo).abs() * b_dhn + (dhn * fo).abs() * b_tc + 5 * U * dO.abs()
    dgates = torch.cat([d3, dO], -1)
    b_dgates = torch.cat([b3, b_dO], -1)
    dc_prev = dcn * gf + dcp_direct
    b_dc_prev = gf.abs() * b_dcn + b_direct + 2 * U * ((dcn * gf).abs() + dcp_direct.abs())
    return dgates, b_dgates, dc_prev, b_dc_prev, dhz, b_dhz


def energy_tanh(q, cum, memTr, prm, mode, wcomb=None):
    """t = tanh(location term + q + bias + memT) [S, B, L, A] and its bound.  persist (forward: decoder_persist_tc.cu:622-702;
    reverse: decoder_persist_bwd.cu:339-346, :438-469): location term on the tensor cores from the bf16 Wcomb and a hi + lo split of
    cum, bf16 memory projection, tanh.approx.  Otherwise the per-step kernels: fp32 location convolution, fp32 projection, tanhf."""
    S, B, L = cum.shape
    Wc = prm['attn_loc_features']
    C, K = Wc.shape[0], Wc.shape[-1]
    half = (K - 1) // 2
    unf = Fn.pad(cum.double(), (half, K - 1 - half)).unfold(-1, K, 1)          # [S, B, L, K]: cum[l + k - half]
    if mode == 'persist':
        wcb = rn(wcomb if wcomb is not None else wcomb_fp32(prm['attn_location'], Wc))       # [A, K] (decoder_persist.cu:32)
        loc = unf @ wcb.t()
        b_loc = (K + 2) * U * (unf.abs() @ wcb.abs().t()) + SPLIT_REL * (unf.abs() @ wcb.abs().t())   # cum hi + lo (:622-633)
    else:
        wl, wc = prm['attn_location'].double(), Wc.reshape(C, K).double()
        loc = unf @ (wl @ wc).t()
        b_loc = (K + C + 2) * U * (unf.abs() @ (wl.abs() @ wc.abs()).t())
    qb = q.double() + prm['attn_bias'].reshape(-1).double()                       # qb = q + bias (:652), one fp32 add
    x = loc + qb[:, :, None, :] + memTr[None]
    b_x = b_loc + U * qb.abs()[:, :, None, :] + 2 * U * (loc.abs() + qb.abs()[:, :, None, :] + memTr.abs()[None])
    t = torch.tanh(x)
    if mode == 'persist':
        b_t = b_x + TANH_APPROX_REL * t.abs() + TANH_APPROX_ABS                   # tanh_fast (:699-702)
    else:
        b_t = b_x + 2 * ULP1 * t.abs()
    return t, b_t


def attention_weights(q, cum, memTr, lengths, prm, mode, wcomb=None):
    """Alignment row of the location-sensitive attention for steps [S] at once: q [S, B, A], cum [S, B, L] (the kernel's own):
    energies from energy_tanh, softmax over the text length (decoder_persist_tc.cu:722-739).  -> (weights [S, B, L], bound, valid)"""
    S, B, L = cum.shape
    t, b_t = energy_tanh(q, cum, memTr, prm, mode, wcomb)
    v = prm['attn_energy'].reshape(-1).double()
    A = v.numel()
    e = t @ v
    b_e = b_t @ v.abs() + (A + 2) * U * (t.abs() @ v.abs())
    lens = lengths.to(cum.device).long().clamp(0, L)
    valid = torch.arange(L, device=cum.device)[None, :] < lens[:, None]           # [B, L]
    em = e.masked_fill(~valid[None], -math.inf)
    w = torch.softmax(em, -1).masked_fill(~valid[None], 0.0)
    spread = (e - em.max(-1, keepdim=True).values).abs().masked_fill(~valid[None], 0.0)
    b_ew = b_e.masked_fill(~valid[None], 0.0)
    b_w = w * (b_ew + (w * b_ew).sum(-1, keepdim=True)) + w * (U * spread + (lens[None, :, None].double() + 8) * U)
    return w, b_w, valid


def _dims(v):
    T, B, D4 = v['ga'].shape
    D = D4 // 4
    return T, B, D, v['ai'].shape[2] - D, v['cum'].shape[2], v['q'].shape[2]


def _chunk(v, budget=2.5e7):
    T, B, D, M, L, A = _dims(v)
    return max(1, min(T, int(budget // max(B * max(L * A, 4 * D, L * M), 1))))


def att_operand(v, i0, i1, mode):
    """[h_att | ctx] operand rows of attention-LSTM steps i0 .. i1-1 as the product read them.  persist: the bf16 rows aib the loop
    fed to wgmma (decoder_persist_tc.cu:523, :817-821); chains: RN of the fp32 rows [ctx | h_att] of ai (decoder_fwd.cu:535)."""
    T, B, D, M, L, A = _dims(v)
    if mode == 'persist':
        return v['aib'][i0:i1, :, :D + M].double()
    ai = v['ai'][i0:i1]
    return torch.cat([ra(ai[..., M:], mode), ra(ai[..., :M], mode)], -1)


def gen_operand(v, i0, i1, mode):
    """h_gen operand rows of generator steps i0 .. i1-1: hgb (persist) or RN of hg."""
    T, B, D, M, L, A = _dims(v)
    return v['hgb'][i0:i1, :, :D].double() if mode == 'persist' else ra(v['hg'][i0:i1], mode)


def att_preact(v, prm, a, i0, i1, mode):
    """attention-LSTM pre-activations of steps i0 .. i1-1 from operand rows a [S, B, D + M] ([h_att | ctx]) -> (z, bound).
    The input projection p1 . W_ih[:, :P]^T + b_ih + b_hh is a time-batched bf16 GEMM (decoder_fwd.cu:655)."""
    P = v['p1'].shape[2]
    W = prm['att_w_ih']
    xp, b_xp = product(ra(v['p1'][i0:i1], mode), rw(W[:, :P], mode))
    bsum = (prm['att_b_ih'].double() + prm['att_b_hh'].double()).float().double()    # bsum_att: one fp32 add (decoder_fwd.cu:641)
    xp = xp + bsum
    b_xp = b_xp + U * bsum.abs() + U * xp.abs()
    Wr = torch.cat([rw(prm['att_w_hh'], mode), rw(W[:, P:], mode)], 1)          # operand column order [h | ctx]
    rec, b_rec = product(a, Wr)
    z = xp + rec
    return z, b_xp + b_rec + U * z.abs()


def gen_preact(v, prm, a_in, h_prev, mode):
    """generator-LSTM pre-activations from the input rows a_in [S, B, D + M] = [h_att | ctx] of step i+1 (the input projection is
    one bf16 GEMM over those rows, decoder_fwd.cu:687-694) and the operand rows h_prev of step i -> (z, bound)"""
    xp, b_xp = product(a_in, rw(prm['gen_w_ih'], mode))
    bsum = (prm['gen_b_ih'].double() + prm['gen_b_hh'].double()).float().double()
    xp = xp + bsum
    rec, b_rec = product(h_prev, rw(prm['gen_w_hh'], mode))
    z = xp + rec
    return z, b_xp + b_rec + 2 * U * (bsum.abs() + xp.abs() + z.abs())


# ------------------------------------------------------------------------------------------------------------------------
# forward
# ------------------------------------------------------------------------------------------------------------------------
def check_forward(v, prm, masks, cfg, lengths, memory, align, mode, report=None):
    """Every stage of every forward step.  v: workspace views (decoder_workspace.py), prm: {DECODER_PARAM_FIELDS name: fp32
    tensor}, masks: {name: uint8 [T, B, D] or None}, align: [B, T, L] output of the decode.  Returns the Report."""
    assert mode in MODES
    T, B, D, M, L, A = _dims(v)
    rep = report or Report(T)
    mem = memory.double() if mode != 'persist' else rn(memory)          # memFf: bf16 memory (decoder_persist.cu:60-67)
    memTr = v['memT'].double() if mode != 'persist' else rn(v['memT'])  # memTf: bf16 projection (decoder_persist.cu:38)
    wcomb = wcomb_fp32(prm['attn_location'], prm['attn_loc_features']) if mode == 'persist' else None
    Wq = prm['attn_query'].double()
    N1 = v['fs'].shape[2]
    wfs = torch.cat([prm['frame_w'], prm['stop_w']], 0)
    bfs = torch.cat([prm['frame_b'].reshape(-1), prm['stop_b'].reshape(-1)]).double()
    m = {k: masks.get(k) if (cfg.training and masks) else None for k in ('att_h', 'att_c', 'gen_h', 'gen_c')}
    al = align.transpose(0, 1)                                          # [T, B, L]
    if mode == 'persist':
        for name, key in (('aib', 'aib'), ('hgb', 'hgb')):
            rep.add(name + '_row0', 0, v[key][0:1].double().abs(), torch.zeros_like(v[key][0:1], dtype=torch.float64))
    chunk = _chunk(v)
    for i0 in range(0, T, chunk):
        i1 = min(T, i0 + chunk)
        sl = slice(i0, i1)
        sl1 = slice(i0 + 1, i1 + 1)
        mk = lambda k: None if m[k] is None else m[k][sl]       # noqa: E731
        # ---- attention LSTM ----
        z, b_z = att_preact(v, prm, att_operand(v, i0, i1, mode), i0, i1, mode)
        g, lip, g_err = activate(z, mode)
        rep.add('ga', i0, (v['ga'][sl].double() - g).abs(), lip * b_z + g_err)
        ai0, ai1 = v['ai'][sl], v['ai'][sl1]
        c, h, b_c, b_h = cell_forward(v['ga'][sl].double(), v['ca'][sl].double(), ai0[..., M:].double(), mk('att_h'), mk('att_c'), cfg, mode)
        rep.add('c_att', i0, (v['ca'][sl1].double() - c).abs(), b_c)
        rep.add('h_att', i0, (ai1[..., M:].double() - h).abs(), b_h)
        # ---- query: h_att . Wq^T, fp32-equivalent (hi + lo bf16 split, decoder_persist_tc.cu:532-559; fp32 in decoder_fwd.cu:130-155)
        h1 = ai1[..., M:].double()
        qr, b_q = product(h1, Wq)
        b_q = b_q + (D // 16 + 2) * U * (h1.abs() @ Wq.abs().t()) + (SPLIT_REL * (h1.abs() @ Wq.abs().t()) if mode == 'persist' else 0)
        rep.add('q', i0, (v['q'][sl].double() - qr).abs(), b_q)
        # ---- attention weights from the kernel's own q and cum ----
        w, b_w, valid = attention_weights(v['q'][sl], v['cum'][sl], memTr, lengths, prm, mode, wcomb)
        got = al[sl].double()
        rep.add('align', i0, ((got - w).abs()).masked_fill(~valid[None], 0.0), b_w)
        rep.add('align_pad', i0, got.abs().masked_fill(valid[None], 0.0), torch.zeros_like(got))
        # ---- context from the kernel's own weights: memory^T . w, w split hi + lo (decoder_persist_tc.cu:741-757, :782-784)
        cr = torch.einsum('sbl,blm->sbm', got, mem)
        a_c = torch.einsum('sbl,blm->sbm', got.abs(), mem.abs())
        b_ctx = (L + 4) * U * a_c + (SPLIT_REL * a_c if mode == 'persist' else 0)
        rep.add('ctx', i0, (ai1[..., :M].double() - cr).abs(), b_ctx)
        # ---- cumulative weights: cum_{i+1} = cum_i + w, one fp32 add (decoder_persist_tc.cu:734)
        cn = v['cum'][sl].double() + got
        rep.add('cum', i0, (v['cum'][sl1].double() - cn).abs(), U * cn.abs())
        # ---- generator LSTM ----
        a_in = att_operand(v, i0 + 1, i1 + 1, mode)
        z, b_z = gen_preact(v, prm, a_in, gen_operand(v, i0, i1, mode), mode)
        g, lip, g_err = activate(z, mode)
        rep.add('gg', i0, (v['gg'][sl].double() - g).abs(), lip * b_z + g_err)
        c, h, b_c, b_h = cell_forward(v['gg'][sl].double(), v['cg'][sl].double(), v['hg'][sl].double(), mk('gen_h'), mk('gen_c'), cfg, mode)
        rep.add('c_gen', i0, (v['cg'][sl1].double() - c).abs(), b_c)
        rep.add('h_gen', i0, (v['hg'][sl1].double() - h).abs(), b_h)
        # ---- frame / stop projection: [h_gen | ctx] . [frame_w ; stop_w]^T + b (decoder_fwd.cu:697-719, two GEMMs into one output)
        x = torch.cat([gen_operand(v, i0 + 1, i1 + 1, mode), a_in[..., D:]], -1)
        fr, b_fr = product(x, rw(wfs, mode))
        fr = fr + bfs
        rep.add('fs', i0, (v['fs'][sl].double() - fr).abs(), b_fr + 3 * U * (fr.abs() + bfs.abs()))
        # ---- the saved bf16 operand rows are the RN of the fp32 rows they mirror ----
        if mode == 'persist':
            rows = v['aib'][sl1].double()
            want = torch.cat([rn(ai1[..., M:]), rn(ai1[..., :M]), torch.zeros_like(rows[..., D + M:])], -1)
            rep.add('aib_rn', i0, (rows - want).abs(), torch.zeros_like(rows))
            rows = v['hgb'][sl1].double()
            want = torch.cat([rn(v['hg'][sl1]), torch.zeros_like(rows[..., D:])], -1)
            rep.add('hgb_rn', i0, (rows - want).abs(), torch.zeros_like(rows))
    return rep


# ------------------------------------------------------------------------------------------------------------------------
# reverse
# ------------------------------------------------------------------------------------------------------------------------
def _reverse(v, cfg, mode, rep, name, hist, hist_b, gates, cstate, static, extra, W, mh, mc, fill=False, hook=None):
    """Shared sweep of both reverse loops: step i from the kernel's gate gradients of step i+1 (its bf16 history in persist mode),
    the static d h of step i and the carried d c / zoneout d h, which are scanned sequentially in fp64 with their bounds.
    fill: write the reference into the history instead (synthetic workspaces)."""
    T = v[hist].shape[0]
    Wr = rw(W, mode)                                                     # [4D, D]
    dc = b_dc = dhz = b_dhz = None
    for i in range(T - 1, -1, -1):
        if hook is not None:
            hook(i)
        dh = v[static][i].double()
        b_dh = torch.zeros_like(dh)
        if extra is not None:
            e, b_e = extra(i)
            dh = dh + e
            b_dh = b_dh + b_e + U * dh.abs()
        if i < T - 1:
            if mode == 'persist':
                nxt = v[hist_b][i + 1].double()        # the bf16 gate gradients the loop saved and multiplied
            else:
                nxt = ra(v[hist][i + 1], mode)         # gemm_run on the fp32 gate gradients (decoder_bwd.cu:886-890, :983-987)
            rec = nxt @ Wr
            b_rec = (Wr.shape[0] + 4) * U * (nxt.abs() @ Wr.abs())
            dh = dh + rec + dhz
            b_dh = b_dh + b_rec + b_dhz + 3 * U * (dh.abs() + rec.abs() + dhz.abs())
            dcin, b_dcin = dc, b_dc
        else:
            dcin, b_dcin = torch.zeros_like(dh), torch.zeros_like(dh)
        g = v[gates][i].double()
        dg, b_dg, dc, b_dc, dhz, b_dhz = cell_backward(dh, b_dh, dcin, b_dcin, g, v[cstate][i].double(),
                                                       None if mh is None else mh[i], None if mc is None else mc[i], cfg, mode)
        if fill:
            v[hist][i] = dg.float()
            if hist_b in v:
                v[hist_b][i] = v[hist][i].to(torch.bfloat16)
        got = v[hist][i].double()
        rep.add(name, i, (got - dg).abs()[None], b_dg[None])
        if mode == 'persist':
            rep.add(name + 'b_rn', i, (v[hist_b][i].double() - rn(v[hist][i])).abs()[None], torch.zeros_like(got)[None])
    return rep


class AttentionReverse:
    """The attention backward of the attention reverse loop, step by step (decoder_persist_bwd.cu:298-545; the per-step chains:
    att_bwd_step, decoder_bwd.cu:937-968), from the kernel's own total d context, alignments, queries and cumulative weights.  The d cum
    carry (the location term of step i feeds on cum_i, and cum_{i+1} = cum_i + w_i) is scanned in fp64 together with its bound; d memT
    is the sum over steps of the per-step products and is checked once the sweep is done.
    Stages: dctxt (d context total: static part + dgab[i+1] . W_ih[:, P:]), dq, dmemT.
    The d cum carry is not saved by the kernels, so the reference carries its own, and its bound: an error of the carry feeds back
    through the softmax and energy backward into the next carry, and the worst-case (absolute value) propagation of that loop grows
    geometrically with the number of reverse steps.  The dq / dmemT bounds are therefore tight for the last steps of a decode (the
    first reverse steps) and for short decodes, and lose their power after a few tens of reverse steps of a long one."""

    def __init__(self, v, prm, lengths, memory, align, dalign, mode, rep, fill=False):
        T, B, D, M, L, A = _dims(v)
        self.v, self.prm, self.mode, self.rep, self.fill = v, prm, mode, rep, fill
        self.T, self.D, self.M, self.L, self.A = T, D, M, L, A
        persist = mode == 'persist'
        self.mem = rn(memory) if persist else memory.double()                 # memFb: bf16 memory (decoder_persist.cu:60-67)
        self.memTr = rn(v['memT']) if persist else v['memT'].double()         # memTf (decoder_persist_bwd.cu:915)
        Wc = prm['attn_loc_features']
        self.K = Wc.shape[-1]
        self.half = (self.K - 1) // 2
        if persist:
            self.wcomb = wcomb_fp32(prm['attn_location'], Wc)
            self.wcb = rn(self.wcomb)                                         # WcB2 (decoder_persist_bwd.cu:909)
            self.wcb_abs = self.wcb.abs()
        else:
            self.wcomb = None
            wl, wc = prm['attn_location'].double(), Wc.reshape(Wc.shape[0], self.K).double()
            self.wcb, self.wcb_abs = wl @ wc, wl.abs() @ wc.abs()            # location conv + Wloc, fp32 (C more terms in the bound)
        P = v['p1'].shape[2]
        self.Wctx = rw(prm['att_w_ih'][:, P:], mode)                         # [4D, M]
        self.v_e = prm['attn_energy'].reshape(-1).double()
        self.lens = lengths.to(v['cum'].device).long().clamp(0, L)
        self.valid = torch.arange(L, device=v['cum'].device)[None, :] < self.lens[:, None]
        self.al = align
        self.dal = dalign
        B_ = v['cum'].shape[1]
        z = lambda *s: torch.zeros(*s, dtype=torch.float64, device=v['cum'].device)   # noqa: E731
        self.dcum, self.b_dcum = z(B_, L), z(B_, L)
        self.lose_carry_at = None           # synthetic workspaces only: the d cum carry is lost on entry to this step
        self.dmemT, self.b_dmemT = z(B_, L, A), z(B_, L, A)

    def step(self, i):
        v, mode, rep = self.v, self.mode, self.rep
        T, M, L, A, K, half = self.T, self.M, self.L, self.A, self.K, self.half
        last = i == T - 1
        valid = self.valid
        if i == self.lose_carry_at:
            self.dcum = torch.zeros_like(self.dcum)
        # ---- total d context: static part + the recurrent part dgates_{i+1} . W_ih[:, P:] (bf16 history x bf16 weights)
        dct = v['dctxs'][i].double()
        b_dct = torch.zeros_like(dct)
        if not last:
            nxt = v['dgab'][i + 1].double() if mode == 'persist' else ra(v['dga'][i + 1], mode)
            r = nxt @ self.Wctx
            dct = dct + r
            b_dct = (nxt.shape[-1] + 4) * U * (nxt.abs() @ self.Wctx.abs()) + 2 * U * (dct.abs() + r.abs())
        if self.fill:
            v['dctxt'][i] = dct.float()
        rep.add('dctxt', i, (v['dctxt'][i].double() - dct).abs()[None], b_dct[None])
        # ---- d weights from the kernel's own d context: memory[l] . dctx (dctx split hi + lo, :349-404) + d cum carry + d alignment
        g = v['dctxt'][i].double()
        dw = torch.einsum('blm,bm->bl', self.mem, g)
        a_dw = torch.einsum('blm,bm->bl', self.mem.abs(), g.abs())
        b_dw = (M + 4) * U * a_dw + (SPLIT_REL * a_dw if mode == 'persist' else 0)
        if self.dal is not None:
            dw = dw + self.dal[:, i].double()
        if not last:
            dw = dw + self.dcum
            b_dw = b_dw + self.b_dcum
        b_dw = (b_dw + 2 * U * dw.abs()).masked_fill(~valid, 0.0)
        dw = dw.masked_fill(~valid, 0.0)
        # ---- softmax backward with the kernel's weights (:411-422)
        w = self.al[:, i].double().masked_fill(~valid, 0.0)
        dot = (w * dw).sum(-1, keepdim=True)
        b_dot = (w * b_dw).sum(-1, keepdim=True) + (self.lens[:, None].double() + 2) * U * (w * dw).abs().sum(-1, keepdim=True)
        de = w * (dw - dot)
        b_de = w * (b_dw + b_dot) + 2 * U * (w * (dw.abs() + dot.abs()))
        # ---- energies backward: ds = de v (1 - t^2) with t recomputed from the kernel's q and cum (:453-473)
        t, b_t = energy_tanh(v['q'][i:i + 1], v['cum'][i:i + 1], self.memTr, self.prm, mode, self.wcomb)
        t, b_t = t[0], b_t[0]                                                  # [B, L, A]
        s = 1 - t * t
        b_s = 2 * t.abs() * b_t + b_t * b_t + 2 * U * (s.abs() + t * t)
        ve = self.v_e
        ds = de[..., None] * ve * s
        b_ds = ve.abs() * (s.abs() * b_de[..., None] + de.abs()[..., None] * b_s) + 3 * U * ds.abs()
        dq = ds.sum(1)
        b_dq = b_ds.sum(1) + (L + 4) * U * ds.abs().sum(1)
        if self.fill:
            v['dq'][i] = dq.float()
        rep.add('dq', i, (v['dq'][i].double() - dq).abs()[None], b_dq[None])
        self.dmemT = self.dmemT + ds
        self.b_dmemT = self.b_dmemT + b_ds + U * self.dmemT.abs()
        # ---- d cum of step i-1: carry + sum_k G[j + half - k, k], G = ds . Wcomb, ds rounded to bf16 in persist mode (:473, :476-492)
        if mode == 'persist':
            dsr = rn(ds)
            b_dsr = b_ds + 2.0 ** -8 * ds.abs()          # RN of the kernel's ds vs RN of the reference: at most one bf16 ulp apart + b_ds
        else:
            dsr, b_dsr = ds, b_ds
        G = dsr @ self.wcb                                                     # [B, L, K]
        aG = dsr.abs() @ self.wcb_abs
        b_G = b_dsr @ self.wcb_abs + (A + 2) * U * aG
        dloc, b_loc, a_loc = torch.zeros_like(self.dcum), torch.zeros_like(self.dcum), torch.zeros_like(self.dcum)
        for k in range(K):
            lo, hi = max(0, k - half), min(L, L + k - half)                   # j with 0 <= l = j + half - k < L
            if lo >= hi:
                continue
            dloc[:, lo:hi] += G[:, lo + half - k:hi + half - k, k]
            b_loc[:, lo:hi] += b_G[:, lo + half - k:hi + half - k, k]
            a_loc[:, lo:hi] += G[:, lo + half - k:hi + half - k, k].abs()
        self.dcum = self.dcum + dloc
        self.b_dcum = self.b_dcum + b_loc + (K + 2) * U * (a_loc + self.dcum.abs())

    def finish(self):
        if self.fill:
            self.v['dmemT'].copy_(self.dmemT.float())
        self.rep.add('dmemT', 0, (self.v['dmemT'].double() - self.dmemT).abs()[None], self.b_dmemT[None])


def check_reverse(v, prm, masks, cfg, mode, report=None, fill=False, attention=None, lose_carry_at=None):
    """Gate gradients of the generator reverse loop (dgg) and of the attention-LSTM part of the attention reverse loop (dga, from the
    loop's own query gradients dq), teacher-forced decodes.  attention = (lengths, memory, align, dalign): also the attention backward
    of the attention reverse loop (AttentionReverse)."""
    assert mode in MODES
    T, B, D, M, L, A = _dims(v)
    rep = report or Report(T)
    att = AttentionReverse(v, prm, *attention, mode, rep, fill) if attention is not None else None
    if att is not None:
        att.lose_carry_at = lose_carry_at
    m = {k: masks.get(k) if (cfg.training and masks) else None for k in ('att_h', 'att_c', 'gen_h', 'gen_c')}
    _reverse(v, cfg, mode, rep, 'dgg', 'dgg', 'dggb', 'gg', 'cg', 'dhgd', None, prm['gen_w_hh'], m['gen_h'], m['gen_c'], fill)
    Wq = prm['attn_query'].double()

    def dq_term(i):
        # d h (query part) = dq . Wq, fp32-equivalent: dq and Wq split into bf16 hi + lo (decoder_persist_bwd.cu:582-611); fp32 in the
        # per-step cell backward (decoder_bwd.cu:191-199)
        dq = v['dq'][i].double()
        y = dq @ Wq
        a = dq.abs() @ Wq.abs()
        return y, (A + 4) * U * a + (SPLIT_REL * a if mode == 'persist' else 0)
    _reverse(v, cfg, mode, rep, 'dga', 'dga', 'dgab', 'ga', 'ca', 'dhas', dq_term, prm['att_w_hh'], m['att_h'], m['att_c'], fill,
             None if att is None else att.step)
    if att is not None:
        att.finish()
    return rep


def closing_products(v, prm, memory, align, mode):
    """fp64 products of the saved histories that form each parameter gradient and d memory (decoder_bwd.cu:850-908, :1210-1239).
    -> [(name, column slice or None, reference [rows, cols], bound)].  Bound: (T B + 2) 2^-24 |A|^T |B| of each product."""
    T, B, D, M, L, A = _dims(v)
    P = v['p1'].shape[2]
    out = []
    persist = mode == 'persist'
    flat = lambda x: x.reshape(-1, x.shape[-1])                     # noqa: E731
    # operand rows as the products read them: the bf16 rows in place (persist) or the RN of the fp32 rows (bf16 GEMM packing)
    if persist:
        aib, hgb = v['aib'].double(), v['hgb'].double()
        h_att, ctx, h_gen = aib[..., :D], aib[..., D:D + M], hgb[..., :D]
        dgg, dga = v['dggb'].double(), v['dgab'].double()
    else:
        ai = v['ai']
        h_att, ctx, h_gen = ra(ai[..., M:], mode), ra(ai[..., :M], mode), ra(v['hg'], mode)
        dgg, dga = ra(v['dgg'], mode), ra(v['dga'], mode)
    dfs, dq = ra(v['dfs'], mode), ra(v['dq'], mode)

    def prod(name, a, b, sl=None):
        """gradient = sum over (step, utterance) of a^T b"""
        a2, b2 = flat(a), flat(b)
        out.append((name, sl, a2.t() @ b2, (a2.shape[0] + 2) * U * (a2.abs().t() @ b2.abs())))

    def colsum(name, a):
        out.append((name, None, flat(a).sum(0)[None], ((flat(a).shape[0] + 2) * U * flat(a).abs().sum(0))[None]))

    prod('gen_w_hh', dgg, h_gen[:T])                                 # hgb rows 0..T-1
    prod('gen_w_ih', dgg, torch.cat([h_att[1:], ctx[1:]], -1))       # aib rows 1..T, [h_att | ctx]
    prod('att_w_hh', dga, h_att[:T])                                 # aib rows 0..T-1
    prod('att_w_ih', dga, ctx[:T], slice(P, P + M))
    prod('att_w_ih', dga, ra(v['p1'], mode), slice(0, P))
    prod('frame_w', dfs[..., :-1], torch.cat([h_gen[1:], ctx[1:]], -1))
    prod('stop_w', dfs[..., -1:], torch.cat([h_gen[1:], ctx[1:]], -1))
    prod('attn_query', dq, h_att[1:])
    prod('attn_memory', ra(v['dmemT'], mode), ra(memory, mode))
    colsum('gen_b_ih', v['dgg'].double())
    colsum('gen_b_hh', v['dgg'].double())
    colsum('att_b_ih', v['dga'].double())
    colsum('att_b_hh', v['dga'].double())
    colsum('attn_bias', v['dq'].double())
    colsum('frame_b', v['dfs'][..., :-1].double())
    colsum('stop_b', v['dfs'][..., -1:].double())
    # d memory = align^T . dctx (per utterance) + dmemT . Wm
    alr, dct = ra(align, mode), ra(v['dctxt'].transpose(0, 1), mode)   # [B, T, L], [B, T, M]
    dmr, wmr = ra(v['dmemT'], mode), ra(prm['attn_memory'], mode)
    ref = torch.einsum('btl,btm->blm', alr, dct) + dmr @ wmr
    bound = (T + 2) * U * torch.einsum('btl,btm->blm', alr.abs(), dct.abs()) + (A + 4) * U * (dmr.abs() @ wmr.abs()) + 2 * U * ref.abs()
    out.append(('memory', None, ref.reshape(B * L, M), bound.reshape(B * L, M)))
    return out


def _grad_view(g, sl):
    g = g.reshape(g.shape[0], -1) if g.dim() > 1 else g.reshape(1, -1)
    return g if sl is None else g[:, sl]


def check_closing(v, prm, grads, memory, align, mode, report=None):
    """Each parameter gradient formed from the saved histories, and d memory, against the fp64 product of those histories.  This pins
    the operand wiring of the in-place MN-major bf16 products: rows 0..T-1 vs 1..T of aib / hgb, and the column offsets into aib
    ([h_att | ctx]).  grads: {parameter name or 'memory': gradient}.  One stage per product, reported at step 0."""
    rep = report or Report(_dims(v)[0])
    for name, sl, ref, bound in closing_products(v, prm, memory, align, mode):
        g = grads[name]
        got = (g.reshape(-1, g.shape[-1]) if name == 'memory' else _grad_view(g, sl)).double()
        rep.add(name if sl is None else f'{name}[{sl.start}:{sl.stop}]', 0, (got - ref).abs()[None], bound[None])
    return rep


def closing_grads(v, prm, memory, align, mode):
    """gradients equal to the closing products (synthetic workspaces)"""
    T, B, D, M, L, A = _dims(v)
    grads = {k: torch.zeros_like(t) for k, t in prm.items()}
    grads['memory'] = torch.zeros_like(memory)
    for name, sl, ref, _ in closing_products(v, prm, memory, align, mode):
        if name == 'memory':
            grads[name].copy_(ref.reshape(memory.shape).float())
        else:
            _grad_view(grads[name], sl).copy_(ref.float())
    return grads


# ------------------------------------------------------------------------------------------------------------------------
# synthetic workspace (CPU tests): an fp64 trajectory with the same rounding points, stored in the same views
# ------------------------------------------------------------------------------------------------------------------------
class Config:
    def __init__(self, kind, training, rate_h, rate_c):
        self.kind, self.training, self.rate_h, self.rate_c = int(kind), bool(training), float(rate_h), float(rate_c)


def synthetic(B=34, L=20, T=6, D=64, M=64, P=32, A=16, C=4, K=5, N=8, kind=1, training=True, mode='persist', seed=0,
              kernel_masks=None, lose_dcum_carry_at=None):
    """-> (views, params, masks, cfg, lengths, memory, align, aux).  kernel_masks: masks the trajectory uses instead of the returned
    ones; lose_dcum_carry_at: the reverse trajectory drops the d cum carry on entry to that step.  aux: d alignments and the parameter
    gradients (the closing products)."""
    g = torch.Generator().manual_seed(seed)
    r = lambda *s, scale=1.0: (torch.randn(*s, generator=g, dtype=torch.float64) * scale).float()   # noqa: E731
    prm = {'prenet_w0': r(P, N, scale=N ** -0.5), 'prenet_b0': r(P, scale=0.1), 'prenet_w1': r(P, P, scale=P ** -0.5),
           'prenet_b1': r(P, scale=0.1), 'att_w_ih': r(4 * D, P + M, scale=2 * D ** -0.5), 'att_w_hh': r(4 * D, D, scale=2 * D ** -0.5),
           'att_b_ih': r(4 * D, scale=0.1), 'att_b_hh': r(4 * D, scale=0.1), 'gen_w_ih': r(4 * D, D + M, scale=D ** -0.5),
           'gen_w_hh': r(4 * D, D, scale=D ** -0.5), 'gen_b_ih': r(4 * D, scale=0.1), 'gen_b_hh': r(4 * D, scale=0.1),
           'attn_query': r(A, D, scale=3 * D ** -0.5), 'attn_memory': r(A, M, scale=3 * M ** -0.5),
           'attn_location': r(A, C, scale=C ** -0.5), 'attn_loc_features': r(C, 1, K, scale=K ** -0.5), 'attn_bias': r(1, A, scale=0.1),
           'attn_energy': r(1, A, scale=6 * A ** -0.5), 'frame_w': r(N, D + M, scale=(D + M) ** -0.5), 'frame_b': r(N, scale=0.1),
           'stop_w': r(1, D + M, scale=(D + M) ** -0.5), 'stop_b': r(1, scale=0.1)}
    lengths = torch.randint(1, L + 1, (B,), generator=g)
    lengths[0], lengths[1] = L, 1
    memory = r(B, L, M)
    cfg = Config(kind, training, 0.1, 0.1 if kind == 1 else 0.0)
    masks = {k: (torch.rand(T, B, D, generator=g) >= 0.1).to(torch.uint8) for k in ('att_h', 'att_c', 'gen_h', 'gen_c')}
    km = kernel_masks or masks
    kmask = lambda k, i: km[k][i:i + 1] if training else None     # noqa: E731
    Kp_att, Kp_gen = -(-(D + M) // 64) * 64, -(-D // 64) * 64
    z = lambda *s: torch.zeros(*s, dtype=torch.float32)          # noqa: E731
    v = {'ai': z(T + 1, B, M + D), 'ca': z(T + 1, B, D), 'hg': z(T + 1, B, D), 'cg': z(T + 1, B, D), 'ga': z(T, B, 4 * D),
         'gg': z(T, B, 4 * D), 'q': z(T, B, A), 'cum': z(T + 1, B, L), 'fs': z(T, B, N + 1),
         'p1': (torch.relu(r(T, B, P)) * 2), 'memT': (rn(memory) @ rn(prm['attn_memory']).t()).float(),
         'aib': z(T + 1, B, Kp_att).to(torch.bfloat16), 'hgb': z(T + 1, B, Kp_gen).to(torch.bfloat16),
         'dfs': r(T, B, N + 1, scale=0.1), 'dhgd': r(T, B, D, scale=0.1), 'dctxs': r(T, B, M, scale=0.1), 'dgg': z(T, B, 4 * D),
         'dhas': r(T, B, D, scale=0.1),
         'dga': z(T, B, 4 * D), 'dq': r(T, B, A, scale=0.1), 'dctxt': z(T, B, M), 'dmemT': z(B, L, A),
         'dggb': z(T, B, 4 * D).to(torch.bfloat16), 'dgab': z(T, B, 4 * D).to(torch.bfloat16)}
    if mode != 'persist':
        for k in ('aib', 'hgb', 'dggb', 'dgab'):
            del v[k]
    align = z(B, T, L)
    mem = rn(memory) if mode == 'persist' else memory.double()
    memTr = rn(v['memT']) if mode == 'persist' else v['memT'].double()
    wcomb = wcomb_fp32(prm['attn_location'], prm['attn_loc_features'])
    wfs = torch.cat([prm['frame_w'], prm['stop_w']], 0)
    bfs = torch.cat([prm['frame_b'], prm['stop_b']]).double()
    for i in range(T):
        zz, _ = att_preact(v, prm, att_operand(v, i, i + 1, mode), i, i + 1, mode)
        v['ga'][i] = activate(zz, mode)[0][0].float()
        c, h, _, _ = cell_forward(v['ga'][i:i + 1].double(), v['ca'][i:i + 1].double(), v['ai'][i:i + 1, :, M:].double(),
                                  kmask('att_h', i), kmask('att_c', i), cfg, mode)
        v['ca'][i + 1], v['ai'][i + 1, :, M:] = c[0].float(), h[0].float()
        v['q'][i] = (v['ai'][i + 1, :, M:].double() @ prm['attn_query'].double().t()).float()
        w, _, _ = attention_weights(v['q'][i:i + 1], v['cum'][i:i + 1], memTr, lengths, prm, mode, wcomb)
        align[:, i] = w[0].float()
        v['cum'][i + 1] = (v['cum'][i].double() + align[:, i].double()).float()
        v['ai'][i + 1, :, :M] = torch.einsum('bl,blm->bm', align[:, i].double(), mem).float()
        if mode == 'persist':
            v['aib'][i + 1, :, :D] = v['ai'][i + 1, :, M:].to(torch.bfloat16)
            v['aib'][i + 1, :, D:D + M] = v['ai'][i + 1, :, :M].to(torch.bfloat16)
        a_in = att_operand(v, i + 1, i + 2, mode)
        zz, _ = gen_preact(v, prm, a_in, gen_operand(v, i, i + 1, mode), mode)
        v['gg'][i] = activate(zz, mode)[0][0].float()
        c, h, _, _ = cell_forward(v['gg'][i:i + 1].double(), v['cg'][i:i + 1].double(), v['hg'][i:i + 1].double(),
                                  kmask('gen_h', i), kmask('gen_c', i), cfg, mode)
        v['cg'][i + 1], v['hg'][i + 1] = c[0].float(), h[0].float()
        if mode == 'persist':
            v['hgb'][i + 1, :, :D] = v['hg'][i + 1].to(torch.bfloat16)
        x = torch.cat([gen_operand(v, i + 1, i + 2, mode), a_in[..., D:]], -1)
        v['fs'][i] = (x @ rw(wfs, mode).t() + bfs)[0].float()
    dalign = r(B, T, L, scale=0.1)
    check_reverse(v, prm, {k: km[k] for k in km}, cfg, mode, fill=True, attention=(lengths, memory, align, dalign),
                  lose_carry_at=lose_dcum_carry_at)
    aux = {'dalign': dalign, 'grads': closing_grads(v, prm, memory, align, mode)}
    return v, prm, masks, cfg, lengths, memory, align, aux


# (B, L, T, M, D) of the GPU step checks (tests/test_gpu_persist_steps.py): every one runs on all three wgmma loops
# (test_step_check_cpu.py pins that and the edges they cover)
GPU_SHAPES = [
    (1, 17, 8, 288, 1024),      # one utterance, L = 1 (mod 16)
    (33, 47, 2, 288, 1024),     # odd B (second batch half of one utterance), L = 15 (mod 16), T = 2
    (64, 300, 8, 288, 1024),    # B = 64, L = 300
    (16, 180, 1, 512, 1024),    # memory dim 512, T = 1
    (8, 100, 6, 288, 512),      # D = 512
]


def check_all(v, prm, masks, cfg, lengths, memory, align, aux, mode):
    """Forward, reverse (with the attention backward: aux['dalign'] is the d alignments of the decode, None for none) and, when
    aux['grads'] is given, the closing products."""
    rep = check_forward(v, prm, masks, cfg, lengths, memory, align, mode)
    check_reverse(v, prm, masks, cfg, mode, rep, attention=(lengths, memory, align, aux.get('dalign')))
    if aux.get('grads') is not None:
        check_closing(v, prm, aux['grads'], memory, align, mode, rep)
    return rep
