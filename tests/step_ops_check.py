"""fp64 oracle and per-element bounds of the per-step decoder ops, as the module-level C ABI runs them in fp32 mode:

    b200tts_attention_step / _backward                    attn_fwd_kernel, attn_bwd_kernel (+ batchsum_add_kernel)
    b200tts_forward_attention_step / _backward            fwd_attn_fwd_kernel, fwd_attn_bwd_kernel (+ batchsum_add_kernel)
    b200tts_lstm_cell_forward / _backward                 lstm_cell_fwd_kernel, lstm_cell_bwd_kernel

Everything is step-local, as in tests/step_check.py, whose fp32-mode primitives this builds on: each output is recomputed in fp64
from the inputs of the call and from the intermediates the kernel exposes (q = query . Wq^T from the head of the forward workspace,
the weights the forward wrote), and gets its own bound

    err = |kernel value - fp64 reference|  <=  bound = fp32 accumulation bound n 2^-24 (|a| . |b|) of each sum
                                                        + the propagated bounds of its inputs + the libm error of expf / tanhf

Every function returns {output name: (reference, bound)}; the bounds of the += outputs are those of the increment (see accumulate).
"""
import math

import numpy as np
import torch
import torch.nn.functional as Fn

import step_check as S

U = S.U
NW = 8                                   # warps per CTA of the attention kernels (ATT_THREADS = 256)
FLOOR = float(np.float32(1e-6))          # FWD_ATT_FLOOR: the fp32 1e-6 of torch.clamp(energies, 1e-6)


def ratio(got, ref, bound):
    """worst err / bound over all elements (0 / 0 = 0, err / 0 = inf) and the flat index where it sits"""
    err = (got.double() - ref.double()).abs()
    r = torch.where(err == 0, torch.zeros_like(err), err / bound.double())
    r = torch.nan_to_num(r, nan=math.inf).reshape(-1)
    if r.numel() == 0:
        return 0.0, -1
    i = int(r.argmax())
    return float(r[i]), i


def accumulate(prefill, inc, b_inc):
    """out = prefill + increment, one fp32 add onto the caller's buffer -> (reference, bound)"""
    out = prefill.double() + inc
    return out, b_inc + U * out.abs()


def batch_sum(x, b_x, a_x, n):
    """per-utterance partials x [B, ...] (bound b_x, each a sum of at most n [B] terms whose |.| sum to a_x), summed in order over
    the batch by batchsum_add_kernel -> (sum, bound)"""
    B = x.shape[0]
    nn = n.double().reshape(B, *([1] * (x.dim() - 1)))
    return x.sum(0), (b_x + (nn + 2) * U * a_x).sum(0) + (B + 1) * U * x.abs().sum(0)


def _lens(lengths, B, L, device):
    lens = lengths.to(device).long().reshape(B).clamp(0, L)
    return lens, torch.arange(L, device=device)[None, :] < lens[:, None]


def _loc_params(prm):
    Wl = prm['attn_location'].double()
    A, C = Wl.shape
    Wc = prm['attn_loc_features'].double().reshape(C, -1)
    return Wl, Wc, prm['attn_energy'].double().reshape(-1), C, Wc.shape[1]


def query_product(query, Wq):
    """q = query . Wq^T (gemm_f32: one fp32 fmaf chain over D) -> (q, bound)"""
    return S.product(query.double(), Wq.double())


def context(w, memory, n):
    """context[m] = sum_l w[l] memory[l, m] from the kernel's own weights: per-warp fmaf chains over every NW-th position, then the NW
    warp partials in order; n [B] positions summed"""
    mem = memory.double()
    c = torch.einsum('bl,blm->bm', w.double(), mem)
    a = torch.einsum('bl,blm->bm', w.double().abs(), mem.abs())
    k = (torch.div(n + NW - 1, NW, rounding_mode='floor') + NW + 1).double()[:, None]
    return c, k * U * a


# ------------------------------------------------------------------------------------------------------------------------
# location-sensitive attention (attn_fwd_kernel / attn_bwd_kernel)
# ------------------------------------------------------------------------------------------------------------------------
def location_forward(q, cum, memT, memory, lengths, prm, w_kernel):
    """weights from the kernel's q and cum_prev (step_check.attention_weights: fp32 location convolution and projection, tanhf, the
    softmax over l < len), the context from the kernel's weights."""
    B, L = cum.shape
    w, b_w, valid = S.attention_weights(q[None], cum[None], memT.double(), lengths, prm, 'fp32')
    lens, _ = _lens(lengths, B, L, cum.device)
    return {'weights': (w[0], b_w[0]), 'context': context(w_kernel, memory, lens)}


def location_backward(q, cum, memT, memory, lengths, prm, w, d_ctx, d_w, d_cum):
    """One attention step backward (b200tts_attention_step_backward) from the kernel's q, the cum_prev the step consumed and the
    weights it wrote.  d_cum is the gradient of the updated cumulative weights (in) and d_w the d weights (None: none).
    -> d_cum (out: d cum_prev), d_q, and the increments d_memT, d_Wloc, d_Wc, d_v"""
    B, L = cum.shape
    Wl, Wc, v_e, C, K = _loc_params(prm)
    M = memory.shape[-1]
    half = (K - 1) // 2
    lens, valid = _lens(lengths, B, L, cum.device)
    mem, g = memory.double(), d_ctx.double()
    # dw[l] = <d ctx, memory[l]> (lane chains over M / 32 + a 5-level warp sum) + d cum + d weights, for l < len
    dw = torch.einsum('blm,bm->bl', mem, g)
    b_dw = (math.ceil(M / 32) + 7) * U * torch.einsum('blm,bm->bl', mem.abs(), g.abs())
    dw = dw + d_cum.double() + (d_w.double() if d_w is not None else 0.0)
    b_dw = (b_dw + 2 * U * dw.abs()).masked_fill(~valid, 0.0)
    dw = dw.masked_fill(~valid, 0.0)
    t, b_t = S.energy_tanh(q[None], cum[None], memT.double(), prm, 'fp32')
    t, b_t = t[0], b_t[0]
    wk = w.double().masked_fill(~valid, 0.0)
    ab = S.attention_backward(dw, b_dw, wk, lens, t, b_t, v_e, Wl @ Wc, Wl.abs() @ Wc.abs(), K, 'fp32')
    ds, b_ds, de, b_de = ab['ds'], ab['b_ds'], ab['de'], ab['b_de']
    out = {}
    out['d_q'] = (ds.sum(1), b_ds.sum(1) + (L + 4) * U * ds.abs().sum(1))
    out['d_memT'] = (ds, b_ds)
    dc = d_cum.double() + ab['dloc']
    out['d_cum'] = (dc, ab['b_loc'] + (K + 2) * U * (ab['a_loc'] + dc.abs()))
    n = lens + NW + 2                                         # each per-utterance sum below: at most len terms + its reduction
    # d v[a] = sum_l de[l] t[l, a]
    dv = torch.einsum('bl,bla->ba', de, t)
    a_dv = torch.einsum('bl,bla->ba', de.abs(), t.abs())
    out['d_v'] = batch_sum(dv, torch.einsum('bl,bla->ba', de.abs(), b_t) + torch.einsum('bl,bla->ba', b_de, t.abs()), a_dv, n)
    # location features f[l, c] = sum_k Wc[c, k] cum[l + k - half] (K fmaf), zero padded
    unf = Fn.pad(cum.double(), (half, K - 1 - half)).unfold(-1, K, 1)           # [B, L, K]
    f = unf @ Wc.t()
    b_f = (K + 2) * U * (unf.abs() @ Wc.abs().t())
    # d Wloc[a, c] = sum_l ds[l, a] f[l, c]
    dWl = torch.einsum('bla,blc->bac', ds, f)
    a_dWl = torch.einsum('bla,blc->bac', ds.abs(), f.abs())
    b_dWl = torch.einsum('bla,blc->bac', b_ds, f.abs()) + torch.einsum('bla,blc->bac', ds.abs(), b_f)
    out['d_Wloc'] = batch_sum(dWl, b_dWl, a_dWl, n)
    # dF[l, c] = sum_a ds[l, a] Wloc[a, c] (A fmaf); d Wc[c, k] = sum_l dF[l, c] cum[l + k - half]
    dF = ds @ Wl
    b_dF = b_ds @ Wl.abs() + (Wl.shape[0] + 2) * U * (ds.abs() @ Wl.abs())
    dWc = torch.einsum('blc,blk->bck', dF, unf)
    a_dWc = torch.einsum('blc,blk->bck', dF.abs(), unf.abs())
    out['d_Wc'] = batch_sum(dWc, torch.einsum('blc,blk->bck', b_dF, unf.abs()), a_dWc, n)
    return out


# ------------------------------------------------------------------------------------------------------------------------
# forward attention (fwd_attn_fwd_kernel / fwd_attn_bwd_kernel)
# ------------------------------------------------------------------------------------------------------------------------
def transition(q, memT, prm):
    """t = tanh(q + bias + memT[l]) [B, L, A] and s = softmax over ALL L of v . t (fwd_att_transition) -> (t, b_t, s, b_s)"""
    B, L, A = memT.shape
    qb = q.double() + prm['attn_bias'].double().reshape(-1)
    x = qb[:, None, :] + memT.double()
    b_x = U * qb.abs()[:, None, :] + U * x.abs()
    t = torch.tanh(x)
    b_t = b_x + 2 * S.ULP1 * t.abs()
    v = prm['attn_energy'].double().reshape(-1)
    e = t @ v
    b_e = b_t @ v.abs() + (A + 2) * U * (t.abs() @ v.abs())
    valid = torch.ones(B, L, dtype=torch.bool, device=memT.device)
    s, b_s = S.softmax(e, b_e, valid, L)
    return t, b_t, s, b_s


def _product(alpha, s, b_s, valid):
    """a[l] = (alpha[l] + alpha[l-1]) s[l] for l < len, 0 beyond (fwd_att_product) -> (p, a, b_a)"""
    al = alpha.double()
    p = al + Fn.pad(al, (1, 0))[:, :-1]
    a = (p * s).masked_fill(~valid, 0.0)
    return p, a, (p.abs() * b_s + 2 * U * a.abs()).masked_fill(~valid, 0.0)


def _normaliser(a, b_a):
    """c = max(a, 1e-6) and its sum over all L (strided partials + a block sum) -> (c, b_c, den, b_den)"""
    L = a.shape[-1]
    c = a.clamp(min=FLOOR)
    den = c.sum(-1, keepdim=True)
    return c, b_a, den, b_a.sum(-1, keepdim=True) + (L + 16) * U * den


def forward_forward(q, alpha, memT, memory, lengths, prm, w_kernel):
    """weights = clamp(a, 1e-6) / sum (the L1 normalisation) from the kernel's q and the alpha the step consumed; the context from the
    kernel's weights over all L."""
    B, L = alpha.shape
    _, _, s, b_s = transition(q, memT, prm)
    lens, valid = _lens(lengths, B, L, alpha.device)
    p, a, b_a = _product(alpha, s, b_s, valid)
    c, b_c, den, b_den = _normaliser(a, b_a)
    w = c / den
    return {'weights': (w, (b_c + w * b_den) / den + U * w),
            'context': context(w_kernel, memory, torch.full_like(lens, L))}


def forward_backward(q, alpha, memT, memory, lengths, prm, w, d_ctx, d_w, d_alpha):
    """One forward-attention step backward (b200tts_forward_attention_step_backward) from the kernel's q, the alpha the step consumed
    and the weights it wrote.  The clamp passes a gradient only where a >= 1e-6; where the fp64 a lies within its bound of the floor
    either decision is accepted (the reference then takes the midpoint and half the difference joins the bound).
    -> d_alpha (out: d alpha_prev), d_q, and the increments d_memT, d_v"""
    B, L = alpha.shape
    M = memory.shape[-1]
    t, b_t, s, b_s = transition(q, memT, prm)
    lens, valid = _lens(lengths, B, L, alpha.device)
    mem, g = memory.double(), d_ctx.double()
    gw = torch.einsum('blm,bm->bl', mem, g) + d_alpha.double() + (d_w.double() if d_w is not None else 0.0)
    b_gw = (math.ceil(M / 32) + 7) * U * torch.einsum('blm,bm->bl', mem.abs(), g.abs()) + 2 * U * gw.abs()
    wk = w.double()
    dot = (gw * wk).sum(-1, keepdim=True)
    b_dot = (wk.abs() * b_gw).sum(-1, keepdim=True) + (L + 16) * U * (gw * wk).abs().sum(-1, keepdim=True)
    p, a, b_a = _product(alpha, s, b_s, valid)
    _, _, den, b_den = _normaliser(a, b_a)
    val = (gw - dot) / den
    b_val = (b_gw + b_dot) / den + val.abs() * b_den / den + 2 * U * val.abs()
    gate = valid & (a >= FLOOR)
    either = valid & ((a - FLOOR).abs() <= b_a)
    da = torch.where(gate, val, torch.zeros_like(val))
    b_da = torch.where(gate, b_val, torch.zeros_like(val))
    da = torch.where(either, 0.5 * val, da)
    b_da = torch.where(either, 0.5 * val.abs() + b_val, b_da)
    # d alpha[l] = da[l] s[l] + da[l+1] s[l+1]
    x, b_x = da * s, da.abs() * b_s + b_da * s
    xn, b_xn = Fn.pad(x, (0, 1))[:, 1:], Fn.pad(b_x, (0, 1))[:, 1:]
    dal = x + xn
    out = {'d_alpha': (dal, b_x + b_xn + 2 * U * (x.abs() + xn.abs()))}
    # softmax backward: de = s (ds - <s, ds>), ds = da (alpha[l] + alpha[l-1])
    ds = da * p
    b_ds = p.abs() * b_da + 2 * U * ds.abs()
    sds = (s * ds).sum(-1, keepdim=True)
    b_sds = (s * b_ds + ds.abs() * b_s).sum(-1, keepdim=True) + (L + 16) * U * (s * ds).abs().sum(-1, keepdim=True)
    de = s * (ds - sds)
    b_de = (ds - sds).abs() * b_s + s * (b_ds + b_sds) + 2 * U * s * (ds.abs() + sds.abs())
    # energies backward over every position: dpre = de v (1 - t^2)
    v = prm['attn_energy'].double().reshape(-1)
    om = 1 - t * t
    b_om = 2 * t.abs() * b_t + b_t * b_t + 2 * U * (om.abs() + t * t)
    dpre = de[..., None] * v * om
    b_dpre = v.abs() * (om.abs() * b_de[..., None] + de.abs()[..., None] * b_om) + 3 * U * dpre.abs()
    out['d_q'] = (dpre.sum(1), b_dpre.sum(1) + (L + 16) * U * dpre.abs().sum(1))
    out['d_memT'] = (dpre, b_dpre)
    dv = torch.einsum('bl,bla->ba', de, t)
    a_dv = torch.einsum('bl,bla->ba', de.abs(), t.abs())
    b_dv = torch.einsum('bl,bla->ba', de.abs(), b_t) + torch.einsum('bl,bla->ba', b_de, t.abs())
    out['d_v'] = batch_sum(dv, b_dv, a_dv, torch.full_like(lens, L + NW + 2))
    return out


# ------------------------------------------------------------------------------------------------------------------------
# LSTM cell (lstm_cell_fwd_kernel / lstm_cell_bwd_kernel)
# ------------------------------------------------------------------------------------------------------------------------
def cell_fwd(z, h_prev, c_prev, mask_h, mask_c, cfg, gates_kernel):
    """gates = activations of the pre-activations z [B, 4D] (i, f, g, o); h / c from the kernel's own gates (step_check.cell_forward)"""
    g, _, g_err = S.activate(z.double(), 'fp32')
    c, h, b_c, b_h = S.cell_forward(gates_kernel.double(), c_prev.double(), h_prev.double(), mask_h, mask_c, cfg, 'fp32')
    return {'gates': (g, g_err), 'c': (c, b_c), 'h': (h, b_h)}


def cell_bwd(gates, c_prev, mask_h, mask_c, d_h, d_c, cfg):
    """d_gates, d_c (out: d c_prev) and d_h_prev (the direct zoneout term; exactly 0 for the dropout cell) from the saved gates
    (step_check.cell_backward with exact incoming gradients)"""
    dh, dc = d_h.double(), d_c.double()
    z = torch.zeros_like(dh)
    dg, b_dg, dcp, b_dcp, dhz, b_dhz = S.cell_backward(dh, z, dc, z, gates.double(), c_prev.double(), mask_h, mask_c, cfg, 'fp32')
    return {'d_gates': (dg, b_dg), 'd_c': (dcp, b_dcp), 'd_h_prev': (dhz, b_dhz)}
