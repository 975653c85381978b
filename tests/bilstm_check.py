"""Step-local fp64 check of the packed bidirectional LSTM (csrc/rnn.cu, csrc/bilstm_persist.cu) from the state the kernels saved.

Step j of each direction (position t = j forward, t = L-1-j reverse) is recomputed in fp64 from the kernel's OWN state of step j-1
(the saved hs / cs rows, and in the backward the kernel's own gate gradients of step j+1), so the reference never drifts off the
kernel's trajectory, and every element gets its own bound as in tests/step_check.py, whose primitives this module uses:

    err   = |kernel value - fp64 reference|
    bound = fp32 accumulation bound of each product + the error of the accurate nonlinearities, through Lipschitz constants

Rounding model (precision, path):
    fp32 mode      every GEMM in fp32 (gemm.cu gemm_f32_kernel); no operand rounding at all
    bf16 mode      the time-batched GEMMs take bf16 RN operands (gemm_bf16.cu:74-82): the input projection (rnn.cu:98-101), dW_ih,
                   dW_hh (rnn.cu:163-168) and dx (rnn.cu:172-175); on the per-step chain also the recurrent products (rnn.cu:107-111,
                   rnn.cu:155-159).  The persistent kernel keeps W_hh in fp32 shared memory and multiplies with fp32 FFMA in both
                   modes (bilstm_persist.cu:91-100, :203-210)
Both paths activate with the accurate sigmoidf_acc / tanhf (bilstm_persist.cu:109, decoder_fwd.cu:100): step_check's non-'persist'
nonlinearity model.  There is no blanket tolerance anywhere.

Stages (Report, per processing step j; the error tensors carry the direction as their first index):
    xp, bsum     the input in processing order and b_ih + b_hh, exact (rnn.cu:13-22, :94)
    gates        activated gates of valid steps from z = (xp . W_ih^T + bsum) + h_prev . W_hh^T
    xproj        persistent kernel, frozen steps: the buffer still holds the input projection (bilstm_persist.cu:83-86, :113)
    c, h         the cell from the saved gates and c_prev
    frozen       hs / cs of a frozen step bitwise equal to those of the step before
    zero_start   the state before a direction's first valid step is exactly zero (the reverse direction starts at each utterance's
                 own last token)
    out, out_pad the output equals the new h at valid positions, exactly 0 at t >= length
    dg, dg_frozen pre-activation gate gradients; exactly 0 at frozen steps
    dW_ih, dW_hh, db_ih, db_hh, dx, dx_pad   the closing products from the kernel's own dg (step 0)
"""
import ctypes

import torch

from step_check import U, Config, Report, activate, cell_backward, cell_forward, product, ra, rw

CELL = Config(0, False, 0.0, 0.0)       # the bi-LSTM runs the dropout cell kind untrained (rnn.cu:117, :151): a plain LSTM cell
VIEWS = ('xp', 'gates', 'hs', 'cs', 'bsum', 'dg', 'dxp')
PARAMS = ('w_ih', 'w_hh', 'b_ih', 'b_hh', 'w_ih_reverse', 'w_hh_reverse', 'b_ih_reverse', 'b_hh_reverse')
AUTO_SPLIT_MAX = 160                    # gemm.cu gemm_auto_impl: most partial sums the dW products are split into


def layout(B, L, E, H):
    """b200tts_debug_bilstm_layout: {view: byte offset}, split, split_b (split-K of the chain's recurrent products) and persist."""
    from multilingual_text_to_speech_b200 import _lib
    out = (ctypes.c_size_t * 10)()
    n = _lib.load().b200tts_debug_bilstm_layout(ctypes.byref(_lib.BiLSTMShape(B, L, E, H)), out, 10)
    assert n == 10, n
    lay = dict(zip(VIEWS, (int(x) for x in out[:7])))
    lay.update(split=int(out[7]), split_b=int(out[8]), persist=bool(out[9]))
    return lay


def views(saved, ws, B, L, E, H, lay):
    """fp32 views of the saved buffer (forward) and the backward workspace, direction-major in processing order."""
    shapes = {'xp': (2, L, B, E), 'gates': (2, L, B, 4 * H), 'hs': (2, L + 1, B, H), 'cs': (2, L + 1, B, H), 'bsum': (2, 4 * H),
              'dg': (2, L, B, 4 * H), 'dxp': (2, L, B, E)}
    v = {}
    for name, shape in shapes.items():
        buf = (ws if name in ('dg', 'dxp') else saved).view(torch.float32)
        o = lay[name] // 4
        n = 1
        for s in shape:
            n *= s
        v[name] = buf[o:o + n].view(shape)
    return v


def _dims(v):
    _, L, B, H4 = v['gates'].shape
    return B, L, v['xp'].shape[3], H4 // 4


def positions(L, device):
    """t[dir, j]: the position processing step j of each direction reads"""
    j = torch.arange(L, device=device)
    return torch.stack([j, L - 1 - j])


def valid_steps(lengths, L, device):
    """[2, L, B]: step j of a direction is valid for utterance b when its position is below the length"""
    return positions(L, device)[:, :, None] < lengths.to(device).long()[None, None, :]


def pair(prm, name):
    """[2, ...] fp32: the forward and reverse tensor of one parameter"""
    return torch.stack([prm[name], prm[name + '_reverse']])


def processing_order(y, H):
    """y [B, L, 2H] (output or its gradient) -> [2, L, B, H] in each direction's processing order"""
    B, L, _ = y.shape
    t = positions(L, y.device)
    return torch.stack([y[:, t[d], d * H:(d + 1) * H].transpose(0, 1) for d in range(2)])


def _modes(precision, persist):
    """(mode of the time-batched GEMM operands, mode of the recurrent product operands), in step_check's names"""
    pm = 'chain_bf16' if precision == 'bf16' else 'fp32'
    return pm, ('fp32' if persist else pm)


def preact(xp, h, w_ih, w_hh, bsum, precision, persist, split):
    """Pre-activations of the steps whose input rows are xp [..., E] and previous hidden rows h [..., H] (one direction).
    Input projection: one GEMM with the fp32 bias bsum in its epilogue (rnn.cu:98-101), stored in fp32.  Recurrent part: the
    persistent kernel's fp32 FFMA chain, added to the projection once (bilstm_persist.cu:107-108); or the chain's split-K GEMM whose
    `split` partial sums the cell kernel adds to the projection one by one (rnn.cu:107-111, decoder_fwd.cu:95-99).
    -> (projection, its bound, z, bound of z)"""
    pm, rm = _modes(precision, persist)
    E, H = xp.shape[-1], h.shape[-1]
    proj, _ = product(ra(xp, pm), rw(w_ih, pm))
    a_proj = ra(xp, pm).abs() @ rw(w_ih, pm).abs().t()
    b = bsum.double()
    proj = proj + b
    b_proj = (E + 3) * U * a_proj + U * (b.abs() + proj.abs())
    rec, _ = product(ra(h, rm), rw(w_hh, rm))
    a_rec = ra(h, rm).abs() @ rw(w_hh, rm).abs().t()
    z = proj + rec
    b_z = b_proj + (H + 2) * U * a_rec + split * U * (proj.abs() + a_rec)
    return proj, b_proj, z, b_z


def gates_ref(z, b_z):
    """activated gates and their bound"""
    g, lip, err = activate(z, 'fp32')
    return g, lip * b_z + err


def dh_ref(dout, nxt, w_hh, precision, persist, split_b):
    """Total d h of the steps whose static output gradient is dout [..., H] and whose following step's gate gradients are nxt
    [..., 4H] (None: the last step).  Persistent kernel: eight fp32 FFMA partial sums over 4H / 8 rows each, added in order and added
    to d out once (bilstm_persist.cu:173, :200-217); chain: the split-K GEMM on bf16 operands in bf16 mode, whose split_b partials the
    cell kernel sums and adds to d out (rnn.cu:154-159, decoder_bwd.cu:209-222).  -> (dh, bound)"""
    dh = dout.double()
    if nxt is None:
        return dh, torch.zeros_like(dh)
    _, rm = _modes(precision, persist)
    a, w = ra(nxt, rm), rw(w_hh, rm)
    rec = a @ w
    a_rec = a.abs() @ w.abs()
    dh = dh + rec
    n = 8 if persist else split_b
    return dh, (w.shape[0] + 2 + n) * U * a_rec + (n + 2) * U * (dout.double().abs() + a_rec)


# ------------------------------------------------------------------------------------------------------------------------
# forward
# ------------------------------------------------------------------------------------------------------------------------
def _steps_first(x):
    """[2, L, ...] -> [L, 2, ...] (Report wants the step first)"""
    return x.transpose(0, 1)


def _add(rep, stage, err, bound, mask=None):
    if mask is not None:
        err = torch.where(mask, err, torch.zeros_like(err))
    rep.add(stage, 0, _steps_first(err), _steps_first(bound))


def check_forward(v, prm, x, lengths, out, precision, persist, split=1, report=None):
    """Every stage of every forward step of both directions.  prm: {PARAMS name: fp32 tensor}, x [B, L, E], out [B, L, 2H]."""
    B, L, E, H = _dims(v)
    rep = report or Report(L)
    dev = v['gates'].device
    t = positions(L, dev)
    valid = valid_steps(lengths, L, dev)                                   # [2, L, B]
    vm = valid[..., None]
    z0 = lambda a: torch.zeros_like(a, dtype=torch.float64)             # noqa: E731
    # ---- the input in processing order, and the summed bias: exact copies (rnn.cu:13-22, :94 launch_add_vec)
    xp_want = torch.stack([x[:, t[d]].transpose(0, 1) for d in range(2)]).double()
    err = (v['xp'].double() - xp_want).abs()
    _add(rep, 'xp', err, z0(err))
    bsum = (pair(prm, 'b_ih').double() + pair(prm, 'b_hh').double()).float()
    rep.add('bsum', 0, (v['bsum'].double() - bsum.double()).abs()[None], torch.zeros(1, 2, 4 * H, dtype=torch.float64, device=dev))
    # ---- gates of every step from the kernel's own h_prev = hs[j]
    w_ih, w_hh = pair(prm, 'w_ih'), pair(prm, 'w_hh')
    g_err, g_bound, p_err, p_bound = [], [], [], []
    for d in range(2):
        proj, b_proj, z, b_z = preact(v['xp'][d], v['hs'][d, :L], w_ih[d], w_hh[d], bsum[d], precision, persist, split)
        g, b_g = gates_ref(z, b_z)
        g_err.append((v['gates'][d].double() - g).abs())
        g_bound.append(b_g)
        p_err.append((v['gates'][d].double() - proj).abs())
        p_bound.append(b_proj)
    g_err, g_bound, p_err, p_bound = map(torch.stack, (g_err, g_bound, p_err, p_bound))
    if persist:
        # valid steps overwrite the projection with the activated gates in place (bilstm_persist.cu:113); frozen steps keep it
        _add(rep, 'gates', g_err, g_bound, vm)
        _add(rep, 'xproj', p_err, p_bound, ~vm)
    else:
        # the chain's cell kernel stores the gates of every step, a frozen one's from the frozen state (decoder_fwd.cu:104)
        _add(rep, 'gates', g_err, g_bound)
    # ---- cell from the saved gates and c_prev
    c, h, b_c, b_h = cell_forward(v['gates'].double(), v['cs'][:, :L].double(), v['hs'][:, :L].double(), None, None, CELL, 'fp32')
    _add(rep, 'c', (v['cs'][:, 1:].double() - c).abs(), b_c, vm)
    _add(rep, 'h', (v['hs'][:, 1:].double() - h).abs(), b_h, vm)
    # ---- frozen steps copy the state bitwise (bilstm_persist.cu:105, :115-117; decoder_fwd.cu:123)
    err = (v['hs'][:, 1:] != v['hs'][:, :L]).double() + (v['cs'][:, 1:] != v['cs'][:, :L]).double()
    _add(rep, 'frozen', err, z0(err), ~vm)
    # ---- the state before each direction's first valid step is exactly zero: hs / cs rows j <= L - length of the reverse direction
    # (its frozen steps come first), row 0 of the forward direction
    lens = lengths.to(dev).long()
    j = torch.arange(L, device=dev)
    before = torch.stack([(j == 0)[:, None].expand(L, B), j[:, None] <= (L - lens)[None, :]])[..., None]
    err = v['hs'][:, :L].double().abs() + v['cs'][:, :L].double().abs()
    _add(rep, 'zero_start', err, z0(err), before)
    # ---- output: the new h at valid positions, exactly zero beyond the length
    o = processing_order(out, H).double()
    _add(rep, 'out', (o - v['hs'][:, 1:].double()).abs(), z0(o), vm)
    _add(rep, 'out_pad', o.abs(), z0(o), ~vm)
    return rep


# ------------------------------------------------------------------------------------------------------------------------
# backward
# ------------------------------------------------------------------------------------------------------------------------
def check_backward(v, prm, lengths, dout, precision, persist, split_b=1, report=None):
    """Gate gradients of every backward step of both directions.  The incoming d h of step j is d out + W_hh^T . dg_{j+1} from the
    kernel's own dg; the d c carry is not saved by the kernels, so the reference scans its own in fp64 with its bound (|f| < 1 keeps
    that bound from growing).  A frozen step passes both carries through and has dg exactly 0."""
    B, L, E, H = _dims(v)
    rep = report or Report(L)
    dev = v['gates'].device
    valid = valid_steps(lengths, L, dev)[..., None]                    # [2, L, B, 1]
    w_hh = pair(prm, 'w_hh')
    dop = processing_order(dout, H)                                    # [2, L, B, H]
    dh, b_dh = [], []
    for d in range(2):
        a, ba = dh_ref(dop[d, :L - 1], v['dg'][d, 1:], w_hh[d], precision, persist, split_b)
        z, bz = dh_ref(dop[d, L - 1:], None, w_hh[d], precision, persist, split_b)
        dh.append(torch.cat([a, z]))
        b_dh.append(torch.cat([ba, bz]))
    dh, b_dh = torch.stack(dh), torch.stack(b_dh)
    dc = torch.zeros(2, B, H, dtype=torch.float64, device=dev)
    b_dc = torch.zeros_like(dc)
    for j in range(L - 1, -1, -1):
        dg, b_dg, dcp, b_dcp, _, _ = cell_backward(dh[:, j], b_dh[:, j], dc, b_dc, v['gates'][:, j].double(), v['cs'][:, j].double(),
                                                   None, None, CELL, 'fp32')
        m = valid[:, j]
        got = v['dg'][:, j].double()
        rep.add('dg', j, torch.where(m, (got - dg).abs(), torch.zeros_like(got))[None], b_dg[None])
        rep.add('dg_frozen', j, torch.where(m, torch.zeros_like(got), got.abs())[None], torch.zeros_like(got)[None])
        dc, b_dc = torch.where(m, dcp, dc), torch.where(m, b_dcp, b_dc)
    return rep


def closing_products(v, prm, precision):
    """fp64 products that form the parameter gradients and dx from the kernel's own dg and saved operand rows.
    -> [(name, direction, reference without the prefill, bound)] for dW_ih, dW_hh (one GEMM each, rnn.cu:163-168, split-K up to
    AUTO_SPLIT_MAX partials), db (colsum_add2_kernel: an fp32 sum over L B / 8 rows per thread, then 8 partials, rnn.cu:31-44), and
    ('dx', None, [B, L, E], bound): the sum of both directions' dg . W_ih (rnn.cu:172-179)."""
    B, L, E, H = _dims(v)
    pm, _ = _modes(precision, False)
    out = []
    flat = lambda a: a.reshape(-1, a.shape[-1])                        # noqa: E731
    t = positions(L, v['dg'].device)
    dx = 0
    b_dx = 0
    for d in range(2):
        dg = flat(ra(v['dg'][d], pm))
        for name, rows in (('w_ih', v['xp'][d]), ('w_hh', v['hs'][d, :L])):
            r = flat(ra(rows, pm))
            out.append((name, d, dg.t() @ r, (dg.shape[0] + 2 + AUTO_SPLIT_MAX) * U * (dg.abs().t() @ r.abs())))
        g32 = flat(v['dg'][d].double())
        s = g32.sum(0)
        bound = (g32.shape[0] // 8 + 8 + 4) * U * g32.abs().sum(0)
        out.append(('b_ih', d, s, bound))
        out.append(('b_hh', d, s, bound))
        a = ra(v['dg'][d][t[d]], pm)                                    # [L (position), B, 4H]
        w = rw(prm['w_ih' + ('_reverse' if d else '')], pm)
        dx = dx + (a @ w).transpose(0, 1)
        b_dx = b_dx + (4 * H + 2) * U * (a.abs() @ w.abs()).transpose(0, 1)
    out.append(('dx', None, dx, b_dx + U * dx.abs()))
    return out


def _grad_name(name, d):
    return name + ('_reverse' if d else '')


def check_closing(v, prm, lengths, grads, prefill, dx, precision, report=None):
    """Each parameter gradient (accumulated onto prefill: {PARAMS name: the value the gradient buffer held before the backward})
    and dx [B, L, E] against the fp64 products of the kernel's own dg.  One stage per product, reported at step 0."""
    B, L, E, H = _dims(v)
    rep = report or Report(L)
    dev = v['dg'].device
    for name, d, ref, bound in closing_products(v, prm, precision):
        if name == 'dx':
            pad = ~(torch.arange(L, device=dev)[None, :, None] < lengths.to(dev).long()[:, None, None])
            err = (dx.double() - ref).abs()
            rep.add('dx', 0, torch.where(pad, torch.zeros_like(err), err)[None], bound[None])
            rep.add('dx_pad', 0, torch.where(pad, dx.double().abs(), torch.zeros_like(err))[None], torch.zeros_like(err)[None])
            continue
        key = _grad_name(name, d)
        want = prefill[key].double() + ref
        stage = 'd' + name[0].upper() + name[1:] if name.startswith('w') else 'd' + name
        rep.add(stage, 0, (grads[key].double() - want).abs()[None, None],
                (bound + U * (prefill[key].double().abs() + want.abs()))[None, None])
    return rep


def check_all(v, prm, x, lengths, out, dout, grads, prefill, dx, precision, persist, split=1, split_b=1):
    rep = check_forward(v, prm, x, lengths, out, precision, persist, split)
    check_backward(v, prm, lengths, dout, precision, persist, split_b, rep)
    check_closing(v, prm, lengths, grads, prefill, dx, precision, rep)
    return rep


# ------------------------------------------------------------------------------------------------------------------------
# synthetic saved state (CPU tests): the same recurrence in fp64, rounded to fp32 where the kernels store
# ------------------------------------------------------------------------------------------------------------------------
def synthetic(B=13, L=11, E=24, H=16, precision='fp32', persist=True, split=1, split_b=1, seed=0, fault=None):
    """-> dict(v, prm, x, lengths, out, dout, grads, prefill, dx).  Lengths are unsorted and ragged, with 1 and L present.
    fault: (kind, ...) a kernel-style mistake made while the trajectory is produced:
        ('gate', d, j, b, k)      the stored gate element moved by 4x its bound (the cell goes on from the moved value)
        ('dh_rec', d, j)          the recurrent d h of step j dropped
        ('dc', d, j)              the d c carry lost on entry to step j
        ('rev_start', b)          the reverse direction of utterance b starts from a nonzero state
        ('out_pad', d, j, b)      a nonzero output at a frozen step
        ('dg_frozen', d, j, b)    a nonzero gate gradient at a frozen step"""
    g = torch.Generator().manual_seed(seed)
    r = lambda *s, scale=1.0: (torch.randn(*s, generator=g, dtype=torch.float64) * scale).float()   # noqa: E731
    k = 2.0 / H ** 0.5
    prm = {}
    for n in PARAMS:
        shape = {'w_ih': (4 * H, E), 'w_hh': (4 * H, H)}.get(n.replace('_reverse', ''), (4 * H,))
        prm[n] = r(*shape, scale=k)
    x = r(B, L, E)
    lengths = torch.randint(1, L + 1, (B,), generator=g)
    lengths[B // 2], lengths[1] = L, 1
    dout = r(B, L, 2 * H)
    fault = fault or ()
    kind = fault[0] if fault else None
    z = lambda *s: torch.zeros(*s, dtype=torch.float32)                # noqa: E731
    v = {'xp': z(2, L, B, E), 'gates': z(2, L, B, 4 * H), 'hs': z(2, L + 1, B, H), 'cs': z(2, L + 1, B, H), 'bsum': z(2, 4 * H),
         'dg': z(2, L, B, 4 * H), 'dxp': z(2, L, B, E)}
    t = positions(L, 'cpu')
    valid = valid_steps(lengths, L, 'cpu')
    out = z(B, L, 2 * H)
    w_ih, w_hh = pair(prm, 'w_ih'), pair(prm, 'w_hh')
    for d in range(2):
        v['xp'][d] = x[:, t[d]].transpose(0, 1)
        v['bsum'][d] = (prm[_grad_name('b_ih', d)].double() + prm[_grad_name('b_hh', d)].double()).float()
        if kind == 'rev_start' and d == 1:
            v['hs'][1, 0, fault[1]] = 0.25
            v['cs'][1, 0, fault[1]] = -0.5
        for j in range(L):
            proj, _, zz, b_z = preact(v['xp'][d, j], v['hs'][d, j], w_ih[d], w_hh[d], v['bsum'][d], precision, persist, split)
            gg, b_g = gates_ref(zz, b_z)
            gs = gg.float()
            if kind == 'gate' and fault[1:3] == (d, j):
                b, kk = fault[3], fault[4]
                gs[b, kk] = float(gg[b, kk] + 4 * b_g[b, kk])
            m = valid[d, j][:, None]
            v['gates'][d, j] = torch.where(m, gs, proj.float()) if persist else gs
            c, h, _, _ = cell_forward(v['gates'][d, j].double(), v['cs'][d, j].double(), v['hs'][d, j].double(), None, None, CELL, 'fp32')
            v['cs'][d, j + 1] = torch.where(m, c.float(), v['cs'][d, j])
            v['hs'][d, j + 1] = torch.where(m, h.float(), v['hs'][d, j])
            out[:, t[d, j], d * H:(d + 1) * H] = torch.where(m, h.float(), torch.zeros_like(h.float()))
            if kind == 'out_pad' and fault[1:3] == (d, j):
                out[fault[3], t[d, j], d * H] = 1e-3
    # backward
    dop = processing_order(dout, H)
    for d in range(2):
        dc = torch.zeros(B, H, dtype=torch.float64)
        for j in range(L - 1, -1, -1):
            nxt = None if (j == L - 1 or (kind == 'dh_rec' and fault[1:] == (d, j))) else v['dg'][d, j + 1]
            dh, b_dh = dh_ref(dop[d, j], nxt, w_hh[d], precision, persist, split_b)
            if kind == 'dc' and fault[1:] == (d, j):
                dc = torch.zeros_like(dc)
            dg, _, dcp, _, _, _ = cell_backward(dh, b_dh, dc, torch.zeros_like(dc), v['gates'][d, j].double(), v['cs'][d, j].double(),
                                                None, None, CELL, 'fp32')
            m = valid[d, j][:, None]
            v['dg'][d, j] = torch.where(m, dg.float(), torch.zeros_like(dg.float()))
            if kind == 'dg_frozen' and fault[1:3] == (d, j):
                v['dg'][d, j, fault[3], 0] = 1e-3
            dc = torch.where(m, dcp, dc)
    prefill = {n: r(*prm[n].shape, scale=0.1) for n in PARAMS}
    grads = {n: p.clone() for n, p in prefill.items()}
    dx = None
    for name, d, ref, _ in closing_products(v, prm, precision):
        if name == 'dx':
            dx = ref.float()
        else:
            key = _grad_name(name, d)
            grads[key] = (prefill[key].double() + ref).float()
    return dict(v=v, prm=prm, x=x, lengths=lengths, out=out, dout=dout, grads=grads, prefill=prefill, dx=dx)


def check_synthetic(s, precision='fp32', persist=True, split=1, split_b=1):
    return check_all(s['v'], s['prm'], s['x'], s['lengths'], s['out'], s['dout'], s['grads'], s['prefill'], s['dx'], precision, persist,
                     split, split_b)


# (B, L, E, H, lengths, expected path) of the GPU step checks (tests/test_gpu_bilstm_steps.py).  lengths: None = random in [1, L]
# with L present, 'unsorted' = groups of 8 whose longest utterance alternates between short and long.  test_bilstm_check_cpu.py
# pins the path of each and the edges they cover.
GPU_CASES = [
    (16, 180, 512, 256, None, 'persist'),          # cfg 1 encoder (LJ Speech): cluster of 8 at the real length
    (64, 180, 512, 256, None, 'persist'),
    (64, 180, 256, 128, None, 'persist'),          # cfg 3 encoder (shared_switching): cluster of 4
    (40, 60, 128, 64, 'unsorted', 'persist'),      # groups of 8 ending far earlier than their neighbours
    (61, 47, 64, 32, None, 'persist'),             # cluster of 1, partial last group; lengths 1 and L present
    (1, 1, 64, 32, None, 'persist'),               # single utterance, L = 1
    (1, 23, 64, 32, None, 'persist'),
    (9, 30, 96, 224, None, 'persist'),             # CS = 7
    (9, 19, 48, 24, None, 'chain'),                # H % 32 != 0
    (8, 20, 64, 288, None, 'chain'),               # H > 256
]


def gpu_lengths(B, L, lengths, seed):
    """The length list of a GPU case: random in [1, L] with 1 and L present, in no particular order; 'unsorted': groups of 8 whose
    longest utterance alternates between L / 6 and L (both directions then skip whole groups for many steps next to running ones)."""
    g = torch.Generator().manual_seed(seed)
    if lengths == 'unsorted':
        out = []
        for b in range(B):
            top = max(1, L // 6) if (b // 8) % 2 == 0 else L
            out.append(int(torch.randint(1, top + 1, (1,), generator=g)))
        for q in range(0, B, 8):
            out[min(B - 1, q + 3)] = max(1, L // 6) if (q // 8) % 2 == 0 else L
        return torch.tensor(out)
    out = torch.randint(1, L + 1, (B,), generator=g)
    perm = torch.randperm(B, generator=g)
    out[perm[0]] = L
    if B > 1:
        out[perm[1]] = 1
    return out
