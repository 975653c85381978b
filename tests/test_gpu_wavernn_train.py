"""WaveRNN training on the GPU at the reference's dimensions (rnn / fc 512, compute / res_out 128, 10 res blocks, factors 5 x 5 x 11), RAW
and MOL:
  1. fp32 mode: logits, loss, every parameter gradient and the updated batch-norm running statistics against the fp64 oracle; eval mode
     (running statistics, none updated) against the oracle;
  2. every step of both GRU loops, forward and reverse, step-checked in fp64 from the loop's own recorded state, for B in {1, 7, 32, 64}
     and T in {275, 1375, 2750}; two identical calls give identical bits;
  3. the loss kernels in each MOL branch against the oracle's autograd;
  4. the weight gradients of the GRUs and of fc3 against fp64 products of the step's own operands (rounded to bf16 in bf16 mode, as the
     tensor-core GEMMs round them), in both precision modes; bf16 mode's gradients against fp32 mode;
  5. five FusedAdam steps (clip 4, lr 1e-4) against torch.optim.Adam on the fp64 oracle, then generate_batch with the trained model.
Bounds: DESIGN.md section 11."""
import numpy as np
import pytest
import torch

import wavernn_train_oracle as TO
from multilingual_text_to_speech_b200 import _lib
from multilingual_text_to_speech_b200.distributed import GradBucket
from multilingual_text_to_speech_b200.modules.wavernn import WaveRNN, label_2_float, wavernn_loss
from multilingual_text_to_speech_b200.optim import FlatParams, FusedAdam

pytestmark = pytest.mark.gpu

REAL = dict(rnn_dims=512, fc_dims=512, bits=9, pad=2, upsample_factors=(5, 5, 11), feat_dims=80, compute_dims=128, res_out_dims=128,
            res_blocks=10, hop_length=275, sample_rate=22050)
U = 2.0 ** -24
# fp32 against fp64, normwise ||got - ref|| / ||ref|| per tensor
LOGITS_RTOL, LOSS_RTOL, GRAD_RTOL, STATS_ATOL = 1e-4, 1e-6, 2e-3, 1e-5
# bf16 mode (tensor-core operands outside the fp32 GRU loops) against fp32 mode, normwise: the whole gradient vector, and each tensor.  At
# random weights and labels the gradients are sums of many cancelling terms, so bf16 operand rounding shows up strongly (measured 0.12 /
# 0.022 whole, 0.17 / 0.15 worst tensor for RAW / MOL, a batch-norm bias)
BF16_GRAD_RTOL, BF16_TENSOR_RTOL = 0.25, 0.3
# FusedAdam against fp64 Adam after 5 steps at lr 1e-4: a step moves an element by at most about lr, so an element whose update differs
# (a near-zero gradient of another sign) may differ by 2 lr per step; 99 % of the elements stay within one step size
LR = 1e-4
ADAM_MAX_ABS, ADAM_Q99 = 10 * LR, LR


def make_model(mode, seed=0):
    torch.manual_seed(seed)
    m = WaveRNN(**dict(REAL, mode=mode))
    with torch.no_grad():
        for name, p in m.named_parameters():
            if 'batch_norm' in name:
                p.copy_(1 + 0.1 * torch.randn_like(p) if name.endswith('weight') else 0.1 * torch.randn_like(p))
        for i in (1, 3, 5):
            w = m.upsample.up_layers[i].weight
            w.add_(0.02 * torch.randn_like(w))
    return m.train()


def make_batch(mode, B, T, seed=1):
    g = torch.Generator().manual_seed(seed)
    mels = torch.randn(B, 80, T // 275 + 4, generator=g)
    if mode == 'RAW':
        lab = torch.randint(0, 512, (B, T + 1), generator=g)
        return label_2_float(lab[:, :T], 9), lab[:, 1:], mels
    lab = torch.randint(0, 65536, (B, T + 1), generator=g)
    lab[:, 1::97] = 0                        # targets at -1 and +1 exercise those branches
    lab[:, 2::89] = 65535
    return label_2_float(lab[:, :T], 16), label_2_float(lab[:, 1:], 16), mels


def gpu_step(m, x, y, mels, mode, trace=None):
    m.zero_grad(set_to_none=True)
    logits = m(x.cuda(), mels.cuda(), trace)
    loss = wavernn_loss(logits, y.cuda(), mode)
    loss.backward()
    torch.cuda.synchronize()
    return logits.detach(), loss.detach(), {n: p.grad.detach().clone() for n, p in m.named_parameters()}


def rel(a, b):
    a, b = a.double().cpu(), b.double().cpu()
    return float((a - b).norm() / b.norm().clamp_min(1e-300))


@pytest.fixture(autouse=True)
def fp32_mode():
    _lib.set_precision('fp32')
    yield
    _lib.set_precision('fp32')


@pytest.mark.parametrize('mode', ['RAW', 'MOL'])
def test_train_step_matches_fp64_oracle(mode):
    m = make_model(mode)
    m64 = TO.double_copy(m)
    m.cuda()
    x, y, mels = make_batch(mode, 7, 1375)
    logits, loss, grads = gpu_step(m, x, y, mels, mode)
    ref_logits, ref_loss = TO.train_step(m64, x.double(), y if mode == 'RAW' else y.double(), mels.double(), mode)
    errs = {'logits': rel(logits, ref_logits), 'loss': rel(loss, ref_loss)}
    assert errs['logits'] <= LOGITS_RTOL and errs['loss'] <= LOSS_RTOL, errs
    worst = max(((rel(grads[n], p.grad), n) for n, p in m64.named_parameters()))
    print(f'\n[{mode}] logits {errs["logits"]:.2e} loss {errs["loss"]:.2e} worst gradient {worst[0]:.2e} ({worst[1]})')
    for n, p in m64.named_parameters():
        assert rel(grads[n], p.grad) <= GRAD_RTOL, (n, rel(grads[n], p.grad))
    b32, b64 = dict(m.named_buffers()), dict(m64.named_buffers())
    for n in b64:
        if 'running' in n:
            torch.testing.assert_close(b32[n].double().cpu(), b64[n], rtol=0, atol=STATS_ATOL * (1 + float(b64[n].abs().max())))
        else:
            assert int(b32[n]) == int(b64[n]), n         # step and num_batches_tracked
    assert int(b32['step']) == 1


@pytest.mark.parametrize('mode', ['RAW', 'MOL'])
def test_eval_mode_forward_matches_fp64_oracle(mode):
    m = make_model(mode)
    with torch.no_grad():
        for name, b in m.named_buffers():
            if name.endswith('running_mean'):
                b.copy_(0.1 * torch.randn_like(b))
            elif name.endswith('running_var'):
                b.copy_(1 + 0.2 * torch.rand_like(b))
    m.eval()
    m64 = TO.double_copy(m)
    m.cuda()
    before = {n: b.clone() for n, b in m.named_buffers()}
    x, _, mels = make_batch(mode, 7, 1375)
    with torch.no_grad():
        logits = m(x.cuda(), mels.cuda())
        ref = TO.forward(m64, x.double(), mels.double())
    assert rel(logits, ref) <= LOGITS_RTOL, rel(logits, ref)
    for n, b in m.named_buffers():
        if n == 'step':
            assert int(b) == int(before[n]) + 1 == int(dict(m64.named_buffers())[n])
        else:
            assert torch.equal(b, before[n]), n          # eval mode reads the running statistics and updates nothing


def bf16(t):
    return t.to(torch.bfloat16).to(torch.float64)


def product_check(got, a, b, rounded):
    """got against a^T b in fp64 (a [K, M], b [K, N]) with operands rounded to bf16 when `rounded`: -> err / ((K + 2) 2^-24 |a|^T |b|)."""
    a, b = a.detach(), b.detach()
    a, b = (bf16(a), bf16(b)) if rounded else (a.double(), b.double())
    ref = a.T @ b
    bound = (a.shape[0] + 2) * U * (a.abs().T @ b.abs()) + 2.0 ** -126
    return float(((got.double() - ref).abs() / bound).max())


@pytest.mark.parametrize('precision', ['fp32', 'bf16'])
@pytest.mark.parametrize('mode', ['RAW', 'MOL'])
def test_weight_gradients_against_their_operands(mode, precision):
    m = make_model(mode).cuda()
    x, y, mels = make_batch(mode, 7, 1375)
    _lib.set_precision(precision)
    trace, dl = {}, {}
    m.zero_grad(set_to_none=True)
    logits = m(x.cuda(), mels.cuda(), trace)
    logits.register_hook(lambda g: dl.setdefault('g', g))
    wavernn_loss(logits, y.cuda(), mode).backward()
    torch.cuda.synchronize()
    rounded = precision == 'bf16'
    n = m.fc3.weight.shape[0]
    ratios = {'fc3.weight': product_check(m.fc3.weight.grad, dl['g'].reshape(-1, n), trace['y2'].reshape(-1, trace['y2'].shape[-1]), rounded)}
    for k, rnn in (('rnn1', m.rnn1), ('rnn2', m.rnn2)):
        tr = trace[k]
        B, T, R = tr['h'].shape
        dgi, dgh = tr['dgi'].reshape(B * T, 3 * R), tr['dgh']
        ratios[k + '.weight_ih'] = product_check(rnn.weight_ih_l0.grad.T, tr['x'], dgi, rounded)
        # d W_hh pairs dgh[b, t] with h[b, t - 1] (t >= 1) only
        ratios[k + '.weight_hh'] = product_check(rnn.weight_hh_l0.grad.T, tr['h'][:, :-1].reshape(-1, R), dgh[:, 1:].reshape(-1, 3 * R), rounded)
        for name, hist in (('bias_ih', dgi), ('bias_hh', dgh.reshape(B * T, 3 * R))):
            ones = torch.ones(B * T, 1, device='cuda')
            ratios[f'{k}.{name}'] = product_check(getattr(rnn, name + '_l0').grad.view(1, -1), ones, hist, False)
    print(f'\n[{mode} {precision}] worst err / bound ' + ' '.join(f'{k} {v:.3f}' for k, v in ratios.items()))
    assert all(v <= 1.0 for v in ratios.values()), ratios


def step_check_forward(tr, w_hh, b_hh):
    """Every step of the forward loop from its own recorded h_{t-1}: -> worst err / bound of h_t and of W_hn h + b_hn."""
    gi, h, saved = tr['gi'], tr['h'], tr['saved']
    B, T, R = h.shape
    W, bh = w_hh.detach().double().cuda(), b_hh.detach().double().cuda()
    worst = 0.0
    for b0 in range(0, B, 8):
        hb = h[b0:b0 + 8].double()
        hp = torch.cat([torch.zeros_like(hb[:, :1]), hb[:, :-1]], 1)
        gh = hp @ W.T + bh
        S = (hp.abs() @ W.abs().T + bh.abs()).view(*hp.shape[:2], 3, R)
        g = gi[b0:b0 + 8].double()
        r = torch.sigmoid(g[..., :R] + gh[..., :R])
        z = torch.sigmoid(g[..., R:2 * R] + gh[..., R:2 * R])
        n = torch.tanh(g[..., 2 * R:] + r * gh[..., 2 * R:])
        href = (1 - z) * n + z * hp
        scale = S.amax(2) + g.abs().view(*hp.shape[:2], 3, R).amax(2)
        bound = (R + 16) * U * scale * (2 + gh[..., 2 * R:].abs()) + 2.0 ** -20
        worst = max(worst, float(((hb - href).abs() / bound).max()))
        ghn = saved[b0:b0 + 8, :, 3 * R:].double()
        bound_n = (R + 2) * U * S[:, :, 2] + 2.0 ** -22
        worst = max(worst, float(((ghn - gh[..., 2 * R:]).abs() / bound_n).max()))
    return worst


def step_check_reverse(tr, w_hh):
    """Every step of the reverse loop from its own recorded dh_{t+1} and dgh_{t+1}: -> worst err / bound of dh_t, dgi_t and dgh_t."""
    dgi, dgh, dh, dh_ext, h, saved = tr['dgi'], tr['dgh'], tr['dh'], tr['dh_ext'], tr['h'], tr['saved']
    B, T, R = h.shape
    W = w_hh.detach().double().cuda()
    worst = 0.0
    shift = lambda a: torch.cat([a[:, 1:], torch.zeros_like(a[:, :1])], 1)      # noqa: E731  value of the later step (0 after the last)
    for b0 in range(0, B, 8):
        sl = slice(b0, b0 + 8)
        d, dn_, dgh_n = dh[sl].double(), shift(dh[sl].double()), shift(dgh[sl].double())
        sv = saved[sl].double()
        r, z, n, ghn = sv[..., :R], sv[..., R:2 * R], sv[..., 2 * R:3 * R], sv[..., 3 * R:]
        zdn = shift(z) * dn_
        dref = dh_ext[sl].double() + zdn + dgh_n @ W
        bound = (3 * R + 8) * U * (dgh_n.abs() @ W.abs() + zdn.abs() + dh_ext[sl].double().abs()) + 2.0 ** -126
        worst = max(worst, float(((d - dref).abs() / bound).max()))
        hb = h[sl].double()
        hp = torch.cat([torch.zeros_like(hb[:, :1]), hb[:, :-1]], 1)
        dnh = d * (1 - z) * (1 - n * n)
        drh = dnh * ghn * r * (1 - r)
        dzh = d * (hp - n) * z * (1 - z)
        cell_bound = 16 * U * d.abs() * (1 + hp.abs() + n.abs()) * (1 + ghn.abs()) + 2.0 ** -126
        for got, ref in ((dgi[sl, :, :R], drh), (dgi[sl, :, R:2 * R], dzh), (dgi[sl, :, 2 * R:], dnh), (dgh[sl, :, :R], drh),
                         (dgh[sl, :, R:2 * R], dzh), (dgh[sl, :, 2 * R:], r * dnh)):
            worst = max(worst, float(((got.double() - ref).abs() / cell_bound).max()))
    return worst


@pytest.mark.parametrize('T', [275, 1375, 2750])
@pytest.mark.parametrize('B', [1, 7, 32, 64])
@pytest.mark.parametrize('mode', ['RAW', 'MOL'])
def test_loops_step_checked_and_reproducible(mode, B, T):
    m = make_model(mode).cuda()
    x, y, mels = make_batch(mode, B, T, seed=B + T)
    trace = {}
    out1 = gpu_step(m, x, y, mels, mode, trace)
    ratios = {}
    for k, rnn in (('rnn1', m.rnn1), ('rnn2', m.rnn2)):
        ratios[k + ' fwd'] = step_check_forward(trace[k], rnn.weight_hh_l0, rnn.bias_hh_l0)
        ratios[k + ' rev'] = step_check_reverse(trace[k], rnn.weight_hh_l0)
    print(f'\n[{mode} B={B} T={T}] worst err / bound ' + ' '.join(f'{k} {v:.3f}' for k, v in ratios.items()))
    assert all(v <= 1.0 for v in ratios.values()), ratios
    del trace
    out2 = gpu_step(m, x, y, mels, mode)
    assert torch.equal(out1[0], out2[0]) and torch.equal(out1[1], out2[1])
    for n in out1[2]:
        assert torch.equal(out1[2][n], out2[2][n]), n


def test_mol_loss_kernel_in_each_branch():
    rng = np.random.default_rng(8)
    N, nr = 4096, 10
    logits = np.concatenate([rng.standard_normal((N, nr)), rng.uniform(-1, 1, (N, nr)), rng.uniform(-12, 2, (N, nr))], 1)
    logits[::7, 2 * nr:] = -40.0                 # below the clamp
    y = rng.uniform(-1, 1, N)
    y[::5], y[1::5] = -1.0, 1.0
    near = rng.integers(0, nr, N)
    logits[2::5, nr + near[2::5]] = y[2::5] + rng.uniform(-1e-3, 1e-3, len(y[2::5]))      # sharp mixtures at the target: cdf_delta > 1e-5
    lg = torch.tensor(logits, dtype=torch.float32)
    yt = torch.tensor(y, dtype=torch.float32)
    l64 = lg.double().view(1, N, 3 * nr).requires_grad_(True)
    ref = TO.mol_loss(l64, yt.double().view(1, N))
    ref.backward()
    lc = lg.cuda().requires_grad_(True)
    loss = wavernn_loss(lc.view(1, N, 3 * nr), yt.cuda().view(1, N), 'MOL')
    loss.backward()
    assert abs(float(loss) - float(ref)) <= 1e-5 * abs(float(ref))
    assert rel(lc.grad, l64.grad.view(N, 3 * nr)) <= 1e-4
    lr = torch.randn(N, 512).cuda().requires_grad_(True)
    lab = torch.randint(0, 512, (N,))
    loss = wavernn_loss(lr.view(1, N, 512), lab.cuda().view(1, N), 'RAW')
    loss.backward()
    l64 = lr.detach().double().cpu().requires_grad_(True)
    ref = TO.raw_loss(l64, lab)
    ref.backward()
    assert abs(float(loss) - float(ref)) <= 1e-5 * abs(float(ref)) and rel(lr.grad, l64.grad) <= 1e-5


@pytest.mark.parametrize('mode', ['RAW', 'MOL'])
def test_bf16_mode_gradients_close_to_fp32(mode):
    m = make_model(mode).cuda()
    x, y, mels = make_batch(mode, 32, 1375)
    _, loss32, g32 = gpu_step(m, x, y, mels, mode)
    _lib.set_precision('bf16')
    _, loss16, g16 = gpu_step(m, x, y, mels, mode)
    worst = max((rel(g16[n], g32[n]), n) for n in g32)
    whole = rel(torch.cat([g16[n].reshape(-1) for n in g32]), torch.cat([g32[n].reshape(-1) for n in g32]))
    print(f'\n[{mode}] bf16 against fp32: loss {rel(loss16, loss32):.2e}, whole gradient {whole:.2e}, worst tensor {worst[0]:.2e} '
          f'({worst[1]})')
    assert whole <= BF16_GRAD_RTOL and worst[0] <= BF16_TENSOR_RTOL, (whole, worst)


@pytest.mark.parametrize('mode', ['RAW', 'MOL'])
def test_fused_adam_tracks_fp64_oracle_then_generates(mode):
    m = make_model(mode)
    m64 = TO.double_copy(m)
    m.cuda()
    flat = FlatParams(m)
    bucket = GradBucket(m)
    opt = FusedAdam(flat, bucket, lr=LR, max_grad_norm=4.0)
    opt64 = torch.optim.Adam(m64.parameters(), lr=LR)
    for k in range(5):
        x, y, mels = make_batch(mode, 4, 550, seed=10 + k)
        bucket.zero()
        logits = m(x.cuda(), mels.cuda())
        wavernn_loss(logits, y.cuda(), mode).backward()
        for n, p in m.named_parameters():
            assert bool((p.grad != 0).any()), f'step {k}: {n} received no gradient'
        opt.step()
        opt64.zero_grad()
        TO.train_step(m64, x.double(), y if mode == 'RAW' else y.double(), mels.double(), mode)
        torch.nn.utils.clip_grad_norm_(m64.parameters(), 4.0)
        opt64.step()
    torch.cuda.synchronize()
    diffs = torch.cat([(p.detach().double().cpu() - p64.detach()).abs().reshape(-1) for p, p64 in zip(m.parameters(), m64.parameters())])
    q = [float(torch.quantile(diffs[::7], v)) for v in (0.5, 0.99)]
    print(f'\n[{mode}] after 5 Adam steps: |p - p64| median {q[0]:.2e}, 99th percentile {q[1]:.2e}, max {float(diffs.max()):.2e}')
    assert float(diffs.max()) <= ADAM_MAX_ABS and q[1] <= ADAM_Q99
    m.eval()
    mel = torch.randn(80, 24, device='cuda')
    wave = m.generate(mel, target=1100, overlap=55, generator=torch.Generator(device='cuda').manual_seed(0))
    assert wave.shape == (23 * 275,) and bool(torch.isfinite(wave).all())
