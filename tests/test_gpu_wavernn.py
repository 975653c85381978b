"""WaveRNN on the GPU at the reference's dimensions (rnn / fc 512, compute / res_out 128, 10 res blocks, factors 5 x 5 x 11) with random
small-norm weights, both modes, ragged mel lengths:
  1. the upsampling network and the conditioning products against the fp64 oracle;
  2. a step-local check of the persistent loop: every step of every fold row recomputed in fp64 from the loop's own recorded state and
     sample of the previous step, with the operand-quantised oracle;
  3. the post-processing against the oracle's mu-law / unfold / fade of the loop's folded samples;
  4. batch invariance: generate_batch equals generate of each mel, bit for bit, given the same uniform tapes;
  5. the optional de-emphasis of the folds against the oracle's lfilter;
  6. state carried across several loop launches equals one launch, bit for bit;
  7. generate_batch computes in fp32 (and restores the caller's precision mode) when the library is in bf16 mode."""
import numpy as np
import pytest
import torch

import wavernn_oracle as O
from multilingual_text_to_speech_b200 import _lib
from multilingual_text_to_speech_b200.modules.wavernn import WaveRNN

pytestmark = pytest.mark.gpu

REAL = dict(rnn_dims=512, fc_dims=512, bits=9, pad=2, upsample_factors=(5, 5, 11), feat_dims=80, compute_dims=128, res_out_dims=128,
            res_blocks=10, hop_length=275, sample_rate=22050)
FRAMES = (21, 26, 33)
TARGET, OVERLAP = 1800, 100                  # 2,000 steps per fold row; 3 + 4 + 5 rows
# fp32 accumulation of a K-term product (tensor-core or SIMT order unknown): |error| <= K 2^-23 sum |w a|
GAMMA = 2.0 ** -23
# fp32 softmax / CDF (RAW) and Gumbel scores (MOL) in the loop against fp64: a decision within this margin of a boundary may go either
# way.  RAW: each lane sums n / 32 exponentials, then a 5-level scan and the threshold u S, each term within a few fp32 roundings of the
# total: 2 (n / 32 + 8) 2^-24 of the CDF.  MOL: scores of magnitude <= ~20 through two logs.
DECISION_EPS = {'RAW': 2 * (512 / 32 + 8) * 2.0 ** -24, 'MOL': 1e-4}
# such steps, at most this fraction of all steps (measured: RAW 85 and MOL 3 of 24,000; the 512 classes lie about 2e-3 apart in the CDF)
AMBIGUOUS_FRACTION = 1e-2
UPSAMPLE_RTOL = 1e-4                         # fp32 MelResNet (10 blocks) and FIR cascade against fp64, relative to each feature's scale


def make_model(mode, seed=0):
    torch.manual_seed(seed)
    m = WaveRNN(**dict(REAL, mode=mode))
    with torch.no_grad():
        for name, p in m.named_parameters():
            if 'batch_norm' in name:
                p.copy_(1 + 0.1 * torch.randn_like(p) if name.endswith('weight') else 0.1 * torch.randn_like(p))
        for name, b in m.named_buffers():
            if name.endswith('running_mean'):
                b.copy_(0.1 * torch.randn_like(b))
            elif name.endswith('running_var'):
                b.copy_(1 + 0.2 * torch.rand_like(b))
        for i in (1, 3, 5):
            w = m.upsample.up_layers[i].weight
            w.add_(0.02 * torch.randn_like(w))
        m.fc3.weight.mul_(20.0)          # a softmax far from uniform
    return m.cuda().eval()


def mels(seed=1):
    rng = np.random.default_rng(seed)
    return [rng.standard_normal((80, f)).astype(np.float32) for f in FRAMES]


def tapes(m, target, overlap, seed=2):
    g = torch.Generator().manual_seed(seed)
    return [torch.rand(m.tape_shape(f, target, overlap), generator=g) for f in FRAMES]


@pytest.fixture(scope='module', params=['RAW', 'MOL'])
def case(request):
    _lib.set_precision('fp32')
    mode = request.param
    m = make_model(mode)
    ms = mels()
    us = tapes(m, TARGET, OVERLAP)
    rows = sum(u.shape[0] for u in us)
    L = TARGET + 2 * OVERLAP
    D = 4 * 512 + 2 * 512 + m.n_classes
    trace = {'dbg': torch.full((L, rows, D), float('nan'), device='cuda')}
    specs = [torch.from_numpy(x).cuda() for x in ms]
    with torch.no_grad():
        wave, wave_off = m._generate(specs, list(FRAMES), us, TARGET, OVERLAP, None, torch.device('cuda'), trace)
    torch.cuda.synchronize()
    return m, ms, us, trace, wave.cpu().numpy(), wave_off


def _oracle_features(p, ms):
    feats = []
    for x in ms:
        mu, aux = O.upsample(p, x.astype(np.float64), (5, 5, 11), 2, 10)
        feats.append(O.fold_with_overlap(np.concatenate([mu, aux], axis=1), TARGET, OVERLAP))
    return np.concatenate(feats).transpose(1, 0, 2)             # [L, rows, 208]


def test_upsampling_and_conditioning_against_fp64(case):
    m, ms, us, trace, _, _ = case
    assert trace['chunk'] == TARGET + 2 * OVERLAP
    p = O.sd64(m)
    ref = _oracle_features(p, ms)
    got = trace['feat'].double().cpu().numpy()
    assert got.shape == ref.shape
    scale = np.abs(ref).max(axis=(0, 1))
    err = np.abs(got - ref) / (scale + 1e-30)
    assert err.max() <= UPSAMPLE_RTOL, err.max()
    # conditioning from the loop's own features: the fp32 GEMM against fp64 with the accumulation bound
    w = O.loop_weights(p, 512, 512, False)
    absw = {k: np.abs(v) for k, v in w.items()}
    ref_c = O.conditioning(w, got, 80, 32)
    mag = O.conditioning(absw, np.abs(got), 80, 32)
    Ks = (112, 512, 32, 32, 32)
    bound_c = None
    for name, g, r, a, K in zip(('c', 'g1', 'c2', 'p1', 'p2'), trace['cond'], ref_c, mag, Ks):
        g = g.double().cpu().numpy()
        bound = K * GAMMA * a + 2 * GAMMA * np.abs(r) + 1e-30
        if name == 'c':
            bound_c = bound
        if name == 'g1':                 # g1 multiplies the loop's fp32 c, which carries c's error
            bound = bound + bound_c @ absw['w_ih1'].T
        ratio = np.abs(g - r) / bound
        assert ratio.max() <= 1.0, (name, ratio.max())


def _tt(x):
    return torch.as_tensor(x, dtype=torch.float64, device='cuda')


def test_step_local_check_of_the_loop(case):
    m, ms, us, trace, _, _ = case
    L, R = TARGET + 2 * OVERLAP, 512
    n = m.n_classes
    dbg = trace['dbg'].double()
    assert not torch.isnan(dbg).any()
    rows = dbg.shape[1]
    h1, x1b, h2, x2b = (dbg[..., i * R:(i + 1) * R] for i in range(4))
    y1b, y2b, logits = dbg[..., 4 * R:5 * R], dbg[..., 5 * R:6 * R], dbg[..., 6 * R:]
    y = trace['folded'].double().t()                                # [L, rows]
    zero = torch.zeros(1, rows, R, dtype=torch.float64, device='cuda')
    h1p, h2p = torch.cat([zero, h1[:-1]]), torch.cat([zero, h2[:-1]])
    prev = torch.cat([torch.zeros(1, rows, dtype=torch.float64, device='cuda'), y[:-1]])[..., None]
    p = O.sd64(m)
    wq = {k: _tt(v) for k, v in O.loop_weights(p, R, 512, True).items()}
    c, g1, c2, p1, p2 = (t.double() for t in trace['cond'])
    q = lambda a: a.to(torch.bfloat16).double()
    wp = _tt(p['I.weight'][:, 0])
    u1 = trace['weights']['u1'].double()                            # the loop's own u1 (fp32 GEMM of W_ih1 and w)

    def gemv(W, a, K):
        return a @ W.T, K * GAMMA * (a.abs() @ W.abs().T)

    def gru(gi, gh, egi, egh, h):
        r = torch.sigmoid(gi[..., :R] + gh[..., :R])
        z = torch.sigmoid(gi[..., R:2 * R] + gh[..., R:2 * R])
        nn_ = torch.tanh(gi[..., 2 * R:] + r * gh[..., 2 * R:])
        e = egi + egh
        bound = 0.25 * e[..., :R] * (gh[..., 2 * R:].abs() + egh[..., 2 * R:]) + 0.25 * e[..., R:2 * R] * (nn_ - h).abs() + \
            e[..., 2 * R:] + 4e-7 * (1 + h.abs())
        return (1 - z) * nn_ + z * h, bound

    def check(name, got, ref, bound):
        ratio = ((got - ref).abs() / bound).max().item()
        assert ratio <= 1.0, (name, ratio)

    def check_bf16(name, got, ref, e):
        check(name, got, ref, 2.0 ** -8 * ref.abs() + e + 1e-30)

    # 1. GRU1 from the loop's h1 and sample of the previous step
    gh, egh = gemv(wq['w_hh1'], q(h1p), R)
    gh = gh + wq['b_hh1']
    gi = g1 + u1 * prev
    h1o, b1 = gru(gi, gh, 4 * GAMMA * gi.abs(), egh + 2 * GAMMA * gh.abs(), h1p)
    check('h1', h1, h1o, b1)
    x1 = c + wp * prev + h1
    check_bf16('x1', x1b, x1, 4 * GAMMA * (c.abs() + (wp * prev).abs() + h1.abs()))
    # 2. GRU2 from the loop's bf16 x and h2
    gi, egi = gemv(wq['w_ih2x'], x1b, R)
    gi = gi + c2
    gh, egh = gemv(wq['w_hh2'], q(h2p), R)
    gh = gh + wq['b_hh2']
    h2o, b2 = gru(gi, gh, egi + 2 * GAMMA * gi.abs(), egh + 2 * GAMMA * gh.abs(), h2p)
    check('h2', h2, h2o, b2)
    check_bf16('x2', x2b, x1 + h2, 4 * GAMMA * (x1.abs() + h2.abs()) + 4 * GAMMA * (c.abs() + (wp * prev).abs() + h1.abs()))
    # 3. - 5. the fc stack, each from the loop's own bf16 input
    for name, W, a, P, got in (('y1', 'w_fc1x', x2b, p1, y1b), ('y2', 'w_fc2x', y1b, p2, y2b)):
        v, e = gemv(wq[W], a, 512)
        v = v + P
        check_bf16(name, got, torch.relu(v), e + 2 * GAMMA * v.abs())
    v, e = gemv(wq['w_fc3'], y2b, 512)
    v = v + wq['b_fc3']
    check('logits', logits, v, e + 2 * GAMMA * v.abs() + 1e-30)
    # 6. the sample from the loop's logits
    uni = trace['uniforms'].double().permute(1, 0, 2)                 # [L, rows, U]
    total = L * rows
    if m.mode == 'RAW':
        pr = torch.softmax(logits, -1)
        cdf = torch.cumsum(pr, -1)
        u = uni[..., 0]
        k = torch.searchsorted(cdf.contiguous(), u[..., None].contiguous(), right=True)[..., 0].clamp(max=n - 1)
        hi = cdf.gather(-1, k[..., None])[..., 0]
        lo = torch.where(k > 0, cdf.gather(-1, (k - 1).clamp(min=0)[..., None])[..., 0], torch.zeros_like(u))
        margin = torch.minimum((hi - u).abs(), (u - lo).abs())
        kk = torch.round((y + 1) * (n - 1) / 2).long()
        kf = kk.cpu().numpy().astype(np.float32)
        cls = np.float32(2) * kf / np.float32(n - 1) - np.float32(1)           # the loop's fp32 arithmetic
        assert np.array_equal(cls.astype(np.float64), y.cpu().numpy()), 'a RAW sample is not a class value'
        ambiguous = margin < DECISION_EPS[m.mode]
        wrong = (kk != k) & ~ambiguous
        assert not wrong.any(), f'{int(wrong.sum())} RAW decisions differ outside the fp32 margin'
    else:
        nr = n // 3
        uu = 1e-5 + (1 - 2e-5) * uni
        score = logits[..., :nr] - torch.log(-torch.log(uu[..., :nr]))
        top = torch.topk(score, 2, dim=-1)
        j = top.indices[..., 0]
        margin = top.values[..., 0] - top.values[..., 1]
        ambiguous = margin < DECISION_EPS[m.mode]
        ls = torch.clamp(logits.gather(-1, (2 * nr + j)[..., None])[..., 0], min=float(np.log(1e-14)))
        mean = logits.gather(-1, (nr + j)[..., None])[..., 0]
        lu = torch.log(uu[..., nr]) - torch.log(1 - uu[..., nr])
        x = torch.clamp(mean + torch.exp(ls) * lu, -1, 1)
        bound = 1e-5 * (1 + torch.exp(ls) * lu.abs())
        wrong = ((x - y).abs() > bound) & ~ambiguous
        assert not wrong.any(), f'{int(wrong.sum())} MOL samples differ beyond {bound.max().item():.2e} outside the margin'
    n_amb = int(ambiguous.sum())
    print(f'{m.mode}: {n_amb} of {total} steps within {DECISION_EPS[m.mode]:.2e} of a decision boundary')
    assert n_amb <= AMBIGUOUS_FRACTION * total, n_amb


def test_postprocessing_against_oracle(case):
    m, ms, us, trace, wave, wave_off = case
    folded = trace['folded'].double().cpu().numpy()
    ro = trace['row_off']
    for b, f in enumerate(FRAMES):
        ref = O.postprocess(folded[ro[b]:ro[b + 1]], f, 275, TARGET, OVERLAP, m.n_classes if m.mode == 'RAW' else None)
        got = wave[wave_off[b]:wave_off[b] + (f - 1) * 275]
        assert got.shape == ref.shape
        np.testing.assert_allclose(got, ref, rtol=1e-6, atol=1e-7)


# de-emphasis runs on the fp32 scan: a few roundings per sample, amplified by up to 1 / (1 - a) through the recurrence
def _deemphasis_bound(a):
    return 32 * 2.0 ** -24 / (1 - abs(a))


@pytest.mark.parametrize('a', [0.97, -0.5])
def test_postprocessing_with_deemphasis_against_oracle(case, a):
    m, ms, us, trace, _, _ = case
    before = trace['folded'].clone()
    wave, wave_off = m.postprocess(trace['folded'], list(FRAMES), TARGET, OVERLAP, a)
    assert torch.equal(before, trace['folded'])                       # the loop's samples are left as they were
    wave = wave.cpu().numpy()
    folded = trace['folded'].double().cpu().numpy()
    ro = trace['row_off']
    for b, f in enumerate(FRAMES):
        ref = O.postprocess(folded[ro[b]:ro[b + 1]], f, 275, TARGET, OVERLAP, m.n_classes if m.mode == 'RAW' else None, a)
        got = wave[wave_off[b]:wave_off[b] + (f - 1) * 275]
        err = np.abs(got - ref).max() / np.abs(ref).max()
        assert err <= _deemphasis_bound(a), err


def test_state_carried_across_chunks(monkeypatch):
    """Several loop launches (h1 / h2 buffer parity, the previous sample and the global step index carried between them) compute
    exactly what one launch computes; the one-launch run is the one the step-local check covers."""
    from multilingual_text_to_speech_b200.modules import wavernn
    _lib.set_precision('fp32')
    m = make_model('RAW', seed=8)
    ms = mels(seed=9)
    us = tapes(m, TARGET, OVERLAP, seed=10)
    specs = [torch.from_numpy(x).cuda() for x in ms]
    runs = []
    for cond_bytes in (wavernn.COND_BYTES, 300 * 12 * 4 * (80 + 128 + 7 * 512 + 2 * 512)):
        monkeypatch.setattr(wavernn, 'COND_BYTES', cond_bytes)
        trace = {}
        with torch.no_grad():
            wave, _ = m._generate(specs, list(FRAMES), us, TARGET, OVERLAP, None, torch.device('cuda'), trace)
        runs.append((trace['chunk'], trace['folded'].clone(), wave.clone()))
    (c1, y1, w1), (c2, y2, w2) = runs
    assert c1 == TARGET + 2 * OVERLAP and c2 == 300, (c1, c2)            # one launch, then seven (the last one partial)
    assert torch.equal(y1, y2) and torch.equal(w1, w2)


def test_generate_batch_runs_in_fp32_whatever_the_precision_mode():
    m = make_model('MOL', seed=11)
    ms = mels(seed=12)
    us = tapes(m, 600, 50, seed=13)
    _lib.set_precision('fp32')
    ref = m.generate_batch(ms, 600, 50, uniforms=us)
    _lib.set_precision('bf16')
    try:
        got = m.generate_batch(ms, 600, 50, uniforms=us)
        assert _lib.get_precision() == 'bf16'                          # restored after the call
    finally:
        _lib.set_precision('fp32')
    for r, g in zip(ref, got):
        assert np.array_equal(r, g)


@pytest.mark.parametrize('mode', ['RAW', 'MOL'])
def test_batch_invariance(mode):
    _lib.set_precision('fp32')
    m = make_model(mode, seed=5)
    ms = mels(seed=6)
    us = tapes(m, 600, 50, seed=7)
    batch = m.generate_batch(ms, 600, 50, uniforms=us)
    for i, x in enumerate(ms):
        one = m.generate(x, 600, 50, uniforms=us[i])
        assert isinstance(one, np.ndarray) and one.shape == ((FRAMES[i] - 1) * 275,)
        assert np.array_equal(one, batch[i]), i
        assert np.isfinite(one).all()
    # torch in -> torch out on the input's device; default tapes from torch.rand
    t = m.generate_batch([torch.from_numpy(ms[0]).cuda()], 600, 50, generator=torch.Generator(device='cuda').manual_seed(0))[0]
    assert t.is_cuda and t.shape == ((FRAMES[0] - 1) * 275,)
