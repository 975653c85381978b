"""Griffin-Lim vocoder on the H100 against the fp64 numpy oracle (tests/audio_oracle.py): single transforms, every step of 60 iterations
recomputed from the kernels' own state, ragged-batch invariance, NNLS optimality, de-emphasis and the text -> waveform path."""
import numpy as np
import pytest
import scipy.signal
import torch

import audio_oracle as O
from test_vocoder_cpu import GL_DRIFT_FACTOR

pytestmark = pytest.mark.gpu

EPS = 2.0 ** -24
C_FFT = 16          # per-frame bound: C_FFT * log2(N) * 2^-24 * (||frame|| + 1e-3 * max frame norm)


@pytest.fixture(scope='module')
def mods():
    import __graft_entry__ as entry
    entry.build()
    from multilingual_text_to_speech_b200 import _lib, configs
    from multilingual_text_to_speech_b200 import functional as F
    from multilingual_text_to_speech_b200.utils import audio
    configs.apply('ljspeech')
    _lib.set_precision('fp32')
    return _lib, F, audio


def _shape(_lib, frames, n_fft, hop, win, n_mels=0, power=1.0, preemphasis=0.0, nnls_iters=0):
    return _lib.VocoderShape(len(frames), int(sum(frames)), n_fft, hop, win, n_mels, power, 0.99, preemphasis, nnls_iters)


def _pack(arrays, dtype):
    """[K, F_i] numpy arrays -> packed frame-major [sum F, K] CUDA tensor and int32 offsets."""
    off = np.concatenate([[0], np.cumsum([a.shape[1] for a in arrays])]).astype(np.int32)
    t = torch.from_numpy(np.concatenate([a.T for a in arrays]).astype(dtype)).cuda().contiguous()
    return t, torch.from_numpy(off).cuda()


def _signal(n, seed, f0=140.0):
    rng = np.random.default_rng(seed)
    t = np.arange(n) / 22050
    return sum(np.sin(2 * np.pi * f0 * k * t * (1 + 0.05 * t) + rng.uniform(0, 6)) / k for k in range(1, 25)) + 0.01 * rng.standard_normal(n)


def _frame_bound(ref, n_fft):
    """ref [K or N, F] -> per-frame bound."""
    norms = np.linalg.norm(ref, axis=0)
    return C_FFT * np.log2(n_fft) * EPS * (norms + 1e-3 * norms.max())


# the default plan [19, 29], [4, 4, 4, 4, 2] with and without a zero-padded window, then the other plans a user's hp.num_fft can give:
# [4, 4, 5, 5] (16 kHz), [2, 5, 5, 11], [3, 7, 13] (N - win odd), [23, 31], [31, 31] and [4, 4, 4, 4, 4]
@pytest.mark.parametrize('n_fft,hop,win', [(1102, 275, 1102), (1024, 256, 1024), (1024, 256, 800), (800, 200, 800), (1100, 275, 1100),
                                           (546, 136, 545), (1426, 356, 1426), (1922, 480, 1922), (2048, 512, 2048)])
def test_single_transforms_against_fp64(mods, n_fft, hop, win):
    _lib, F, _ = mods
    rng = np.random.default_rng(n_fft + win)
    Fr = 40
    S = np.abs(O.stft(_signal(hop * (Fr - 1), 1), n_fft, hop, win)).astype(np.float32)
    u = rng.uniform(0, 1, S.shape)
    ang = O.angles_from_uniform(u)
    St, off = _pack([S], np.float32)
    shape = _shape(_lib, [Fr], n_fft, hop, win)
    # iters = 0: the inverse path alone
    angles = _pack([ang], np.complex64)[0]
    rebuilt = torch.zeros_like(angles)
    wave = torch.empty(hop * (Fr - 1), device='cuda')
    F.griffinlim(shape, St, off, angles, rebuilt, True, 0, wave)
    ref = O.istft(S.astype(np.float64) * ang.astype(np.complex128), n_fft, hop, win)
    err = np.abs(wave.cpu().numpy() - ref)
    # per output hop block: the frames overlapping it bound its error
    inv_bound = C_FFT * np.log2(n_fft) * EPS * np.abs(ref).max() * 8
    assert err.max() <= inv_bound, (err.max(), inv_bound)
    # one iteration from `first`: the forward path on the kernel's own inverse
    F.griffinlim(shape, St, off, angles, rebuilt, True, 1)
    inverse = O.istft(S.astype(np.float64) * ang.astype(np.complex128), n_fft, hop, win)
    rb_ref = O.stft(inverse, n_fft, hop, win)
    rb = rebuilt.cpu().numpy().T
    e = np.linalg.norm(rb - rb_ref, axis=0)
    assert (e <= _frame_bound(rb_ref, n_fft)).all(), (e / _frame_bound(rb_ref, n_fft)).max()


def test_every_step_of_60_iterations_and_fused_equals_chain(mods):
    _lib, F, _ = mods
    n_fft, hop, win, Fr = 1102, 275, 1102, 24
    S = np.abs(O.stft(_signal(hop * (Fr - 1), 2), n_fft, hop, win)).astype(np.float32) ** 1.5
    u = np.random.default_rng(5).uniform(0, 1, S.shape)
    St, off = _pack([S], np.float32)
    shape = _shape(_lib, [Fr], n_fft, hop, win)
    a0 = _pack([O.angles_from_uniform(u)], np.complex64)[0]
    angles, rebuilt = a0.clone(), torch.zeros_like(a0)
    S64 = S.astype(np.float64)
    worst = [0.0, 0.0]
    for i in range(60):
        a_prev = angles.cpu().numpy().T.astype(np.complex128)
        t_prev = rebuilt.cpu().numpy().T.astype(np.complex128) if i else np.zeros_like(a_prev)
        F.griffinlim(shape, St, off, angles, rebuilt, i == 0, 1)
        rb_ref, upd_ref, _ = O.griffinlim_step(S64, a_prev, t_prev, n_fft, hop, win)
        rb = rebuilt.cpu().numpy().T
        bound = _frame_bound(rb_ref, n_fft)
        e = np.linalg.norm(rb - rb_ref, axis=0)
        assert (e <= bound).all(), (i, (e / bound).max())
        # The kernel does not store its unnormalised update, so the momentum arithmetic is checked through the normalised angles it
        # writes, against the fp64 update from the kernel's previous state.  Only where the update is well conditioned: its error is
        # the rebuilt error (<= bound) plus the rounding of the momentum term, and that moves the phase by at most 2 e / |update|.
        ang = angles.cpu().numpy().T
        mag = np.abs(upd_ref)
        ok = mag > 1e-3 * mag.max(axis=0, keepdims=True)
        ea = np.abs(ang - upd_ref / (mag + 1e-16))
        lim = 2 * bound[None, :] / np.maximum(mag, 1e-30) + 4 * EPS
        assert (ea[ok] <= lim[ok]).all(), (i, (ea[ok] / lim[ok]).max())
        worst = [max(worst[0], (e / bound).max()), max(worst[1], (ea[ok] / lim[ok]).max())]
    print(f'worst err/bound over 60 steps: rebuilt {worst[0]:.3f}, angles {worst[1]:.3f}')
    chained_wave = torch.empty(hop * (Fr - 1), device='cuda')
    F.griffinlim(shape, St, off, angles, rebuilt, False, 0, chained_wave)
    fa, fr = a0.clone(), torch.zeros_like(a0)
    fused_wave = torch.empty_like(chained_wave)
    F.griffinlim(shape, St, off, fa, fr, True, 60, fused_wave)
    assert torch.equal(fa, angles) and torch.equal(fr, rebuilt) and torch.equal(fused_wave, chained_wave)


def test_ragged_batch_equals_single_calls(mods):
    _lib, F, audio = mods
    lengths = [2, 3, 4, 5, 77, 900, 1201]
    rng = np.random.default_rng(7)
    frames = [lengths[i % len(lengths)] for i in range(64)][:24] + [1201, 900, 2, 3]
    specs = [(rng.standard_normal((80, f)) * 10 - 40).astype(np.float32) for f in frames]
    phases = [rng.uniform(0, 1, (552, f)) for f in frames]
    batch = audio.inverse_spectrogram_batch(specs, mel=True, phases=phases)
    hop = audio.ms_to_frames(12.5)
    for s, p, w, f in zip(specs, phases, batch, frames):
        assert isinstance(w, np.ndarray) and w.shape == (hop * (f - 1),)
        single = audio.inverse_spectrogram(s, mel=True, phases=p)
        assert np.array_equal(single, w), f
        assert np.isfinite(w).all() and w.max() == 1.0


@pytest.mark.parametrize('Fr', [2, 3, 4, 5])
def test_short_utterances_follow_repeated_reflection(mods, Fr):
    """hop * (F - 1) <= N / 2: np.pad reflects more than once; one iteration's forward transform sees exactly that padding."""
    _lib, F, _ = mods
    n_fft, hop, win = 1102, 275, 1102
    rng = np.random.default_rng(Fr)
    S = rng.uniform(0.1, 1, (552, Fr)).astype(np.float32)
    ang = O.angles_from_uniform(rng.uniform(0, 1, S.shape))
    St, off = _pack([S], np.float32)
    angles = _pack([ang], np.complex64)[0]
    rebuilt = torch.zeros_like(angles)
    F.griffinlim(_shape(_lib, [Fr], n_fft, hop, win), St, off, angles, rebuilt, True, 1)
    inverse = O.istft(S.astype(np.float64) * ang, n_fft, hop, win)
    ref = O.stft(inverse, n_fft, hop, win)
    e = np.linalg.norm(rebuilt.cpu().numpy().T - ref, axis=0)
    assert (e <= _frame_bound(ref, n_fft)).all(), (e / _frame_bound(ref, n_fft)).max()


def _kkt(A, B, X):
    G = A.T @ (A @ X - B)
    return G, np.abs(G * X).max(axis=0), np.maximum(-G, 0).max(axis=0)


def test_nnls_optimality(mods):
    _lib, F, audio = mods
    A = audio.mel_basis(22050, 1102, 80).astype(np.float64)
    rng = np.random.default_rng(11)
    real = A @ np.abs(O.stft(_signal(275 * 99, 3), 1102, 275, 1102))
    smooth = 10 ** (0.05 * (np.cumsum(rng.standard_normal((80, 100)), axis=0) * 3 - 40))    # model-like: smooth in frequency
    adversarial = 10 ** (-4 * rng.uniform(0, 1, (80, 100)))
    basis, pinv_t, step = audio.mel_tables(22050, 1102, 80, 'cuda')
    P = np.linalg.pinv(A)
    for name, Bm in (('real', real), ('model-like', smooth), ('adversarial', adversarial)):
        log_mel = (20 * np.log10(np.maximum(Bm, 1e-30))).astype(np.float32)      # db_to_amplitude inverts this
        t, _ = _pack([log_mel], np.float32)
        # no steps: librosa's start point clip(pinv(A) b, 0); each bin is an 80-term fp32 dot product of rounded operands
        shape0 = _shape(_lib, [Bm.shape[1]], 1102, 275, 1102, n_mels=80, power=1.0, nnls_iters=0)
        X0 = F.spectrogram_magnitude(shape0, t, basis, pinv_t, step).cpu().numpy().T.astype(np.float64)
        b0 = O.db_to_amplitude(log_mel.astype(np.float64))
        ref0 = np.maximum(P @ b0, 0)
        bound0 = 2 * (80 + 8) * EPS * (np.abs(P) @ np.abs(b0))
        assert (np.abs(X0 - ref0) <= bound0).all(), (name, (np.abs(X0 - ref0) / bound0).max())
        shape = _shape(_lib, [Bm.shape[1]], 1102, 275, 1102, n_mels=80, power=1.0, nnls_iters=audio.NNLS_ITERS)
        X = F.spectrogram_magnitude(shape, t, basis, pinv_t, step).cpu().numpy().T.astype(np.float64)
        b = O.db_to_amplitude(log_mel.astype(np.float64))
        assert (X >= 0).all()
        _, opt = O.nnls_optimum(A, b)
        gap = O.nnls_gap(A, b, X, opt)
        assert gap.max() <= audio.NNLS_GAP_BOUND, (name, gap.max())
        # KKT: no more violation than the fp32 oracle of the same algorithm shows, with 4x margin
        Xo = O.fista_nnls(A, b, audio.NNLS_ITERS, np.float32).astype(np.float64)
        _, comp, neg = _kkt(A, b, X)
        _, comp_o, neg_o = _kkt(A, b, Xo)
        # tau: the fp32 rounding floor of g_i x_i, 168 * 2^-24 (~1e-5) of |A^T b| |b| -- a gradient sums up to 2 x 44 products
        tau = 168 * EPS * np.abs(A.T @ b).max(axis=0) * np.abs(b).max(axis=0)
        # (worst over the set: the two fp32 solvers sum in different orders, so single frames trade places at the rounding floor)
        assert comp.max() <= 4 * comp_o.max() + tau.max() and neg.max() <= 4 * neg_o.max() + tau.max(), name
        print(f'{name}: worst gap {gap.max():.2e}')


def test_deemphasis_and_normalisation(mods):
    _lib, F, _ = mods
    rng = np.random.default_rng(13)
    hop, frames = 275, [2, 3, 77, 900, 5]
    waves = [rng.standard_normal(hop * (f - 1)).astype(np.float32) for f in frames]
    off = torch.from_numpy(np.concatenate([[0], np.cumsum(frames)]).astype(np.int32)).cuda()
    wave = torch.from_numpy(np.concatenate(waves)).cuda()
    for a in (0.97, 0.0):
        w = wave.clone()
        F.deemphasis_normalize(_shape(_lib, frames, 1102, hop, 1102, preemphasis=a), w, off)
        got, pos = w.cpu().numpy(), 0
        for x in waves:
            y = scipy.signal.lfilter([1], [1, -a], x.astype(np.float64)) if a else x.astype(np.float64)
            ref = y / max(y)
            g = got[pos:pos + len(x)]
            pos += len(x)
            bound = 64 * EPS / (1 - a) * np.abs(y).max() / max(y)
            assert np.abs(g - ref).max() <= bound, (len(x), a)
            assert g.max() == 1.0


def test_text_to_waveform(mods):
    _lib, F, audio = mods
    from multilingual_text_to_speech_b200 import configs
    from multilingual_text_to_speech_b200.modules.tacotron2 import Tacotron
    hp = configs.apply('ljspeech', max_output_length=120)
    hp.mel_normalize_mean, hp.mel_normalize_variance = -40.0, 15.0
    torch.manual_seed(0)
    model = Tacotron().cuda().eval()
    with torch.no_grad():
        model._decoder._stop_prediction.bias.fill_(-100.0)      # random weights never stop: every utterance runs to 120 frames
    rng = np.random.default_rng(0)
    texts = [torch.from_numpy(rng.integers(1, hp.symbols_count() + 1, size=L)).cuda() for L in (12, 30, 21)]
    with torch.no_grad():
        specs = model.inference_batch(texts)
    specs = [audio.denormalize_spectrogram(s, True) for s in specs]
    phases = [rng.uniform(0, 1, (552, s.shape[1])) for s in specs]
    waves = audio.inverse_spectrogram_batch(specs, mel=True, phases=phases)
    hop = audio.ms_to_frames(hp.stft_shift_ms)
    for s, w in zip(specs, waves):
        assert isinstance(w, torch.Tensor) and w.is_cuda and w.shape == (hop * (s.shape[1] - 1),)
        assert torch.isfinite(w).all() and float(w.max()) == 1.0
    # spectral convergence of the Griffin-Lim output against the fp64 oracle from the same phases and the same NNLS magnitudes
    s, u = specs[0], phases[0]
    Fr = s.shape[1]
    basis, pinv_t, step = audio.mel_tables(hp.sample_rate, hp.num_fft, hp.num_mels, 'cuda')
    shape = _shape(_lib, [Fr], 1102, hop, 1102, n_mels=80, power=1.5, nnls_iters=audio.NNLS_ITERS)
    S = F.spectrogram_magnitude(shape, s.t().contiguous().float(), basis, pinv_t, step)
    _, off = _pack([np.zeros((1, Fr))], np.float32)
    angles = _pack([O.angles_from_uniform(u)], np.complex64)[0]
    y = torch.empty(hop * (Fr - 1), device='cuda')
    F.griffinlim(shape, S, off, angles, torch.zeros_like(angles), True, 60, y)
    Sn = S.cpu().numpy().T.astype(np.float64)
    y = y.cpu().numpy().astype(np.float64)
    y64 = O.griffinlim(Sn, u, 60, 1102, hop, 1102, dtype=np.float64)
    y32 = O.griffinlim(Sn, u, 60, 1102, hop, 1102, dtype=np.float32)
    drift32 = np.linalg.norm(y32 - y64) / np.linalg.norm(y64)
    drift = np.linalg.norm(y - y64) / np.linalg.norm(y64)
    sc, sc64 = O.spectral_convergence(Sn, y, 1102, hop, 1102), O.spectral_convergence(Sn, y64, 1102, hop, 1102)
    print(f'text->wave: drift {drift:.2e} (fp32 oracle {drift32:.2e}), spectral convergence {sc:.4f} vs fp64 {sc64:.4f}')
    assert drift <= GL_DRIFT_FACTOR * drift32 + 1e-5
    assert sc <= sc64 * (1 + GL_DRIFT_FACTOR * drift32) + 1e-5


def test_harmonic_signal_spectral_convergence(mods):
    _lib, F, _ = mods
    n_fft, hop, win, Fr = 1102, 275, 1102, 200
    S = np.abs(O.stft(_signal(hop * (Fr - 1), 4), n_fft, hop, win))
    u = np.random.default_rng(17).uniform(0, 1, S.shape)
    St, off = _pack([S], np.float32)
    angles = _pack([O.angles_from_uniform(u)], np.complex64)[0]
    y = torch.empty(hop * (Fr - 1), device='cuda')
    F.griffinlim(_shape(_lib, [Fr], n_fft, hop, win), St, off, angles, torch.zeros_like(angles), True, 60, y)
    sc = O.spectral_convergence(S, y.cpu().numpy().astype(np.float64), n_fft, hop, win)
    sc64 = O.spectral_convergence(S, O.griffinlim(S, u, 60, n_fft, hop, win), n_fft, hop, win)
    print(f'harmonic: spectral convergence {sc:.4f} (fp64 oracle {sc64:.4f})')
    assert sc <= 1.05 * sc64 and sc < 0.15


def test_linear_magnitude_and_power(mods):
    """The linear path's magnitude kernel: (10^(0.1 s))^0.5 ** power against fp64, over the 120 dB a log spectrogram spans."""
    _lib, F, _ = mods
    s = np.random.default_rng(19).uniform(-100, 20, (300, 552)).astype(np.float32)
    for power in (1.5, 1.0):
        S = F.spectrogram_magnitude(_shape(_lib, [300], 1102, 275, 1102, power=power), torch.from_numpy(s).cuda()).cpu().numpy()
        ref = np.power(np.power(10.0, 0.1 * s.astype(np.float64)), 0.5) ** power
        # 0.1 s rounds to 2^-24 |0.1 s| in the exponent: relative ln(10) |0.1 s| 2^-24 in 10^x, scaled by 0.5 * power; a few ulps besides
        bound = EPS * (8 + np.log(10) * np.abs(0.1 * s.astype(np.float64)) * 0.5 * power * 2)
        rel = np.abs(S - ref) / ref
        assert (rel <= bound).all(), (power, (rel / bound).max())


@pytest.mark.parametrize('mel', [False, True])
def test_inverse_spectrogram_batch_matches_reference_composition(mods, mel):
    """The public function under hp (ljspeech: power 1.5, 60 iterations, de-emphasis 0.97, y / max(y)) against the oracle's composition
    of the reference's inverse_spectrogram in fp64, from the same phases and with the same NNLS routine; hop and win come from hp by the
    reference's formula.  Bound: GL_DRIFT_FACTOR times the fp32 oracle's drift from the fp64 one on the same input."""
    _lib, F, audio = mods
    from multilingual_text_to_speech_b200.params.params import Params as hp
    assert (hp.griffin_lim_power, hp.griffin_lim_iters, hp.use_preemphasis, hp.preemphasis) == (1.5, 60, True, 0.97)
    n_fft = hp.num_fft
    hop, win = int(hp.sample_rate * hp.stft_shift_ms / 1000), int(hp.sample_rate * hp.stft_window_ms / 1000)
    A = audio.mel_basis(hp.sample_rate, n_fft, hp.num_mels).astype(np.float64)
    rng = np.random.default_rng(23 + mel)
    frames = [3, 41, 120]
    specs, phases = [], []
    for i, f in enumerate(frames):
        mag = np.abs(O.stft(_signal(hop * (f - 1), 30 + i, f0=110.0 + 40 * i), n_fft, hop, win))
        if mel:
            mag = A @ mag
        specs.append((20 * np.log10(mag + 1e-5)).astype(np.float32))
        phases.append(rng.uniform(0, 1, (n_fft // 2 + 1, f)))
    waves = audio.inverse_spectrogram_batch(specs, mel=mel, phases=phases)
    for s, u, w, f in zip(specs, phases, waves, frames):
        assert w.shape == (hop * (f - 1),) and w.max() == 1.0
        args = (s, u, n_fft, hop, win, hp.griffin_lim_iters, hp.griffin_lim_power, hp.preemphasis, A if mel else None, audio.NNLS_ITERS)
        y64 = O.inverse_spectrogram(*args, dtype=np.float64)
        y32 = O.inverse_spectrogram(*args, dtype=np.float32)
        drift32 = np.linalg.norm(y32 - y64) / np.linalg.norm(y64)
        err = np.linalg.norm(w.astype(np.float64) - y64) / np.linalg.norm(y64)
        print(f'mel={mel} F={f}: error {err:.2e}, fp32 oracle drift {drift32:.2e}')
        assert err <= GL_DRIFT_FACTOR * drift32 + 1e-6, (f, err, drift32)
