"""Audio analysis on the H100 against the numpy oracle (tests/analysis_oracle.py): the fp64 STFT magnitude (linear and mel) with a bound per
element, the dB step, the cepstrum, the three MCD modes, ragged-batch invariance and an evaluation-shaped run through inference_batch."""
import numpy as np
import pytest
import torch

import analysis_oracle as AO

pytestmark = pytest.mark.gpu

EPS = 2.0 ** -24
DB = 20 / np.log(10)            # d(20 log10 x) / (dx / x)
WORST = {}                      # worst err / bound per check, printed at the end of the module


def _worst(name, ratio):
    WORST[name] = max(WORST.get(name, 0.0), float(ratio))


@pytest.fixture(scope='module')
def mods():
    import __graft_entry__ as entry
    entry.build()
    from multilingual_text_to_speech_b200 import _lib, configs
    from multilingual_text_to_speech_b200 import functional as F
    from multilingual_text_to_speech_b200.utils import audio
    configs.apply('ljspeech')
    _lib.set_precision('fp32')
    yield _lib, F, audio
    print('worst err/bound:', {k: round(v, 3) for k, v in sorted(WORST.items())})


def _signal(n, seed, f0=140.0):
    """Harmonics falling 80 dB over 24 partials plus noise 120 dB down: the spectrum spans more than 80 dB."""
    rng = np.random.default_rng(seed)
    t = np.arange(n) / 22050
    y = sum(10 ** (-k / 6) * np.sin(2 * np.pi * f0 * (k + 1) * t * (1 + 0.05 * t) + rng.uniform(0, 6)) for k in range(24))
    return (0.5 * y + 1e-6 * rng.standard_normal(n)).astype(np.float32)


def _run_stft(_lib, F, waves, n_fft, hop, win, A=None, preemph=0.0):
    lengths = [len(w) for w in waves]
    frames = [1 + n // hop for n in lengths]
    soff = torch.from_numpy(np.concatenate([[0], np.cumsum(lengths)]).astype(np.int32)).cuda()
    off_h = np.concatenate([[0], np.cumsum(frames)]).astype(np.int64)
    off = torch.from_numpy(off_h.astype(np.int32)).cuda()
    shape = _lib.AnalysisShape(len(waves), sum(lengths), sum(frames), n_fft, hop, win, 0 if A is None else A.shape[0], preemph)
    wave = torch.from_numpy(np.concatenate(waves).astype(np.float32)).cuda()
    basis = None if A is None else torch.from_numpy(A).cuda()
    out = F.stft_magnitude(shape, wave, soff, off, basis)
    return shape, out, off, [out[off_h[i]:off_h[i + 1]].cpu().numpy().T for i in range(len(waves))]


def _mag_bound(X64, norms):
    """|fp32 magnitude - |X||: the complex64 rounding (2^-24 |X|), hypotf (3 ulp <= 6 * 2^-24 |X|) and the fp64 transform's error (far
    below 2^-40 of the frame norm for N <= 2048)."""
    return 8 * EPS * X64 + 2.0 ** -40 * norms[None, :] + 1e-38


def _mel_bound(A, X64, kb):
    """sum_k A_mk (magnitude bound_k) plus an fp32 sum of n_m products: (n_m + 1) 2^-24 sum_k A_mk |X_k|."""
    nm = (A != 0).sum(1)[:, None]
    return A.astype(np.float64) @ kb + (nm + 1) * EPS * (A.astype(np.float64) @ X64) + 1e-38


# the default plan [19, 29], [4, 4, 4, 4, 2] with and without a zero-padded window, then the other plans a user's hp.num_fft can give:
# [4, 4, 5, 5] (16 kHz), [2, 5, 5, 11], [3, 7, 13] (N - win odd), [23, 31], [31, 31] and [4, 4, 4, 4, 4]
@pytest.mark.parametrize('n_fft,hop,win', [(1102, 275, 1102), (1024, 256, 1024), (1024, 256, 800), (800, 200, 800), (1100, 275, 1100),
                                           (546, 136, 545), (1426, 356, 1426), (1922, 480, 1922), (2048, 512, 2048)])
def test_stft_magnitude_against_fp64(mods, n_fft, hop, win):
    _lib, F, audio = mods
    lengths = [1, 2, 3, n_fft // 2 - 1, n_fft // 2, n_fft // 2 + 1, hop * 40, hop * 41 + 17]
    waves = [_signal(L, 100 + i) for i, L in enumerate(lengths)]
    A = audio.mel_basis(22050, n_fft, 80)
    for preemph in (0.97, 0.0):
        _, _, _, lin = _run_stft(_lib, F, waves, n_fft, hop, win, preemph=preemph)
        _, _, _, mel = _run_stft(_lib, F, waves, n_fft, hop, win, A=A, preemph=preemph)
        for w, g, gm in zip(waves, lin, mel):
            X64, norms = AO.magnitude64(w, n_fft, hop, win, preemph)
            assert g.shape == X64.shape == (n_fft // 2 + 1, 1 + len(w) // hop)
            kb = _mag_bound(X64, norms)
            r = np.abs(g - X64) / kb
            assert (r <= 1).all(), (len(w), preemph, r.max())
            _worst('stft linear', r.max())
            mb = _mel_bound(A, X64, kb)
            rm = np.abs(gm - A.astype(np.float64) @ X64) / mb
            assert (rm <= 1).all(), (len(w), preemph, rm.max())
            _worst('stft mel', rm.max())
    # the bound means something: a single-precision transform of the same input breaks it
    w = waves[-1]
    X64, norms = AO.magnitude64(w, n_fft, hop, win, 0.97)
    X32 = AO.magnitude(w, n_fft, hop, win, 0.97, fp32_fft=True).astype(np.float64)
    assert (np.abs(X32 - X64) / _mag_bound(X64, norms)).max() > 10


def test_amplitude_to_db_from_the_kernels_magnitudes(mods):
    """The dB step recomputed in float32 by the oracle from the kernel's own magnitudes.  Each term 10 log10(.) carries log10f's 2 ulp
    and the multiply's rounding: 4 ulp of each term and one of the difference."""
    _lib, F, audio = mods
    waves = [_signal(L, 7 + L) for L in (3, 2000, 22050)]
    waves[1][:600] = 0.0                                            # exact zeros: the amin floor
    A = audio.mel_basis(22050, 1102, 80)
    for mel in (False, True):
        shape, S, off, per = _run_stft(_lib, F, waves, 1102, 275, 1102, A=A if mel else None, preemph=0.97)
        db = F.amplitude_to_db(shape, S, off)
        off_h = off.cpu().numpy()
        for i, s in enumerate(per):
            got = db[off_h[i]:off_h[i + 1]].cpu().numpy().T
            ref = AO.amplitude_to_db(s)
            a = 10 * np.log10(np.maximum(1e-10, s.astype(np.float64) ** 2))
            r = 10 * np.log10(max(1e-10, float(np.abs(s).max()) ** 2))
            bound = 8 * EPS * (np.abs(a) + abs(r)) + 2 * EPS * np.abs(ref)
            assert (np.abs(got - ref) <= bound).all(), (mel, i, (np.abs(got - ref) / bound).max())
            _worst('amplitude_to_db', (np.abs(got - ref) / bound).max())
            assert got.max() == 0.0
        inplace = S.clone()
        F.amplitude_to_db(shape, inplace, off, out=inplace)
        assert torch.equal(inplace, db)


def test_ragged_batch_is_bitwise_its_single_calls(mods):
    _lib, F, audio = mods
    lengths = [1, 2, 3, 551, 552, 275 * 80 + 13, 22050 * 3, 1000]
    waves = [_signal(L, 200 + i) for i, L in enumerate(lengths)]
    for mel in (False, True):
        batch = audio.spectrogram_batch(waves, mel=mel)
        for w, b in zip(waves, batch):
            assert isinstance(b, np.ndarray) and b.shape == ((80 if mel else 552), 1 + len(w) // 275)
            assert np.array_equal(audio.spectrogram(w, mel), b)
        # torch in -> torch out on the input's device
        tb = audio.spectrogram_batch([torch.from_numpy(w).cuda() for w in waves[:3]] + [torch.from_numpy(waves[3])], mel=mel)
        assert tb[0].is_cuda and not tb[3].is_cuda
        assert all(np.array_equal(t.cpu().numpy(), b) for t, b in zip(tb, batch))


@pytest.mark.parametrize('mel', [False, True])
def test_spectrogram_batch_end_to_end_under_hp(mods, mel):
    """spectrogram_batch / mel_spectrogram under hp ljspeech against the oracle's fp64 composition.  The dB error of an element follows from
    its magnitude bound (relative, times 20 / ln 10), the same for the utterance's maximum, and the float32 log arithmetic."""
    _lib, F, audio = mods
    from multilingual_text_to_speech_b200.params.params import Params as hp
    n_fft = hp.num_fft
    hop, win = int(hp.sample_rate * hp.stft_shift_ms / 1000), int(hp.sample_rate * hp.stft_window_ms / 1000)
    A = audio.mel_basis(hp.sample_rate, n_fft, hp.num_mels)
    waves = [_signal(L, 300 + L) for L in (2, 551, 22050 * 2 + 5)]
    got = audio.spectrogram_batch(waves, mel=mel)
    assert np.array_equal(got[2], audio.mel_spectrogram(waves[2]) if mel else audio.spectrogram(waves[2]))
    for w, g in zip(waves, got):
        X64, norms = AO.magnitude64(w, n_fft, hop, win, hp.preemphasis)
        kb = _mag_bound(X64, norms)
        if mel:
            kb, X64 = _mel_bound(A, X64, kb), A.astype(np.float64) @ X64
        ref = 20 * np.log10(np.maximum(1e-5, X64)) - 20 * np.log10(max(1e-5, X64.max()))
        rel = np.where(X64 > 1e-5, kb / np.maximum(X64 - kb, 1e-300), np.where(X64 + kb > 1e-5, np.inf, 0))
        ref_rel = kb.flat[np.argmax(X64)] / X64.max()
        # (2 DB 2^-24: the fp32 squares of the element and of the maximum)
        bound = DB * (rel + ref_rel) + 8 * EPS * (np.abs(ref) + 2 * abs(20 * np.log10(X64.max()))) + 2 * DB * EPS
        r = np.abs(g - ref) / bound
        assert (r <= 1).all(), (len(w), r.max())
        _worst(f'spectrogram_batch mel={mel}', r.max())


def test_cepstrum_against_fp64(mods):
    """The kernel's cepstra against the fp64 DCT of the same dB input: the matrix rounding, the /10 rounding and an fp32 sum of n_mels
    products give (n_mels + 3) 2^-24 sum_n |D_kn x_n / 10| per coefficient."""
    _lib, F, audio = mods
    rng = np.random.default_rng(5)
    mel_db = np.minimum(rng.normal(-40, 20, (1000, 80)), 0).astype(np.float32)
    got = F.mel_cepstrum(torch.from_numpy(mel_db).cuda(), 13).cpu().numpy()
    D = AO.dct_matrix(80, 13)
    x = mel_db.astype(np.float64).T / 10
    ref = (D @ x).T
    bound = ((80 + 3) * EPS * (np.abs(D) @ np.abs(x))).T
    r = np.abs(got - ref) / bound
    assert (r <= 1).all(), r.max()
    _worst('cepstrum', r.max())
    # the public wrapper: [n_mfcc, F] in the input's container
    c = audio.get_spectrogram_mfcc(mel_db.T)
    assert isinstance(c, np.ndarray) and c.shape == (13, 1000) and np.array_equal(c, got.T)
    # librosa's own arithmetic (scipy.fftpack in single precision) is within the same bound
    assert (np.abs(AO.mfcc(mel_db.T, 13).T - ref) <= bound).all()


def _cepstra_pairs(rng, sizes, n_mfcc=13):
    return [(rng.normal(0, 3, (fa, n_mfcc)).astype(np.float32), rng.normal(0, 3, (fb, n_mfcc)).astype(np.float32)) for fa, fb in sizes]


def _mcd_direct(F, pairs, mode):
    ca = torch.from_numpy(np.concatenate([a for a, _ in pairs])).cuda()
    cb = torch.from_numpy(np.concatenate([b for _, b in pairs])).cuda()
    oa = torch.from_numpy(np.concatenate([[0], np.cumsum([len(a) for a, _ in pairs])]).astype(np.int32)).cuda()
    ob = torch.from_numpy(np.concatenate([[0], np.cumsum([len(b) for _, b in pairs])]).astype(np.int32)).cuda()
    mcd, plen = F.mel_cepstral_distortion(ca, oa, cb, ob, mode)
    return mcd.cpu().numpy(), plen.cpu().numpy()


def test_dtw_bitwise_against_the_mirror_and_fp64(mods):
    """(cost / length, path length) bit for bit against the numpy mirror (fp32 distances in the kernel's order, fp64 accumulation) on the
    same cepstra; against all-fp64 within (C + 4) 2^-24 of the value where the fp64 path is the same (random inputs have no near-ties)."""
    _lib, F, _ = mods
    rng = np.random.default_rng(9)
    sizes = [(1, 1), (1, 40), (40, 1), (2, 3), (37, 50), (120, 97), (300, 333), (5, 5)]
    pairs = _cepstra_pairs(rng, sizes)
    mcd, plen = _mcd_direct(F, pairs, 'dtw')
    for (a, b), m, n in zip(pairs, mcd, plen):
        mm, nn = AO.mcd_from_cepstra(a.T, b.T, 'dtw')
        assert m == mm and n == nn, (a.shape, b.shape, m, mm, n, nn)
        m64, n64 = AO.mcd_from_cepstra(a.T, b.T, 'dtw', np.float64)
        assert n64 == n
        bound = (12 + 4) * EPS * m64 + 1e-300
        assert abs(m - m64) <= bound, (abs(m - m64) / bound)
        _worst('dtw vs fp64', abs(m - m64) / bound)
    # 1 x F and F x 1: the only path runs along the long side
    assert plen[1] == 40 and plen[2] == 40


def test_dtw_at_the_shared_memory_cap_and_over_it(mods):
    _lib, F, audio = mods
    cap = _lib.DTW_MAX_FRAMES
    rng = np.random.default_rng(11)
    a = rng.normal(0, 3, (cap, 13)).astype(np.float32)
    b = np.concatenate([a, a[-1:]])                                 # the diagonal, then one step along b: cost 0, cap + 1 cells
    mcd, plen = _mcd_direct(F, [(a, a), (a, b), (b, a)], 'dtw')
    assert list(mcd) == [0.0, 0.0, 0.0] and list(plen) == [cap, cap + 1, cap + 1]
    over = np.concatenate([b, b[-1:]])
    mcd, plen = _mcd_direct(F, [(b, over), (a[:3], a[:4])], 'dtw')
    assert np.isnan(mcd[0]) and plen[0] == -1 and plen[1] == 4      # the C ABI marks the pair; the others are computed
    S = rng.normal(-40, 10, (80, cap + 1)).astype(np.float32)
    with pytest.raises(ValueError, match='at most'):
        audio.mel_cepstral_distortion_batch([S], [S], 'dtw')


@pytest.mark.parametrize('mode', ['cut', 'stretch'])
def test_cut_and_stretch_against_fp64(mods, mode):
    _lib, F, _ = mods
    rng = np.random.default_rng(13)
    sizes = [(1, 1), (1, 9), (9, 1), (50, 50), (77, 300), (300, 77), (1000, 999)]
    pairs = _cepstra_pairs(rng, sizes)
    mcd, plen = _mcd_direct(F, pairs, mode)
    for (a, b), m, n in zip(pairs, mcd, plen):
        m64, n64 = AO.mcd_from_cepstra(a.T, b.T, mode, np.float64)
        assert n == n64
        bound = (12 + 4) * EPS * m64 + n * 1e-16 * m64
        assert abs(m - m64) <= bound, (a.shape, b.shape, abs(m - m64) / bound)
        _worst(mode, abs(m - m64) / bound)


def test_batch_of_pairs_is_bitwise_its_single_calls(mods):
    _lib, F, audio = mods
    rng = np.random.default_rng(15)
    S1 = [rng.normal(-40, 15, (80, f)).astype(np.float32) for f in (1, 7, 200, 333)]
    S2 = [rng.normal(-40, 15, (80, f)).astype(np.float32) for f in (5, 7, 180, 350)]
    for mode in ('dtw', 'cut', 'stretch'):
        batch = audio.mel_cepstral_distortion_batch(S1, S2, mode)
        assert isinstance(batch, np.ndarray) and batch.dtype == np.float64 and batch.shape == (4,)
        for i in range(4):
            assert audio.mel_cepstral_distorision(S1[i], S2[i], mode) == batch[i]
        assert audio.mel_cepstral_distorision(S1[2], S1[2], mode) == 0.0
    t = audio.mel_cepstral_distortion_batch([torch.from_numpy(s).cuda() for s in S1], S2, 'dtw')
    assert isinstance(t, torch.Tensor) and t.is_cuda and t.dtype == torch.float64
    assert np.array_equal(t.cpu().numpy(), audio.mel_cepstral_distortion_batch(S1, S2, 'dtw'))


def test_evaluation_shaped_run(mods):
    """train.py's evaluate: MCD of inference_batch outputs against targets of other lengths, through mel_cepstral_distortion_batch, against
    the mirror on the library's own cepstra (bitwise) and the fp64 oracle from the spectrograms (within its bound)."""
    _lib, F, audio = mods
    from multilingual_text_to_speech_b200 import configs
    from multilingual_text_to_speech_b200.modules.tacotron2 import Tacotron
    hp = configs.apply('ljspeech', max_output_length=90)
    hp.mel_normalize_mean, hp.mel_normalize_variance = -40.0, 15.0
    torch.manual_seed(0)
    model = Tacotron().cuda().eval()
    with torch.no_grad():
        model._decoder._stop_prediction.bias.fill_(-100.0)
    rng = np.random.default_rng(0)
    texts = [torch.from_numpy(rng.integers(1, hp.symbols_count() + 1, size=L)).cuda() for L in (12, 30, 21)]
    with torch.no_grad():
        gen = [audio.denormalize_spectrogram(s, True) for s in model.inference_batch(texts)]
    targets = audio.spectrogram_batch([_signal(275 * f, 400 + f) for f in (70, 95, 60)], mel=True)
    for mode in ('dtw', 'cut', 'stretch'):
        mcd = audio.mel_cepstral_distortion_batch(gen, targets, mode)
        assert isinstance(mcd, torch.Tensor) and mcd.is_cuda
        mcd = mcd.cpu().numpy()
        for g, t, m in zip(gen, targets, mcd):
            ca = audio.get_spectrogram_mfcc(g).cpu().numpy()
            cb = audio.get_spectrogram_mfcc(t)
            mm, _ = AO.mcd_from_cepstra(ca, cb, mode)
            assert m == mm, (mode, m, mm)
            # fp64 from the spectrograms: the cepstrum bound carried through the distance, plus the distance arithmetic
            D = AO.dct_matrix(80, 13)
            ga, ta = g.cpu().numpy().astype(np.float64), t.astype(np.float64)
            c64a, c64b = D @ (ga / 10), D @ (ta / 10)
            m64, _ = AO.mcd_from_cepstra(c64a, c64b, mode, np.float64)
            cb_a = (80 + 3) * EPS * (np.abs(D) @ np.abs(ga / 10))[1:]
            cb_b = (80 + 3) * EPS * (np.abs(D) @ np.abs(ta / 10))[1:]
            bound = np.sqrt((cb_a.max(1) ** 2).sum()) + np.sqrt((cb_b.max(1) ** 2).sum()) + 16 * EPS * m64
            assert abs(m - m64) <= bound, (mode, abs(m - m64) / bound)
            _worst(f'evaluation {mode}', abs(m - m64) / bound)
