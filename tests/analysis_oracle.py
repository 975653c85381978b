"""numpy restatement of the reference's audio analysis (utils/audio.py:66-78, 117-161 with librosa 0.7.0), the yardstick of the analysis tests.

librosa and fastdtw cannot be installed here, so each piece is written with the calls they make and tests/test_audio_analysis_cpu.py pins it
to an independent computation.  The dtypes follow librosa 0.7.0: an fp64 FFT of the fp64 (pre-emphasised) signal rounded to complex64, abs
in float32, the mel dot in float32, power_to_db in float32, and scipy.fftpack's single-precision DCT of float32 input.  `fp32_fft=True`
runs the transform in single precision instead, to show the bounds of the GPU tests are tight enough to tell the two apart."""
import numpy as np
import scipy.fft
import scipy.fftpack
import scipy.signal

import audio_oracle as AO


def preemphasis(y, a):
    """scipy.signal.lfilter([1, -a], [1], y) in fp64."""
    return scipy.signal.lfilter([1, -a], [1], np.asarray(y, dtype=np.float64))


def stft_complex(y, n_fft, hop, win, preemph=0.0, fp32_fft=False):
    """librosa.stft(preemphasis(y), center=True, pad_mode='reflect', window='hann') -> complex64 [K, 1 + len(y) // hop]."""
    y = np.asarray(y, dtype=np.float64)
    if preemph:
        y = preemphasis(y, preemph)
    if fp32_fft:
        return AO.stft(y, n_fft, hop, win, dtype=np.float32)
    return AO.stft(y, n_fft, hop, win).astype(np.complex64)


def magnitude(y, n_fft, hop, win, preemph=0.0, fp32_fft=False):
    """np.abs of the complex64 STFT (float32)."""
    return np.abs(stft_complex(y, n_fft, hop, win, preemph, fp32_fft))


def magnitude64(y, n_fft, hop, win, preemph=0.0):
    """|STFT| in fp64 without the complex64 rounding, and the fp64 frame norms of the windowed frames: the centre of the GPU bounds."""
    y = np.asarray(y, dtype=np.float64)
    if preemph:
        y = preemphasis(y, preemph)
    X = AO.stft(y, n_fft, hop, win)
    return np.abs(X), np.sqrt((np.abs(X) ** 2).sum(0) * 2 / n_fft)


def mel_project(A, S):
    """np.dot(mel_basis, S) in float32 (librosa.feature.melspectrogram(S=S))."""
    return np.dot(np.asarray(A, np.float32), np.asarray(S, np.float32))


def amplitude_to_db(S):
    """librosa.amplitude_to_db(S, ref=np.max, amin=1e-5, top_db=None) in float32: power_to_db(S^2, ref=max(S)^2, amin=1e-10)."""
    mag = np.abs(np.asarray(S, np.float32))
    ref = np.max(mag)
    power = np.square(mag)
    log_spec = np.float32(10.0) * np.log10(np.maximum(np.float32(1e-10), power))
    log_spec -= np.float32(10.0) * np.log10(np.maximum(np.float32(1e-10), np.square(ref)))
    return log_spec.astype(np.float32)


def spectrogram(y, n_fft, hop, win, preemph=0.0, A=None, fp32_fft=False):
    """The reference's spectrogram(y, mel=A is not None)."""
    S = magnitude(y, n_fft, hop, win, preemph, fp32_fft)
    if A is not None:
        S = mel_project(A, S)
    return amplitude_to_db(S)


def dct_matrix(n_mels, n_mfcc):
    """DCT-II with norm='ortho' as an fp64 matrix [n_mfcc, n_mels]."""
    k = np.arange(n_mfcc)[:, None]
    n = np.arange(n_mels)[None, :]
    D = np.cos(np.pi * k * (2 * n + 1) / (2 * n_mels))
    D *= np.where(k == 0, np.sqrt(1.0 / n_mels), np.sqrt(2.0 / n_mels))
    return D


def mfcc(S, n_mfcc):
    """librosa 0.7.0 mfcc(S=S/10, n_mfcc): scipy.fftpack.dct(S / 10, type=2, norm='ortho', axis=0)[:n_mfcc] (single precision for float32)."""
    S = np.asarray(S, np.float32)
    return scipy.fftpack.dct(S / np.float32(10), type=2, norm='ortho', axis=0)[:n_mfcc]


def frame_distances(x, y):
    """The library's frame distance of every pair: x [Fa, C], y [Fb, C] float32 (coefficients 1.. already selected) -> float32 [Fa, Fb],
    squares summed in index order with one rounding per operation, then a correctly rounded sqrt."""
    x = np.asarray(x, np.float32)
    y = np.asarray(y, np.float32)
    acc = np.zeros((x.shape[0], y.shape[0]), np.float32)
    for c in range(x.shape[1]):
        d = x[:, c][:, None] - y[:, c][None, :]
        acc = acc + d * d
    return np.sqrt(acc)


def dtw(dist):
    """Exact DTW over a distance matrix [Fa, Fb] with fastdtw.dtw's recurrence: D[0,0] = 0, borders infinite, predecessor the first minimum
    of the sums over (i-1, j), (i, j-1), (i-1, j-1); costs in fp64.  -> (cost, path length)."""
    Fa, Fb = dist.shape
    D = np.full((Fa + 1, Fb + 1), np.inf)
    Ln = np.zeros((Fa + 1, Fb + 1), np.int64)
    D[0, 0] = 0.0
    d64 = np.asarray(dist, np.float64)
    for s in range(2, Fa + Fb + 1):
        i = np.arange(max(1, s - Fb), min(Fa, s - 1) + 1)
        j = s - i
        dd = d64[i - 1, j - 1]
        best, bl = D[i - 1, j] + dd, Ln[i - 1, j].copy()
        cl = D[i, j - 1] + dd
        m = cl < best
        best[m], bl[m] = cl[m], Ln[i, j - 1][m]
        cd = D[i - 1, j - 1] + dd
        m = cd < best
        best[m], bl[m] = cd[m], Ln[i - 1, j - 1][m]
        D[i, j], Ln[i, j] = best, bl + 1
    return D[Fa, Fb], int(Ln[Fa, Fb])


def mcd_pairs(n_a, n_b, mode):
    """Frame index pairs of 'cut' and 'stretch': a literal restatement of the reference's utils/audio.py:143-153."""
    if mode == 'cut':
        n = min(n_a, n_b)
        return list(range(n)), list(range(n))
    if n_a > n_b:
        m = n_a
        return list(range(m)), [i * n_b // m for i in range(m)]
    m = n_b
    return [i * n_a // m for i in range(m)], list(range(m))


def mcd_from_cepstra(ca, cb, mode, dtype=np.float32):
    """MCD of cepstra [n_mfcc, F] (c0 dropped here) -> (value, pairs averaged over).  dtype float32: the library's distances (bit for bit)
    with fp64 accumulation; float64: every step in fp64."""
    x, y = np.asarray(ca)[1:].T.astype(dtype), np.asarray(cb)[1:].T.astype(dtype)
    if dtype == np.float32:
        dist = frame_distances(x, y).astype(np.float64)
    else:
        dist = np.sqrt(((x[:, None, :] - y[None, :, :]) ** 2).sum(-1))
    if mode == 'dtw':
        cost, n = dtw(dist)
        return cost / n, n
    ia, ib = mcd_pairs(x.shape[0], y.shape[0], mode)
    return float(np.mean(dist[ia, ib])), len(ia)
