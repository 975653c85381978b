"""CPU checks of the audio analysis: the numpy oracle (tests/analysis_oracle.py) pinned to independent computations, host validation and the
workspace formula, the no-GPU failure mode, the Python input checks and the register report of csrc/analysis.cu."""
import ctypes
import itertools
import os
import re
import shutil
import subprocess

import numpy as np
import pytest
import scipy.fftpack
import scipy.signal
import torch

import __graft_entry__ as entry
import analysis_oracle as AO
from multilingual_text_to_speech_b200 import _lib, build
from multilingual_text_to_speech_b200.utils import audio

N, HOP, WIN = 1102, 275, 1102


@pytest.fixture(scope='module')
def lib():
    entry.build()
    return _lib.load()


def test_oracle_preemphasis_is_the_difference_equation():
    x = np.random.default_rng(0).standard_normal(1000)
    y = AO.preemphasis(x, 0.97)
    ref = x.copy()
    ref[1:] = x[1:] - 0.97 * x[:-1]
    assert np.array_equal(y, ref)
    assert np.array_equal(y, scipy.signal.lfilter([1, -0.97], [1], x))


@pytest.mark.parametrize('L', [1, 2, 3, N // 2 - 1, N // 2, N // 2 + 1, 40 * HOP, 40 * HOP + 123])
def test_frame_count_and_reflect_padding(L):
    """1 + L // hop frames, and the kernel's index map (reflect_index in fft.cuh, restated) equals np.pad(mode='reflect')."""
    y = np.arange(L, dtype=np.float64) + 1
    X = AO.stft_complex(y, N, HOP, WIN)
    assert X.shape == (N // 2 + 1, 1 + L // HOP)
    pad = N // 2
    ref = np.pad(y, pad, mode='reflect')
    idx = np.arange(L + 2 * pad) - pad
    if L == 1:
        s = np.zeros_like(idx)
    else:
        s = np.mod(idx, 2 * (L - 1))
        s = np.where(s >= L, 2 * (L - 1) - s, s)
    assert np.array_equal(y[s], ref)
    # the last frame starts inside the padded signal and ends inside it
    assert (X.shape[1] - 1) * HOP + N <= L + 2 * pad


def test_amplitude_to_db_closed_form():
    rng = np.random.default_rng(1)
    S = (10 ** rng.uniform(-7, 1, (552, 30))).astype(np.float32)
    S[5, 3] = 0.0
    db = AO.amplitude_to_db(S)
    ref = 20 * np.log10(np.maximum(S.astype(np.float64), 1e-5)) - 20 * np.log10(S.max())
    assert db.dtype == np.float32
    assert np.abs(db - ref).max() < 1e-4
    assert db.max() == 0.0 and db[5, 3] == pytest.approx(-100 - 20 * np.log10(S.max()), abs=1e-4)
    # the reference is the utterance's own maximum: scaling the utterance changes nothing above the floor
    assert np.abs(AO.amplitude_to_db(S * np.float32(4)) - db)[S > 1e-5].max() < 1e-4


def test_dct_matrix_is_scipy_orthonormal_dct2():
    D = AO.dct_matrix(80, 13)
    ref = scipy.fftpack.dct(np.eye(80), type=2, norm='ortho', axis=0)[:13]
    assert np.abs(D - ref).max() < 1e-14
    assert np.abs(D @ D.T - np.eye(13)).max() < 1e-14
    x = np.random.default_rng(2).normal(-40, 10, (80, 7)).astype(np.float32)
    assert np.abs(AO.mfcc(x, 13) - D @ (x.astype(np.float64) / 10)).max() < 1e-4


def _brute_force_dtw(dist):
    """Minimum cost over every monotone path from (0, 0) to (Fa-1, Fb-1) with steps (1, 0), (0, 1), (1, 1)."""
    Fa, Fb = dist.shape
    best = [np.inf, None]

    def walk(i, j, cost, n):
        cost += dist[i, j]
        n += 1
        if i == Fa - 1 and j == Fb - 1:
            if cost < best[0]:
                best[:] = [cost, n]
            return
        if i + 1 < Fa:
            walk(i + 1, j, cost, n)
        if j + 1 < Fb:
            walk(i, j + 1, cost, n)
        if i + 1 < Fa and j + 1 < Fb:
            walk(i + 1, j + 1, cost, n)
    walk(0, 0, 0.0, 0)
    return best[0]


def test_exact_dtw_equals_brute_force():
    rng = np.random.default_rng(3)
    for Fa, Fb in itertools.product(range(1, 6), range(1, 7)):
        dist = rng.uniform(0, 1, (Fa, Fb))
        cost, n = AO.dtw(dist)
        assert abs(cost - _brute_force_dtw(dist)) < 1e-12, (Fa, Fb)
        assert max(Fa, Fb) <= n <= Fa + Fb - 1


def test_dtw_tie_order_and_path_length():
    """Ties take the first minimum among (i-1, j), (i, j-1), (i-1, j-1), as fastdtw's min(..., key=cost) does."""
    # all distances 0: every cell ties; the first candidate (i-1, j) is taken wherever it is finite, so the path runs along the first
    # row and then down the last column: Fa + Fb - 1 cells
    cost, n = AO.dtw(np.zeros((3, 4)))
    assert cost == 0.0 and n == 3 + 4 - 1
    # equal cost through (i-1, j) and (i-1, j-1): the up move wins and lengthens the path
    d = np.array([[0.0, 1.0], [1.0, 0.0]])
    d2 = np.array([[0.0, 0.0], [0.0, 0.0]])
    assert AO.dtw(d) == (0.0, 2)                                    # the diagonal is strictly cheapest
    assert AO.dtw(d2) == (0.0, 3)
    # (i, j-1) beats (i-1, j-1) on a tie: 1 x 3 has a single path
    assert AO.dtw(np.array([[1.0, 1.0, 1.0]])) == (3.0, 3)


def test_cut_and_stretch_pairs_restate_the_reference():
    rng = np.random.default_rng(4)
    for na, nb in [(5, 5), (3, 7), (7, 3), (1, 4), (4, 1), (10, 9)]:
        x = rng.standard_normal((12, na))
        y = rng.standard_normal((12, nb))
        # utils/audio.py:143-153, literally
        xc, yc = x, y
        if yc.shape[1] > xc.shape[1]: yc = yc[:, :xc.shape[1]]
        if xc.shape[1] > yc.shape[1]: xc = xc[:, :yc.shape[1]]
        ia, ib = AO.mcd_pairs(na, nb, 'cut')
        assert np.array_equal(x[:, ia], xc) and np.array_equal(y[:, ib], yc)
        xs, ys = x, y
        if xs.shape[1] > ys.shape[1]:
            m = xs.shape[1]
            ys = np.array([ys[:, i * ys.shape[1] // m] for i in range(m)]).T
        else:
            m = ys.shape[1]
            xs = np.array([xs[:, i * xs.shape[1] // m] for i in range(m)]).T
        ia, ib = AO.mcd_pairs(na, nb, 'stretch')
        assert np.array_equal(x[:, ia], xs) and np.array_equal(y[:, ib], ys)


def test_mcd_of_a_spectrogram_with_itself_is_zero():
    c = AO.mfcc(np.random.default_rng(5).normal(-40, 10, (80, 50)), 13)
    for mode in ('cut', 'stretch', 'dtw'):
        for dtype in (np.float32, np.float64):
            m, n = AO.mcd_from_cepstra(c, c, mode, dtype)
            assert m == 0.0 and n == 50


def test_frame_distance_mirror_is_the_sequential_fp32_sum():
    rng = np.random.default_rng(6)
    x = rng.standard_normal((4, 12)).astype(np.float32)
    y = rng.standard_normal((3, 12)).astype(np.float32)
    d = AO.frame_distances(x, y)
    for i in range(4):
        for j in range(3):
            acc = np.float32(0)
            for c in range(12):
                t = np.float32(x[i, c] - y[j, c])
                acc = np.float32(acc + np.float32(t * t))
            assert d[i, j] == np.sqrt(acc)


def test_header_constants_match_the_binding():
    h = open(os.path.join(build.ROOT, 'include', 'b200tts.h')).read()
    for name, v in _lib.MCD_MODES.items():
        assert re.search(rf'#define B200TTS_MCD_{name.upper()} {v}\b', h)
    assert re.search(rf'#define B200TTS_DTW_MAX_FRAMES {_lib.DTW_MAX_FRAMES}\b', h)
    # three diagonals of (fp64, int32) over the shorter side plus the border cell within 227 KB
    assert (_lib.DTW_MAX_FRAMES + 1) * 36 <= 227 * 1024 < (_lib.DTW_MAX_FRAMES + 2) * 36


def _shape(B=2, samples=3000, frames=12, n=N, hop=HOP, win=WIN, n_mels=80, pre=0.97):
    return _lib.AnalysisShape(B, samples, frames, n, hop, win, n_mels, pre)


def test_shape_validation_and_workspace_formula(lib):
    def ws(s):
        return lib.b200tts_analysis_workspace_bytes(ctypes.byref(s))
    up = lambda x: -(-x // 256) * 256
    for n, n_mels in ((N, 80), (1024, 0), (2048, 128)):
        M = n // 2
        assert ws(_shape(n=n, win=n, n_mels=n_mels)) == up(up(up(up(16 * M) + 16 * (M + 1)) + 8 * n) + 8 * n_mels)
    cases = [(_shape(n=1101), 'unsupported FFT size'), (_shape(win=1103), 'window length'), (_shape(win=0), 'window length'),
             (_shape(hop=0), 'hop'), (_shape(B=0), 'B >= 1'), (_shape(samples=1), 'at least one sample'),
             (_shape(frames=1), 'one frame'), (_shape(n_mels=-1), 'n_mels'), (_shape(n_mels=553), 'n_mels'),
             (_shape(pre=float('nan')), 'finite')]
    for s, msg in cases:
        assert ws(s) == 0
        assert msg.encode() in lib.b200tts_last_error(), (msg, lib.b200tts_last_error())
    buf = torch.zeros(64)
    p = _lib.ptr(buf)
    for args, msg in (((0, 80, 13), 'total_frames'), ((5, 0, 13), 'n_mels'), ((5, 80, 81), 'n_mfcc'), ((5, 2000, 13), 'n_mels')):
        assert lib.b200tts_mel_cepstrum(*args, p, p, None) != 0
        assert msg.encode() in lib.b200tts_last_error()
    for args, msg in (((0, 13, 2), 'B'), ((1, 1, 2), 'n_mfcc'), ((1, 13, 3), 'unknown mode')):
        assert lib.b200tts_mel_cepstral_distortion(*args, p, p, p, p, p, None, None) != 0
        assert msg.encode() in lib.b200tts_last_error()


@pytest.mark.skipif(torch.cuda.is_available(), reason='checks the no-GPU failure mode')
def test_analysis_entry_points_fail_without_gpu(lib):
    s = _shape()
    buf = torch.zeros(1 << 16)
    off = torch.tensor([0, 6, 12], dtype=torch.int32)
    p, po = _lib.ptr(buf), _lib.ptr(off)
    assert lib.b200tts_stft_magnitude(ctypes.byref(s), p, po, po, p, p, p, buf.numel() * 4, None) != 0
    assert lib.b200tts_amplitude_to_db(ctypes.byref(s), p, po, p, None) != 0
    assert lib.b200tts_mel_cepstrum(12, 80, 13, p, p, None) != 0
    assert lib.b200tts_mel_cepstral_distortion(2, 13, 2, p, po, p, po, p, None, None) != 0
    assert b'no CPU fallback' in lib.b200tts_last_error() or b'CUDA' in lib.b200tts_last_error()
    with pytest.raises((_lib.B200TTSError, RuntimeError, AssertionError)):
        audio.spectrogram(np.zeros(1000, np.float32))
    with pytest.raises((_lib.B200TTSError, RuntimeError, AssertionError)):
        audio.mel_cepstral_distorision(np.zeros((80, 5), np.float32), np.zeros((80, 5), np.float32), 'dtw')


def test_python_input_validation():
    S = np.zeros((80, 5), np.float32)
    bad_spectrogram = [[], [np.zeros((2, 5), np.float32)], [np.zeros(0, np.float32)], [np.zeros(100, np.int16)],
                       [torch.zeros(100, dtype=torch.int32)], 'not a list']
    for arg in bad_spectrogram:
        with pytest.raises(ValueError):
            audio.spectrogram_batch(arg)
    with pytest.raises(ValueError):
        audio.get_spectrogram_mfcc(np.zeros(80, np.float32))
    with pytest.raises(ValueError):
        audio.get_spectrogram_mfcc(np.zeros((12, 5), np.float32))              # fewer mel bands than hp.num_mfcc
    with pytest.raises(ValueError):
        audio.mel_cepstral_distortion_batch([S], [S, S])
    with pytest.raises(ValueError):
        audio.mel_cepstral_distortion_batch([], [])
    with pytest.raises(ValueError):
        audio.mel_cepstral_distortion_batch([S], [S], 'fast')
    with pytest.raises(ValueError):
        audio.mel_cepstral_distorision(S, np.zeros((40, 5), np.float32), 'cut')
    with pytest.raises(ValueError):
        audio.mel_cepstral_distorision(S, S.astype(np.int32), 'cut')
    with pytest.raises(ValueError, match='at most'):
        big = np.zeros((80, _lib.DTW_MAX_FRAMES + 1), np.float32)
        audio.mel_cepstral_distortion_batch([big], [big], 'dtw')


def test_normalize_inverts_denormalize(monkeypatch):
    from multilingual_text_to_speech_b200.params.params import Params as hp
    for name, v in (('mel_normalize_mean', -40.0), ('mel_normalize_variance', 15.0), ('lin_normalize_mean', -50.0),
                    ('lin_normalize_variance', 20.0)):
        monkeypatch.setattr(hp, name, v, raising=False)
    S = np.random.default_rng(7).normal(-40, 10, (80, 9))
    assert np.allclose(audio.normalize_spectrogram(S, True), (S + 40) / 15, rtol=0, atol=1e-12)
    for is_mel in (True, False):
        assert np.allclose(audio.denormalize_spectrogram(audio.normalize_spectrogram(S, is_mel), is_mel), S, rtol=0, atol=1e-12)


def test_analysis_kernels_do_not_spill():
    nvcc = next((c for c in (os.environ.get('NVCC'), '/usr/local/cuda/bin/nvcc', shutil.which('nvcc')) if c and os.path.exists(c)), None)
    if nvcc is None:
        pytest.skip('nvcc not available')
    src = os.path.join(build.CSRC, 'analysis.cu')
    cmd = [nvcc] + build.NVCC_FLAGS + ['-I', os.path.join(build.ROOT, 'include'), '-Xptxas', '-v', '-cubin', src, '-o', os.devnull]
    res = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    assert res.returncode == 0, res.stdout
    found = re.findall(r'Function properties for \S*(analysis_\w+?_kernel)\S*\n\s*\d+ bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads',
                       res.stdout)
    names = {f[0] for f in found}
    assert names == {'analysis_tables_kernel', 'analysis_stft_kernel', 'analysis_db_kernel', 'analysis_cepstrum_kernel',
                     'analysis_mcd_linear_kernel', 'analysis_mcd_dtw_kernel'}, names
    for name, st, ld in found:
        assert st == '0' and ld == '0', (name, st, ld)
