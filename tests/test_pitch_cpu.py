"""Pitch analysis without a GPU: the pYIN oracle against its own definitions and against signals of known pitch, the banded Viterbi against
the dense one and brute force, every ValueError of the Python entry points, the library's argument checks and the kernels' registers."""
import ctypes
import os
import re
import shutil
import subprocess

import numpy as np
import pytest
import torch

import pitch_oracle as P

SR, HOP = 22050, 275


def tone(f0, seconds=0.5, harmonics=4, sr=SR):
    t = np.arange(int(seconds * sr)) / sr
    return sum(0.5 / k * np.sin(2 * np.pi * k * f0 * t) for k in range(1, harmonics + 1)).astype(np.float32).astype(np.float64)


def glide(f_start, f_end, seconds=0.5, sr=SR):
    t = np.arange(int(seconds * sr)) / sr
    phase = 2 * np.pi * (f_start * t + (f_end - f_start) * t ** 2 / (2 * seconds))
    return (0.5 * np.sin(phase) + 0.2 * np.sin(2 * phase)).astype(np.float32).astype(np.float64)


def noise(seconds=0.5, seed=0):
    return (0.3 * np.random.default_rng(seed).standard_normal(int(seconds * SR))).astype(np.float32).astype(np.float64)


def test_fft_cmnd_equals_direct_sums():
    g = P.geometry(SR, HOP, 65.406, 2093.0, 1024)
    y = np.concatenate([tone(110.0, 0.2), np.zeros(2000), noise(0.2)])
    yf = P.frames(y, 1024, HOP)
    a = P.cmnd(yf, 1024, g['win_length'], g['min_period'], g['max_period'])
    b = P.cmnd_direct(yf, g['win_length'], g['min_period'], g['max_period'])
    assert a.shape == b.shape == (g['max_period'] - g['min_period'] + 1, 1 + len(y) // HOP)
    np.testing.assert_allclose(a, b, rtol=1e-9, atol=1e-11)


def _random_case(rng, n, F, zero=False):
    obs = np.zeros((F, n)) if zero else rng.random((F, n)) * (rng.random((F, n)) < 0.3)
    vp = np.clip(obs.sum(1), 0, 1)
    full = np.concatenate([obs.T, np.tile((1 - vp) / n, (n, 1))], 0)
    return obs, vp, full


@pytest.mark.parametrize('n,W', [(5, 3), (9, 5), (12, 11), (20, 7), (31, 31)])
@pytest.mark.parametrize('kind', ['random', 'zero', 'ties'])
def test_banded_viterbi_equals_dense(n, W, kind):
    rng = np.random.default_rng(n * 100 + W)
    F = 12
    obs, vp, full = _random_case(rng, n, F, zero=kind == 'zero')
    if kind == 'ties':
        # exact ties: a few equal probabilities, repeated on neighbouring bins and frames
        obs = np.zeros((F, n))
        obs[:, ::3] = 0.25
        obs[::2, 1::4] = 0.25
        vp = np.clip(obs.sum(1), 0, 1)
        full = np.concatenate([obs.T, np.tile((1 - vp) / n, (n, 1))], 0)
    s_dense, v_dense = P.viterbi(full, P.transition(n, W), P.p_init(n))
    s_band, v_band = P.viterbi_banded(obs, vp, n, W)
    np.testing.assert_array_equal(s_band, s_dense)
    assert v_band == v_dense


@pytest.mark.parametrize('n,W,F', [(1, 1, 4), (2, 1, 4), (3, 3, 3), (3, 1, 4)])
def test_viterbi_against_brute_force(n, W, F):
    rng = np.random.default_rng(7 + n + F)
    for kind in ('random', 'zero'):
        obs, vp, full = _random_case(rng, n, F, zero=kind == 'zero')
        trans, init = P.transition(n, W), P.p_init(n)
        best = P.brute_force(full, trans, init)
        s_dense, v_dense = P.viterbi(full, trans, init)
        s_band, v_band = P.viterbi_banded(obs, vp, n, W)
        assert v_dense == best and P.path_score(full, trans, init, s_dense) == best
        np.testing.assert_array_equal(s_band, s_dense)


def _interior(y):
    F = 1 + len(y) // HOP
    return slice(4, F - 4)


@pytest.mark.parametrize('f0', [80.0, 123.0, 200.0, 311.0, 400.0])
def test_oracle_tracks_tones(f0):
    f, voiced, _ = P.pyin(tone(f0), SR, HOP)
    s = _interior(tone(f0))
    assert voiced[s].all()
    bins = 120 * np.log2(f[s] / 65.406)
    assert np.abs(bins - 120 * np.log2(f0 / 65.406)).max() <= 1.0


def test_oracle_follows_a_glide_and_marks_silence_and_noise():
    y = glide(120.0, 180.0, 1.0)
    f, voiced, _ = P.pyin(y, SR, HOP)
    s = _interior(y)
    assert voiced[s].all()
    # the difference function of frame t looks at samples t hop - 512 + [1, 1024): its window y[1 .. 512] is centred 256 samples early
    t = ((np.arange(len(f)) * HOP - 256) / SR)[s]
    truth = 120.0 + (180.0 - 120.0) * t / 1.0
    assert np.abs(120 * np.log2(f[s] / truth)).max() <= 1.0
    f, voiced, vp = P.pyin(np.zeros(8000), SR, HOP)
    assert not voiced.any() and np.isnan(f).all() and (vp == 0).all()
    f, voiced, _ = P.pyin(noise(), SR, HOP)
    assert voiced[_interior(noise())].mean() < 0.5


def test_oracle_tone_silence_tone():
    y = np.concatenate([tone(150.0, 0.4), np.zeros(int(0.4 * SR)), tone(250.0, 0.4)])
    f, voiced, _ = P.pyin(y, SR, HOP)
    fr = lambda sec: int(sec * SR / HOP)                # noqa: E731
    assert voiced[fr(0.05):fr(0.35)].all() and not voiced[fr(0.45):fr(0.75)].any() and voiced[fr(0.85):fr(1.15)].all()
    assert np.abs(120 * np.log2(f[fr(0.05):fr(0.35)] / 150.0)).max() <= 1.0
    assert np.abs(120 * np.log2(f[fr(0.85):fr(1.15)] / 250.0)).max() <= 1.0


def test_library_tables_equal_the_oracle():
    from multilingual_text_to_speech_b200.utils import audio
    g = audio.pitch_geometry()
    assert g == dict(sr=SR, hop=HOP, **P.geometry(SR, HOP, 65.406, 2093.0, 1024))
    assert (g['min_period'], g['max_period'], g['n_bins'], g['transition_width']) == (10, 338, 601, 51)
    np.testing.assert_array_equal(audio._pitch_log_transitions(41, 11), P.banded_log_transitions(41, 11))


# ---- ValueErrors -----------------------------------------------------------------------------------------------------------------------
def test_pitch_batch_errors():
    from multilingual_text_to_speech_b200.utils import audio
    y = np.zeros(1000, dtype=np.float32)
    for bad in ([], 'x', [np.zeros((2, 10))], [np.zeros(0)], [np.zeros(10, dtype=np.int16)], [torch.zeros(10, dtype=torch.int32)]):
        with pytest.raises(ValueError):
            audio.pitch_batch(bad)
    for kw in (dict(fmin=0.0), dict(fmin=-5.0), dict(fmin=300.0, fmax=300.0), dict(fmin=400.0, fmax=300.0), dict(fmax=12000.0),
               dict(fmin=1.0, fmax=11000.0), dict(fmin=200.0, fmax=240.0), dict(frame_length=1023), dict(frame_length=4096),
               dict(frame_length=16), dict(frame_length=22)):
        with pytest.raises(ValueError):
            audio.pitch_batch([y], **kw)
    with pytest.raises(ValueError):
        audio.pitch(np.zeros((3, 3)))


def test_energy_batch_errors():
    from multilingual_text_to_speech_b200.utils import audio
    for bad in ([], None, [np.zeros((2, 10))], [np.zeros(0)], [np.arange(10)]):
        with pytest.raises(ValueError):
            audio.energy_batch(bad)


def test_symbol_average_errors():
    from multilingual_text_to_speech_b200.functional import symbol_average
    x = torch.ones(2, 10)
    d = torch.tensor([[3, 4], [5, 5]])
    for args in ((np.ones((2, 10)), d), (torch.ones(10), d), (torch.ones(2, 10, dtype=torch.int64), d), (x, d.float()),
                 (x, torch.tensor([3, 4])), (x, d[:1]), (x, torch.tensor([[3, -1], [5, 5]])), (x, torch.tensor([[3, 4], [5, 6]])),
                 (x, d, torch.ones(2, 10)), (x, d, torch.ones(2, 9, dtype=torch.bool))):
        with pytest.raises(ValueError):
            symbol_average(*args)


def test_symbol_average_hand_computed():
    from multilingual_text_to_speech_b200.functional import symbol_average
    x = torch.tensor([[1.0, 2.0, 3.0, 4.0, 5.0, 6.0], [10.0, float('nan'), 30.0, 40.0, 50.0, 60.0]])
    d = torch.tensor([[2, 0, 3], [1, 2, 2]])
    got = symbol_average(x[:1], d[:1])
    assert got.dtype == torch.float64 and got.tolist() == [[1.5, 0.0, 4.0]]
    voiced = torch.tensor([[True, False, True, True, False, True], [True, False, True, False, False, True]])
    assert symbol_average(x, d, voiced).tolist() == [[1.0, 0.0, 3.5], [10.0, 30.0, 0.0]]


def test_pitch_errors_batch():
    from multilingual_text_to_speech_b200.utils import audio
    nan = np.nan
    ref = np.array([100.0, 100.0, 200.0, nan, nan, 100.0])
    gen = np.array([100.0, 130.0, 200.0 * 2 ** (50 / 1200), 90.0, nan, nan, 7.0])
    r = audio.pitch_errors_batch([ref], [gen])
    # 6 frames: VV = {0, 1, 2}, gross = {1} (30 % off), voicing errors = {3, 5}
    assert r['gpe'][0] == 1 / 3 and r['vde'][0] == 2 / 6 and r['ffe'][0] == 3 / 6
    cents = np.array([0.0, 1200 * np.log2(1.3), 1200 * np.log2(200.0 * 2 ** (50 / 1200) / 200.0)])
    assert np.isclose(r['f0_rmse_cents'][0], np.sqrt(np.mean(cents ** 2)), rtol=1e-14)
    r = audio.pitch_errors_batch([torch.tensor([nan, nan])], [torch.tensor([nan, 100.0, 100.0])])
    assert torch.isnan(r['gpe'][0]) and torch.isnan(r['f0_rmse_cents'][0]) and r['vde'][0] == 0.5 and r['ffe'][0] == 0.5
    for a, b in (([], []), (ref, [gen]), ([ref], [gen, gen]), ([ref], [np.array([1.0, -2.0])]), ([np.zeros((2, 2))], [gen]),
                 ([np.array([], dtype=np.float64)], [gen]), ([np.array([1, 2])], [gen]), ([np.array([np.inf])], [gen])):
        with pytest.raises(ValueError):
            audio.pitch_errors_batch(a, b)


# ---- the library -----------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope='module')
def lib():
    import __graft_entry__ as entry
    entry.build()
    from multilingual_text_to_speech_b200 import _lib
    return _lib.load()


def _shape(**kw):
    from multilingual_text_to_speech_b200 import _lib
    s = _lib.PitchShape(2, 4000, 16, 1024, 512, 275, 10, 338, 601, 51, 22050.0, 65.406, float(np.log(P.TINY)), float(np.log(1 / 601)))
    for k, v in kw.items():
        setattr(s, k, v)
    return s


def test_library_argument_checks(lib):
    good = _shape()
    assert lib.b200tts_pitch_workspace_bytes(ctypes.byref(good)) == 16 * 2 * 601 * 2
    for kw, msg in ((dict(B=0), b'B >= 1'), (dict(frame_length=1023, win_length=511), b'even'), (dict(win_length=500), b'win_length'),
                    (dict(hop=0), b'hop'), (dict(max_period=10), b'min_period'), (dict(max_period=512), b'max_period'),
                    (dict(n_bins=1202), b'n_bins'), (dict(transition_width=50), b'transition_width'),
                    (dict(transition_width=603), b'transition_width'), (dict(fmin=0.0), b'fmin')):
        assert lib.b200tts_pitch_workspace_bytes(ctypes.byref(_shape(**kw))) == 0, kw
        assert msg in lib.b200tts_last_error(), (kw, lib.b200tts_last_error())
    x = torch.zeros(64, dtype=torch.float64)
    p = ctypes.c_void_p(x.data_ptr())
    assert lib.b200tts_pitch_cmnd(None, p, p, p, p, None) != 0
    assert lib.b200tts_pitch_cmnd(ctypes.byref(good), p, None, p, p, None) != 0 and b'null' in lib.b200tts_last_error()
    assert lib.b200tts_pitch_observations(ctypes.byref(_shape(B=0)), p, p, p, None) != 0
    assert lib.b200tts_pitch_viterbi(ctypes.byref(good), p, p, p, p, p, p, 10, None) != 0
    assert b'workspace' in lib.b200tts_last_error()


@pytest.mark.skipif(torch.cuda.is_available(), reason='checks the no-GPU failure mode')
def test_calls_without_gpu_fail_loudly(lib):
    good = _shape()
    x = torch.zeros(1 << 16, dtype=torch.float64)
    p = ctypes.c_void_p(x.data_ptr())
    for st in (lib.b200tts_pitch_cmnd(ctypes.byref(good), p, p, p, p, None),
               lib.b200tts_pitch_observations(ctypes.byref(good), p, p, p, None),
               lib.b200tts_pitch_viterbi(ctypes.byref(good), p, p, p, p, p, p, x.numel() * 8, None)):
        assert st != 0
    from multilingual_text_to_speech_b200 import _lib
    from multilingual_text_to_speech_b200.utils import audio
    with pytest.raises((_lib.B200TTSError, RuntimeError, AssertionError)):
        audio.pitch_batch([np.zeros(2000, dtype=np.float32)])


# measured (CUDA 12.9, sm_90a, -Xptxas -v): registers of each kernel; none spills
PITCH_REGS = {'pitch_cmnd_kernel': 32, 'pitch_obs_kernel': 56, 'pitch_viterbi_kernel': 56}


def test_kernel_registers_and_spills():
    from multilingual_text_to_speech_b200 import build
    nvcc = next((c for c in (os.environ.get('NVCC'), '/usr/local/cuda/bin/nvcc', shutil.which('nvcc')) if c and os.path.exists(c)), None)
    if nvcc is None:
        pytest.skip('nvcc not available')
    import tempfile
    with tempfile.TemporaryDirectory() as tmp:
        cmd = [nvcc] + build.NVCC_FLAGS + ['-I', os.path.join(build.ROOT, 'include'), '-Xptxas', '-v', '-cubin',
               os.path.join(build.CSRC, 'pitch.cu'), '-o', os.path.join(tmp, 'pitch.cubin')]
        res = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    assert res.returncode == 0, res.stdout
    for name, regs in PITCH_REGS.items():
        m = re.search(r'Function properties for \S*' + name + r'\S*\n\s*(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes '
                      r'spill loads\n[^\n]*Used (\d+) registers', res.stdout)
        assert m, (name, res.stdout)
        stack, st, ld, used = map(int, m.groups())
        assert (stack, st, ld) == (0, 0, 0), (name, stack, st, ld)
        assert used <= regs, (name, used)
