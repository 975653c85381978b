"""Time-scale modification without a GPU: the WSOLA oracle against its own contract (identity at rate 1 and at unchanged durations,
output lengths, pitch kept under stretching, onsets moved, symbols retimed), the library's warps against the oracle's, every ValueError
of time_stretch_batch and retime_batch, the library's argument checks and the kernels' registers."""
import ctypes
import os
import re
import shutil
import subprocess

import numpy as np
import pytest
import torch

import pitch_oracle as P
import wsola_oracle as O
from test_pitch_cpu import glide, noise, tone

SR, HOP = 22050, 275
RATES = (0.5, 0.8, 1.25, 2.0)


def onset_case():
    """tone - silence - tone, and the sample where the second tone starts."""
    a, gap = tone(150.0, 0.2), np.zeros(2500)
    return np.concatenate([a, gap, tone(250.0, 0.2)]), len(a) + len(gap)


def identity_cases():
    out = [(f'tone{f:g}', tone(f, 0.3)) for f in (80.0, 200.0, 311.0)]
    out += [('glide', glide(120.0, 180.0, 0.5)), ('noise', noise(0.3)), ('silence', np.zeros(3000)),
            ('tone-silence-tone', onset_case()[0]), ('one sample', np.array([0.25])), ('one negative sample', np.array([-0.5]))]
    return out


CASES = identity_cases()


def partition(total, parts, seed):
    """A random split of `total` frames into `parts` non-negative durations (some of them 0)."""
    rng = np.random.default_rng(seed)
    cuts = np.sort(rng.integers(0, total + 1, parts - 1))
    return np.diff(np.concatenate([[0], cuts, [total]])).astype(np.int64)


def _check_identity(name, x, y, p, tau):
    x32 = x.astype(np.float32).astype(np.float64)
    assert len(y) == len(x)
    assert np.abs(y - x32).max() <= 1e-6 * max(np.abs(x32).max(), 1e-30), name
    if name in ('noise', 'glide'):
        # p_k = kH on every frame: d = 0 where kH <= L, and where the nominal position is clamped to L the search finds kH - L
        np.testing.assert_array_equal(p, np.rint(tau))


@pytest.mark.parametrize('case', range(len(CASES)), ids=[c[0] for c in CASES])
def test_identity_at_rate_one(case):
    name, x = CASES[case]
    y, p, tau = O.time_stretch(x, 1.0, HOP)
    np.testing.assert_array_equal(tau, np.arange(len(tau)) * HOP)
    _check_identity(name, x, y, p, tau)


@pytest.mark.parametrize('case', range(len(CASES)), ids=[c[0] for c in CASES])
def test_identity_at_unchanged_durations(case):
    name, x = CASES[case]
    F = 1 + len(x) // HOP
    d = partition(F, min(F, 5) + 1, case)
    y, p, tau = O.retime(x, d, d, HOP)
    np.testing.assert_array_equal(tau, np.arange(len(tau)) * HOP)
    _check_identity(name, x, y, p, tau)


def test_lengths():
    for L in (1, 2, 274, 275, 276, 549, 550, 12345):
        for rate in (0.25, 0.5, 0.8, 1.0, 1.25, 2.0, 4.0):
            Lp, tau = O.stretch_warp(L, HOP, rate)
            assert Lp == max(1, int(round(L / rate))) and len(tau) == (Lp - 1) // HOP + 2
            # the synthesis frames cover [0, L'): sample n reads frames n // H and n // H + 1
            assert (Lp - 1) // HOP + 1 < len(tau)
        F = 1 + L // HOP
        for seed in range(4):
            d = partition(F, 6, seed)
            dp = partition(max(1, int(F * (0.5 + seed / 2))), 6, 10 + seed)
            Lp, tau = O.retime_warp(L, HOP, d, dp)
            assert 1 + Lp // HOP == dp.sum(), (L, d, dp, Lp)


def test_library_warps_equal_the_oracle():
    from multilingual_text_to_speech_b200.utils import audio
    for L in (1, 274, 550, 12345, 220500):
        for rate in (0.25, 0.8, 1.0, 1.2, 3.7, 4.0):
            Lp, tau = audio._stretch_plan(L, HOP, rate)
            Lp_o, tau_o = O.stretch_warp(L, HOP, rate)
            assert Lp == Lp_o and tau.dtype == np.float64 and np.array_equal(tau, tau_o)
        F = 1 + L // HOP
        for seed in range(6):
            d = partition(F, 1 + seed * 3, seed)
            dp = partition(max(1, int(F * (0.3 + seed / 3))), 1 + seed * 3, 20 + seed)
            Lp, tau = audio._retime_plan(L, HOP, d, dp)
            Lp_o, tau_o = O.retime_warp(L, HOP, d, dp)
            assert Lp == Lp_o and np.array_equal(tau, tau_o), (L, seed)
            from multilingual_text_to_speech_b200.functional import scale_durations
            ds = scale_durations(d, 1.2)
            if ds.sum() >= 1:
                assert np.array_equal(audio._retime_plan(L, HOP, d, ds)[1], O.retime_warp(L, HOP, d, ds)[1])


def test_retime_warp_rules():
    """Symbols with d' = 0 are dropped, those with d = 0 hold their boundary, and past the last boundary the slope is 1."""
    d, dp = [3, 0, 4, 2], [6, 2, 0, 1]
    L = HOP * (sum(d) - 1) + 10
    Lp, tau = O.retime_warp(L, HOP, d, dp)
    phi = tau / HOP
    np.testing.assert_allclose(phi[:6], -0.5 + (np.arange(6) + 0.5) * 0.5)        # symbol 0: 6 output frames onto 3 input frames
    np.testing.assert_array_equal(phi[6:8], [2.5, 2.5])                           # symbol 1 (d = 0) holds the boundary 3 - 1/2
    np.testing.assert_allclose(phi[8], 2.5 + 4 + 0.5 * 2)                         # symbol 2 is dropped; symbol 3 follows at slope 2
    assert len(phi) == 10 and phi[9] == 9.0                                       # past the last boundary 9 - 1/2, slope 1


@pytest.mark.parametrize('f', [100.0, 160.0, 300.0])
def test_pitch_is_kept(f):
    x = tone(f, 2.0)
    for rate in RATES:
        y, _, _ = O.time_stretch(x, rate, HOP)
        assert len(y) == int(round(len(x) / rate))
        g, voiced, _ = P.pyin(y.astype(np.float32).astype(np.float64), SR, HOP)
        inner = slice(4, len(g) - 4)
        assert voiced[inner].all(), (f, rate)
        cents = np.abs(1200 * np.log2(g[inner] / f))
        print(f'{f:g} Hz at rate {rate}: median |cents| {np.median(cents):.2f}')
        assert np.median(cents) <= 10.0, (f, rate, np.median(cents))


@pytest.mark.parametrize('rate', RATES)
def test_second_onset_moves(rate):
    x, onset = onset_case()
    y, _, _ = O.time_stretch(x, rate, HOP)
    mid_gap = int(np.rint((onset - 1250) / rate))          # the middle of the 2,500-sample gap, more than D + H from either tone
    assert np.abs(y[mid_gap - int(1250 / rate) + 2 * HOP:mid_gap]).max() == 0.0
    got = mid_gap + int(np.flatnonzero(np.abs(y[mid_gap:]) > 1e-3)[0])
    want = int(np.rint(onset / rate))
    print(f'rate {rate}: onset {got}, expected {want}')
    assert abs(got - want) <= 2 * HOP, (rate, got, want)                          # within D + H, D = H


SEGMENT_TONES = (110.0, 150.0, 200.0, 260.0, 180.0)
SEGMENT_FRAMES = np.array([16, 24, 12, 20, 18])


def segmented_tones():
    """Five tones, tone j over the samples of mel frames [B_j, B_{j+1}) (B the cumulative SEGMENT_FRAMES), frame k owning the samples
    nearest kH; -> (x, durations) with sum(durations) = 1 + L // H."""
    B = np.concatenate([[0], np.cumsum(SEGMENT_FRAMES)])
    L = HOP * (int(B[-1]) - 1) + 100
    x = np.zeros(L)
    t = np.arange(L) / SR
    for j, f in enumerate(SEGMENT_TONES):
        lo, hi = max(0, B[j] * HOP - HOP // 2), (L if j == len(SEGMENT_TONES) - 1 else B[j + 1] * HOP - HOP // 2)
        x[lo:hi] = sum(0.5 / h * np.sin(2 * np.pi * h * f * t[lo:hi]) for h in range(1, 4))
    return x.astype(np.float32).astype(np.float64), SEGMENT_FRAMES.copy()


def retimed_frames_on_tone(y, dp, margin=3, cents=20.0):
    """Every output frame at least `margin` frames inside symbol j re-tracks to tone j within `cents`; -> worst |cents|."""
    g, voiced, _ = P.pyin(np.asarray(y, dtype=np.float32).astype(np.float64), SR, HOP)
    Bp = np.concatenate([[0], np.cumsum(dp)])
    worst = 0.0
    for j, f in enumerate(SEGMENT_TONES):
        k = np.arange(Bp[j] + margin, Bp[j + 1] - margin)
        if len(k) == 0:
            continue
        assert voiced[k].all(), (j, k[~voiced[k]])
        err = np.abs(1200 * np.log2(g[k] / f))
        worst = max(worst, float(err.max()))
        assert (err <= cents).all(), (j, err.max())
    return worst


def retime_targets(d):
    from multilingual_text_to_speech_b200.functional import scale_durations
    return {'rotated': np.roll(d, 1), 'reversed': d[::-1].copy(), 'scaled 1.5': scale_durations(d, 1.5),
            'scaled 0.7': scale_durations(d, 0.7)}


@pytest.mark.parametrize('target', ['rotated', 'reversed', 'scaled 1.5', 'scaled 0.7'])
def test_retime_moves_each_tone_into_its_new_span(target):
    x, d = segmented_tones()
    dp = retime_targets(d)[target]
    y, _, _ = O.retime(x, d, dp, HOP)
    assert 1 + len(y) // HOP == dp.sum()
    print(f'{target}: worst |cents| {retimed_frames_on_tone(y, dp):.2f}')


# ---- ValueErrors -----------------------------------------------------------------------------------------------------------------------
def test_time_stretch_batch_errors():
    from multilingual_text_to_speech_b200.utils import audio
    y = tone(150.0, 0.1).astype(np.float32)
    bad_calls = [
        dict(waveforms=[], rate=1.0), dict(waveforms='x', rate=1.0), dict(waveforms=[np.zeros((2, 10))], rate=1.0),
        dict(waveforms=[np.zeros(0)], rate=1.0), dict(waveforms=[np.arange(10)], rate=1.0),
        dict(waveforms=[np.array([0.0, np.nan])], rate=1.0), dict(waveforms=[np.array([0.0, np.inf])], rate=1.0),
        dict(waveforms=[y], rate=[1.0, 2.0]), dict(waveforms=[y, y], rate=[1.0]), dict(waveforms=[y], rate=np.ones((1, 1))),
        dict(waveforms=[y], rate=0.24), dict(waveforms=[y], rate=4.01), dict(waveforms=[y], rate=0.0), dict(waveforms=[y], rate=-1.0),
        dict(waveforms=[y], rate=float('nan')), dict(waveforms=[y], rate=float('inf')), dict(waveforms=[y], rate='fast'),
        dict(waveforms=[y, y], rate=[1.0, 5.0]),
    ]
    for kw in bad_calls:
        with pytest.raises(ValueError):
            audio.time_stretch_batch(**kw)
    with pytest.raises(ValueError):
        audio.time_stretch(np.zeros((3, 3)), 1.0)
    with pytest.raises(ValueError):
        audio.time_stretch(torch.zeros(100, dtype=torch.int32), 1.0)


def test_retime_batch_errors():
    from multilingual_text_to_speech_b200.utils import audio
    y = tone(150.0, 0.1).astype(np.float32)
    F = 1 + len(y) // HOP
    d = np.array([3, F - 3])
    bad_calls = [
        dict(waveforms=[], durations=[], new_durations=[]), dict(waveforms=[np.array([np.nan])], durations=[[1]], new_durations=[[1]]),
        dict(waveforms=[y], durations=d, new_durations=[d]), dict(waveforms=[y], durations=[d], new_durations=d),
        dict(waveforms=[y], durations=[d, d], new_durations=[d]), dict(waveforms=[y, y], durations=[d], new_durations=[d]),
        dict(waveforms=[y], durations=[d + 1], new_durations=[d]),                      # total is not 1 + L // hop
        dict(waveforms=[y], durations=[d], new_durations=[d[:1]]),                      # lengths differ
        dict(waveforms=[y], durations=[d], new_durations=[np.array([2, -1])]),
        dict(waveforms=[y], durations=[np.array([-1, F + 1])], new_durations=[d]),
        dict(waveforms=[y], durations=[d], new_durations=[np.array([0, 0])]),
        dict(waveforms=[y], durations=[d.astype(np.float64)], new_durations=[d]),
        dict(waveforms=[y], durations=[d], new_durations=[np.array([[1, 2]])]),
        dict(waveforms=[y], durations=[np.array([], dtype=np.int64)], new_durations=[np.array([], dtype=np.int64)]),
        dict(waveforms=[y], durations=[d], new_durations=[np.array([1, 2 ** 31 // HOP + 1])]),   # 2^31 + 154 output samples
    ]
    for kw in bad_calls:
        with pytest.raises(ValueError):
            audio.retime_batch(**kw)
    with pytest.raises(ValueError):
        audio.retime(y, d, d[:1])


# ---- the library -----------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope='module')
def lib():
    import __graft_entry__ as entry
    entry.build()
    from multilingual_text_to_speech_b200 import _lib
    return _lib.load()


def _shape(**kw):
    from multilingual_text_to_speech_b200 import _lib
    s = _lib.WsolaShape(2, 4000, 3000, 16, 275, 275)
    for k, v in kw.items():
        setattr(s, k, v)
    return s


def test_library_argument_checks(lib):
    x = torch.zeros(64, dtype=torch.float64)
    p = ctypes.c_void_p(x.data_ptr())
    q = ctypes.c_void_p(x.data_ptr() + 8)
    for kw, msg in ((dict(B=0), b'B >= 1'), (dict(total_samples=1), b'B >= 1'), (dict(total_out_samples=1), b'B >= 1'),
                    (dict(total_frames=3), b'B >= 1'), (dict(total_samples=2 ** 31 - 1), b'INT_MAX'), (dict(hop=0), b'hop'),
                    (dict(hop=1025), b'hop'), (dict(tolerance=-1), b'tolerance'), (dict(tolerance=1025), b'tolerance')):
        s = ctypes.byref(_shape(**kw))
        assert lib.b200tts_wsola_positions(s, p, p, p, p, q, None) != 0, kw
        assert msg in lib.b200tts_last_error(), (kw, lib.b200tts_last_error())
        assert lib.b200tts_wsola_overlap_add(s, p, p, p, p, p, q, None) != 0, kw
        assert msg in lib.b200tts_last_error(), (kw, lib.b200tts_last_error())
    good = ctypes.byref(_shape())
    assert lib.b200tts_wsola_positions(None, p, p, p, p, q, None) != 0 and b'null' in lib.b200tts_last_error()
    for i in range(5):
        args = [p, p, p, p, q]
        args[i] = None
        assert lib.b200tts_wsola_positions(good, *args, None) != 0 and b'null' in lib.b200tts_last_error(), i
    assert lib.b200tts_wsola_overlap_add(None, p, p, p, p, p, q, None) != 0 and b'null' in lib.b200tts_last_error()
    for i in range(6):
        args = [p, p, p, p, p, q]
        args[i] = None
        assert lib.b200tts_wsola_overlap_add(good, *args, None) != 0 and b'null' in lib.b200tts_last_error(), i
    assert lib.b200tts_wsola_overlap_add(good, p, p, p, p, p, p, None) != 0 and b'alias' in lib.b200tts_last_error()


@pytest.mark.skipif(torch.cuda.is_available(), reason='checks the no-GPU failure mode')
def test_calls_without_gpu_fail_loudly(lib):
    good = ctypes.byref(_shape())
    x = torch.zeros(1 << 16, dtype=torch.float64)
    p = ctypes.c_void_p(x.data_ptr())
    q = ctypes.c_void_p(x.data_ptr() + 8)
    assert lib.b200tts_wsola_positions(good, p, p, p, p, q, None) != 0
    assert lib.b200tts_wsola_overlap_add(good, p, p, p, p, p, q, None) != 0
    from multilingual_text_to_speech_b200 import _lib
    from multilingual_text_to_speech_b200.utils import audio
    y = np.zeros(2000, dtype=np.float32)
    with pytest.raises((_lib.B200TTSError, RuntimeError, AssertionError)):
        audio.time_stretch_batch([y], 1.25)
    with pytest.raises((_lib.B200TTSError, RuntimeError, AssertionError)):
        audio.retime_batch([y], [np.array([1 + 2000 // HOP])], [np.array([3])])


# measured (CUDA 12.9, sm_90a, -Xptxas -v): registers of each kernel; none spills or keeps a stack frame
WSOLA_REGS = {'wsola_search_kernel': 56, 'wsola_ola_kernel': 40}


def test_kernel_registers_and_spills():
    from multilingual_text_to_speech_b200 import build
    nvcc = next((c for c in (os.environ.get('NVCC'), '/usr/local/cuda/bin/nvcc', shutil.which('nvcc')) if c and os.path.exists(c)), None)
    if nvcc is None:
        pytest.skip('nvcc not available')
    import tempfile
    with tempfile.TemporaryDirectory() as tmp:
        cmd = [nvcc] + build.NVCC_FLAGS + ['-I', os.path.join(build.ROOT, 'include'), '-Xptxas', '-v', '-cubin',
               os.path.join(build.CSRC, 'wsola.cu'), '-o', os.path.join(tmp, 'wsola.cubin')]
        res = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    assert res.returncode == 0, res.stdout
    for name, regs in WSOLA_REGS.items():
        m = re.search(r'Function properties for \S*' + name + r'\S*\n\s*(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes '
                      r'spill loads\n[^\n]*Used (\d+) registers', res.stdout)
        assert m, (name, res.stdout)
        stack, st, ld, used = map(int, m.groups())
        assert (stack, st, ld) == (0, 0, 0), (name, stack, st, ld)
        assert used <= regs, (name, used)
