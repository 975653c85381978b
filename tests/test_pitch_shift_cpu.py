"""Pitch shifting without a GPU: the TD-PSOLA oracle against its own contract (identity at ratio 1, mark invariants, coverage, shift
accuracy re-tracked by the pYIN oracle), every ValueError of pitch_shift_batch and f0_ratio, the library's argument checks and the
kernels' registers."""
import ctypes
import os
import re
import shutil
import subprocess

import numpy as np
import pytest
import torch

import pitch_oracle as P
import psola_oracle as O
from test_pitch_cpu import glide, noise, tone

SR, HOP = 22050, 275
SHIFTS = (-12, -7, -3, 3, 7, 12)
RETRACK_FMIN = 45.0          # a 100 Hz tone an octave down is below pitch_batch's default 65.406 Hz floor


def random_track(F, seed, flip=False):
    """A random f0 track (Hz, NaN unvoiced) of F frames: voiced runs of 70-800 Hz, or voicing that flips every frame."""
    rng = np.random.default_rng(seed)
    f = rng.uniform(70.0, 800.0, F).astype(np.float32)
    unvoiced = (np.arange(F) % 2 == 1) if flip else (rng.random(F) < 0.3)
    f[unvoiced] = np.nan
    return f


def cases():
    """(name, x, f0): the signals with their oracle pYIN tracks, and random tracks on tones and noise."""
    out = []
    for f in (80.0, 123.0, 200.0, 311.0, 400.0):
        out.append((f'tone{f:g}', tone(f, 0.3)))
    out += [('glide', glide(120.0, 180.0, 0.5)), ('noise', noise(0.3)), ('silence', np.zeros(3000)),
            ('tone-silence-tone', np.concatenate([tone(150.0, 0.2), np.zeros(2500), tone(250.0, 0.2)])), ('one sample', np.array([0.25]))]
    out = [(n, x, P.pyin(x, SR, HOP)[0].astype(np.float32)) for n, x in out]
    for seed, flip in ((1, False), (2, True), (3, False)):
        x = tone(150.0, 0.3) if seed != 3 else noise(0.3, seed=3)
        out.append((f'random track {seed}{" flips" if flip else ""}', x, random_track(1 + len(x) // HOP, seed, flip)))
    out.append(('random track, one sample', np.array([-0.5]), np.array([300.0], dtype=np.float32)))
    return out


CASES = cases()


@pytest.mark.parametrize('case', range(len(CASES)), ids=[c[0] for c in CASES])
def test_identity_at_ratio_one(case):
    _, x, f0 = CASES[case]
    y, info = O.pitch_shift(x, f0, np.ones(len(f0), np.float32), SR, HOP)
    x32 = x.astype(np.float32).astype(np.float64)
    assert np.abs(y - x32).max() <= 1e-12 * max(np.abs(x32).max(), 1e-30)
    np.testing.assert_array_equal(info['c'], info['marks'])
    np.testing.assert_array_equal(info['k'], np.arange(len(info['marks'])))


@pytest.mark.parametrize('case', range(len(CASES)), ids=[c[0] for c in CASES])
def test_all_unvoiced_is_identity_at_any_ratio(case):
    _, x, f0 = CASES[case]
    unvoiced = np.full_like(f0, np.nan)
    x32 = x.astype(np.float32).astype(np.float64)
    for r in (0.5, 0.8, 1.7, 2.0):
        y, info = O.pitch_shift(x, unvoiced, np.full(len(f0), r, np.float32), SR, HOP)
        assert np.abs(y - x32).max() <= 1e-12 * max(np.abs(x32).max(), 1e-30)
        assert (np.diff(info['marks']) == HOP).all()


@pytest.mark.parametrize('case', range(len(CASES)), ids=[c[0] for c in CASES])
def test_mark_invariants(case):
    _, x, f0 = CASES[case]
    L = len(x)
    Pf = O.periods(f0, SR)
    rng = np.random.default_rng(case)
    for ratio in (np.full(len(f0), 0.5, np.float32), np.full(len(f0), 2.0, np.float32), rng.uniform(0.5, 2.0, len(f0)).astype(np.float32)):
        marks, d, voiced, a0 = O.analysis_marks(x, f0, SR, HOP)
        assert marks[0] >= 0 and marks[-1] < L and (np.diff(marks) > 0).all()
        for i in range(len(marks) - 1):
            if voiced[i]:
                p = int(Pf[O.frame_of(int(marks[i]), HOP, len(f0))])
                c = marks[i] + p
                if Pf[O.frame_of(int(c), HOP, len(f0))]:
                    assert p - p // 4 <= d[i] <= p + p // 4, (i, p, d[i])
                else:
                    assert d[i] == p
        c, k = O.synthesis_marks(L, marks, d, voiced, ratio, HOP)
        assert c[0] == marks[0] and (c < L).all() and (np.diff(c) >= 0).all()
        dist = np.abs(marks[None, :] - c[:, None])
        np.testing.assert_array_equal(k, dist.argmin(1))          # nearest, and the lower on ties (argmin takes the first)
        y, _ = O.overlap_add(x, marks, d, a0, c, k)
        assert y.shape == (L,)
        assert np.abs(y).max() <= float(np.abs(x.astype(np.float32)).max()) * (1 + 1e-12)


def _uncovered(x, f0, r):
    marks, d, voiced, a0 = O.analysis_marks(x, f0, SR, HOP)
    c, k = O.synthesis_marks(len(x), marks, d, voiced, np.full(len(f0), r, np.float32), HOP)
    _, den = O.overlap_add(x, marks, d, a0, c, k)
    return np.flatnonzero(den == 0), int(d.max())


@pytest.mark.parametrize('r', [0.5, 0.6, 0.8, 1.0, 1.25, 1.6, 2.0])
def test_no_interior_sample_is_uncovered(r):
    """Below r = 1 the last grain can end before the waveform does; the interior, [0, L - 2 max d), is covered at every ratio on tones.
    On a glide at r = 0.5 grains of falling periods placed two periods apart can leave one sample between them (d_k > d_{k+1} + 1), the
    only interior gaps found; they are listed."""
    for f in (100.0, 150.0, 220.0, 300.0):
        x = tone(f, 0.5)
        gaps, dmax = _uncovered(x, P.pyin(x, SR, HOP)[0], r)
        assert (gaps >= len(x) - 2 * dmax).all(), (f, r, gaps)
    x = glide(120.0, 180.0, 1.0)
    gaps, dmax = _uncovered(x, P.pyin(x, SR, HOP)[0], r)
    interior = gaps[gaps < len(x) - 2 * dmax]
    print(f'glide 120->180 Hz at r = {r}: uncovered interior samples {interior.tolist()}, tail {gaps[len(interior):].tolist()[:3]}...')
    if r > 0.5:
        assert len(interior) == 0, (r, interior)
    else:
        assert len(interior) <= 3, interior


@pytest.mark.parametrize('f', [100.0, 150.0, 220.0, 300.0])
def test_shift_accuracy_retracked(f):
    x = tone(f, 0.5)
    f0 = P.pyin(x, SR, HOP)[0].astype(np.float32)
    F = len(f0)
    inner = slice(4, F - 4)
    before = P.pyin(x, SR, HOP, fmin=RETRACK_FMIN)[1][inner]
    for s in SHIFTS:
        y, _ = O.pitch_shift(x, f0, np.full(F, 2.0 ** (s / 12), np.float32), SR, HOP)
        g, voiced, _ = P.pyin(y, SR, HOP, fmin=RETRACK_FMIN)
        np.testing.assert_array_equal(voiced[inner], before)
        cents = np.abs(1200 * np.log2(g[inner][voiced[inner]] / (f * 2.0 ** (s / 12))))
        assert np.median(cents) <= 15.0, (f, s, np.median(cents))


# ---- ValueErrors -----------------------------------------------------------------------------------------------------------------------
def test_pitch_shift_batch_errors():
    from multilingual_text_to_speech_b200.utils import audio
    y = tone(150.0, 0.1).astype(np.float32)
    F = 1 + len(y) // HOP
    f0 = np.full(F, 150.0, np.float32)
    ones = np.ones(F, np.float32)
    bad_calls = [
        dict(waveforms=[], semitones=1.0), dict(waveforms='x', semitones=1.0), dict(waveforms=[np.zeros((2, 10))], semitones=1.0),
        dict(waveforms=[np.zeros(0)], semitones=1.0), dict(waveforms=[np.arange(10)], semitones=1.0),
        dict(waveforms=[np.array([0.0, np.nan])], semitones=1.0, f0s=[np.array([100.0], np.float32)]),
        dict(waveforms=[y]), dict(waveforms=[y], semitones=1.0, ratios=[ones]),
        dict(waveforms=[y], semitones=[1.0, 2.0]), dict(waveforms=[y], semitones=12.5), dict(waveforms=[y], semitones=-13.0),
        dict(waveforms=[y], semitones=float('nan')), dict(waveforms=[y], semitones=float('inf')),
        dict(waveforms=[y], ratios=ones), dict(waveforms=[y], ratios=[ones, ones]), dict(waveforms=[y], ratios=[ones[:-1]]),
        dict(waveforms=[y], ratios=[np.concatenate([ones[:-1], [2.5]])]), dict(waveforms=[y], ratios=[ones * 0.49]),
        dict(waveforms=[y], ratios=[np.concatenate([ones[:-1], [np.nan]])]), dict(waveforms=[y], ratios=[np.ones((F, 1))]),
        dict(waveforms=[y], ratios=[np.ones(F, dtype=np.int32)]),
        dict(waveforms=[y], semitones=1.0, f0s=[f0[:-1]]), dict(waveforms=[y], semitones=1.0, f0s=[f0, f0]),
        dict(waveforms=[y], semitones=1.0, f0s=f0), dict(waveforms=[y], semitones=1.0, f0s=[-f0]),
        dict(waveforms=[y], semitones=1.0, f0s=[f0 * 0]), dict(waveforms=[y], semitones=1.0, f0s=[f0 * np.inf]),
        dict(waveforms=[y], semitones=1.0, f0s=[np.full(F, 20.0, np.float32)]),        # period 1,102 > 1,024
        dict(waveforms=[y], semitones=1.0, f0s=[np.full(F, 15000.0, np.float32)]),     # period 1 < 2
    ]
    for kw in bad_calls:
        with pytest.raises(ValueError):
            audio.pitch_shift_batch(**kw)
    with pytest.raises(ValueError):
        audio.pitch_shift(np.zeros((3, 3)), semitones=1.0)
    with pytest.raises(ValueError):
        audio.pitch_shift(y, ratios=ones[:-1], f0=f0)


def test_f0_ratio():
    from multilingual_text_to_speech_b200.utils import audio
    nan = np.nan
    tgt = np.array([200.0, nan, 100.0, 1000.0, 10.0, 300.0])
    src = np.array([100.0, 100.0, nan, 100.0, 100.0])
    got = audio.f0_ratio(tgt, src)
    assert got.dtype == np.float32 and got.tolist() == [2.0, 1.0, 1.0, 2.0, 0.5]
    got = audio.f0_ratio(np.array([150.0, 120.0]), torch.tensor([100.0, 100.0, 100.0]))
    assert torch.is_tensor(got) and got.tolist() == [1.5, 1.2000000476837158, 1.0]
    for a, b in ((np.zeros((2, 2)), src), (tgt, np.array([], dtype=np.float64)), (np.array([1, 2]), src), (tgt, np.array([100.0, -1.0])),
                 (np.array([np.inf]), src), (tgt, np.array([0.0]))):
        with pytest.raises(ValueError):
            audio.f0_ratio(a, b)


# ---- the library -----------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope='module')
def lib():
    import __graft_entry__ as entry
    entry.build()
    from multilingual_text_to_speech_b200 import _lib
    return _lib.load()


def _shape(**kw):
    from multilingual_text_to_speech_b200 import _lib
    s = _lib.PsolaShape(2, 4000, 16, 275, 275, 22050.0)
    for k, v in kw.items():
        setattr(s, k, v)
    return s


def test_library_argument_checks(lib):
    good = _shape()
    assert lib.b200tts_psola_workspace_bytes(ctypes.byref(good)) == 2 * 16 + 4000 * 17
    for kw, msg in ((dict(B=0), b'B >= 1'), (dict(total_samples=1), b'B >= 1'), (dict(total_frames=1), b'B >= 1'), (dict(hop=0), b'hop'),
                    (dict(unvoiced_spacing=0), b'unvoiced_spacing'), (dict(unvoiced_spacing=1025), b'unvoiced_spacing'),
                    (dict(sr=0.0), b'sr'), (dict(sr=float('inf')), b'sr')):
        assert lib.b200tts_psola_workspace_bytes(ctypes.byref(_shape(**kw))) == 0, kw
        assert msg in lib.b200tts_last_error(), (kw, lib.b200tts_last_error())
    assert lib.b200tts_psola_workspace_bytes(None) == 0
    x = torch.zeros(64, dtype=torch.float64)
    p = ctypes.c_void_p(x.data_ptr())
    assert lib.b200tts_psola_marks(None, p, p, p, p, p, p, 1 << 20, None) != 0
    assert lib.b200tts_psola_marks(ctypes.byref(good), p, None, p, p, p, p, 1 << 20, None) != 0 and b'null' in lib.b200tts_last_error()
    assert lib.b200tts_psola_marks(ctypes.byref(good), p, p, p, p, p, p, 10, None) != 0 and b'workspace' in lib.b200tts_last_error()
    assert lib.b200tts_psola_overlap_add(ctypes.byref(good), p, p, p, 10, ctypes.c_void_p(x.data_ptr() + 8), None) != 0
    assert b'workspace' in lib.b200tts_last_error()
    assert lib.b200tts_psola_overlap_add(ctypes.byref(good), p, p, p, 1 << 20, p, None) != 0 and b'alias' in lib.b200tts_last_error()
    assert lib.b200tts_psola_overlap_add(ctypes.byref(_shape(hop=0)), p, p, p, 1 << 20, p, None) != 0


@pytest.mark.skipif(torch.cuda.is_available(), reason='checks the no-GPU failure mode')
def test_calls_without_gpu_fail_loudly(lib):
    good = _shape()
    x = torch.zeros(1 << 16, dtype=torch.float64)
    p = ctypes.c_void_p(x.data_ptr())
    q = ctypes.c_void_p(x.data_ptr() + 8)
    assert lib.b200tts_psola_marks(ctypes.byref(good), p, p, p, p, p, p, x.numel() * 8, None) != 0
    assert lib.b200tts_psola_overlap_add(ctypes.byref(good), p, p, p, x.numel() * 8, q, None) != 0
    from multilingual_text_to_speech_b200 import _lib
    from multilingual_text_to_speech_b200.utils import audio
    y = np.zeros(2000, dtype=np.float32)
    with pytest.raises((_lib.B200TTSError, RuntimeError, AssertionError)):
        audio.pitch_shift_batch([y], semitones=3.0, f0s=[np.full(1 + 2000 // HOP, 150.0, np.float32)])


# measured (CUDA 12.9, sm_90a, -Xptxas -v): registers of each kernel; none spills or keeps a stack frame
PSOLA_REGS = {'psola_marks_kernel': 48, 'psola_ola_kernel': 39}


def test_kernel_registers_and_spills():
    from multilingual_text_to_speech_b200 import build
    nvcc = next((c for c in (os.environ.get('NVCC'), '/usr/local/cuda/bin/nvcc', shutil.which('nvcc')) if c and os.path.exists(c)), None)
    if nvcc is None:
        pytest.skip('nvcc not available')
    import tempfile
    with tempfile.TemporaryDirectory() as tmp:
        cmd = [nvcc] + build.NVCC_FLAGS + ['-I', os.path.join(build.ROOT, 'include'), '-Xptxas', '-v', '-cubin',
               os.path.join(build.CSRC, 'psola.cu'), '-o', os.path.join(tmp, 'psola.cubin')]
        res = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    assert res.returncode == 0, res.stdout
    for name, regs in PSOLA_REGS.items():
        m = re.search(r'Function properties for \S*' + name + r'\S*\n\s*(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes '
                      r'spill loads\n[^\n]*Used (\d+) registers', res.stdout)
        assert m, (name, res.stdout)
        stack, st, ld, used = map(int, m.groups())
        assert (stack, st, ld) == (0, 0, 0), (name, stack, st, ld)
        assert used <= regs, (name, used)
