"""The waveform front end without a GPU: the resampling oracle against scipy.signal.resample_poly, the host's polyphase tables against the
flat filter, output lengths, the trimming oracle on cases with known answers (librosa is not installed here, so the oracle restates
librosa 0.7.0's effects.trim and has not been run against librosa itself), every ValueError of resample_batch and trim_silence_batch,
the library's argument checks and the kernels' registers."""
import ctypes
import itertools
import math
import os
import re
import shutil
import subprocess

import numpy as np
import pytest
import scipy.signal
import torch

import resample_oracle as O

SR = 22050
RATES = (8000, 11025, 16000, 22050, 24000, 32000, 44100, 48000, 96000)
PAIRS = [(a, b) for a, b in itertools.permutations(RATES, 2)]


def ratio(a, b):
    g = math.gcd(a, b)
    return b // g, a // g


@pytest.mark.parametrize('pair', PAIRS, ids=[f'{a}-{b}' for a, b in PAIRS])
def test_oracle_equals_scipy_resample_poly(pair):
    up, down = ratio(*pair)
    assert max(up, down) <= O.MAX_FACTOR
    rng = np.random.default_rng(up * 7919 + down)
    for L in (1, 2, 37, 2000 if max(up, down) > 400 else 6000):
        x = rng.standard_normal(L)
        want = scipy.signal.resample_poly(x, up, down)
        got, mag = O.resample(x, up, down)
        assert len(got) == len(want) == O.out_length(L, up, down)
        assert (np.abs(got - want) <= 1e-12 * mag + 1e-300).all(), (pair, L, np.abs(got - want).max())


def test_largest_ratio_is_within_the_limit():
    assert max(max(ratio(*p)) for p in PAIRS) == 1280 <= O.MAX_FACTOR
    assert ratio(11025, 96000) == (1280, 147) and ratio(11025, 32000) == (1280, 441)


@pytest.mark.parametrize('pair', [(48000, 22050), (16000, 22050), (22050, 16000), (44100, 22050), (22050, 44100), (11025, 96000),
                                  (96000, 8000), (1, 2048), (2048, 1)])
def test_host_polyphase_table_equals_the_flat_filter(pair):
    from multilingual_text_to_speech_b200.utils import audio
    up, down = audio.resample_ratio(*pair)
    table, h_len = audio.resample_taps(up, down)
    h, h_len_o = O.taps(up, down)
    T = -(-len(h) // up)
    assert h_len == h_len_o and table.shape == (up, T) and table.dtype == np.float64 and table.flags.c_contiguous
    for phase in range(0, up, max(1, up // 37)):
        n = len(h[phase::up])
        # firwin's sinc(fc n) and the closed form's sinc(n / m) round their arguments differently: a few ulps of the peak tap
        np.testing.assert_allclose(table[phase, :n], h[phase::up], rtol=1e-13, atol=1e-15 * np.abs(h).max())
        assert (table[phase, n:] == 0).all()


def test_output_lengths():
    for a, b in PAIRS:
        up, down = ratio(a, b)
        for L in (1, 2, 3, 100, 12345):
            assert O.out_length(L, up, down) == len(scipy.signal.resample_poly(np.zeros(L), up, down)) == math.ceil(L * up / down)


# ---- trimming oracle -------------------------------------------------------------------------------------------------------------------
W, HOP = 1102, 275                 # ms_to_frames(50), ms_to_frames(12.5) at 22,050 Hz


def quarter_tone(n):
    """sin(pi i / 2 + pi / 4) / 2: every sample is +-0.354, so any frame touching it is within 31 dB of the loudest."""
    return 0.5 * np.sin(np.pi / 2 * np.arange(n) + np.pi / 4)


def test_reflect_index_equals_numpy_pad():
    for L in (1, 2, 3, 5, 40, 700):
        x = np.arange(L, dtype=np.float64)
        for pad in (1, 3, 551, 2000):
            want = np.pad(x, pad, mode='reflect')
            got = x[O.reflect_index(np.arange(len(want)) - pad, L)]
            np.testing.assert_array_equal(got, want)


@pytest.mark.parametrize('lead,n,tail', [(5000, 3000, 7000), (0, 4000, 2000), (3000, 800, 0), (551, 275, 552), (20000, 1, 20000)])
def test_tone_between_digital_silences(lead, n, tail):
    """Frames that touch a tone sample are non-silent and the others are exactly silent, so the bounds follow from the lengths."""
    x = np.concatenate([np.zeros(lead), quarter_tone(n), np.zeros(tail)])
    L, p = len(x), W // 2
    F = 1 + (L + 2 * p - W) // HOP
    # frame f reads x[f hop - p, f hop - p + W): it touches [lead, lead + n) when f hop > lead - W + p - 1 and f hop <= lead + n - 1 + p
    a = max(0, -(-(lead - W + 1 + p) // HOP))
    b = min(F - 1, (lead + n - 1 + p) // HOP)
    if lead <= p or tail <= p:
        # within W // 2 of an end the padding mirrors the tone back in, and frames touching the mirror image count too
        touched = [f for f in range(F) if (np.abs(x[O.reflect_index(np.arange(W) + f * HOP - p, L)]) > 0).any()]
        a, b = touched[0], touched[-1]
    (start, end), _ = O.trim(x, W, HOP, top_db=50)
    assert (start, end) == (a * HOP, min(L, (b + 1) * HOP))
    assert start <= lead and end >= lead + n


def test_all_zero_input_comes_back_whole():
    for L in (1, 7, 1000, 30000):
        (start, end), db = O.trim(np.zeros(L), W, HOP)
        assert (start, end) == (0, L) and (db == 0).all()


def test_single_sample():
    (start, end), db = O.trim(np.array([0.3]), W, HOP)
    assert (start, end) == (0, 1) and len(db) == 1
    np.testing.assert_allclose(O.frame_power(np.array([0.3]), W, HOP), [0.09], rtol=1e-15)


def test_signal_shorter_than_half_a_frame_reflects_repeatedly():
    x = np.array([0.0, 0.0, 0.0, 0.0, 1.0])
    # padded by 551 on each side, x repeats with period 8 as 0 0 0 0 1 0 0 0: every W-sample frame holds 1102 / 8 ones, near enough
    p = O.frame_power(x, W, HOP)
    padded = np.pad(x, W // 2, mode='reflect')
    want = np.array([np.mean(padded[f * HOP:f * HOP + W] ** 2) for f in range(len(p))])
    np.testing.assert_allclose(p, want, rtol=1e-15)
    assert len(p) == 1 + (5 + 2 * 551 - W) // HOP
    assert O.trim(x, W, HOP)[0] == (0, 5)


def test_margin_crop():
    """Bursts inside the margins are cut away before the decision, and the index is relative to the cropped signal."""
    M = 2205
    x = np.concatenate([quarter_tone(M), np.zeros(8000), quarter_tone(3000), np.zeros(8000), quarter_tone(M)])
    (start, end), _ = O.trim(x, W, HOP, margin=M)
    (s0, e0), _ = O.trim(x[M:-M], W, HOP)
    assert (start, end) == (s0, e0) and 0 < start <= 8000 and 11000 <= end < 19000
    (start, end), _ = O.trim(x, W, HOP)
    assert (start, end) == (0, len(x))


@pytest.mark.parametrize('top_db', [0.0, -5.0])
def test_no_frame_is_non_silent_at_non_positive_top_db(top_db):
    x = np.concatenate([np.zeros(3000), quarter_tone(3000)])
    assert O.trim(x, W, HOP, top_db=top_db)[0] == (0, 0)


# ---- ValueErrors -----------------------------------------------------------------------------------------------------------------------
def test_resample_batch_errors():
    from multilingual_text_to_speech_b200.utils import audio
    y = np.zeros(1000, dtype=np.float32)
    bad_calls = [
        dict(waveforms=[], orig_sr=16000), dict(waveforms='x', orig_sr=16000), dict(waveforms=[np.zeros((2, 10))], orig_sr=16000),
        dict(waveforms=[np.zeros(0)], orig_sr=16000), dict(waveforms=[np.arange(10)], orig_sr=16000),
        dict(waveforms=[np.array([0.0, np.nan])], orig_sr=16000), dict(waveforms=[np.array([0.0, -np.inf])], orig_sr=16000),
        dict(waveforms=[y], orig_sr=0), dict(waveforms=[y], orig_sr=-16000), dict(waveforms=[y], orig_sr=16000.0),
        dict(waveforms=[y], orig_sr='16000'), dict(waveforms=[y], orig_sr=True), dict(waveforms=[y], orig_sr=None),
        dict(waveforms=[y], orig_sr=16000, target_sr=0), dict(waveforms=[y], orig_sr=16000, target_sr=22050.5),
        dict(waveforms=[y, y], orig_sr=[16000]), dict(waveforms=[y], orig_sr=[16000, 22050]), dict(waveforms=[y, y], orig_sr=[16000, 0]),
        dict(waveforms=[y], orig_sr=4099, target_sr=2), dict(waveforms=[y], orig_sr=1, target_sr=2049),
        dict(waveforms=[y, y], orig_sr=[16000, 22051]),                                      # 22050 / 22051: factor 22051
        dict(waveforms=[np.zeros(1 << 20, dtype=np.float32)], orig_sr=1, target_sr=2048),   # 2^31 output samples
    ]
    for kw in bad_calls:
        with pytest.raises(ValueError):
            audio.resample_batch(**kw)
    with pytest.raises(ValueError, match='2049/1'):
        audio.resample_batch([y], 1, 2049)
    with pytest.raises(ValueError):
        audio.resample(np.zeros((3, 3)), 16000)
    with pytest.raises(ValueError):
        audio.resample(torch.zeros(100, dtype=torch.int32), 16000)


def test_trim_silence_batch_errors():
    from multilingual_text_to_speech_b200.utils import audio
    y = np.zeros(5000, dtype=np.float32)
    bad_calls = [
        dict(waveforms=[], window_ms=50, hop_ms=12.5), dict(waveforms=[np.zeros((2, 10))], window_ms=50, hop_ms=12.5),
        dict(waveforms=[np.zeros(0)], window_ms=50, hop_ms=12.5), dict(waveforms=[np.arange(10)], window_ms=50, hop_ms=12.5),
        dict(waveforms=[np.array([0.0, np.nan])], window_ms=50, hop_ms=12.5), dict(waveforms=[y], window_ms=0, hop_ms=12.5),
        dict(waveforms=[y], window_ms=50, hop_ms=0.01), dict(waveforms=[y], window_ms=-5, hop_ms=12.5),
        dict(waveforms=[y], window_ms=50, hop_ms=12.5, top_db=float('nan')), dict(waveforms=[y], window_ms=50, hop_ms=12.5, top_db=np.inf),
        dict(waveforms=[y], window_ms=50, hop_ms=12.5, margin_ms=-1),
        dict(waveforms=[y, np.zeros(100)], window_ms=50, hop_ms=12.5, margin_ms=5),       # 2 x 110 >= 100 samples
        dict(waveforms=[np.zeros(220)], window_ms=50, hop_ms=12.5, margin_ms=5),          # 2 x 110 = 220
    ]
    for kw in bad_calls:
        with pytest.raises(ValueError):
            audio.trim_silence_batch(**kw)
    with pytest.raises(ValueError):
        audio.trim_silence(np.zeros((3, 3)), 50, 12.5)


def test_duration():
    from multilingual_text_to_speech_b200.utils import audio
    assert audio.duration(np.zeros(SR * 3)) == 3.0 and audio.duration(torch.zeros(SR // 2)) == 0.5


# ---- the library -----------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope='module')
def lib():
    import __graft_entry__ as entry
    entry.build()
    from multilingual_text_to_speech_b200 import _lib
    return _lib.load()


def _rshape(**kw):
    from multilingual_text_to_speech_b200 import _lib
    s = _lib.ResampleShape(2, 4000, 3000, 6468, 320)
    for k, v in kw.items():
        setattr(s, k, v)
    return s


def _tshape(**kw):
    from multilingual_text_to_speech_b200 import _lib
    s = _lib.TrimShape(2, 4000, 30, W, HOP, 50.0)
    for k, v in kw.items():
        setattr(s, k, v)
    return s


def test_library_argument_checks(lib):
    x = torch.zeros(64, dtype=torch.float64)
    p = ctypes.c_void_p(x.data_ptr())
    q = ctypes.c_void_p(x.data_ptr() + 16)
    r = ctypes.c_void_p(x.data_ptr() + 32)
    for kw, msg in ((dict(B=0), b'B >= 1'), (dict(total_samples=1), b'B >= 1'), (dict(total_out_samples=1), b'B >= 1'),
                    (dict(total_taps=0), b'B >= 1'), (dict(max_factor=0), b'max_factor'), (dict(max_factor=2049), b'max_factor')):
        assert lib.b200tts_resample(ctypes.byref(_rshape(**kw)), p, p, p, p, q, r, None) != 0, kw
        assert msg in lib.b200tts_last_error(), (kw, lib.b200tts_last_error())
    good = ctypes.byref(_rshape())
    assert lib.b200tts_resample(None, p, p, p, p, q, r, None) != 0 and b'null' in lib.b200tts_last_error()
    for i in range(6):
        args = [p, p, p, p, q, r]
        args[i] = None
        assert lib.b200tts_resample(good, *args, None) != 0 and b'null' in lib.b200tts_last_error(), i
    assert lib.b200tts_resample(good, p, p, p, p, q, p, None) != 0 and b'alias' in lib.b200tts_last_error()
    assert lib.b200tts_resample(good, p, p, p, p, q, q, None) != 0 and b'alias' in lib.b200tts_last_error()
    assert lib.b200tts_resample(good, p, p, p, ctypes.c_void_p(x.data_ptr() + 4), q, r, None) != 0
    assert b'aligned' in lib.b200tts_last_error()

    for kw, msg in ((dict(B=0), b'B >= 1'), (dict(total_samples=1), b'B >= 1'), (dict(total_frames=1), b'B >= 1'),
                    (dict(frame_length=0), b'frame_length'), (dict(hop=0), b'hop'), (dict(top_db=float('nan')), b'top_db'),
                    (dict(top_db=float('-inf')), b'top_db')):
        assert lib.b200tts_trim_silence(ctypes.byref(_tshape(**kw)), p, p, p, q, r, None) != 0, kw
        assert msg in lib.b200tts_last_error(), (kw, lib.b200tts_last_error())
    good = ctypes.byref(_tshape())
    assert lib.b200tts_trim_silence(None, p, p, p, q, r, None) != 0 and b'null' in lib.b200tts_last_error()
    for i in range(5):
        args = [p, p, p, q, r]
        args[i] = None
        assert lib.b200tts_trim_silence(good, *args, None) != 0 and b'null' in lib.b200tts_last_error(), i
    for args in ([p, p, p, p, r], [p, p, p, q, p], [p, p, p, q, q]):
        assert lib.b200tts_trim_silence(good, *args, None) != 0 and b'alias' in lib.b200tts_last_error()


@pytest.mark.skipif(torch.cuda.is_available(), reason='checks the no-GPU failure mode')
def test_calls_without_gpu_fail_loudly(lib):
    x = torch.zeros(1 << 16, dtype=torch.float64)
    p = ctypes.c_void_p(x.data_ptr())
    q = ctypes.c_void_p(x.data_ptr() + 16)
    r = ctypes.c_void_p(x.data_ptr() + 32)
    assert lib.b200tts_resample(ctypes.byref(_rshape()), p, p, p, p, q, r, None) != 0
    assert lib.b200tts_trim_silence(ctypes.byref(_tshape()), p, p, p, q, r, None) != 0
    from multilingual_text_to_speech_b200 import _lib
    from multilingual_text_to_speech_b200.utils import audio
    y = np.zeros(2000, dtype=np.float32)
    for call in (lambda: audio.resample_batch([y], 16000), lambda: audio.resample_batch([y], 22050),
                 lambda: audio.trim_silence_batch([y], 50, 12.5)):
        with pytest.raises((_lib.B200TTSError, RuntimeError, AssertionError)):
            call()


# measured (CUDA 12.9, sm_90a, -Xptxas -v): registers of each kernel; none spills or keeps a stack frame
FRONT_END_REGS = {'resample.cu': {'resample_kernel': 32}, 'trim.cu': {'trim_power_kernel': 30, 'trim_bounds_kernel': 32}}


@pytest.mark.parametrize('source', sorted(FRONT_END_REGS))
def test_kernel_registers_and_spills(source):
    from multilingual_text_to_speech_b200 import build
    nvcc = next((c for c in (os.environ.get('NVCC'), '/usr/local/cuda/bin/nvcc', shutil.which('nvcc')) if c and os.path.exists(c)), None)
    if nvcc is None:
        pytest.skip('nvcc not available')
    import tempfile
    with tempfile.TemporaryDirectory() as tmp:
        cmd = [nvcc] + build.NVCC_FLAGS + ['-I', os.path.join(build.ROOT, 'include'), '-Xptxas', '-v', '-cubin',
               os.path.join(build.CSRC, source), '-o', os.path.join(tmp, 'k.cubin')]
        res = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    assert res.returncode == 0, res.stdout
    for name, regs in FRONT_END_REGS[source].items():
        m = re.search(r'Function properties for \S*' + name + r'\S*\n\s*(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes '
                      r'spill loads\n[^\n]*Used (\d+) registers', res.stdout)
        assert m, (name, res.stdout)
        stack, st, ld, used = map(int, m.groups())
        assert (stack, st, ld) == (0, 0, 0), (name, stack, st, ld)
        assert used <= regs, (name, used)
