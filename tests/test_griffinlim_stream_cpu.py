"""CPU checks of streaming Griffin-Lim (RTISI-LA): the oracle's chunking invariance and output length, its quality against batch
Griffin-Lim, the fp32 rounding drift that sets the GPU tolerance, the argument checks (all before any device work), the workspace query,
the no-GPU failure mode and the register report of csrc/vocoder_stream.cu."""
import ctypes
import os
import re
import shutil
import subprocess

import numpy as np
import pytest
import torch

import __graft_entry__ as entry
import audio_oracle as O
import griffinlim_stream_oracle as G
from gl_stream_slot import GlLayout
from multilingual_text_to_speech_b200 import _lib, build
from multilingual_text_to_speech_b200 import functional as F
from multilingual_text_to_speech_b200.modules.griffinlim import GriffinLimVocoder
from test_vocoder_cpu import _harmonic

N, HOP, WIN = 1102, 275, 1102

# How far rounding alone moves the streaming inversion, as GL_DRIFT_FACTOR does for batch Griffin-Lim: the GPU tests allow this many
# times the drift the fp32 oracle shows against the fp64 one on their own input.  test_fp32_rounding_drift records that drift on the
# harmonic signal (about 1.4e-4 over 199 frames).  The kernels' fp32 arithmetic differs from the fp32 oracle's (FFT order, fused
# multiply-adds) about as much as either differs from fp64, so the same margin as the batch vocoder's applies.
GL_STREAM_DRIFT_FACTOR = 10.0


@pytest.fixture(scope='module')
def lib():
    entry.build()
    return _lib.load()


def _chirp(n, seed=0):
    """100 -> 2100 Hz linear chirp, 3 Hz amplitude modulation, 5 % white noise."""
    rng = np.random.default_rng(seed)
    t = np.arange(n) / 22050
    f = 100 + 2000 * t / t[-1]
    return (0.5 + 0.5 * np.sin(2 * np.pi * 3 * t)) * np.sin(2 * np.pi * np.cumsum(f) / 22050) + 0.05 * rng.standard_normal(n)


def _mag(y):
    return np.abs(O.stft(y, N, HOP, WIN))


@pytest.mark.parametrize('lookahead', [0, 1, 3])
@pytest.mark.parametrize('dtype', [np.float64, np.float32])
def test_oracle_chunked_equals_one_shot(dtype, lookahead):
    S = _mag(_harmonic(HOP * 40))
    kw = dict(lookahead=lookahead, iters=4, dtype=dtype)
    whole = G.rtisi(S, N, HOP, WIN, **kw)
    assert whole.shape == (HOP * 40,) and whole.dtype == dtype
    rng = np.random.default_rng(0)
    for _ in range(3):
        cuts = sorted(set(rng.integers(1, 41, 6).tolist()) | {41})
        assert np.array_equal(G.rtisi_chunked(S, cuts, N, HOP, WIN, **kw), whole), cuts
    # one frame at a time; every frame before the end is known (with lookahead 0 the last frame is committed before it: the run that
    # learns of the end releases the rest); and a stream of two frames
    assert np.array_equal(G.rtisi_chunked(S, list(range(1, 42)), N, HOP, WIN, **kw), whole)
    assert np.array_equal(G.rtisi_chunked(S, [41], N, HOP, WIN, **kw), whole)
    assert G.rtisi(S[:, :2], N, HOP, WIN, **kw).shape == (HOP,)
    assert G.rtisi_chunked(S[:, :2], [2], N, HOP, WIN, **kw).shape == (HOP,)


def test_oracle_releases_k_frames_plus_half_a_window_behind():
    st = G.Stream(N, HOP, WIN, lookahead=3, iters=2)
    S = _mag(_harmonic(HOP * 20))
    got = []
    for t in range(21):
        st.feed(S[:, t:t + 1])
        got.append(len(st.run()))
    # frame m is committed once frame m + 3 has arrived; then the output below (m + 1) hop - N/2 is final
    assert got == [max(0, (t - 2) * HOP - N // 2) - max(0, (t - 3) * HOP - N // 2) for t in range(21)]


@pytest.mark.parametrize('signal', ['harmonic', 'chirp'])
def test_quality_against_batch_griffinlim(signal):
    y = _harmonic(HOP * 198) if signal == 'harmonic' else _chirp(HOP * 198)
    S = _mag(y)
    u = np.random.default_rng(1).uniform(0, 1, S.shape)
    sc_gl = O.spectral_convergence(S, O.griffinlim(S, u, 60, N, HOP, WIN), N, HOP, WIN)
    sc = O.spectral_convergence(S, G.rtisi(S, N, HOP, WIN), N, HOP, WIN)
    assert sc <= 1.6 * sc_gl, (sc, sc_gl)
    if signal == 'chirp':
        # iterating pays: 0.06 against 0.15 (on the harmonic signal a single iteration already lands at 0.060, 32 at 0.068: DESIGN)
        assert sc < O.spectral_convergence(S, G.rtisi(S, N, HOP, WIN, iters=1), N, HOP, WIN)


def test_fp32_rounding_drift():
    S = _mag(_harmonic(HOP * 198))
    y64 = G.rtisi(S, N, HOP, WIN)
    y32 = G.rtisi(S, N, HOP, WIN, dtype=np.float32)
    drift = np.linalg.norm(y64 - y32) / np.linalg.norm(y64)
    assert 1e-6 < drift < 1e-3, drift


def _no_device(monkeypatch):
    def fail(*a, **k):
        raise AssertionError('device work before the argument checks')
    for name in ('gl_stream_workspace', 'gl_stream_reset', 'gl_stream_run', 'spectrogram_magnitude'):
        monkeypatch.setattr(F, name, fail)


def test_stream_value_errors_come_before_any_device_work(lib, monkeypatch):
    _no_device(monkeypatch)
    for kw in (dict(lookahead=-1), dict(iters=0), dict(lookahead=1.5), dict(iters=True), dict(lookahead=_lib.GL_STREAM_MAX_LOOKAHEAD + 1)):
        with pytest.raises(ValueError):
            GriffinLimVocoder(**kw)
    from multilingual_text_to_speech_b200.params.params import Params as hp
    try:
        hp.num_fft = 1101                      # odd: the FFT plan rejects it
        with pytest.raises(ValueError, match='unsupported FFT size'):
            GriffinLimVocoder()
    finally:
        hp.reset()
    voc = GriffinLimVocoder()
    ok = np.zeros((80, 4), np.float32)
    for kw in (dict(uniforms=np.zeros((1, 10, 1))), dict(target=100), dict(overlap=10), dict(preemphasis=1.0)):
        with pytest.raises(ValueError):
            next(voc.generate_stream([ok], **kw))
    for chunk in (np.zeros((81, 4), np.float32), np.zeros((80, 4), np.int32), np.zeros(80, np.float32)):
        with pytest.raises(ValueError):
            next(voc.generate_stream([chunk]))
    with pytest.raises(ValueError, match='at least 2'):
        next(voc.generate_stream([np.zeros((80, 1), np.float32)]))
    with pytest.raises(ValueError, match='at least 2'):
        next(voc.generate_stream([]))
    for bad in (0, 65, True):
        with pytest.raises(ValueError):
            voc.stream_pool(bad)
    with pytest.raises(ValueError):
        voc.stream_pool(2, target=10, overlap=2)
    with pytest.raises(ValueError):
        voc.stream_pool(2, preemphasis=-1.0)
    pool = voc.stream_pool(2)
    assert voc.lookahead() == 3 and pool.check_tape(None) is None
    with pytest.raises(ValueError, match='draws nothing'):
        pool.check_tape(np.zeros((1, 10, 1)))
    a = pool.open(seed=3)
    with pytest.raises(ValueError):
        pool.open(uniforms=np.zeros((1, 10, 1)))
    b = pool.open()
    with pytest.raises(ValueError, match='full'):
        pool.open()
    with pytest.raises(ValueError):
        pool.feed(a, np.zeros((552, 3), np.float32))
    pool.feed(a, ok[:, :1])
    with pytest.raises(ValueError, match='at least 2'):
        pool.end(a)
    pool.feed(a, ok)
    pool.end(a)
    with pytest.raises(ValueError, match='ended'):
        pool.feed(a, ok)
    with pytest.raises(ValueError, match='ended'):
        pool.end(a)
    for op in (lambda: pool.feed(99, ok), lambda: pool.end(99), lambda: pool.close(99)):
        with pytest.raises(ValueError, match='unknown'):
            op()
    pool.close(b)
    assert pool.open() == 2 and pool.rows == 2 and sorted(pool.streams) == [0, 2]


def test_workspace_query_and_validation(lib):
    def ws(**kw):
        s = dict(N=N, hop=HOP, win=WIN, lookahead=3, iters=32, slots=4, preemphasis=0.97)
        s.update(kw)
        return lib.b200tts_gl_stream_workspace_bytes(ctypes.byref(_lib.GLStreamShape(*s.values())))
    assert ws() == GlLayout(N, 3, 4).bytes
    for kw, msg in ((dict(N=1101), 'unsupported FFT size'), (dict(win=N + 1), 'window length'), (dict(hop=0), 'hop'),
                    (dict(lookahead=-1), 'lookahead'), (dict(lookahead=8), 'lookahead'), (dict(lookahead=0, hop=N // 2 + 1), 'lookahead 0'), (dict(iters=0), 'iters'), (dict(slots=0), 'slots'),
                    (dict(slots=65), 'slots'), (dict(preemphasis=1.0), 'preemphasis'), (dict(N=2048, win=2048, hop=512, lookahead=7), 'shared memory')):
        assert ws(**kw) == 0, kw
        assert msg.encode() in lib.b200tts_last_error(), (kw, lib.b200tts_last_error())


@pytest.mark.skipif(torch.cuda.is_available(), reason='checks the no-GPU failure mode')
def test_entry_points_fail_without_gpu(lib):
    shape = _lib.GLStreamShape(N, HOP, WIN, 3, 32, 2, 0.0)
    n = lib.b200tts_gl_stream_workspace_bytes(ctypes.byref(shape))
    buf = np.zeros(n + 256, np.uint8)
    base = ctypes.c_void_p((buf.ctypes.data + 255) // 256 * 256)
    assert lib.b200tts_gl_stream_reset(ctypes.byref(shape), base, n, (ctypes.c_int * 1)(0), 1, None) != 0
    row = _lib.GLStreamRow(0, 4, 1, 0, 0)
    out = np.zeros(4096, np.float32)
    assert lib.b200tts_gl_stream_run(ctypes.byref(shape), ctypes.byref(row), 1, out.ctypes.data, out.ctypes.data, base, n, None) != 0
    assert b'no CPU fallback' in lib.b200tts_last_error() or b'CUDA' in lib.b200tts_last_error()
    assert lib.b200tts_gl_stream_run(ctypes.byref(shape), ctypes.byref(row), 1, None, out.ctypes.data, base, n, None) != 0
    assert b'null argument' in lib.b200tts_last_error()
    voc = GriffinLimVocoder()
    with pytest.raises((_lib.B200TTSError, RuntimeError, AssertionError)):
        list(voc.generate_stream([np.zeros((80, 5), np.float32)]))


def test_stream_kernels_do_not_spill():
    nvcc = next((c for c in (os.environ.get('NVCC'), '/usr/local/cuda/bin/nvcc', shutil.which('nvcc')) if c and os.path.exists(c)), None)
    if nvcc is None:
        pytest.skip('nvcc not available')
    src = os.path.join(build.CSRC, 'vocoder_stream.cu')
    cmd = [nvcc] + build.NVCC_FLAGS + ['-I', os.path.join(build.ROOT, 'include'), '-Xptxas', '-v', '-cubin', src, '-o', os.devnull]
    res = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    assert res.returncode == 0, res.stdout
    found = re.findall(r'Function properties for \S*(gl_stream_\w+?_kernel)\S*\n\s*(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads',
                       res.stdout)
    assert {f[0] for f in found} == {'gl_stream_reset_kernel', 'gl_stream_run_kernel'}, found
    for name, stack, st, ld in found:
        assert stack == '0' and st == '0' and ld == '0', (name, stack, st, ld)
