"""Forced synthesis (durations= / alignments=) without a GPU: durations_to_alignment against brute force and against the monotonic
path of Tacotron.align, the scale_durations rule, every ValueError of the public entry points, the library's argument checks and the
registers of attn_forced_fwd_kernel."""
import ctypes
import os
import re
import subprocess

import numpy as np
import pytest
import torch

import align_oracle as AO
import forced_synthesis_oracle as FO
from multilingual_text_to_speech_b200 import _lib, build
from multilingual_text_to_speech_b200 import functional as F
from multilingual_text_to_speech_b200.params.params import Params as hp
from multilingual_text_to_speech_b200.modules import tacotron2 as T
from test_wavernn_cpu import _nvcc


@pytest.fixture
def params():
    hp.reset()
    yield hp
    hp.reset()


@pytest.mark.parametrize('r', [1, 2, 4])
def test_durations_to_alignment_matches_brute_force(r):
    rng = np.random.default_rng(r)
    cases = [[1], [3], [0, 2], [2, 0, 0, 1], [0, 0, 5, 0]] + [list(rng.integers(0, 6, size=n)) for n in (1, 7, 30, 64) for _ in range(5)]
    for d in cases:
        if sum(d) == 0:
            continue
        got = F.durations_to_alignment(torch.tensor(d, dtype=torch.int32), r)
        want = FO.brute_rows(d, r)
        assert got.dtype == torch.float32 and got.shape == (-(-sum(d) // r), len(d)), (d, r)
        assert np.array_equal(got.numpy(), want), (d, r)
        assert not got[:, np.asarray(d) == 0].any(), (d, r)           # a symbol without frames is never attended
    assert np.array_equal(F.durations_to_alignment([2, 1], r).numpy(), FO.brute_rows([2, 1], r))


@pytest.mark.parametrize('r', [1, 2, 3])
def test_align_durations_round_trip(r):
    """Tacotron.align's durations (step durations times r, the last symbol cut to the target) give back the search's path."""
    rng = np.random.default_rng(10 + r)
    for _ in range(20):
        L = int(rng.integers(1, 12))
        S = int(rng.integers(L, 3 * L + 2))
        frames = int(rng.integers((S - 1) * r + 1, S * r + 1))
        P = rng.dirichlet(np.ones(L), size=S)
        step_d, _, path = AO.mas(P, L, S)
        d = step_d.astype(np.int64) * r
        d[-1] -= S * r - frames
        assert d.sum() == frames and (d >= 1).all()
        got = F.durations_to_alignment(torch.from_numpy(d), r).numpy()
        assert got.shape == (S, L)
        assert np.array_equal(got, np.eye(L)[path])


def test_scale_durations_rule():
    d = torch.tensor([3, 0, 5, 2, 7], dtype=torch.int32)
    for f in (0.37, 0.5, 1.0, 1.25, 2.0, 3.3):
        got = F.scale_durations(d, f)
        assert got.dtype == torch.int32
        bounds = np.floor(f * np.cumsum(d.numpy()).astype(np.float64) + 0.5)
        assert np.array_equal(got.numpy(), np.diff(bounds, prepend=0)), f
        assert int(got.sum()) == int(bounds[-1]) and (got >= 0).all()
    assert torch.equal(F.scale_durations(d, 1.0), d)
    assert int(F.scale_durations(torch.tensor([1, 1, 1, 1]), 0.3).eq(0).sum()) >= 2     # strong speed-ups drop symbols to 0 frames
    assert F.scale_durations(np.array([4, 4]), 0.5).tolist() == [2, 2]
    for bad in (0.0, -1.0, float('nan'), float('inf')):
        with pytest.raises(ValueError, match='factor'):
            F.scale_durations(d, bad)
    with pytest.raises(ValueError, match='0 frames'):
        F.scale_durations(torch.tensor([1, 0]), 0.4)
    with pytest.raises(ValueError, match='integer'):
        F.scale_durations(torch.tensor([1.0, 2.0]), 2.0)
    with pytest.raises(ValueError, match='>= 0'):
        F.scale_durations(torch.tensor([1, -2]), 2.0)


def test_durations_to_alignment_errors():
    with pytest.raises(ValueError, match='0 frames'):
        F.durations_to_alignment(torch.tensor([0, 0]), 1)
    with pytest.raises(ValueError, match='r must be'):
        F.durations_to_alignment(torch.tensor([1]), 0)
    with pytest.raises(ValueError, match='1-D integer'):
        F.durations_to_alignment(torch.ones(2, 2, dtype=torch.int64), 1)


def _bad_plans(L, max_frames):
    d = torch.ones(L, dtype=torch.int64)
    a = torch.full((4, L), 0.25)
    nan = a.clone()
    nan[1, 0] = float('nan')
    return [
        (dict(durations=d, alignment=a), 'not both'),
        (dict(durations=torch.ones(L, dtype=torch.float32)), 'integer'),
        (dict(durations=torch.ones(1, L, dtype=torch.int64)), 'integer'),
        (dict(durations=torch.ones(L + 1, dtype=torch.int64)), 'durations for a text'),
        (dict(durations=torch.tensor([-1] + [2] * (L - 1))), '>= 0'),
        (dict(durations=torch.zeros(L, dtype=torch.int64)), '0 frames'),
        (dict(durations=torch.full((L,), max_frames, dtype=torch.int64)), 'max_output_length'),
        (dict(alignment=torch.ones(4, L, dtype=torch.int64)), 'float tensor'),
        (dict(alignment=torch.ones(4 * L)), 'float tensor'),
        (dict(alignment=torch.ones(4, L + 2)), 'symbols for a text'),
        (dict(alignment=nan), 'finite'),
        (dict(alignment=-a), 'finite and >= 0'),
        (dict(alignment=torch.ones(0, L)), '0 frames'),
        (dict(alignment=torch.ones(max_frames + 1, L)), 'max_output_length'),
    ]


def test_every_entry_point_raises(params):
    """Each malformed plan fails in every entry point before any device work (the model lives on the CPU here)."""
    from multilingual_text_to_speech_b200.modules.streaming import SpeechServer, speech_stream, speech_streams
    hp.max_output_length = 50
    model = T.Tacotron().eval()
    text = torch.tensor([3, 4, 5, 6, 7])
    pool = model.decoder_pool()

    class _Voc:
        def stream_pool(self, *a):
            return None

        def generate_stream(self, mels, *a):
            yield from mels
    for kw, match in _bad_plans(5, 50):
        one = {'durations' if k == 'durations' else 'alignment': v for k, v in kw.items()}
        many = {('durations' if k == 'durations' else 'alignments'): [None, v] for k, v in kw.items()}
        calls = [lambda: model.inference(text, **one),
                 lambda: model.inference_batch([text[:3], text], **many),
                 lambda: next(model.inference_stream(text, **one)),
                 lambda: next(model.inference_streams([text[:3], text], **many)),
                 lambda: pool.check(text, **one),
                 lambda: pool.open(text, **one),
                 lambda: next(speech_stream(model, _Voc(), text, **one)),
                 lambda: next(speech_streams(model, _Voc(), [text[:3], text], **many))]
        for call in calls:
            with pytest.raises(ValueError, match=match):
                call()
    assert pool.ids == []
    server = SpeechServer(model, _Voc(), 2)
    for kw, match in _bad_plans(5, 50):
        with pytest.raises(ValueError, match=match):
            server.submit(text, **kw)
    assert server.pending == []
    with pytest.raises(ValueError, match='1 durations for 2 texts'):
        model.inference_batch([text, text], durations=[None])


def _shape(**kw):
    s = _lib.DecoderShape(2, 12, 8, 16, 24, 8, 8, 4, 5, 6, 0, 0, 0.1, 0.0, 0.5)
    for k, v in kw.items():
        setattr(s, k, v)
    return s


def test_library_argument_checks():
    lib = _lib.load()
    one = ctypes.c_void_p(16)
    P, O_, G = _lib.DecoderParams(), _lib.DecoderOutputs(), _lib.DecoderOutputGrads()
    s = _shape()
    for fields in (dict(forced_count=1, forced_rows=one, forced_alignment=one), dict(forced_rows=one), dict(forced_alignment=one)):
        I = _lib.DecoderInputs(**fields)
        assert lib.b200tts_decoder_forward(ctypes.byref(s), ctypes.byref(P), ctypes.byref(I), ctypes.byref(O_), one, 1, None) == -1
        assert b'decoder_forward: forced attention rows are for synthesis only' in lib.b200tts_last_error()
        assert lib.b200tts_decoder_backward(ctypes.byref(s), ctypes.byref(P), ctypes.byref(I), ctypes.byref(O_), ctypes.byref(G), one,
                                            one, 1, ctypes.byref(P), None, None) == -1
        assert b'decoder_backward: forced attention rows are for synthesis only' in lib.b200tts_last_error()
    st = _lib.DecoderState(*([one] * 8))
    chunk = lambda I: lib.b200tts_decoder_forward_chunk(ctypes.byref(s), ctypes.byref(P), ctypes.byref(I), ctypes.byref(O_),  # noqa: E731
                                                        ctypes.byref(st), 1, one, 1, None)
    for count in (-1, 3):
        assert chunk(_lib.DecoderInputs(forced_count=count, forced_rows=one, forced_alignment=one)) == -1
        assert b'forced_count %d outside [0, B=2]' % count in lib.b200tts_last_error()
    for fields in (dict(forced_count=1, forced_rows=one), dict(forced_count=2, forced_alignment=one), dict(forced_rows=one),
                   dict(forced_alignment=one)):
        assert chunk(_lib.DecoderInputs(**fields)) == -1
        assert b'given exactly when forced_count > 0' in lib.b200tts_last_error(), fields


# measured (CUDA 12.9, sm_90a): attn_forced_fwd_kernel 39 registers, no spills
FORCED_REG_BOUND = 48


def test_forced_kernel_registers_and_spills():
    nvcc = _nvcc()
    if nvcc is None:
        pytest.skip('nvcc not available')
    import tempfile
    with tempfile.TemporaryDirectory() as tmp:
        cmd = [nvcc] + build.NVCC_FLAGS + ['-I', os.path.join(build.ROOT, 'include'), '-Xptxas', '-v', '-cubin',
                                           os.path.join(build.CSRC, 'decoder_fwd.cu'), '-o', os.path.join(tmp, 'decoder_fwd.cubin')]
        res = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    assert res.returncode == 0, res.stdout
    m = re.search(r'Function properties for \S*attn_forced_fwd_kernel\S*\n\s*(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes '
                  r'spill loads\n[^\n]*Used (\d+) registers', res.stdout)
    assert m, res.stdout
    stack, st, ld, regs = map(int, m.groups())
    assert st == 0 and ld == 0 and stack == 0, m.group(0)
    assert regs <= FORCED_REG_BOUND, regs
