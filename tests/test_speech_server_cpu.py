"""Continuous-batching synthesis without a GPU: the SpeechServer's admission, queue and cancel bookkeeping over stand-in pools; the decoder
rows' per-row step counters, re-padding and mask sources on host tensors with the library calls replaced by host models; the ValueErrors;
the argument checks of the three new entry points; the registers and spills of the new kernels."""
import ctypes
import os
import re
import subprocess

import numpy as np
import pytest
import torch

from multilingual_text_to_speech_b200 import _lib, build
from multilingual_text_to_speech_b200 import functional as F
from multilingual_text_to_speech_b200.modules import tacotron2 as T
from multilingual_text_to_speech_b200.modules.streaming import SpeechServer
from multilingual_text_to_speech_b200.params.params import Params as hp
from test_wavernn_cpu import _nvcc


# ---- the server over stand-in pools ----
class _Decoder:
    """DecoderPool stand-in: every text decodes `frames[text length]` frames, 8 per call, and leaves after its last call."""

    def __init__(self, frames):
        self.frames, self.rows, self.queue, self.next_id, self.calls = frames, {}, [], 0, []

    @property
    def ids(self):
        return self.queue + list(self.rows)

    def check(self, text, speaker=None, language=None, seed=None, masks=None):
        T.DecoderPool.check(_CHECKER, text, speaker, language, seed, masks)

    def open(self, text, speaker=None, language=None, seed=None, masks=None):
        tid = self.next_id
        self.next_id += 1
        self.queue.append(tid)
        self.rows[tid] = [self.frames[int(text.shape[0])], 0]
        return tid

    def close(self, tid):
        if tid not in self.rows:
            raise ValueError('unknown')
        del self.rows[tid]
        if tid in self.queue:
            self.queue.remove(tid)

    def run(self):
        self.queue = []
        self.calls.append(len(self.rows))
        out = {}
        for tid, row in list(self.rows.items()):
            n = min(8, row[0] - row[1])
            row[1] += n
            out[tid] = torch.zeros(80, n)
            if row[1] == row[0]:
                del self.rows[tid]
        return out


class _Pool:
    """StreamPool stand-in: a stream releases its whole mel's samples (1 per frame) at the second run() after end()."""

    def __init__(self, rows):
        self.rows, self.streams, self.next_sid = rows, {}, 0

    def open(self, uniforms=None, seed=None):
        assert len(self.streams) < self.rows
        sid = self.next_sid
        self.next_sid += 1
        self.streams[sid] = [0, False]
        return sid

    def close(self, sid):
        del self.streams[sid]

    def feed(self, sid, chunk):
        self.streams[sid][0] += chunk.shape[1]

    def end(self, sid):
        if self.streams[sid][0] < 21:
            raise ValueError(f'the mel stream ended after {self.streams[sid][0]} frames; the 20-hop fade-out needs at least 21')
        self.streams[sid][1] = 1

    def run(self):
        out = {sid: torch.zeros(st[0]) for sid, st in self.streams.items() if st[1] == 2}
        for sid in out:
            del self.streams[sid]
        for st in self.streams.values():
            st[1] += bool(st[1])
        return out


class _Voc:
    @staticmethod
    def _check_stream_tape(uniforms):
        return uniforms


def _server(rows, frames):
    s = SpeechServer.__new__(SpeechServer)
    s.decoder, s.pool, s.wavernn, s.mel_transform = _Decoder(frames), _Pool(rows), _Voc(), None
    s.requests, s.pending, s.failed, s.next_id = {}, [], {}, 0
    return s


_CHECKER = None


@pytest.fixture(autouse=True)
def _model():
    global _CHECKER
    hp.reset()
    torch.manual_seed(0)
    model = T.Tacotron()
    _CHECKER = T.DecoderPool(model, 4)
    yield model
    hp.reset()


def _text(n):
    return torch.full((n,), 5, dtype=torch.int64)


def test_admission_fifo_and_capacity():
    frames = {n: 21 + 3 * n for n in range(1, 80)}
    s = _server(64, frames)
    ids = [s.submit(_text(1 + i % 70)) for i in range(70)]
    assert s.pending == ids and s.active == []
    s.step()
    assert s.active == ids[:64] and s.pending == ids[64:]
    assert s.decoder.calls == [64]
    done = {}
    while s.pending or s.active:
        before = set(s.active)
        for rid, chunk in s.step().items():
            done[rid] = chunk.shape[0]
        assert len(s.active) <= 64
        # the queue is admitted in order as rows free up
        assert s.pending == ids[ids.index(s.pending[0]):] if s.pending else True
        assert before - set(s.active) <= set(done)
    assert done == {rid: frames[1 + i % 70] for i, rid in enumerate(ids)}


def test_cancel_queued_decoding_and_vocoding():
    s = _server(2, {3: 40, 4: 24, 5: 40})
    a, b, c = s.submit(_text(3)), s.submit(_text(4)), s.submit(_text(5))
    s.step()
    assert s.active == [a, b] and s.pending == [c]
    s.cancel(c)                                  # queued
    assert s.pending == []
    s.step()
    s.step()                                     # b has decoded its 24 frames
    s.step()                                     # b's stream has ended: vocoding
    assert b in s.active and s.requests[b].tid is None and s.pool.streams[s.requests[b].sid][1] and s.decoder.rows.keys() == {0}
    s.cancel(b)                                  # vocoding
    s.cancel(a)                                  # decoding
    assert not s.active and not s.pool.streams and not s.decoder.rows
    with pytest.raises(ValueError, match='unknown or finished request'):
        s.cancel(a)


def test_short_request_fails_alone():
    s = _server(4, {3: 40, 4: 12, 5: 30})
    a, b, c = s.submit(_text(3)), s.submit(_text(4)), s.submit(_text(5))
    out = {}
    while s.pending or s.active:
        for rid, chunk in s.step().items():
            out[rid] = chunk.shape[0]
    assert list(s.failed) == [b] and 'at least 21' in s.failed[b]
    assert out == {a: 40, c: 30}


# ---- the decoder rows on the host ----
def _host_rows(monkeypatch, forward=False, stops=None):
    """_DecodeRows of the default model with the library calls replaced: reset_rows writes the initial state on the host, a decoder call
    returns zero frames and the stop logits stops[key](frames decoded) -> fired, and records (B, L, frames, masks)."""
    calls = []

    def reset_rows(self, rows, fwd):
        for name in ('att_h', 'att_c', 'gen_h', 'gen_c', 'context', 'cum_weights', 'frame'):
            getattr(self, name)[list(rows)] = 0.0
        if fwd:
            self.cum_weights[list(rows), 0] = 1.0

    def chunk(cfg, memory, lengths, params, state, frames):
        B, L = memory.shape[0], memory.shape[1]
        assert state.cum_weights.shape == (B, L) and lengths.shape == (B,) and int(lengths.max()) == L
        calls.append((B, L, frames, {k: v.clone() for k, v in cfg.masks.items()}))
        stop = torch.full((B, frames), -1.0)
        for j, key in enumerate(rows.keys):
            for i in range(frames):
                if stops and stops.get(key) is not None and stops[key](rows.done[j] + i):
                    stop[j, i] = 1.0
        return torch.zeros(B, frames, 80), stop, torch.zeros(B, frames, L)
    monkeypatch.setattr(F.DecoderState, 'reset_rows', reset_rows)
    monkeypatch.setattr(F, 'decoder_forward_chunk', chunk)
    monkeypatch.setattr(F, 'fill_keep_mask', lambda shape, rate, seed, stream_id, device: torch.ones(shape, dtype=torch.uint8))
    model = T.Tacotron()
    rows = T._DecodeRows(model._decoder, 1)
    return rows, calls


def _memory(lengths, M=4, fill=1.0):
    m = torch.zeros(len(lengths), max(lengths), M)
    for b, n in enumerate(lengths):
        m[b, :n] = fill + b
    return m


def test_rows_repad_and_step_counters(monkeypatch):
    hp.max_output_length = 40
    rows, calls = _host_rows(monkeypatch, stops={'b': lambda t: t >= 9})
    rows.add(_memory([5, 3]), [5, 3], ['a', 'b'], [('shared', 0), ('shared', 1)])
    rows.state.cum_weights += 0.5                        # a running decode's weights
    rows.step(8)
    assert rows.done == [8, 8] and calls[-1][:3] == (2, 5, 8)
    # a text longer than every open one joins: memory and cum_weights re-pad to 9, the old rows keep their values, the new row is reset
    rows.add(_memory([9], fill=7.0), [9], ['c'], [('shared', 2)])
    assert rows.memory.shape == (3, 9, 4) and bool((rows.memory[:2, 5:] == 0).all()) and bool((rows.memory[2] == 7.0).all())
    assert bool((rows.state.cum_weights[:2, :5] == 0.5).all()) and bool((rows.state.cum_weights[:2, 5:] == 0).all())
    assert bool((rows.state.cum_weights[2] == 0).all()) and rows.done == [8, 8, 0]
    rows.step(8)
    assert rows.done == [16, 16, 8]
    # b's stop token fires from frame 9 on: its cut is the one-shot rule's over the same logits
    cut = T.Decoder._stop_cut(torch.tensor([1.0 if t >= 9 else -1.0 for t in range(16)]), hp.stop_frames)
    assert cut < 16 and rows.rules[1].cut == cut and rows.rules[0].cut is None
    assert rows.retire() == ['b'] and rows.keys == ['a', 'c'] and rows.done == [16, 8]
    # the longest leaves: memory and cum_weights shrink to the longest left
    rows.close('c')
    assert rows.memory.shape[1] == 5 and rows.state.cum_weights.shape[1] == 5
    # per-row max_output_length: 'a' reaches 40 frames before a row opened later
    rows.add(_memory([2]), [2], ['d'], [('shared', 3)])
    while 'a' in rows.keys:
        rows.step(8)
        rows.retire()
    assert rows.keys == ['d'] and rows.done[0] < 40
    # the last call of a row near its limit is as long as the row furthest from it needs
    steps = [c[2] for c in calls]
    assert all(s <= 8 for s in steps)


def test_rows_mask_sources(monkeypatch):
    from multilingual_text_to_speech_b200.rng import MaskSource
    rows, calls = _host_rows(monkeypatch)
    P = rows.dec._prenet._layers[0].weight.shape[0]
    tape = {k: torch.arange(12 * P).reshape(12, P).remainder(2).to(torch.uint8) for k in T.PRENET_SITES}
    shared = {k: torch.zeros(20, 4, P, dtype=torch.uint8) for k in T.PRENET_SITES}
    for k in shared:
        shared[k][:, 2] = 1
    monkeypatch.setattr(F, 'fill_keep_mask_rows', lambda steps, width, rate, seeds, step0, stream, device:
                        torch.stack([torch.full((steps, width), 7 + 10 * s0, dtype=torch.uint8) for s0 in step0], 1))
    MaskSource.use_tape(shared)
    try:
        rows.add(_memory([3, 4, 2]), [3, 4, 2], ['t', 's', 'c'], [('tape', tape), ('seed', 1), ('shared', 2)])
        rows.step(5)
        rows.step(5)
    finally:
        MaskSource.use_tape(None)
    for k in T.PRENET_SITES:
        m0, m1 = calls[0][3][k], calls[1][3][k]
        assert torch.equal(m0[:, 0], tape[k][:5]) and torch.equal(m1[:, 0], tape[k][5:10])    # the row's own tape at its own steps
        assert bool((m0[:, 1] == 7).all()) and bool((m1[:, 1] == 57).all())                   # seeded at step0 = 0, then 5
        assert bool((m0[:, 2] == 1).all())                                                    # column 2 of the shared tape


# ---- argument errors ----
def test_value_errors(_model):
    pool = T.DecoderPool(_model, 2)
    P = _model._decoder._prenet._layers[0].weight.shape[0]
    bad = [dict(text=torch.zeros(0, dtype=torch.int64)), dict(text=torch.ones(3)),
           dict(text=_text(3), masks={'step_prenet0': torch.ones(4, P)}),
           dict(text=_text(3), masks={'step_prenet0': torch.ones(4, P), 'step_prenet1': torch.ones(4, P + 1)}),
           dict(text=_text(3), masks={'step_prenet0': torch.ones(4, P), 'step_prenet1': 2 * torch.ones(4, P)}),
           dict(text=_text(3), seed=-1), dict(text=_text(3), seed=1 << 64), dict(text=_text(3), seed=1.5), dict(text=_text(3), seed=True)]
    for kw in bad:
        with pytest.raises(ValueError):
            pool.open(**kw)
    assert pool.ids == []
    a = pool.open(_text(3), seed=3)
    pool.open(_text(4), masks={k: torch.ones(4, P) for k in T.PRENET_SITES})
    with pytest.raises(ValueError, match='pool is full'):
        pool.open(_text(5))
    pool.close(a)
    with pytest.raises(ValueError, match='unknown or finished text'):
        pool.close(a)
    with pytest.raises(ValueError, match='1 to 64 texts'):
        T.DecoderPool(_model, 65)
    with pytest.raises(ValueError, match='chunk_frames'):
        T.DecoderPool(_model, 2, chunk_frames=0)
    s = _server(2, {3: 30})
    with pytest.raises(ValueError):
        s.submit(_text(3), seed=-2)
    assert s.pending == [] and s.next_id == 0


def test_abi_argument_checks_without_a_device():
    lib = _lib.load()
    one = ctypes.c_void_p(16)
    shape = _lib.DecoderShape(B=4, L=10, M=8, D=8, N=80)
    st = _lib.DecoderState(*([one] * 7))
    rows = (ctypes.c_int * 2)(1, 4)
    assert lib.b200tts_decoder_state_reset_rows(ctypes.byref(shape), ctypes.byref(st), rows, 2, None) == -1
    assert b'row 4 outside [0, 4)' in lib.b200tts_last_error()
    assert lib.b200tts_decoder_state_reset_rows(ctypes.byref(shape), ctypes.byref(st), rows, 5, None) == -1
    assert b'5 rows of a state of 4' in lib.b200tts_last_error()
    st_missing = _lib.DecoderState(*([one] * 6 + [None]))
    assert lib.b200tts_decoder_state_reset_rows(ctypes.byref(shape), ctypes.byref(st_missing), rows, 1, None) == -1
    assert b'every state buffer' in lib.b200tts_last_error()
    assert lib.b200tts_decoder_state_reset_rows(ctypes.byref(_lib.DecoderShape(B=4, L=10, M=8, D=8, N=80, att_kind=7)), ctypes.byref(st),
                                                rows, 1, None) == -1
    assert b'bad attention kind' in lib.b200tts_last_error()
    assert lib.b200tts_fill_keep_mask_rows(one, 3, 0, 4, 0.5, one, one, 1, None) == -1
    assert b'0 rows' in lib.b200tts_last_error()
    assert lib.b200tts_fill_keep_mask_rows(one, 3, 2, 4, 1.0, one, one, 1, None) == -1
    assert b'rate must be in [0,1)' in lib.b200tts_last_error()
    assert lib.b200tts_fill_keep_mask_rows(one, 3, 2, 4, 0.5, None, one, 1, None) == -1
    assert b'null mask, seeds or step0' in lib.b200tts_last_error()
    assert lib.b200tts_fill_uniform_rows(one, 2, -1, 1, one, one, 3, None) == -1
    assert b'-1 steps' in lib.b200tts_last_error()
    assert lib.b200tts_fill_uniform_rows(one, 2, 5, 1, one, None, 3, None) == -1
    assert b'null output, seeds or t0' in lib.b200tts_last_error()
    # valid arguments pass the checks and stop only for want of a device
    assert lib.b200tts_fill_uniform_rows(one, 2, 5, 1, one, one, 3, None) != 0
    assert b'fill_uniform_rows' not in lib.b200tts_last_error()


# measured (CUDA 12.9, sm_90a): decoder_init_rows_kernel 28 registers, fill_keep_mask_rows_kernel 32, fill_uniform_rows_kernel 30
BOUNDS = {'decoder_fwd.cu': {'decoder_init_rows_kernel': 40}, 'api.cu': {'fill_keep_mask_rows_kernel': 40, 'fill_uniform_rows_kernel': 40}}


@pytest.mark.parametrize('source', sorted(BOUNDS))
def test_new_kernels_registers_and_spills(source, tmp_path):
    nvcc = _nvcc()
    if nvcc is None:
        pytest.skip('nvcc not available')
    cmd = [nvcc] + build.NVCC_FLAGS + ['-I', os.path.join(build.ROOT, 'include'), '-Xptxas', '-v', '-cubin',
                                       os.path.join(build.CSRC, source), '-o', str(tmp_path / 'k.cubin')]
    res = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    assert res.returncode == 0, res.stdout
    for name, bound in BOUNDS[source].items():
        m = re.search(r'Function properties for \S*' + name + r'\S*\n\s*(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes '
                      r'spill loads\n[^\n]*Used (\d+) registers', res.stdout)
        assert m, (name, res.stdout[-2000:])
        stack, st, ld, regs = map(int, m.groups())
        assert st == 0 and ld == 0 and stack == 0, m.group(0)
        assert regs <= bound, (name, regs)


def test_timing_tool_arguments_and_trace():
    import importlib.util
    spec = importlib.util.spec_from_file_location('time_speech_server', os.path.join(build.ROOT, 'tools', 'time_speech_server.py'))
    tool = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(tool)
    a = tool.parse_args(['--rates', '2,16', '--requests', '5'])
    assert a.rates == [2.0, 16.0] and a.modes == ['RAW', 'MOL'] and a.requests == 5
    with pytest.raises(SystemExit):
        tool.parse_args(['--rates', '0'])
    trace = tool.make_trace(8.0, 2000, 200, 0)
    assert trace == tool.make_trace(8.0, 2000, 200, 0) and trace[0][0] == 0.0
    t = np.array([x for x, _ in trace])
    assert np.all(np.diff(t) >= 0) and abs(np.diff(t).mean() - 1 / 8) < 0.01
    assert [c for _, c in trace[:4]] == [21, 58, 95, 132] and max(c for _, c in trace) <= 400
