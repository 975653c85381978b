"""Concurrent streaming synthesis without a GPU: the pool's per-call budgets, releases and window layout on hand-computed cases, the
checks every vocoder stream pool makes before any device work, the argument checks of the new entry points, and the registers of the new
kernels and of both sample-loop instantiations."""
import ctypes
import os
import re
import subprocess

import numpy as np
import pytest
import torch

from multilingual_text_to_speech_b200 import _lib, build
from multilingual_text_to_speech_b200.modules.griffinlim import GriffinLimVocoder
from multilingual_text_to_speech_b200.modules.stream_pool import VocoderStreamPool
from multilingual_text_to_speech_b200.modules.wavernn import FoldedStreamPool, StreamPool, WaveRNN, _PoolStream, _Row, _SampleLoop
from multilingual_text_to_speech_b200.params.params import Params as hp
from test_wavernn_cpu import REAL, _nvcc


def _pool(S, lookahead=2, hop=275):
    p = StreamPool.__new__(StreamPool)
    p.S, p.lookahead, p.hop, p.streams = S, lookahead, hop, {}
    return p


def _stream(slot, frames, steps, ended=False, released=0):
    st = _PoolStream(slot, torch.device('cpu'), 80, None)
    st.mel = torch.zeros(80, frames)
    st.steps, st.ended, st.released = steps, ended, released
    return st


def test_pool_releases():
    p = _pool(S=4400)
    p.streams = {
        0: _stream(0, 40, 25 * 275 + 100),                      # whole hops run more than 20 hops ago: 5
        1: _stream(1, 40, 20 * 275),                            # nothing older than 20 hops
        2: _stream(2, 30, 29 * 275, True, 5 * 275),             # ended and run out: the final chunk of the 25 frames left
        3: _stream(3, 30, 28 * 275, True, 5 * 275),             # ended but not run out: 3 whole hops, no fade
    }
    assert p.release_plan() == [(0, 5 * 275, 26), (2, 24 * 275, 25), (3, 3 * 275, 24)]


def test_loop_window_layout():
    """Two streams at the reference's settings (pad 2, factors 5 x 5 x 11): row 0 ended at 30 frames and runs its last two hops, row 1
    has 10 frames and runs its first hop."""
    loop = _SampleLoop.__new__(_SampleLoop)
    loop.m = WaveRNN(**REAL)
    rows = [_Row(0, torch.zeros(80, 30), True, 27 * 275, 550, 27 * 275, None, None, 27 * 275),
            _Row(1, torch.zeros(80, 10), False, 0, 275, 0, None, None, 0)]
    srcs, idx, lens, widths, W, desc = loop.window_layout(rows)
    # mel-path windows: padded-mel frames [27, 33) (frames 25..29 of row 0, then zero) and [0, 5) (zero, zero, frames 0..2 of row 1);
    # MelResNet windows: frames [25, 30) and [0, 3)
    assert srcs == [(0, 25, 30), (1, 0, 3), (0, 25, 30), (1, 0, 3)]
    assert lens == [6, 5] and widths == [5, 3] and W == 5
    Wt = 17                                                   # 16 packed columns and the zero column
    assert idx.shape == (80 * 11 + 2 * 80 * 5,)
    assert list(idx[:6]) == [0, 1, 2, 3, 4, 16] and list(idx[6:12]) == [Wt + c for c in (0, 1, 2, 3, 4, 16)]
    assert list(idx[480:485]) == [16, 16, 5, 6, 7]
    assert list(idx[880:885]) == [8, 9, 10, 11, 12] and list(idx[1280:1285]) == [13, 14, 15, 16, 16]
    assert np.all(idx < 80 * Wt)
    # (slot, frames or 0, m0, mel_len, a0, aux_len, s0, mel_off, aux row, n): m0 and the mel lengths in samples of the penultimate layer
    assert desc == [(0, 30, 27 * 25, 6 * 25, 25, 5, 27 * 275, 0, 0, 550), (1, 0, 0, 5 * 25, 0, 3, 0, 80 * 6 * 25, 5, 275)]


def test_pool_budgets():
    p = _pool(S=4400)
    p.streams = {
        0: _stream(0, 10, 0),                      # 10 frames, 2 of lookahead: samples of frames [0, 8) are ready
        1: _stream(1, 10, 8 * 275),                # nothing more until frames arrive
        2: _stream(2, 100, 0),                     # 98 frames ready: capped at 4400 steps
        3: _stream(3, 21, 19 * 275, ended=True),   # ended: the last frame's lookahead no longer waits, up to (F - 1) hop
        4: _stream(4, 2, 0),                       # fewer frames than the lookahead
        5: _stream(5, 30, 29 * 275, ended=True),   # every step run: only its final release is left
    }
    assert p.plan() == {0: (0, 8 * 275), 2: (0, 4400), 3: (19 * 275, 275)}


def _host_pools():
    """The three vocoder stream pools' host state, without the WaveRNN pools' device set-up."""
    m = WaveRNN(**REAL)
    unfolded = StreamPool.__new__(StreamPool)
    VocoderStreamPool.__init__(unfolded, m, 2)
    folded = FoldedStreamPool.__new__(FoldedStreamPool)
    folded._layout(m, 2, 300, 7, 64)
    return {'unfolded': (unfolded, np.zeros((2, 100, 1), np.float32)), 'folded': (folded, np.zeros((2, 100, 1), np.float32)),
            'griffinlim': (GriffinLimVocoder().stream_pool(2), np.zeros((1, 100, 1), np.float32))}


def test_pool_checks_before_device_work():
    """max_streams and preemphasis at construction, the tape and the seed at open(): ValueError before any device work, and nothing
    opened."""
    hp.reset()
    m = WaveRNN(**REAL)
    for make in (lambda n, a: StreamPool(m, n, a), lambda n, a: FoldedStreamPool(m, n, 300, 7, a),
                 lambda n, a: GriffinLimVocoder().stream_pool(n, a)):
        for n in (0, 65, True, 2.0):
            with pytest.raises(ValueError, match='1 to 64 streams'):
                make(n, 0.0)
        for a in (1.0, -1.0):
            with pytest.raises(ValueError, match='preemphasis'):
                make(2, a)
    for name, (pool, bad_tape) in _host_pools().items():
        for seed in (-1, 1 << 64, 1.5, True, '3'):
            with pytest.raises(ValueError, match=r'a seed is an int in \[0, 2\^64\)'):
                pool.open(seed=seed)
        with pytest.raises(ValueError, match='uniform tape'):
            pool.open(uniforms=bad_tape)
        assert pool.streams == {} and pool.next_sid == 0, name


def test_abi_argument_checks_without_a_device():
    lib = _lib.load()
    shape = _lib.WaveRNNShape(4, 512, 512, 512, 0, 100)
    ws = ctypes.c_void_p(1 << 20)
    nbytes = lib.b200tts_wavernn_workspace_bytes(ctypes.byref(shape))
    params, cond = _lib.WaveRNNParams(), _lib.WaveRNNCond()
    one = ctypes.c_void_p(16)
    for active, n in ((5, 10), (0, 10), (4, 101), (4, 0)):
        assert lib.b200tts_wavernn_run_rows(ctypes.byref(shape), ctypes.byref(params), ctypes.byref(cond), one, one, active, n, one, one, ws,
                                            nbytes, None) == -1
        assert b'active rows' in lib.b200tts_last_error()
    rows = (ctypes.c_int * 2)(1, 4)
    assert lib.b200tts_wavernn_reset_rows(ctypes.byref(shape), ws, nbytes, rows, 2, None) == -1
    assert b'row 4 outside [0, 4)' in lib.b200tts_last_error()
    # window rows: each row checked against its own windows
    good = _lib.WaveRNNWindowShape(80, 128, 275, 2, 11, 0, 0, 100, 0, 5)
    short = _lib.WaveRNNWindowShape(80, 128, 275, 2, 11, 0, 0, 60, 0, 5)
    other = _lib.WaveRNNWindowShape(80, 64, 275, 2, 11, 0, 0, 100, 0, 5)
    W = _lib.WaveRNNWindowRow * 2
    assert lib.b200tts_wavernn_window_rows(W(_lib.WaveRNNWindowRow(good, 0, 0, 0, 275), _lib.WaveRNNWindowRow(short, 0, 0, 0, 275)), 2, 275,
                                           one, one, one, one, None) == -1
    assert b'outside the window' in lib.b200tts_last_error()
    # a row that runs no steps is not checked against its window: the call passes the checks and stops only for want of a device
    rows_ok = W(_lib.WaveRNNWindowRow(good, 0, 0, 0, 275), _lib.WaveRNNWindowRow(short, 0, 0, 0, 0))
    lib.b200tts_wavernn_window_rows(rows_ok, 2, 275, one, one, one, one, None)
    assert b'wavernn_window_rows' not in lib.b200tts_last_error()
    assert lib.b200tts_wavernn_window_rows(rows_ok, 2, 274, one, one, one, one, None) == -1
    assert b'runs 275 of 274 steps' in lib.b200tts_last_error()
    assert lib.b200tts_wavernn_window_rows(W(_lib.WaveRNNWindowRow(good, 0, 0, 0, 275), _lib.WaveRNNWindowRow(other, 0, 0, 0, 0)), 2, 275,
                                           one, one, one, one, None) == -1
    assert b'differ from row 0' in lib.b200tts_last_error()
    assert lib.b200tts_wavernn_window_rows(rows_ok, 65, 275, one, one, one, one, None) == -1
    lens = (ctypes.c_int * 2)(5, 0)
    assert lib.b200tts_wavernn_upsample_segments(80, 2, lens, 5, one, one, one, None) == -1
    assert b'bad dimensions' in lib.b200tts_last_error()
    assert lib.b200tts_wavernn_upsample_segments(80, 65, lens, 5, one, one, one, None) == -1


# measured (CUDA 12.9, sm_90a): wavernn_window_rows_kernel 40 registers, wavernn_upsample_segments_kernel 32, wavernn_reset_rows_kernel 24;
# the loop kernel 158 registers for the existing instantiation (as before the ragged one was added) and 156 for the ragged one
BOUNDS = {'wavernn_window_rows_kernel': 64, 'wavernn_upsample_segments_kernel': 64, 'wavernn_reset_rows_kernel': 64,
          'wavernn_loop_kernelILb0E': 158, 'wavernn_loop_kernelILb1E': 168}


def test_new_kernels_registers_and_spills(tmp_path):
    nvcc = _nvcc()
    if nvcc is None:
        pytest.skip('nvcc not available')
    cmd = [nvcc] + build.NVCC_FLAGS + ['-I', os.path.join(build.ROOT, 'include'), '-Xptxas', '-v', '-cubin',
                                       os.path.join(build.CSRC, 'wavernn.cu'), '-o', str(tmp_path / 'wavernn.cubin')]
    res = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    assert res.returncode == 0, res.stdout
    for name, bound in BOUNDS.items():
        m = re.search(r'Function properties for \S*' + name + r'\S*\n\s*(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes '
                      r'spill loads\n[^\n]*Used (\d+) registers', res.stdout)
        assert m, (name, res.stdout)
        stack, st, ld, regs = map(int, m.groups())
        assert st == 0 and ld == 0 and stack == 0, m.group(0)
        assert regs <= bound, (name, regs)
    # the existing instantiation keeps the register count it had
    m = re.search(r'Function properties for \S*wavernn_loop_kernelILb0E\S*\n[^\n]*\n[^\n]*Used (\d+) registers', res.stdout)
    assert int(m.group(1)) == 158
