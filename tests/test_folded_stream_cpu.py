"""Folded streaming synthesis without a GPU: fold existence and opening against fold_count, the plan, release and row-grant order on
hand-computed cases, a host-model simulation of a few rows under many long streams, the ValueErrors, the argument checks of
b200tts_wavernn_unfold_streams, its registers, and the unchanged SASS of wavernn_unfold_kernel."""
import contextlib
import ctypes
import hashlib
import os
import re
import subprocess

import numpy as np
import pytest
import torch

from multilingual_text_to_speech_b200 import _lib, build
from multilingual_text_to_speech_b200 import functional as F
from multilingual_text_to_speech_b200.modules.wavernn import FoldedStreamPool, WaveRNN, _FoldedStream, fold_count
from test_wavernn_cpu import REAL, _nvcc

HOP = 275


class _HostPool(FoldedStreamPool):
    """A FoldedStreamPool with the device work replaced: a loop call only advances the folds' step counters, and a release checks that
    every fold its positions read exists, has run those positions and still holds its storage."""

    def __init__(self, model, max_streams, target, overlap, nrows):
        self._layout(model, max_streams, target, overlap, nrows)

    def _fp32(self):
        return contextlib.nullcontext()

    def _reset(self, slots):
        assert all(self.slots[r] is not None and self.slots[r].steps == 0 for r in slots)

    def _loop(self, plan):
        for f, (t, n) in plan.items():
            assert self.slots[f.slot] is f and t == f.start + f.steps and n >= 1
            assert f.steps + n <= self.needed(f.st, f.k) and (f.st.tape is None or f.k < f.st.tape.shape[0])
        self._advance(plan)

    def _release(self, rel):
        descs, base = self.unfold_layout(rel)
        for d, (sid, q0, q1, frames) in zip(descs, rel):
            st = self.streams[sid]
            assert q0 == st.released and (frames == 0 or q1 <= (frames - 1) * self.hop)
            n_exist = fold_count(st.frames * self.hop, self.target, self.overlap)
            for e in range(d.nfolds):
                k = d.fold0 + e
                if base[d.src + e] < 0:
                    assert st.ended and k >= n_exist          # absent: the fold does not exist
                    continue
                f = st.folds[k]
                assert f.store is not None and base[d.src + e] == f.store * self.fold_len
                assert f.start + f.steps >= min(q1, f.start + self.fold_len)      # it has run every position of the range it covers
        self._mark_released(rel)
        return {sid: q1 - q0 for sid, q0, q1, _ in rel}


@pytest.fixture
def model():
    return WaveRNN(**REAL)


@pytest.fixture
def no_device(monkeypatch):
    monkeypatch.setattr(F, 'wavernn_aborted', lambda shape, ws: False)


def _host(model, max_streams, target, overlap, nrows=64):
    p = _HostPool(model, max_streams, target, overlap, nrows)
    p.shape = p.ws = None
    p.device = torch.device('cpu')
    return p


def _stream(p, frames, ended=False, tape_folds=None):
    sid = p.next_sid
    tape = None if tape_folds is None else torch.zeros(tape_folds, p.fold_len, 1)
    st = _FoldedStream(sid, torch.device('cpu'), 80, tape)
    st.mel = torch.zeros(80, frames)
    st.ended = ended
    p.streams[sid] = st
    p.next_sid += 1
    return st


GEOMETRIES = [(11000, 550), (300, 0), (300, 7), (1000, 137), (550, 275), (40, 900)]


# ---- geometry ----
@pytest.mark.parametrize('target,overlap', GEOMETRIES)
def test_fold_existence_and_opening_follow_fold_count(model, target, overlap):
    p = _host(model, 1, target, overlap)
    step = target + overlap
    for F_ in range(21, 201):
        n = fold_count(F_ * HOP, target, overlap)
        # fold k exists iff k (t + o) + o < F hop
        assert n == sum(1 for k in range(F_ * HOP) if k * step + overlap < F_ * HOP), F_
        ended = _stream(p, F_, True)
        assert p.folds_known(ended) == n
        # the folds the stream runs: those with a position before the cut, each up to the cut
        needs = [p.needed(ended, k) for k in range(n)]
        cut = (F_ - 1) * HOP
        assert all(s == min(target + 2 * overlap, cut - k * step) for k, s in enumerate(needs))
        # while the mel arrives, a fold opens only once it exists for the frames that have arrived
        for known in (1, F_ // 2, F_ - 1):
            st = _stream(p, known)
            assert p.folds_known(st) == fold_count(known * HOP, target, overlap) <= n
        p.streams.clear()


def test_plan_release_and_grant_order_by_hand(model, no_device):
    p = _host(model, 4, 11000, 550, nrows=3)
    step = 11550
    a = _stream(p, 80)                   # 22000 samples: folds 0 and 1 certain (11550 + 550 < 22000), fold 2 undecided (23650)
    b = _stream(p, 40)                   # 11000 samples: fold 0 only (11550 + 550 > 11000)
    assert p.folds_known(a) == 2 and p.folds_known(b) == 1
    # keys k (t + o) - released: a0 0, b0 0, a1 11550
    assert [(st.sid, k) for st, k in p.grants()] == [(0, 0), (1, 0), (0, 1)]
    a.released = 11550                   # a's fold 1 (key 0) now ties with b's fold 0 and goes first by stream id
    assert [(st.sid, k) for st, k in p.grants()] == [(0, 0), (0, 1), (1, 0)]
    a.released = 0
    p.run()
    assert [(f.st.sid, f.k) for f in p.slots] == [(0, 0), (1, 0), (0, 1)]
    # one call: 16 hops (COND_BYTES allows more at 3 rows)
    assert all(f.steps == 4400 for f in p.slots)
    assert {(f.st.sid, f.k): v for f, v in p.plan().items()} == {(0, 0): (4400, 4400), (1, 0): (4400, 4400), (0, 1): (step + 4400, 4400)}
    # a's final positions end at fold 0's 4400; nothing is released within 20 hops of them
    assert p.final(a) == 4400 and p.release_plan() == []
    for _ in range(2):
        p.run()
    # a's fold 0 has run its 12100 steps and left its row; fold 1 stops at the ready positions, (80 - 2) hops: 9900 steps; b's fold 0
    # at (40 - 2) hops
    assert p.slots[0] is None and a.folds[0].done
    assert a.folds[1].steps == 78 * HOP - step and b.folds[0].steps == 38 * HOP
    assert p.final(a) == 78 * HOP and a.released == (58 * HOP) // HOP * HOP
    assert a.folds[0].store is None                              # every sample of fold 0 (below 12100) is released
    assert p.grants() == [] and p.plan() == {}                   # nothing more until frames arrive
    # b ends: fold 0 runs to the cut, (40 - 1) hops, and the last chunk carries the fade-out
    b.ended = True
    assert p.release_plan() == [(1, 18 * HOP, 38 * HOP, 40)]    # after end() every final position goes, fade-out included
    p.run()
    assert 1 not in p.streams and len(p.free_store) == p.nstore - 1
    # a ends at 90 frames (24750 samples): fold 2 exists (23100 + 550 < 24750) and runs to the cut 24475
    a.mel = torch.zeros(80, 90)
    a.ended = True
    assert p.folds_known(a) == 3 and p.needed(a, 2) == 89 * HOP - 2 * step
    assert [(st.sid, k) for st, k in p.grants()] == [(0, 2)]
    while 0 in p.streams:
        p.run()
    assert sorted(p.free_store) == list(range(p.nstore)) and all(f is None for f in p.slots)


def test_release_rule_by_hand(model):
    p = _host(model, 2, 300, 7)
    st = _stream(p, 60)                                          # 16500 samples
    p._grant([(st, 0), (st, 1)])
    st.folds[0].steps, st.folds[1].steps = 314, 200             # fold 0 complete, fold 1 at position 307 + 200
    p._retire()
    assert st.folds[0].done and st.folds[0].slot is None and not st.folds[1].done
    # fold 2 (at 614) has no row: it blocks from 614; fold 1 blocks from 507
    assert p.final(st) == 507
    st.ended = True
    st.mel = torch.zeros(80, 3)                                  # pretend a 3-frame mel: the cut 550 lies inside fold 1
    assert p.final(st) == 507 and p.needed(st, 1) == 550 - 307
    st.folds[1].steps = 243
    p._retire()
    assert st.folds[1].done and p.final(st) == 550               # fold 2 starts past the cut: it never runs
    assert p.release_plan() == [(0, 0, 550, 3)]


def test_grant_keys_favour_the_listener(model):
    """A new stream's fold 0 goes before an old stream's later folds, whose keys are far ahead of what the old stream has released."""
    p = _host(model, 3, 11000, 550, nrows=2)
    old = _stream(p, 900)
    old.released = 3 * 11550 - 100
    old.folds = [None] * 3                                       # folds 0..2 opened (bookkeeping only)
    new = _stream(p, 50)
    # keys: old fold 3 at 3 * 11550 - released = 100, new fold 0 at 0
    assert [(st.sid, k) for st, k in p.grants()][:2] == [(1, 0), (0, 3)]


@pytest.mark.parametrize('target,overlap,nrows', [(11000, 550, 4), (1000, 137, 3), (300, 7, 5), (550, 275, 2)])
def test_host_simulation_every_stream_finishes(model, no_device, target, overlap, nrows):
    """Few rows, many long streams joining, feeding, cancelling and ending at random: every stream that is not cancelled finishes with
    all its samples released exactly once, no row is ever held by a finished fold, and every row and storage slot is free at the end."""
    rng = np.random.default_rng(target + overlap + nrows)
    p = _host(model, 8, target, overlap, nrows=nrows)
    todo = {}                          # sid -> (frames in all, frames fed)
    finished, cancelled, out = set(), set(), {}
    opened = 0
    for call in range(20000):
        if opened < 40 and len(p.streams) < p.rows and rng.random() < 0.3:
            sid = p.open()
            todo[sid] = [int(rng.integers(21, 900)), 0]
            out[sid] = 0
            opened += 1
        for sid in list(p.streams):
            tot, fed = todo[sid]
            if p.streams[sid].ended:
                continue
            if rng.random() < 0.005:
                p.close(sid)
                cancelled.add(sid)
                continue
            n = min(int(rng.integers(0, 40)), tot - fed)
            if n:
                p.feed(sid, torch.zeros(80, n))
                todo[sid][1] += n
            if todo[sid][1] == tot and rng.random() < 0.5:
                p.end(sid)
        for sid, n in p.run().items():
            out[sid] += n
        assert all(f is None or not f.done for f in p.slots)
        held = sum(1 for f in p.slots if f is not None)
        assert held + len(p.free_store) <= p.nstore
        for sid in list(todo):
            if sid not in p.streams and sid not in cancelled and sid not in finished:
                finished.add(sid)
                assert out[sid] == (todo[sid][0] - 1) * HOP, (sid, out[sid], todo[sid])
        if opened == 40 and not p.streams:
            break
    assert not p.streams and opened == 40, (call, len(p.streams))
    assert len(finished) + len(cancelled) == 40 and len(finished) > 30
    assert all(f is None for f in p.slots) and sorted(p.free_store) == list(range(p.nstore))


# ---- errors ----
def test_value_errors(model, no_device):
    with pytest.raises(ValueError, match='target >= 1'):
        FoldedStreamPool(model, 2, 0, 10)
    with pytest.raises(ValueError, match='overlap >= 0'):
        FoldedStreamPool(model, 2, 100, -1)
    with pytest.raises(ValueError, match='target >= 1'):
        model.stream_pool(2, target=100)
    with pytest.raises(ValueError, match='1 to 64 streams'):
        FoldedStreamPool(model, 65, 11000, 550)
    with pytest.raises(ValueError, match='exceeds 512 MiB'):
        FoldedStreamPool(model, 64, 10 ** 7, 0)
    # a tape's fold length must be target + 2 overlap
    with pytest.raises(ValueError, match=r'expected \[folds, 12100, 1\]'):
        model._check_stream_tape(torch.zeros(2, 12000, 1), 12100)
    with pytest.raises(ValueError, match='outside'):
        model._check_stream_tape(torch.ones(2, 12100, 1), 12100)
    assert model._check_stream_tape(torch.zeros(3, 12100, 1), 12100).shape == (3, 12100, 1)
    # a fold beyond the tape: ValueError before any device work of that run()
    p = _host(model, 2, 300, 7)
    st = _stream(p, 30, tape_folds=2)
    with pytest.raises(ValueError, match='holds 2 folds; stream 0 needs fold 2'):
        p.run()
    assert not st.folds and all(f is None for f in p.slots)


def test_server_rejects_an_unfolded_tape_for_a_folded_pool(model):
    from multilingual_text_to_speech_b200.modules.streaming import SpeechServer
    s = SpeechServer.__new__(SpeechServer)
    s.pool, s.wavernn = _host(model, 2, 11000, 550), model
    s.decoder = type('D', (), {'check': staticmethod(lambda *a: None)})()
    s.requests, s.pending, s.failed, s.next_id = {}, [], {}, 0
    with pytest.raises(ValueError, match=r'expected \[folds, 12100, 1\]'):
        s.submit(torch.zeros(5, dtype=torch.long), uniforms=torch.zeros(1, 5000, 1))
    assert s.submit(torch.zeros(5, dtype=torch.long), uniforms=torch.zeros(2, 12100, 1)) == 0


# ---- the C ABI ----
def test_unfold_streams_argument_checks_without_a_device():
    lib = _lib.load()
    one = ctypes.c_void_p(16)
    S = _lib.WaveRNNUnfoldStream

    def call(streams, nsrc=8, total=None, hop=275, target=1000, overlap=100, mu=511):
        arr = (S * len(streams))(*streams) if streams else None
        total = sum(s.q1 - s.q0 for s in streams) if total is None else total
        return lib.b200tts_wavernn_unfold_streams(len(streams), hop, target, overlap, mu, arr, one, one, nsrc, total, one, one, None)

    # step 1100, L 1200: positions [0, 2000) read folds 0 and 1, [2000, 2100) fold 1 only (fold 0 ends at 1200, fold 2 starts at 2200)
    good = [S(0, 2000, 0, 0, 0, 2, 0), S(2000, 2100, 2000, 0, 1, 1, 2)]
    assert call(good) != 0 and b'wavernn_unfold_streams' not in lib.b200tts_last_error()      # stops only for want of a device
    assert call(good, target=0) == -1 and b'bad arguments' in lib.b200tts_last_error()
    assert call([]) == -1 and b'0 streams' in lib.b200tts_last_error()
    assert call([S(0, 10, 0, 0, 0, 1, 0)] * 65, total=650) == -1 and b'65 streams' in lib.b200tts_last_error()
    assert call([S(5, 5, 0, 0, 0, 1, 0)], total=1) == -1 and b'writes positions [5, 5)' in lib.b200tts_last_error()
    assert call([good[0], S(2000, 2100, 1999, 0, 1, 1, 2)]) == -1 and b'(expected 2000' in lib.b200tts_last_error()
    assert call([S(0, 2000, 0, 0, 0, 1, 0)]) == -1 and b'read folds 0 to 1' in lib.b200tts_last_error()
    assert call([S(2000, 2100, 0, 0, 2, 1, 0)]) == -1 and b'read folds 1 to 1' in lib.b200tts_last_error()
    assert call([S(0, 2000, 0, 0, 0, 2, 7)]) == -1 and b'sources [7, 9) of 8' in lib.b200tts_last_error()
    assert call([S(0, 2000, 0, 7, 0, 2, 0)]) == -1 and b'past the cut 1650 of its 7 frames' in lib.b200tts_last_error()
    assert call(good, total=5) == -1 and b'total 5' in lib.b200tts_last_error()


# measured (CUDA 12.9, sm_90a): wavernn_unfold_streams_kernel 48 registers, no spills
BOUNDS = {'wavernn_unfold_streams_kernel': 64}
# sha256 of wavernn_unfold_kernel's SASS instructions (addresses stripped) as the parent commit built them with CUDA 12.9 for sm_90a
UNFOLD_SASS_SHA256 = '394b40114b60fde597abcedf4a38b16575aadf1366bb9a24a3c71c7c9fabe64c'


def _compile(tmp_path):
    nvcc = _nvcc()
    if nvcc is None:
        pytest.skip('nvcc not available')
    cubin = tmp_path / 'wavernn.cubin'
    cmd = [nvcc] + build.NVCC_FLAGS + ['-I', os.path.join(build.ROOT, 'include'), '-Xptxas', '-v', '-cubin',
                                       os.path.join(build.CSRC, 'wavernn.cu'), '-o', str(cubin)]
    res = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    assert res.returncode == 0, res.stdout
    return nvcc, cubin, res.stdout


def test_new_kernel_registers_and_spills(tmp_path):
    _, _, log = _compile(tmp_path)
    for name, bound in BOUNDS.items():
        m = re.search(r'Function properties for \S*' + name + r'\S*\n\s*(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes '
                      r'spill loads\n[^\n]*Used (\d+) registers', log)
        assert m, (name, log)
        stack, st, ld, regs = map(int, m.groups())
        assert st == 0 and ld == 0 and stack == 0, m.group(0)
        assert regs <= bound, (name, regs)


def test_unfold_kernel_sass_unchanged(tmp_path):
    """wavernn_unfold_kernel now reads its per-sample arithmetic from the device functions it shares with the streams kernel; its SASS
    is the parent's instruction for instruction."""
    nvcc, cubin, _ = _compile(tmp_path)
    version = subprocess.run([nvcc, '--version'], stdout=subprocess.PIPE, text=True).stdout
    if 'release 12.9' not in version:
        pytest.skip('the recorded SASS is CUDA 12.9\'s')
    cuobjdump = os.path.join(os.path.dirname(nvcc), 'cuobjdump')
    out = subprocess.run([cuobjdump, '-sass', str(cubin)], stdout=subprocess.PIPE, text=True).stdout
    funcs = [f for f in re.split(r'\n\s*Function : ', out) if 'wavernn_unfold_kernel' in f.split('\n', 1)[0]]
    assert len(funcs) == 1
    ins = [re.sub(r'/\*[0-9a-f]{4}\*/', '', line).split(';')[0].strip() for line in funcs[0].split('\n')[1:]
           if re.match(r'\s*/\*[0-9a-f]{4}\*/', line)]
    assert hashlib.sha256('\n'.join(ins).encode()).hexdigest() == UNFOLD_SASS_SHA256
