"""Streaming Griffin-Lim (b200tts_gl_stream_run) checked call by call against fp64 from its own slot state (tests/gl_stream_check.py), through
the C ABI on a raw workspace, at every look-ahead each shape's shared memory admits and across the FFT plans:
  * recorded streams (iters 1 and 2, one frame per call, then the end): each slot read before and after every call, the call recomputed
    from the "before" state; with de-emphasis, each call also runs with a = 0 from the same state and is checked against lfilter of that;
  * crafted single-pass states (one Jacobi pass, with or without an admission before it) at m = 0, inside the partial envelope, at steady
    state and at the largest frame count the host accepts, many in one launch;
  * translation invariance: a steady state shifted to the 2^31 edge gives the same bits;
  * isolation: released samples land exactly at each row's wave_off (NaN-poisoned buffer, sentinel guard bands), in the number
    GriffinLimStreamPool predicts; unlisted slots and the FFT tables stay bitwise unchanged.
The worst err / bound of each stage and shape is printed under -s."""
import time
from types import SimpleNamespace

import numpy as np
import pytest
import torch

import audio_oracle as O
import gl_stream_check as C
import gl_stream_slot as L

pytestmark = pytest.mark.gpu

# (N, hop, win) -> the plan of the half-length transform
SHAPES = {(1102, 275, 1102): (19, 29), (1024, 256, 1024): (4, 4, 4, 4, 2), (1024, 256, 800): (4, 4, 4, 4, 2), (800, 200, 800): (4, 4, 5, 5),
          (1100, 275, 1100): (2, 5, 5, 11), (546, 136, 545): (3, 7, 13), (1426, 356, 1426): (23, 31), (1922, 480, 1922): (31, 31),
          (2048, 512, 2048): (4, 4, 4, 4, 4), (1102, 551, 1102): (19, 29), (1102, 1102, 1102): (19, 29), (4, 2, 4): (2,)}
IDS = [f'{n}-{h}-{w}' for n, h, w in SHAPES]
GUARD = 64
SENTINEL = np.float32(-12345.5)
WORST = {}
T0 = []


@pytest.fixture(scope='module', autouse=True)
def mods():
    import __graft_entry__ as entry
    entry.build()
    from multilingual_text_to_speech_b200 import _lib
    from multilingual_text_to_speech_b200 import functional as F
    assert torch.cuda.is_available()
    T0.append(time.perf_counter())
    yield _lib, F
    print(f'\nworst err / bound by shape and stage ({time.perf_counter() - T0[0]:.1f} s):')
    for key in sorted(WORST):
        print(' ', key, {s: f'{r:.2e}' for s, r in sorted(WORST[key].items())})


def _note(key, worst):
    d = WORST.setdefault(key, {})
    for s, r in worst.items():
        d[s] = max(d.get(s, 0.0), r)


def _lookaheads(N, H, W):
    return [k for k in range(L.MAX_LOOKAHEAD + 1) if L.accepted(N, H, W, k)]


class Rig:
    """A raw workspace of `slots` slots, reset; junk() fills the slots a test does not use with random bytes."""

    def __init__(self, mods, N, H, W, k, iters, slots, seed=0):
        self._lib, self.F = mods
        self.N, self.H, self.W, self.k, self.iters, self.slots = N, H, W, k, iters, slots
        self.lay = L.GlLayout(N, k, slots)
        self.ws = self.F.gl_stream_workspace(self.shape(0.0), 'cuda')
        assert self.ws.numel() == self.lay.bytes
        self.F.gl_stream_reset(self.shape(0.0), self.ws, list(range(slots)))
        buf = self.host()
        _, _, w = L.read_tables(buf, self.lay)
        assert np.array_equal(w, O.hann(W, N).astype(np.float32)) or np.abs(w - O.hann(W, N)).max() < 1e-7
        self.window = w
        self.rng = np.random.default_rng(seed)

    def shape(self, a):
        return self._lib.GLStreamShape(self.N, self.H, self.W, self.k, self.iters, self.slots, float(a))

    def host(self):
        torch.cuda.synchronize()
        return self.ws.cpu().numpy().copy()

    def put(self, buf):
        self.ws.copy_(torch.from_numpy(buf).cuda())

    def junk(self, buf, keep):
        for s in range(self.slots):
            if s not in keep:
                b = self.lay.slot_base(s)
                buf[b:b + self.lay.slot_bytes] = self.rng.integers(0, 256, self.lay.slot_bytes, dtype=np.uint8)
        return buf

    def run(self, rows, S_new, counts, a=0.0):
        """rows: [(slot, frames, ended, new frames)], S_new: their new frames in row order, counts: samples each row should release ->
        (released samples per row, workspace bytes after).  Each row's span has a sentinel band before it and NaN poison after it."""
        offs, off = [], 0
        for n in counts:
            offs.append(off + GUARD)
            off += n + 2 * GUARD
        wave = np.full(off + GUARD, np.nan, np.float32)
        for o, n in zip(offs, counts):
            wave[o - GUARD:o] = SENTINEL
        wave[off:] = SENTINEL
        S = torch.from_numpy(np.ascontiguousarray(S_new, np.float32) if S_new is not None and len(S_new) else
                             np.zeros((1, self.N // 2 + 1), np.float32)).cuda()
        glrows, so = [], 0
        for (slot, frames, ended, s_rows), o in zip(rows, offs):
            glrows.append(self._lib.GLStreamRow(slot, frames, int(ended), so, o))
            so += s_rows
        w = torch.from_numpy(wave).cuda()
        self.F.gl_stream_run(self.shape(a), glrows, S, w, self.ws)
        got = w.cpu().numpy()
        outs = []
        for o, n in zip(offs, counts):
            assert np.array_equal(got[o - GUARD:o].view(np.uint32), wave[o - GUARD:o].view(np.uint32)), 'guard band before a row written'
            seg = got[o:o + n]
            assert np.isfinite(seg).all(), 'a released sample is missing or not finite'
            outs.append(seg.copy())
        assert np.array_equal(got[off:].view(np.uint32), wave[off:].view(np.uint32)), 'trailing guard band written'
        spans = np.zeros(len(got), bool)
        for o, n in zip(offs, counts):
            spans[o - GUARD:o + n] = True
        spans[off:] = True
        assert np.isnan(got[~spans]).all(), 'a row wrote past the samples it releases'
        return outs, self.host()


def _predicted(N, H, k, fed, ended, committed, released):
    """Samples the pool's bookkeeping (GriffinLimStreamPool._committed_after, _released) expects the next call to release."""
    from multilingual_text_to_speech_b200.modules.griffinlim import GriffinLimStreamPool as P
    pool = SimpleNamespace(v=SimpleNamespace(hop=H, N=N, k=k))
    st = SimpleNamespace(fed=fed, ended=ended, committed=committed)
    return P._released(pool, st, P._committed_after(pool, st)) - released


def _unchanged(before, after, lay, listed):
    assert np.array_equal(before[:lay.slots_at], after[:lay.slots_at]), 'FFT tables changed'
    for s in range(lay.slots):
        if s not in listed:
            b = lay.slot_base(s)
            assert np.array_equal(before[b:b + lay.slot_bytes], after[b:b + lay.slot_bytes]), f'unlisted slot {s} changed'


def _check(key, exp, before, after, out, row, sh, window):
    worst = C.compare(exp, after, out, a0=float(np.float32(sh.a)) == 0)
    fails = C.exact_checks(before, after, out, row, sh, window, exp)
    _note(key, worst)
    assert not fails, (key, row, fails)
    assert all(r <= 1 for r in worst.values()), (key, row, worst)


def _signal(kind, n, seed=0):
    t = np.arange(n) / 22050
    if kind == 'chirp':
        f = 100 + 2000 * t / max(t[-1], 1e-9)
        return np.sin(2 * np.pi * np.cumsum(f) / 22050) * (0.5 + 0.5 * np.sin(2 * np.pi * 3 * t)) + 0.05 * np.random.default_rng(seed).standard_normal(n)
    return sum(np.sin(2 * np.pi * 140 * h * t + h) / h for h in range(1, 20))


@pytest.mark.parametrize('N,H,W', list(SHAPES), ids=IDS)
def test_recorded_streams_call_by_call(mods, N, H, W):
    from multilingual_text_to_speech_b200 import _lib
    plan = C.fft_plan(_lib.load(), N)
    assert plan == SHAPES[(N, H, W)]
    frames = 40
    for k in _lookaheads(N, H, W):
        for I, kind, a in ((1, 'harmonic', 0.97), (2, 'chirp', 0.0)):
            rig = Rig(mods, N, H, W, k, I, slots=3, seed=k)
            sh = C.Shape(N, H, W, k, I, a, plan)
            sh0 = C.Shape(N, H, W, k, I, 0.0, plan)
            S = np.abs(O.stft(_signal(kind, H * (frames - 1)), N, H, W)).astype(np.float32)
            buf = rig.junk(rig.host(), {1})
            rig.put(buf)
            released = committed = 0
            calls = [(t + 1, False, S[:, t:t + 1].T) for t in range(frames)] + [(frames, True, None)]
            for F_, ended, new in calls:
                before_buf = rig.host()
                before = L.read_slot(before_buf, rig.lay, 1)
                exp0 = C.one_call(before, new, (F_, ended), sh0, rig.window)
                n = _predicted(N, H, k, F_, ended, committed, released)
                assert n == len(exp0.out), (n, len(exp0.out))
                s_rows = 0 if new is None else len(new)
                (out0,), after_buf = rig.run([(1, F_, ended, s_rows)], new, [n], 0.0)
                _unchanged(before_buf, after_buf, rig.lay, {1})
                after = L.read_slot(after_buf, rig.lay, 1)
                _check((N, H, W, f'k={k}'), exp0, before, after, out0, (F_, ended), sh0, rig.window)
                if a:
                    rig.put(before_buf)                            # the same call again, de-emphasised
                    (out, ), after_buf = rig.run([(1, F_, ended, s_rows)], new, [n], a)
                    after_a = L.read_slot(after_buf, rig.lay, 1)
                    assert np.array_equal(after_a.c, after.c) and np.array_equal(after_a.x, after.x)
                    r = C.deemphasis_ratio(out0, before.carry, a, out)
                    assert not n or after_a.carry.view(np.uint32) == out[-1].view(np.uint32)
                    exp = C.one_call(before, new, (F_, ended), sh, rig.window)
                    r64 = C.compare(exp, after_a, out, a0=False)['deemphasis']
                    _note((N, H, W, f'k={k}'), {'deemphasis': r, 'deemphasis (fp64 from the state)': r64})
                    assert r <= 1 and r64 <= 1, (r, r64)
                released += n
                committed = L.read_slot(rig.host(), rig.lay, 1).committed
            assert released == H * (frames - 1)


KINDS = ('noise', 'zero', 'tone', 'tiny')


def _placements(N, H, k):
    part = -(-(N - 1) // H)
    steady = 3 * part + 7
    return sorted({0, 1, max(1, part - 1), steady, L.max_frames(N, H) - k - 1})


@pytest.mark.parametrize('N,H,W', list(SHAPES), ids=IDS)
def test_crafted_single_passes_and_translation(mods, N, H, W):
    from multilingual_text_to_speech_b200 import _lib
    plan = C.fft_plan(_lib.load(), N)
    for k in _lookaheads(N, H, W):
        places = _placements(N, H, k)
        cases = [(m, kind, admit) for m in places for kind in KINDS for admit in (False, True)]
        slots = min(L.MAX_SLOTS, len(cases) + 2 + 3)
        cases = cases[:slots - 5]
        rig = Rig(mods, N, H, W, k, 1, slots=slots, seed=100 + k)
        sh = C.Shape(N, H, W, k, 1, 0.0, plan)
        rng = np.random.default_rng(k)
        states = [C.crafted_state(sh, rig.window, m, kind, rng, admit) for m, kind, admit in cases]
        # translation: a steady noise state and the same state shifted by d frames to the largest frame count
        m0 = 3 * -(-(N - 1) // H) + 7
        d = L.max_frames(N, H) - k - 1 - m0
        b0, _, row0 = C.crafted_state(sh, rig.window, m0, 'noise', rng)
        A = k + 1
        b1 = L.Slot(b0.committed + d, b0.admitted + d, b0.frames + d, b0.carry, np.roll(b0.c, (d * H) % N), np.roll(b0.x, d % A, axis=0),
                    np.roll(b0.S, d % A, axis=0))
        states += [(b0, None, row0), (b1, None, (row0[0] + d, False))]
        listed = list(range(len(states)))
        buf = rig.junk(rig.host(), set(listed))
        for s, (before, _, _) in zip(listed, states):
            L.write_slot(buf, rig.lay, s, before)
        rig.put(buf)
        before_buf = rig.host()
        exps = [C.one_call(b, new, row, sh, rig.window) for b, new, row in states]
        news = [new for _, new, _ in states if new is not None]
        S_new = np.concatenate(news) if news else None
        rows = [(s, row[0], row[1], 0 if new is None else len(new)) for s, (_, new, row) in zip(listed, states)]
        outs, after_buf = rig.run(rows, S_new, [len(e.out) for e in exps])
        _unchanged(before_buf, after_buf, rig.lay, set(listed))
        for s, (before, new, row), exp, out in zip(listed, states, exps, outs):
            after = L.read_slot(after_buf, rig.lay, s)
            _check((N, H, W, f'k={k}', 'crafted'), exp, before, after, out, row, sh, rig.window)
        a0, a1 = L.read_slot(after_buf, rig.lay, listed[-2]), L.read_slot(after_buf, rig.lay, listed[-1])
        assert (a1.committed - a0.committed, a1.admitted - a0.admitted) == (d, d)
        assert np.array_equal(np.roll(a0.c, (d * H) % N).view(np.uint32), a1.c.view(np.uint32))
        assert np.array_equal(np.roll(a0.x, d % A, axis=0).view(np.uint32), a1.x.view(np.uint32))
        assert np.array_equal(outs[-2].view(np.uint32), outs[-1].view(np.uint32)) and len(outs[-1]) == H
        assert a0.carry.view(np.uint32) == a1.carry.view(np.uint32)
