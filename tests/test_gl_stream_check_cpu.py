"""CPU checks of tests/gl_stream_check.py, the per-call fp64 check of streaming Griffin-Lim: chained over a stream's calls it is the
specification (tests/griffinlim_stream_oracle.py); an fp32 emulation in the kernel's order passes every bound; and each planted fault fails
a bound or an exact check.  Also the slot layout of tests/gl_stream_slot.py against the library's workspace query."""
import ctypes

import numpy as np
import pytest

import audio_oracle as O
import gl_stream_check as C
import gl_stream_slot as L
import griffinlim_stream_oracle as G
from multilingual_text_to_speech_b200 import _lib
from test_griffinlim_stream_cpu import _chirp, lib  # noqa: F401 -- lib is a fixture
from test_vocoder_cpu import _harmonic


def _spec(N, H, W, frames, signal='chirp', seed=0):
    y = (_chirp if signal == 'chirp' else _harmonic)(H * (frames - 1), seed)
    return np.abs(O.stft(y, N, H, W)).astype(np.float32)


@pytest.mark.parametrize('N', [2, 4, 546, 800, 1024, 1100, 1102, 1426, 1922, 2048])
def test_slot_layout_equals_the_workspace_query(lib, N):  # noqa: F811
    ok = 0
    for k in range(L.MAX_LOOKAHEAD + 2):
        for hop in sorted({1, max(1, N // 4), N // 2 or 1, N // 2 + 1, N}):
            for slots in (1, 2, 7, 64):
                shape = _lib.GLStreamShape(N, hop, N, k, 1, slots, 0.0)
                n = lib.b200tts_gl_stream_workspace_bytes(ctypes.byref(shape))
                if not L.accepted(N, hop, N, k):
                    assert n == 0, (N, hop, k)
                    continue
                assert n == L.GlLayout(N, k, slots).bytes, (N, hop, k, slots)
                ok += 1
    assert ok
    # the shared-memory edge of the issue's shapes: N = 2048 up to lookahead 4, N = 1922 up to 5
    assert [L.accepted(2048, 512, 2048, k) for k in (4, 5)] == [True, False]
    assert [L.accepted(1922, 480, 1922, k) for k in (5, 6)] == [True, False]


def test_slot_readers_and_writers_round_trip():
    lay = L.GlLayout(546, 3, 3)
    buf = np.zeros(lay.bytes, np.uint8)
    rng = np.random.default_rng(0)
    st = L.Slot(5, 9, 9, np.float32(-0.25), rng.standard_normal(546).astype(np.float32), rng.standard_normal((4, 546)).astype(np.float32),
                rng.uniform(0, 1, (4, 274)).astype(np.float32))
    L.write_slot(buf, lay, 1, st)
    got = L.read_slot(buf, lay, 1)
    assert (got.committed, got.admitted, got.frames, got.carry) == (5, 9, 9, np.float32(-0.25))
    assert np.array_equal(got.c, st.c) and np.array_equal(got.x, st.x) and np.array_equal(got.S, st.S)
    assert not buf[:lay.slot_base(1)].any() and not buf[lay.slot_base(2):].any()


@pytest.mark.parametrize('N,H,W,k,cuts', [(1102, 275, 1102, 3, [1, 5, 6, 13, 20]), (1102, 275, 1102, 0, list(range(1, 25))),
                                          (1102, 275, 1102, 0, [24]), (546, 136, 545, 1, [2, 3, 17]), (800, 200, 800, 2, [9]),
                                          (1102, 1102, 1102, 1, [4, 11]), (64, 16, 60, 0, [3, 4, 5, 23]), (4, 2, 4, 7, [1, 2, 8])])
def test_chained_one_call_equals_the_spec(lib, N, H, W, k, cuts):  # noqa: F811
    Fr, I = 24, 3
    S = _spec(N, H, W, Fr)
    sh = C.Shape(N, H, W, k, I, 0.0, C.fft_plan(lib, N))
    w = O.hann(W, N)
    st, out, t0 = L.empty_slot(L.GlLayout(N, k)), [], 0
    for t1 in cuts:
        exp = C.one_call(st, S[:, t0:t1].T, (t1, False), sh, w)
        out.append(exp.out)
        st, t0 = exp.after, t1
    exp = C.one_call(st, S[:, t0:].T if t0 < Fr else None, (Fr, True), sh, w)
    out.append(exp.out)
    got = np.concatenate(out)
    ref = G.rtisi_chunked(S.astype(np.float64), cuts + ([Fr] if cuts[-1] < Fr else []), N, H, W, k, I)
    assert got.shape == ref.shape == (H * (Fr - 1),)
    assert np.linalg.norm(got - ref) <= 1e-12 * np.linalg.norm(ref), np.linalg.norm(got - ref) / np.linalg.norm(ref)
    assert exp.after.committed == exp.after.admitted == Fr


def recorded(lib, N, H, W, k, I, a=0.0, frames=12, signal='chirp', fault=None):  # noqa: F811
    """The fp32 emulation fed one frame per call, then ended; every call checked from its own before-state -> ({stage: worst}, fails)."""
    sh = C.Shape(N, H, W, k, I, a, C.fft_plan(lib, N))
    w32 = O.hann(W, N).astype(np.float32)
    S = _spec(N, H, W, frames, signal)
    st = L.empty_slot(L.GlLayout(N, k))
    worst, fails = {}, []
    rows = [((t + 1, False), S[:, t:t + 1].T) for t in range(frames)] + [((frames, True), None)]
    for row, new in rows:
        exp = C.one_call(st, new, row, sh, w32)
        got, out = C.emulate_call(st, new, row, sh, w32, fault)
        for name, r in C.compare(exp, got, out, a0=float(np.float32(a)) == 0).items():
            worst[name] = max(worst.get(name, 0.0), r)
        fails += C.exact_checks(st, got, out, row, sh, w32, exp)
        st = got
    return worst, fails


EMULATED = [(1102, 275, 1102, 3, 2, 0.0), (1102, 275, 1102, 0, 1, 0.97), (546, 136, 545, 1, 2, 0.0), (800, 200, 800, 2, 1, 0.97),
            (1426, 356, 1426, 4, 1, 0.0), (1100, 1100, 1100, 1, 2, 0.0), (4, 2, 4, 7, 2, 0.0)]


@pytest.mark.parametrize('N,H,W,k,I,a', EMULATED)
def test_fp32_emulation_passes_every_bound(lib, N, H, W, k, I, a):  # noqa: F811
    worst, fails = recorded(lib, N, H, W, k, I, a)
    print(f'\nfp32 emulation N={N} H={H} W={W} k={k} I={I} a={a}:', {s: f'{r:.2e}' for s, r in sorted(worst.items())})
    assert not fails, fails
    assert all(r <= 1 for r in worst.values()), worst


def crafted(lib, N, H, W, k, m, kind, admit=False, fault=None, seed=0):  # noqa: F811
    """One call from a crafted single-pass state (gl_stream_check.crafted_state), fp32 emulation against one_call."""
    sh = C.Shape(N, H, W, k, 1, 0.0, C.fft_plan(lib, N))
    w32 = O.hann(W, N).astype(np.float32)
    before, new, row = C.crafted_state(sh, w32, m, kind, np.random.default_rng(seed), admit)
    exp = C.one_call(before, new, row, sh, w32)
    got, out = C.emulate_call(before, new, row, sh, w32, fault)
    return C.compare(exp, got, out), C.exact_checks(before, got, out, row, sh, w32, exp)


@pytest.mark.parametrize('kind', ['noise', 'zero', 'tone', 'tiny'])
@pytest.mark.parametrize('N,H,W,k', [(1102, 275, 1102, 3), (546, 136, 545, 0), (1922, 480, 1922, 5), (4, 2, 4, 1)])
def test_fp32_emulation_passes_crafted_single_steps(lib, N, H, W, k, kind):  # noqa: F811
    for m in (0, 1, 12, L.max_frames(N, H) - k - 1):
        for admit in (False, True):
            worst, fails = crafted(lib, N, H, W, k, m, kind, admit)
            assert not fails, (m, admit, fails)
            assert all(r <= 1 for r in worst.values()), (m, admit, worst)


# a planted fault, and the stream (recorded: one frame per call) or crafted state that shows it
FAULT_CASES = {'window_lpad_off_by_one': ('recorded', 546, 136, 545, 1, 1, 0.0),
               'tail_release_frames_F_minus_2': ('recorded', 1102, 275, 1102, 0, 1, 0.0),
               'carry_reset_per_call': ('recorded', 1102, 275, 1102, 1, 1, 0.97),
               'gauss_seidel': ('crafted', 1102, 275, 1102, 2, 12, 'noise'),
               'admission_includes_own_frame': ('crafted', 1102, 275, 1102, 2, 12, 'zero', True)}


@pytest.mark.parametrize('fault', C.FAULTS)
def test_planted_faults_fail(lib, fault):  # noqa: F811
    how, *args = FAULT_CASES.get(fault, ('recorded', 1102, 275, 1102, 2, 1, 0.0))
    worst, fails = (recorded if how == 'recorded' else crafted)(lib, *args, fault=fault)
    bad = {s: r for s, r in worst.items() if r > 1}
    print(f'\n{fault}:', bad, fails[:3])
    assert bad or fails, worst
