"""The waveform front end on the H100: resample_batch against the fp64 oracle (tests/resample_oracle.py) on ragged batches that mix source
rates, the equal-rate identity, batch independence, guard regions, a waveform whose n down passes 2^31, and trim_silence_batch's bounds
and frame powers against the oracle, with the trimmed audio returned as the caller's own samples."""
import ctypes
import math

import numpy as np
import pytest
import torch

import resample_oracle as O

pytestmark = pytest.mark.gpu

SR = 22050
SOURCES = (8000, 16000, 22050, 24000, 44100, 48000)


@pytest.fixture(scope='module', autouse=True)
def _built():
    import __graft_entry__ as entry
    entry.build()
    assert torch.cuda.is_available(), 'GPU tests need a CUDA device'


def ratio(a, b):
    g = math.gcd(a, b)
    return b // g, a // g


def speech_like(n, sr, rng):
    """A harmonic glide with a little noise."""
    t = np.arange(n) / sr
    f = rng.uniform(90, 250) * 2 ** (0.5 * np.sin(2 * np.pi * rng.uniform(0.2, 1.0) * t))
    ph = 2 * np.pi * np.cumsum(f) / sr
    return 0.4 * np.sin(ph) + 0.2 * np.sin(2 * ph) + 0.01 * rng.standard_normal(n)


def ragged(count, seed, rates):
    """Seeded waveforms of up to 10 s at rates drawn from `rates` -> (fp32 waveforms, their rates)."""
    rng = np.random.default_rng(seed)
    srs = [int(rng.choice(rates)) for _ in range(count)]
    lengths = [int(rng.uniform(0.01, 10.0) * sr) for sr in srs]
    if count >= 7:
        lengths[:3] = [1, 2, 5]
    return [speech_like(n, sr, rng).astype(np.float32) for n, sr in zip(lengths, srs)], srs


def check_against_oracle(x, y, up, down, n=None):
    want, mag = O.resample(x.astype(np.float64), up, down, n)
    got = y if n is None else y[n]
    assert len(got) == len(want)
    err = np.abs(got.astype(np.float64) - want)
    bound = np.spacing(np.abs(want).astype(np.float32)).astype(np.float64) + 1e-12 * mag
    assert (err <= bound).all(), (up, down, np.flatnonzero(err > bound)[:5], err[err > bound][:5])
    big = np.abs(want) > 1e-3
    return float((err[big] / np.spacing(np.abs(want[big]).astype(np.float32))).max(initial=0.0))


@pytest.mark.parametrize('count', [1, 7, 64])
def test_resample_batch_matches_the_oracle(count):
    from multilingual_text_to_speech_b200.utils import audio
    worst = 0.0
    waves, srs = ragged(count, 100 + count, SOURCES)
    outs = audio.resample_batch(waves, srs, SR)
    for x, sr, y in zip(waves, srs, outs):
        assert isinstance(y, np.ndarray) and y.dtype == np.float32
        up, down = ratio(sr, SR)
        if sr == SR:
            assert np.array_equal(y, x)
            continue
        worst = max(worst, check_against_oracle(x, y, up, down))
    for target in (16000, 44100):
        waves = ragged(count, 200 + count + target, (SR,))[0]
        up, down = ratio(SR, target)
        for x, y in zip(waves, audio.resample_batch(waves, SR, target)):
            worst = max(worst, check_against_oracle(x, y, up, down))
    print(f'{count} waveforms: worst {worst:.3f} fp32 ulps from the fp64 oracle where |y| > 1e-3')


def test_equal_rates_return_the_fp32_input():
    from multilingual_text_to_speech_b200.utils import audio
    x = np.random.default_rng(1).standard_normal(5000)
    y = audio.resample(x, 22050, 22050)
    assert y.dtype == np.float32 and np.array_equal(y, x.astype(np.float32))
    t = torch.from_numpy(x.astype(np.float32)).cuda()
    yt = audio.resample(t, 16000, 16000)
    assert yt.is_cuda and torch.equal(yt, t) and yt.data_ptr() != t.data_ptr()
    yc = audio.resample(torch.from_numpy(x), SR)
    assert not yc.is_cuda and yc.dtype == torch.float32 and np.array_equal(yc.numpy(), x.astype(np.float32))


def test_each_waveform_is_bit_identical_alone_and_in_any_batch():
    from multilingual_text_to_speech_b200.utils import audio
    waves, srs = ragged(64, 7, SOURCES)
    together = audio.resample_batch(waves, srs)
    order = np.random.default_rng(5).permutation(len(waves))
    shuffled = audio.resample_batch([waves[i] for i in order], [srs[i] for i in order])
    for b in range(len(waves)):
        alone = audio.resample(waves[b], srs[b])
        assert np.array_equal(alone, together[b])
        assert np.array_equal(shuffled[int(np.flatnonzero(order == b)[0])], together[b])
    t = audio.resample_batch([torch.from_numpy(w).cuda() for w in waves[:5]], srs[:5])
    assert all(y.is_cuda and np.array_equal(y.cpu().numpy(), together[i]) for i, y in enumerate(t))


def _launch(waves, ratios, guard):
    """b200tts_resample on a packed batch, the output inside NaN guard regions -> (guarded buffer, host output offsets)."""
    from multilingual_text_to_speech_b200 import _lib
    from multilingual_text_to_speech_b200.utils import audio
    dev = torch.device('cuda:0')
    pairs = sorted(set(ratios))
    tables = [audio._resample_table(up, down, dev) for up, down in pairs]
    toff = np.concatenate([[0], np.cumsum([len(t) for t in tables])])
    plan = np.array([[up, down, 10 * max(up, down), toff[pairs.index((up, down))]] for up, down in ratios], dtype=np.int32)
    soff = np.concatenate([[0], np.cumsum([len(w) for w in waves])])
    ooff = np.concatenate([[0], np.cumsum([O.out_length(len(w), up, down) for w, (up, down) in zip(waves, ratios)])])
    shape = _lib.ResampleShape(len(waves), int(soff[-1]), int(ooff[-1]), int(toff[-1]), max(max(p) for p in pairs))
    wave = torch.from_numpy(np.concatenate(waves).astype(np.float32)).to(dev)
    d_soff, d_ooff = (torch.from_numpy(o.astype(np.int32)).to(dev) for o in (soff, ooff))
    d_plan, taps = torch.from_numpy(plan).to(dev), torch.cat(tables)
    buf = torch.full((int(ooff[-1]) + 2 * guard,), float('nan'), dtype=torch.float32, device=dev)
    ptr = lambda t: ctypes.c_void_p(t.data_ptr())          # noqa: E731
    lib = _lib.load()
    assert lib.b200tts_resample(ctypes.byref(shape), ptr(wave), ptr(d_soff), ptr(d_ooff), ptr(d_plan), ptr(taps), ptr(buf[guard:]),
                                ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)) == 0, lib.b200tts_last_error()
    torch.cuda.synchronize()
    return buf, ooff


def test_kernel_writes_nothing_outside_its_output():
    guard = 4096
    for count in (1, 7, 64):
        waves, srs = ragged(count, 300 + count, SOURCES + (11025, 96000))
        ratios = [ratio(sr, SR) if sr != SR else (2, 1) for sr in srs]
        buf, ooff = _launch(waves, ratios, guard)
        total = int(ooff[-1])
        assert bool(torch.isnan(buf[:guard]).all()) and bool(torch.isnan(buf[guard + total:]).all())
        assert bool(torch.isfinite(buf[guard:guard + total]).all())


def test_n_down_beyond_two_to_the_thirty_one():
    """One waveform of 2^25 samples at 16 kHz -> 22,050 Hz: n down passes 2^31 from output 6,710,887 on.  A strided subset of outputs,
    both ends and the outputs around the crossing, against the oracle."""
    L = 1 << 25
    up, down = ratio(16000, SR)
    x = (0.5 * np.sin(2 * np.pi * 0.01 * np.arange(L)) + 0.05 * np.random.default_rng(9).standard_normal(L)).astype(np.float32)
    buf, ooff = _launch([x], [(up, down)], 1024)
    Lp = int(ooff[-1])
    assert Lp == O.out_length(L, up, down) and (Lp - 1) * down > 2 ** 31
    cross = 2 ** 31 // down
    n = np.unique(np.concatenate([np.arange(3000), np.arange(Lp - 3000, Lp), np.arange(cross - 500, cross + 500),
                                  np.arange(0, Lp, 4099)]))
    y = buf[1024:1024 + Lp][torch.from_numpy(n).cuda()].cpu().numpy()
    full = np.full(Lp, np.nan, dtype=np.float32)
    full[n] = y
    check_against_oracle(x, full, up, down, n)
    assert bool(torch.isnan(buf[:1024]).all()) and bool(torch.isnan(buf[1024 + Lp:]).all())


# ---- trimming --------------------------------------------------------------------------------------------------------------------------
W_MS, HOP_MS = 50, 12.5
W, HOP = 1102, 275


def floored(n, rng):
    """Speech-like audio between noise floors of different levels (some under the threshold, some over) at both ends."""
    lead, tail = (int(rng.uniform(0, 1.5) * SR) for _ in range(2))
    body = speech_like(n, SR, rng)
    levels = 10.0 ** rng.uniform(-5, -1, 2)
    return np.concatenate([levels[0] * rng.standard_normal(lead), body, levels[1] * rng.standard_normal(tail)]).astype(np.float32)


def trim_cases(count, seed):
    rng = np.random.default_rng(seed)
    waves = [floored(int(rng.uniform(0.01, 8.0) * SR), rng) for _ in range(count)]
    if count > 1:
        waves[1] = np.zeros(int(rng.integers(1, 20000)), dtype=np.float32)
        waves[-1] = waves[-1][:int(rng.integers(1, 500))]
    return waves


@pytest.mark.parametrize('count', [1, 7, 64])
@pytest.mark.parametrize('top_db,margin_ms', [(50, 0), (40, 10), (60, 0)])
def test_trim_bounds_match_the_oracle(count, top_db, margin_ms):
    from multilingual_text_to_speech_b200.utils import audio
    waves = trim_cases(count, 17 * count + top_db)
    M = audio.ms_to_frames(margin_ms)
    waves = [w for w in waves if len(w) > 2 * M]
    got = audio.trim_silence_batch(waves, W_MS, HOP_MS, top_db=top_db, margin_ms=margin_ms)
    for i, (x, (y, index)) in enumerate(zip(waves, got)):
        (start, end), db = O.trim(x.astype(np.float64), W, HOP, top_db, M)
        # fp64 sums in another order move a frame's dB by far less than 1e-6: no decision can flip
        assert np.abs(db + top_db).min() > 1e-6, (i, np.abs(db + top_db).min())
        assert index.dtype == np.int64 and index.shape == (2,) and (int(index[0]), int(index[1])) == (start, end), (i, index, start, end)
        assert np.array_equal(y, x[M:len(x) - M][start:end])


def test_frame_powers_match_the_oracle():
    from multilingual_text_to_speech_b200 import _lib
    from multilingual_text_to_speech_b200 import functional as F
    waves = trim_cases(7, 3) + [np.array([0.25], dtype=np.float32), np.arange(5, dtype=np.float32)]
    soff = np.concatenate([[0], np.cumsum([len(w) for w in waves])])
    frames = [1 + (len(w) + 2 * (W // 2) - W) // HOP for w in waves]
    foff = np.concatenate([[0], np.cumsum(frames)])
    shape = _lib.TrimShape(len(waves), int(soff[-1]), int(foff[-1]), W, HOP, 50.0)
    dev = torch.device('cuda:0')
    wave = torch.from_numpy(np.concatenate(waves)).to(dev)
    power, bounds = F.trim_silence(shape, wave, *(torch.from_numpy(o.astype(np.int32)).to(dev) for o in (soff, foff)))
    power = power.cpu().numpy()
    for b, x in enumerate(waves):
        want = O.frame_power(x.astype(np.float64), W, HOP)
        np.testing.assert_allclose(power[foff[b]:foff[b + 1]], want, rtol=1e-12, atol=0)
        assert tuple(bounds[b].tolist()) == O.trim(x.astype(np.float64), W, HOP)[0]


def test_trimmed_audio_is_the_callers_own():
    from multilingual_text_to_speech_b200.utils import audio
    rng = np.random.default_rng(21)
    x = np.concatenate([np.zeros(8000), speech_like(20000, SR, rng), np.zeros(9000)])          # float64
    M = audio.ms_to_frames(5)
    (start, end), _ = O.trim(x.astype(np.float32).astype(np.float64), W, HOP, 50, M)
    y, index = audio.trim_silence(x, W_MS, HOP_MS, margin_ms=5)
    assert y.dtype == np.float64 and np.shares_memory(y, x) and (index[0], index[1]) == (start, end)
    assert y.ctypes.data == x.ctypes.data + 8 * (M + start) and len(y) == end - start
    for t in (torch.from_numpy(x), torch.from_numpy(x).cuda(), torch.from_numpy(x.astype(np.float32)).cuda()):
        y, index = audio.trim_silence(t, W_MS, HOP_MS, margin_ms=5)
        assert y.device == t.device and y.dtype == t.dtype and y.untyped_storage().data_ptr() == t.untyped_storage().data_ptr()
        assert y.data_ptr() == t.data_ptr() + t.element_size() * (M + start) and (index[0], index[1]) == (start, end)


def test_trim_results_are_batch_independent():
    from multilingual_text_to_speech_b200.utils import audio
    waves = trim_cases(64, 8)
    together = audio.trim_silence_batch(waves, W_MS, HOP_MS, top_db=40)
    order = np.random.default_rng(2).permutation(len(waves))
    shuffled = audio.trim_silence_batch([waves[i] for i in order], W_MS, HOP_MS, top_db=40)
    for b in range(len(waves)):
        alone = audio.trim_silence(waves[b], W_MS, HOP_MS, top_db=40)[1]
        assert np.array_equal(alone, together[b][1])
        assert np.array_equal(shuffled[int(np.flatnonzero(order == b)[0])][1], together[b][1])


def test_front_end_chain_stays_on_the_device():
    """48 and 16 kHz recordings with silent ends -> resample_batch -> trim_silence_batch -> spectrogram_batch, all CUDA tensors."""
    from multilingual_text_to_speech_b200.utils import audio
    rng = np.random.default_rng(4)
    srs = [48000, 16000]
    ys = [torch.from_numpy(np.concatenate([np.zeros(sr // 2), speech_like(sr, sr, rng), np.zeros(sr // 3)]).astype(np.float32)).cuda()
          for sr in srs]
    ys = audio.resample_batch(ys, srs)
    assert all(y.is_cuda and abs(len(y) - int(SR * 1.8333)) < 3 for y in ys)
    trimmed = [y for y, _ in audio.trim_silence_batch(ys, 50, 12.5, top_db=40)]
    assert all(y.is_cuda and abs(len(y) - SR) <= 2 * W for y in trimmed)
    mels = audio.spectrogram_batch(trimmed, mel=True)
    assert all(m.is_cuda and m.shape[1] == 1 + len(y) // HOP for m, y in zip(mels, trimmed))
