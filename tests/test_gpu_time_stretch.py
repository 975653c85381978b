"""Time-scale modification on the H100: the search kernel's positions and the overlap-add against the numpy oracle (tests/wsola_oracle.py),
identity at rate 1 and at unchanged durations, batch independence, time_stretch_batch and retime_batch end to end re-tracked by
pitch_batch, a retime of the Griffin-Lim output of a golden model, an overlap-add of more than 2^30 output samples, and compute-sanitizer
memcheck and racecheck runs of both kernels."""
import numpy as np
import pytest
import torch

import model_cases
import wsola_oracle as O
from helpers import Golden
from test_pitch_cpu import tone
from test_time_stretch_cpu import CASES, SEGMENT_TONES, partition, retime_targets, segmented_tones

pytestmark = pytest.mark.gpu

SR, HOP = 22050, 275


@pytest.fixture(scope='module', autouse=True)
def _built():
    import __graft_entry__ as entry
    entry.build()
    assert torch.cuda.is_available(), 'GPU tests need a CUDA device'


def _run(waves, plans):
    """Both kernels on cuda:0 for plans (L', warp) -> positions int64 per utterance, y fp32 numpy per utterance."""
    from multilingual_text_to_speech_b200 import _lib
    from multilingual_text_to_speech_b200 import functional as F
    dev = torch.device('cuda:0')
    soff = np.concatenate([[0], np.cumsum([len(w) for w in waves])])
    ooff = np.concatenate([[0], np.cumsum([Lp for Lp, _ in plans])])
    foff = np.concatenate([[0], np.cumsum([len(t) for _, t in plans])])
    shape = _lib.WsolaShape(len(waves), int(soff[-1]), int(ooff[-1]), int(foff[-1]), HOP, HOP)
    wave = torch.from_numpy(np.concatenate(waves).astype(np.float32)).to(dev)
    d_soff, d_ooff, d_foff = (torch.from_numpy(o.astype(np.int32)).to(dev) for o in (soff, ooff, foff))
    warp = torch.from_numpy(np.concatenate([t for _, t in plans])).to(dev)
    pos = F.wsola_positions(shape, wave, d_soff, warp, d_foff)
    y = F.wsola_overlap_add(shape, wave, d_soff, pos, d_foff, d_ooff).cpu().numpy()
    pos = pos.cpu().numpy().astype(np.int64)
    return [pos[foff[b]:foff[b + 1]] for b in range(len(waves))], [y[ooff[b]:ooff[b + 1]] for b in range(len(waves))]


def _plan(i, x, rng):
    """Alternately a stretch at a random rate and a retime to randomly perturbed durations (some symbols dropped or held)."""
    from multilingual_text_to_speech_b200.utils import audio
    if i % 2 == 0:
        return audio._stretch_plan(len(x), HOP, float(rng.uniform(0.25, 4.0)))
    F = 1 + len(x) // HOP
    d = partition(F, int(rng.integers(1, 40)), int(rng.integers(1 << 30)))
    dp = np.maximum(0, np.rint(d * rng.uniform(0.3, 2.5, len(d)))).astype(np.int64)
    dp[int(rng.integers(len(dp)))] += 1
    return audio._retime_plan(len(x), HOP, d, dp)


def _ragged(count, seed):
    """Seeded harmonic glides with noise and a silent stretch, up to about 10 s, each with a stretch or a retime."""
    rng = np.random.default_rng(seed)
    waves = []
    for _ in range(count):
        n = int(rng.uniform(0.05, 10.0) * SR)
        t = np.arange(n) / SR
        f = rng.uniform(90, 250) * 2 ** (0.5 * np.sin(2 * np.pi * rng.uniform(0.2, 1.0) * t))
        ph = 2 * np.pi * np.cumsum(f) / SR
        y = 0.4 * np.sin(ph) + 0.2 * np.sin(2 * ph) + 0.01 * rng.standard_normal(n)
        y[int(rng.uniform(0, 1) * n):][:int(rng.uniform(0, 0.3) * n)] = 0.0
        waves.append(y.astype(np.float32))
    return waves, [_plan(i, x, rng) for i, x in enumerate(waves)]


def _cpu_cases():
    rng = np.random.default_rng(0)
    waves = [np.asarray(x, np.float32) for _, x in CASES]
    return waves, [_plan(i, x, rng) for i, x in enumerate(waves)]


@pytest.fixture(scope='module')
def batches():
    return [_cpu_cases()] + [_ragged(B, 40 + B) for B in (1, 7, 64)]


def test_positions_match_the_oracle(batches):
    """Each frame's search against the oracle's from the GPU's previous position; every frame except in the 64-waveform batch, where 24
    frames per utterance (the first, the last and 22 at random) keep the file's run time to minutes."""
    rng = np.random.default_rng(1)
    checked = 0
    for waves, plans in batches:
        got, _ = _run(waves, plans)
        for x, (Lp, tau), p in zip(waves, plans, got):
            a = O.nominal(tau, len(x))
            assert p[0] == a[0]
            ks = np.arange(1, len(tau))
            if len(waves) == 64 and len(ks) > 24:
                ks = np.unique(np.concatenate([[1, len(tau) - 1], rng.choice(ks, 22, replace=False)]))
            for k in ks:
                want = a[k] + O.search(x, int(a[k]), int(p[k - 1]), HOP, HOP)[0]
                assert p[k] == want, (len(x), int(k), int(p[k]), int(want))
                checked += 1
    print(f'positions: {checked} frames equal to the oracle')


def _ulps(got, want):
    w = want.astype(np.float32)
    return np.abs(got.astype(np.float64) - w.astype(np.float64)) / np.spacing(np.abs(w))


def test_overlap_add_matches_the_oracle_from_the_gpu_positions(batches):
    worst = 0.0
    for waves, plans in batches:
        got, ys = _run(waves, plans)
        for b, (x, (Lp, _)) in enumerate(zip(waves, plans)):
            want = O.overlap_add_fast(x, got[b], HOP, Lp)
            assert len(ys[b]) == Lp
            floor = np.spacing(np.float32(2.0 ** -40 * max(float(np.abs(x).max()), 1e-30)))
            err = np.abs(ys[b].astype(np.float64) - want.astype(np.float32).astype(np.float64))
            ok = err <= 2 * np.maximum(np.spacing(np.abs(want.astype(np.float32))), floor)
            assert ok.all(), (b, np.flatnonzero(~ok)[:5], _ulps(ys[b], want)[~ok][:5])
            worst = max(worst, float(_ulps(ys[b], want)[np.abs(want) > 1e-6].max(initial=0.0)))
    print(f'overlap-add: worst {worst:.2f} fp32 ulps from the fp64 oracle')


def test_identity_at_rate_one_and_unchanged_durations(batches):
    from multilingual_text_to_speech_b200.utils import audio
    for waves, _ in batches[:3]:
        same = [partition(1 + len(x) // HOP, 7, i) for i, x in enumerate(waves)]
        for ys in (audio.time_stretch_batch(waves, 1.0), audio.retime_batch(waves, same, same)):
            for x, y in zip(waves, ys):
                assert isinstance(y, np.ndarray) and y.dtype == np.float32 and y.shape == x.shape
                assert np.abs(y.astype(np.float64) - x).max() <= 1e-6 * max(float(np.abs(x).max()), 1e-30)


def test_each_utterance_is_bit_identical_alone_and_in_any_batch(batches):
    waves, plans = batches[2]
    _, together = _run(waves, plans)
    order = np.random.default_rng(5).permutation(len(waves))
    _, shuffled = _run([waves[i] for i in order], [plans[i] for i in order])
    for b in range(len(waves)):
        _, alone = _run([waves[b]], [plans[b]])
        assert np.array_equal(alone[0], together[b])
        assert np.array_equal(shuffled[int(np.flatnonzero(order == b)[0])], together[b])
    from multilingual_text_to_speech_b200.utils import audio
    a = audio.time_stretch_batch(waves[:3], [0.7, 1.3, 2.9])
    c = audio.time_stretch_batch(waves[2::-1], [2.9, 1.3, 0.7])
    assert all(np.array_equal(a[i], c[2 - i]) for i in range(3))


@pytest.mark.parametrize('f', [100.0, 160.0, 300.0])
def test_time_stretch_batch_keeps_f0(f):
    from multilingual_text_to_speech_b200.utils import audio
    x = tone(f, 2.0).astype(np.float32)
    rates = [0.5, 0.8, 1.25, 2.0]
    f_src, _ = audio.pitch(x)
    outs = audio.time_stretch_batch([x] * len(rates), rates)
    tracks = audio.pitch_batch(outs)
    for r, y, (g, _) in zip(rates, outs, tracks):
        assert len(y) == int(round(len(x) / r))
        inner = np.arange(4, len(g) - 4)
        src = f_src[np.minimum(np.rint(inner * r).astype(int), len(f_src) - 1)]
        err = audio.pitch_errors_batch([src], [g[inner]])
        print(f'{f:g} Hz at rate {r}: gpe {err["gpe"][0]}, vde {err["vde"][0]}, f0 rmse {err["f0_rmse_cents"][0]:.2f} cents')
        assert err['gpe'][0] == 0.0 and err['vde'][0] == 0.0, (f, r)
    t = torch.from_numpy(x).cuda()
    y = audio.time_stretch(t, 1.25)
    assert y.is_cuda and np.array_equal(y.cpu().numpy(), outs[2])


def test_retime_batch_moves_each_tone_into_its_new_span():
    from multilingual_text_to_speech_b200.utils import audio
    x, d = segmented_tones()
    x = x.astype(np.float32)
    targets = retime_targets(d)
    outs = audio.retime_batch([x] * len(targets), [d] * len(targets), list(targets.values()))
    for (name, dp), y, (g, _) in zip(targets.items(), outs, audio.pitch_batch(outs)):
        Bp = np.concatenate([[0], np.cumsum(dp)])
        assert 1 + len(y) // HOP == Bp[-1] == audio.spectrogram(y).shape[1]
        worst = 0.0
        for j, f in enumerate(SEGMENT_TONES):
            k = np.arange(Bp[j] + 3, Bp[j + 1] - 3)
            assert not np.isnan(g[k]).any(), (name, j)
            cents = np.abs(1200 * np.log2(g[k] / f))
            worst = max(worst, float(cents.max(initial=0.0)))
            assert (cents <= 20.0).all(), (name, j, cents.max())
        print(f'{name}: worst |cents| {worst:.2f}')


def test_retime_of_griffin_lim_synthesis_from_a_golden_model():
    from multilingual_text_to_speech_b200.functional import scale_durations
    from multilingual_text_to_speech_b200.params.params import Params as hp
    from multilingual_text_to_speech_b200.utils import audio
    try:
        g = Golden('generated_training')
        model = model_cases.build_model(g, torch.device('cuda:0')).eval()
        hp.mel_normalize_mean, hp.mel_normalize_variance = -40.0, 15.0          # set by training from its data; the golden carries none
        i = g.inputs
        texts = [i['text'][b, :int(i['text_length'][b])].cuda() for b in range(2)]
        languages = [torch.nn.functional.one_hot(i['languages'][b:b + 1], hp.language_number).float()[:, None, :].expand(1, len(t), -1)
                     .contiguous().cuda() for b, t in enumerate(texts)]
        durations = [torch.full((len(t),), 8, dtype=torch.int64) for t in texts]
        with torch.no_grad():
            specs = model.inference_batch(texts, None, languages, durations=durations)
        specs = [audio.denormalize_spectrogram(s, True) for s in specs]
        phases = [np.random.default_rng(b).uniform(0, 1, (hp.num_fft // 2 + 1, s.shape[1])) for b, s in enumerate(specs)]
        waves = audio.inverse_spectrogram_batch(specs, mel=True, phases=phases)
        ds = []
        for w, d in zip(waves, durations):
            d = d.clone()
            d[-1] += 1 + len(w) // HOP - int(d.sum())          # the vocoder's length decides the mel frames of the waveform
            assert d[-1] >= 0
            ds.append(d)
        new = [scale_durations(d, 1.3) for d in ds]
        outs = audio.retime_batch(waves, ds, new)
        for y, dp in zip(outs, new):
            assert y.is_cuda and bool(torch.isfinite(y).all())
            assert audio.mel_spectrogram(y).shape[1] == int(dp.sum())
    finally:
        hp.reset()


def test_overlap_add_beyond_two_to_the_thirty_output_samples():
    """2^30 + 1 output samples in one batch, a range where a 32-bit grid index or grid stride would overflow: sampled outputs equal the
    oracle's sums, and guard regions on both sides of the output stay untouched."""
    import ctypes
    from multilingual_text_to_speech_b200 import _lib
    dev = torch.device('cuda:0')
    L, Lp, guard = 10000, 2 ** 30 + 1, 4096
    K = (Lp - 1) // HOP + 2
    x = np.random.default_rng(3).standard_normal(L).astype(np.float32)
    p = (np.arange(K, dtype=np.int64) * 7919) % (L + 2 * HOP) - HOP          # positions anywhere in [-H, L + H)
    shape = _lib.WsolaShape(1, L, Lp, K, HOP, HOP)
    wave = torch.from_numpy(x).to(dev)
    pos = torch.from_numpy(p.astype(np.int32)).to(dev)
    soff, ooff, foff = (torch.tensor([0, v], dtype=torch.int32, device=dev) for v in (L, Lp, K))
    buf = torch.full((Lp + 2 * guard,), float('nan'), dtype=torch.float32, device=dev)
    out = buf[guard:guard + Lp]
    ptr = lambda t: ctypes.c_void_p(t.data_ptr())          # noqa: E731
    lib = _lib.load()
    assert lib.b200tts_wsola_overlap_add(ctypes.byref(shape), ptr(wave), ptr(soff), ptr(pos), ptr(foff), ptr(ooff), ptr(out),
                                         ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)) == 0, lib.b200tts_last_error()
    torch.cuda.synchronize()
    assert bool(torch.isnan(buf[:guard]).all()) and bool(torch.isnan(buf[guard + Lp:]).all())
    rng = np.random.default_rng(4)
    n = np.unique(np.concatenate([np.arange(2000), np.arange(Lp - 2000, Lp), rng.integers(0, Lp, 2000), [2 ** 30 - 256, 2 ** 30]]))
    got = out[torch.from_numpy(n).to(dev)].cpu().numpy()
    w = O.window(HOP)
    want = np.zeros(len(n))
    for j in (0, 1):
        k = n // HOP + j
        ok = k < K
        src = np.where(ok, p[np.minimum(k, K - 1)] + n - k * HOP, -1)
        xs = np.where((src >= 0) & (src < L), x[np.clip(src, 0, L - 1)].astype(np.float64), 0.0)
        want = want + np.where(ok, w[n - k * HOP + HOP] * xs, 0.0)
    err = np.abs(got.astype(np.float64) - want.astype(np.float32).astype(np.float64))
    floor = np.spacing(np.float32(2.0 ** -40 * float(np.abs(x).max())))
    assert (err <= 2 * np.maximum(np.spacing(np.abs(want.astype(np.float32))), floor)).all()
    del buf, out


def test_kernels_write_nothing_outside_their_outputs(batches):
    """Both kernels on the ragged batches, with guard regions before and after the positions and the output: the guards stay untouched."""
    import ctypes
    from multilingual_text_to_speech_b200 import _lib
    dev = torch.device('cuda:0')
    lib = _lib.load()
    stream = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    ptr = lambda t: ctypes.c_void_p(t.data_ptr())          # noqa: E731
    guard, sentinel = 1024, -2 ** 31
    for waves, plans in batches:
        soff = np.concatenate([[0], np.cumsum([len(w) for w in waves])])
        ooff = np.concatenate([[0], np.cumsum([Lp for Lp, _ in plans])])
        foff = np.concatenate([[0], np.cumsum([len(t) for _, t in plans])])
        shape = _lib.WsolaShape(len(waves), int(soff[-1]), int(ooff[-1]), int(foff[-1]), HOP, HOP)
        wave = torch.from_numpy(np.concatenate(waves).astype(np.float32)).to(dev)
        d_soff, d_ooff, d_foff = (torch.from_numpy(o.astype(np.int32)).to(dev) for o in (soff, ooff, foff))
        warp = torch.from_numpy(np.concatenate([t for _, t in plans])).to(dev)
        pbuf = torch.full((int(foff[-1]) + 2 * guard,), sentinel, dtype=torch.int32, device=dev)
        obuf = torch.full((int(ooff[-1]) + 2 * guard,), float('nan'), dtype=torch.float32, device=dev)
        pos, out = pbuf[guard:guard + int(foff[-1])], obuf[guard:guard + int(ooff[-1])]
        assert lib.b200tts_wsola_positions(ctypes.byref(shape), ptr(wave), ptr(d_soff), ptr(warp), ptr(d_foff), ptr(pos), stream) == 0
        assert lib.b200tts_wsola_overlap_add(ctypes.byref(shape), ptr(wave), ptr(d_soff), ptr(pos), ptr(d_foff), ptr(d_ooff), ptr(out),
                                             stream) == 0
        torch.cuda.synchronize()
        assert bool((pbuf[:guard] == sentinel).all()) and bool((pbuf[guard + int(foff[-1]):] == sentinel).all())
        assert bool((pos != sentinel).all())
        assert bool(torch.isnan(obuf[:guard]).all()) and bool(torch.isnan(obuf[guard + int(ooff[-1]):]).all())
        assert bool(torch.isfinite(out).all())


@pytest.mark.parametrize('tool', ['memcheck', 'racecheck'])
def test_compute_sanitizer_is_clean(tool):
    """tools/wsola_small.py under compute-sanitizer, only the wsola_ kernels instrumented.  Skipped where the sanitizer is not installed
    or cannot attach to the device; any reported error or hazard fails."""
    import os
    import re
    import shutil
    import signal
    import subprocess
    import sys
    exe = next((c for c in ('/usr/local/cuda/bin/compute-sanitizer', shutil.which('compute-sanitizer')) if c and os.path.exists(c)), None)
    if exe is None:
        pytest.skip('compute-sanitizer not installed')
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    cmd = [exe, '--tool', tool, '--kernel-name', 'kns=wsola_', '--error-exitcode', '3', sys.executable,
           os.path.join(root, 'tools', 'wsola_small.py')]
    proc = subprocess.Popen(cmd, cwd=root, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, start_new_session=True)
    try:
        out, _ = proc.communicate(timeout=900)
    except subprocess.TimeoutExpired:
        os.killpg(proc.pid, signal.SIGKILL)              # the sanitizer and the program it runs: nothing is left behind
        proc.communicate()
        pytest.fail(f'compute-sanitizer {tool} did not finish in 900 s')
    print(out[-3000:])
    summary = re.search(r'(ERROR|RACECHECK) SUMMARY: (\d+)', out)
    # the sanitizer refuses some devices: then the program's first CUDA call fails, before either wsola kernel is reached
    ours = re.search(r'wsola_(search|ola)_kernel|b200tts_wsola|wsola_positions|wsola_overlap_add', out)
    if summary is None or 'Device not supported' in out or ('wsola_small ok' not in out and ours is None):
        pytest.skip(f'compute-sanitizer {tool} could not run the program on this device (exit {proc.returncode}): {out[-400:]}')
    assert int(summary.group(2)) == 0 and proc.returncode == 0 and 'wsola_small ok' in out, out[-3000:]
