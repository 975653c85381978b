"""Pitch shifting on the H100: the marks kernel and the overlap-add against the numpy oracle (tests/psola_oracle.py), the identity at
ratio 1, batch independence, pitch_shift_batch end to end re-tracked by pitch_batch, contour transfer with f0_ratio, and a shift of the
Griffin-Lim output of a golden model."""
import numpy as np
import pytest
import torch

import model_cases
import psola_oracle as O
from helpers import Golden
from test_pitch_cpu import glide, tone
from test_pitch_shift_cpu import CASES, SHIFTS

pytestmark = pytest.mark.gpu

SR, HOP = 22050, 275
RETRACK_FMIN = 45.0          # an octave below 100 Hz is below pitch_batch's default floor


@pytest.fixture(scope='module', autouse=True)
def _built():
    import __graft_entry__ as entry
    entry.build()
    assert torch.cuda.is_available(), 'GPU tests need a CUDA device'


def _run(waves, f0s, ratios):
    """Both kernels on cuda:0 -> (per utterance: dict of marks, d, voiced, a0, c, k), y per utterance (fp32 numpy)."""
    from multilingual_text_to_speech_b200 import _lib
    from multilingual_text_to_speech_b200 import functional as F
    dev = torch.device('cuda:0')
    lengths = [len(w) for w in waves]
    soff = np.concatenate([[0], np.cumsum(lengths)])
    off = np.concatenate([[0], np.cumsum([1 + n // HOP for n in lengths])])
    shape = _lib.PsolaShape(len(waves), int(soff[-1]), int(off[-1]), HOP, HOP, float(SR))
    wave = torch.from_numpy(np.concatenate(waves).astype(np.float32)).to(dev)
    d_soff = torch.from_numpy(soff.astype(np.int32)).to(dev)
    d_off = torch.from_numpy(off.astype(np.int32)).to(dev)
    f0 = torch.from_numpy(np.concatenate(f0s).astype(np.float32)).to(dev)
    r = torch.from_numpy(np.concatenate(ratios).astype(np.float32)).to(dev)
    ws = F.psola_marks(shape, wave, d_soff, f0, r, d_off)
    y = F.psola_overlap_add(shape, wave, d_soff, ws).cpu().numpy()
    info, marks, spacing, centre, nearest, voiced = (t.cpu().numpy() for t in F.psola_workspace_views(shape, ws))
    out = []
    for b in range(len(waves)):
        K, J, a0, _ = info[b]
        s = slice(soff[b], soff[b] + K)
        t = slice(soff[b], soff[b] + J)
        out.append(dict(marks=marks[s], d=spacing[s], voiced=voiced[s].astype(bool), a0=int(a0), c=centre[t], k=nearest[t],
                        W=int(info[b][3])))
    return out, [y[soff[b]:soff[b + 1]] for b in range(len(waves))]


def _ragged(count, seed):
    """Ragged waveforms up to about 10 s with their pitch_batch tracks, and mixed constant and per-frame ratios."""
    from multilingual_text_to_speech_b200.utils import audio
    rng = np.random.default_rng(seed)
    waves = []
    for i in range(count):
        n = int(rng.uniform(0.05, 10.0) * SR)
        t = np.arange(n) / SR
        f = rng.uniform(90, 250) * 2 ** (0.5 * np.sin(2 * np.pi * rng.uniform(0.2, 1.0) * t))
        ph = 2 * np.pi * np.cumsum(f) / SR
        y = 0.4 * np.sin(ph) + 0.2 * np.sin(2 * ph) + 0.01 * rng.standard_normal(n)
        y[int(rng.uniform(0, 1) * n):][:int(rng.uniform(0, 0.3) * n)] = 0.0       # a silent stretch
        waves.append(y.astype(np.float32))
    f0s = [f for f, _ in audio.pitch_batch(waves)]
    ratios = []
    for i, w in enumerate(waves):
        F = 1 + len(w) // HOP
        ratios.append(np.full(F, 2.0 ** (rng.uniform(-12, 12) / 12), np.float32) if i % 2 else
                      rng.uniform(0.5, 2.0, F).astype(np.float32))
    return waves, f0s, ratios


def _cpu_cases():
    waves = [np.asarray(x, np.float32) for _, x, _ in CASES]
    f0s = [f for _, _, f in CASES]
    rng = np.random.default_rng(0)
    ratios = [rng.uniform(0.5, 2.0, len(f)).astype(np.float32) if i % 2 else np.full(len(f), 2 ** (3 / 12), np.float32)
              for i, f in enumerate(f0s)]
    return waves, f0s, ratios


def _batches():
    return [_cpu_cases()] + [_ragged(B, 20 + B) for B in (1, 7, 64)]


@pytest.fixture(scope='module')
def batches():
    return _batches()


def _ulps(got, want):
    """Distance in fp32 ulps of got from want rounded to fp32."""
    w = want.astype(np.float32)
    return np.abs(got.astype(np.float64) - w.astype(np.float64)) / np.spacing(np.abs(w))


def test_marks_match_the_oracle(batches):
    for waves, f0s, ratios in batches:
        got, _ = _run(waves, f0s, ratios)
        for b, (x, f0, r) in enumerate(zip(waves, f0s, ratios)):
            marks, d, voiced, a0 = O.analysis_marks(x, f0, SR, HOP)
            c, k = O.synthesis_marks(len(x), marks, d, voiced, r, HOP)
            g = got[b]
            np.testing.assert_array_equal(g['marks'], marks)
            np.testing.assert_array_equal(g['d'], d)
            np.testing.assert_array_equal(g['voiced'], voiced)
            assert g['a0'] == a0 and g['W'] == max(HOP, a0, int(d.max()))
            np.testing.assert_array_equal(g['c'], c)
            np.testing.assert_array_equal(g['k'], k)


def test_overlap_add_matches_the_oracle_from_the_gpu_marks(batches):
    worst = 0.0
    for waves, f0s, ratios in batches:
        got, ys = _run(waves, f0s, ratios)
        for b, x in enumerate(waves):
            g = got[b]
            want, _ = O.overlap_add(x, g['marks'], g['d'], g['a0'], g['c'], g['k'])
            # 2 ulps of the value, or of 2^-40 max|x| where the weighted sum cancels to near zero
            floor = np.spacing(np.float32(2.0 ** -40 * max(float(np.abs(x).max()), 1e-30)))
            err = np.abs(ys[b].astype(np.float64) - want.astype(np.float32).astype(np.float64))
            ok = err <= 2 * np.maximum(np.spacing(np.abs(want.astype(np.float32))), floor)
            assert ok.all(), (b, np.flatnonzero(~ok)[:5], _ulps(ys[b], want)[~ok][:5])
            worst = max(worst, float(_ulps(ys[b], want)[np.abs(want) > 1e-6].max(initial=0.0)))
    print(f'overlap-add: worst {worst:.2f} fp32 ulps from the fp64 oracle')


def test_identity_at_ratio_one(batches):
    for waves, f0s, _ in batches:
        _, ys = _run(waves, f0s, [np.ones(len(f), np.float32) for f in f0s])
        for x, y in zip(waves, ys):
            assert (_ulps(y, x.astype(np.float64)) <= 1).all()


def test_each_utterance_is_bit_identical_alone_and_in_any_batch(batches):
    waves, f0s, ratios = batches[2]
    _, together = _run(waves, f0s, ratios)
    order = np.random.default_rng(5).permutation(len(waves))
    _, shuffled = _run([waves[i] for i in order], [f0s[i] for i in order], [ratios[i] for i in order])
    for b in range(len(waves)):
        _, alone = _run([waves[b]], [f0s[b]], [ratios[b]])
        assert np.array_equal(alone[0], together[b])
        assert np.array_equal(shuffled[int(np.flatnonzero(order == b)[0])], together[b])
    from multilingual_text_to_speech_b200.utils import audio
    a = audio.pitch_shift_batch(waves[:3], semitones=[2.0, -5.0, 7.0], f0s=f0s[:3])
    c = audio.pitch_shift_batch(waves[2::-1], semitones=[7.0, -5.0, 2.0], f0s=f0s[2::-1])
    assert all(np.array_equal(a[i], c[2 - i]) for i in range(3))


def _inner(F):
    return slice(4, F - 4)


@pytest.mark.parametrize('kind', ['tone100', 'tone160', 'tone300', 'glide'])
def test_pitch_shift_batch_end_to_end(kind):
    from multilingual_text_to_speech_b200.utils import audio
    x = (glide(130.0, 190.0, 2.0) if kind == 'glide' else tone(float(kind[4:]), 2.0)).astype(np.float32)
    f_src, _ = audio.pitch_batch([x], fmin=RETRACK_FMIN)[0]
    s_in = _inner(len(f_src))
    outs = audio.pitch_shift_batch([x] * len(SHIFTS), semitones=list(SHIFTS))
    tracks = audio.pitch_batch(outs, fmin=RETRACK_FMIN)
    for s, y, (f, _) in zip(SHIFTS, outs, tracks):
        assert isinstance(y, np.ndarray) and y.dtype == np.float32 and y.shape == x.shape
        target = f_src * np.float32(2.0 ** (s / 12))
        np.testing.assert_array_equal(~np.isnan(f[s_in]), ~np.isnan(f_src[s_in]))
        cents = np.abs(1200 * np.log2(f[s_in] / target[s_in]))
        err = audio.pitch_errors_batch([target[s_in]], [f[s_in]])
        print(f'{kind} {s:+d} st: median |cents| {np.nanmedian(cents):.2f}, gpe {err["gpe"][0]}')
        assert np.nanmedian(cents) <= 15.0 and err['gpe'][0] == 0.0, (kind, s)
    t = torch.from_numpy(x).cuda()
    y = audio.pitch_shift(t, semitones=3.0)
    assert y.is_cuda and np.array_equal(y.cpu().numpy(), outs[SHIFTS.index(3)])


def test_contour_transfer_on_synthetic_glides():
    from multilingual_text_to_speech_b200.utils import audio
    src = glide(120.0, 180.0, 2.0).astype(np.float32)
    tgt = glide(200.0, 140.0, 2.0).astype(np.float32)
    (f_tgt, _), (f_src, _) = audio.pitch_batch([tgt, src])
    r = audio.f0_ratio(f_tgt, f_src)
    out = audio.pitch_shift_batch([src], ratios=[r], f0s=[f_src])[0]
    f_out, _ = audio.pitch(out)
    s = _inner(len(f_src))
    after = audio.pitch_errors_batch([f_tgt[s]], [f_out[s]])
    before = audio.pitch_errors_batch([f_tgt[s]], [f_src[s]])
    print(f'contour transfer: f0_rmse_cents {after["f0_rmse_cents"][0]:.2f} after, {before["f0_rmse_cents"][0]:.2f} unshifted; '
          f'gpe {after["gpe"][0]} after, {before["gpe"][0]} unshifted')
    assert after['gpe'][0] == 0.0 and after['vde'][0] == 0.0
    assert after['f0_rmse_cents'][0] < 0.1 * before['f0_rmse_cents'][0]


def test_shift_of_griffin_lim_synthesis_from_a_golden_model():
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
        durations = [torch.full((len(t),), 8, dtype=torch.int64) for t in texts]          # a fixed length whatever the stop token does
        with torch.no_grad():
            specs = model.inference_batch(texts, None, languages, durations=durations)
        specs = [audio.denormalize_spectrogram(s, True) for s in specs]
        phases = [np.random.default_rng(b).uniform(0, 1, (hp.num_fft // 2 + 1, s.shape[1])) for b, s in enumerate(specs)]
        waves = audio.inverse_spectrogram_batch(specs, mel=True, phases=phases)
        up = audio.pitch_shift_batch(waves, semitones=3.0)
        same = audio.pitch_shift_batch(waves, semitones=0.0)
        for w, u, z in zip(waves, up, same):
            assert u.is_cuda and u.shape == w.shape and bool(torch.isfinite(u).all())
            assert (_ulps(z.cpu().numpy(), w.cpu().numpy().astype(np.float64)) <= 1).all()
    finally:
        hp.reset()
