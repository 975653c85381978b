"""Pitch analysis on the H100: each pYIN stage against the numpy oracle (tests/pitch_oracle.py) from the previous stage's GPU output,
pitch_batch end to end, batch independence, per-symbol averages on Tacotron.align durations and the export tool's pitch and energy files."""
import numpy as np
import pytest
import torch

import model_cases
import pitch_oracle as P
from helpers import Golden
from test_pitch_cpu import glide, noise, tone

pytestmark = pytest.mark.gpu

SR, HOP = 22050, 275


@pytest.fixture(scope='module', autouse=True)
def _built():
    import __graft_entry__ as entry
    entry.build()
    assert torch.cuda.is_available(), 'GPU tests need a CUDA device'


def _signals():
    return [tone(80.0, 0.3), tone(123.0, 0.25), tone(200.0, 0.3), tone(311.0, 0.2), tone(400.0, 0.25), glide(120.0, 180.0, 0.4),
            noise(0.2), np.zeros(3000), np.concatenate([tone(150.0, 0.15), np.zeros(2500), tone(250.0, 0.15)]),
            np.float32(0.3) * tone(95.0, 0.02), np.array([0.25])]


def _ragged(count, seed):
    rng = np.random.default_rng(seed)
    out = []
    for i in range(count):
        sec = float(rng.uniform(0.05, 0.3))
        kind = i % 4
        if kind == 0:
            out.append(tone(float(rng.uniform(70, 450)), sec))
        elif kind == 1:
            out.append(glide(float(rng.uniform(90, 200)), float(rng.uniform(90, 200)), sec))
        elif kind == 2:
            out.append(noise(sec, seed=i))
        else:
            out.append(np.concatenate([tone(float(rng.uniform(70, 450)), sec / 2), np.zeros(int(rng.integers(1, 3000)))]))
    return out


def _stages(waves, fmin=65.406, fmax=2093.0, frame_length=1024):
    """Every stage on the GPU: (shape, host frame offsets, d', obs, voiced_prob, state, log_trans)."""
    from multilingual_text_to_speech_b200 import functional as F
    from multilingual_text_to_speech_b200.utils import audio
    dev = torch.device('cuda:0')
    lengths = [len(w) for w in waves]
    soff = np.concatenate([[0], np.cumsum(lengths)])
    off = np.concatenate([[0], np.cumsum([1 + n // HOP for n in lengths])])
    shape, log_trans, _ = audio.pitch_shape(len(waves), soff[-1], off[-1], fmin, fmax, frame_length, dev)
    wave = torch.from_numpy(np.concatenate(waves).astype(np.float32)).to(dev)
    d_soff = torch.from_numpy(soff.astype(np.int32)).to(dev)
    d_off = torch.from_numpy(off.astype(np.int32)).to(dev)
    cmnd = F.pitch_cmnd(shape, wave, d_soff, d_off)
    obs, vp = F.pitch_observations(shape, cmnd)
    state = F.pitch_viterbi(shape, obs, vp, d_off, log_trans)
    torch.cuda.synchronize()
    return shape, off, cmnd.cpu().numpy(), obs.cpu().numpy(), vp.cpu().numpy(), state.cpu().numpy(), log_trans


def _near_zeroing(y, g):
    """Frames with an acf or e within 1e-12 of the 1e-6 zeroing threshold, where the two evaluations may fall on either side of it."""
    acf, e = P.difference_terms(P.frames(y, 1024, HOP), g['win_length'], g['max_period'])
    near = lambda v: (np.abs(np.abs(v) - 1e-6) < 1e-12).any(0)    # noqa: E731
    return near(acf) | near(e)


def test_cmnd_matches_the_oracle():
    waves = _signals() + _ragged(12, 1)
    shape, off, got, _, _, _, _ = _stages(waves)
    g = P.geometry(SR, HOP, 65.406, 2093.0, 1024)
    checked = 0
    for b, y in enumerate(waves):
        want = P.cmnd(P.frames(np.asarray(y, dtype=np.float32).astype(np.float64), 1024, HOP), 1024, g['win_length'], g['min_period'],
                      g['max_period']).T
        mine = got[off[b]:off[b + 1]]
        assert mine.shape == want.shape
        keep = ~_near_zeroing(np.asarray(y, dtype=np.float32).astype(np.float64), g)
        # rtol 1e-12, with a floor of 1e-13 for the rounding of the fp64 sums (relative to the frame energy, not to the lag's d)
        err = np.abs(mine[keep] - want[keep])
        assert (err <= 1e-12 * np.abs(want[keep]) + 1e-13).all(), (b, err.max())
        checked += int(keep.sum())
    assert checked > 200


def _oracle_obs(cmnd_rows, n):
    yin = cmnd_rows.T
    return P.observations(yin, P.parabolic_shifts(yin), SR, 65.406, 10, n)


def test_observations_match_the_oracle_from_the_gpu_cmnd():
    waves = _signals() + _ragged(24, 2)
    shape, off, cmnd, obs, vp, _, _ = _stages(waves)
    n = shape.n_bins
    want, want_vp = _oracle_obs(cmnd, n)
    want = want[:n].T
    np.testing.assert_array_equal(obs != 0, want != 0)
    np.testing.assert_allclose(obs, want, rtol=1e-12, atol=1e-15)
    np.testing.assert_allclose(vp, want_vp, rtol=1e-12, atol=1e-15)


def test_viterbi_matches_the_oracle_from_the_gpu_observations():
    waves = _signals() + _ragged(20, 3)
    shape, off, _, obs, vp, state, _ = _stages(waves)
    n, W = shape.n_bins, shape.transition_width
    trans, init = P.transition(n, W), P.p_init(n)
    ties = 0
    for b in range(len(waves)):
        o, v = obs[off[b]:off[b + 1]], vp[off[b]:off[b + 1]]
        full = np.concatenate([o.T, np.tile((1 - v) / n, (n, 1))], 0)
        want, _ = P.viterbi(full, trans, init)
        got = state[off[b]:off[b + 1]].astype(np.int64)
        if not np.array_equal(got, want):
            a, c = P.path_score(full, trans, init, got), P.path_score(full, trans, init, want)
            assert abs(a - c) <= 1e-12 * abs(c), (b, a, c)
            ties += 1
    assert ties <= 2


def _check_end_to_end(waves, got):
    for b, y in enumerate(waves):
        f0, voiced, vp = P.pyin(np.asarray(y, dtype=np.float32).astype(np.float64), SR, HOP)
        g_f0, g_vp = got[b]
        assert g_f0.dtype == np.float32 and g_vp.dtype == np.float32 and g_f0.shape == f0.shape == (1 + len(y) // HOP,)
        np.testing.assert_array_equal(~np.isnan(g_f0), voiced)
        np.testing.assert_array_equal(g_f0[voiced], f0[voiced].astype(np.float32))
        np.testing.assert_allclose(g_vp, vp.astype(np.float32), rtol=1e-6, atol=1e-7)


def test_pitch_batch_end_to_end_on_synthetic_signals():
    from multilingual_text_to_speech_b200.utils import audio
    waves = _signals()
    got = audio.pitch_batch([np.asarray(w, dtype=np.float32) for w in waves])
    _check_end_to_end(waves, got)
    f0, vp = audio.pitch(torch.from_numpy(waves[2].astype(np.float32)).cuda())
    assert f0.is_cuda and vp.is_cuda and np.array_equal(f0.cpu().numpy(), got[2][0], equal_nan=True)


@pytest.mark.parametrize('B', [1, 7, 64])
def test_pitch_batch_end_to_end_on_ragged_batches(B):
    from multilingual_text_to_speech_b200.utils import audio
    waves = [np.asarray(w, dtype=np.float32) for w in _ragged(B, 10 + B)]
    _check_end_to_end(waves, audio.pitch_batch(waves))


def test_each_utterance_is_bit_identical_alone_and_in_any_batch():
    from multilingual_text_to_speech_b200.utils import audio
    waves = [np.asarray(w, dtype=np.float32) for w in _ragged(16, 4)]
    alone = [_stages([w]) for w in waves[:4]]
    batch = _stages(waves)
    order = np.random.default_rng(5).permutation(len(waves))
    shuffled = _stages([waves[i] for i in order])
    for b in range(4):
        _, _, c, o, v, s, _ = alone[b]
        for res, pos in ((batch, b), (shuffled, int(np.flatnonzero(order == b)[0]))):
            off = res[1]
            sl = slice(off[pos], off[pos + 1])
            assert np.array_equal(res[2][sl], c) and np.array_equal(res[3][sl], o)
            assert np.array_equal(res[4][sl], v) and np.array_equal(res[5][sl], s)
    f_alone = audio.pitch_batch(waves[:1])[0][0]
    f_batch = audio.pitch_batch(waves[::-1])[-1][0]
    assert np.array_equal(f_alone, f_batch, equal_nan=True)


def _aligned_golden():
    from multilingual_text_to_speech_b200.rng import MaskSource
    g = Golden('generated_training')
    dev = torch.device('cuda:0')
    model = model_cases.build_model(g, dev)
    batch = {k: v.to(dev) for k, v in g.inputs.items()}
    MaskSource.manual_seed(0)
    res = model.align(batch['text'], batch['text_length'], batch['target'], batch['target_length'], batch.get('speakers'),
                      batch.get('languages'))
    return g, res


def test_symbol_average_on_align_durations():
    from multilingual_text_to_speech_b200 import functional as F
    from multilingual_text_to_speech_b200.params.params import Params as hp
    from multilingual_text_to_speech_b200.utils import audio
    try:
        g, res = _aligned_golden()
        frames = g.inputs['target_length'].tolist()
        rng = np.random.default_rng(0)
        waves = [np.float32(0.5) * tone(float(rng.uniform(90, 300)), ((t - 1) * HOP + 100) / SR) for t in frames]
        waves = [np.asarray(w[:(t - 1) * HOP + 100], dtype=np.float32) for w, t in zip(waves, frames)]
        pitches, energies = audio.pitch_batch(waves), audio.energy_batch(waves)
        T = max(frames)
        f0 = np.zeros((len(waves), T))
        en = np.zeros((len(waves), T))
        voiced = np.zeros((len(waves), T), dtype=bool)
        for b, ((f, _), e) in enumerate(zip(pitches, energies)):
            assert len(f) == len(e) == frames[b]
            f0[b, :len(f)] = np.nan_to_num(f)
            voiced[b, :len(f)] = ~np.isnan(f)
            en[b, :len(e)] = e
        d = res.durations.cpu()
        got_p = F.symbol_average(torch.from_numpy(f0), d, torch.from_numpy(voiced)).numpy()
        got_e = F.symbol_average(torch.from_numpy(en).cuda(), res.durations).cpu().numpy()
        d = d.numpy()
        for b in range(len(waves)):
            ends = np.cumsum(d[b])
            for l in range(d.shape[1]):
                fr = slice(ends[l] - d[b, l], ends[l])
                v = voiced[b, fr]
                want_p = f0[b, fr][v].sum() / v.sum() if v.any() else 0.0
                want_e = en[b, fr].sum() / d[b, l] if d[b, l] else 0.0
                assert abs(got_p[b, l] - want_p) <= 1e-12 * abs(want_p) and abs(got_e[b, l] - want_e) <= 1e-12 * abs(want_e)
        assert (got_p[np.arange(d.shape[1])[None, :] < g.inputs['text_length'].numpy()[:, None]] > 0).mean() > 0.5
    finally:
        hp.reset()


def test_export_writes_pitch_and_energy(tmp_path):
    import importlib.util
    import os
    from helpers import ROOT
    from multilingual_text_to_speech_b200.params.params import Params as hp
    spec = importlib.util.spec_from_file_location('export_alignments', os.path.join(ROOT, 'tools', 'export_alignments.py'))
    tool = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(tool)
    try:
        g = Golden('generated_training')
        model = model_cases.build_model(g, torch.device('cuda:0'))
        i = g.inputs
        items = [(0, int(i['languages'][b]), i['text'][b, :int(i['text_length'][b])].tolist(),
                  i['target'][b, :, :int(i['target_length'][b])].numpy(), None) for b in range(g.B)]
        waves = [tone(100.0 + 20 * b, (int(i['target_length'][b]) * HOP) / SR) for b in range(g.B)]
        ids = [f'utt{b:03}' for b in range(g.B)]
        tool.export(model, tool.ItemDataset(items), ids, str(tmp_path), batch_size=4, waveforms=waves)
        for b, uid in enumerate(ids):
            L = len(items[b][2])
            pitch = np.load(os.path.join(tmp_path, f'{uid}.pitch.npy'))
            energy = np.load(os.path.join(tmp_path, f'{uid}.energy.npy'))
            assert pitch.shape == energy.shape == (L,) and pitch.dtype == energy.dtype == np.float64
            assert np.isfinite(pitch).all() and (energy >= 0).all()
            assert np.load(os.path.join(tmp_path, f'{uid}.durations.npy')).shape == (L,)
    finally:
        hp.reset()


def test_energy_batch_is_the_norm_of_the_linear_magnitudes():
    from multilingual_text_to_speech_b200 import functional as F
    from multilingual_text_to_speech_b200.utils import audio
    waves = [np.asarray(w, dtype=np.float32) for w in _ragged(5, 6)]
    got = audio.energy_batch(waves)
    dev = torch.device('cuda:0')
    for w, e in zip(waves, got):
        shape = audio.analysis_shape(1, len(w), 1 + len(w) // HOP, False)
        S = F.stft_magnitude(shape, torch.from_numpy(w).to(dev), torch.tensor([0, len(w)], dtype=torch.int32, device=dev),
                             torch.tensor([0, 1 + len(w) // HOP], dtype=torch.int32, device=dev)).cpu().numpy().astype(np.float64)
        np.testing.assert_allclose(e, np.sqrt((S ** 2).sum(1)), rtol=1e-6)
