"""Streaming synthesis without a GPU: the decoder stream's release rule on recorded stop-logit sequences, the post-net window plan against
the fp64 oracle post-net, the WaveRNN lookahead and window plan against the fp64 upsampling, and argument checks."""
import ctypes
import json
import os

import numpy as np
import pytest
import torch

import wavernn_oracle as O
from helpers import GOLDEN_DIR
from multilingual_text_to_speech_b200 import _lib
from multilingual_text_to_speech_b200.modules.tacotron2 import Decoder, postnet_window, stream_release
from multilingual_text_to_speech_b200.modules.wavernn import WaveRNN
from test_wavernn_cpu import REAL


# ---- decoder stream: which frames each chunk releases ----
def _releases(stop_logits, chunk, r, max_frames, stop_frames, halo=10):
    """Replays the stream's per-chunk release on a recorded stop-logit sequence: -> (frames released after each chunk, the cut)."""
    rule = Decoder._StopRule(stop_frames)
    done, out = 0, []
    steps = max(1, chunk // r)
    while done < max_frames:
        Tc = min(steps, -(-(max_frames - done) // r)) * r
        rule.feed(torch.as_tensor(stop_logits[done:done + Tc]))
        done += Tc
        out.append(stream_release(done, rule.cut, max_frames, halo))
        if rule.cut is not None:
            break
    return out, rule.cut


def _logits(n, fires):
    x = -np.ones(n, dtype=np.float32)
    x[list(fires)] = 1.0
    return x


@pytest.mark.parametrize('chunk, r, fires, max_frames, want', [
    # the cut inside a chunk: stop fires at 50 and twice more (stop_frames 2), cut after frame 53
    (16, 1, [50, 51, 52], 200, [6, 22, 38, 53]),
    # the cut on a chunk boundary: cut = 48 = 3 chunks of 16
    (16, 1, [45, 46, 47], 200, [6, 22, 48]),
    # no cut: max_output_length ends the decode, the last chunk partial (60 = 3 x 16 + 12)
    (16, 1, [], 60, [6, 22, 38, 60]),
    # r = 2: chunks of 7 frames round down to 3 steps (6 frames); the cut after frame 21 falls inside a step
    (7, 2, [18, 19, 20], 200, [0, 2, 8, 21]),
    # a chunk shorter than the halo releases nothing until 10 frames follow
    (4, 1, [], 24, [0, 0, 2, 6, 10, 24]),
])
def test_decoder_stream_release_rule(chunk, r, fires, max_frames, want):
    got, cut = _releases(_logits(300, fires), chunk, r, max_frames, 2)
    assert got == want, got
    assert all(b >= a for a, b in zip(got, got[1:]))
    # the whole stream is the stop cut of the one-shot rule, and no release lags the decoder by more than the halo plus one chunk
    assert got[-1] == min(Decoder._stop_cut(torch.as_tensor(_logits(300, fires)[:max_frames]), 2), max_frames)


def test_postnet_window_plan_reproduces_the_oracle_postnet():
    import oracle.tacotron_oracle as TO
    from multilingual_text_to_speech_b200.params.params import Params as hp
    z = np.load(os.path.join(GOLDEN_DIR, 'inf_lj.npz'))
    meta = json.loads(bytes(z['meta']).decode())
    hp.reset()
    hp.load_state_dict(meta['hp'])
    sd = {k[3:]: torch.from_numpy(z[k]).double() for k in z.files if k.startswith('sd.') and '_postnet' in k}
    T = 57
    pre = torch.from_numpy(np.random.default_rng(0).standard_normal((1, hp.num_mels, T)))
    whole = TO.postnet(sd, hp, pre, None, training=False)
    halo = hp.postnet_blocks * (hp.postnet_kernel_size - 1) // 2
    assert halo == 10
    for chunk in (1, 7, 16, 57):
        released = 0
        for done in range(chunk, T + chunk, chunk):
            final = done >= T
            end = T if final else max(done - halo, 0)
            w0, w1 = postnet_window(released, end, halo, T if final else done)
            if end > released:
                got = TO.postnet(sd, hp, pre[:, :, w0:w1], None, training=False)[:, :, released - w0:end - w0]
                np.testing.assert_allclose(got.numpy(), whole[:, :, released:end].numpy(), rtol=1e-12, atol=1e-12)
            released = end
        assert released == T


# ---- vocoder stream: lookahead and windows ----
def _small():
    torch.manual_seed(3)
    m = WaveRNN(**dict(REAL, res_blocks=1))
    with torch.no_grad():
        for i in (1, 3, 5):
            w = m.upsample.up_layers[i].weight
            w.add_(0.05 * torch.randn_like(w))
        for name, b in m.named_buffers():
            if name.endswith('running_mean'):
                b.copy_(0.1 * torch.randn_like(b))
    return m


def _windowed_features(m, p, mel, s0, s1, known, final):
    """fp64 features of positions [s0, s1) computed on the windows of window_plan, [s1 - s0, 80 + 128]."""
    hop, pad = m.hop_length, m.pad
    (P0, P1), (r0, r1), _ = m.window_plan(s0, s1, known, final)
    padded = np.pad(mel[:, :known], ((0, 0), (pad, pad)))
    win = np.zeros((mel.shape[0], P1 - P0))
    hi = min(P1, padded.shape[1] if final else known + pad)
    win[:, :hi - P0] = padded[:, P0:hi]
    x = win
    for i, s in enumerate(m.upsample_factors):
        fir = p[f'upsample.up_layers.{2 * i + 1}.weight'].reshape(-1)
        st = np.repeat(x, s, axis=1)
        sp = np.pad(st, ((0, 0), (s, s)))
        x = sum(fir[j] * sp[:, j:j + st.shape[1]] for j in range(2 * s + 1))
    q = np.arange(s0, s1)
    mel_cols = x[:, q + pad * hop - P0 * hop].T
    _, aux = O.upsample(p, mel[:, r0:r1], m.upsample_factors, pad, 1)
    return np.concatenate([mel_cols, aux[q - r0 * hop]], axis=1)


def test_lookahead_is_the_reach_of_the_features():
    m = _small()
    assert m.lookahead() == 2
    assert WaveRNN(**dict(REAL, res_blocks=1, pad=0)).lookahead() == 2          # the mel path alone: one frame per stretch layer, rounded
    assert WaveRNN(**dict(REAL, res_blocks=1, pad=5)).lookahead() == 5
    p = O.sd64(m)
    rng = np.random.default_rng(1)
    mel = rng.standard_normal((80, 30))
    mu, aux = O.upsample(p, mel, (5, 5, 11), 2, 1)
    f, hop, la = 10, 275, m.lookahead()
    for d, changes in ((la, True), (la + 1, False)):
        bumped = mel.copy()
        bumped[:, f + d] += 1.0
        mu2, aux2 = O.upsample(p, bumped, (5, 5, 11), 2, 1)
        moved = not (np.array_equal(mu[f * hop:(f + 1) * hop], mu2[f * hop:(f + 1) * hop])
                     and np.array_equal(aux[f * hop:(f + 1) * hop], aux2[f * hop:(f + 1) * hop]))
        assert moved == changes, d


@pytest.mark.parametrize('frames', [21, 45])
@pytest.mark.parametrize('chunking', ['ones', 'irregular', 'whole'])
def test_window_plan_reproduces_the_whole_mel_upsampling(frames, chunking):
    m = _small()
    p = O.sd64(m)
    mel = np.random.default_rng(frames).standard_normal((80, frames))
    mu, aux = O.upsample(p, mel, (5, 5, 11), 2, 1)
    ref = np.concatenate([mu, aux], axis=1)
    sizes = {'ones': [1] * frames, 'irregular': [3, 0, 8, 1], 'whole': [frames]}[chunking]
    sizes = sizes + [frames - sum(sizes)] if sum(sizes) < frames else sizes
    hop, la = m.hop_length, m.lookahead()
    known, steps = 0, 0
    for n in sizes:
        known += n
        ready = min(known - la, known - 1) * hop
        if ready > steps:
            got = _windowed_features(m, p, mel, steps, ready, known, False)
            np.testing.assert_allclose(got, ref[steps:ready], rtol=1e-12, atol=1e-12)
            steps = ready
    got = _windowed_features(m, p, mel, steps, (frames - 1) * hop, frames, True)
    np.testing.assert_allclose(got, ref[steps:(frames - 1) * hop], rtol=1e-12, atol=1e-12)


def test_window_plan_refuses_frames_that_have_not_arrived():
    m = _small()
    with pytest.raises(ValueError, match='past the 10'):
        m.window_plan(0, 9 * 275, 10, False)
    m.window_plan(0, 8 * 275, 10, False)


# ---- argument checks ----
def test_stream_argument_checks():
    m = _small()
    mel = np.zeros((80, 30), np.float32)
    with pytest.raises(ValueError, match='ended after 0 frames'):
        list(m.generate_stream([]))
    with pytest.raises(ValueError, match='shape'):
        next(m.generate_stream([np.zeros((79, 5), np.float32)]))
    with pytest.raises(ValueError, match='shape'):
        next(m.generate_stream([np.zeros(80, np.float32)]))
    bad = mel.copy()
    bad[3, 4] = np.nan
    with pytest.raises(ValueError, match='non-finite'):
        next(m.generate_stream([bad]))
    with pytest.raises(ValueError, match='preemphasis'):
        next(m.generate_stream([mel], preemphasis=1.0))
    with pytest.raises(ValueError, match='uniform tape'):
        next(m.generate_stream([mel], uniforms=np.zeros((30 * 275, 1), np.float32)))
    with pytest.raises(ValueError, match='outside'):
        next(m.generate_stream([mel], uniforms=np.full((1, 30 * 275, 1), 1.0, np.float32)))


def test_decoder_stream_rejects_a_bad_chunk_size():
    from multilingual_text_to_speech_b200.modules.tacotron2 import Tacotron
    from multilingual_text_to_speech_b200.params.params import Params as hp
    hp.reset()
    model = Tacotron()
    text = torch.tensor([3, 4, 5])
    for bad in (0, -8):
        with pytest.raises(ValueError, match='chunk_frames'):
            next(model.inference_stream(text, chunk_frames=bad))
    with pytest.raises(ValueError, match='non-empty int64'):
        next(model.inference_stream(torch.tensor([], dtype=torch.int64)))


def test_window_rows_abi_rejects_each_bad_window_without_a_device():
    """b200tts_wavernn_window_rows refuses each shape alone in a one-row call: reads outside the mel or aux window, bad dimensions, a hop
    that is not a multiple of the last factor, a negative first position."""
    lib = _lib.load()
    one = ctypes.c_void_p(16)
    W = _lib.WaveRNNWindowShape
    for shape, s0, what in [
        # positions [0, 275) read penultimate samples up to 3 x 25 (pad 2, last factor 11): a window of 60 samples is too short
        (W(80, 128, 275, 2, 11, 0, 0, 60, 0, 5), 0, b'outside the window'),
        (W(80, 128, 275, 2, 11, 0, 0, 100, 1, 5), 0, b'aux frames'),          # aux frames start at 1, frame 0 is read
        (W(0, 128, 275, 2, 11, 0, 0, 100, 0, 5), 0, b'bad dimensions'),
        (W(80, 128, 270, 2, 11, 0, 0, 100, 0, 5), 0, b'must be a multiple'),
        (W(80, 128, 275, 2, 11, 0, 0, 100, 0, 5), -1, b'positions [-1, 274)'),
    ]:
        row = (_lib.WaveRNNWindowRow * 1)(_lib.WaveRNNWindowRow(shape, s0, 0, 0, 275))
        assert lib.b200tts_wavernn_window_rows(row, 1, 275, one, one, one, one, None) == -1
        assert what in lib.b200tts_last_error(), (what, lib.b200tts_last_error())
