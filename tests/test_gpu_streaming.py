"""Streaming synthesis on the GPU:
  * Tacotron.inference_stream on the reference's inference goldens: the stream's length equals inference()'s, its decoded frames equal
    inference()'s bit for bit, its post-net meets the golden tolerance and an fp32 bound against an fp64 post-net of the same frames, in
    both precision modes, at chunks of 7 and 128 frames and with r = 2; the first chunk comes after one decoder call;
  * WaveRNN.generate_stream: the stream equals generate(mel, target=F hop, overlap=0) bit for bit over several chunkings in RAW and MOL,
    at 21 and 900 frames; with de-emphasis, within its bound;
  * speech_stream equals generate of the concatenated streamed mel."""
import json
import os

import numpy as np
import pytest
import torch

import oracle.tacotron_oracle as TO
from helpers import GOLDEN_DIR, assert_close
from multilingual_text_to_speech_b200 import _lib
from multilingual_text_to_speech_b200 import functional as F
from test_gpu_wavernn import make_model, _deemphasis_bound

pytestmark = pytest.mark.gpu


@pytest.fixture(scope='module', autouse=True)
def _built():
    import __graft_entry__ as entry
    entry.build()
    assert torch.cuda.is_available()
    yield
    _lib.set_precision('fp32')


def _golden(name):
    """-> (model, [(text, language, tape, reference post-net)])"""
    from multilingual_text_to_speech_b200.params.params import Params as hp
    from multilingual_text_to_speech_b200.modules.tacotron2 import Tacotron
    z = np.load(os.path.join(GOLDEN_DIR, name + '.npz'))
    meta = json.loads(bytes(z['meta']).decode())
    hp.reset()
    hp.load_state_dict(meta['hp'])
    model = Tacotron()
    model.load_state_dict({k[3:]: torch.from_numpy(z[k]) for k in z.files if k.startswith('sd.')}, strict=True)
    model = model.cuda().eval()
    get = lambda k: torch.from_numpy(z[k]).cuda() if k in z.files else None     # noqa: E731
    if name == 'inf_batch_forward':
        utts = [(get(f'text{j}'), get(f'language{j}'), {'step_prenet0': torch.from_numpy(z[f'tape{j}.step_prenet0']).unsqueeze(1),
                                                        'step_prenet1': torch.from_numpy(z[f'tape{j}.step_prenet1']).unsqueeze(1)},
                 torch.from_numpy(z[f'out{j}'])) for j in range(meta['n'])]
    else:
        tape = {k[5:]: torch.from_numpy(z[k]) for k in z.files if k.startswith('tape.')}
        utts = [(get('in.text'), get('in.language'), tape, torch.from_numpy(z['out.post']))]
    return model, utts


def _record(fn):
    """Runs fn() with F.decoder_forward_chunk wrapped: -> (fn's result, the decoded frames of every call)."""
    frames = []
    orig = F.decoder_forward_chunk

    def wrapped(*a, **k):
        out = orig(*a, **k)
        frames.append(out[0][0].clone())
        return out
    F.decoder_forward_chunk = wrapped
    try:
        return fn(), frames
    finally:
        F.decoder_forward_chunk = orig


def _taped(tape, fn):
    from multilingual_text_to_speech_b200.rng import MaskSource
    MaskSource.use_tape(tape)
    try:
        return fn()
    finally:
        MaskSource.use_tape(None)


def _fp64_postnet(model, pre):
    from multilingual_text_to_speech_b200.params.params import Params as hp
    sd = {k: v.detach().double().cpu() for k, v in model.state_dict().items() if k.startswith('_postnet')}
    x = pre.double().cpu().unsqueeze(0)
    post = TO.postnet(sd, hp, x, None, training=False)[0]
    # magnitude: the same post-net on |weights| and |inputs| bounds each fp32 accumulation's error
    mag = x.abs()
    for j in range(hp.postnet_blocks):
        p = f'_postnet._convs.{j}'
        w = sd[f'{p}._block.1.weight'].abs()
        mag = TO.conv1d_same(mag, w) * (sd[f'{p}._block.2.weight'].abs() / torch.sqrt(sd[f'{p}._block.2.running_var'] + 1e-5))[None, :, None]
    return post, mag[0]


@pytest.mark.parametrize('precision', ['fp32', 'bf16'])
@pytest.mark.parametrize('chunk', [7, 128])
@pytest.mark.parametrize('name', ['inf_lj', 'inf_generated_mix', 'inf_batch_forward'])
def test_decoder_stream_matches_inference(name, chunk, precision):
    from multilingual_text_to_speech_b200.modules.tacotron2 import Decoder
    model, utts = _golden(name)
    _lib.set_precision(precision)
    old = Decoder.inference_chunk
    Decoder.inference_chunk = chunk
    try:
        for text, language, tape, ref in utts:
            lang = None if language is None else language
            whole, whole_frames = _record(lambda: _taped(tape, lambda: model.inference(text, None, lang)))
            parts, stream_frames = _record(lambda: _taped(tape, lambda: list(model.inference_stream(text, None, lang))))
            assert len(parts) == len(stream_frames)                     # one item per decoder call
            post = torch.cat(parts, 1)
            assert post.shape == whole.shape, (post.shape, whole.shape)
            pre = torch.cat(stream_frames, 0)
            assert torch.equal(pre, torch.cat(whole_frames, 0))
            T = post.shape[1]
            if precision == 'fp32':           # bf16 mode may stop elsewhere than the reference did
                assert post.shape == ref.shape, (post.shape, ref.shape)
                assert_close(post, ref, 1e-3, 1e-4, f'{name}: streamed post-net')
            ref64, mag = _fp64_postnet(model, pre[:T].t())
            K = 5 * 512
            bound = (K * 2.0 ** -23 if precision == 'fp32' else 2 * 2.0 ** -8) * mag * 4 + 1e-5
            err = (post.double().cpu() - ref64).abs()
            assert bool((err <= bound + 1e-3 * ref64.abs()).all()), float((err - bound).max())
    finally:
        Decoder.inference_chunk = old
        _lib.set_precision('fp32')


def test_decoder_stream_first_chunk_after_one_call():
    from multilingual_text_to_speech_b200.rng import MaskSource
    model, utts = _golden('inf_lj')
    text, language, tape, ref = utts[0]
    calls = []
    orig = F.decoder_forward_chunk
    F.decoder_forward_chunk = lambda *a, **k: (calls.append(a[-1]), orig(*a, **k))[1]
    MaskSource.use_tape(tape)
    try:
        stream = model.inference_stream(text, None, language)
        first = next(stream)
        assert len(calls) == 1 and first.shape[1] == min(128 - 10, ref.shape[1]), (calls, first.shape)
        stream.close()
    finally:
        MaskSource.use_tape(None)
        F.decoder_forward_chunk = orig


def test_decoder_stream_outputs_per_step_2():
    """r = 2 on seeded weights, decoded to max_output_length: the stream equals inference() at the same chunk, frames bit for bit."""
    from multilingual_text_to_speech_b200.params.params import Params as hp
    from multilingual_text_to_speech_b200.modules.tacotron2 import Decoder, Tacotron
    from multilingual_text_to_speech_b200.rng import MaskSource
    hp.reset()
    hp.outputs_per_step = 2
    hp.max_output_length = 61
    torch.manual_seed(5)
    model = Tacotron().cuda().eval()
    text = torch.randint(3, 20, (17,)).cuda()
    old = Decoder.inference_chunk
    try:
        for chunk in (7, 128):
            Decoder.inference_chunk = chunk
            MaskSource.manual_seed(11)
            whole, wf = _record(lambda: model.inference(text))
            MaskSource.manual_seed(11)
            parts, sf = _record(lambda: list(model.inference_stream(text)))
            post = torch.cat(parts, 1)
            assert post.shape == whole.shape
            assert torch.equal(torch.cat(sf, 0), torch.cat(wf, 0))
            assert_close(post, whole, 1e-5, 1e-6, f'r = 2, chunk {chunk}')
    finally:
        Decoder.inference_chunk = old
        hp.reset()


# ---- vocoder ----
def _mel(frames, seed):
    return torch.from_numpy(np.random.default_rng(seed).standard_normal((80, frames)).astype(np.float32)).cuda()


def _chunks(mel, sizes):
    out, i = [], 0
    for n in sizes:
        out.append(mel[:, i:i + n])
        i += n
    if i < mel.shape[1]:
        out.append(mel[:, i:])
    return out


@pytest.mark.parametrize('mode', ['RAW', 'MOL'])
@pytest.mark.parametrize('frames', [21, 900])
def test_generate_stream_equals_unbatched_generate(mode, frames):
    _lib.set_precision('fp32')
    m = make_model(mode, seed=23)
    mel = _mel(frames, 24)
    hop = m.hop_length
    tape = torch.rand(m.tape_shape(frames, frames * hop, 0), generator=torch.Generator().manual_seed(25))
    assert tape.shape[0] == 1
    ref = m.generate(mel, target=frames * hop, overlap=0, uniforms=tape)
    assert ref.shape == ((frames - 1) * hop,)
    chunkings = {'one frame': [1] * frames, 'irregular': [5, 0, 1, 13, 2, 130, 64], 'whole': [frames]}
    for what, sizes in chunkings.items():
        if frames == 900 and what == 'one frame':
            sizes = [1] * 40 + [3] * 40              # one-frame chunks at the start, then the rest in one
        parts = list(m.generate_stream(_chunks(mel, sizes), uniforms=tape))
        got = torch.cat(parts)
        assert got.shape == ref.shape, (what, got.shape)
        assert torch.equal(got, ref), (what, int((got != ref).sum()))
        if frames == 900 and what == 'irregular':
            assert len(parts) > 3


def test_generate_stream_with_deemphasis_within_bound():
    _lib.set_precision('fp32')
    m = make_model('RAW', seed=26)
    frames, hop, a = 60, 275, 0.97
    mel = _mel(frames, 27)
    tape = torch.rand(m.tape_shape(frames, frames * hop, 0), generator=torch.Generator().manual_seed(28))
    ref = m.generate(mel, target=frames * hop, overlap=0, uniforms=tape, preemphasis=a)
    got = torch.cat(list(m.generate_stream(_chunks(mel, [7, 1, 20]), uniforms=tape, preemphasis=a)))
    err = float((got - ref).abs().max() / ref.abs().max())
    assert err <= _deemphasis_bound(a), err


def test_single_fold_generate_against_oracle():
    """generate(mel, target=F hop, overlap=0) is accepted and post-processes as the oracle's unbatched path."""
    _lib.set_precision('fp32')
    m = make_model('MOL', seed=29)
    frames, hop = 25, 275
    mel = _mel(frames, 30)
    trace = {}
    with torch.no_grad():
        wave, _ = m._generate([mel], [frames], None, frames * hop, 0, None, torch.device('cuda'), trace)
    y = trace['folded'].double().cpu().numpy()
    assert y.shape == (1, frames * hop)
    # one fold without cross-fade: the loop's samples, cut to (F - 1) hop, times linspace(1, 0, 20 hop) over the last 20 hops
    ref = y[0, :(frames - 1) * hop].copy()
    ref[-20 * hop:] *= np.linspace(1, 0, 20 * hop)
    np.testing.assert_allclose(wave.cpu().numpy(), ref, rtol=1e-6, atol=1e-7)


def test_speech_stream_equals_generate_of_the_streamed_mel():
    from multilingual_text_to_speech_b200.modules.streaming import speech_stream
    model, utts = _golden('inf_generated_mix')              # 51 frames: the vocoder needs at least 21
    text, language, tape, _ = utts[0]
    voc = make_model('RAW', seed=31)
    _lib.set_precision('fp32')
    widen = lambda m: torch.cat([m] * 7)[:80]                  # noqa: E731 -- frame-local: the golden model has 12 mel channels
    mels = _taped(tape, lambda: list(model.inference_stream(text, None, language, chunk_frames=32)))
    mel = widen(torch.cat(mels, 1))
    frames = mel.shape[1]
    u = torch.rand(voc.tape_shape(frames, frames * 275, 0), generator=torch.Generator().manual_seed(32))
    audio = _taped(tape, lambda: torch.cat(list(speech_stream(model, voc, text, None, language, widen, chunk_frames=32, uniforms=u))))
    ref = voc.generate(mel, target=frames * 275, overlap=0, uniforms=u)
    assert torch.equal(audio, ref)
