"""Streaming Griffin-Lim on the GPU (GriffinLimVocoder, b200tts_gl_stream_run):
  * a stream's magnitudes are b200tts_spectrogram_magnitude's bit for bit, mel and linear, whatever the chunk;
  * one stream against the fp64 oracle of tests/griffinlim_stream_oracle.py, mel and linear, within GL_STREAM_DRIFT_FACTOR times the
    drift the fp32 oracle shows on the same input; with de-emphasis, against the oracle followed by lfilter;
  * the bits do not depend on the chunking, on when run() is called, or on the streams around a stream in a pool;
  * speech_stream and SpeechServer run on it, bit for bit as the vocoder alone on the decoded mel, in fp32 mode."""
import numpy as np
import pytest
import scipy.signal
import torch

import audio_oracle as O
import griffinlim_stream_oracle as G
from multilingual_text_to_speech_b200 import _lib
from multilingual_text_to_speech_b200 import functional as F
from multilingual_text_to_speech_b200.modules.griffinlim import GriffinLimVocoder
from multilingual_text_to_speech_b200.utils import audio
from test_griffinlim_stream_cpu import GL_STREAM_DRIFT_FACTOR, N, HOP, WIN, _harmonic
from test_gpu_speech_server import _fresh_model, _serve, _taped, fixed_cuts  # noqa: F401 -- fixed_cuts is a fixture

pytestmark = pytest.mark.gpu


@pytest.fixture(scope='module', autouse=True)
def _built():
    import __graft_entry__ as entry
    from multilingual_text_to_speech_b200.params.params import Params as hp
    entry.build()
    assert torch.cuda.is_available()
    hp.reset()
    yield
    _lib.set_precision('fp32')


def _denorm(m):
    return audio.denormalize_spectrogram(m, True)


@pytest.fixture
def mel_constants(monkeypatch):
    """The normalisation constants train.py sets from the training set (absent from the defaults)."""
    from multilingual_text_to_speech_b200.params.params import Params as hp
    monkeypatch.setattr(hp, 'mel_normalize_mean', -40.0, raising=False)
    monkeypatch.setattr(hp, 'mel_normalize_variance', 20.0, raising=False)


def _log_spec(frames, mel, seed=0):
    """A dB spectrogram [bins, frames] of a harmonic signal (20 log10 of its |STFT|, mel-projected when `mel`)."""
    X = np.abs(O.stft(_harmonic(HOP * (frames - 1), seed=seed), N, HOP, WIN))
    if mel:
        X = audio.mel_basis(22050, N, 80).astype(np.float64) @ X
    return (20 * np.log10(np.maximum(X, 1e-5))).astype(np.float32)


def _stream(voc, spec, sizes, **kw):
    chunks, t = [], 0
    for n in sizes:
        chunks.append(spec[:, t:t + n])
        t += n
    assert t == spec.shape[1]
    out = list(voc.generate_stream(chunks, **kw))
    return torch.cat(out) if out and isinstance(out[0], torch.Tensor) else np.concatenate(out)


@pytest.mark.parametrize('mel', [True, False])
def test_magnitudes_equal_spectrogram_magnitude(mel):
    voc = GriffinLimVocoder(mel)
    spec = torch.from_numpy(_log_spec(40, mel)).cuda()
    shape = audio.vocoder_shape(1, 40, mel)
    tables = audio.mel_tables(22050, N, 80, spec.device) if mel else ()
    whole = F.spectrogram_magnitude(shape, spec.t().contiguous(), *tables)
    t = 0
    for n in (1, 3, 17, 19):
        got = voc.magnitudes(spec[:, t:t + n].t().contiguous())
        assert torch.equal(got, whole[t:t + n]), n
        t += n


@pytest.mark.parametrize('mel', [True, False])
def test_one_stream_against_the_oracle(mel):
    voc = GriffinLimVocoder(mel)
    spec = _log_spec(120, mel)
    S = voc.magnitudes(torch.from_numpy(spec).cuda().t().contiguous()).double().cpu().numpy().T
    y64 = G.rtisi(S, N, HOP, WIN)
    y32 = G.rtisi(S, N, HOP, WIN, dtype=np.float32)
    drift32 = np.linalg.norm(y64 - y32) / np.linalg.norm(y64)
    got = _stream(voc, spec, [120])
    assert got.shape == (HOP * 119,) and got.dtype == np.float32
    err = np.linalg.norm(got - y64) / np.linalg.norm(y64)
    assert err <= GL_STREAM_DRIFT_FACTOR * drift32, (err, drift32)
    # de-emphasis carried across chunks: the oracle followed by lfilter
    pre = _stream(voc, spec, [7, 50, 63], preemphasis=0.97)
    ref = scipy.signal.lfilter([1], [1, -0.97], y64)
    err = np.linalg.norm(pre - ref) / np.linalg.norm(ref)
    assert err <= GL_STREAM_DRIFT_FACTOR * drift32, (err, drift32)


def test_lookahead_0_releases_the_whole_stream():
    """Without look-ahead the last frame is committed before the end is known: the run() that learns of the end releases the rest."""
    voc = GriffinLimVocoder(True, lookahead=0, iters=4)
    spec = torch.from_numpy(_log_spec(60, True, seed=2)).cuda()
    whole = _stream(voc, spec, [60])
    assert whole.shape == (HOP * 59,)
    for sizes in ([1] * 60, [7] * 8 + [4], [0, 60]):
        assert torch.equal(_stream(voc, spec, sizes), whole), sizes
    pool = voc.stream_pool(2)
    a = pool.open()
    pool.feed(a, spec)
    first = pool.run()[a]
    pool.end(a)
    rest = pool.run()
    assert list(rest) == [a] and not pool.streams and first.shape[0] < HOP * 59
    assert torch.equal(torch.cat([first, rest[a]]), whole)
    S = voc.magnitudes(spec.t().contiguous()).double().cpu().numpy().T
    y64 = G.rtisi(S, N, HOP, WIN, lookahead=0, iters=4)
    y32 = G.rtisi(S, N, HOP, WIN, lookahead=0, iters=4, dtype=np.float32)
    err = np.linalg.norm(whole.cpu().numpy() - y64) / np.linalg.norm(y64)
    assert err <= GL_STREAM_DRIFT_FACTOR * np.linalg.norm(y64 - y32) / np.linalg.norm(y64), err


def test_chunking_and_run_calls_do_not_change_the_bits():
    voc = GriffinLimVocoder(True)
    spec = torch.from_numpy(_log_spec(200, True, seed=4)).cuda()
    whole = _stream(voc, spec, [200])
    assert whole.shape == (HOP * 199,)
    for size in (1, 3, 17, 64):
        sizes = [size] * (200 // size) + ([200 % size] if 200 % size else [])
        assert torch.equal(_stream(voc, spec, sizes), whole), size
    assert torch.equal(_stream(voc, spec, [0, 5, 0, 195]), whole)
    # a pool: run() after every feed, or once at the end
    pool = voc.stream_pool(2)
    a, b = pool.open(), pool.open(seed=7)
    got = {a: [], b: []}
    for t in range(0, 200, 9):
        pool.feed(a, spec[:, t:t + 9])
        pool.feed(b, spec[:, t:t + 9])
        for sid, w in pool.run().items():
            got[sid].append(w)
    pool.end(a)
    for sid, w in pool.run().items():
        got[sid].append(w)
    assert torch.equal(torch.cat(got[a]), whole)
    pool.end(b)
    assert list(pool.run()) == [b] and not pool.streams
    once = voc.stream_pool(1)
    s = once.open()
    once.feed(s, spec)
    once.end(s)
    assert torch.equal(once.run()[s], whole)


def test_ragged_pool_streams_equal_their_solo_runs():
    voc = GriffinLimVocoder(True)
    rng = np.random.default_rng(11)
    lens = [2, 3, 5, 900, 40, 7, 123, 64, 250, 17, 4, 333, 90, 11, 2, 600]
    specs = [torch.from_numpy(_log_spec(n, True, seed=i)).cuda() for i, n in enumerate(lens)]
    solo = [_stream(voc, s, [s.shape[1]], preemphasis=0.97) for s in specs]
    pool = voc.stream_pool(16, preemphasis=0.97)
    join = {i: int(rng.integers(0, 12)) for i in range(16)}
    chunk = {i: int(rng.integers(1, 80)) for i in range(16)}
    sid, pos, got, closed = {}, {i: 0 for i in range(16)}, {i: [] for i in range(16)}, set()
    call = 0
    while call < 12 or pool.streams:
        for i in range(16):
            if join[i] == call:
                sid[i] = pool.open()
            if i in sid and sid[i] in pool.streams and i not in closed and not pool.streams[sid[i]].ended:
                n = min(chunk[i], lens[i] - pos[i])
                pool.feed(sid[i], specs[i][:, pos[i]:pos[i] + n])
                pos[i] += n
                if pos[i] == lens[i] and (i + call) % 2 == 0:
                    pool.end(sid[i])
        if call == 5 and sid.get(13) in pool.streams:             # dropped mid-stream: the others do not notice
            pool.close(sid[13])
            closed.add(13)
        key = {s: i for i, s in sid.items()}
        for s, w in pool.run().items():
            got[key[s]].append(w)
        for i in sid:
            if sid[i] in pool.streams and pos[i] == lens[i] and not pool.streams[sid[i]].ended:
                pool.end(sid[i])
        call += 1
    for i in range(16):
        if i in closed:
            continue
        assert torch.equal(torch.cat(got[i]), solo[i]), (i, lens[i])
    full = voc.stream_pool(64)
    for _ in range(64):
        full.open()
    with pytest.raises(ValueError, match='full'):
        full.open()


def test_speech_stream_equals_the_vocoder_on_the_decoded_mel(mel_constants):
    from multilingual_text_to_speech_b200.params.params import Params as hp
    from multilingual_text_to_speech_b200.modules.streaming import speech_stream
    try:
        model = _fresh_model(70, max_output_length=60)
        with torch.no_grad():
            model._decoder._stop_prediction.bias.fill_(-1e4)      # decodes max_output_length frames
        _lib.set_precision('fp32')
        voc = GriffinLimVocoder()
        P = model._decoder._prenet._layers[0].weight.shape[0]
        g = torch.Generator().manual_seed(71)
        text = torch.randint(3, 20, (17,), generator=g).cuda()
        tape = {k: (torch.rand(60, 1, P, generator=g) >= 0.5).to(torch.uint8) for k in ('step_prenet0', 'step_prenet1')}
        mel = _taped(tape, lambda: model.inference(text))
        ref = torch.cat(list(voc.generate_stream([_denorm(mel)], preemphasis=hp.preemphasis)))
        got = _taped(tape, lambda: torch.cat(list(speech_stream(model, voc, text, mel_transform=_denorm, chunk_frames=16,
                                                                preemphasis=hp.preemphasis))))
        assert got.shape == ref.shape == (HOP * (mel.shape[1] - 1),)
        assert torch.equal(got, ref)
    finally:
        hp.reset()


def test_server_requests_equal_their_solo_speech_stream(fixed_cuts, mel_constants):  # noqa: F811
    from multilingual_text_to_speech_b200.params.params import Params as hp
    from multilingual_text_to_speech_b200.modules.streaming import SpeechServer, speech_stream
    try:
        model = _fresh_model(96, max_output_length=120)
        _lib.set_precision('fp32')
        voc = GriffinLimVocoder()
        P, rate = model._decoder._prenet._layers[0].weight.shape[0], model._decoder._prenet._dropout_rate
        g = torch.Generator().manual_seed(97)
        lens = [5, 9, 14, 22, 31, 40]
        cuts = {5: 2, 9: 70, 14: 1, 22: 33, 31: 110, 40: 9}       # 14 decodes one frame: it fails alone
        fixed_cuts.update(cuts)
        texts = {n: torch.randint(3, 20, (n,), generator=g).cuda() for n in lens}

        def script(call):
            return [('submit', n, dict(text=texts[n], seed=300 + n)) for n in lens if lens.index(n) == call]
        server = SpeechServer(model, voc, 3, _denorm, 8, hp.preemphasis)
        got, ids = _serve(server, script, len(lens))
        assert list(server.failed) == [ids[14]] and 'at least 2' in server.failed[ids[14]]
        for n in lens:
            if n == 14:
                continue
            mk = {k: F.fill_keep_mask((120, P), rate, 300 + n, _lib.SEED_STREAMS[k], 'cuda').cpu().unsqueeze(1)
                  for k in ('step_prenet0', 'step_prenet1')}
            ref = _taped(mk, lambda: torch.cat(list(speech_stream(model, voc, texts[n], mel_transform=_denorm, chunk_frames=8,
                                                                  preemphasis=hp.preemphasis))))
            assert got[n].shape == ref.shape == (HOP * (cuts[n] - 1),), n
            assert torch.equal(got[n], ref), n
    finally:
        hp.reset()
