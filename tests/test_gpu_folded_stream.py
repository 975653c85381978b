"""Folded streaming synthesis on the GPU, at the reference's vocoder dimensions with random weights, RAW and MOL:
  * folded generate_stream equals generate(mel, target, overlap, uniforms=tape) bit for bit at the fold edges of 11000 / 550 and hop 275
    (F = 21, 43, 44, 45, 86, 87, 900), at a small target with odd overlap and at overlap 0, under one-frame, irregular and whole-mel chunkings;
  * a seeded folded stream equals generate with the tape its seed denotes, alone, in a full pool and at another chunking;
  * eight 900-frame streams (176 folds on 64 rows) joining at staggered calls each equal their own generate;
  * preemphasis within generate_batch's bound;
  * SpeechServer(…, target=11000, overlap=550): each request equals speech_stream of it alone and generate of its mel, with tapes and with
    seeds; a cancel mid-vocode leaves the others unchanged; a request under 21 frames fails alone."""
import pytest
import torch

from multilingual_text_to_speech_b200 import _lib
from multilingual_text_to_speech_b200 import functional as F
from test_gpu_speech_server import _fresh_model, _serve, _widen, fixed_cuts  # noqa: F401 -- fixed_cuts is a fixture
from test_gpu_streaming import _chunks, _mel, _taped
from test_gpu_wavernn import _deemphasis_bound, make_model

pytestmark = pytest.mark.gpu


@pytest.fixture(scope='module', autouse=True)
def _built():
    import __graft_entry__ as entry
    entry.build()
    assert torch.cuda.is_available()
    yield
    _lib.set_precision('fp32')


def _tape(m, frames, target, overlap, seed):
    return torch.rand(m.tape_shape(frames, target, overlap), generator=torch.Generator().manual_seed(seed))


def _seed_tape(m, frames, target, overlap, seed):
    K, L, U = m.tape_shape(frames, target, overlap)
    return F.fill_uniform_rows(K * L, U, [seed], [0], _lib.SEED_STREAMS['vocoder'], 'cuda').reshape(K, L, U).cpu()


def _irregular(frames):
    sizes, n, i = [], 0, 0
    while n < frames:
        sizes.append([1, 7, 0, 30, 3, 64, 2][i % 7])
        n += sizes[-1]
        i += 1
    return sizes


def _stream(m, parts, target, overlap, tape):
    return torch.cat([torch.as_tensor(c) for c in m.generate_stream(parts, tape, target=target, overlap=overlap)])


@pytest.mark.parametrize('mode', ['RAW', 'MOL'])
def test_folded_generate_stream_equals_generate(mode):
    _lib.set_precision('fp32')
    m = make_model(mode, seed=80)
    cases = [(f, 11000, 550) for f in (21, 43, 44, 45, 86, 87, 900)] + [(60, 300, 7), (45, 500, 0)]
    for i, (frames, target, overlap) in enumerate(cases):
        mel, tape = _mel(frames, 81 + i), _tape(m, frames, target, overlap, 91 + i)
        ref = m.generate(mel, target=target, overlap=overlap, uniforms=tape)
        chunkings = {'whole': [frames], 'irregular': _irregular(frames)}
        if frames <= 100:
            chunkings['one-frame'] = [1] * frames
        for name, sizes in chunkings.items():
            got = _stream(m, _chunks(mel, sizes), target, overlap, tape)
            assert got.shape == ref.shape, (frames, target, overlap, name)
            assert torch.equal(got, ref), (frames, target, overlap, name, int((got != ref).sum()))


def _drive(pool, mels, tapes, seeds, opens, chunk):
    """Opens stream i at call opens[i] (tape or seed), feeds `chunk` frames per call, ends it after its last; runs until every stream has
    finished -> [audio of stream i]."""
    sid, out, fed, call = {}, {}, {}, 0
    while len(sid) < len(mels) or pool.streams:
        for i, c in enumerate(opens):
            if c == call:
                sid[i] = pool.open(tapes[i], seeds[i])
                out[sid[i]], fed[i] = [], 0
        for i in sid:
            if fed[i] < mels[i].shape[1]:
                pool.feed(sid[i], mels[i][:, fed[i]:fed[i] + chunk])
                fed[i] += chunk
                if fed[i] >= mels[i].shape[1]:
                    pool.end(sid[i])
        for s, w in pool.run().items():
            out[s].append(w)
        call += 1
    return [torch.cat(out[sid[i]]) for i in range(len(mels))]


@pytest.mark.parametrize('mode', ['RAW', 'MOL'])
def test_seeded_folded_stream_alone_full_and_rechunked(mode):
    _lib.set_precision('fp32')
    m = make_model(mode, seed=82)
    mel, seed = _mel(150, 83), 2 ** 64 - 11
    ref = m.generate(mel, 11000, 550, uniforms=_seed_tape(m, 150, 11000, 550, seed))
    alone = _drive(m.stream_pool(1, target=11000, overlap=550), [mel], [None], [seed], [0], 32)[0]
    assert torch.equal(alone, ref)
    others = [_mel(f, 84 + i) for i, f in enumerate((300, 90, 200))]
    full = _drive(m.stream_pool(4, target=11000, overlap=550), others[:2] + [mel] + others[2:], [None] * 4, [1, 2, seed, 3], [0, 0, 2, 1],
                  64)
    assert torch.equal(full[2], ref)
    assert torch.equal(_drive(m.stream_pool(1, target=11000, overlap=550), [mel], [None], [seed], [0], 7)[0], ref)


@pytest.mark.parametrize('mode', ['RAW', 'MOL'])
def test_eight_long_streams_share_64_rows(mode):
    _lib.set_precision('fp32')
    m = make_model(mode, seed=85)
    mels = [_mel(900, 86 + i) for i in range(8)]
    tapes = [_tape(m, 900, 11000, 550, 96 + i) for i in range(8)]
    assert sum(t.shape[0] for t in tapes) == 176
    pool = m.stream_pool(8, target=11000, overlap=550)
    got = _drive(pool, mels, tapes, [None] * 8, [0, 0, 1, 3, 4, 9, 14, 30], 64)
    assert all(f is None for f in pool.slots) and sorted(pool.free_store) == list(range(pool.nstore))
    refs = m.generate_batch(mels, 11000, 550, uniforms=tapes)
    for i in range(8):
        assert torch.equal(got[i], refs[i]), i


def test_folded_stream_with_deemphasis_within_bound():
    _lib.set_precision('fp32')
    m = make_model('RAW', seed=87)
    a = 0.97
    for frames, target, overlap in ((120, 11000, 550), (60, 300, 7)):
        mel, tape = _mel(frames, 88), _tape(m, frames, target, overlap, 89)
        ref = m.generate(mel, target, overlap, uniforms=tape, preemphasis=a)
        got = torch.cat(list(m.generate_stream(_chunks(mel, _irregular(frames)), tape, preemphasis=a, target=target, overlap=overlap)))
        assert got.shape == ref.shape
        assert float((got - ref).abs().max() / ref.abs().max()) <= _deemphasis_bound(a)


# ---- the server ----
def _solo_folded(model, voc, text, masks, uniforms, chunk):
    """(speech_stream of the text alone, folded; its decoded mel through the frame transform)."""
    from multilingual_text_to_speech_b200.modules.streaming import speech_stream
    tape = {k: v.unsqueeze(1) for k, v in masks.items()}
    audio = _taped(tape, lambda: torch.cat(list(speech_stream(model, voc, text, None, None, _widen, chunk, uniforms, target=11000,
                                                               overlap=550))))
    mel = _taped(tape, lambda: torch.cat([_widen(c) for c in model.inference_stream(text, chunk_frames=chunk)], 1))
    return audio, mel


@pytest.mark.parametrize('mode', ['RAW', 'MOL'])
def test_folded_server_parity(mode, fixed_cuts):
    from multilingual_text_to_speech_b200.params.params import Params as hp
    from multilingual_text_to_speech_b200.modules.streaming import SpeechServer
    try:
        model = _fresh_model(110, max_output_length=120)
        _lib.set_precision('fp32')
        voc = make_model(mode, seed=111)
        U, hop = voc.uniforms_per_step(), voc.hop_length
        P, rate = model._decoder._prenet._layers[0].weight.shape[0], model._decoder._prenet._dropout_rate
        g = torch.Generator().manual_seed(112)
        lens = [5, 9, 14, 22, 31, 40]
        for i, n in enumerate(lens):
            fixed_cuts[n] = 21 + (37 * i) % 99
        texts = {n: torch.randint(3, 20, (n,), generator=g).cuda() for n in lens}
        masks = {n: {k: (torch.rand(120, P, generator=g) >= 0.5).to(torch.uint8) for k in ('step_prenet0', 'step_prenet1')} for n in lens}
        unis = {n: torch.rand(voc.tape_shape(fixed_cuts[n], 11000, 550), generator=g) for n in lens}
        seeded = {lens[1]: 5, lens[4]: 2 ** 64 - 3}

        def script(call):
            if call < len(lens):
                n = lens[::-1][call]
                kw = dict(text=texts[n])
                kw.update(dict(seed=seeded[n]) if n in seeded else dict(masks=masks[n], uniforms=unis[n]))
                return [('submit', n, kw)]
            return []
        server = SpeechServer(model, voc, 3, _widen, 16, target=11000, overlap=550)
        got, _ = _serve(server, script, len(lens))
        assert not server.failed and not server.active and not server.pending
        for n in lens:
            if n in seeded:
                s = seeded[n]
                mk = {k: F.fill_keep_mask((120, P), rate, s, _lib.SEED_STREAMS[k], 'cuda').cpu() for k in ('step_prenet0', 'step_prenet1')}
                un = _seed_tape(voc, fixed_cuts[n], 11000, 550, s)
            else:
                mk, un = masks[n], unis[n]
            ref, mel = _solo_folded(model, voc, texts[n], mk, un, 16)
            assert got[n].shape == ref.shape == ((fixed_cuts[n] - 1) * hop,), (n, got[n].shape, ref.shape)
            assert torch.equal(got[n], ref), n
            assert torch.equal(got[n], voc.generate(mel, 11000, 550, uniforms=un)), n
    finally:
        hp.reset()


def test_folded_server_cancel_and_failure(fixed_cuts):
    from multilingual_text_to_speech_b200.params.params import Params as hp
    from multilingual_text_to_speech_b200.modules.streaming import SpeechServer
    try:
        model = _fresh_model(113, max_output_length=100)
        _lib.set_precision('fp32')
        voc = make_model('RAW', seed=114)
        g = torch.Generator().manual_seed(115)
        lens = [6, 11, 17, 25]
        fixed_cuts.update({6: 90, 11: 60, 17: 12, 25: 70})            # 17 cuts under 21 frames: it fails alone
        texts = {n: torch.randint(3, 20, (n,), generator=g).cuda() for n in lens}

        def run(cancel):
            server = SpeechServer(model, voc, 8, _widen, 8, target=11000, overlap=550)
            ids = {n: server.submit(texts[n], seed=200 + n) for n in lens}
            key = {i: n for n, i in ids.items()}
            out, vocoding = {n: [] for n in lens}, None
            while server.pending or server.active:
                if cancel and vocoding is None and ids[6] in server.requests and server.requests[ids[6]].tid is None:
                    vocoding = True
                    server.cancel(ids[6])                        # its decode has ended: it is vocoding
                for rid, chunk in server.step().items():
                    out[key[rid]].append(chunk)
            return {n: torch.cat(v) if v else None for n, v in out.items()}, server, vocoding
        base, server, _ = run(False)
        assert list(server.failed) == [2] and 'at least 21' in server.failed[2] and base[17] is None
        got, server, vocoding = run(True)
        assert list(server.failed) == [2] and vocoding
        assert all(f is None for f in server.pool.slots) and sorted(server.pool.free_store) == list(range(server.pool.nstore))
        for n in (11, 25):
            assert torch.equal(got[n], base[n]), n
        assert got[6] is None or got[6].shape[0] < base[6].shape[0]
    finally:
        hp.reset()
