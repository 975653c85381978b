"""Continuous-batching synthesis on the GPU:
  * b200tts_decoder_state_reset_rows then a chunk with first = 0 equals a chunk with first != 0, bit for bit, for both attention types;
  * b200tts_fill_keep_mask_rows rows are slices of b200tts_fill_keep_mask under random chunkings; b200tts_fill_uniform_rows is
    chunk-invariant and uniform on [0, 1);
  * DecoderPool texts opened at staggered calls equal inference_stream of each text alone (every test_gpu_batch_inference case, fp32 bit
    for bit and bf16 within tolerance, chunks of 7 and 128 frames, and a model with two frames per step);
  * SpeechServer requests equal speech_stream of each alone given the same tapes, or the tapes their seed denotes (RAW and MOL), through
    joins at every call, a queue beyond the capacity, cancels mid-decode and mid-vocode, and a request that fails alone."""
import numpy as np
import pytest
import torch

from helpers import assert_close
from multilingual_text_to_speech_b200 import _lib
from multilingual_text_to_speech_b200 import functional as F
from test_gpu_batch_inference import CASES, _case
from test_gpu_streaming import _taped
from test_gpu_wavernn import make_model

pytestmark = pytest.mark.gpu


@pytest.fixture(scope='module', autouse=True)
def _built():
    import __graft_entry__ as entry
    entry.build()
    assert torch.cuda.is_available()
    yield
    _lib.set_precision('fp32')


# ---- library entry points ----
@pytest.mark.parametrize('name', ['inf_batch_lj', 'inf_batch_forward'])
def test_reset_rows_equals_first_chunk(name):
    model, utts, _ = _case(name)
    _lib.set_precision('fp32')
    dec = model._decoder
    texts = [u[0] for u in utts]
    with torch.no_grad():
        encoded, mask, speaker, language = model._encode_group(texts, None if utts[0][1] is None else [u[1] for u in utts],
                                                                None if utts[0][2] is None else [u[2] for u in utts])
        memory = dec._memory(encoded, speaker, language)
        B, L, M = memory.shape
        lengths = mask.sum(1).to(torch.int32)
        P = dec._prenet._layers[0].weight.shape[0]
        g = torch.Generator(device='cuda').manual_seed(5)
        masks = {k: (torch.rand(6, B, P, device='cuda', generator=g) > 0.5).to(torch.uint8) for k in ('step_prenet0', 'step_prenet1')}
        kind, rh, rc = dec._cell_config()
        cfg = F.DecoderConfig(kind, False, rh, rc, dec._prenet._dropout_rate, masks, np.zeros(6, np.uint8), 1)
        fresh = F.DecoderState(B, dec._decoder_dim, M, L, dec._output_dim, memory.device)
        ref = F.decoder_forward_chunk(cfg, memory, lengths, dec._param_list(), fresh, 6)
        carried = F.DecoderState(B, dec._decoder_dim, M, L, dec._output_dim, memory.device)
        for name_ in ('att_h', 'att_c', 'gen_h', 'gen_c', 'context', 'cum_weights', 'frame'):
            getattr(carried, name_).normal_(generator=g)
        carried.first = False
        rows = list(range(B))[::-1]
        carried.reset_rows(rows, getattr(dec._attention, '_location', None) is None)
        got = F.decoder_forward_chunk(cfg, memory, lengths, dec._param_list(), carried, 6)
        for a, b in zip(got, ref):
            assert torch.equal(a, b)
        for name_ in ('att_h', 'att_c', 'gen_h', 'gen_c', 'context', 'cum_weights', 'frame'):
            assert torch.equal(getattr(carried, name_), getattr(fresh, name_)), name_


def _cut_points(total, rng):
    cuts = sorted(set(int(c) for c in rng.integers(0, total + 1, 4)) | {0, total})
    return list(zip(cuts[:-1], cuts[1:]))


def test_keep_mask_rows_are_slices_of_fill_keep_mask():
    rng = np.random.default_rng(3)
    S, P, rate, stream = 57, 256, 0.5, _lib.SEED_STREAMS['step_prenet0']
    seeds = [0, 1, 2 ** 64 - 1, 123456789123, 77]
    full = [F.fill_keep_mask((S, P), rate, s, stream, 'cuda') for s in seeds]
    for trial in range(3):
        got = [[] for _ in seeds]
        spans = [_cut_points(S, rng) for _ in seeds]
        for k in range(max(len(sp) for sp in spans)):
            live = [r for r in range(len(seeds)) if k < len(spans[r])]
            n = max(spans[r][k][1] - spans[r][k][0] for r in live)
            m = F.fill_keep_mask_rows(n, P, rate, [seeds[r] for r in live], [spans[r][k][0] for r in live], stream, 'cuda')
            for j, r in enumerate(live):
                a, b = spans[r][k]
                got[r].append(m[:b - a, j])
        for r in range(len(seeds)):
            assert torch.equal(torch.cat(got[r]), full[r]), (trial, r)
    big = F.fill_keep_mask_rows(400, 256, 0.3, [11, 12], [0, 1000], stream, 'cuda').double()
    n = big.numel()
    assert abs(float(big.mean()) - 0.7) < 5 * (0.7 * 0.3 / n) ** 0.5
    assert not torch.equal(big[:, 0], big[:, 1])


def test_uniform_rows_chunk_invariant_and_uniform():
    rng = np.random.default_rng(4)
    T, U, stream = 3000, 3, _lib.SEED_STREAMS['vocoder']
    seeds = [9, 10, 2 ** 63 + 5]
    full = F.fill_uniform_rows(T, U, seeds, [0] * len(seeds), stream, 'cuda')
    for r, s in enumerate(seeds):
        got = torch.cat([F.fill_uniform_rows(b - a, U, [s], [a], stream, 'cuda')[0] for a, b in _cut_points(T, rng)])
        assert torch.equal(got, full[r])
    x = F.fill_uniform_rows(20000, 8, [1, 2, 3], [0, 5, 7], stream, 'cuda').double()
    assert float(x.min()) >= 0.0 and float(x.max()) < 1.0
    n = x.numel()
    assert abs(float(x.mean()) - 0.5) < 5 * (1 / 12 / n) ** 0.5
    assert abs(float(x.var()) - 1 / 12) < 5 * (1 / 180 / n) ** 0.5 + 1e-4


# ---- DecoderPool ----
def _solo_stream(model, text, speaker, language, masks, chunk):
    tape = {k: v.unsqueeze(1) for k, v in masks.items()}
    return _taped(tape, lambda: torch.cat(list(model.inference_stream(text, speaker, language, chunk_frames=chunk)), 1))


def _drive_pool(pool, opens, closes=None):
    """opens: {call: [(key, open args)]}; closes: {call: [key]} before that call.  -> ({key: concatenated chunks}, {call: open rows})"""
    ids, out, sizes, call = {}, {}, {}, 0
    while call <= max(opens) or pool.ids:
        for key, args in opens.get(call, []):
            ids[key] = pool.open(*args[:3], masks=args[3] if len(args) > 3 else None, seed=args[4] if len(args) > 4 else None)
            out[key] = []
        for key in (closes or {}).get(call, []):
            pool.close(ids[key])
        sizes[call] = len(pool.ids)
        for tid, chunk in pool.run().items():
            out[next(k for k, i in ids.items() if i == tid)].append(chunk)
        call += 1
    return {k: torch.cat(v, 1) for k, v in out.items() if v}, sizes


@pytest.mark.parametrize('precision', ['fp32', 'bf16'])
@pytest.mark.parametrize('chunk', [7, 128])
@pytest.mark.parametrize('name', CASES)
def test_decoder_pool_staggered_opens(name, chunk, precision):
    model, utts, _ = _case(name)
    _lib.set_precision(precision)
    try:
        masks = [{'step_prenet0': u[3], 'step_prenet1': u[4]} for u in utts]
        # the longest text joins last, after the others have started; one text per call before it
        order = sorted(range(len(utts)), key=lambda j: int(utts[j][0].shape[0]))
        opens = {c: [(j, (utts[j][0], utts[j][1], utts[j][2], masks[j]))] for c, j in enumerate(order)}
        got, _ = _drive_pool(model.decoder_pool(8, chunk), opens)
        for j, u in enumerate(utts):
            ref = _solo_stream(model, u[0], u[1], u[2], masks[j], chunk)
            assert got[j].shape == ref.shape, (j, got[j].shape, ref.shape)
            if precision == 'fp32':
                assert torch.equal(got[j], ref), (name, chunk, j)
            else:
                assert_close(got[j], ref, 1e-3, 1e-4, f'{name}: text {j}')
    finally:
        _lib.set_precision('fp32')


def _fresh_model(seed, **hp_values):
    from multilingual_text_to_speech_b200.params.params import Params as hp
    from multilingual_text_to_speech_b200.modules.tacotron2 import Tacotron
    hp.reset()
    for k, v in hp_values.items():
        setattr(hp, k, v)
    torch.manual_seed(seed)
    return Tacotron().cuda().eval()


def test_decoder_pool_two_frames_per_step_and_close():
    from multilingual_text_to_speech_b200.params.params import Params as hp
    try:
        model = _fresh_model(80, outputs_per_step=2, max_output_length=60)
        with torch.no_grad():
            model._decoder._stop_prediction.bias.fill_(-1e4)      # every text decodes 60 frames: text 2 is still open at call 2
        _lib.set_precision('fp32')
        P = model._decoder._prenet._layers[0].weight.shape[0]
        g = torch.Generator().manual_seed(81)
        texts = [torch.randint(3, 20, (n,), generator=g).cuda() for n in (12, 30, 7, 45, 20)]
        masks = [{k: (torch.rand(30, P, generator=g) >= 0.5).to(torch.uint8) for k in ('step_prenet0', 'step_prenet1')} for _ in texts]
        opens = {0: [(0, (texts[0], None, None, masks[0])), (1, (texts[1], None, None, masks[1]))], 1: [(2, (texts[2], None, None, masks[2]))],
                 3: [(3, (texts[3], None, None, masks[3])), (4, (texts[4], None, None, masks[4]))]}
        got, _ = _drive_pool(model.decoder_pool(4, 9), opens, closes={2: [2]})
        assert got[2].shape[1] < 60
        for j in (0, 1, 3, 4):
            assert torch.equal(got[j], _solo_stream(model, texts[j], None, None, masks[j], 9)), j
    finally:
        hp.reset()


# ---- SpeechServer ----
class _Cut:
    """A stop rule that cuts at a fixed frame (the stop token is ignored): texts of chosen lengths end where the test needs them to."""

    def __init__(self, frames):
        self.target, self.seen, self.cut = frames, 0, None

    def feed(self, logits):
        self.seen += len(logits)
        if self.cut is None and self.seen >= self.target:
            self.cut = self.target
        return self.cut


@pytest.fixture
def fixed_cuts(monkeypatch):
    """Text length n cuts at cuts[n] frames (default 40)."""
    from multilingual_text_to_speech_b200.modules import tacotron2 as T
    cuts = {}
    orig = T._DecodeRows.add

    def add(self, memory, lengths, keys, sources):
        orig(self, memory, lengths, keys, sources)
        for j in range(len(self.keys) - len(keys), len(self.keys)):
            self.rules[j] = _Cut(cuts.get(self.text_len[j], 40))
    monkeypatch.setattr(T._DecodeRows, 'add', add)
    return cuts


def _widen(m):
    return torch.cat([m] * (80 // m.shape[0] + 1))[:80]


def _speech_solo(model, voc, text, masks, uniforms, chunk):
    from multilingual_text_to_speech_b200.modules.streaming import speech_stream
    tape = {k: v.unsqueeze(1) for k, v in masks.items()}
    return _taped(tape, lambda: torch.cat(list(speech_stream(model, voc, text, None, None, _widen, chunk, uniforms))))


def _serve(server, script, last):
    """script(call) -> [(op, key, kwargs)] before that call ('submit' / 'cancel'), for calls up to `last`; then steps until idle.
    -> ({key: audio or None}, {key: id})"""
    ids, out, call = {}, {}, 0
    while call <= last or server.pending or server.active:
        for op, key, kw in script(call):
            if op == 'submit':
                ids[key] = server.submit(**kw)
                out[key] = []
            else:
                server.cancel(ids[key])
        for rid, chunk in server.step().items():
            out[next(k for k, i in ids.items() if i == rid)].append(chunk)
        call += 1
    return {k: torch.cat(v) if v else None for k, v in out.items()}, ids


@pytest.mark.parametrize('mode', ['RAW', 'MOL'])
def test_server_tape_and_seed_parity(mode, fixed_cuts):
    from multilingual_text_to_speech_b200.params.params import Params as hp
    from multilingual_text_to_speech_b200.modules.streaming import SpeechServer
    try:
        model = _fresh_model(90, max_output_length=120)
        _lib.set_precision('fp32')
        voc = make_model(mode, seed=91)
        U, hop = voc.uniforms_per_step(), voc.hop_length
        P, rate = model._decoder._prenet._layers[0].weight.shape[0], model._decoder._prenet._dropout_rate
        g = torch.Generator().manual_seed(92)
        lens = [5, 9, 14, 22, 31, 40, 47, 55]
        for i, n in enumerate(lens):
            fixed_cuts[n] = 21 + (37 * i) % 80
        texts = {n: torch.randint(3, 20, (n,), generator=g).cuda() for n in lens}
        masks = {n: {k: (torch.rand(120, P, generator=g) >= 0.5).to(torch.uint8) for k in ('step_prenet0', 'step_prenet1')} for n in lens}
        unis = {n: torch.rand(1, fixed_cuts[n] * hop, U, generator=g) for n in lens}
        # capacity 3 with 8 requests: a queue; a join at every call while rows are free; seeded requests mixed with taped ones
        seeded = {lens[1]: 5, lens[4]: 2 ** 64 - 3, lens[6]: 17}

        def script(call):
            if call < len(lens):
                n = lens[::-1][call]            # longest first: later joins are shorter, the longest leaves first
                kw = dict(text=texts[n])
                kw.update(dict(seed=seeded[n]) if n in seeded else dict(masks=masks[n], uniforms=unis[n]))
                return [('submit', n, kw)]
            return []
        server = SpeechServer(model, voc, 3, _widen, 16)
        got, _ = _serve(server, script, len(lens))
        assert not server.failed and not server.active and not server.pending
        for n in lens:
            if n in seeded:
                s = seeded[n]
                mk = {k: F.fill_keep_mask((120, P), rate, s, _lib.SEED_STREAMS[k], 'cuda').cpu() for k in ('step_prenet0', 'step_prenet1')}
                un = F.fill_uniform_rows(fixed_cuts[n] * hop, U, [s], [0], _lib.SEED_STREAMS['vocoder'], 'cuda').cpu()
                ref = _speech_solo(model, voc, texts[n], mk, un, 16)
            else:
                ref = _speech_solo(model, voc, texts[n], masks[n], unis[n], 16)
            assert got[n].shape == ref.shape == ((fixed_cuts[n] - 1) * hop,), (n, got[n].shape, ref.shape)
            assert torch.equal(got[n], ref), n
        # a seeded request alone, at another chunk size, gives the same bits
        n = lens[4]
        alone = SpeechServer(model, voc, 1, _widen, 7)
        solo, _ = _serve(alone, lambda c: [('submit', 'x', dict(text=texts[n], seed=seeded[n]))] if c == 2 else [], 2)
        assert torch.equal(solo['x'], got[n])
    finally:
        hp.reset()


def test_server_cancel_and_failure(fixed_cuts):
    from multilingual_text_to_speech_b200.params.params import Params as hp
    from multilingual_text_to_speech_b200.modules.streaming import SpeechServer
    try:
        model = _fresh_model(93, max_output_length=100)
        _lib.set_precision('fp32')
        voc = make_model('RAW', seed=94)
        g = torch.Generator().manual_seed(95)
        lens = [6, 11, 17, 25, 33]
        cuts = {6: 50, 11: 60, 17: 12, 25: 70, 33: 45}            # 17 cuts under 21 frames: it fails alone
        fixed_cuts.update(cuts)
        texts = {n: torch.randint(3, 20, (n,), generator=g).cuda() for n in lens}

        def run(cancel=False):
            """All five submitted at once; with cancel, 25 is cancelled before call 3 (24 of its 70 frames decoded) and 6 at the first call
            after its decode has ended (its stream is vocoding)."""
            server = SpeechServer(model, voc, 8, _widen, 8)
            ids = {n: server.submit(texts[n], seed=100 + n) for n in lens}
            key = {i: n for n, i in ids.items()}
            out, call, vocoding = {n: [] for n in lens}, 0, None
            while server.pending or server.active:
                if cancel and call == 3:
                    assert server.requests[ids[25]].tid is not None
                    server.cancel(ids[25])
                if cancel and vocoding is None and ids[6] in server.requests and server.requests[ids[6]].tid is None:
                    vocoding = call
                    server.cancel(ids[6])
                for rid, chunk in server.step().items():
                    out[key[rid]].append(chunk)
                call += 1
            return {n: torch.cat(v) if v else None for n, v in out.items()}, server, vocoding
        base, server, _ = run()
        assert list(server.failed) == [2] and 'at least 21' in server.failed[2]
        assert base[17] is None
        got, server, vocoding = run(cancel=True)
        assert list(server.failed) == [2] and vocoding is not None
        for n in (11, 33):
            assert torch.equal(got[n], base[n]), n
        assert got[6] is None or got[6].shape[0] < base[6].shape[0]
        # a queued request cancelled before admission
        s = SpeechServer(model, voc, 1, _widen, 8)
        a, b = s.submit(texts[6], seed=1), s.submit(texts[11], seed=2)
        assert s.pending == [a, b]
        s.step()
        assert s.active == [a] and s.pending == [b]
        s.cancel(b)
        assert s.pending == []
        with pytest.raises(ValueError, match='unknown'):
            s.cancel(b)
        s.cancel(a)
        assert not s.active and not s.pool.streams and not s.decoder.ids
    finally:
        hp.reset()
