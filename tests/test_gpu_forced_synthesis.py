"""Forced synthesis (durations= / alignments=) on the GPU:
  * one step from crafted states against fp64, both attention kinds, all rows forced and mixed with computed rows;
  * replay: a free decode's own alignment rows, supplied back, give that decode bit for bit (fp32 and bf16, r = 1 and 2, with and
    without a window; location-sensitive attention);
  * inference with durations against the CPU oracle with its attention step replaced by the plan, at r = 1 and 2;
  * a forced text in a mixed inference_batch, a DecoderPool with forced and free rows joining, leaving and closed, and a SpeechServer
    request each equal the text alone, and free rows are unchanged by forced neighbours."""
import numpy as np
import pytest
import torch

import forced_synthesis_oracle as FO
import outputs_per_step_oracle as R
from decoder_cases import PARAM_KEYS, _decoder_sd_alias
from helpers import assert_close
from oracle import tacotron_oracle as O
from multilingual_text_to_speech_b200 import _lib
from multilingual_text_to_speech_b200 import functional as F
from test_gpu_attention_window import _sharpen, _small_sd, _texts_and_tape, _with_window
from test_gpu_outputs_per_step import _synthesis_model
from test_gpu_speech_server import _fresh_model, _widen
from test_gpu_streaming import _taped
from test_gpu_wavernn import make_model

pytestmark = pytest.mark.gpu


@pytest.fixture(scope='module', autouse=True)
def _built():
    import __graft_entry__ as entry
    entry.build()
    assert torch.cuda.is_available()


@pytest.fixture(autouse=True)
def _reset():
    from multilingual_text_to_speech_b200.params.params import Params as hp
    yield
    hp.reset()
    _lib.set_precision('fp32')


# ---- one step against fp64 ----
@pytest.mark.parametrize('att', ['location', 'forward'])
@pytest.mark.parametrize('L', [1, 3, 37, 128, 300])
def test_one_step_against_fp64(L, att):
    M, D, P, A, C, K, N = 64, 64, 32, 32, 8, 7, 8
    g = torch.Generator().manual_seed(200 + L)
    sd = {k: v.float().double() for k, v in _small_sd(g, M, D, P, A, C, K, N).items()}
    lens = [L, max(1, L - 1), max(1, L // 2), max(1, L // 3)]
    B, dev = len(lens), torch.device('cuda:0')
    skip = ('_attention._location.weight', '_attention._loc_features.weight') if att == 'forward' else ()
    params = [None if key in skip else sd[key].float().to(dev) for _, key in PARAM_KEYS]
    memory = torch.randn(B, L, M, generator=g).to(dev)
    prev = torch.rand(B, L, generator=g).to(dev)
    keep = [torch.ones(1, B, P, dtype=torch.uint8, device=dev) for _ in range(2)]
    mask = O.lengths_to_mask(torch.tensor(lens), L).to(dev)
    for rows in ([0, 1, 2, 3], [3, 1], [2]):
        st = F.DecoderState(B, D, M, L, N, dev)
        st.cum_weights.copy_(prev)
        st.first = False
        w = torch.rand(1, len(rows), L, generator=g).to(dev) * 3
        cfg = F.DecoderConfig(_lib.CELL_DROPOUT, False, 0.1, 0.0, 0.5, {'step_prenet0': keep[0], 'step_prenet1': keep[1]},
                              np.zeros(1, dtype=np.uint8), 1)
        forced = (torch.tensor(rows, dtype=torch.int32, device=dev), w)
        _, _, align = F.decoder_forward_chunk(cfg, memory, torch.tensor(lens, device=dev), params, st, 1, forced)
        for k, b in enumerate(rows):
            want = torch.where(mask[b], w[0, k], torch.zeros_like(w[0, k]))
            what = f'L={L} att={att} rows={rows} b={b}'
            assert torch.equal(align[b, 0], want), what                        # the supplied row, exact zeros past the length
            if att == 'forward':
                assert torch.equal(st.cum_weights[b], want), what              # alpha is the row
            else:
                assert torch.allclose(st.cum_weights[b].double(), prev[b].double() + want.double(), rtol=1e-7, atol=0), what
            ctx64 = (want.double()[:, None] * memory[b].double()).sum(0)
            bound = 2e-5 * (want.double()[:, None] * memory[b].double().abs()).sum(0) + 1e-5
            assert bool(((st.context[b].double() - ctx64).abs() <= bound).all()), what
        free = [b for b in range(B) if b not in rows]
        if free:        # the computed rows: weights of a softmax within their lengths
            sums = align[free, 0].double().sum(1)
            assert torch.allclose(sums, torch.ones_like(sums), atol=1e-5)


# ---- replay ----
def _decode(model, texts, tape, window, plans=None):
    from multilingual_text_to_speech_b200.rng import MaskSource
    encoded, mask, speaker, language = model._encode_group(texts, None, None)
    MaskSource.use_tape(tape)
    try:
        with torch.no_grad():
            return model._decoder._decode_inference(encoded, mask, speaker, language, att_extent=1, att_window=window, plans=plans)
    finally:
        MaskSource.use_tape(None)


@pytest.mark.parametrize('window', [None, (1, 3)])
@pytest.mark.parametrize('r', [1, 2])
@pytest.mark.parametrize('precision', ['fp32', 'bf16'])
def test_replay_is_bitwise(precision, r, window):
    model = _fresh_model(300 + r, max_output_length=60, outputs_per_step=r)
    _sharpen(model)
    texts, tape = _texts_and_tape(model, [23, 9, 40, 5], 60, 301)
    _lib.set_precision(precision)
    spec, stop, align, cuts = _decode(model, texts, tape, window)
    S = [-(-c // r) for c in cuts]
    plans = [(align[b, :S[b], :t.shape[0]].contiguous(), S[b] * r) for b, t in enumerate(texts)]
    spec2, _, align2, cuts2 = _decode(model, texts, tape, window, plans)
    assert cuts2 == [s * r for s in S]
    for b in range(len(texts)):
        assert torch.equal(spec2[b, :cuts[b]], spec[b, :cuts[b]]), (precision, r, window, b)
        assert torch.equal(align2[b, :S[b]], align[b, :S[b]]), (precision, r, window, b)
    if r == 1:        # the post-net output through the public entry point
        def run(**kw):
            return _taped(tape, lambda: model.inference_batch(texts, **kw))
        replay = lambda: run(alignments=[p[0] for p in plans])      # noqa: E731
        free, forced = (_with_window(window, run), _with_window(window, replay)) if window else (run(), replay())
        for a, b in zip(forced, free):
            assert torch.equal(a, b), (precision, window)


# ---- against the oracle ----
@pytest.mark.parametrize('r', [1, 2])
def test_durations_against_oracle(r):
    from multilingual_text_to_speech_b200.rng import MaskSource
    from multilingual_text_to_speech_b200.params.params import Params as hp
    dev = torch.device('cuda:0')
    try:
        model, ohp = _synthesis_model(r, dev)
        ohp.stop_frames = 10 ** 6
        g = torch.Generator().manual_seed(400 + r)
        L = 17
        d = torch.randint(0, 5, (L,), generator=g)
        d[0] = 2
        frames = int(d.sum())
        rows = F.durations_to_alignment(d, r)
        S = rows.shape[0]
        tape = {k: (torch.rand(S, 1, ohp.prenet_dimension, generator=g) >= 0.5).float() for k in ('step_prenet0', 'step_prenet1')}
        encoded = torch.randn(1, L, ohp.encoder_dimension, generator=g)
        mask = O.lengths_to_mask(torch.tensor([L]), L)
        MaskSource.use_tape({k: v.to(dev) for k, v in tape.items()})
        try:
            spec, stop, align, cuts = model._decoder._decode_inference(encoded.to(dev), mask.to(dev), None, None,
                                                                       plans=[(rows.to(dev), frames)])
        finally:
            MaskSource.use_tape(None)
        assert cuts == [frames] and spec.shape[1] == frames and align.shape[1] == S
        sd = {k: v.detach().cpu().double() for k, v in model.state_dict().items() if v.is_floating_point()}
        _decoder_sd_alias(sd)
        with FO.forced(rows.double()[:, None, :]):
            spec_o, _, align_o = R.decoder_forward(sd, ohp, encoded.double(), mask, None, None, None,
                                                   {k: v.double() for k, v in tape.items()}, training=False, max_frames=frames)
        assert spec_o.shape[1] == frames
        assert_close(spec.cpu(), spec_o, 1e-3, 1e-4, 'forced inference spectrogram')
        assert torch.equal(align[0].argmax(1).cpu(), rows.argmax(1)) and torch.equal(align[0].cpu(), rows)
        assert torch.equal(align_o[0].float(), rows)
    finally:
        hp.reset()


# ---- independence ----
def _durations(g, texts, scale=3):
    return [torch.randint(0, scale, (int(t.shape[0]),), generator=g) + (torch.arange(int(t.shape[0])) == 0).long() for t in texts]


def test_batch_equals_single():
    model = _fresh_model(500, max_output_length=60)
    _sharpen(model)
    g = torch.Generator().manual_seed(501)
    texts, tape = _texts_and_tape(model, [12, 30, 7, 25, 18], 60, 502)
    dur = _durations(g, texts)
    durations = [dur[0], None, dur[2], dur[3], None]
    singles = []
    for i, t in enumerate(texts):
        col = {k: v[:, i:i + 1] for k, v in tape.items()}
        singles.append(_taped(col, lambda: model.inference(t, durations=durations[i])))
    for i in (0, 2, 3):
        assert singles[i].shape[1] == int(dur[i].sum())
    for max_batch in (1, 3, 64):
        outs = _taped(tape, lambda: model.inference_batch(texts, max_batch=max_batch, durations=durations))
        for i, (a, b) in enumerate(zip(outs, singles)):
            assert a.shape == b.shape and torch.equal(a, b), (max_batch, i)


def test_pool_equals_solo_stream():
    """Forced and free rows join at different calls, a longer forced text joins a running group, one row is closed."""
    model = _fresh_model(600, max_output_length=60)
    with torch.no_grad():
        model._decoder._stop_prediction.bias.fill_(-1e4)
    P = model._decoder._prenet._layers[0].weight.shape[0]
    g = torch.Generator().manual_seed(601)
    texts = [torch.randint(3, 20, (n,), generator=g).cuda() for n in (12, 30, 7, 45, 20)]
    masks = [{k: (torch.rand(60, P, generator=g) >= 0.5).to(torch.uint8) for k in ('step_prenet0', 'step_prenet1')} for _ in texts]
    dur = _durations(g, texts, scale=2)
    durations = [dur[0], None, torch.full((7,), 6), dur[3], None]        # the closed text is forced, with 42 frames
    opens, closes = {0: [0, 1], 1: [2], 3: [3, 4]}, {2: [2]}
    pool = model.decoder_pool(4, 9)
    ids, out, call = {}, {}, 0
    while call <= max(opens) or pool.ids:
        for j in opens.get(call, []):
            ids[j] = pool.open(texts[j], masks=masks[j], durations=durations[j])
            out[j] = []
        for j in closes.get(call, []):
            pool.close(ids[j])
        for tid, chunk in pool.run().items():
            out[next(k for k, i in ids.items() if i == tid)].append(chunk)
        call += 1
    for j in (0, 1, 3, 4):
        got = torch.cat(out[j], 1)
        tape = {k: v.unsqueeze(1) for k, v in masks[j].items()}
        ref = _taped(tape, lambda: torch.cat(list(model.inference_stream(texts[j], chunk_frames=9, durations=durations[j])), 1))
        assert torch.equal(got, ref), j
        if durations[j] is not None:
            assert got.shape[1] == int(durations[j].sum()), j


def test_server_request_equals_speech_stream():
    from multilingual_text_to_speech_b200.modules.streaming import SpeechServer, speech_stream
    model = _fresh_model(700, max_output_length=120)
    _sharpen(model)
    voc = make_model('RAW', seed=701)
    U, hop = voc.uniforms_per_step(), voc.hop_length
    P = model._decoder._prenet._layers[0].weight.shape[0]
    g = torch.Generator().manual_seed(702)
    lens = [14, 40, 22]
    texts = [torch.randint(3, 20, (n,), generator=g).cuda() for n in lens]
    dur = [torch.randint(0, 3, (n,), generator=g) + 2 for n in lens]      # at least the 21 frames a WaveRNN stream needs
    durations = [dur[0], None, dur[2]]
    masks = [{k: (torch.rand(120, P, generator=g) >= 0.5).to(torch.uint8) for k in ('step_prenet0', 'step_prenet1')} for _ in lens]
    unis = [torch.rand(1, 120 * hop, U, generator=g) for _ in lens]
    server = SpeechServer(model, voc, 2, _widen, 16)
    ids = {server.submit(texts[j], masks=masks[j], uniforms=unis[j], durations=durations[j]): j for j in range(3)}
    out = {j: [] for j in range(3)}
    while server.pending or server.active:
        for rid, chunk in server.step().items():
            out[ids[rid]].append(chunk)
    for j in (0, 2):
        tape = {k: v.unsqueeze(1) for k, v in masks[j].items()}
        ref = _taped(tape, lambda: torch.cat(list(speech_stream(model, voc, texts[j], None, None, _widen, 16, unis[j],
                                                                durations=durations[j]))))
        got = torch.cat(out[j])
        assert got.shape == ref.shape and torch.equal(got, ref), j
