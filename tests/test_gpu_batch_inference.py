"""Tacotron.inference_batch: batched synthesis with per-utterance stop.  Every utterance's output must equal the unmodified reference's
own batch-1 `inference()` (tests/golden/make_golden_batch_inference.py) and the library's own `inference()` of that utterance alone,
given the same prenet dropout masks; finished utterances leave the decode; the length-masked conv block matches an fp64 conv1d."""
import json
import os
import numpy as np
import pytest
import torch

from helpers import GOLDEN_DIR, assert_close

pytestmark = pytest.mark.gpu

CASES = ['inf_batch_lj', 'inf_batch_generated', 'inf_batch_convolutional', 'inf_batch_forward']


@pytest.fixture(scope='module', autouse=True)
def _built():
    import __graft_entry__ as entry
    entry.build()
    assert torch.cuda.is_available()


class _Precision:
    def __init__(self, name):
        self.name = name

    def __enter__(self):
        from multilingual_text_to_speech_b200 import _lib
        _lib.set_precision(self.name)

    def __exit__(self, *exc):
        from multilingual_text_to_speech_b200 import _lib
        _lib.set_precision('fp32')


def _case(name):
    """-> (model on cuda, utterances [(text, speaker, language, tape0, tape1, out)], meta)"""
    from multilingual_text_to_speech_b200.params.params import Params as hp
    from multilingual_text_to_speech_b200.modules.tacotron2 import Tacotron
    z = np.load(os.path.join(GOLDEN_DIR, name + '.npz'))
    meta = json.loads(bytes(z['meta']).decode())
    hp.reset()
    hp.load_state_dict(meta['hp'])
    model = Tacotron()
    model.load_state_dict({k[3:]: torch.from_numpy(z[k]) for k in z.files if k.startswith('sd.')}, strict=True)
    model = model.cuda().eval()
    dev = torch.device('cuda:0')
    utts = []
    for j in range(meta['n']):
        get = lambda k: torch.from_numpy(z[k]).to(dev) if k in z.files else None   # noqa: E731
        utts.append((get(f'text{j}'), get(f'speaker{j}'), get(f'language{j}'), torch.from_numpy(z[f'tape{j}.step_prenet0']),
                     torch.from_numpy(z[f'tape{j}.step_prenet1']), torch.from_numpy(z[f'out{j}'])))
    return model, utts, meta


def _stacked_tape(tapes):
    """Per-utterance tapes [T_i, P] -> one [max T_i, n, P] tape, padded with ones (frames past an utterance's own tape are discarded)."""
    T = max(t.shape[0] for t in tapes)
    out = torch.ones(T, len(tapes), tapes[0].shape[1], dtype=torch.uint8)
    for j, t in enumerate(tapes):
        out[:t.shape[0], j] = t
    return out


def _batch(model, utts, max_batch=64):
    from multilingual_text_to_speech_b200.rng import MaskSource
    MaskSource.use_tape({'step_prenet0': _stacked_tape([u[3] for u in utts]), 'step_prenet1': _stacked_tape([u[4] for u in utts])})
    try:
        speakers = None if utts[0][1] is None else [u[1] for u in utts]
        languages = None if utts[0][2] is None else [u[2] for u in utts]
        return model.inference_batch([u[0] for u in utts], speakers, languages, max_batch=max_batch)
    finally:
        MaskSource.use_tape(None)


def _single(model, u):
    from multilingual_text_to_speech_b200.rng import MaskSource
    MaskSource.use_tape({'step_prenet0': u[3].unsqueeze(1), 'step_prenet1': u[4].unsqueeze(1)})
    try:
        return model.inference(u[0], speaker=u[1], language=u[2])
    finally:
        MaskSource.use_tape(None)


@pytest.mark.parametrize('chunk', [7, 128])
@pytest.mark.parametrize('name', CASES)
def test_batch_matches_reference(name, chunk):
    from multilingual_text_to_speech_b200.modules.tacotron2 import Decoder
    model, utts, meta = _case(name)
    old = Decoder.inference_chunk
    Decoder.inference_chunk = chunk
    try:
        outs = _batch(model, utts)
    finally:
        Decoder.inference_chunk = old
    assert len(outs) == len(utts)
    for j, (out, u) in enumerate(zip(outs, utts)):
        assert tuple(out.shape) == tuple(u[5].shape) == (model._decoder._output_dim, meta['T'][j]), (j, out.shape, u[5].shape)
        assert_close(out, u[5], 1e-3, 1e-4, f'{name}: utterance {j}')


@pytest.mark.parametrize('max_batch', [2, 64])
@pytest.mark.parametrize('precision', ['fp32', 'bf16'])
@pytest.mark.parametrize('name', CASES)
def test_batch_equals_single(name, precision, max_batch):
    """Per-row arithmetic does not depend on the batch at these shapes (no split-K change below 64 rows, fixed k order), and the
    padded positions are exact zeros, so a batched utterance is bit-identical to the same utterance decoded alone."""
    model, utts, _ = _case(name)
    with _Precision(precision):
        outs = _batch(model, utts, max_batch)
        singles = [_single(model, u) for u in utts]
    for j, (a, b) in enumerate(zip(outs, singles)):
        assert a.shape == b.shape, (j, a.shape, b.shape)
        assert torch.equal(a, b), f'{name} {precision} max_batch={max_batch} utterance {j}: max |diff| {float((a - b).abs().max())}'


def test_finished_utterances_leave_the_decode():
    from multilingual_text_to_speech_b200 import functional as F
    from multilingual_text_to_speech_b200.modules.tacotron2 import Decoder
    model, utts, meta = _case('inf_batch_lj')
    chunk, calls = 7, []
    orig = F.decoder_forward_chunk
    F.decoder_forward_chunk = lambda *a, **k: (calls.append((a[1].shape[0], a[-1])), orig(*a, **k))[1]
    old = Decoder.inference_chunk
    Decoder.inference_chunk = chunk
    try:
        _batch(model, utts)
    finally:
        F.decoder_forward_chunk = orig
        Decoder.inference_chunk = old
    cuts, T = meta['T'], model._decoder._max_frames
    need = [min(-(-c // chunk) * chunk, T) for c in cuts]
    done = 0
    for B, frames in calls:       # after a chunk that finished an utterance, the next call has one row fewer per finished utterance
        assert B == sum(1 for n in need if n > done), (calls, need)
        done += frames
    assert sum(B * f for B, f in calls) == sum(need), (calls, need)
    assert calls[-1][0] < calls[0][0]


def _conv_reference(x, n_len, conv_w, gamma, beta, mean, var, eps, G, k, dil, act, highway):
    """One block on one utterance alone, fp64: pad -> grouped conv1d -> eval batch norm -> activation (-> highway gate)."""
    import torch.nn.functional as TF
    x = x[:, :, :n_len].double()
    pad = (k - 1) * dil // 2
    y = TF.conv1d(TF.pad(x, (pad, pad)), conv_w.double(), dilation=dil, groups=G)
    y = (y - mean.double()[None, :, None]) / torch.sqrt(var.double()[None, :, None] + eps) * gamma.double()[None, :, None] + beta.double()[None, :, None]
    y = {'relu': torch.relu, 'tanh': torch.tanh, 'identity': lambda v: v}[act](y)
    if highway:
        C = y.shape[1] // (2 * G)
        y = y.view(1, G, 2, C, -1)
        s = torch.sigmoid(y[:, :, 0])
        y = (y[:, :, 1] * s + x.view(1, G, C, -1) * (1 - s)).reshape(1, G * C, -1)
    return y


@pytest.mark.parametrize('precision', ['fp32', 'bf16'])
@pytest.mark.parametrize('case', [
    dict(G=1, Cin=512, Cout=512, k=5, dil=1, act='relu', highway=False, L=64),          # encoder conv5 blocks
    dict(G=1, Cin=512, Cout=512, k=5, dil=1, act='relu', highway=False, L=67),
    dict(G=5, Cin=32, Cout=64, k=3, dil=27, act='identity', highway=True, L=40),        # generated grouped highway, dilation 27
    dict(G=5, Cin=32, Cout=64, k=3, dil=27, act='identity', highway=True, L=41),
    dict(G=1, Cin=80, Cout=512, k=5, dil=1, act='tanh', highway=False, L=200),          # post-net 80 -> 512
    dict(G=1, Cin=512, Cout=80, k=5, dil=1, act='identity', highway=False, L=201),      # post-net 512 -> 80
])
def test_masked_conv_block_against_fp64(case, precision):
    from multilingual_text_to_speech_b200 import functional as F
    g = torch.Generator().manual_seed(case['L'] + case['G'])
    G, Cin, Cout, k, dil, L = case['G'], case['Cin'], case['Cout'], case['k'], case['dil'], case['L']
    NB = 4
    lens = [1, L, max(2, L // 3), min(L, 2 * dil + 1)]          # 1, L, and lengths shorter than the receptive field
    dev = torch.device('cuda:0')
    x = torch.randn(NB, G * Cin, L, generator=g)
    for n, ln in enumerate(lens):
        x[n, :, ln:] = 0
    w = torch.randn(G * Cout, Cin, k, generator=g) / (Cin * k) ** 0.5
    gamma, beta = torch.rand(G * Cout, generator=g) + 0.5, torch.randn(G * Cout, generator=g) * 0.1
    mean, var = torch.randn(G * Cout, generator=g) * 0.1, torch.rand(G * Cout, generator=g) + 0.5
    cuda = [t.to(dev) for t in (x, w, gamma, beta, mean, var)]
    lengths = torch.tensor(lens, dtype=torch.int32, device=dev)
    with _Precision(precision):
        out = F.conv_block_masked(cuda[0], lengths, cuda[1], cuda[2], cuda[3], cuda[4], cuda[5], G, k, dil, case['act'],
                                  case['highway'], 1e-5, Cout).cpu()
        full = F.conv_block_masked(cuda[0], torch.full((NB,), L, dtype=torch.int32, device=dev), *cuda[1:], G, k, dil, case['act'],
                                   case['highway'], 1e-5, Cout)
        plain = F.conv_block(cuda[0], *cuda[1:], None, G, k, dil, case['act'], case['highway'], False, 1e-5, 0.1, 0.0, Cout)
    assert torch.equal(full, plain), 'every length == L must be bit-identical to the unmasked block'
    tol = 2e-4 if precision == 'fp32' else 3e-2
    for n, ln in enumerate(lens):
        ref = _conv_reference(x[n:n + 1], ln, w, gamma, beta, mean, var, 1e-5, G, k, dil, case['act'], case['highway'])[0]
        got = out[n, :, :ln].double()
        err = float((got - ref).abs().max() / max(1.0, float(ref.abs().max())))
        assert err < tol, (case, precision, n, ln, err)
        assert bool((out[n, :, ln:] == 0).all()), (case, n, ln)


def _random_lj_model():
    from multilingual_text_to_speech_b200.params.params import Params as hp
    from multilingual_text_to_speech_b200.modules.tacotron2 import Tacotron
    hp.reset()
    hp.max_output_length = 64
    torch.manual_seed(5)
    return Tacotron().cuda().eval()


def test_many_utterances_in_order_and_reproducible():
    """150 utterances in 3 groups: two identical runs are bit-identical, and each utterance equals its own single decode."""
    from multilingual_text_to_speech_b200.rng import MaskSource
    from multilingual_text_to_speech_b200.params.params import Params as hp
    model = _random_lj_model()
    g = torch.Generator().manual_seed(11)
    n, T, P = 150, 64, hp.prenet_dimension
    texts = [torch.randint(1, hp.symbols_count() + 3, (int(L),), generator=g).cuda() for L in torch.randint(5, 60, (n,), generator=g)]
    tape = {k: (torch.rand(T, n, P, generator=g) >= 0.5).to(torch.uint8) for k in ('step_prenet0', 'step_prenet1')}
    runs = []
    for _ in range(2):
        MaskSource.use_tape(tape)
        try:
            runs.append(model.inference_batch(texts, max_batch=64))
        finally:
            MaskSource.use_tape(None)
    assert all(torch.equal(a, b) for a, b in zip(*runs))
    for i in (0, 37, 149):
        MaskSource.use_tape({k: v[:, i:i + 1] for k, v in tape.items()})
        try:
            single = model.inference(texts[i])
        finally:
            MaskSource.use_tape(None)
        assert torch.equal(single, runs[0][i]), i


@pytest.mark.parametrize('precision', ['fp32', 'bf16'])
@pytest.mark.parametrize('encoder_type', ['separate', 'shared'])
def test_separate_and_shared_encoders_batch_equals_single(encoder_type, precision):
    """The padded paths of MultiEncoder (each utterance normalised by its own language sums, padding weighted 0) and ConditionalEncoder
    (the language embedding concatenated, then the padding zeroed): per-character mixes, a code-switched and an accent-blended text."""
    from multilingual_text_to_speech_b200.rng import MaskSource
    from multilingual_text_to_speech_b200.params.params import Params as hp
    from multilingual_text_to_speech_b200.modules.tacotron2 import Tacotron
    hp.reset()
    hp.load_state_dict(dict(embedding_dimension=16, encoder_dimension=16, prenet_dimension=16, decoder_dimension=32, postnet_dimension=16,
                            attention_dimension=16, max_output_length=40, encoder_type=encoder_type, multi_language=True,
                            languages=['a', 'b', 'c'], language_embedding_dimension=4, input_language_embedding=4))
    hp.language_number = 3
    torch.manual_seed(3)
    model = Tacotron().cuda().eval()
    g = torch.Generator().manual_seed(4)
    lengths = [2, 30, 11, 17]
    texts = [torch.randint(1, hp.symbols_count() + 3, (L,), generator=g).cuda() for L in lengths]
    languages = []
    for i, L in enumerate(lengths):
        w = torch.zeros(1, L, 3)
        if i == 2:                          # code-switching a | c
            w[0, :5, 0] = 1.0; w[0, 5:, 2] = 1.0
        elif i == 3:                        # accent: b*0.75 + a*0.25, un-normalised weights at the end
            w[0, :, 1] = 0.75; w[0, :, 0] = 0.25; w[0, 12:, 1] = 2.0
        else:
            w[0, :, i] = 1.0
        languages.append(w.cuda())
    T, P = hp.max_output_length, hp.prenet_dimension
    tape = {k: (torch.rand(T, len(texts), P, generator=g) >= 0.5).to(torch.uint8) for k in ('step_prenet0', 'step_prenet1')}
    with _Precision(precision):
        MaskSource.use_tape(tape)
        try:
            outs = model.inference_batch(texts, None, languages)
        finally:
            MaskSource.use_tape(None)
        for i in range(len(texts)):
            MaskSource.use_tape({k: v[:, i:i + 1] for k, v in tape.items()})
            try:
                single = model.inference(texts[i], language=languages[i])
            finally:
                MaskSource.use_tape(None)
            assert bool(torch.isfinite(outs[i]).all()), i
            assert torch.equal(single, outs[i]), (encoder_type, precision, i, float((single - outs[i]).abs().max()))
