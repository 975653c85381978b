"""Windowed synthesis (hp.inference_attention_window) on the GPU:
  * the reference's own inference with its attention windowed (tests/golden/make_golden_attention_window.py) at chunks of 7 and 128;
  * a window covering every position gives the bits of no window, in both precision modes;
  * from the returned alignments alone, every row lies in the window of the previous row's first argmax and sums to 1 (r = 1 and 2);
  * inference_batch, a DecoderPool with joins, leaves and a close, and a SpeechServer request each equal the text decoded alone;
  * one-step chunks from crafted states against the fp64 oracle, including the window centre the kernel writes back;
  * the library refuses a window with forward attention and outside b200tts_decoder_forward_chunk."""
import json
import os

import numpy as np
import pytest
import torch

import attention_window_oracle as AW
from helpers import GOLDEN_DIR, assert_close
from oracle import tacotron_oracle as O
from multilingual_text_to_speech_b200 import _lib
from multilingual_text_to_speech_b200 import functional as F
from test_gpu_batch_inference import _batch, _case, _single
from test_gpu_speech_server import _drive_pool, _fresh_model, _serve, _solo_stream, _speech_solo, _widen, fixed_cuts  # noqa: F401
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


class _Capture:
    """Records the alignment of every decoder call: {call: [b, S_c, L]}."""

    def __init__(self):
        self.aligns = []

    def __enter__(self):
        self.orig = F.decoder_forward_chunk

        def chunk(*a, **k):
            spec, stop, align = self.orig(*a, **k)
            self.aligns.append(align.clone())
            return spec, stop, align
        F.decoder_forward_chunk = chunk
        return self

    def __exit__(self, *exc):
        F.decoder_forward_chunk = self.orig


@pytest.mark.parametrize('chunk', [7, 128])
@pytest.mark.parametrize('name', ['inf_window_lj', 'inf_window_generated_mix'])
def test_window_matches_reference(name, chunk):
    from multilingual_text_to_speech_b200.params.params import Params as hp
    from multilingual_text_to_speech_b200.modules.tacotron2 import Tacotron, Decoder
    from multilingual_text_to_speech_b200.rng import MaskSource
    z = np.load(os.path.join(GOLDEN_DIR, name + '.npz'))
    meta = json.loads(bytes(z['meta']).decode())
    hp.reset()
    hp.load_state_dict(meta['hp'])
    hp.inference_attention_window = meta['window']
    model = Tacotron()
    model.load_state_dict({k[3:]: torch.from_numpy(z[k]) for k in z.files if k.startswith('sd.')}, strict=True)
    dev = torch.device('cuda:0')
    model = model.to(dev).eval()
    tape = {k[5:]: torch.from_numpy(z[k]) for k in z.files if k.startswith('tape.')}
    language = torch.from_numpy(z['in.language']).to(dev) if 'in.language' in z.files else None
    old = Decoder.inference_chunk
    Decoder.inference_chunk = chunk
    MaskSource.use_tape(tape)
    try:
        with _Capture() as cap:
            out = model.inference(torch.from_numpy(z['in.text']).to(dev), speaker=None, language=language)
    finally:
        MaskSource.use_tape(None)
        Decoder.inference_chunk = old
    T = meta['T']
    ref = torch.from_numpy(z['out.post'])
    assert tuple(out.shape) == tuple(ref.shape) == (hp.num_mels, T), (out.shape, ref.shape)
    assert_close(out, ref, 1e-3, 1e-4, f'{name}: windowed inference spectrogram')
    align = torch.cat(cap.aligns, 1)[0, :T]
    assert torch.equal(align.argmax(1).cpu().to(torch.int32), torch.from_numpy(z['out.argmax']))
    AW.check_window_property(align[None], [meta['L']], meta['window'])


def _group(model, texts, window, tape):
    """One padded decode of `texts` through the chunk loop -> (spectrogram, stop, alignment, cuts, lengths)."""
    from multilingual_text_to_speech_b200.rng import MaskSource
    encoded, mask, speaker, language = model._encode_group(texts, None, None)
    MaskSource.use_tape(tape)
    try:
        with torch.no_grad():
            out = model._decoder._decode_inference(encoded, mask, speaker, language, att_extent=1, att_window=window)
    finally:
        MaskSource.use_tape(None)
    return out + ([int(t.shape[0]) for t in texts],)


def _texts_and_tape(model, lens, frames, seed):
    g = torch.Generator().manual_seed(seed)
    texts = [torch.randint(3, 20, (n,), generator=g).cuda() for n in lens]
    P = model._decoder._prenet._layers[0].weight.shape[0]
    tape = {k: (torch.rand(frames, len(lens), P, generator=g) >= 0.5).to(torch.uint8) for k in ('step_prenet0', 'step_prenet1')}
    return texts, tape


def _sharpen(model):
    with torch.no_grad():
        model._attention._energy.weight.mul_(6.0)
        model._attention._query.weight.mul_(3.0)
        model._decoder._stop_prediction.bias.fill_(-1e4)          # every text decodes max_output_length frames


@pytest.mark.parametrize('precision', ['fp32', 'bf16'])
def test_full_coverage_window_is_bitwise_no_window(precision):
    model = _fresh_model(70, max_output_length=50)
    _sharpen(model)
    texts, tape = _texts_and_tape(model, [23, 9, 40], 50, 71)
    _lib.set_precision(precision)
    off = _group(model, texts, None, tape)
    for window in ((40, 40), (1000, 64)):
        on = _group(model, texts, window, tape)
        for k in range(3):
            assert torch.equal(on[k], off[k]), (precision, window, k)
        assert on[3] == off[3]


@pytest.mark.parametrize('r', [1, 2])
@pytest.mark.parametrize('precision', ['fp32', 'bf16'])
def test_window_property(precision, r):
    model = _fresh_model(72 + r, max_output_length=60, outputs_per_step=r)
    _sharpen(model)
    texts, tape = _texts_and_tape(model, [31, 12, 50, 3], 60, 74)
    _lib.set_precision(precision)
    free = _group(model, texts, None, tape)[2]
    for window in ((1, 3), (0, 1), (4, 2)):
        spec, stop, align, cuts, lens = _group(model, texts, window, tape)
        assert align.shape[1] == -(-60 // r)
        AW.check_window_property(align, lens, window)
        assert not torch.equal(align, free), window            # the window binds on these texts


def _with_window(window, fn):
    from multilingual_text_to_speech_b200.params.params import Params as hp
    hp.inference_attention_window = list(window)
    try:
        return fn()
    finally:
        hp.inference_attention_window = None


def test_batch_equals_single():
    """inference_batch's groups (1, 3 and all texts at once) give every text its own decode, bit for bit."""
    model, utts, meta = _case('inf_batch_lj')
    assert len(set(meta['T'])) > 1                            # the texts stop at different frames
    for window in ((1, 3), (0, 2)):
        singles = _with_window(window, lambda: [_single(model, u) for u in utts])
        for max_batch in (1, 3, 64):
            outs = _with_window(window, lambda: _batch(model, utts, max_batch))
            for j, (a, b) in enumerate(zip(outs, singles)):
                assert a.shape == b.shape and torch.equal(a, b), (window, max_batch, j)


def test_pool_equals_solo_stream(fixed_cuts):  # noqa: F811
    """Staggered opens, a longer text joining a running group, the longest leaving first, and a close."""
    model = _fresh_model(80, max_output_length=60)
    _sharpen(model)
    fixed_cuts.update({12: 50, 30: 40, 7: 60, 45: 25, 20: 55})     # text length -> cut: the 45-character text joins last, leaves first
    P = model._decoder._prenet._layers[0].weight.shape[0]
    g = torch.Generator().manual_seed(81)
    texts = [torch.randint(3, 20, (n,), generator=g).cuda() for n in (12, 30, 7, 45, 20)]
    masks = [{k: (torch.rand(60, P, generator=g) >= 0.5).to(torch.uint8) for k in ('step_prenet0', 'step_prenet1')} for _ in texts]

    def run():
        from multilingual_text_to_speech_b200.params.params import Params as hp
        pool = model.decoder_pool(4, 9)
        assert pool.rows.att_window == (1, 3)
        hp.inference_attention_window = None            # a running pool keeps the window it was built with
        opens = {0: [(0, (texts[0], None, None, masks[0])), (1, (texts[1], None, None, masks[1]))], 1: [(2, (texts[2], None, None, masks[2]))],
                 3: [(3, (texts[3], None, None, masks[3])), (4, (texts[4], None, None, masks[4]))]}
        return _drive_pool(pool, opens, closes={2: [2]})[0]
    got = _with_window((1, 3), run)
    assert got[2].shape[1] < 60 and got[3].shape[1] == 25
    for j in (0, 1, 3, 4):
        ref = _with_window((1, 3), lambda: _solo_stream(model, texts[j], None, None, masks[j], 9))
        assert torch.equal(got[j], ref), j
    off = _drive_pool(model.decoder_pool(4, 9), {0: [(0, (texts[3], None, None, masks[3]))]})[0][0]
    assert not torch.equal(off, got[3])


def test_server_request_equals_speech_stream(fixed_cuts):  # noqa: F811
    from multilingual_text_to_speech_b200.modules.streaming import SpeechServer
    model = _fresh_model(90, max_output_length=120)
    _sharpen(model)
    voc = make_model('RAW', seed=91)
    U, hop = voc.uniforms_per_step(), voc.hop_length
    P = model._decoder._prenet._layers[0].weight.shape[0]
    g = torch.Generator().manual_seed(92)
    lens = [14, 40, 22]
    for i, n in enumerate(lens):
        fixed_cuts[n] = 30 + 17 * i
    texts = {n: torch.randint(3, 20, (n,), generator=g).cuda() for n in lens}
    masks = {n: {k: (torch.rand(120, P, generator=g) >= 0.5).to(torch.uint8) for k in ('step_prenet0', 'step_prenet1')} for n in lens}
    unis = {n: torch.rand(1, fixed_cuts[n] * hop, U, generator=g) for n in lens}

    def serve():
        server = SpeechServer(model, voc, 2, _widen, 16)
        script = lambda c: [('submit', lens[c], dict(text=texts[lens[c]], masks=masks[lens[c]], uniforms=unis[lens[c]]))] if c < 3 else []  # noqa: E731
        return _serve(server, script, 3)[0]
    got = _with_window((1, 3), serve)
    for n in lens:
        ref = _with_window((1, 3), lambda: _speech_solo(model, voc, texts[n], masks[n], unis[n], 16))
        assert got[n].shape == ref.shape and torch.equal(got[n], ref), n


# ---- one step against fp64 ----
def _small_sd(g, M, D, P, A, C, K, N):
    rn = lambda *s, scale=1.0: torch.randn(*s, generator=g, dtype=torch.float64) * scale     # noqa: E731
    s_in = lambda n: 1.0 / np.sqrt(n)   # noqa: E731
    sd = {'_prenet._layers.0.weight': rn(P, N, scale=s_in(N)), '_prenet._layers.0.bias': rn(P, scale=0.1),
          '_prenet._layers.1.weight': rn(P, P, scale=s_in(P)), '_prenet._layers.1.bias': rn(P, scale=0.1),
          '_decoder._attention_lstm.weight_ih': rn(4 * D, P + M, scale=s_in(D)), '_decoder._attention_lstm.weight_hh': rn(4 * D, D, scale=s_in(D)),
          '_decoder._attention_lstm.bias_ih': rn(4 * D, scale=0.1), '_decoder._attention_lstm.bias_hh': rn(4 * D, scale=0.1),
          '_decoder._generator_lstm.weight_ih': rn(4 * D, D + M, scale=s_in(D)), '_decoder._generator_lstm.weight_hh': rn(4 * D, D, scale=s_in(D)),
          '_decoder._generator_lstm.bias_ih': rn(4 * D, scale=0.1), '_decoder._generator_lstm.bias_hh': rn(4 * D, scale=0.1),
          '_attention._query.weight': rn(A, D, scale=3 * s_in(D)), '_attention._memory.weight': rn(A, M, scale=3 * s_in(M)),
          '_attention._location.weight': rn(A, C, scale=s_in(C)), '_attention._loc_features.weight': rn(C, 1, K, scale=s_in(K)),
          '_attention._bias': rn(1, A, scale=0.1), '_attention._energy.weight': rn(1, A, scale=6 * s_in(A)),
          '_decoder._frame_prediction.weight': rn(N, D + M, scale=s_in(D + M)), '_decoder._frame_prediction.bias': rn(N, scale=0.1),
          '_decoder._stop_prediction.weight': rn(1, D + M, scale=s_in(D + M)), '_decoder._stop_prediction.bias': rn(1, scale=0.1)}
    return sd


@pytest.mark.parametrize('L', [1, 2, 5, 37, 128, 300])
def test_one_step_against_fp64(L):
    from decoder_cases import PARAM_KEYS
    M, D, P, A, C, K, N = 64, 64, 32, 32, 8, 7, 8
    g = torch.Generator().manual_seed(100 + L)
    sd = {k: v.float().double() for k, v in _small_sd(g, M, D, P, A, C, K, N).items()}     # the weights the kernels read
    lens = [L, max(1, L - 1), max(1, L // 2)]
    B = len(lens)
    memory = torch.randn(B, L, M, generator=g, dtype=torch.float64).float().double()
    cum0 = (torch.rand(B, L, generator=g) * 2 * O.lengths_to_mask(torch.tensor(lens), L)).double()
    h0 = [(torch.randn(B, D, generator=g) * 0.5).double() for _ in range(4)]
    ctx0 = (torch.randn(B, M, generator=g) * 0.5).double()
    frame0 = torch.randn(B, N, generator=g).double()
    keep = [(torch.rand(1, B, P, generator=g) >= 0.5).to(torch.uint8) for _ in range(2)]
    dev = torch.device('cuda:0')
    params = [sd[key].float().to(dev) for _, key in PARAM_KEYS]
    _lib.set_precision('fp32')
    mask = O.lengths_to_mask(torch.tensor(lens), L)
    # fp64: prenet of the carried frame, attention LSTM (eval), then the windowed attention step
    x = O.prenet(sd, '_prenet', frame0, 0.5, keep[0][0].double(), keep[1][0].double())
    w_att = tuple(sd[f'_decoder._attention_lstm.{n}'] for n in ('weight_ih', 'weight_hh', 'bias_ih', 'bias_hh'))
    h_att, _ = O.regularised_cell('dropout', False, torch.cat((x, ctx0), 1), h0[0], h0[1], w_att, (0.1, 0.0))
    memT, _, _ = O.attention_reset(sd, '_attention', memory)
    for centres in ([0, 0, 0], [l - 1 for l in lens], [l // 2 for l in lens]):
        for window in ((0, 1), (1, 3), (40, 90)):
            st = F.DecoderState(B, D, M, L, N, dev)
            st.att_h.copy_(h0[0]); st.att_c.copy_(h0[1]); st.gen_h.copy_(h0[2]); st.gen_c.copy_(h0[3])
            st.context.copy_(ctx0); st.cum_weights.copy_(cum0); st.frame.copy_(frame0)
            st.attended.copy_(torch.tensor(centres, dtype=torch.int32))
            st.first = False
            cfg = F.DecoderConfig(_lib.CELL_DROPOUT, False, 0.1, 0.0, 0.5, {'step_prenet0': keep[0].to(dev), 'step_prenet1': keep[1].to(dev)},
                                  np.zeros(1, dtype=np.uint8), 1, att_window=window)
            _, _, align = F.decoder_forward_chunk(cfg, memory.float().to(dev), torch.tensor(lens, device=dev), params, st, 1)
            ctx64, w64, cum64, c64 = AW.attention_step(sd, '_attention', h_att, memory, memT, cum0, mask, torch.tensor(centres), window)
            w = align[:, 0].double().cpu()
            what = f'L={L} centres={centres} window={window}'
            assert float((w - w64).abs().max()) <= 2e-5, (what, float((w - w64).abs().max()))
            assert torch.equal(w == 0, w64 == 0), what            # the same positions outside the window
            bound = 2e-5 * (w64[:, :, None] * memory.abs()).sum(1) + 1e-5
            assert bool(((st.context.double().cpu() - ctx64).abs() <= bound).all()), what
            assert torch.allclose(st.cum_weights.double().cpu(), cum64, atol=2e-5), what
            got = st.attended.cpu().long()
            assert torch.equal(got, w.argmax(1)), what             # the first argmax of the row the kernel wrote
            top2 = w64.topk(min(2, L), dim=1).values
            clear = (top2[:, 0] - top2[:, -1] > 1e-3 * top2[:, 0]) | (top2.shape[1] == 1)
            assert torch.equal(got[clear], c64[clear]), what


def test_library_errors():
    model = _fresh_model(60, max_output_length=20)
    texts, tape = _texts_and_tape(model, [9, 4], 20, 61)
    dec = model._decoder
    encoded, mask, _, _ = model._encode_group(texts, None, None)
    kind, rate_h, rate_c = dec._cell_config()
    lengths = mask.sum(1).to(torch.int32)
    cfg = F.DecoderConfig(kind, False, rate_h, rate_c, 0.5, None, None, att_window=(1, 3))
    target = torch.zeros(2, dec._output_dim, 20, device='cuda')
    with pytest.raises(_lib.B200TTSError, match='attention window is for synthesis only'):
        F.decoder_forward(cfg, encoded, target, lengths, dec._param_list())
    fwd = _fresh_model(62, max_output_length=20, attention_type='forward')
    dec = fwd._decoder
    encoded, mask, _, _ = fwd._encode_group(texts, None, None)
    st = F.DecoderState(2, dec._decoder_dim, encoded.shape[2], encoded.shape[1], dec._output_dim, 'cuda')
    cfg = F.DecoderConfig(kind, False, rate_h, rate_c, 0.5, None, np.zeros(4, dtype=np.uint8), 1, att_window=(1, 3))
    with pytest.raises(_lib.B200TTSError, match='forward attention'):
        F.decoder_forward_chunk(cfg, encoded, mask.sum(1), dec._param_list(), st, 4)
