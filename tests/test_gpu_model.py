"""GPU parity of the whole model (embedding, encoders, classifier, fused decoder, postnet, loss) against the golden
vectors recorded from the unmodified reference, including every parameter gradient and the BN running statistics."""
import pytest
import torch

import model_cases
from helpers import GOLDEN_CASES

pytestmark = pytest.mark.gpu


@pytest.fixture(scope='module', autouse=True)
def _built():
    import __graft_entry__ as entry
    entry.build()
    assert torch.cuda.is_available()


@pytest.mark.parametrize('name', GOLDEN_CASES)
def test_model_matches_reference_golden(name):
    model_cases.run_golden(name, check_grads=True, verbose=True)


# the full-size model of each encoder family: generated_training (G=10), and the vanilla encoder's ljspeech (E=512, bi-LSTM H=256,
# decoder memory M=512) and shared_switching (E=256, H=128, M=256+32 speaker+4 language=292, with the speaker classifier)
FULL_SIZE_CONFIGS = ('generated_training', 'ljspeech', 'shared_switching')


def test_full_size_model_fp32_and_bf16_modes():
    """Every configuration of FULL_SIZE_CONFIGS at the real dimensions (D=1024, A=128): fp32 mode meets the parity gate against the
    fp64 oracle; bf16 perf mode (persistent kernels + tensor-core GEMMs) meets the north_star gate mel L1 < 1e-3."""
    for config in FULL_SIZE_CONFIGS:
        _full_size_model(config)
        torch.cuda.empty_cache()


def _full_size_model(config):
    import types
    from multilingual_text_to_speech_b200 import configs, _lib
    from multilingual_text_to_speech_b200.modules.tacotron2 import Tacotron
    from multilingual_text_to_speech_b200.rng import MaskSource
    from oracle import tacotron_oracle as O
    from helpers import assert_close
    hp = configs.apply(config, decoder_regularization='zoneout')
    B, L, T = 20, 48, 24
    torch.manual_seed(0)
    model = Tacotron().train()
    g = torch.Generator().manual_seed(5)
    text = torch.randint(1, hp.symbols_count() + 3, (B, L), generator=g)
    lens = torch.sort(torch.randint(L // 2, L + 1, (B,), generator=g), descending=True).values; lens[0] = L
    for b in range(B):
        text[b, lens[b]:] = 0
    mel = torch.randn(B, hp.num_mels, T, generator=g)
    tlens = torch.full((B,), T)
    lang = torch.arange(B) % hp.language_number if hp.multi_language else None
    spk = torch.randint(0, hp.speaker_number, (B,), generator=g) if hp.multi_speaker else None
    D, P = hp.decoder_dimension, hp.prenet_dimension
    keep = lambda shape, p: (torch.rand(*shape, generator=g) >= p).float()   # noqa: E731
    tape = {'teacher': torch.ones(T, dtype=torch.bool), 'prenet0': keep((B, T + 1, P), 0.5), 'prenet1': keep((B, T + 1, P), 0.5),
            'att_h': keep((T, B, D), 0.1), 'att_c': keep((T, B, D), 0.1), 'gen_h': keep((T, B, D), 0.1), 'gen_c': keep((T, B, D), 0.1)}
    if hp.encoder_type == 'simple':     # the vanilla encoder's conv dropout (ConvBlock._mask_key enc0 .. enc2)
        tape.update({f'enc{j}': keep((B, hp.encoder_dimension, L), hp.dropout) for j in range(hp.encoder_blocks)})
    sd = {k: v.detach().double() for k, v in model.state_dict().items()}
    for k in list(sd):
        if k.startswith('_decoder._prenet.') or k.startswith('_decoder._attention.'):
            sd[k] = sd[k[len('_decoder.'):]]
    ns = types.SimpleNamespace(**hp.state_dict())
    with torch.no_grad():
        post_o, pre_o, stop_o, align_o, spk_o, enc_o = O.tacotron_forward(sd, ns, text, lens, mel.double(), tlens, spk, lang, tape,
                                                                           training=True)
    dev = torch.device('cuda:0')
    model = model.to(dev)
    results = {}
    for mode in ('fp32', 'bf16'):
        _lib.set_precision(mode)
        MaskSource.use_tape(tape)
        try:
            with torch.no_grad():
                post, pre, stop, align, spk_pred, enc = model(text.to(dev), lens.to(dev), mel.to(dev), tlens.to(dev),
                                                              None if spk is None else spk.to(dev), None if lang is None else lang.to(dev), 1.0)
        finally:
            MaskSource.use_tape(None)
            _lib.set_precision('fp32')
        results[mode] = {'pre_l1': float((pre.cpu().double() - pre_o).abs().mean()), 'post_l1': float((post.cpu().double() - post_o).abs().mean()),
                         'align_l1': float((align.cpu().double() - align_o).abs().mean()),
                         'argmax': float((align.cpu().argmax(2) == align_o.argmax(2)).float().mean())}
        if mode == 'fp32':
            assert_close(enc, enc_o, 1e-3, 1e-4, f'{config} enc'); assert_close(pre, pre_o, 1e-3, 1e-4, f'{config} pre')
            assert_close(align, align_o, 1e-3, 1e-4, f'{config} align'); assert_close(stop, stop_o, 1e-3, 1e-4, f'{config} stop')
            assert torch.equal(align.cpu().argmax(2), align_o.argmax(2)), f'{config} alignment argmax'
            if spk_o is not None:
                assert_close(spk_pred, spk_o, 1e-3, 1e-4, f'{config} speaker prediction')
    print(f'full-size {config} model vs fp64 oracle:', results, 'mean |pre| =', float(pre_o.abs().mean()))
    # mel gate on the decoder output; `post` adds 5 train-mode BatchNorm layers that amplify ANY input difference ~50x at
    # random init (SURVEY 7.3: a 3.5e-4 pre difference became 1.7e-2 in post with an exact fp32 postnet), so it is only bounded loosely
    assert results['bf16']['pre_l1'] < 1e-3 and results['bf16']['post_l1'] < 5e-2, (config, results)
