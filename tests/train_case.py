"""Two optimisation steps of the reference's training procedure (train.py:29-95) at small dimensions, shared by the golden generator
(tests/golden/make_golden_train.py, which runs the UNMODIFIED reference's own `train()` on its own modules, CPU fp32) and the GPU test
(tests/test_gpu_reference_train.py, this package).  Every regularisation rate is zero and teacher forcing is constant 1, so the two
runs see the same arithmetic; the model weights come from `torch.manual_seed(0); Tacotron()` in both (parameters are constructed in the
reference's order).
"""
import torch

CONFIGS = ('generated_switching', 'ljspeech')
SPEAKERS = 3
SMALL = dict(embedding_dimension=32, encoder_dimension=32, prenet_dimension=24, attention_dimension=16, attention_kernel_size=7,
             attention_location_dimension=8, decoder_dimension=48, postnet_dimension=32, num_mels=12, reversal_classifier_dim=16,
             speaker_embedding_dimension=8)
DETERMINISTIC = dict(dropout=0.0, zoneout_hidden=0.0, zoneout_cell=0.0, dropout_hidden=0.0, constant_teacher_forcing=True, teacher_forcing=1.0)
REGULARIZATION = {'generated_switching': 'zoneout', 'ljspeech': 'dropout'}


def overrides(config):
    return dict(SMALL, decoder_regularization=REGULARIZATION[config], **DETERMINISTIC)


def make_batch(hp):
    """The batch tuple train() unpacks: (src, src_len, trg_mel, trg_lin, trg_len, stop_trg, spkrs, langs)."""
    G = max(hp.language_number, 1)
    B, L, T = 2 * G, 14, 20
    g = torch.Generator().manual_seed(3)
    lens = torch.sort(torch.randint(L // 2, L + 1, (B,), generator=g), descending=True).values
    lens[0] = L
    text = torch.randint(1, hp.symbols_count() + 3, (B, L), generator=g)
    for b in range(B):
        text[b, lens[b]:] = 0
    tlens = torch.full((B,), T)
    stop = torch.zeros(B, T)
    stop[:, -hp.stop_frames:] = 1
    return (text, lens, torch.randn(B, hp.num_mels, T, generator=g), None, tlens, stop,
            torch.randint(0, SPEAKERS, (B,), generator=g) if hp.multi_speaker else None,
            (torch.arange(B) % G) if hp.multi_language else None)


def param_sums(model):
    """Per-parameter float64 sums (name order): identical weights on both sides."""
    return torch.tensor([float(p.detach().double().sum()) for _, p in sorted(model.named_parameters())], dtype=torch.float64)
