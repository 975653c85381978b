"""Two optimisation steps of the reference's training procedure (train.py:29-95) at small dimensions, shared by the golden generator
(tests/golden/make_golden_train.py, which runs the UNMODIFIED reference's own `train()` on its own modules, CPU fp32), the CPU test
that replays it through the fp64 oracle (tests/test_reference_train_cpu.py) and the GPU test (tests/test_gpu_reference_train.py, this
package).  Teacher forcing is constant 1 and every rate that hp sets is zero (DETERMINISTIC), but the generated encoder's dropout is
fixed at 0.05 by the reference (tacotron2.py:300-302) whatever hp.dropout says: the golden records the masks the reference drew at
each step, and the other two replay them from that tape (`MaskSource.use_tape`).  The model weights come from
`torch.manual_seed(0); Tacotron()` on every side (parameters are constructed in the reference's order).

The widths are narrower than the other goldens' so that the fixture can hold every parameter's gradient at both steps (the generated
encoder's weight generators grow with the square of the encoder width).
"""
import json
import os

import numpy as np
import torch

CONFIGS = ('generated_switching', 'ljspeech')
SPEAKERS = 3
SMALL = dict(embedding_dimension=16, encoder_dimension=16, prenet_dimension=24, attention_dimension=16, attention_kernel_size=7,
             attention_location_dimension=8, decoder_dimension=32, postnet_dimension=16, num_mels=12, reversal_classifier_dim=16,
             speaker_embedding_dimension=8)
# generated_switching: the 5-language encoder is 5x as wide as encoder_dimension
WIDTHS = {'generated_switching': dict(embedding_dimension=8, encoder_dimension=8), 'ljspeech': dict()}
DETERMINISTIC = dict(dropout=0.0, zoneout_hidden=0.0, zoneout_cell=0.0, dropout_hidden=0.0, constant_teacher_forcing=True, teacher_forcing=1.0)
REGULARIZATION = {'generated_switching': 'zoneout', 'ljspeech': 'dropout'}
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'reference_train.npz')


def overrides(config):
    return dict(SMALL, **WIDTHS[config], decoder_regularization=REGULARIZATION[config], **DETERMINISTIC)


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


def quantise(tensors):
    """Per-tensor 16-bit fixed point of a list of tensors: (int16 [sum of numel], float64 scales); the rounding error is at most
    1.5e-5 of each tensor's largest magnitude."""
    q, scales = [], []
    for t in tensors:
        t = t.detach().double().reshape(-1)
        s = float(t.abs().max()) / 32767.0 if t.numel() else 0.0
        q.append(torch.round(t / s).to(torch.int16) if s > 0 else torch.zeros_like(t, dtype=torch.int16))
        scales.append(s)
    return torch.cat(q).numpy(), np.array(scales, dtype=np.float64)


class Fixture:
    """One config of reference_train.npz, in sorted parameter-name order (`names`, `shapes`):
    losses [2, K] over `loss_keys`, gradient [2] (the norm before clipping), classifier [2] (accuracy), param_sums;
    grad(step) -> {name: float64 tensor} of the gradients train() clipped at that step, from per-tensor int16 fixed point;
    update() -> {name: float64 tensor} of parameter after two steps minus parameter before, stored as float16;
    tape(step) -> {'enc{j}': uint8 mask [NB, G * Cout', L], 'teacher': bool [T]} for MaskSource.use_tape."""

    def __init__(self, config, path=GOLDEN):
        z = np.load(path)
        meta = json.loads(bytes(z['meta']).decode())[config]
        self.loss_keys = meta['loss_keys']
        self.names = [n for n, _ in meta['params']]
        self.shapes = [tuple(s) for _, s in meta['params']]
        self.mask_shapes = [tuple(s) for s in meta['masks']]
        self.losses, self.gradient, self.classifier = z[f'{config}.losses'], z[f'{config}.gradient'], z[f'{config}.classifier']
        self.param_sums = z[f'{config}.param_sums']
        self._grad, self._scale = z[f'{config}.grad'], z[f'{config}.grad_scale']
        self._update, self._tape = z[f'{config}.update'], z[f'{config}.tape']
        self.T = 20

    def _split(self, flat, scales=None):
        out, pos = {}, 0
        for i, (name, shape) in enumerate(zip(self.names, self.shapes)):
            n = int(np.prod(shape))
            t = torch.from_numpy(flat[pos:pos + n].astype(np.float64)).reshape(shape)
            out[name] = t * scales[i] if scales is not None else t
            pos += n
        assert pos == flat.size
        return out

    def grad(self, step):
        return self._split(self._grad[step], self._scale[step])

    def update(self):
        return self._split(self._update)

    def conditioned(self):
        """{name: bool mask} of the elements whose gradient at both steps is at least 1 % of its tensor's largest.  Adam's second
        step divides a mix of the two gradients by their root mean square, so where an element's gradients are tiny its change
        follows their rounding, not the arithmetic: there neither the int16 record nor another fp32 run pins the update."""
        g0, g1 = self.grad(0), self.grad(1)
        return {n: (g0[n].abs() >= 1e-2 * g0[n].abs().max()) & (g1[n].abs() >= 1e-2 * g1[n].abs().max()) for n in self.names}

    def tape(self, step):
        tape, pos = {'teacher': torch.ones(self.T, dtype=torch.bool)}, 0
        for j, shape in enumerate(self.mask_shapes):
            n = int(np.prod(shape))
            tape[f'enc{j}'] = torch.from_numpy(self._tape[step, pos:pos + n].copy()).reshape(shape)
            pos += n
        assert pos == self._tape.shape[1]
        return tape
