"""Time WaveRNN training: one full step (forward + loss + backward + FusedAdam with clip 4) at the reference's dimensions with random
weights, against the same model and inputs as plain torch eager (cuDNN GRU, torch.optim.Adam) alternated in the same process.

    python tools/time_wavernn_train.py [--configs 32x1375,64x2750] [--modes RAW,MOL] [--precisions fp32,bf16] [--rounds 5]

Per-kernel times of the GRU loops come from the library's kernel timers in a separate step; the per-step loop latency is a loop's time
over its T steps.  The run also trains one step end to end on ground-truth-aligned mels from teacher-forced Tacotron.forward in eval mode
(random weights) through vocoder_batch.  The card's name and power limit are read in the same run."""
import argparse
import copy
import json
import os
import statistics
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tests'))

DIMS = dict(rnn_dims=512, fc_dims=512, bits=9, pad=2, upsample_factors=(5, 5, 11), feat_dims=80, compute_dims=128, res_out_dims=128,
            res_blocks=10, hop_length=275, sample_rate=22050)


def card():
    try:
        q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'], capture_output=True, text=True)
        return q.stdout.strip().splitlines()[0]
    except (OSError, IndexError):
        return torch.cuda.get_device_name(0) + ', power limit unknown'


def batch(mode, B, T, dev, seed=0):
    from multilingual_text_to_speech_b200.modules.wavernn import label_2_float
    g = torch.Generator().manual_seed(seed)
    mels = torch.randn(B, 80, T // 275 + 4, generator=g)
    if mode == 'RAW':
        lab = torch.randint(0, 512, (B, T + 1), generator=g)
        return label_2_float(lab[:, :T], 9).to(dev), lab[:, 1:].to(dev), mels.to(dev)
    lab = torch.randint(0, 65536, (B, T + 1), generator=g)
    return label_2_float(lab[:, :T], 16).to(dev), label_2_float(lab[:, 1:], 16).to(dev), mels.to(dev)


class Library:
    """The library path: FlatParams + GradBucket + FusedAdam around WaveRNN.forward and wavernn_loss."""

    def __init__(self, model):
        from multilingual_text_to_speech_b200.distributed import GradBucket
        from multilingual_text_to_speech_b200.optim import FlatParams, FusedAdam
        self.m = model
        self.bucket = GradBucket(model)
        self.opt = FusedAdam(FlatParams(model), self.bucket, lr=1e-4, max_grad_norm=4.0)

    def step(self, x, y, mels, mode):
        from multilingual_text_to_speech_b200.modules.wavernn import wavernn_loss
        self.bucket.zero()
        wavernn_loss(self.m(x, mels), y, mode).backward()
        self.opt.step()


class Eager:
    """Plain torch fp32 on the same GPU: the oracle's forward over nn modules (cuDNN GRU), torch losses, clip_grad_norm_ and Adam."""

    def __init__(self, model):
        self.m = copy.deepcopy(model)
        self.opt = torch.optim.Adam(self.m.parameters(), lr=1e-4)

    def step(self, x, y, mels, mode):
        import wavernn_train_oracle as TO
        self.opt.zero_grad(set_to_none=True)
        TO.loss(TO.forward(self.m, x, mels), y, mode).backward()
        torch.nn.utils.clip_grad_norm_(self.m.parameters(), 4.0)
        self.opt.step()


def timed(arms, rounds):
    for f in arms.values():
        f()
    torch.cuda.synchronize()
    times = {k: [] for k in arms}
    for _ in range(rounds):
        for k, f in arms.items():
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            f()
            e1.record()
            torch.cuda.synchronize()
            times[k].append(e0.elapsed_time(e1))
    return {k: (statistics.median(t), max(t) - min(t)) for k, t in times.items()}


def end_to_end(dev):
    """GTA mels (teacher-forced Tacotron.forward, eval mode, random weights) -> vocoder_batch -> one training step."""
    from multilingual_text_to_speech_b200 import configs
    from multilingual_text_to_speech_b200.modules.tacotron2 import Tacotron
    from multilingual_text_to_speech_b200.modules.wavernn import WaveRNN, draw_offsets, vocoder_batch, wavernn_loss
    hp = configs.apply('ljspeech')
    torch.manual_seed(0)
    taco = Tacotron().to(dev).eval()
    rng = np.random.default_rng(0)
    B, L, F = 4, 40, 48
    text = torch.from_numpy(rng.integers(1, hp.symbols_count() + 3, size=(B, L))).to(dev)
    target = torch.randn(B, hp.num_mels, F, device=dev)
    lengths = torch.full((B,), L, dtype=torch.long, device=dev)
    tl = torch.full((B,), F, dtype=torch.long, device=dev)
    with torch.no_grad():
        gta = taco(text, lengths, target, tl, None, None, teacher_forcing_ratio=1.0)[0]
    mels = [g.cpu().numpy() for g in gta]
    labels = [rng.integers(0, 512, F * 275) for _ in range(B)]
    offsets = draw_offsets([F] * B, 1375, 275, 2, rng)
    x, y, m = vocoder_batch(mels, labels, offsets, 'RAW', 9, 1375, 2, 275)
    voc = WaveRNN(**DIMS).to(dev).train()
    loss = wavernn_loss(voc(x.to(dev), m.to(dev)), y.to(dev), 'RAW')
    loss.backward()
    return {'gta_mels': [list(g.shape) for g in gta], 'window': list(m.shape), 'loss': float(loss.detach()),
            'all_gradients_finite': all(bool(torch.isfinite(p.grad).all()) for p in voc.parameters())}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--configs', default='32x1375,64x2750')
    ap.add_argument('--modes', default='RAW,MOL')
    ap.add_argument('--precisions', default='fp32,bf16')
    ap.add_argument('--rounds', type=int, default=5)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('time_wavernn_train needs a CUDA device')
    from multilingual_text_to_speech_b200 import _lib
    from multilingual_text_to_speech_b200.modules.wavernn import WaveRNN
    dev = torch.device('cuda:0')
    torch.backends.cudnn.benchmark = True
    result = {'card': card(), 'steps': {}}
    for cfg in a.configs.split(','):
        B, T = (int(v) for v in cfg.split('x'))
        for mode in a.modes.split(','):
            torch.manual_seed(0)
            base = WaveRNN(**DIMS, mode=mode).to(dev).train()
            lib, eager = Library(copy.deepcopy(base)), Eager(base)
            x, y, mels = batch(mode, B, T, dev)
            for prec in a.precisions.split(','):
                _lib.set_precision(prec)
                t = timed({'library': lambda: lib.step(x, y, mels, mode), 'torch_eager': lambda: eager.step(x, y, mels, mode)}, a.rounds)
                _lib.kernel_timing(True)
                lib.step(x, y, mels, mode)
                torch.cuda.synchronize()
                kernels = {k: (round(v[0], 3), v[1]) for k, v in _lib.kernel_timing_read().items()}
                _lib.kernel_timing(False)
                loops = {k: {'ms': kernels[k][0], 'launches': kernels[k][1], 'us_per_step': round(1e3 * kernels[k][0] / kernels[k][1] / T, 3)}
                         for k in ('gru_seq_fwd', 'gru_seq_bwd') if k in kernels}
                result['steps'][f'B={B} T={T} {mode} {prec}'] = {
                    'library_ms': round(t['library'][0], 2), 'library_spread_ms': round(t['library'][1], 2),
                    'torch_eager_ms': round(t['torch_eager'][0], 2), 'torch_eager_spread_ms': round(t['torch_eager'][1], 2),
                    'gru_loops': loops, 'kernel_ms': {k: v[0] for k, v in kernels.items()}}
            _lib.set_precision('fp32')
            del lib, eager, base
            torch.cuda.empty_cache()
    result['gta_to_training_step'] = end_to_end(dev)
    print(json.dumps(result))


if __name__ == '__main__':
    main()
