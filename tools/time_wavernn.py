"""Time the WaveRNN vocoder: WaveRNN.generate_batch (mel -> waveform) at the reference's dimensions with random weights.

    python tools/time_wavernn.py [--frames 900] [--batches 1,16,64] [--modes RAW,MOL] [--rounds 3] [--target 11000] [--overlap 550]

Each batch holds mels of --frames frames (900 frames are about 11 s at hop 275 / 22,050 Hz: 22 folds of 12,100 steps at target 11,000 /
overlap 550).  Inputs are CUDA tensors.  Arms alternate within each round; the figures are medians with their spread over the rounds.
Per-kernel times come from the library's kernel timers in a separate call.  The run also turns Tacotron.inference_batch output (random
weights, default config) into waveforms end to end.  The card's name and power limit are read in the same run."""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

DIMS = dict(rnn_dims=512, fc_dims=512, bits=9, pad=2, upsample_factors=(5, 5, 11), feat_dims=80, compute_dims=128, res_out_dims=128,
            res_blocks=10, hop_length=275, sample_rate=22050)


def card():
    try:
        q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'], capture_output=True, text=True)
        return q.stdout.strip().splitlines()[0]
    except (OSError, IndexError):
        return torch.cuda.get_device_name(0) + ', power limit unknown'


def timed(fn, rounds, arms):
    for arm in arms:
        fn(arm)
    torch.cuda.synchronize()
    times = {arm: [] for arm in arms}
    for _ in range(rounds):
        for arm in arms:
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            fn(arm)
            e1.record()
            torch.cuda.synchronize()
            times[arm].append(e0.elapsed_time(e1))
    return {arm: (statistics.median(t), max(t) - min(t)) for arm, t in times.items()}


def end_to_end(models, dev):
    """Tacotron.inference_batch (random weights, 3 texts, 60 frames) -> generate_batch on the GPU."""
    import numpy as np
    from multilingual_text_to_speech_b200 import configs
    from multilingual_text_to_speech_b200.modules.tacotron2 import Tacotron
    hp = configs.apply('ljspeech', max_output_length=60)
    torch.manual_seed(0)
    taco = Tacotron().to(dev).eval()
    with torch.no_grad():
        taco._decoder._stop_prediction.bias.fill_(-100.0)
    rng = np.random.default_rng(0)
    texts = [torch.from_numpy(rng.integers(1, hp.symbols_count() + 3, size=n)).to(dev) for n in (30, 45, 60)]
    with torch.no_grad():
        mels = taco.inference_batch(texts, None, None)
    out = {}
    for mode, m in models.items():
        waves = m.generate_batch([s[:hp.num_mels] for s in mels], generator=torch.Generator(device=dev).manual_seed(0))
        out[mode] = {'mel_frames': [int(s.shape[-1]) for s in mels], 'samples': [int(w.shape[0]) for w in waves],
                     'on_gpu': all(w.is_cuda for w in waves), 'finite': all(bool(torch.isfinite(w).all()) for w in waves)}
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--frames', type=int, default=900)
    ap.add_argument('--batches', default='1,16,64')
    ap.add_argument('--modes', default='RAW,MOL')
    ap.add_argument('--rounds', type=int, default=3)
    ap.add_argument('--target', type=int, default=11000)
    ap.add_argument('--overlap', type=int, default=550)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('time_wavernn needs a CUDA device')
    from multilingual_text_to_speech_b200 import _lib
    from multilingual_text_to_speech_b200.modules.wavernn import WaveRNN
    _lib.set_precision('fp32')
    dev = torch.device('cuda:0')
    torch.manual_seed(0)
    models = {mode: WaveRNN(**DIMS, mode=mode).to(dev).eval() for mode in a.modes.split(',')}
    batches = [int(b) for b in a.batches.split(',')]
    gen = torch.Generator(device=dev).manual_seed(0)
    mels = [torch.randn(80, a.frames, device=dev, generator=gen) for _ in range(max(batches))]
    result = {'card': card(), 'frames': a.frames, 'target': a.target, 'overlap': a.overlap, 'generate_batch': {}}
    arms = [(B, mode) for B in batches for mode in models]
    call = lambda arm: models[arm[1]].generate_batch(mels[:arm[0]], a.target, a.overlap, generator=gen)
    t = timed(call, a.rounds, arms)
    for B, mode in arms:
        ms, spread = t[(B, mode)]
        audio_s = B * (a.frames - 1) * DIMS['hop_length'] / DIMS['sample_rate']
        _lib.kernel_timing(True)
        call((B, mode))
        torch.cuda.synchronize()
        kernels = {k: round(v[0], 3) for k, v in _lib.kernel_timing_read().items()}
        _lib.kernel_timing(False)
        folds = models[mode].tape_shape(a.frames, a.target, a.overlap)[0]
        result['generate_batch'][f'{B} {mode}'] = {'ms': round(ms, 2), 'spread_ms': round(spread, 2), 'fold_rows': B * folds,
                                                   'audio_s_per_s': round(audio_s / (ms / 1e3), 2), 'kernel_ms': kernels}
    result['tacotron_to_waveform'] = end_to_end(models, dev)
    print(json.dumps(result))


if __name__ == '__main__':
    main()
