"""Time the audio analysis: utils.audio.spectrogram_batch (waveform -> log (mel) spectrogram) and mel_cepstral_distortion_batch.

    python tools/time_audio_analysis.py [--seconds 10] [--batches 1,16,64] [--pairs 64] [--rounds 5]

Inputs are CUDA tensors, so the figures are the library calls plus the packing the public functions do on the device; no host copies.
Arms alternate within each round; the figures are medians with their spread over the rounds.  Per-kernel times come from the library's
kernel timers in a separate call.  The card's name and power limit are read in the same run."""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def card():
    try:
        q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'], capture_output=True, text=True)
        return q.stdout.strip().splitlines()[0]
    except (OSError, IndexError):
        return torch.cuda.get_device_name(0) + ', power limit unknown'


def timed(fn, rounds_of, arms):
    """Median and spread (ms) per arm, arms alternating within each round."""
    for arm in arms:
        fn(arm)
    torch.cuda.synchronize()
    times = {arm: [] for arm in arms}
    for _ in range(rounds_of):
        for arm in arms:
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            fn(arm)
            e1.record()
            torch.cuda.synchronize()
            times[arm].append(e0.elapsed_time(e1))
    return {arm: (statistics.median(t), max(t) - min(t)) for arm, t in times.items()}


def kernel_ms(_lib, fn, arm):
    _lib.kernel_timing(True)
    fn(arm)
    torch.cuda.synchronize()
    out = {k: round(v[0], 3) for k, v in _lib.kernel_timing_read().items()}
    _lib.kernel_timing(False)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--seconds', type=float, default=10.0)
    ap.add_argument('--batches', default='1,16,64')
    ap.add_argument('--pairs', type=int, default=64)
    ap.add_argument('--rounds', type=int, default=5)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('time_audio_analysis needs a CUDA device')
    from multilingual_text_to_speech_b200 import _lib, configs
    from multilingual_text_to_speech_b200.utils import audio
    hp = configs.apply('ljspeech')
    dev = torch.device('cuda:0')
    gen = torch.Generator(device=dev)
    gen.manual_seed(0)
    sr = hp.sample_rate
    batches = [int(b) for b in a.batches.split(',')]
    # waveforms of about --seconds each (lengths spread by +-5 %), harmonic-like content does not change the work
    lens = torch.randint(int(0.95 * a.seconds * sr), int(1.05 * a.seconds * sr), (max(batches),), generator=gen, device=dev).tolist()
    waves = [torch.randn(n, device=dev, generator=gen) * 0.1 for n in lens]
    result = {'card': card(), 'seconds_per_waveform': a.seconds, 'spectrogram_batch': {}, 'mcd': {}}

    arms = [(B, mel) for B in batches for mel in (True, False)]
    spec = lambda arm: audio.spectrogram_batch(waves[:arm[0]], mel=arm[1])
    t = timed(spec, a.rounds, arms)
    for B, mel in arms:
        ms, spread = t[(B, mel)]
        audio_s = sum(lens[:B]) / sr
        result['spectrogram_batch'][f'{B} {"mel" if mel else "linear"}'] = {
            'ms': round(ms, 3), 'spread_ms': round(spread, 3), 'audio_s_per_s': round(audio_s / (ms / 1e3), 1),
            'kernel_ms': kernel_ms(_lib, spec, (B, mel))}

    # MCD: pairs of about 900 x 1000 frames of log-mel spectrograms
    fa = torch.randint(860, 941, (a.pairs,), generator=gen, device=dev).tolist()
    fb = torch.randint(960, 1041, (a.pairs,), generator=gen, device=dev).tolist()
    S1 = [torch.randn(hp.num_mels, f, device=dev, generator=gen) * 15 - 40 for f in fa]
    S2 = [torch.randn(hp.num_mels, f, device=dev, generator=gen) * 15 - 40 for f in fb]
    mcd = lambda mode: audio.mel_cepstral_distortion_batch(S1, S2, mode)
    t = timed(mcd, a.rounds, ['dtw', 'cut'])
    for mode in ('dtw', 'cut'):
        ms, spread = t[mode]
        cells = sum(x * y for x, y in zip(fa, fb)) if mode == 'dtw' else sum(min(x, y) for x, y in zip(fa, fb))
        result['mcd'][mode] = {'pairs': a.pairs, 'ms': round(ms, 3), 'spread_ms': round(spread, 3),
                               'frame_pairs_per_s': round(cells / (ms / 1e3)), 'kernel_ms': kernel_ms(_lib, mcd, mode)}
    print(json.dumps(result))


if __name__ == '__main__':
    main()
