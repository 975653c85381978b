"""Time time-scale modification on the GPU: utils.audio.time_stretch_batch on 1, 16 and 64 waveforms of about --seconds seconds each at
rates 0.8 and 1.25, and retime_batch from seeded durations d to scale_durations(d, 1.2), with the library's per-kernel times.

Waveforms are the seeded harmonic glides of tools/time_pitch.py, at hp.sample_rate; d splits each waveform's mel frames into symbols of
2 to 14 frames.  Every arm runs once untimed, then --rounds timed rounds, each a host clock ending in torch.cuda.synchronize(); kernel
times come from the library's named CUDA-event timers in a separate pass.  The search's achieved FP64 rate counts the 2 (2D + 1) 2H
multiply-adds of each frame after the first (C and E of every candidate) over its kernel time.  The card's name, power limit and max SM
clock are read in the same run.  One JSON line on stdout, and the same under --out.

    python tools/time_time_stretch.py [--seconds 10 --rounds 5 --out time_time_stretch.json]
"""
import argparse
import json
import os
import statistics
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tools'))

from time_pitch import card, waveforms          # noqa: E402


def durations(frames, rng):
    """A split of `frames` mel frames into symbols of 2 to 14 frames."""
    d = []
    while sum(d) < frames:
        d.append(int(rng.integers(2, 15)))
    d[-1] -= sum(d) - frames
    return np.array(d, dtype=np.int64)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--seconds', type=float, default=10.0)
    ap.add_argument('--rounds', type=int, default=5)
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    import __graft_entry__ as entry
    entry.build()
    from multilingual_text_to_speech_b200 import _lib
    from multilingual_text_to_speech_b200.functional import scale_durations
    from multilingual_text_to_speech_b200.params.params import Params as hp
    from multilingual_text_to_speech_b200.utils import audio
    if not torch.cuda.is_available():
        raise SystemExit('time_time_stretch.py measures the GPU: no CUDA device')
    sr, hop = hp.sample_rate, audio.ms_to_frames(hp.stft_shift_ms)
    result = {'card': card(), 'seconds': args.seconds, 'rounds': args.rounds, 'sample_rate': sr, 'hop': hop, 'tolerance': hop}
    dev = torch.device('cuda:0')
    for B in (1, 16, 64):
        waves = [torch.from_numpy(w).to(dev) for w in waveforms(B, args.seconds, sr, B)]
        audio_s = sum(len(w) for w in waves) / sr
        rng = np.random.default_rng(B)
        ds = [durations(1 + len(w) // hop, rng) for w in waves]
        new = [scale_durations(d, 1.2) for d in ds]
        arms = {'rate0.8': lambda: audio.time_stretch_batch(waves, 0.8),                   # noqa: E731
                'rate1.25': lambda: audio.time_stretch_batch(waves, 1.25),                 # noqa: E731
                'retime1.2': lambda: audio.retime_batch(waves, ds, new)}                    # noqa: E731
        for name, call in arms.items():
            outs = call()
            torch.cuda.synchronize()
            search_frames = sum((len(y) - 1) // hop + 1 for y in outs)                    # K - 1 per waveform
            ts = []
            for _ in range(args.rounds):
                t0 = time.perf_counter()
                call()
                torch.cuda.synchronize()
                ts.append(time.perf_counter() - t0)
            _lib.kernel_timing(True)
            for _ in range(args.rounds):
                call()
            torch.cuda.synchronize()
            kt = _lib.kernel_timing_read()
            _lib.kernel_timing(False)
            med = statistics.median(ts)
            kms = {k: v[0] / v[1] for k, v in kt.items() if k.startswith('wsola_')}
            row = {'audio_seconds': audio_s, 'median_ms': med * 1e3, 'min_ms': min(ts) * 1e3, 'max_ms': max(ts) * 1e3,
                   'audio_seconds_per_s': audio_s / med, 'kernel_ms': kms, 'search_frames': search_frames}
            if 'wsola_positions' in kms:
                fmas = search_frames * 2 * (2 * hop + 1) * 2 * hop
                row['search_fp64_TFLOPs'] = 2 * fmas / (kms['wsola_positions'] * 1e-3) / 1e12
            key = f'B{B}_{name}'
            result[key] = row
            print(json.dumps({key: row}), file=sys.stderr)
    line = json.dumps(result)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, 'w') as f:
            f.write(line + '\n')


if __name__ == '__main__':
    main()
