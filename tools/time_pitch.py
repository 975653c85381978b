"""Time pitch analysis on the GPU: utils.audio.pitch_batch on 1, 16 and 64 waveforms of about --seconds seconds each, with the library's
per-stage kernel times, and the numpy oracle (tests/pitch_oracle.py) on the host for the same inputs.

Waveforms are seeded harmonic glides with noise, at hp.sample_rate.  Every arm runs once untimed, then --rounds timed rounds, each a host
clock ending in torch.cuda.synchronize(); kernel times come from the library's named CUDA-event timers in a separate pass.  The oracle is a
host-CPU figure, timed once per batch size on --oracle-utterances of the waveforms (it decodes 1,202 states densely per frame) and scaled
to the batch.  The card's name, power limit and clocks are read in the same run.  One JSON line on stdout, and the same under --out.

    python tools/time_pitch.py [--seconds 10 --rounds 5 --oracle-utterances 1 --out time_pitch.json]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tests'))


def card():
    try:
        q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'], capture_output=True,
                           text=True, timeout=30)
        return q.stdout.strip().splitlines()[0]
    except Exception:                  # noqa: BLE001
        return torch.cuda.get_device_name(0) + ', power limit unknown'


def waveforms(count, seconds, sr, seed):
    rng = np.random.default_rng(seed)
    out = []
    for _ in range(count):
        n = int(seconds * sr * rng.uniform(0.9, 1.1))
        t = np.arange(n) / sr
        f = rng.uniform(90, 250) * 2 ** (0.5 * np.sin(2 * np.pi * rng.uniform(0.2, 1.0) * t))
        phase = 2 * np.pi * np.cumsum(f) / sr
        y = 0.4 * np.sin(phase) + 0.2 * np.sin(2 * phase) + 0.1 * np.sin(3 * phase) + 0.01 * rng.standard_normal(n)
        out.append(y.astype(np.float32))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--seconds', type=float, default=10.0)
    ap.add_argument('--rounds', type=int, default=5)
    ap.add_argument('--oracle-utterances', type=int, default=1)
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    import __graft_entry__ as entry
    entry.build()
    import pitch_oracle as P
    from multilingual_text_to_speech_b200 import _lib
    from multilingual_text_to_speech_b200.params.params import Params as hp
    from multilingual_text_to_speech_b200.utils import audio
    if not torch.cuda.is_available():
        raise SystemExit('time_pitch.py measures the GPU: no CUDA device')
    sr, hop = hp.sample_rate, audio.ms_to_frames(hp.stft_shift_ms)
    result = {'card': card(), 'seconds': args.seconds, 'rounds': args.rounds, 'sample_rate': sr, 'hop': hop,
              'params': {'fmin': 65.406, 'fmax': 2093.0, 'frame_length': 1024}}
    dev = torch.device('cuda:0')
    for B in (1, 16, 64):
        waves = [torch.from_numpy(w).to(dev) for w in waveforms(B, args.seconds, sr, B)]
        audio_s = sum(len(w) for w in waves) / sr
        call = lambda: audio.pitch_batch(waves)            # noqa: E731
        call()
        torch.cuda.synchronize()
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
        row = {'audio_seconds': audio_s, 'frames': sum(1 + len(w) // hop for w in waves), 'median_ms': med * 1e3, 'min_ms': min(ts) * 1e3,
               'max_ms': max(ts) * 1e3, 'audio_seconds_per_s': audio_s / med,
               'kernel_ms': {k: v[0] / v[1] for k, v in kt.items() if k.startswith('pitch_')}}
        m = min(B, args.oracle_utterances)
        host = [w.cpu().numpy().astype(np.float64) for w in waves[:m]]
        t0 = time.perf_counter()
        for y in host:
            P.pyin(y, sr, hop)
        per = (time.perf_counter() - t0) / m
        row['host_cpu_numpy_oracle'] = {'utterances_timed': m, 'ms_per_utterance': per * 1e3, 'ms_for_batch_scaled': per * B * 1e3}
        got = audio.pitch_batch([waves[i] for i in range(m)])
        row['oracle_f0_equal'] = all(np.array_equal(g[0].cpu().numpy(), P.pyin(y, sr, hop)[0].astype(np.float32), equal_nan=True)
                                     for g, y in zip(got, host))
        result[f'B{B}'] = row
        print(json.dumps({f'B{B}': row}), file=sys.stderr)
    line = json.dumps(result)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, 'w') as f:
            f.write(line + '\n')


if __name__ == '__main__':
    main()
