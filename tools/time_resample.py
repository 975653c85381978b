"""Time the waveform front end on the GPU: utils.audio.resample_batch on 1, 16 and 64 waveforms of about --seconds seconds each for
48000 -> 22050, 16000 -> 22050 and 22050 -> 16000 Hz, and trim_silence_batch(ys, 50, 12.5, top_db=40) on 64 of them, with the inputs
already on the device.

Waveforms are the seeded harmonic glides of tools/time_pitch.py, generated at each source rate; the trimming inputs get 0.5 s of digital
silence at both ends.  Every arm runs once untimed, then --rounds timed rounds, each a pair of CUDA events around one call (the call ends
in its own device-to-host copies only for trimming, whose bounds come back to the host).  Kernel times come from the library's named
CUDA-event timers in a separate pass.  For resampling, achieved bytes count 4 (L + L') per waveform (each input and output sample once)
and achieved FP64 work counts one multiply-add per filter tap an output uses; each is set against the H100 SXM data sheet's 3.35 TB/s
and 34 TFLOP/s non-tensor FP64 (17 T multiply-adds/s).  scipy.signal.resample_poly on the host, on the same batch, is a context line.
The card's name, power limit and max SM clock are read in the same run.  One JSON line on stdout, and the same under --out.

    python tools/time_resample.py [--seconds 10 --rounds 10 --scipy-waveforms 4 --out time_resample.json]
"""
import argparse
import json
import math
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

HBM_BYTES_PER_S = 3.35e12
FP64_FMA_PER_S = 34e12 / 2
PAIRS = ((48000, 22050), (16000, 22050), (22050, 16000))


def taps_used(L, up, down):
    """Filter taps summed over all L' outputs: output n uses the h indices h_len + n down - k up in [0, 2 h_len] with k in [0, L)."""
    m = max(up, down)
    h_len = 10 * m
    n = np.arange(-(-L * up // down), dtype=np.int64)
    t = h_len + n * down
    hi = np.minimum(t // up, L - 1)
    lo = np.maximum(-(-(t - 2 * h_len) // up), 0)
    return int(np.maximum(hi - lo + 1, 0).sum())


def timed(call, rounds):
    ts = []
    for _ in range(rounds):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        call()
        b.record()
        b.synchronize()
        ts.append(a.elapsed_time(b))
    return ts


def kernel_ms(call, rounds, prefix):
    from multilingual_text_to_speech_b200 import _lib
    _lib.kernel_timing(True)
    for _ in range(rounds):
        call()
    torch.cuda.synchronize()
    kt = _lib.kernel_timing_read()
    _lib.kernel_timing(False)
    return {k: v[0] / v[1] for k, v in kt.items() if k.startswith(prefix)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--seconds', type=float, default=10.0)
    ap.add_argument('--rounds', type=int, default=10)
    ap.add_argument('--scipy-waveforms', type=int, default=4, help='waveforms per batch timed through scipy, scaled to the batch')
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    import __graft_entry__ as entry
    entry.build()
    import scipy.signal
    from multilingual_text_to_speech_b200.utils import audio
    if not torch.cuda.is_available():
        raise SystemExit('time_resample.py measures the GPU: no CUDA device')
    result = {'card': card(), 'seconds': args.seconds, 'rounds': args.rounds}
    dev = torch.device('cuda:0')
    for src, dst in PAIRS:
        up, down = audio.resample_ratio(src, dst)
        for B in (1, 16, 64):
            host = waveforms(B, args.seconds, src, B)
            waves = [torch.from_numpy(w).to(dev) for w in host]
            call = lambda: audio.resample_batch(waves, src, dst)          # noqa: E731
            call()
            torch.cuda.synchronize()
            ts = timed(call, args.rounds)
            kms = kernel_ms(call, args.rounds, 'resample')
            L = sum(len(w) for w in host)
            Lp = sum(-(-len(w) * up // down) for w in host)
            fmas = sum(taps_used(len(w), up, down) for w in host)
            k = kms.get('resample', float('nan')) * 1e-3
            med = statistics.median(ts) * 1e-3
            n_sp = min(B, args.scipy_waveforms)
            t0 = time.perf_counter()
            for w in host[:n_sp]:
                scipy.signal.resample_poly(w, up, down)
            scipy_s = (time.perf_counter() - t0) * sum(len(w) for w in host) / sum(len(w) for w in host[:n_sp])
            row = {'ratio': f'{up}/{down}', 'audio_seconds': L / src, 'median_ms': med * 1e3, 'min_ms': min(ts), 'max_ms': max(ts),
                   'audio_seconds_per_s': L / src / med, 'kernel_ms': k * 1e3, 'bytes': 4 * (L + Lp), 'fp64_fma': fmas,
                   'achieved_TBps': 4 * (L + Lp) / k / 1e12, 'achieved_fp64_TFLOPs': 2 * fmas / k / 1e12,
                   'hbm_floor_us': 4 * (L + Lp) / HBM_BYTES_PER_S * 1e6, 'fp64_floor_us': fmas / FP64_FMA_PER_S * 1e6,
                   'scipy_host_ms': scipy_s * 1e3}
            key = f'resample_{src}_{dst}_B{B}'
            result[key] = row
            print(json.dumps({key: row}), file=sys.stderr)
    B, sr = 64, audio.hp.sample_rate
    host = [np.concatenate([np.zeros(sr // 2, np.float32), w, np.zeros(sr // 2, np.float32)]) for w in waveforms(B, args.seconds, sr, 5)]
    waves = [torch.from_numpy(w).to(dev) for w in host]
    call = lambda: audio.trim_silence_batch(waves, 50, 12.5, top_db=40)          # noqa: E731
    call()
    ts = timed(call, args.rounds)
    kms = kernel_ms(call, args.rounds, 'trim')
    L = sum(len(w) for w in host)
    med = statistics.median(ts) * 1e-3
    row = {'audio_seconds': L / sr, 'median_ms': med * 1e3, 'min_ms': min(ts), 'max_ms': max(ts), 'audio_seconds_per_s': L / sr / med,
           'kernel_ms': kms.get('trim_silence', float('nan')), 'hbm_floor_us': 4 * L / HBM_BYTES_PER_S * 1e6}
    result[f'trim_B{B}'] = row
    print(json.dumps({f'trim_B{B}': row}), file=sys.stderr)
    line = json.dumps(result)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, 'w') as f:
            f.write(line + '\n')


if __name__ == '__main__':
    main()
