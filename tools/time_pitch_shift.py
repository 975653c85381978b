"""Time pitch shifting on the GPU: utils.audio.pitch_shift_batch on 1, 16 and 64 waveforms of about --seconds seconds each, at +4 and -4
semitones, with the F0 tracks given (f0s=) and tracked by pitch_batch inside the call (f0s=None), with the library's per-kernel times.

Waveforms are seeded harmonic glides with noise, at hp.sample_rate.  Every arm runs once untimed, then --rounds timed rounds, each a host
clock ending in torch.cuda.synchronize(); kernel times come from the library's named CUDA-event timers in a separate pass.  The
overlap-add's achieved bandwidth is the bytes it must move (the waveform read once, the output written once, and each utterance's marks
read once: 4 + 4 + 17 bytes per sample plus 16 per utterance) over its kernel time; reads of the same samples by neighbouring threads are
not counted.  The card's name, power limit and max SM clock are read in the same run.  One JSON line on stdout, and the same under --out.

    python tools/time_pitch_shift.py [--seconds 10 --rounds 5 --out time_pitch_shift.json]
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--seconds', type=float, default=10.0)
    ap.add_argument('--rounds', type=int, default=5)
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    import __graft_entry__ as entry
    entry.build()
    from multilingual_text_to_speech_b200 import _lib
    from multilingual_text_to_speech_b200.params.params import Params as hp
    from multilingual_text_to_speech_b200.utils import audio
    if not torch.cuda.is_available():
        raise SystemExit('time_pitch_shift.py measures the GPU: no CUDA device')
    sr, hop = hp.sample_rate, audio.ms_to_frames(hp.stft_shift_ms)
    result = {'card': card(), 'seconds': args.seconds, 'rounds': args.rounds, 'sample_rate': sr, 'hop': hop}
    dev = torch.device('cuda:0')
    for B in (1, 16, 64):
        waves = [torch.from_numpy(w).to(dev) for w in waveforms(B, args.seconds, sr, B)]
        samples = sum(len(w) for w in waves)
        audio_s = samples / sr
        f0s = [f for f, _ in audio.pitch_batch(waves)]
        for semis in (4.0, -4.0):
            for given in (True, False):
                call = lambda: audio.pitch_shift_batch(waves, semitones=semis, f0s=f0s if given else None)   # noqa: E731
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
                kms = {k: v[0] / v[1] for k, v in kt.items() if k.startswith(('psola_', 'pitch_'))}
                row = {'audio_seconds': audio_s, 'median_ms': med * 1e3, 'min_ms': min(ts) * 1e3, 'max_ms': max(ts) * 1e3,
                       'audio_seconds_per_s': audio_s / med, 'kernel_ms': kms}
                if 'psola_overlap_add' in kms:
                    moved = samples * (4 + 4 + 17) + 16 * B
                    row['overlap_add_achieved_GBps'] = moved / (kms['psola_overlap_add'] * 1e-3) / 1e9
                key = f'B{B}_{semis:+g}st_{"f0_given" if given else "f0_tracked"}'
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
