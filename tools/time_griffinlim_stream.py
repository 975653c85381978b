"""Time streaming Griffin-Lim (modules/griffinlim.py: GriffinLimVocoder.stream_pool, b200tts_gl_stream_run) on N concurrent streams of
900-frame log-mel spectrograms fed in chunks, against batch Griffin-Lim (utils.audio.inverse_spectrogram_batch) of the same spectrograms.

    python tools/time_griffinlim_stream.py [--frames 900] [--streams 1,16,64] [--chunks 32,64] [--iters 32,16] [--rounds 3] [--out FILE]

The spectrograms are utils.audio.spectrogram_batch of harmonic test signals (a different fundamental per stream).  Every arm feeds each
stream `chunk` frames per call, as a decoder would, then makes one pool.run() and synchronises.  Every arm runs once untimed before the
timed rounds.  Reported per arm, medians over rounds with the [min, max] over rounds in `spread`:
  * rtf worst / median: per stream, wall time to its last chunk over its audio duration (below 1: faster than real time);
  * first audio: wall time to a stream's first chunk (worst over streams); gap: the largest wall time between two chunks of a stream;
  * us per frame: the gl_stream_run kernel time over the frames each stream commits (the streams run side by side, one CTA each);
  * kernels: b200tts_kernel_timing totals per name (gl_stream_run, gl_stream_reset, vocoder_magnitude) in ms per round.
The batch arm (hp.griffin_lim_iters iterations over the whole spectrograms) alternates with the streaming arms round by round.  Wall times
are host clocks that end in torch.cuda.synchronize().  The card's name and power limit are read in the same run."""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def card():
    try:
        q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'], capture_output=True,
                           text=True, timeout=30)
        return q.stdout.strip().splitlines()[0]
    except Exception:                  # noqa: BLE001
        return torch.cuda.get_device_name(0) + ', power limit unknown'


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--frames', type=int, default=900)
    ap.add_argument('--streams', default='1,16,64')
    ap.add_argument('--chunks', default='32,64')
    ap.add_argument('--iters', default='32,16')
    ap.add_argument('--rounds', type=int, default=3)
    ap.add_argument('--out', default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('time_griffinlim_stream: no CUDA device')
    import __graft_entry__ as entry
    entry.build()
    from multilingual_text_to_speech_b200 import _lib
    from multilingual_text_to_speech_b200.modules.griffinlim import GriffinLimVocoder
    from multilingual_text_to_speech_b200.params.params import Params as hp
    from multilingual_text_to_speech_b200.utils import audio
    hp.reset()
    hop, sr = audio.ms_to_frames(hp.stft_shift_ms), hp.sample_rate
    nmax = max(int(s) for s in a.streams.split(','))
    t = np.arange(hop * (a.frames - 1)) / sr
    waves = [sum(np.sin(2 * np.pi * (90 + 7 * i) * k * t * (1 + 0.03 * t)) / k for k in range(1, 20)).astype(np.float32) for i in range(nmax)]
    mels = [m.cuda() for m in audio.spectrogram_batch([torch.from_numpy(w) for w in waves], mel=True)]
    assert all(m.shape[1] == a.frames for m in mels)
    dur = hop * (a.frames - 1) / sr
    info = card()
    print(f'card: {info}', flush=True)

    def stream_arm(voc, n, chunk):
        pool = voc.stream_pool(n, preemphasis=hp.preemphasis)
        sids = [pool.open() for _ in range(n)]
        stamps = {s: [] for s in sids}
        _lib.kernel_timing(True)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for f0 in range(0, a.frames, chunk):
            for i, s in enumerate(sids):
                pool.feed(s, mels[i][:, f0:f0 + chunk])
                if f0 + chunk >= a.frames:
                    pool.end(s)
            out = pool.run()
            torch.cuda.synchronize()
            now = time.perf_counter() - t0
            for s in out:
                stamps[s].append(now)
        kern = _lib.kernel_timing_read()
        _lib.kernel_timing(False)
        rtf = [stamps[s][-1] / dur for s in sids]
        gaps = [max(np.diff([0.0] + stamps[s])) for s in sids]
        return dict(rtf_worst=max(rtf), rtf_median=statistics.median(rtf), first_audio_s=max(stamps[s][0] for s in sids),
                    gap_worst_s=max(gaps), us_per_frame=1e3 * kern.get('gl_stream_run', (0, 0))[0] / a.frames,
                    kernels_ms={k: round(v[0], 3) for k, v in kern.items()})

    def batch_arm(n):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        audio.inverse_spectrogram_batch(mels[:n], mel=True)
        torch.cuda.synchronize()
        return dict(wall_s=time.perf_counter() - t0, rtf=(time.perf_counter() - t0) / dur)

    arms = [(n, c, it) for n in map(int, a.streams.split(',')) for c in map(int, a.chunks.split(',')) for it in map(int, a.iters.split(','))]
    vocs = {it: GriffinLimVocoder(True, 3, it) for it in map(int, a.iters.split(','))}
    for n, c, it in arms:                       # warm-up of every shape: tables, allocator, mel tables
        stream_arm(vocs[it], n, c)
    for n in sorted({x[0] for x in arms}):
        batch_arm(n)
    res = {}
    for r in range(a.rounds):
        for n, c, it in arms:
            res.setdefault(('stream', n, c, it), []).append(stream_arm(vocs[it], n, c))
        for n in sorted({x[0] for x in arms}):
            res.setdefault(('batch', n), []).append(batch_arm(n))
    lines = []
    for key, rows in res.items():
        med = {k: statistics.median(r[k] for r in rows) for k in rows[0] if k != 'kernels_ms'}
        med['spread'] = {k: [min(r[k] for r in rows), max(r[k] for r in rows)] for k in rows[0] if k != 'kernels_ms'}
        if 'kernels_ms' in rows[0]:
            med['kernels_ms'] = rows[-1]['kernels_ms']
        rec = dict(arm=key[0], streams=key[1], frames=a.frames, card=info, **({'chunk': key[2], 'iters': key[3]} if key[0] == 'stream' else
                                                                             {'iters': hp.griffin_lim_iters}), **med)
        lines.append(json.dumps(rec))
        print(lines[-1], flush=True)
    if a.out:
        with open(a.out, 'w') as f:
            f.write('\n'.join(lines) + '\n')


if __name__ == '__main__':
    main()
