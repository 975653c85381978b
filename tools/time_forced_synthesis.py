"""Cost of forced synthesis (durations=): a free decode against a forced one of the same length and a decode with the window [1, 3],
random weights, seeded texts.

Every utterance decodes --frames frames.  The free and windowed arms have the stop bias at -100 and every stop logit
F.decoder_forward_chunk returns rewritten to -10 (the stop-disable of tools/time_batch_synthesis.py); the forced arm gives every text one
symbol per frame run (durations_to_alignment of an even split of --frames frames), so its one-hot rows decode the same number of steps.
Workloads:
  inference_batch  --n texts of 20 to 200 characters at max_batch 1 (only the first --single-n texts), 16 and 64 (every row forced:
                   only the forced attention step runs);
  pool             DecoderPool.run() until idle with 8 texts open from the first call, every other one forced (mixed chunks: the
                   computed step runs over every row, then the forced step over the forced rows).
The arms alternate round by round; the tool prints medians and spreads of mel frames/s and the card name and power limit read in the
same run.
    python tools/time_forced_synthesis.py --config generated_switching
"""
import argparse
import json
import os
import statistics
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from tools.time_batch_synthesis import card     # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--config', default='generated_switching')
    ap.add_argument('--n', type=int, default=64)
    ap.add_argument('--single-n', type=int, default=4)
    ap.add_argument('--frames', type=int, default=900)
    ap.add_argument('--precision', default='bf16')
    ap.add_argument('--rounds', type=int, default=3)
    a = ap.parse_args()
    from multilingual_text_to_speech_b200 import configs, _lib
    from multilingual_text_to_speech_b200 import functional as F
    hp = configs.apply(a.config, max_output_length=a.frames)
    _lib.set_precision(a.precision)
    dev = torch.device('cuda:0')
    torch.manual_seed(0)
    from multilingual_text_to_speech_b200.modules.tacotron2 import Tacotron
    model = Tacotron().to(dev).eval()
    with torch.no_grad():
        model._decoder._stop_prediction.bias.fill_(-100.0)
    rng = np.random.default_rng(0)
    lens = rng.integers(20, 201, size=a.n)
    texts = [torch.from_numpy(rng.integers(1, hp.symbols_count() + 3, size=int(L))).to(dev) for L in lens]
    G = hp.language_number if hp.multi_language else 0
    languages = None
    if G:
        languages = []
        for L in lens:
            w = torch.zeros(1, int(L), G, device=dev)
            w[0, :, int(rng.integers(G))] = 1.0
            languages.append(w)
    speakers = [torch.zeros(1, dtype=torch.long, device=dev) for _ in lens] if hp.multi_speaker else None
    pick = lambda seq, idx: None if seq is None else [seq[i] for i in idx]     # noqa: E731

    orig = F.decoder_forward_chunk

    def chunk(*args, **kw):
        spec, stop, align = orig(*args, **kw)
        return spec, torch.full_like(stop, -10.0), align
    F.decoder_forward_chunk = chunk

    def even(L):        # --frames frames split over L symbols as evenly as whole frames allow
        return torch.from_numpy(np.diff(np.floor(np.arange(L + 1) * a.frames / L).astype(np.int64)))
    durations = [even(int(L)) for L in lens]

    def batch(mb, forced):
        idx = range(a.single_n) if mb == 1 else range(a.n)
        outs = model.inference_batch(pick(texts, idx), pick(speakers, idx), pick(languages, idx), max_batch=mb,
                                     durations=pick(durations, idx) if forced else None)
        return sum(o.shape[-1] for o in outs)

    def pool(k, forced):
        p = model.decoder_pool(k)
        for i in range(k):
            p.open(texts[i], None if speakers is None else speakers[i], None if languages is None else languages[i],
                   durations=durations[i] if forced and i % 2 == 0 else None)
        frames = 0
        while p.ids:
            frames += sum(c.shape[-1] for c in p.run().values())
        return frames

    work = {f'inference_batch max_batch {mb}': (lambda forced, mb=mb: batch(mb, forced)) for mb in (1, 16, 64)}
    work['pool 8 texts, 4 forced'] = lambda forced: pool(8, forced)
    arms = {'free': (None, False), 'forced': (None, True), 'window [1, 3]': ([1, 3], False)}

    def timed(fn, arm):
        hp.inference_attention_window, forced = arm
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        with torch.no_grad():
            frames = fn(forced)
        torch.cuda.synchronize()
        return frames, time.perf_counter() - t0

    report = {'card': card(), 'config': a.config, 'precision': a.precision, 'frames': a.frames, 'n': a.n, 'single_n': a.single_n,
              'workloads': {}}
    for name, fn in work.items():
        for arm in arms.values():               # warm-up of every shape the timed window uses
            timed(fn, arm)
        res = {name: [] for name in arms}
        frames_of = {}
        for _ in range(a.rounds):
            for arm_name, arm in arms.items():
                frames, dt = timed(fn, arm)
                frames_of[arm_name] = frames
                res[arm_name].append(frames / dt)
        out = {arm: {'frames_per_s': statistics.median(r), 'spread': max(r) - min(r), 'frames': frames_of[arm]} for arm, r in res.items()}
        free = out['free']['frames_per_s']
        out['forced / free'] = out['forced']['frames_per_s'] / free
        out['window / free'] = out['window [1, 3]']['frames_per_s'] / free
        print(name, json.dumps(out), flush=True)
        report['workloads'][name] = out
    hp.inference_attention_window = None
    F.decoder_forward_chunk = orig
    print(json.dumps(report))


if __name__ == '__main__':
    main()
