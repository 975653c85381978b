"""Time forced alignment on the GPU: Tacotron.align on a batch of utterances (eval forward at teacher forcing 1.0, then the monotonic
alignment search and the scores) and the search alone against the fp64 numpy oracle on the host.

The model is generated_training's configuration (10 languages, generated encoder) with seeded random weights; the batch is --batch
utterances of --symbols symbols and --frames target frames, languages b % 10.  Every arm runs once untimed, then --rounds timed rounds,
each a host clock ending in torch.cuda.synchronize(); kernel times come from the library's named CUDA-event timers in a separate pass.
The card's name and power limit are read in the same run.  One JSON line on stdout, and the same under --out.

    python tools/time_align.py [--batch 64 --symbols 180 --frames 900 --rounds 5 --out time_align.json]
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


def rounds(fn, n):
    fn()
    torch.cuda.synchronize()
    out = []
    for _ in range(n):
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        out.append(time.perf_counter() - t0)
    return out


def summary(ts, batch):
    med = statistics.median(ts)
    return {'median_ms': med * 1e3, 'min_ms': min(ts) * 1e3, 'max_ms': max(ts) * 1e3, 'utterances_per_s': batch / med}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--batch', type=int, default=64)
    ap.add_argument('--symbols', type=int, default=180)
    ap.add_argument('--frames', type=int, default=900)
    ap.add_argument('--rounds', type=int, default=5)
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    import __graft_entry__ as entry
    entry.build()
    import align_oracle as A
    from multilingual_text_to_speech_b200 import _lib, configs, functional as F
    from multilingual_text_to_speech_b200.modules.tacotron2 import Tacotron
    from multilingual_text_to_speech_b200.rng import MaskSource
    if not torch.cuda.is_available():
        raise SystemExit('time_align.py measures the GPU: no CUDA device')
    dev = torch.device('cuda:0')
    hp = configs.apply('generated_training')
    torch.manual_seed(0)
    model = Tacotron().to(dev).eval()
    B, L, T = args.batch, args.symbols, args.frames
    g = torch.Generator().manual_seed(1)
    text = torch.randint(1, hp.symbols_count(), (B, L), generator=g).to(dev)
    text_length = torch.full((B,), L, dtype=torch.long, device=dev)
    target = torch.randn(B, hp.num_mels, T, generator=g).to(dev)
    target_length = torch.full((B,), T, dtype=torch.long, device=dev)
    languages = (torch.arange(B) % hp.language_number).to(dev)
    result = {'card': card(), 'batch': B, 'symbols': L, 'frames': T, 'rounds': args.rounds, 'config': 'generated_training'}

    for precision in ('fp32', 'bf16'):
        _lib.set_precision(precision)
        MaskSource.manual_seed(0)
        align = lambda: model.align(text, text_length, target, target_length, None, languages)       # noqa: E731
        forward = lambda: model(text, text_length, target, target_length, None, languages, 1.0)     # noqa: E731
        with torch.no_grad():
            result[f'align_{precision}'] = summary(rounds(align, args.rounds), B)
            result[f'eval_forward_{precision}'] = summary(rounds(forward, args.rounds), B)
    _lib.set_precision('fp32')

    weights = model.align(text, text_length, target, target_length, None, languages).alignment
    tl, sl = [L] * B, [T] * B
    search = lambda: F.monotonic_alignment(weights, tl, sl)        # noqa: E731
    scores = lambda: F.alignment_scores(weights, tl, sl)            # noqa: E731
    result['search'] = summary(rounds(search, args.rounds), B)
    result['scores'] = summary(rounds(scores, args.rounds), B)
    _lib.kernel_timing(True)
    for _ in range(args.rounds):
        search()
        scores()
    torch.cuda.synchronize()
    kt = _lib.kernel_timing_read()
    _lib.kernel_timing(False)
    result['kernel_ms'] = {k: v[0] / v[1] for k, v in kt.items() if k in ('monotonic_alignment', 'alignment_scores')}

    P = weights.cpu().numpy()
    t0 = time.perf_counter()
    want_d, want_v, _ = A.mas_batch(P, tl, sl)
    host = time.perf_counter() - t0
    got_d, got_v = search()
    result['numpy_oracle'] = {'ms': host * 1e3, 'utterances_per_s': B / host}
    result['durations_equal_oracle'] = bool(np.array_equal(got_d.cpu().numpy(), want_d))
    result['path_logp_max_rel'] = float(np.max(np.abs(got_v.cpu().numpy() - want_v) / np.abs(want_v)))
    line = json.dumps(result)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, 'w') as f:
            f.write(line + '\n')


if __name__ == '__main__':
    main()
