"""Eager training-step times at teacher forcing below 1.0 beside the teacher-forced step, on the benchmark workload (generated_training,
zoneout, B = 60, L = 180, T = 900, bf16 by default).

One step = Tacotron.forward + TacotronLoss + backward into the gradient bucket, ending in a device synchronise.  Steps with free-running
decoder steps run eagerly (GraphedTrainStep refuses them: the host-drawn coins decide the launch sequence), so every ratio is timed
eagerly here, including 1.0.  The ratios alternate round by round in one process so that all of them see the same card state; the coins
are fresh at every step (MaskSource), as in training.  Prints one JSON line with the card, its power limit and SM clock (read in the same
call), and per ratio the median and spread (max - min) of the per-round means, and the mean number of free-running steps per decode.

    python tools/time_teacher_forcing.py [--rounds 3] [--steps 3] [--warmup 1] [--ratios 1.0,0.9,0.5]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    q = 'name,power.limit,clocks.sm,clocks.max.sm'
    try:
        out = subprocess.run(['nvidia-smi', f'--query-gpu={q}', '--format=csv,noheader'], capture_output=True, text=True, timeout=30)
        return out.stdout.strip().splitlines()[0]
    except Exception as exc:        # noqa: BLE001 -- reported, not fatal
        return f'nvidia-smi unavailable: {exc!r}'


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--config', default='generated_training')
    ap.add_argument('--batch', type=int, default=60)
    ap.add_argument('--text-len', type=int, default=180)
    ap.add_argument('--frames', type=int, default=900)
    ap.add_argument('--precision', default='bf16', choices=['bf16', 'fp32'])
    ap.add_argument('--rounds', type=int, default=3)
    ap.add_argument('--steps', type=int, default=3, help='timed steps per ratio and round')
    ap.add_argument('--warmup', type=int, default=1, help='untimed steps per ratio and round')
    ap.add_argument('--ratios', default='1.0,0.9,0.5')
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('time_teacher_forcing.py needs a CUDA device: the hot path has no CPU fallback')
    import __graft_entry__ as entry
    entry.build()
    import bench
    from multilingual_text_to_speech_b200 import _lib, configs
    from multilingual_text_to_speech_b200 import functional as F
    from multilingual_text_to_speech_b200.distributed import GradBucket
    from multilingual_text_to_speech_b200.modules.tacotron2 import Tacotron, TacotronLoss
    from multilingual_text_to_speech_b200.rng import MaskSource
    _lib.set_precision(a.precision)
    dev = torch.device('cuda:0')
    hp = configs.apply(a.config, decoder_regularization='zoneout')
    torch.manual_seed(0)
    model = Tacotron().to(dev).train()
    crit = TacotronLoss(hp.guided_attention_steps, hp.guided_attention_toleration, hp.guided_attention_gain)
    bucket = GradBucket(model, 1)
    MaskSource.manual_seed(1234)
    batch = bench.synth_batch(hp, a.batch, a.text_len, a.frames, 1234, dev)
    free_steps = []
    decode = F.decoder_forward

    def counting_decode(cfg, *args):          # records the number of free-running steps of each decode
        free_steps.append(0 if cfg.teacher is None else int((cfg.teacher == 0).sum()))
        return decode(cfg, *args)

    def step(tf):
        bucket.zero()
        post, pre, stop, align, spk, enc = model(batch['text'], batch['text_length'], batch['target'], batch['target_length'],
                                                 batch.get('speakers'), batch.get('languages'), tf)
        loss, _ = crit(batch['text_length'], batch['target_length'], pre, batch['target'], post, batch['target'], stop,
                       batch['stop_target'], align, batch.get('speakers'), spk, enc, None)
        loss.backward()
        torch.cuda.synchronize()

    ratios = [float(r) for r in a.ratios.split(',')]
    samples = {r: [] for r in ratios}
    frees = {r: [] for r in ratios}
    F.decoder_forward = counting_decode
    try:
        before = card()
        for _ in range(a.rounds):
            for r in ratios:
                for _ in range(a.warmup):
                    step(r)
                del free_steps[:]
                t0 = time.perf_counter()
                for _ in range(a.steps):
                    step(r)
                samples[r].append((time.perf_counter() - t0) * 1e3 / a.steps)
                frees[r].extend(free_steps)
        after = card()
    finally:
        F.decoder_forward = decode
    result = {'card_before': before, 'card_after': after, 'precision': a.precision, 'mode': 'eager',
              'workload': dict(config=a.config, B=a.batch, L=a.text_len, T=a.frames, regularization='zoneout'), 'teacher_forcing': {}}
    for r in ratios:
        v = samples[r]
        result['teacher_forcing'][str(r)] = {'step_ms': {'median': statistics.median(v), 'spread': max(v) - min(v), 'all': v},
                                             'free_running_steps': statistics.mean(frees[r]) if frees[r] else 0.0}
    print(json.dumps(result))


if __name__ == '__main__':
    main()
