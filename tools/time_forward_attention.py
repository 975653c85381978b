"""Step times of forward attention (hp.attention_type = "forward") beside the location-sensitive default, on the benchmark workload
(generated_training, zoneout, B = 60, L = 180, T = 900, bf16 by default):

  * one training step: forward + TacotronLoss + backward captured as a CUDA graph (GraphedTrainStep) and replayed;
  * one evaluation decode: eval mode, teacher forcing 0.0 (every frame free-running), what train.py:125 runs every epoch.

The attention types alternate round by round in one process so that both see the same card state.  Prints one JSON line with the
card, its power limit and SM clock, and per attention type the median and spread (max - min) over the rounds.

    python tools/time_forward_attention.py [--rounds 3] [--steps 5] [--warmup 3] [--precision bf16]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

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


def timed_ms(fn, n):
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(n):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n


def one_round(attention, a, dev):
    import bench
    from multilingual_text_to_speech_b200 import configs
    from multilingual_text_to_speech_b200.modules.tacotron2 import Tacotron, TacotronLoss
    from multilingual_text_to_speech_b200.rng import MaskSource
    from multilingual_text_to_speech_b200.distributed import GradBucket
    from multilingual_text_to_speech_b200.graph import GraphedTrainStep
    hp = configs.apply(a.config, decoder_regularization='zoneout', attention_type=attention)
    torch.manual_seed(0)
    model = Tacotron().to(dev).train()
    crit = TacotronLoss(hp.guided_attention_steps, hp.guided_attention_toleration, hp.guided_attention_gain)
    bucket = GradBucket(model, 1)
    MaskSource.manual_seed(1234)
    batch = bench.synth_batch(hp, a.batch, a.text_len, a.frames, 1234, dev)
    graphed = GraphedTrainStep(model, crit, bucket, batch, teacher_forcing=hp.teacher_forcing, warmup=a.warmup)
    train_ms = timed_ms(lambda: graphed(batch), a.steps)

    def evaluate():
        with torch.no_grad():
            model(batch['text'], batch['text_length'], batch['target'], batch['target_length'], batch.get('speakers'),
                  batch.get('languages'), 0.0)
    model.eval()
    evaluate()
    eval_ms = timed_ms(evaluate, max(1, a.steps // 2))
    del graphed, model, bucket
    torch.cuda.empty_cache()
    return train_ms, eval_ms


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--config', default='generated_training')
    ap.add_argument('--batch', type=int, default=60)
    ap.add_argument('--text-len', type=int, default=180)
    ap.add_argument('--frames', type=int, default=900)
    ap.add_argument('--precision', default='bf16', choices=['bf16', 'fp32'])
    ap.add_argument('--rounds', type=int, default=3)
    ap.add_argument('--steps', type=int, default=5)
    ap.add_argument('--warmup', type=int, default=3)
    ap.add_argument('--attention', default='forward,location_sensitive')
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('time_forward_attention.py needs a CUDA device: the hot path has no CPU fallback')
    import __graft_entry__ as entry
    entry.build()
    from multilingual_text_to_speech_b200 import _lib
    _lib.set_precision(a.precision)
    dev = torch.device('cuda:0')
    kinds = a.attention.split(',')
    samples = {k: {'train_ms': [], 'eval_ms': []} for k in kinds}
    before = card()
    for _ in range(a.rounds):
        for k in kinds:
            tr, ev = one_round(k, a, dev)
            samples[k]['train_ms'].append(tr)
            samples[k]['eval_ms'].append(ev)
    result = {'card_before': before, 'card_after': card(), 'precision': a.precision,
              'workload': dict(config=a.config, B=a.batch, L=a.text_len, T=a.frames, regularization='zoneout'), 'attention': {}}
    for k, s in samples.items():
        result['attention'][k] = {m: {'median': statistics.median(v), 'spread': max(v) - min(v), 'all': v} for m, v in s.items()}
    print(json.dumps(result))


if __name__ == '__main__':
    main()
