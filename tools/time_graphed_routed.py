"""Training step of generated_training (G = 10 languages, zoneout) captured as a CUDA graph on routed batches, against the eager routed
step and the graphed reference-layout step, alternated round by round in one process:

- graphed_routed_B64: B = 64 (languages b % 10: counts 7 x 4, 6 x 6) in one graph captured at capacity 7 (GraphedTrainStep
  max_per_language=7);
- eager_routed_B64: the same batch issued from Python; its forward reads the CUDA labels on the host (one device-to-host copy);
- graphed_reference_B60: B = 60 in the reference layout (utterance b of language b % 10), the benchmark's graphed step;
- graphed_imbalanced_B60: the imbalanced B = 60 batch (language 2 absent, language 1 alone, language 0 with 9) in one graph at
  capacity --imbalanced-capacity (default 9).

The graphed arms take their labels from the host, as batches from a data loader come, so the per-call layout read does not wait on
the device.  Prints, per arm, ms per step of every round, the median and the spread (max - min over rounds) and mel frames per second
at the median, with the GPU name, power limit and peak memory.  Needs a CUDA device.

    python tools/time_graphed_routed.py [--steps 10] [--rounds 7] [--precision bf16] [--out DIR]
"""
import argparse
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tools'))

from time_routed_encoder import gpu_info, imbalanced_60  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=10)
    ap.add_argument('--rounds', type=int, default=7)
    ap.add_argument('--warmup', type=int, default=3)
    ap.add_argument('--text-len', type=int, default=180)
    ap.add_argument('--frames', type=int, default=900)
    ap.add_argument('--imbalanced-capacity', type=int, default=9)
    ap.add_argument('--precision', default='bf16', choices=['fp32', 'bf16'])
    ap.add_argument('--out', default=None)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit('time_graphed_routed.py needs a CUDA device')
    import __graft_entry__ as entry
    entry.build()
    from multilingual_text_to_speech_b200 import configs, _lib
    from multilingual_text_to_speech_b200.distributed import GradBucket
    from multilingual_text_to_speech_b200.graph import GraphedTrainStep, capture_stream
    from multilingual_text_to_speech_b200.modules.tacotron2 import Tacotron, TacotronLoss
    from multilingual_text_to_speech_b200.rng import MaskSource
    hp = configs.apply('generated_training', decoder_regularization='zoneout')
    G, L, T = hp.language_number, a.text_len, a.frames
    _lib.set_precision(a.precision)
    dev = torch.device('cuda:0')
    torch.manual_seed(0)
    model = Tacotron().to(dev).train()
    crit = TacotronLoss(hp.guided_attention_steps, hp.guided_attention_toleration, hp.guided_attention_gain)
    bucket = GradBucket(model, 1)
    MaskSource.manual_seed(1234)
    layouts = {'graphed_routed_B64': ([b % G for b in range(64)], 7), 'eager_routed_B64': ([b % G for b in range(64)], None),
               'graphed_reference_B60': ([b % G for b in range(60)], None),
               'graphed_imbalanced_B60': (imbalanced_60(G), a.imbalanced_capacity)}
    g = torch.Generator().manual_seed(1)
    batches = {}
    for name, (ids, _) in layouts.items():
        B = len(ids)
        stop = torch.zeros(B, T)
        stop[:, T - hp.stop_frames:] = 1.0
        b = {k: v.to(dev) for k, v in dict(
            text=torch.randint(1, hp.symbols_count() + 3, (B, L), generator=g), text_length=torch.full((B,), L),
            target=torch.randn(B, hp.num_mels, T, generator=g), target_length=torch.full((B,), T), stop_target=stop).items()}
        b['speakers'] = None
        b['languages'] = torch.tensor(ids) if name.startswith('graphed') else torch.tensor(ids, device=dev)
        batches[name] = b

    def eager(b):
        bucket.zero()
        post, pre, stop, align, spk, enc = model(b['text'], b['text_length'], b['target'], b['target_length'], None, b['languages'],
                                                 hp.teacher_forcing)
        loss, _ = crit(b['text_length'], b['target_length'], pre, b['target'], post, b['target'], stop, b['stop_target'], align, None,
                       spk, enc, None)
        loss.backward()
        return loss

    steps = {}
    for name, (ids, capacity) in layouts.items():
        if name.startswith('graphed'):
            step = GraphedTrainStep(model, crit, bucket, batches[name], teacher_forcing=hp.teacher_forcing, warmup=a.warmup,
                                    max_per_language=capacity)
            steps[name] = step
        else:
            side = capture_stream(dev)              # eager steps on the stream the captures bound the gradient accumulators to
            side.wait_stream(torch.cuda.current_stream(dev))
            with torch.cuda.stream(side):
                for _ in range(a.warmup):
                    eager(batches[name])
            torch.cuda.current_stream(dev).wait_stream(side)
            steps[name] = None
    torch.cuda.synchronize()
    times = {name: [] for name in layouts}
    side = capture_stream(dev)
    for _ in range(a.rounds):
        for name, b in batches.items():
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            torch.cuda.synchronize()
            with torch.cuda.stream(side):
                e0.record()
                for _ in range(a.steps):
                    loss = steps[name](b) if steps[name] is not None else eager(b)
                e1.record()
            torch.cuda.synchronize()
            assert bool(torch.isfinite(loss)), name
            times[name].append(e0.elapsed_time(e1) / a.steps)
    for step in steps.values():
        if step is not None:
            step.close()
    result = {'gpu': gpu_info(), 'precision': a.precision, 'L': L, 'T': T, 'steps_per_round': a.steps, 'rounds': a.rounds,
              'peak_memory_GiB': round(torch.cuda.max_memory_allocated(dev) / 2 ** 30, 1), 'arms': {}}
    for name, ts in times.items():
        ids, capacity = layouts[name]
        med = statistics.median(ts)
        result['arms'][name] = {'B': len(ids), 'capacity': capacity, 'ms_per_step': [round(t, 2) for t in ts], 'median_ms': round(med, 2),
                                'spread_ms': round(max(ts) - min(ts), 2), 'mel_frames_per_s': round(len(ids) * T / (med / 1e3))}
    print(json.dumps(result, indent=1))
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, f'time_graphed_routed_{a.precision}.json'), 'w') as f:
            json.dump(result, f, indent=1)


if __name__ == '__main__':
    main()
