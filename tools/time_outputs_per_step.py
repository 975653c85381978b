"""Training-step and synthesis times at several mel frames per decoder step (hp.outputs_per_step = r).

Training: the graphed training step (GraphedTrainStep, bf16, zoneout, teacher forcing 1.0) at r = 1, 2 and 4 on the benchmark workload
(generated_training, B = 60, L = 180, T = 900) and on the config-5 shape (generated_switching, B = 60, L = 300, T = 1200).  Each r is its
own model with the same seed; the r values alternate round by round in one process so that all of them see the same card state.
Synthesis: Tacotron.inference_batch over 64 texts at r = 1 and 2 (stop bias -100, decoding up to --synth-frames frames per utterance;
the rate counts the frames actually returned).
Prints one JSON line with the card, its power limit and SM clock (read in the same call), and per workload and r the median and spread
(max - min) of the per-round means in ms and mel frames per second.

    python tools/time_outputs_per_step.py [--rounds 3] [--steps 5] [--warmup 3]
"""
import argparse
import json
import os
import statistics
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tools'))

WORKLOADS = (('generated_training', 60, 180, 900), ('generated_switching', 60, 300, 1200))


def summary(v, frames):
    med = statistics.median(v)
    return {'ms': {'median': med, 'spread': max(v) - min(v), 'all': v}, 'mel_frames_per_s': frames / (med * 1e-3)}


def time_training(a, config, B, L, T, rs, dev):
    import bench
    from multilingual_text_to_speech_b200 import configs
    from multilingual_text_to_speech_b200.distributed import GradBucket
    from multilingual_text_to_speech_b200.graph import GraphedTrainStep
    from multilingual_text_to_speech_b200.modules.tacotron2 import Tacotron, TacotronLoss
    from multilingual_text_to_speech_b200.rng import MaskSource
    steps = {}
    MaskSource.manual_seed(1234)
    try:
        for r in rs:
            hp = configs.apply(config, decoder_regularization='zoneout', outputs_per_step=r)
            torch.manual_seed(0)
            model = Tacotron().to(dev).train()
            crit = TacotronLoss(hp.guided_attention_steps, hp.guided_attention_toleration, hp.guided_attention_gain)
            bucket = GradBucket(model, 1)
            batch = bench.synth_batch(hp, B, L, T, 1234, dev)
            steps[r] = (GraphedTrainStep(model, crit, bucket, batch, teacher_forcing=1.0, warmup=a.warmup), batch)
        samples = {r: [] for r in rs}
        for _ in range(a.rounds):
            for r in rs:
                step, batch = steps[r]
                for _ in range(a.warmup):
                    step(batch)
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                for _ in range(a.steps):
                    step(batch)
                torch.cuda.synchronize()
                samples[r].append((time.perf_counter() - t0) * 1e3 / a.steps)
    finally:
        for step, _ in steps.values():
            step.close()
    frames = B * T
    return {str(r): dict(summary(samples[r], frames), decoder_steps=-(-T // r)) for r in rs}


def time_synthesis(a, rs, dev):
    from multilingual_text_to_speech_b200 import configs
    from multilingual_text_to_speech_b200.modules.tacotron2 import Tacotron
    models = {}
    for r in rs:
        hp = configs.apply('generated_training', decoder_regularization='zoneout', outputs_per_step=r, max_output_length=a.synth_frames)
        torch.manual_seed(0)
        model = Tacotron().to(dev).eval()
        with torch.no_grad():
            model._decoder._stop_prediction.bias.fill_(-100.0)      # random weights: keep the stop token from firing
        models[r] = (model, hp.symbols_count())
    g = torch.Generator().manual_seed(5)
    texts = [torch.randint(1, models[rs[0]][1] + 3, (int(n),), generator=g) for n in torch.randint(100, 181, (a.synth_texts,), generator=g)]
    lang = []                   # one language per text, as per-character weights [1, L, G] (the generated encoder's input form)
    for i, t in enumerate(texts):
        w = torch.zeros(1, t.shape[0], 10, device=dev)
        w[0, :, i % 10] = 1.0
        lang.append(w)
    texts = [t.to(dev) for t in texts]
    samples, frames = {r: [] for r in rs}, {}
    for _ in range(a.rounds):
        for r in rs:
            model = models[r][0]
            model.inference_batch(texts, languages=lang)
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            outs = model.inference_batch(texts, languages=lang)
            torch.cuda.synchronize()
            samples[r].append((time.perf_counter() - t0) * 1e3)
            frames[r] = sum(int(o.shape[1]) for o in outs)
    return {str(r): dict(summary(samples[r], frames[r]), frames_decoded=frames[r]) for r in rs}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--rounds', type=int, default=3)
    ap.add_argument('--steps', type=int, default=5, help='timed graph replays per r and round')
    ap.add_argument('--warmup', type=int, default=3, help='untimed replays per r and round')
    ap.add_argument('--train-r', default='1,2,4')
    ap.add_argument('--synth-r', default='1,2')
    ap.add_argument('--synth-texts', type=int, default=64)
    ap.add_argument('--synth-frames', type=int, default=600)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('time_outputs_per_step.py needs a CUDA device: the hot path has no CPU fallback')
    import __graft_entry__ as entry
    entry.build()
    from time_teacher_forcing import card
    from multilingual_text_to_speech_b200 import _lib
    _lib.set_precision('bf16')
    dev = torch.device('cuda:0')
    before = card()
    result = {'card_before': before, 'precision': 'bf16', 'training': {}, 'synthesis': {}}
    for config, B, L, T in WORKLOADS:
        key = f'{config} B{B} L{L} T{T} zoneout graphed'
        result['training'][key] = time_training(a, config, B, L, T, [int(r) for r in a.train_r.split(',')], dev)
        torch.cuda.empty_cache()
    result['synthesis'][f'inference_batch {a.synth_texts} texts, at most {a.synth_frames} frames'] = \
        time_synthesis(a, [int(r) for r in a.synth_r.split(',')], dev)
    result['card_after'] = card()
    print(json.dumps(result))


if __name__ == '__main__':
    main()
