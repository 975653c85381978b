"""Eager training step of generated_training (G = 10 languages) on three batch layouts and one label feed, timed alternately:

- B = 60 in the reference layout (utterance b of language b % 10): the grouped encoder's plain reshape, as before;
- B = 64 with languages b % 10: routed through the padded layout (n_max = 7, languages 4..9 with one vacant row);
- B = 60 imbalanced (one language absent, one a single utterance, n_max = 9): routed;
- B = 60 in the reference layout with its labels copied to the GPU afresh before every step, as a training loop feeding new batches does.

Every forward reads its CUDA labels on the host (one device-to-host copy, a synchronisation): a resident labels tensor and a fresh one
cost the same; the last row shows it.

Prints ms per step and mel frames per second for each, with the GPU name and power limit.  Needs a CUDA device.

    python tools/time_routed_encoder.py [--steps 10] [--rounds 3] [--precision bf16] [--out DIR]
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def gpu_info():
    import torch
    info = {'name': torch.cuda.get_device_name(0)}
    try:
        q = subprocess.run(['nvidia-smi', '--query-gpu=power.limit,clocks.max.sm', '--format=csv,noheader'], stdout=subprocess.PIPE,
                           stderr=subprocess.DEVNULL, text=True, timeout=30).stdout.strip().splitlines()
        info['power_limit, max_sm_clock'] = q[0] if q else 'unknown'
    except (OSError, subprocess.SubprocessError):
        info['power_limit, max_sm_clock'] = 'unknown'
    return info


def imbalanced_60(G):
    import torch
    ids = []
    for lang, n in enumerate([9, 1, 0, 8, 7, 6, 8, 7, 6, 8][:G]):
        ids += [lang] * n
    return [ids[i] for i in torch.randperm(len(ids), generator=torch.Generator().manual_seed(9)).tolist()]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=10)
    ap.add_argument('--rounds', type=int, default=3)
    ap.add_argument('--warmup', type=int, default=3)
    ap.add_argument('--text-len', type=int, default=180)
    ap.add_argument('--frames', type=int, default=900)
    ap.add_argument('--precision', default='bf16', choices=['fp32', 'bf16'])
    ap.add_argument('--out', default=None)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit('time_routed_encoder.py needs a CUDA device')
    import __graft_entry__ as entry
    entry.build()
    from multilingual_text_to_speech_b200 import configs, _lib
    from multilingual_text_to_speech_b200.modules.tacotron2 import Tacotron, TacotronLoss
    from multilingual_text_to_speech_b200.distributed import GradBucket
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
    layouts = {'B60_reference': [b % G for b in range(60)], 'B64_routed': [b % G for b in range(64)], 'B60_imbalanced': imbalanced_60(G),
               'B60_reference_fresh_labels': [b % G for b in range(60)]}
    g = torch.Generator().manual_seed(1)
    batches = {}
    for name, ids in layouts.items():
        B = len(ids)
        stop = torch.zeros(B, T)
        stop[:, T - hp.stop_frames:] = 1.0
        batches[name] = {k: v.to(dev) for k, v in dict(
            text=torch.randint(1, hp.symbols_count() + 3, (B, L), generator=g), text_length=torch.full((B,), L),
            target=torch.randn(B, hp.num_mels, T, generator=g), target_length=torch.full((B,), T), stop_target=stop,
            languages=torch.tensor(ids)).items()}
        if name.endswith('fresh_labels'):
            batches[name]['host_languages'] = torch.tensor(ids).pin_memory()

    def step(b):
        if 'host_languages' in b:
            b['languages'] = b['host_languages'].to(dev, non_blocking=True)
        bucket.zero()
        post, pre, stop, align, spk, enc = model(b['text'], b['text_length'], b['target'], b['target_length'], None, b['languages'],
                                                 hp.teacher_forcing)
        loss, _ = crit(b['text_length'], b['target_length'], pre, b['target'], post, b['target'], stop, b['stop_target'], align, None,
                       spk, enc, None)
        loss.backward()
        return loss

    for b in batches.values():
        for _ in range(a.warmup):
            step(b)
    torch.cuda.synchronize()
    times = {name: [] for name in batches}
    for _ in range(a.rounds):
        for name, b in batches.items():
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            torch.cuda.synchronize()
            e0.record()
            for _ in range(a.steps):
                loss = step(b)
            e1.record()
            torch.cuda.synchronize()
            assert bool(torch.isfinite(loss)), name
            times[name].append(e0.elapsed_time(e1) / a.steps)
    result = {'gpu': gpu_info(), 'precision': a.precision, 'L': L, 'T': T, 'steps_per_round': a.steps, 'rounds': a.rounds, 'layouts': {}}
    for name, ts in times.items():
        B = len(layouts[name])
        best = min(ts)
        result['layouts'][name] = {'B': B, 'ms_per_step': [round(t, 2) for t in ts], 'best_ms': round(best, 2),
                                   'mel_frames_per_s': round(B * T / (best / 1e3))}
    print(json.dumps(result, indent=1))
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, f'time_routed_encoder_{a.precision}.json'), 'w') as f:
            json.dump(result, f, indent=1)


if __name__ == '__main__':
    main()
