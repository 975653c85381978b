"""Time the graph-captured WaveRNN training step (GraphedVocoderStep: windows cut on the device from a resident VocoderCorpus, forward, loss
and backward replayed as one CUDA graph) against the eager step as users run it without it (vocoder_batch on the host, the copy to the
device, forward, loss, backward), both followed by the same FusedAdam step (clip 4, lr 1e-4), at the reference's dimensions with random
weights.

    python tools/time_wavernn_graph.py [--configs 32x1375,64x2750] [--modes RAW,MOL] [--precisions fp32,bf16] [--rounds 7] [--steps 3]

Each round runs `steps` steps of one arm, then of the other, each timed from a device event before its first step to a host synchronise
after its last; the table gives the median and the spread (max - min) over the rounds, in ms per step and samples per second.  It also
times one corpus.batch call against vocoder_batch plus its host-to-device copy (host clock around 50 calls ending in a synchronise).  With
two or more GPUs it runs the example trainer under torchrun on all of them; otherwise it says so.  The card's name and power limit are read
in the same run.  Prints one JSON object."""
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

DIMS = dict(rnn_dims=512, fc_dims=512, bits=9, pad=2, upsample_factors=(5, 5, 11), feat_dims=80, compute_dims=128, res_out_dims=128,
            res_blocks=10, hop_length=275, sample_rate=22050)
HOP, PAD = 275, 2


def card():
    try:
        q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'], capture_output=True, text=True)
        return q.stdout.strip().splitlines()[0]
    except (OSError, IndexError):
        return torch.cuda.get_device_name(0) + ', power limit unknown'


def host_corpus(mode, seq_len, n=256, seed=0):
    """n random utterances of 10 to 50 frames beyond one window: mels [80, F] fp32 and labels (RAW 9-bit, MOL 16-bit) of F hop samples."""
    rng = np.random.default_rng(seed)
    win = seq_len // HOP + 2 * PAD
    mels, labels = [], []
    for f in rng.integers(win + 10, win + 50, n):
        mels.append(rng.standard_normal((80, int(f))).astype(np.float32))
        labels.append(rng.integers(0, 512 if mode == 'RAW' else 65536, int(f) * HOP))
    return mels, labels


class Arm:
    def __init__(self, mode, dev):
        from multilingual_text_to_speech_b200.distributed import GradBucket
        from multilingual_text_to_speech_b200.modules.wavernn import WaveRNN
        from multilingual_text_to_speech_b200.optim import FlatParams, FusedAdam
        torch.manual_seed(0)
        self.model = WaveRNN(**DIMS, mode=mode).to(dev).train()
        self.bucket = GradBucket(self.model)
        self.opt = FusedAdam(FlatParams(self.model), self.bucket, lr=1e-4, max_grad_norm=4.0)


def run(B, T, mode, prec, rounds, steps, dev):
    from multilingual_text_to_speech_b200 import _lib
    from multilingual_text_to_speech_b200.graph import GraphedVocoderStep
    from multilingual_text_to_speech_b200.modules.wavernn import VocoderCorpus, vocoder_batch, wavernn_loss
    _lib.set_precision(prec)
    mels, labels = host_corpus(mode, T)
    corpus = VocoderCorpus(mels, labels, mode, 9, T, PAD, HOP, dev)
    rng = np.random.default_rng(1)

    def draw():
        ids = [int(u) for u in rng.integers(0, len(corpus), B)]
        return ids, corpus.draw_offsets(ids, rng)

    eager, graphed = Arm(mode, dev), Arm(mode, dev)
    step = GraphedVocoderStep(graphed.model, graphed.bucket, corpus, B)

    def eager_step():
        ids, offs = draw()
        x, y, m = vocoder_batch([mels[u] for u in ids], [labels[u] for u in ids], offs, mode, 9, T, PAD, HOP)
        x, y, m = x.to(dev), y.to(dev), m.to(dev)
        eager.bucket.zero()
        wavernn_loss(eager.model(x, m), y, mode).backward()
        eager.opt.step()

    def graphed_step():
        step(*draw())
        graphed.opt.step()

    arms = {'eager': eager_step, 'graphed': graphed_step}
    for f in arms.values():
        f()
    torch.cuda.synchronize()
    ms = {k: [] for k in arms}
    for _ in range(rounds):
        for k, f in arms.items():
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(steps):
                f()
            e1.record()
            torch.cuda.synchronize()
            ms[k].append(e0.elapsed_time(e1) / steps)
    step.close()
    out = {}
    for k, t in ms.items():
        med = statistics.median(t)
        out[f'{k}_ms'] = round(med, 2)
        out[f'{k}_spread_ms'] = round(max(t) - min(t), 2)
        out[f'{k}_samples_per_s'] = round(B * T / med * 1e3)
    out['graphed_gain_pct'] = round(100 * (out['eager_ms'] - out['graphed_ms']) / out['eager_ms'], 1)
    # one batch of windows: the device cut against the host collate plus its copy
    n = 50
    ids, offs = draw()
    for name, f in (('corpus_batch_ms', lambda: corpus.batch(ids, offs)),
                    ('vocoder_batch_and_copy_ms', lambda: [t.to(dev) for t in vocoder_batch([mels[u] for u in ids], [labels[u] for u in ids],
                                                                                            offs, mode, 9, T, PAD, HOP)])):
        f()
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for _ in range(n):
            f()
        torch.cuda.synchronize()
        out[name] = round((time.perf_counter() - t0) * 1e3 / n, 3)
    _lib.set_precision('fp32')
    return out


def multi_gpu(count):
    if count < 2:
        return f'not run: this machine has {count} GPU'
    cmd = [sys.executable, '-m', 'torch.distributed.run', '--nproc-per-node', str(count), '--master-addr', '127.0.0.1', '--master-port', '29533',
           os.path.join(ROOT, 'examples', 'train_wavernn_synthetic.py'), '--steps', '30', '--batch', '32']
    res = subprocess.run(cmd, capture_output=True, text=True, timeout=1800)
    lines = [ln for ln in res.stdout.splitlines() if ln.startswith('{')]
    return json.loads(lines[-1]) if res.returncode == 0 and lines else {'returncode': res.returncode, 'tail': res.stdout[-2000:] + res.stderr[-2000:]}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--configs', default='32x1375,64x2750')
    ap.add_argument('--modes', default='RAW,MOL')
    ap.add_argument('--precisions', default='fp32,bf16')
    ap.add_argument('--rounds', type=int, default=7)
    ap.add_argument('--steps', type=int, default=3, help='steps per arm per round')
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('time_wavernn_graph needs a CUDA device')
    dev = torch.device('cuda:0')
    result = {'card': card(), 'steps': {}}
    for cfg in a.configs.split(','):
        B, T = (int(v) for v in cfg.split('x'))
        for mode in a.modes.split(','):
            for prec in a.precisions.split(','):
                result['steps'][f'B={B} T={T} {mode} {prec}'] = run(B, T, mode, prec, a.rounds, a.steps, dev)
                torch.cuda.empty_cache()
    result['multi_gpu'] = multi_gpu(torch.cuda.device_count())
    print(json.dumps(result))


if __name__ == '__main__':
    main()
