#!/usr/bin/env python
"""Minimal WaveRNN training loop on a synthetic corpus: fatchord's vocoder training (train_wavernn.py) on this framework.

    python examples/train_wavernn_synthetic.py --steps 50                                               # one GPU, graph-captured steps
    python examples/train_wavernn_synthetic.py --steps 50 --eager                                       # the eager step
    torchrun --nproc-per-node 8 --master-addr 127.0.0.1 examples/train_wavernn_synthetic.py --steps 50  # data parallel, one rank per GPU

Pieces (all from this repository): a seeded synthetic corpus (waveforms -> `spectrogram_batch(mel=True)` mels, `encode_mu_law` (RAW) or
`float_2_label` (MOL) labels) packed into device memory once as a `VocoderCorpus`; a shuffled sampler that gives each rank its own shard
of the utterance ids every epoch; `GraphedVocoderStep` (window cutting, forward, loss and backward as one CUDA graph) or, with --eager,
the same step launched eagerly; `GradBucket` (flat gradient, one NCCL all-reduce per step) and `FlatParams` + `FusedAdam` (clip 4,
lr 1e-4).  Each rank cuts its own windows and keeps its own batch-norm statistics (no SyncBN).  The last line is a JSON summary: losses,
ms per step over the steps after the first five, and whether every rank ends with the same parameters.  Needs an H100: there is no CPU
path."""
import argparse
import json
import os
import sys

import numpy as np
import torch
import torch.distributed as dist

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

DIMS = dict(rnn_dims=512, fc_dims=512, pad=2, upsample_factors=(5, 5, 11), feat_dims=80, compute_dims=128, res_out_dims=128, res_blocks=10,
            hop_length=275, sample_rate=22050)


def synthetic_corpus(n, mode, bits, seq_len, device, seed=0):
    """n seeded utterances of 1.5 to 4 s: a few decaying partials and a little noise, peak 0.9."""
    from multilingual_text_to_speech_b200.modules.wavernn import VocoderCorpus, encode_mu_law, float_2_label
    from multilingual_text_to_speech_b200.utils.audio import spectrogram_batch
    rng = np.random.default_rng(seed)
    sr = DIMS['sample_rate']
    waves = []
    for _ in range(n):
        t = np.arange(int(rng.uniform(1.5, 4.0) * sr)) / sr
        w = sum(rng.uniform(0.2, 1.0) * np.sin(2 * np.pi * rng.uniform(80, 4000) * t + rng.uniform(0, 2 * np.pi)) * np.exp(-t * rng.uniform(0, 2))
                for _ in range(4))
        w = w + 0.05 * rng.standard_normal(t.shape)
        waves.append((0.9 * w / np.abs(w).max()).astype(np.float32))
    mels = spectrogram_batch(waves, mel=True)
    labels = [encode_mu_law(w, 2 ** bits) if mode == 'RAW' else float_2_label(w, 16) for w in waves]
    return VocoderCorpus(mels, labels, mode, bits, seq_len, DIMS['pad'], DIMS['hop_length'], device)


def shard_batches(n, batch, rank, world, epoch, seed=0):
    """The epoch's shuffle of the n ids (the same on every rank), cut into global batches of batch * world; rank r takes items r, r + world,
    ... of each.  A short last global batch is dropped."""
    perm = np.random.default_rng((seed, epoch)).permutation(n)
    g = batch * world
    for i in range(0, n - g + 1, g):
        yield [int(u) for u in perm[i + rank:i + g:world]]


def main():
    ap = argparse.ArgumentParser(description=__doc__.split('\n')[0])
    ap.add_argument('--steps', type=int, default=50)
    ap.add_argument('--batch', type=int, default=32, help='windows per GPU per step (1 to 64)')
    ap.add_argument('--seq-len', type=int, default=1375, help='samples per window, a multiple of the hop (275), at most 16 hops')
    ap.add_argument('--mode', default='RAW', choices=['RAW', 'MOL'])
    ap.add_argument('--bits', type=int, default=9, help='RAW label bits')
    ap.add_argument('--precision', default='fp32', choices=['fp32', 'bf16'])
    ap.add_argument('--utterances', type=int, default=256, help='synthetic utterances in the corpus')
    ap.add_argument('--eager', action='store_true', help='run the step eagerly instead of as a CUDA graph')
    ap.add_argument('--log-every', type=int, default=10)
    a = ap.parse_args()
    from multilingual_text_to_speech_b200 import _lib
    from multilingual_text_to_speech_b200.distributed import GradBucket
    from multilingual_text_to_speech_b200.graph import GraphedVocoderStep
    from multilingual_text_to_speech_b200.modules.wavernn import WaveRNN, wavernn_loss
    from multilingual_text_to_speech_b200.optim import FlatParams, FusedAdam

    world, rank, local = (int(os.environ.get(k, d)) for k, d in (('WORLD_SIZE', 1), ('RANK', 0), ('LOCAL_RANK', 0)))
    torch.cuda.set_device(local)
    dev = torch.device('cuda', local)
    if world > 1:
        os.environ.setdefault('MASTER_ADDR', '127.0.0.1')
        dist.init_process_group('nccl', device_id=dev)
    _lib.set_precision(a.precision)
    corpus = synthetic_corpus(a.utterances, a.mode, a.bits, a.seq_len, dev)
    torch.manual_seed(0)                                  # the same initial weights on every rank
    model = WaveRNN(**DIMS, bits=a.bits, mode=a.mode).to(dev).train()
    flat, bucket = FlatParams(model), GradBucket(model, world)
    opt = FusedAdam(flat, bucket, lr=1e-4, max_grad_norm=4.0)
    step = None if a.eager else GraphedVocoderStep(model, bucket, corpus, a.batch)
    rng = np.random.default_rng((1, rank))                 # each rank draws its own window offsets
    losses, times, n = [], [], 0
    for epoch in range(1 << 30):
        for ids in shard_batches(len(corpus), a.batch, rank, world, epoch):
            offsets = corpus.draw_offsets(ids, rng)
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            if step is None:
                bucket.zero()
                x, y, m = corpus.batch(ids, offsets)
                loss = wavernn_loss(model(x, m), y, a.mode)
                loss.backward()
            else:
                loss = step(ids, offsets)
            bucket.allreduce()
            info = opt.step()
            e1.record()
            times.append((e0, e1))
            n += 1
            if n % a.log_every == 0 or n == a.steps:
                losses.append((n, float(loss)))
                if rank == 0:
                    print(f'step {n}: loss {losses[-1][1]:.4f}  grad norm {float(info[0]):.3f}  clip x{float(info[1]):.3f}', flush=True)
            if n >= a.steps:
                break
        if n >= a.steps:
            break
    if step is not None:
        step.close()
    torch.cuda.synchronize()
    ms = [s.elapsed_time(e) for s, e in times[5:]] or [s.elapsed_time(e) for s, e in times]
    same = True
    if world > 1:
        ref = flat.flat.clone()
        dist.broadcast(ref, 0)
        ok = torch.tensor([int(torch.equal(ref, flat.flat))], device=dev)
        dist.all_reduce(ok, op=dist.ReduceOp.MIN)
        same = bool(ok.item())
    if rank == 0:
        print(json.dumps({'world': world, 'mode': a.mode, 'precision': a.precision, 'graphed': step is not None, 'batch_per_rank': a.batch,
                          'seq_len': a.seq_len, 'steps': n, 'losses': losses, 'all_finite': all(np.isfinite(v) for _, v in losses),
                          'ms_per_step_median': float(np.median(ms)), 'ms_per_step_spread': float(np.max(ms) - np.min(ms)),
                          'parameters_identical_across_ranks': same}), flush=True)
    if world > 1:
        dist.destroy_process_group()


if __name__ == '__main__':
    main()
