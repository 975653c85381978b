#!/usr/bin/env python
"""Minimal training loop on synthetic data: what `train.py:49-95, 255-272` of the reference looks like on this framework.

    python examples/train_synthetic.py --steps 20                                   # one GPU
    python examples/train_synthetic.py --steps 20 --tf-start 5 --tf-steps 20        # teacher forcing decays from 1.0 after step 5
    torchrun --nproc-per-node 8 --master-addr 127.0.0.1 examples/train_synthetic.py  # data parallel, one rank per GPU

Pieces (all from this repository): `Tacotron` / `TacotronLoss` with the reference's surface, `BucketedPerfectBatchSampler` + `shard`
for language-balanced, length-bucketed batches, `GradBucket` (flat gradient, one NCCL all-reduce per step), `FlatParams` + `FusedAdam`
(global-norm clip + Adam + StepLR in one library call).  Needs an H100: there is no CPU path.
"""
import argparse
import math
import os
import random
import sys

import torch
import torch.distributed as dist

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def cos_decay(global_step, decay_steps):
    """The reference's teacher-forcing schedule (train.py:18-26): 1.0 at step 0, cosine down to 0.0 at `decay_steps`."""
    global_step = min(global_step, decay_steps)
    return 0.5 * (1 + math.cos(math.pi * global_step / decay_steps))


def teacher_forcing_ratio(hp, global_step):
    """train.py:58-60: the constant hp.teacher_forcing, or the cosine decay that starts at hp.teacher_forcing_start_steps."""
    if hp.constant_teacher_forcing:
        return hp.teacher_forcing
    return cos_decay(max(global_step - hp.teacher_forcing_start_steps, 0), hp.teacher_forcing_steps)


class SyntheticCorpus:
    """Stands in for TextToSpeechDataset: items with a language id and a text length; mels are 5 frames per symbol."""

    def __init__(self, hp, n_per_language=400, seed=0):
        rng = random.Random(seed)
        self.items = [{'language': lang, 'len': rng.randint(40, 180)} for lang in range(max(hp.language_number, 1))
                      for _ in range(n_per_language)]
        self.hp = hp

    def __len__(self):
        return len(self.items)

    def collate(self, indices, device):
        hp, g = self.hp, torch.Generator().manual_seed(indices[0])
        lens = torch.tensor([self.items[i]['len'] for i in indices])
        L, T = int(lens.max()), 5 * int(lens.max())
        text = torch.randint(1, hp.symbols_count() + 3, (len(indices), L), generator=g)
        text[torch.arange(L)[None, :] >= lens[:, None]] = 0
        mel = torch.randn(len(indices), hp.num_mels, T, generator=g)
        tlens = 5 * lens
        stop = (torch.arange(T)[None, :] >= (tlens - hp.stop_frames)[:, None]).float()
        lang = torch.tensor([self.items[i]['language'] for i in indices])
        batch = dict(text=text, text_length=lens, target=mel, target_length=tlens, stop_target=stop, languages=lang)
        return {k: v.pin_memory().to(device, non_blocking=True) for k, v in batch.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--config', default='generated_training')
    ap.add_argument('--steps', type=int, default=20)
    ap.add_argument('--batch', type=int, default=60, help='per-GPU batch (a multiple of the number of languages)')
    ap.add_argument('--tf-start', type=int, default=None,
                    help='decay teacher forcing from this step on (hp.teacher_forcing_start_steps; default: the config\'s schedule)')
    ap.add_argument('--tf-steps', type=int, default=None, help='length of the decay (hp.teacher_forcing_steps)')
    ap.add_argument('--outputs-per-step', type=int, default=1, help='mel frames predicted per decoder step (hp.outputs_per_step)')
    a = ap.parse_args()
    from multilingual_text_to_speech_b200 import configs, _lib
    from multilingual_text_to_speech_b200.modules.tacotron2 import Tacotron, TacotronLoss
    from multilingual_text_to_speech_b200.distributed import GradBucket
    from multilingual_text_to_speech_b200.optim import FlatParams, FusedAdam
    from multilingual_text_to_speech_b200.rng import MaskSource
    from multilingual_text_to_speech_b200.utils.samplers import BucketedPerfectBatchSampler, shard

    world, rank, local = (int(os.environ.get(k, d)) for k, d in (('WORLD_SIZE', 1), ('RANK', 0), ('LOCAL_RANK', 0)))
    torch.cuda.set_device(local)
    dev = torch.device('cuda', local)
    if world > 1:
        os.environ.setdefault('MASTER_ADDR', '127.0.0.1')
        dist.init_process_group('nccl', device_id=dev)
    schedule = {}
    if a.tf_start is not None or a.tf_steps is not None:
        schedule['constant_teacher_forcing'] = False
        if a.tf_start is not None:
            schedule['teacher_forcing_start_steps'] = a.tf_start
        if a.tf_steps is not None:
            schedule['teacher_forcing_steps'] = a.tf_steps
    hp = configs.apply(a.config, decoder_regularization='zoneout', outputs_per_step=a.outputs_per_step, **schedule)
    _lib.set_precision('bf16')
    torch.manual_seed(0)
    model = Tacotron().to(dev).train()
    flat, bucket = FlatParams(model), GradBucket(model, world)
    opt = FusedAdam(flat, bucket, lr=hp.learning_rate, weight_decay=hp.weight_decay, max_grad_norm=hp.gradient_clipping,
                    lr_decay_every=hp.learning_rate_decay_each, lr_decay=hp.learning_rate_decay)
    crit = TacotronLoss(hp.guided_attention_steps, hp.guided_attention_toleration, hp.guided_attention_gain)
    MaskSource.manual_seed(1234 + rank)
    corpus = SyntheticCorpus(hp)
    G = max(hp.language_number, 1)
    sampler = BucketedPerfectBatchSampler(corpus, list(range(G)), a.batch * world, [it['len'] for it in corpus.items], bucket_batches=8,
                                          data_parallel_devices=world, seed=0)
    step = 0
    for epoch in range(1000):
        sampler.set_epoch(epoch)
        for global_batch in sampler:
            if len(global_batch) != a.batch * world:
                continue
            b = corpus.collate(shard(global_batch, rank, world, G), dev)
            bucket.zero()
            tf = teacher_forcing_ratio(hp, step)
            post, pre, stop, align, spk, enc = model(b['text'], b['text_length'], b['target'], b['target_length'], None, b['languages'],
                                                     tf)
            loss, parts = crit(b['text_length'], b['target_length'], pre, b['target'], post, b['target'], stop, b['stop_target'], align,
                               None, spk, enc, None)
            loss.backward()
            bucket.allreduce()
            info = opt.step()
            crit.update_states()
            step += 1
            if rank == 0 and step % 5 == 0:
                print(f'step {step}: tf {tf:.3f}  loss {float(loss):.4f}  grad norm {float(info[0]):.3f}  clip x{float(info[1]):.3f}  lr {opt.current_lr():.2e}',
                      flush=True)
            if step >= a.steps:
                if world > 1:
                    dist.destroy_process_group()
                return


if __name__ == '__main__':
    main()
