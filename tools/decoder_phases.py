"""Where a step of the persistent decoder loops goes: per-phase SM cycles of one eager training step of the benchmark workload.

Every persistent decoder loop accumulates clock64() deltas per phase on thread 0 of each CTA and writes them, at the end of the launch,
to a [132][8] int64 row block of its workspace (b200tts_debug_persist_profile_offset / b200tts_debug_persist_bwd_profile_offset).  This
script runs one eager training step of the bench.py workload with the workspaces kept, reads the counters of all four loops and prints
cycles per step for each phase: the median and the maximum over the CTAs, next to the card, its power limit and its SM clock.

    python tools/decoder_phases.py [--config generated_training] [--batch 0] [--text-len 180] [--frames 900]

Needs a CUDA device; there is no CPU path.
"""
import argparse
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

NUM_SMS = 132           # rows of each counter block (common.cuh)

# phase slots of each loop, in the order of its PROF_MARK / BPROF_MARK calls (slot: name)
LOOPS = [
    ('attention forward (lstm_loop_tc_kernel<att>)', 'fwd', 0,
     {0: 'wait for the ctx product', 1: 'cell + query projection', 2: 'barrier', 3: 'query reduction', 4: 'energies + exchange',
      5: 'softmax + B fragments', 6: 'context', 7: 'barrier + prefetch'}),
    ('generator forward (lstm_loop_tc_kernel<gen>)', 'fwd', 1,
     {0: 'wait for the product', 1: 'cell', 2: 'barrier'}),
    ('generator reverse (lstm_bwd_loop_tc_kernel)', 'bwd', 0,
     {0: 'cell backward', 1: 'barrier', 2: 'operand prefetch', 4: 'product + barrier'}),
    ('attention reverse (att_bwd_loop_kernel)', 'bwd', 1,
     {0: 'staging + dw + softmax', 1: 'energies + exchanges + dcum', 2: 'barrier', 3: 'PB cell backward', 4: 'barrier + prefetch',
      5: 'P2 product', 6: 'barrier'}),
]


def gpu_info():
    q = 'name,power.limit,clocks.sm,clocks.max.sm'
    try:
        out = subprocess.run(['nvidia-smi', f'--query-gpu={q}', '--format=csv,noheader'], capture_output=True, text=True, timeout=30).stdout
        return out.strip().splitlines()[0]
    except (OSError, subprocess.SubprocessError, IndexError):
        return 'nvidia-smi not available'


def counters(ws, offset):
    import torch
    raw = ws[offset:offset + NUM_SMS * 8 * 8].clone()
    return raw.view(torch.int64).reshape(NUM_SMS, 8).cpu().numpy()


def launched_rows(c):
    """Rows of CTAs outside the grid keep whatever the workspace held.  Every launched CTA's slots add up to the duration of the loop, so
    the rows whose sum lies within 5 % of the median sum are the launched ones (each loop runs on more than half of the rows)."""
    import numpy as np
    tot = c.sum(axis=1).astype(np.float64)
    med = np.median(tot)
    return c[(tot > 0) & (np.abs(tot - med) <= 0.05 * med)]


def main():
    ap = argparse.ArgumentParser(description=__doc__.split('\n')[0])
    ap.add_argument('--config', default='generated_training')
    ap.add_argument('--batch', type=int, default=0)
    ap.add_argument('--text-len', type=int, default=180)
    ap.add_argument('--frames', type=int, default=900)
    ap.add_argument('--regularization', default='zoneout', choices=['zoneout', 'dropout'])
    a = ap.parse_args()

    import numpy as np
    import torch
    if not torch.cuda.is_available():
        raise SystemExit('decoder_phases.py needs a CUDA device: the counters are written by the GPU loops')
    import __graft_entry__ as entry
    entry.build()
    import bench
    from multilingual_text_to_speech_b200 import _lib, functional as F
    from multilingual_text_to_speech_b200.modules.tacotron2 import Tacotron, TacotronLoss
    from multilingual_text_to_speech_b200.rng import MaskSource
    from multilingual_text_to_speech_b200.distributed import GradBucket
    import ctypes

    hp, B, L, T = bench.workload(a)
    _lib.set_precision('bf16')
    dev = torch.device('cuda', 0)
    torch.manual_seed(0)
    model = Tacotron().to(dev).train()
    crit = TacotronLoss(hp.guided_attention_steps, hp.guided_attention_toleration, hp.guided_attention_gain)
    bucket = GradBucket(model, 1)
    MaskSource.manual_seed(1234)
    batch = bench.synth_batch(hp, B, L, T, 1234, dev)

    F.PROFILE.clear()
    F.PROFILE['keep_ws'] = True
    bucket.zero()
    post, pre, stop, align, spk, enc = model(batch['text'], batch['text_length'], batch['target'], batch['target_length'],
                                             batch.get('speakers'), batch.get('languages'), hp.teacher_forcing)
    loss, _ = crit(batch['text_length'], batch['target_length'], pre, batch['target'], post, batch['target'], stop,
                   batch['stop_target'], align, batch.get('speakers'), spk, enc, None)
    loss.backward()
    torch.cuda.synchronize()
    F.PROFILE['keep_ws'] = False
    if 'last_ws' not in F.PROFILE or 'last_bws' not in F.PROFILE:
        raise SystemExit('the decoder op kept no workspace: this workload does not run the fused decoder')

    lib = _lib.load()
    shape = ctypes.byref(F.PROFILE['last_shape'])
    path = lib.b200tts_decoder_path(shape)
    if path & 0b10101 != 0b10101:
        raise SystemExit(f'this shape does not run all persistent loops (path bits {path:#b})')
    fwd_off = lib.b200tts_debug_persist_profile_offset(shape)
    ws = {'fwd': F.PROFILE['last_ws'], 'bwd': F.PROFILE['last_bws']}

    print(f'device: {torch.cuda.get_device_name(0)} | nvidia-smi name, power limit, SM clock, max SM clock: {gpu_info()}')
    print(f'workload: {a.config}, B = {B}, L = {L}, T = {T}, bf16, one eager training step; SM cycles per decoder step')
    for title, which, idx, slots in LOOPS:
        off = fwd_off + idx * NUM_SMS * 8 * 8 if which == 'fwd' else lib.b200tts_debug_persist_bwd_profile_offset(shape, idx)
        c = launched_rows(counters(ws[which], off)) / T
        print(f'\n{title}: {len(c)} CTAs')
        print(f'  {"slot":<4} {"phase":<30} {"median":>9} {"max":>9}')
        for s, name in slots.items():
            print(f'  {s:<4} {name:<30} {np.median(c[:, s]):9.0f} {c[:, s].max():9.0f}')
        tot = c.sum(axis=1)
        print(f'  {"":<4} {"total":<30} {np.median(tot):9.0f} {tot.max():9.0f}')


if __name__ == '__main__':
    main()
