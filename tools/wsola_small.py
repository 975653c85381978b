"""A small ragged batch through both WSOLA kernels (csrc/wsola.cu), for compute-sanitizer memcheck and racecheck runs.

It runs time_stretch_batch and retime_batch at the default hop and tolerance (9 warps per search CTA, one candidate pair per thread),
then the kernels directly at tolerance 1,024 and hop 100, where the search launches 1,024 threads and some score two candidate pairs
per frame.  Inputs cover a 1-sample waveform, silence, and frames whose spans reach past both ends of the input.

    compute-sanitizer --tool memcheck --kernel-name kns=wsola_ python tools/wsola_small.py
"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    import __graft_entry__ as entry
    entry.build()
    from multilingual_text_to_speech_b200 import _lib
    from multilingual_text_to_speech_b200 import functional as F
    from multilingual_text_to_speech_b200.utils import audio
    rng = np.random.default_rng(0)
    waves = [rng.standard_normal(n).astype(np.float32) * 0.3 for n in (1, 700, 3000)] + [np.zeros(1200, np.float32)]
    ys = audio.time_stretch_batch(waves, [0.5, 1.3, 0.8, 2.0])
    hop = audio.ms_to_frames(audio.hp.stft_shift_ms)
    ds = [np.array([1 + len(w) // hop], dtype=np.int64) for w in waves]
    zs = audio.retime_batch(waves, ds, [d * 2 for d in ds])
    assert all(np.isfinite(y).all() for y in ys + zs)

    H, D = 100, _lib.WSOLA_MAX_TOLERANCE
    dev = torch.device('cuda:0')
    lengths, outs = [len(w) for w in waves], [2 * len(w) for w in waves]
    frames = [(n - 1) // H + 2 for n in outs]
    soff, ooff, foff = (torch.tensor(np.concatenate([[0], np.cumsum(v)]), dtype=torch.int32, device=dev) for v in (lengths, outs, frames))
    shape = _lib.WsolaShape(len(waves), sum(lengths), sum(outs), sum(frames), H, D)
    wave = torch.from_numpy(np.concatenate(waves)).to(dev)
    warp = torch.from_numpy(np.concatenate([np.arange(K) * H * 0.5 for K in frames])).to(dev)
    positions = F.wsola_positions(shape, wave, soff, warp, foff)
    y = F.wsola_overlap_add(shape, wave, soff, positions, foff, ooff)
    torch.cuda.synchronize()
    assert bool(torch.isfinite(y).all())
    print('wsola_small ok')


if __name__ == '__main__':
    main()
