"""Throughput of batched synthesis (Tacotron.inference_batch) against one-by-one Tacotron.inference, random weights, seeded texts.

Two regimes:
  fixed   the stop bias is -100 (as tools/time_inference.py does) and every stop logit F.decoder_forward_chunk returns is rewritten to
          -10, since random weights can still fire the token: every utterance decodes --frames frames;
  ragged  this tool (not the product) rewrites the stop logits F.decoder_forward_chunk returns, so that an utterance fires from a seeded
          frame T in [100, --frames] on; T is drawn per text length, the one key a chunk call carries for each of its rows.
For each regime the arms (one-by-one, max_batch 16 / 32 / 64) alternate over --rounds rounds; the tool prints medians and spreads of
utterances/s, mel frames/s and the real-time factor (80 frames per second of audio), the frames decoded with and without the
retirement of finished utterances, and the card name and power limit read in the same run.
    python tools/time_batch_synthesis.py --config generated_switching --n 256
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def card():
    try:
        q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True, text=True)
        return q.stdout.strip().splitlines()[0]
    except (OSError, IndexError):
        return torch.cuda.get_device_name(0) + ', power limit unknown'


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--config', default='generated_switching')
    ap.add_argument('--n', type=int, default=256)
    ap.add_argument('--single-n', type=int, default=0, help='utterances of the one-by-one arm (default: all --n)')
    ap.add_argument('--frames', type=int, default=900)
    ap.add_argument('--precision', default='bf16')
    ap.add_argument('--rounds', type=int, default=3)
    ap.add_argument('--batches', default='16,32,64')
    ap.add_argument('--regimes', default='fixed,ragged')
    a = ap.parse_args()
    from multilingual_text_to_speech_b200 import configs, _lib
    from multilingual_text_to_speech_b200 import functional as F
    from multilingual_text_to_speech_b200.modules.tacotron2 import Tacotron, Decoder
    hp = configs.apply(a.config, max_output_length=a.frames)
    _lib.set_precision(a.precision)
    dev = torch.device('cuda:0')
    torch.manual_seed(0)
    model = Tacotron().to(dev).eval()
    with torch.no_grad():
        model._decoder._stop_prediction.bias.fill_(-100.0)
    rng = np.random.default_rng(0)
    lens = rng.integers(20, 201, size=a.n)
    texts = [torch.from_numpy(rng.integers(1, hp.symbols_count() + 3, size=int(L))).to(dev) for L in lens]
    G = hp.language_number if hp.multi_language else 0
    languages = None
    if G:
        languages = []
        for L in lens:
            w = torch.zeros(1, int(L), G, device=dev)
            w[0, :, int(rng.integers(G))] = 1.0
            languages.append(w)
    speakers = [torch.zeros(1, dtype=torch.long, device=dev) for _ in lens] if hp.multi_speaker else None
    stop_at = {int(L): int(rng.integers(100, a.frames + 1)) for L in range(20, 201)}
    single_n = a.single_n or a.n

    orig = F.decoder_forward_chunk
    log = {'done': 0, 'rows': 0, 'ragged': False}

    def chunk(cfg, memory, lengths, params, state, frames):
        if state.first:
            log['done'] = 0
        spec, stop, align = orig(cfg, memory, lengths, params, state, frames)
        if log['ragged']:
            at = torch.tensor([stop_at[int(L)] for L in lengths.tolist()], device=stop.device)
            t = torch.arange(log['done'] + 1, log['done'] + frames + 1, device=stop.device)
            stop = torch.where(t.unsqueeze(0) >= at.unsqueeze(1), 10.0, -10.0)
        else:
            stop = torch.full_like(stop, -10.0)
        log['done'] += frames
        log['rows'] += memory.shape[0] * frames
        return spec, stop, align
    F.decoder_forward_chunk = chunk

    def arm(mb):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        with torch.no_grad():
            if mb == 0:
                outs = [model.inference(texts[i], None if speakers is None else speakers[i], None if languages is None else languages[i])
                        for i in range(single_n)]
            else:
                outs = model.inference_batch(texts, speakers, languages, max_batch=mb)
        torch.cuda.synchronize()
        dt = time.perf_counter() - t0
        return dt, len(outs), sum(o.shape[-1] for o in outs)

    batches = [int(b) for b in a.batches.split(',')]
    report = {'card': card(), 'config': a.config, 'precision': a.precision, 'n': a.n, 'single_n': single_n, 'frames': a.frames,
              'chunk': Decoder.inference_chunk, 'regimes': {}}
    for regime in a.regimes.split(','):
        log['ragged'] = regime == 'ragged'
        arm(batches[0])                                  # warm-up of every shape the timed window uses
        res = {mb: [] for mb in [0] + batches}
        decoded = {}
        for _ in range(a.rounds):
            for mb in [0] + batches:
                log['rows'] = 0
                dt, n, frames = arm(mb)
                res[mb].append((n / dt, frames / dt, frames / 80.0 / dt))
                decoded[mb] = (log['rows'], frames)
        out = {}
        for mb, rows in res.items():
            name = 'one-by-one' if mb == 0 else f'max_batch {mb}'
            med = [statistics.median(r[k] for r in rows) for k in range(3)]
            spread = [max(r[k] for r in rows) - min(r[k] for r in rows) for k in range(3)]
            out[name] = {'utt_per_s': med[0], 'frames_per_s': med[1], 'rtf': med[2], 'spread': spread,
                         'frames_decoded': decoded[mb][0], 'frames_kept': decoded[mb][1]}
            if mb and regime == 'ragged':      # without retirement every utterance of a group runs until its group's last cut
                order = sorted(range(a.n), key=lambda i: int(lens[i]))
                cut = lambda i: min(-(-(stop_at[int(lens[i])] + hp.stop_frames) // Decoder.inference_chunk) * Decoder.inference_chunk,  # noqa: E731
                                    a.frames)
                out[name]['frames_without_retirement'] = sum(len(order[k:k + mb]) * max(cut(i) for i in order[k:k + mb])
                                                             for k in range(0, a.n, mb))
            print(regime, name, json.dumps(out[name]), flush=True)
        report['regimes'][regime] = out
    F.decoder_forward_chunk = orig
    print(json.dumps(report))


if __name__ == '__main__':
    main()
