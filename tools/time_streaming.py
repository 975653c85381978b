"""Time streaming synthesis (modules/streaming.py: speech_stream) against the one-shot paths, at the reference's dimensions with random
weights and seeded texts.

    python tools/time_streaming.py [--frames 200] [--text-len 60] [--chunks 32,64,128] [--modes RAW,MOL] [--rounds 3] [--out FILE]

The stop projection's bias is set so that the stop token never fires: every utterance runs to --frames (hp.max_output_length).  Arms, alternated
round by round on the same text:
  * stream/<chunk>: speech_stream at that decoder chunk: time to first audio, the wall time between chunks, and the real-time factor
    (wall time / audio duration);
  * fstream/<chunk>: speech_stream(…, target=11000, overlap=550): folded streaming, whose audio equals the folded arm's;
  * unfolded: Tacotron.inference, then WaveRNN.generate(mel, target=F hop, overlap=0) (one row);
  * folded: Tacotron.inference, then WaveRNN.generate_batch([mel], 11000, 550).
Every time is a host clock that ends in torch.cuda.synchronize().  The card's name and power limit are read in the same run."""
import argparse
import json
import os
import statistics
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from time_wavernn import DIMS, card  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--frames', type=int, default=200)
    ap.add_argument('--text-len', type=int, default=60)
    ap.add_argument('--chunks', default='32,64,128')
    ap.add_argument('--modes', default='RAW,MOL')
    ap.add_argument('--rounds', type=int, default=3)
    ap.add_argument('--out', default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('time_streaming: no CUDA device')
    import __graft_entry__ as entry
    entry.build()
    from multilingual_text_to_speech_b200 import _lib
    from multilingual_text_to_speech_b200.params.params import Params as hp
    from multilingual_text_to_speech_b200.modules.tacotron2 import Tacotron
    from multilingual_text_to_speech_b200.modules.wavernn import WaveRNN
    from multilingual_text_to_speech_b200.modules.streaming import speech_stream
    hp.reset()
    hp.max_output_length = a.frames
    torch.manual_seed(0)
    taco = Tacotron().cuda().eval()
    with torch.no_grad():
        taco._decoder._stop_prediction.bias.fill_(-1e4)      # the stop token never fires: every decode runs to --frames
    text = torch.randint(3, hp.symbols_count() + 3, (a.text_len,), generator=torch.Generator().manual_seed(1)).cuda()
    hop, sr = DIMS['hop_length'], DIMS['sample_rate']
    audio_s = (a.frames - 1) * hop / sr
    chunks = [int(c) for c in a.chunks.split(',')]
    rows = []
    for mode in a.modes.split(','):
        torch.manual_seed(2)
        voc = WaveRNN(**dict(DIMS, mode=mode)).cuda().eval()
        arms = [f'stream/{c}' for c in chunks] + [f'fstream/{c}' for c in chunks] + ['unfolded', 'folded']

        def run(arm):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            stamps = []
            if '/' in arm:
                fold = dict(target=11000, overlap=550) if arm.startswith('fstream/') else {}
                for w in speech_stream(taco, voc, text, chunk_frames=int(arm.split('/')[1]), **fold):
                    torch.cuda.synchronize()
                    stamps.append((time.perf_counter() - t0, int(w.shape[0])))
            else:
                mel = taco.inference(text)
                F = mel.shape[1]
                w = voc.generate(mel, target=F * hop, overlap=0) if arm == 'unfolded' else voc.generate_batch([mel], 11000, 550)[0]
                torch.cuda.synchronize()
                stamps.append((time.perf_counter() - t0, int(w.shape[0])))
            return stamps

        for arm in arms:             # warm-up: module loads, every shape once
            run(arm)
        res = {arm: [] for arm in arms}
        for _ in range(a.rounds):
            for arm in arms:
                res[arm].append(run(arm))
        for arm in arms:
            first = [s[0][0] for s in res[arm] if s and s[0][1] > 0] or [s[-1][0] for s in res[arm]]
            total = [s[-1][0] for s in res[arm]]
            gaps = [t1 - t0 for s in res[arm] for (t0, _), (t1, _) in zip(s, s[1:])]
            samples = sum(n for _, n in res[arm][0])
            rows.append(dict(mode=mode, arm=arm, first_audio_s=statistics.median(first), total_s=statistics.median(total),
                             total_spread_s=max(total) - min(total), rtf=statistics.median(total) / audio_s,
                             gap_median_s=statistics.median(gaps) if gaps else None, gap_max_s=max(gaps) if gaps else None,
                             chunks=len(res[arm][0]), samples=samples))
            print(json.dumps(rows[-1]), flush=True)
    out = dict(card=card(), frames=a.frames, audio_s=audio_s, text_len=a.text_len, rounds=a.rounds, rows=rows)
    print(json.dumps(dict(card=out['card'], frames=a.frames, audio_s=audio_s)))
    if a.out:
        with open(a.out, 'w') as f:
            json.dump(out, f, indent=1)
    _lib.set_precision('fp32')


if __name__ == '__main__':
    main()
