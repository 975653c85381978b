"""Time concurrent streaming synthesis (modules/streaming.py: speech_streams, one WaveRNN.stream_pool shared by N texts) against N
speech_stream runs one after another and against inference_batch + folded generate_batch, at the reference's dimensions with random weights
and seeded texts.

    python tools/time_stream_pool.py [--frames 200] [--text-len 60] [--streams 1,8,16,32,64] [--ragged 64] [--serial-max 8] [--chunk 64]
                                     [--modes RAW,MOL] [--rounds 2] [--out FILE]

The stop projection's bias is set so that the stop token never fires: every text runs to --frames (hp.max_output_length).  The ragged mix
(--ragged N texts, 0: none) instead cuts text i at 21 + (i * 37) % (2 --frames - 20) frames (21 to 2 --frames, mean about --frames) through
the decoder's stop rule, so that streams end and leave the pool at different calls.  Arms, alternated round by round:
  * pool/N: speech_streams of N texts.  Per stream: the real-time factor (wall time to its last chunk / its audio duration), the time to
    its first audio and the largest gap between its chunks; aggregate audio-seconds per wall second; the loop's microseconds per sample
    step (CUDA events around each loop call: b200tts_wavernn_run_rows, or b200tts_wavernn_run_stream in a one-stream pool); the time per
    pool.run() outside the loop kernel, host work and the feature and GEMM kernels (the wall time of the run() calls, each ending in the abort-flag read that synchronises, minus the loop's event time);
  * serial/N (N <= --serial-max): speech_stream of each text, one after another;
  * batch/N: inference_batch of the N texts, then generate_batch(mels, 11000, 550).
Wall times are host clocks that end in torch.cuda.synchronize().  The card's name and power limit are read in the same run."""
import argparse
import json
import os
import statistics
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from time_wavernn import DIMS, card  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--frames', type=int, default=200)
    ap.add_argument('--text-len', type=int, default=60)
    ap.add_argument('--streams', default='1,8,16,32,64')
    ap.add_argument('--ragged', type=int, default=64)
    ap.add_argument('--serial-max', type=int, default=8)
    ap.add_argument('--chunk', type=int, default=64)
    ap.add_argument('--modes', default='RAW,MOL')
    ap.add_argument('--rounds', type=int, default=2)
    ap.add_argument('--out', default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('time_stream_pool: no CUDA device')
    import __graft_entry__ as entry
    entry.build()
    from multilingual_text_to_speech_b200 import _lib
    from multilingual_text_to_speech_b200 import functional as F
    from multilingual_text_to_speech_b200.params.params import Params as hp
    from multilingual_text_to_speech_b200.modules import wavernn as W
    from multilingual_text_to_speech_b200.modules.tacotron2 import Decoder, Tacotron
    from multilingual_text_to_speech_b200.modules.streaming import speech_stream, speech_streams
    hp.reset()
    hp.max_output_length = 2 * a.frames if a.ragged else a.frames
    torch.manual_seed(0)
    taco = Tacotron().cuda().eval()
    with torch.no_grad():
        taco._decoder._stop_prediction.bias.fill_(-1e4)
    g = torch.Generator().manual_seed(1)
    Nmax = max([int(n) for n in a.streams.split(',')] + [a.ragged])
    texts = [torch.randint(3, hp.symbols_count() + 3, (a.text_len,), generator=g).cuda() for _ in range(Nmax)]
    hop, sr = DIMS['hop_length'], DIMS['sample_rate']
    StopRule = Decoder._StopRule

    class CutRule(StopRule):
        """The stop rule with a given cut: the decoder makes one per text, in text order."""
        def __init__(self, stop_frames):
            super().__init__(stop_frames)
            self.at = lengths[CutRule.made % len(lengths)]
            CutRule.made += 1

        def feed(self, logits):
            self.seen += int(logits.numel())
            if self.cut is None and self.seen >= self.at:
                self.cut = self.at
            return self.cut

    loop_events, run_walls = [], []
    orig_loops, orig_run = (F.wavernn_run_rows, F.wavernn_run_stream), W.StreamPool.run

    def timed(loop, nsteps_arg):
        def call(*args):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            loop(*args)
            e1.record()
            loop_events.append((e0, e1, int(args[nsteps_arg])))
        return call

    def pool_run(self):
        t0 = time.perf_counter()
        out = orig_run(self)
        run_walls.append(time.perf_counter() - t0)
        return out
    F.wavernn_run_rows, F.wavernn_run_stream, W.StreamPool.run = timed(F.wavernn_run_rows, 5), timed(F.wavernn_run_stream, 4), pool_run

    rows = []
    for mode in a.modes.split(','):
        torch.manual_seed(2)
        voc = W.WaveRNN(**dict(DIMS, mode=mode)).cuda().eval()
        cases = [(int(n), False) for n in a.streams.split(',')] + ([(a.ragged, True)] if a.ragged else [])
        for N, ragged in cases:
            lengths = [21 + (i * 37) % (2 * a.frames - 20) for i in range(N)] if ragged else [a.frames] * N
            tag = f'{N}ragged' if ragged else f'{N}'
            arms = [f'pool/{tag}', f'batch/{tag}'] + ([f'serial/{tag}'] if N <= a.serial_max else [])
            audio = [(f - 1) * hop / sr for f in lengths]

            def run(arm):
                CutRule.made = 0
                Decoder._StopRule = CutRule
                try:
                    return run_arm(arm)
                finally:
                    Decoder._StopRule = StopRule

            def run_arm(arm):
                loop_events.clear()
                run_walls.clear()
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                stamps = {i: [] for i in range(N)}
                if arm.startswith('pool/'):
                    for i, w in speech_streams(taco, voc, texts[:N], chunk_frames=a.chunk):
                        stamps[i].append(time.perf_counter() - t0)        # run() ends in a synchronising read
                elif arm.startswith('serial/'):
                    for i in range(N):
                        for w in speech_stream(taco, voc, texts[i], chunk_frames=a.chunk):
                            torch.cuda.synchronize()
                            stamps[i].append(time.perf_counter() - t0)
                else:
                    mels = taco.inference_batch(texts[:N], max_batch=N)
                    voc.generate_batch(mels, 11000, 550)
                    torch.cuda.synchronize()
                    for i in range(N):
                        stamps[i].append(time.perf_counter() - t0)
                total = time.perf_counter() - t0
                loop_ms = sum(e0.elapsed_time(e1) for e0, e1, _ in loop_events)
                steps = sum(n for *_, n in loop_events)
                return dict(total=total, stamps=stamps, loop_ms=loop_ms, steps=steps, runs=len(run_walls), run_wall=sum(run_walls))

            for arm in arms:
                run(arm)                 # warm-up
            res = {arm: [] for arm in arms}
            for _ in range(a.rounds):
                for arm in arms:
                    res[arm].append(run(arm))
            for arm in arms:
                rs = res[arm]
                rtf = [max(s[-1] for s in r['stamps'].values()) / max(audio) for r in rs]
                worst_rtf = [max(s[-1] / audio[i] for i, s in r['stamps'].items()) for r in rs]
                first = [max(s[0] for s in r['stamps'].values()) for r in rs]
                gaps = [max((t1 - t0 for s in r['stamps'].values() for t0, t1 in zip(s, s[1:])), default=0.0) for r in rs]
                row = dict(mode=mode, arm=arm, streams=N, ragged=ragged, rtf_worst_stream=statistics.median(worst_rtf), rtf_last=statistics.median(rtf),
                           first_audio_worst_s=statistics.median(first), gap_max_s=statistics.median(gaps),
                           audio_s_per_s=statistics.median([sum(audio) / r['total'] for r in rs]),
                           total_s=statistics.median([r['total'] for r in rs]), total_spread_s=max(r['total'] for r in rs) - min(r['total'] for r in rs))
                if arm.startswith('pool/'):
                    r = rs[-1]
                    row.update(us_per_step=1e3 * r['loop_ms'] / max(r['steps'], 1), runs=r['runs'],
                               host_ms_per_run=(r['run_wall'] * 1e3 - r['loop_ms']) / max(r['runs'], 1))
                rows.append(row)
                print(json.dumps(row), flush=True)
    (F.wavernn_run_rows, F.wavernn_run_stream), W.StreamPool.run = orig_loops, orig_run
    real_time = {}
    for r in rows:
        if r['arm'].startswith('pool/') and not r['ragged'] and r['rtf_worst_stream'] < 1:
            real_time[r['mode']] = max(real_time.get(r['mode'], 0), r['streams'])
    out = dict(card=card(), frames=a.frames, chunk=a.chunk, rounds=a.rounds, largest_real_time_pool=real_time, rows=rows)
    print(json.dumps({k: v for k, v in out.items() if k != 'rows'}))
    if a.out:
        with open(a.out, 'w') as f:
            json.dump(out, f, indent=1)
    _lib.set_precision('fp32')


if __name__ == '__main__':
    main()
