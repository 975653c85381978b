"""Time continuous-batching synthesis (modules/streaming.py: SpeechServer) against a group-at-a-time dispatcher on an open-loop request
trace, at the reference's dimensions with random weights and seeded texts.

    python tools/time_speech_server.py [--rates 2,8,16] [--requests 32] [--frames 200] [--text-len 60] [--chunk 64] [--modes RAW,MOL]
                                       [--rounds 1] [--seed 0] [--out FILE]

Workload: for each rate, a seeded Poisson arrival trace of --requests requests (exponential gaps of mean 1 / rate s).  Request i's text
is --text-len random symbols and cuts at 21 + (i * 37) % (2 --frames - 20) frames (the ragged mix of DESIGN §10.2: 21 to 400 frames at the
default --frames 200, through the decoder's stop rule; the stop token itself never fires).  Arms, replaying the same trace, alternated
round by round after one warm-up of each:
  * server: one SpeechServer(max_streams=64); a request is submitted at its arrival time and every step() runs one decoder call and one
    vocoder call over everything admitted;
  * server-folded: the server arm with target=11000, overlap=550: folded vocoding (the library's default, generate_batch's), each
    request's folds running as rows of the shared 64-row loop;
  * groups: each time the previous group has ended, one speech_streams group of whatever has arrived (at most 64), run to its end.
Per request: queueing delay (arrival to admission), time to first audio and RTF from arrival (time to its last chunk / its audio
duration), and the largest gap between its chunks; p50, p95 and max over the trace.  Overall: audio-seconds per wall second (trace start
to last chunk).  Server arm only: wall time per DecoderPool.run() by the number of open rows, and the cost of a join (the encoder and
re-padding of the calls that admit texts: DecoderPool._admit).  Times are host clocks; each ends in torch.cuda.synchronize() or in a
call that synchronises.  The card's name and power limit are read in the same run."""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ARMS = ('server', 'server-folded', 'groups')


def parse_args(argv=None):
    ap = argparse.ArgumentParser()
    ap.add_argument('--rates', default='2,8,16')
    ap.add_argument('--requests', type=int, default=32)
    ap.add_argument('--frames', type=int, default=200)
    ap.add_argument('--text-len', type=int, default=60)
    ap.add_argument('--chunk', type=int, default=64)
    ap.add_argument('--modes', default='RAW,MOL')
    ap.add_argument('--rounds', type=int, default=1)
    ap.add_argument('--seed', type=int, default=0)
    ap.add_argument('--out', default=None)
    a = ap.parse_args(argv)
    a.rates = [float(r) for r in a.rates.split(',')]
    a.modes = a.modes.split(',')
    if a.requests < 1 or a.frames < 21 or a.text_len < 1 or a.chunk < 1 or a.rounds < 1 or any(r <= 0 for r in a.rates):
        ap.error('requests, frames (>= 21), text-len, chunk, rounds and rates must be positive')
    return a


def make_trace(rate, n, frames, seed):
    """[(arrival s, cut frames)] of n requests: Poisson arrivals at `rate` per second from t = 0, request i cutting at 21 + 37 i mod
    (2 frames - 20) frames."""
    gaps = np.random.default_rng(seed).exponential(1.0 / rate, n)
    arrivals = np.concatenate([[0.0], np.cumsum(gaps[1:])])
    return [(float(t), 21 + (i * 37) % (2 * frames - 20)) for i, t in enumerate(arrivals)]


def percentiles(xs):
    xs = np.asarray(xs, dtype=np.float64)
    return dict(p50=float(np.percentile(xs, 50)), p95=float(np.percentile(xs, 95)), max=float(xs.max()))


def main(argv=None):
    a = parse_args(argv)
    import torch
    if not torch.cuda.is_available():
        raise SystemExit('time_speech_server: no CUDA device')
    sys.path.insert(0, ROOT)
    sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
    import __graft_entry__ as entry
    entry.build()
    from time_wavernn import DIMS, card
    from multilingual_text_to_speech_b200 import _lib
    from multilingual_text_to_speech_b200.params.params import Params as hp
    from multilingual_text_to_speech_b200.modules import tacotron2 as T
    from multilingual_text_to_speech_b200.modules.wavernn import WaveRNN
    from multilingual_text_to_speech_b200.modules.streaming import SpeechServer, speech_streams
    hp.reset()
    hp.max_output_length = 2 * a.frames
    torch.manual_seed(0)
    taco = T.Tacotron().cuda().eval()
    with torch.no_grad():
        taco._decoder._stop_prediction.bias.fill_(-1e4)
    g = torch.Generator().manual_seed(1)
    texts = [torch.randint(3, hp.symbols_count() + 3, (a.text_len,), generator=g).cuda() for _ in range(a.requests)]
    hop, sr = DIMS['hop_length'], DIMS['sample_rate']
    StopRule = T.Decoder._StopRule
    cuts = []

    class CutRule(StopRule):
        """The stop rule with a given cut: the decoder makes one per text in admission order, which is arrival order in both arms."""
        def __init__(self, stop_frames):
            super().__init__(stop_frames)
            self.at = cuts[CutRule.made]
            CutRule.made += 1

        def feed(self, logits):
            self.seen += int(logits.numel())
            if self.cut is None and self.seen >= self.at:
                self.cut = self.at
            return self.cut

    dec_runs, joins = [], []
    orig_run, orig_admit = T.DecoderPool.run, T.DecoderPool._admit

    def pool_run(self):
        n = len(self.ids)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        out = orig_run(self)
        torch.cuda.synchronize()
        dec_runs.append((n, time.perf_counter() - t0))
        return out

    def admit(self):
        n = len(self.queue)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        orig_admit(self)
        torch.cuda.synchronize()
        joins.append((n, time.perf_counter() - t0))

    def serve(voc, trace, folded=False):
        server = SpeechServer(taco, voc, 64, None, a.chunk, target=11000 if folded else None, overlap=550 if folded else None)
        n, ids, stamps, admitted = len(trace), {}, {i: [] for i in range(len(trace))}, {}
        nxt = 0
        t0 = time.perf_counter()
        while nxt < n or server.pending or server.active:
            now = time.perf_counter() - t0
            while nxt < n and trace[nxt][0] <= now:
                ids[server.submit(texts[nxt])] = nxt
                nxt += 1
            if not server.pending and not server.active:
                time.sleep(max(trace[nxt][0] - now, 0.0))
                continue
            start = time.perf_counter() - t0
            waiting = list(server.pending)
            out = server.step()
            for rid in waiting:
                if rid not in server.pending:
                    admitted[ids[rid]] = start
            t = time.perf_counter() - t0                  # step() ends in the pool's synchronising abort-flag read
            for rid in out:
                stamps[ids[rid]].append(t)
        assert not server.failed, server.failed
        return stamps, admitted

    def groups(voc, trace):
        n, stamps, admitted, nxt = len(trace), {i: [] for i in range(len(trace))}, {}, 0
        t0 = time.perf_counter()
        while nxt < n:
            now = time.perf_counter() - t0
            if trace[nxt][0] > now:
                time.sleep(trace[nxt][0] - now)
                continue
            group = [i for i in range(nxt, n) if trace[i][0] <= now][:64]
            nxt = group[-1] + 1
            for i in group:
                admitted[i] = now
            for j, _ in speech_streams(taco, voc, [texts[i] for i in group], chunk_frames=a.chunk):
                stamps[group[j]].append(time.perf_counter() - t0)
        return stamps, admitted

    def run(arm, voc, trace):
        cuts[:] = [c for _, c in trace]
        CutRule.made = 0
        T.Decoder._StopRule = CutRule
        T.DecoderPool.run, T.DecoderPool._admit = pool_run, admit
        dec_runs.clear()
        joins.clear()
        try:
            torch.cuda.synchronize()
            stamps, admitted = groups(voc, trace) if arm == 'groups' else serve(voc, trace, arm == 'server-folded')
        finally:
            T.Decoder._StopRule = StopRule
            T.DecoderPool.run, T.DecoderPool._admit = orig_run, orig_admit
        arrival = [t for t, _ in trace]
        audio = [(c - 1) * hop / sr for _, c in trace]
        end = max(s[-1] for s in stamps.values())
        return dict(queue=[admitted[i] - arrival[i] for i in stamps], first=[s[0] - arrival[i] for i, s in stamps.items()],
                    gap=[max((y - x for x, y in zip(s, s[1:])), default=0.0) for s in stamps.values()],
                    rtf=[(s[-1] - arrival[i]) / audio[i] for i, s in stamps.items()], audio_per_s=sum(audio) / end,
                    dec_runs=list(dec_runs), joins=list(joins))

    rows = []
    for mode in a.modes:
        torch.manual_seed(2)
        voc = WaveRNN(**dict(DIMS, mode=mode)).cuda().eval()
        warm = make_trace(64.0, 8, a.frames, a.seed + 1000)
        for arm in ARMS:
            run(arm, voc, warm)
        for rate in a.rates:
            trace = make_trace(rate, a.requests, a.frames, a.seed)
            res = {arm: [] for arm in ARMS}
            for _ in range(a.rounds):
                for arm in ARMS:
                    res[arm].append(run(arm, voc, trace))
            for arm, rs in res.items():
                pool = lambda k: [x for r in rs for x in r[k]]       # noqa: E731 -- every request of every round
                row = dict(mode=mode, arm=arm, rate=rate, requests=a.requests, queue_s=percentiles(pool('queue')),
                           first_audio_s=percentiles(pool('first')), gap_s=percentiles(pool('gap')), rtf=percentiles(pool('rtf')),
                           audio_s_per_s=float(np.median([r['audio_per_s'] for r in rs])))
                if arm != 'groups':
                    runs = pool('dec_runs')
                    row['decoder_run_ms'] = {f'{lo}-{hi}': round(1e3 * float(np.median([t for n, t in runs if lo <= n <= hi])), 2)
                                             for lo, hi in ((1, 8), (9, 16), (17, 32), (33, 64)) if any(lo <= n <= hi for n, _ in runs)}
                    js = pool('joins')
                    row['join_ms'] = dict(p50=round(1e3 * float(np.median([t for _, t in js])), 2), max=round(1e3 * max(t for _, t in js), 2),
                                          texts_per_join=float(np.mean([n for n, _ in js])))
                rows.append(row)
                print(json.dumps(row), flush=True)
    out = dict(card=card(), frames=a.frames, text_len=a.text_len, chunk=a.chunk, requests=a.requests, rounds=a.rounds, rows=rows)
    print(json.dumps({k: v for k, v in out.items() if k != 'rows'}))
    if a.out:
        with open(a.out, 'w') as f:
            json.dump(out, f, indent=1)
    _lib.set_precision('fp32')


if __name__ == '__main__':
    main()
