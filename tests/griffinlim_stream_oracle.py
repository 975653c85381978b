"""numpy restatement of streaming Griffin-Lim (RTISI-LA) as DESIGN ("Griffin-Lim vocoder", "Streaming") specifies it, the yardstick of
tests/test_griffinlim_stream_cpu.py and tests/test_gpu_griffinlim_stream.py.  Built on audio_oracle (window, window sum-square, the rfft
conventions).  dtype=np.float64 computes in fp64; np.float32 mirrors the kernel's fp32 roundings at the stage boundaries (fp32 signals and
envelopes summed in the kernel's order, complex64 spectra, single-precision FFTs).  No de-emphasis: the tests apply scipy's lfilter to the
output."""
import numpy as np
import scipy.fft

import audio_oracle as O


class Stream:
    """One stream: feed() magnitude frames [K, n], end(), run() -> the samples released by processing every ready frame."""

    def __init__(self, n_fft, hop, win, lookahead=3, iters=32, dtype=np.float64):
        self.N, self.H, self.k, self.I, self.dt = n_fft, hop, lookahead, iters, dtype
        self.w = O.hann(win, n_fft).astype(dtype)
        self.w2 = (self.w * self.w).astype(dtype)
        self.S = []                          # magnitudes of the frames received, [K] each
        self.c = np.zeros(n_fft, dtype)      # committed overlap-add over the untrimmed signal (grows)
        self.x = {}                          # look-ahead set: frame -> w * x_j
        self.m = 0                           # frames committed
        self.rel = 0                         # output samples released
        self.ended = False
        self.env = {}                        # one-sided envelope over frame j's span, by min(j, ceil((N - 1) / hop))

    @property
    def frames(self):
        return len(self.S)

    def feed(self, S):
        S = np.asarray(S)
        self.S += [S[:, t].astype(self.dt) for t in range(S.shape[1])]

    def end(self):
        assert self.frames >= 2
        self.ended = True

    def _sumsquare(self, z, last):
        """sum_{0 <= i <= last} w^2(z - i hop) at the samples z, in ascending i (the kernel's order)."""
        e = np.zeros(len(z), self.dt)
        for i in range(max(0, -(-(int(z.min()) - self.N + 1) // self.H)), min(last, int(z.max()) // self.H) + 1):
            d = z - i * self.H
            ok = (d >= 0) & (d < self.N)
            e[ok] = (e[ok] + self.w2[d[ok]]).astype(self.dt)
        return e

    def _p(self, j, upto):
        """w * p_j: (c + the overlap-add of the frames of the look-ahead set before `upto`) / e over frame j's span (0 where e = 0)."""
        N, H = self.N, self.H
        z = j * H + np.arange(N)
        need = j * H + N
        if len(self.c) < need:
            self.c = np.concatenate([self.c, np.zeros(need - len(self.c), self.dt)])
        seg = self.c[j * H:j * H + N].copy()
        for q in sorted(self.x):
            if q >= upto:
                continue
            lo, hi = max(q * H, j * H), min(q * H + N, j * H + N)
            if lo < hi:
                seg[lo - j * H:hi - j * H] += self.x[q][lo - q * H:hi - q * H]
        key = min(j, -(-(N - 1) // H))        # the one-sided envelope over a frame's span is the same from here on
        if key not in self.env:
            self.env[key] = self._sumsquare(z, 1 << 40)
        e = self.env[key]
        p = np.where(e != 0, seg / np.where(e != 0, e, 1), 0).astype(self.dt)
        return (self.w * p).astype(self.dt)

    def _project(self, j, wp):
        X = scipy.fft.rfft(wp)
        mag = np.abs(X)
        ph = np.where(mag > 0, X / np.where(mag > 0, mag, 1), 1)
        if self.dt == np.float32:
            ph = ph.astype(np.complex64)
        y = scipy.fft.irfft((self.S[j] * ph).astype(ph.dtype), n=self.N)
        return (self.w * y.astype(self.dt)).astype(self.dt)

    def run(self):
        N, H, F = self.N, self.H, self.frames
        out = []
        while True:
            process = self.m < F and (self.m + self.k < F or self.ended)
            # lookahead 0: the last frame may be committed before the end is known; the run that learns of it releases the rest
            tail = not process and self.ended and self.m == F and self.rel < H * (F - 1)
            if not process and not tail:
                break
            m = self.m if process else F - 1
            if process:
                last = min(m + self.k, F - 1)
                for j in range(m, last + 1):
                    if j not in self.x:
                        self.x[j] = self._project(j, self._p(j, j))
                for _ in range(self.I):
                    ps = {j: self._p(j, F) for j in sorted(self.x)}
                    for j in sorted(ps):
                        self.x[j] = self._project(j, ps[j])
                self.c[m * H:m * H + N] = (self.c[m * H:m * H + N] + self.x.pop(m)).astype(self.dt)
            final = self.ended and m == F - 1
            rel_end = H * (F - 1) if final else max(0, (m + 1) * H - N // 2)
            if rel_end > self.rel:
                z = np.arange(self.rel, rel_end) + N // 2
                wss = self._sumsquare(z, m)
                v = self.c[z]
                big = wss > np.finfo(np.float32).tiny
                out.append(np.where(big, v / np.where(big, wss, 1), v).astype(self.dt))
                self.rel = rel_end
            if process:
                self.m += 1
        return np.concatenate(out) if out else np.zeros(0, self.dt)


def rtisi(S, n_fft, hop, win, lookahead=3, iters=32, dtype=np.float64):
    """The whole magnitude spectrogram S [K, F] at once -> hop (F - 1) samples."""
    st = Stream(n_fft, hop, win, lookahead, iters, dtype)
    st.feed(S)
    st.end()
    return st.run()


def rtisi_chunked(S, cuts, n_fft, hop, win, lookahead=3, iters=32, dtype=np.float64):
    """S fed in chunks ending at the frame indices `cuts` (ascending, the last F), run() after every feed, then end() and a last run()."""
    st = Stream(n_fft, hop, win, lookahead, iters, dtype)
    out, t0 = [], 0
    for t1 in cuts:
        st.feed(S[:, t0:t1])
        out.append(st.run())
        t0 = t1
    st.end()
    out.append(st.run())
    return np.concatenate(out)
