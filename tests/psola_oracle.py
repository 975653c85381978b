"""numpy oracle of TD-PSOLA pitch shifting (utils.audio.pitch_shift_batch, csrc/psola.cu): the contract the kernels are checked against.

One waveform x [L] at a time, with an F0 track f0 [F] (Hz, NaN unvoiced) and a ratio track r [F] on the mel frames, F = 1 + L // hop;
sample n belongs to frame min(F - 1, (n + hop // 2) // hop) and is voiced when that frame's f0 is not NaN, with period
P(n) = rint(sr / f0) in fp64 (half to even).  U = hop is the mark spacing of unvoiced regions.

1. Analysis marks m_0 < m_1 < ... in [0, L) with voiced flags: m_0 = argmax x over [0, min(L, P(0))) when sample 0 is voiced, else 0.
   From a voiced mark (p = P(m)): c = m + p, stop when c >= L; the next mark is argmax x over [c - p//4, min(L - 1, c + p//4)] when c is
   voiced, else c.  From an unvoiced mark, o = the first voiced sample after it (L if none): the next mark is m + U when m + U < o (stop
   when that is >= L), else argmax x over [o, min(L, o + P(o))) (stop when o = L).  argmax: signed x, first index on ties.
   d_k = m_{k+1} - m_k; the last mark's d is its nominal period (P when voiced, U when not).
2. Synthesis marks t_0 = m_0, t_{j+1} = t_j + q_j in fp64, centres c_j = rint(t_j), until c_j >= L.  k(j) is the analysis mark nearest c_j
   (the lower one on ties); q_j = d_k / r[frame(c_j)] when mark k is voiced, else d_k.
3. Overlap-add: grain j takes x around m = m_{k(j)} and adds it around c_j with half-widths a = d_{k-1} (left) and b = d_k (right), weight
   w(u) = (1 + cos(pi u / (a + 1))) / 2 for -a <= u <= 0 and (1 + cos(pi u / (b + 1))) / 2 for 0 <= u <= b; the left half of mark 0's
   grains and the right half of the last mark's grains weigh 1 (the signal is not tapered before the first mark or after the last).
   y(n) = sum_j w x[m + n - c_j] / max(1, sum_j w) over the grains whose support holds n and whose source index lies in [0, L), both sums
   fp64 in increasing j; y = 0 where no grain covers n.  |y| <= max |x|: a convex combination where the weights sum to 1 or more, a
   shrunk one where they do not.
   Two details differ from a plain normalised overlap-add, each for a reason:
   - max(1, sum w), not sum w: dividing by the weight sum erases the window wherever only one grain covers a sample, so below r = 1 the
     output is a splice of the input, and at r = 0.5 the splices fall exactly two periods apart and the pitch does not move at all (a
     tone re-tracks at its source F0, 1,200 cents from the target).  Where grains overlap enough (r >= 1, and r = 1 exactly, where the
     two windows about every sample sum to at least 1) the two are the same.
   - Grain 0's left half-width is max(nominal period of mark 0, m_0), not the nominal period alone: when sample 0 is voiced, m_0 can lie
     in a later frame whose period is shorter than m_0, and the samples before m_0 - P(m_0) would otherwise belong to no grain.  With it
     and the untapered outer halves, y = x at r = 1 whatever the tracks are.
"""
import numpy as np

MAX_PERIOD = 1024              # include/b200tts.h B200TTS_PSOLA_MAX_PERIOD
MIN_RATIO, MAX_RATIO = 0.5, 2.0


def frame_of(n, hop, F):
    return min(F - 1, (n + hop // 2) // hop)


def periods(f0, sr):
    """Per-frame periods rint(sr / f0) in fp64 from the fp32 track, 0 on unvoiced frames."""
    f = np.asarray(f0, dtype=np.float32).astype(np.float64)
    out = np.zeros(len(f), dtype=np.int64)
    v = ~np.isnan(f)
    out[v] = np.rint(sr / f[v]).astype(np.int64)
    return out


def _argmax(x, lo, hi):
    """First index of the maximum of x[lo .. hi] (inclusive)."""
    return lo + int(np.argmax(x[lo:hi + 1]))


def analysis_marks(x, f0, sr, hop):
    """-> (marks int64 [K], spacings d int64 [K], voiced bool [K], left half-width of grain 0)."""
    L = len(x)
    F = 1 + L // hop
    assert len(f0) == F, (len(f0), F)
    Pf = periods(f0, sr)
    P = lambda n: int(Pf[frame_of(n, hop, F)])         # noqa: E731
    U = hop
    x = np.asarray(x, dtype=np.float32)
    marks, voiced = [], []
    m = _argmax(x, 0, min(L, P(0)) - 1) if P(0) else 0
    while True:
        p = P(m)
        marks.append(m)
        voiced.append(p > 0)
        if p:
            c = m + p
            if c >= L:
                break
            m = _argmax(x, c - p // 4, min(L - 1, c + p // 4)) if P(c) else c
        else:
            o = m + 1
            while o < L and not P(o):
                o += 1
            if m + U < o:
                if m + U >= L:
                    break
                m = m + U
            else:
                if o >= L:
                    break
                m = _argmax(x, o, min(L, o + P(o)) - 1)
    marks = np.array(marks, dtype=np.int64)
    voiced = np.array(voiced, dtype=bool)
    d = np.empty_like(marks)
    d[:-1] = np.diff(marks)
    d[-1] = P(int(marks[-1])) if voiced[-1] else U
    a0 = max(int(P(int(marks[0])) if voiced[0] else U), int(marks[0]))
    return marks, d, voiced, a0


def synthesis_marks(L, marks, d, voiced, ratio, hop):
    """-> (centres c int64 [J], nearest analysis mark k int64 [J])."""
    F = 1 + L // hop
    r = np.asarray(ratio, dtype=np.float32).astype(np.float64)
    assert len(r) == F
    K = len(marks)
    t = float(marks[0])
    k = 0
    cs, ks = [], []
    while True:
        c = int(np.rint(t))
        if c >= L:
            break
        while k + 1 < K and marks[k] + marks[k + 1] < 2 * c:
            k += 1
        cs.append(c)
        ks.append(k)
        q = float(d[k]) / r[frame_of(c, hop, F)] if voiced[k] else float(d[k])
        t = t + q
    return np.array(cs, dtype=np.int64), np.array(ks, dtype=np.int64)


def overlap_add(x, marks, d, a0, c, k):
    """-> (y float64 [L], weight sum float64 [L])."""
    K = len(marks)
    x = np.asarray(x, dtype=np.float32).astype(np.float64)
    L = len(x)
    num = np.zeros(L)
    den = np.zeros(L)
    for j in range(len(c)):
        kk = int(k[j])
        m = int(marks[kk])
        a = a0 if kk == 0 else int(d[kk - 1])
        b = int(d[kk])
        u = np.arange(-a, b + 1)
        n = c[j] + u
        s = m + u
        ok = (n >= 0) & (n < L) & (s >= 0) & (s < L)
        u, n, s = u[ok], n[ok], s[ok]
        w = np.where(u <= 0, 0.5 * (1.0 + np.cos(np.pi * u / (a + 1))), 0.5 * (1.0 + np.cos(np.pi * u / (b + 1))))
        if kk == 0:
            w[u <= 0] = 1.0
        if kk == K - 1:
            w[u >= 0] = 1.0
        num[n] += w * x[s]
        den[n] += w
    return num / np.maximum(den, 1.0), den


def pitch_shift(x, f0, ratio, sr, hop):
    """The whole contract on one waveform: (y float64 [L], a dict of the intermediate marks)."""
    marks, d, voiced, a0 = analysis_marks(x, f0, sr, hop)
    c, k = synthesis_marks(len(x), marks, d, voiced, ratio, hop)
    y, den = overlap_add(x, marks, d, a0, c, k)
    return y, dict(marks=marks, d=d, voiced=voiced, a0=a0, c=c, k=k, den=den)
