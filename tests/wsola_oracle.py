"""numpy oracle of WSOLA time-scale modification (utils.audio.time_stretch_batch / retime_batch, csrc/wsola.cu): the contract the kernels
are checked against.

One waveform x [L] at a time, read as 0 outside [0, L); output length L'; synthesis hop H (the mel hop), frame length N = 2H, tolerance
D (= H from Python).  There are K = (L' - 1) // H + 2 synthesis frames; frame k is centred on output sample kH and has an fp64 input
position tau_k (the warp).

1. Nominal positions a_k = rint(clamp(tau_k, 0, L)), half to even.
2. Search: p_0 = a_0.  For k >= 1, u_m = x[p_{k-1} + H + m] (the natural continuation of frame k - 1) and v_{d,m} = x[a_k + d + m] for m
   in [-H, H) and d in [-D, D].  C(d) = sum u v and E(d) = sum v^2, fp64 sums of the (exact) fp64 products of fp32 samples, accumulated
   one term at a time in increasing m.  s(d) = C / sqrt(E), and s = 0 where E = 0.  p_k = a_k + argmax s; on exact ties the smallest |d|
   wins, then the negative d.  At tau_k = kH, d = 0 is the Cauchy-Schwarz maximum, so y = x up to rounding, and silence copies the
   nominal positions.
3. Overlap-add: y[n] = sum over k in {n // H, n // H + 1} of w(n - kH + H) x[p_k + n - kH], fp64 in increasing k, rounded to fp32;
   w(i) = 0.5 - 0.5 cos(pi i / H) (periodic Hann of length 2H), and w(i) + w(i + H) = 1, so nothing is normalised.

Warps (Python):
- time stretch by `rate` (> 1 faster): L' = max(1, round(L / rate)), tau_k = k H rate.
- retime from durations d to d' (int frames per symbol, sum d = 1 + L // H): L' = max(1, H (sum d' - 1) + L mod H), so a spectrogram of y'
  has sum d' frames.  With B, B' the cumulative durations, symbol j's output interval [B'_j - 1/2, B'_{j+1} - 1/2) maps linearly onto
  [B_j - 1/2, B_{j+1} - 1/2) (phi, on frame coordinates); a symbol with d'_j = 0 is dropped, one with d_j = 0 holds its boundary, and past
  the last boundary the slope is 1.  tau_k = H phi(k); with d' = d, tau_k = kH exactly.
"""
import numpy as np
from numpy.lib.stride_tricks import sliding_window_view

MAX_HOP = 1024               # include/b200tts.h B200TTS_WSOLA_MAX_HOP
MAX_TOLERANCE = 1024         # include/b200tts.h B200TTS_WSOLA_MAX_TOLERANCE


def frames(Lp, H):
    return (Lp - 1) // H + 2


def stretch_warp(L, H, rate):
    """(L', tau fp64 [K]) of a time stretch by `rate`."""
    Lp = max(1, int(round(L / rate)))
    return Lp, np.array([k * H * rate for k in range(frames(Lp, H))], dtype=np.float64)


def retime_warp(L, H, d, dp):
    """(L', tau fp64 [K]) of a retime from durations d to dp."""
    d = [int(v) for v in d]
    dp = [int(v) for v in dp]
    assert len(d) == len(dp) and sum(d) == 1 + L // H and sum(dp) >= 1 and min(d + dp) >= 0
    Lp = max(1, H * (sum(dp) - 1) + L % H)
    B = np.concatenate([[0], np.cumsum(d)])
    Bp = np.concatenate([[0], np.cumsum(dp)])
    tau = []
    for k in range(frames(Lp, H)):
        j = next((j for j in range(len(d)) if Bp[j + 1] > k), None)       # the output interval that holds frame k
        if j is None:
            phi = (B[-1] - 0.5) + (k - (Bp[-1] - 0.5)) * 1.0 / 1.0
        else:
            phi = (B[j] - 0.5) + (k - (Bp[j] - 0.5)) * float(d[j]) / float(dp[j])
        tau.append(H * phi)
    return Lp, np.array(tau, dtype=np.float64)


def nominal(tau, L):
    return np.rint(np.clip(np.asarray(tau, dtype=np.float64), 0.0, float(L))).astype(np.int64)


def _padded(x, lo, n):
    """x[lo .. lo + n) as fp64, 0 outside [0, L)."""
    out = np.zeros(n)
    a, b = max(lo, 0), min(lo + n, len(x))
    if b > a:
        out[a - lo:b - lo] = x[a:b]
    return out


def search(x, a, p_prev, H, D):
    """-> (d of the best candidate, scores s [2D + 1]) for a frame at nominal position a after a frame placed at p_prev."""
    x = np.asarray(x, dtype=np.float32).astype(np.float64)
    u = _padded(x, p_prev, 2 * H)                            # u_m, m = -H .. H-1
    span = _padded(x, a - D - H, 2 * D + 2 * H)              # x[a - D - H ...]
    V = sliding_window_view(span, 2 * H)[:2 * D + 1]        # V[c, i] = v_{c - D, i - H}
    C = np.cumsum(u[None, :] * V, axis=1)[:, -1]             # one term at a time, in increasing m
    E = np.cumsum(V * V, axis=1)[:, -1]
    s = np.zeros(2 * D + 1)
    nz = E > 0
    s[nz] = C[nz] / np.sqrt(E[nz])
    d = np.arange(-D, D + 1)
    best = max(range(2 * D + 1), key=lambda c: (s[c], -abs(d[c]), -d[c]))
    return int(d[best]), s


def positions(x, tau, H, D):
    """-> p int64 [K] for the warp tau [K]."""
    a = nominal(tau, len(x))
    p = np.empty(len(a), dtype=np.int64)
    p[0] = a[0]
    for k in range(1, len(a)):
        p[k] = a[k] + search(x, int(a[k]), int(p[k - 1]), H, D)[0]
    return p


def window(H):
    return 0.5 - 0.5 * np.cos(np.pi * np.arange(2 * H) / H)


def overlap_add(x, p, H, Lp):
    """-> y float64 [L'] (the contract rounds it to fp32) from the frame positions p [K]."""
    x = np.asarray(x, dtype=np.float32).astype(np.float64)
    w = window(H)
    y = np.zeros(Lp)
    for n in range(Lp):
        for k in (n // H, n // H + 1):
            if k < len(p):
                s = int(p[k]) + n - k * H
                y[n] += w[n - k * H + H] * (x[s] if 0 <= s < len(x) else 0.0)
    return y


def overlap_add_fast(x, p, H, Lp):
    """overlap_add vectorised over n: the same two terms per sample, added in the same order."""
    x = np.asarray(x, dtype=np.float32).astype(np.float64)
    w = window(H)
    n = np.arange(Lp)
    y = np.zeros(Lp)
    for j in (0, 1):
        k = n // H + j
        ok = k < len(p)
        s = np.where(ok, p[np.minimum(k, len(p) - 1)] + n - k * H, -1)
        xs = np.where((s >= 0) & (s < len(x)), x[np.clip(s, 0, len(x) - 1)], 0.0)
        y = y + np.where(ok, w[n - k * H + H] * xs, 0.0)
    return y


def time_stretch(x, rate, H, D=None):
    """The whole contract on one waveform: (y float64 [L'], p [K], tau [K])."""
    Lp, tau = stretch_warp(len(x), H, rate)
    p = positions(x, tau, H, H if D is None else D)
    return overlap_add_fast(x, p, H, Lp), p, tau


def retime(x, d, dp, H, D=None):
    """(y float64 [L'], p [K], tau [K]) of a retime from durations d to dp."""
    Lp, tau = retime_warp(len(x), H, d, dp)
    p = positions(x, tau, H, H if D is None else D)
    return overlap_add_fast(x, p, H, Lp), p, tau
