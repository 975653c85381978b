"""numpy restatement of librosa 0.10's librosa.pyin, the yardstick of the pitch kernels (csrc/pitch.cu).

librosa cannot be installed where this project is built and tested, so this module IS the specification the kernels are checked against:
it restates librosa 0.10.x's pyin, _cumulative_mean_normalized_difference, _parabolic_interpolation, __pyin_helper, localmin,
transition_local, transition_loop and sequence.viterbi with librosa's expressions, in the same order, at librosa's defaults for everything
pitch_batch does not expose.  Agreement with librosa itself is unverified.

Beside the definitions it has a direct O(N^2) evaluation of the difference function, and a banded Viterbi that takes the best in-band
predecessor of each half plus the best out-of-band one (prefix and suffix maxima), which the kernel implements; the CPU tests check both
against the definitions.
"""
import itertools

import numpy as np
import scipy.signal
import scipy.stats

TINY = np.finfo(np.float64).tiny
N_THRESHOLDS = 100
BETA = (2, 18)
BOLTZMANN = 2
BINS_PER_SEMITONE = 10
MAX_TRANSITION_RATE = 35.92
SWITCH_PROB = 0.01
NO_TROUGH_PROB = 0.01


def geometry(sr, hop, fmin, fmax, frame_length):
    win = frame_length // 2
    min_period = int(np.floor(sr / fmax))
    max_period = min(int(np.ceil(sr / fmin)), frame_length - win - 1)
    n_bins = int(np.floor(12 * BINS_PER_SEMITONE * np.log2(fmax / fmin))) + 1
    width = round(MAX_TRANSITION_RATE * 12 * hop / sr) * BINS_PER_SEMITONE + 1
    return dict(win_length=win, min_period=min_period, max_period=max_period, n_bins=n_bins, transition_width=width)


def frames(y, frame_length, hop):
    """center=True with zero padding of frame_length // 2, then util.frame: [frame_length, F] float64."""
    y = np.pad(np.asarray(y, dtype=np.float64), (frame_length // 2, frame_length // 2), mode='constant')
    F = 1 + (len(y) - frame_length) // hop
    idx = np.arange(frame_length)[:, None] + hop * np.arange(F)[None, :]
    return y[idx]


def cmnd(y_frames, frame_length, win_length, min_period, max_period):
    """librosa's _cumulative_mean_normalized_difference (FFT autocorrelation): [K, F]."""
    a = np.fft.rfft(y_frames, frame_length, axis=-2)
    b = np.fft.rfft(y_frames[..., win_length:0:-1, :], frame_length, axis=-2)
    acf = np.fft.irfft(a * b, frame_length, axis=-2)[..., win_length:, :]
    acf[np.abs(acf) < 1e-6] = 0
    energy = np.cumsum(y_frames ** 2, axis=-2)
    energy = energy[..., win_length:, :] - energy[..., :-win_length, :]
    energy[np.abs(energy) < 1e-6] = 0
    yin = energy[..., :1, :] + energy - 2 * acf
    numerator = yin[..., min_period:max_period + 1, :]
    tau = np.arange(1, max_period + 1)[:, None]
    cumulative_mean = np.cumsum(yin[..., 1:max_period + 1, :], axis=-2) / tau
    denominator = cumulative_mean[..., min_period - 1:max_period, :]
    return numerator / (denominator + TINY)


def difference_terms(y_frames, win_length, max_period):
    """(acf, e) [max_period + 1, F] by the direct sums of the header's formulas, before the 1e-6 zeroing."""
    acf = np.empty((max_period + 1, y_frames.shape[1]))
    e = np.empty_like(acf)
    for tau in range(max_period + 1):
        acf[tau] = np.sum(y_frames[1:win_length + 1] * y_frames[1 + tau:win_length + 1 + tau], axis=0)
        e[tau] = np.sum(y_frames[tau + 1:tau + win_length + 1] ** 2, axis=0)
    return acf, e


def cmnd_direct(y_frames, win_length, min_period, max_period):
    """The same d' from the direct O(N^2) sums."""
    acf, e = difference_terms(y_frames, win_length, max_period)
    acf[np.abs(acf) < 1e-6] = 0
    e[np.abs(e) < 1e-6] = 0
    d = e[:1] + e - 2 * acf
    out = np.empty((max_period - min_period + 1, y_frames.shape[1]))
    for k, tau in enumerate(range(min_period, max_period + 1)):
        out[k] = d[tau] / (np.sum(d[1:tau + 1], axis=0) / tau + TINY)
    return out


def parabolic_shifts(x):
    """librosa's _parabolic_interpolation over axis 0 of [K, F]."""
    a = x[2:] + x[:-2] - 2 * x[1:-1]
    b = (x[2:] - x[:-2]) / 2
    shifts = np.zeros_like(x)
    with np.errstate(divide='ignore', invalid='ignore'):
        inner = -b / a
    inner[np.abs(b) >= np.abs(a)] = 0
    shifts[1:-1] = inner
    return shifts


def localmin(x):
    """librosa.util.localmin over a 1-D array (edge padding)."""
    xp = np.pad(x, (1, 1), mode='edge')
    return (x < xp[:-2]) & (x <= xp[2:])


def thresholds_and_beta():
    thresholds = np.linspace(0, 1, N_THRESHOLDS + 1)
    return thresholds, np.diff(scipy.stats.beta.cdf(thresholds, BETA[0], BETA[1]))


def troughs(frame):
    is_trough = localmin(frame)
    is_trough[0] = frame[0] < frame[1]
    return np.nonzero(is_trough)[0]


def observations(yin, shifts, sr, fmin, min_period, n_bins):
    """librosa's __pyin_helper: (observation probabilities [2 n, F], voiced_prob [F])."""
    thresholds, beta_probs = thresholds_and_beta()
    yin_probs = np.zeros_like(yin)
    for i, frame in enumerate(yin.T):
        trough_index = troughs(frame)
        if len(trough_index) == 0:
            continue
        heights = frame[trough_index]
        below = np.less.outer(heights, thresholds[1:])
        positions = np.cumsum(below, axis=0) - 1
        n_troughs = np.count_nonzero(below, axis=0)
        with np.errstate(divide='ignore', invalid='ignore'):
            prior = scipy.stats.boltzmann.pmf(positions, BOLTZMANN, n_troughs)
        prior[~below] = 0
        probs = prior.dot(beta_probs)
        global_min = np.argmin(heights)
        n_below_min = np.count_nonzero(~below[global_min, :])
        probs[global_min] += NO_TROUGH_PROB * np.sum(beta_probs[:n_below_min])
        yin_probs[trough_index, i] = probs
    period, frame_index = np.nonzero(yin_probs)
    candidates = min_period + period + shifts[period, frame_index]
    f0 = sr / candidates
    bins = 12 * BINS_PER_SEMITONE * np.log2(f0 / fmin)
    bins = np.clip(np.round(bins), 0, n_bins).astype(int)
    obs = np.zeros((2 * n_bins, yin.shape[1]))
    obs[bins, frame_index] = yin_probs[period, frame_index]
    voiced_prob = np.clip(np.sum(obs[:n_bins, :], axis=0, keepdims=True), 0, 1)
    obs[n_bins:, :] = (1 - voiced_prob) / n_bins
    return obs, voiced_prob[0]


def transition_local(n, width):
    """librosa.sequence.transition_local(n, width, window='triangle', wrap=False)."""
    window = scipy.signal.get_window('triangle', width, fftbins=False)
    lpad = (n - width) // 2
    padded = np.pad(window, (lpad, n - width - lpad))
    T = np.zeros((n, n))
    for i in range(n):
        row = np.roll(padded, n // 2 + i + 1)
        row[min(n, i + width // 2 + 1):] = 0
        row[:max(0, i - width // 2)] = 0
        T[i] = row
    T /= T.sum(axis=1, keepdims=True)
    return T


def transition(n, width):
    """kron(transition_loop(2, 1 - switch_prob), transition_local(n, width)): [2 n, 2 n]."""
    p = 1 - SWITCH_PROB
    loop = np.array([[p, (1.0 - p) / 1], [(1.0 - p) / 1, p]])
    return np.kron(loop, transition_local(n, width))


def p_init(n):
    p = np.zeros(2 * n)
    p[n:] = 1 / n
    return p


def log_terms(obs, trans, init):
    return np.log(obs + TINY).T, np.log(trans + TINY), np.log(init + TINY)


def viterbi(obs, trans, init):
    """librosa.sequence.viterbi(obs [S, F], trans, p_init=init) -> (states [F], value of the last state)."""
    log_prob, log_trans, log_init = log_terms(obs, trans, init)
    F, S = log_prob.shape
    value = log_prob[0] + log_init
    ptr = np.zeros((F, S), dtype=np.int64)
    for t in range(1, F):
        trans_out = value + log_trans.T          # [j, k]
        ptr[t] = np.argmax(trans_out, axis=1)
        value = log_prob[t] + trans_out[np.arange(S), ptr[t]]
    states = np.zeros(F, dtype=np.int64)
    states[-1] = np.argmax(value)
    for t in range(F - 2, -1, -1):
        states[t] = ptr[t + 1, states[t + 1]]
    return states, value[states[-1]]


def banded_log_transitions(n, width):
    """[2, W, n]: log_trans[s, q, i] of the source bin i - h + q (h = W // 2) into bin i, s = 0 for the same voicing, 1 for a switch."""
    trans = transition(n, width)
    lt = np.log(trans + TINY)
    h, dst = width // 2, np.arange(n)
    out = np.zeros((2, width, n))
    for s in range(2):
        for q in range(width):
            src = dst - h + q
            ok = (src >= 0) & (src < n)
            out[s, q, ok] = lt[s * n + src[ok], dst[ok]]
    return out


def _prefix_max(w):
    """(running max of w[0..m], its first index) for every m."""
    m = np.maximum.accumulate(w)
    new = np.r_[True, w[1:] > m[:-1]]
    return m, np.maximum.accumulate(np.where(new, np.arange(len(w)), 0))


def _suffix_max(w):
    """(max of w[m..], its first index) for every m."""
    r = w[::-1]
    m = np.maximum.accumulate(r)
    new = np.r_[True, r[1:] >= m[:-1]]
    idx = np.maximum.accumulate(np.where(new, np.arange(len(w)), 0))
    return m[::-1], (len(w) - 1 - idx)[::-1]


def viterbi_banded(obs, voiced_prob, n, width, log_tiny=None):
    """The kernel's algorithm: obs [F, n] voiced-bin probabilities and voiced_prob [F] -> (states [F], value of the last state).  Six source
    groups per destination in index order (before the band, the band, after it, for each half), strict comparisons."""
    LT = np.log(TINY) if log_tiny is None else log_tiny
    lt = banded_log_transitions(n, width)
    h = width // 2
    F = obs.shape[0]

    def log_obs(t):
        return np.concatenate([np.log(obs[t] + TINY), np.full(n, np.log((1 - voiced_prob[t]) / n + TINY))])

    value = log_obs(0) + np.log(p_init(n) + TINY)
    ptr = np.zeros((F, 2 * n), dtype=np.int64)
    dst = np.arange(n)
    q = np.arange(width)
    src = dst[:, None] - h + q[None, :]                      # [n, W]
    ok = (src >= 0) & (src < n)
    srcc = np.clip(src, 0, n - 1)
    for t in range(1, F):
        scans = []
        for c in range(2):
            w = value[c * n:(c + 1) * n] + LT
            scans.append((_prefix_max(w), _suffix_max(w)))
        new = np.empty(2 * n)
        lo = log_obs(t)
        for a in range(2):
            vals, idxs = [], []
            for c in range(2):
                (pv, pi), (sv, si) = scans[c]
                pre, suf = dst - h - 1, dst + h + 1
                vals.append(np.where(pre >= 0, pv[np.clip(pre, 0, n - 1)], -np.inf))
                idxs.append(c * n + pi[np.clip(pre, 0, n - 1)])
                cand = np.where(ok, value[c * n + srcc] + lt[0 if a == c else 1, q[None, :], dst[:, None]], -np.inf)
                j = np.argmax(cand, axis=1)
                vals.append(cand[dst, j])
                idxs.append(c * n + src[dst, j])
                vals.append(np.where(suf < n, sv[np.clip(suf, 0, n - 1)], -np.inf))
                idxs.append(c * n + si[np.clip(suf, 0, n - 1)])
            V, I = np.stack(vals), np.stack(idxs)
            g = np.argmax(V, axis=0)
            ptr[t, a * n:(a + 1) * n] = I[g, dst]
            new[a * n:(a + 1) * n] = lo[a * n:(a + 1) * n] + V[g, dst]
        value = new
    states = np.zeros(F, dtype=np.int64)
    states[-1] = np.argmax(value)
    for t in range(F - 2, -1, -1):
        states[t] = ptr[t + 1, states[t + 1]]
    return states, value[states[-1]]


def path_score(obs, trans, init, states):
    """The log probability of a state path, summed as the Viterbi recursion sums it."""
    log_prob, log_trans, log_init = log_terms(obs, trans, init)
    v = log_prob[0, states[0]] + log_init[states[0]]
    for t in range(1, len(states)):
        v = log_prob[t, states[t]] + (v + log_trans[states[t - 1], states[t]])
    return v


def brute_force(obs, trans, init):
    """max over every state path of path_score (tiny problems only)."""
    S, F = obs.shape
    return max(path_score(obs, trans, init, np.array(p)) for p in itertools.product(range(S), repeat=F))


def pyin(y, sr, hop, fmin=65.406, fmax=2093.0, frame_length=1024):
    """librosa.pyin(y, fmin, fmax, sr, frame_length, hop_length=hop) -> (f0 [F] with NaN unvoiced, voiced flag [F], voiced_prob [F])."""
    g = geometry(sr, hop, fmin, fmax, frame_length)
    n = g['n_bins']
    yf = frames(y, frame_length, hop)
    yin = cmnd(yf, frame_length, g['win_length'], g['min_period'], g['max_period'])
    obs, voiced_prob = observations(yin, parabolic_shifts(yin), sr, fmin, g['min_period'], n)
    states, _ = viterbi(obs, transition(n, g['transition_width']), p_init(n))
    freqs = fmin * 2 ** (np.arange(n) / (12 * BINS_PER_SEMITONE))
    f0 = freqs[states % n]
    voiced = states < n
    f0[~voiced] = np.nan
    return f0, voiced, voiced_prob
