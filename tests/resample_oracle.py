"""numpy oracle of the waveform front end (utils.audio.resample_batch / trim_silence_batch, csrc/resample.cu and csrc/trim.cu): the
contracts the kernels are checked against.

Resampling, scipy.signal.resample_poly(x, up, down) with its defaults, in closed form.  With m = max(up, down) and h_len = 10 m:
- h[j] = up w[j] / sum(w), j in [0, 2 h_len], w[j] = (1/m) sinc((j - h_len) / m) kaiser(2 h_len + 1, 5.0)[j] (firwin's filter);
- L' = ceil(L up / down);
- y[n] = sum_k x[k] h[h_len + n down - k up] over the k in [0, L) whose h index lies in [0, 2 h_len], in fp64.

Silence trimming, librosa 0.7.0's effects.trim(x, top_db, frame_length=W, hop_length=hop) restated line by line (_signal_to_frame_nonsilent,
feature.rms(center=True, pad_mode='reflect') and power_to_db(ref=np.max, amin=1e-10, top_db=None)); the reference crops x[M:-M] first
when its margin M is not 0:
- x is reflect-padded by W // 2 with numpy's repeated reflection: padded index i reads x[r], m = (i - W // 2) mod 2 (L - 1), r = m if
  m < L else 2 (L - 1) - m; a single sample repeats;
- F = 1 + (L + 2 (W // 2) - W) // hop frames, frame f covering padded [f hop, f hop + W); p_f = mean of its squares, in fp64;
- db_f = 10 log10(max(1e-10, p_f)) - 10 log10(max(1e-10, max p)); frame f is non-silent when db_f > -top_db;
- (start, end) = (a hop, min(L, (b + 1) hop)) for the first and last non-silent frames a and b, (0, 0) when there is none.
librosa is not installed where these tests run, so this restatement has not been run against librosa itself.
"""
import numpy as np

MAX_FACTOR = 2048            # include/b200tts.h B200TTS_RESAMPLE_MAX_FACTOR
AMIN = 1e-10


def taps(up, down):
    """(h fp64 [2 h_len + 1], h_len)."""
    m = max(up, down)
    h_len = 10 * m
    j = np.arange(2 * h_len + 1)
    w = np.sinc((j - h_len) / m) / m * np.kaiser(2 * h_len + 1, 5.0)
    return up * w / w.sum(), h_len


def out_length(L, up, down):
    return -(-L * up // down)


def _terms(L, up, down, h_len, n):
    """For outputs n: (k [len(n), T], h index [len(n), T], valid mask), T = the most taps any output has."""
    T = -(-(2 * h_len + 1) // up)
    t = h_len + n.astype(np.int64) * down
    k = (t // up)[:, None] - np.arange(T)[None, :]
    j = t[:, None] - k * up
    return k, j, (k >= 0) & (k < L) & (j <= 2 * h_len)


def resample(x, up, down, n=None, chunk=1 << 22):
    """(y fp64 at outputs n (default all L'), sum_k |x[k]| |h[.]| per output, the scale of its rounding error)."""
    x = np.asarray(x, dtype=np.float64)
    h, h_len = taps(up, down)
    n = np.arange(out_length(len(x), up, down)) if n is None else np.asarray(n)
    T = -(-(2 * h_len + 1) // up)
    y, mag = np.empty(len(n)), np.empty(len(n))
    step = max(1, chunk // T)
    for s in range(0, len(n), step):
        k, j, ok = _terms(len(x), up, down, h_len, n[s:s + step])
        xv = np.where(ok, x[np.clip(k, 0, len(x) - 1)], 0.0)
        hv = np.where(ok, h[np.clip(j, 0, 2 * h_len)], 0.0)
        y[s:s + step] = (xv * hv).sum(1)
        mag[s:s + step] = (np.abs(xv) * np.abs(hv)).sum(1)
    return y, mag


def reflect_index(i, L):
    """numpy's repeated reflection of padded-signal index i (relative to x[0]) onto [0, L)."""
    i = np.asarray(i, dtype=np.int64)
    if L == 1:
        return np.zeros_like(i)
    period = 2 * (L - 1)
    m = np.mod(i, period)
    return np.where(m >= L, period - m, m)


def frame_power(x, W, hop):
    """fp64 mean square of each of the F frames of x reflect-padded by W // 2."""
    x = np.asarray(x, dtype=np.float64)
    L = len(x)
    F = 1 + (L + 2 * (W // 2) - W) // hop
    idx = (np.arange(F)[:, None] * hop + np.arange(W)[None, :]) - W // 2
    return (x[reflect_index(idx, L)] ** 2).mean(1)


def frame_db(p):
    return 10 * np.log10(np.maximum(AMIN, p)) - 10 * np.log10(np.maximum(AMIN, p.max()))


def trim(x, W, hop, top_db=50, margin=0):
    """(start, end) in x[margin:L - margin], and the frame dBs the decision was taken on."""
    x = np.asarray(x, dtype=np.float64)
    if margin:
        x = x[margin:-margin]
    db = frame_db(frame_power(x, W, hop))
    nz = np.flatnonzero(db > -top_db)
    if len(nz) == 0:
        return (0, 0), db
    return (int(nz[0]) * hop, min(len(x), (int(nz[-1]) + 1) * hop)), db
