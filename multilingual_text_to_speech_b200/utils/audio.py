"""Audio with the reference's names (reference utils/audio.py:30-161; librosa 0.7.0): spectrogram -> waveform (mel_to_stft + griffinlim),
waveform -> log (mel) spectrogram (stft, melspectrogram, amplitude_to_db), MFCCs and the mel cepstral distortion, silence trimming
(effects.trim) and duration, and the front end the reference leaves to ffmpeg: resampling to hp.sample_rate (scipy's resample_poly).

Every stage runs in the library's kernels on the GPU whatever the precision mode is.  Spectrograms go in and out as [bins, F] (numpy or
torch); a batch is packed frame-major, and each result equals what its input gives on its own.  Reading and writing audio files are not
provided."""
import math

import numpy as np
import torch

from .. import _lib
from .. import functional as F
from ..params.params import Params as hp

# FISTA steps of the mel inversion: the least count whose worst NNLS residual gap on the convergence table in DESIGN ("Griffin-Lim vocoder")
# is within NNLS_GAP_BOUND of scipy's optimum
NNLS_ITERS = 800
NNLS_GAP_BOUND = 2e-3
MOMENTUM = 0.99          # librosa 0.7.0 griffinlim default

_MEL_CACHE = {}


def ms_to_frames(ms):
    """Convert milliseconds into number of frames."""
    return int(hp.sample_rate * ms / 1000)


def duration(data):
    """Return duration of an audio signal in seconds (at hp.sample_rate)."""
    return len(data) / hp.sample_rate


def db_to_amplitude(x):
    """Convert decibels to amplitude: (10 ** (0.1 x)) ** 0.5 (librosa.db_to_amplitude)."""
    if isinstance(x, torch.Tensor):
        return torch.pow(torch.pow(10.0, 0.1 * x), 0.5)
    return np.power(np.power(10.0, 0.1 * np.asarray(x)), 0.5)


def normalize_spectrogram(S, is_mel):
    """Normalize log-magnitude spectrogram (the constants are the ones train.py sets from the training set)."""
    if is_mel: return (S - hp.mel_normalize_mean) / hp.mel_normalize_variance
    else:      return (S - hp.lin_normalize_mean) / hp.lin_normalize_variance


def denormalize_spectrogram(S, is_mel):
    """Denormalize log-magnitude spectrogram (the constants are the ones train.py sets from the training set)."""
    if is_mel: return S * hp.mel_normalize_variance + hp.mel_normalize_mean
    else:      return S * hp.lin_normalize_variance + hp.lin_normalize_mean


def _hz_to_mel(f):
    f = np.asarray(f, dtype=np.float64)
    f_sp, min_log_hz = 200.0 / 3, 1000.0
    min_log_mel, logstep = min_log_hz / f_sp, np.log(6.4) / 27.0
    return np.where(f >= min_log_hz, min_log_mel + np.log(np.maximum(f, min_log_hz) / min_log_hz) / logstep, f / f_sp)


def _mel_to_hz(m):
    m = np.asarray(m, dtype=np.float64)
    f_sp, min_log_hz = 200.0 / 3, 1000.0
    min_log_mel, logstep = min_log_hz / f_sp, np.log(6.4) / 27.0
    return np.where(m >= min_log_mel, min_log_hz * np.exp(logstep * (m - min_log_mel)), f_sp * m)


def mel_basis(sr, n_fft, n_mels):
    """librosa.filters.mel(sr, n_fft, n_mels) of librosa 0.7.0: Slaney scale (htk=False), norm=1, fmin 0, fmax sr / 2, float32 -- the
    triangles are rounded to float32 and then scaled by the fp64 area norm and rounded again, as librosa's in-place float32 update does."""
    fftfreqs = np.linspace(0, sr / 2.0, 1 + n_fft // 2, endpoint=True)
    mel_f = _mel_to_hz(np.linspace(_hz_to_mel(0.0), _hz_to_mel(sr / 2.0), n_mels + 2))
    fdiff = np.diff(mel_f)
    ramps = np.subtract.outer(mel_f, fftfreqs)
    weights = np.zeros((n_mels, 1 + n_fft // 2), dtype=np.float32)
    for i in range(n_mels):
        lower = -ramps[i] / fdiff[i]
        upper = ramps[i + 2] / fdiff[i + 1]
        weights[i] = np.maximum(0, np.minimum(lower, upper))
    enorm = 2.0 / (mel_f[2:n_mels + 2] - mel_f[:n_mels])
    weights *= enorm[:, np.newaxis]
    return weights


def mel_tables(sr, n_fft, n_mels, device):
    """(basis [n_mels, K], pinv(basis)^T [n_mels, K], 1 / ||basis||_2^2) on `device`, built once per (sr, n_fft, n_mels) in fp64 and
    rounded to fp32.  The vocoder kernel relies on every linear bin lying in at most two adjacent filters; that is checked here."""
    key = (int(sr), int(n_fft), int(n_mels), str(device))
    if key not in _MEL_CACHE:
        A = mel_basis(sr, n_fft, n_mels)
        nz = A != 0
        if (nz.sum(0) > 2).any() or any(len(np.flatnonzero(c)) == 2 and np.diff(np.flatnonzero(c))[0] != 1 for c in nz.T):
            raise ValueError(f'mel basis (sr={sr}, n_fft={n_fft}, n_mels={n_mels}) has a bin in more than two adjacent filters')
        A64 = A.astype(np.float64)
        pinv_t = np.ascontiguousarray(np.linalg.pinv(A64).T)            # [n_mels, K] row-major, as the kernel reads it
        step = 1.0 / np.linalg.norm(A64, 2) ** 2
        _MEL_CACHE[key] = (torch.from_numpy(A).to(device), torch.from_numpy(pinv_t.astype(np.float32)).to(device), float(step))
    return _MEL_CACHE[key]


def _work_device(tensors=()):
    """The device of the first CUDA tensor, else the current CUDA device (`cuda` when none is visible: the first device work then raises)."""
    device = next((t.device for t in tensors if t.is_cuda), None)
    if device is None:
        device = torch.device('cuda', torch.cuda.current_device()) if torch.cuda.is_available() else torch.device('cuda')
    return device


def _return_like(t, as_numpy, src):
    """Result t (on the work device) as its input src came: numpy for numpy, the tensor itself for CUDA, a CPU copy for CPU."""
    if as_numpy:
        return t.cpu().numpy()
    return t if src.is_cuda else t.cpu()


def _as_float_tensor(x, what, dims):
    """numpy or torch -> (tensor, came as numpy); ValueError unless it is a non-empty floating array of `dims` dimensions."""
    is_np = not isinstance(x, torch.Tensor)
    if is_np:
        x = np.asarray(x)
        if not np.issubdtype(x.dtype, np.floating):
            raise ValueError(f'{what} has dtype {x.dtype}; expected floating point')
        x = torch.from_numpy(np.ascontiguousarray(x))
    elif not torch.is_floating_point(x):
        raise ValueError(f'{what} has dtype {x.dtype}; expected floating point')
    if x.dim() != dims or x.numel() == 0:
        raise ValueError(f'{what} has shape {tuple(x.shape)}; expected a non-empty {dims}-D array')
    return x, is_np


def _offsets(lengths, what, margin=0):
    """Host int64 offsets [B + 1] of items of these lengths packed end to end.  The kernels index a batch with int32, so ValueError unless
    the total is at most 2^31 - 1 - margin."""
    off = np.concatenate([[0], np.cumsum(lengths)]).astype(np.int64)
    if off[-1] > 2 ** 31 - 1 - margin:
        raise ValueError(f'{off[-1]} {what} in one batch; at most 2^31 - 1' + (f' - {margin}' if margin else ''))
    return off


class _Batch:
    """The inputs of a batch function -- waveforms [L_i] (dims 1) or spectrograms [bins, F_i] (dims 2), numpy or torch -- checked and
    packed end to end along their last axis, under the device and numpy / torch rules spectrogram_batch states.  `finite` rejects
    non-finite samples; `margin` is kept free below the int32 limit on the packed length."""

    def __init__(self, inputs, caller, name, dims=1, finite=False, margin=0):
        if not isinstance(inputs, (list, tuple)) or len(inputs) == 0:
            raise ValueError(f'{caller}: {name} must be a non-empty list of {dims}-D arrays')
        checked = [_as_float_tensor(x, f'{name}[{i}]', dims) for i, x in enumerate(inputs)]
        self.tensors = [t for t, _ in checked]
        self.as_numpy = [is_np for _, is_np in checked]
        if finite:
            for i, t in enumerate(self.tensors):
                if not bool(torch.isfinite(t).all()):
                    raise ValueError(f'{name}[{i}] has non-finite samples')
        self.lengths = [int(t.shape[-1]) for t in self.tensors]
        self.off = _offsets(self.lengths, 'samples' if dims == 1 else 'frames', margin)
        self.device = _work_device(self.tensors)

    def __len__(self):
        return len(self.tensors)

    def frame_offsets(self):
        """Host offsets of the mel frames of a waveform batch, F_i = 1 + L_i // hop."""
        hop = ms_to_frames(hp.stft_shift_ms)
        return _offsets([1 + n // hop for n in self.lengths], 'frames')

    def upload(self, *offsets):
        """(the inputs packed in fp32 -- [total] or [total, bins] --, then each host offset array as int32) on the work device."""
        packed = torch.cat([t.to(device=self.device, dtype=torch.float32).movedim(-1, 0) for t in self.tensors]).contiguous()
        return (packed,) + tuple(torch.from_numpy(o.astype(np.int32)).to(self.device) for o in offsets)

    def out(self, i, t):
        """Result t of input i under the return rule."""
        return _return_like(t, self.as_numpy[i], self.tensors[i])

    def split(self, packed, off):
        """packed[off[i]:off[i + 1]] of each input under the return rule."""
        return [self.out(i, packed[off[i]:off[i + 1]]) for i in range(len(self))]


def vocoder_shape(B, total_frames, mel):
    """The library shape of a batch under the current hp."""
    return _lib.VocoderShape(int(B), int(total_frames), int(hp.num_fft), ms_to_frames(hp.stft_shift_ms), ms_to_frames(hp.stft_window_ms),
                             int(hp.num_mels) if mel else 0, float(hp.griffin_lim_power), MOMENTUM,
                             float(hp.preemphasis) if hp.use_preemphasis else 0.0, NNLS_ITERS)


def inverse_spectrogram_batch(spectrograms, mel=False, phases=None, generator=None):
    """Log-magnitude spectrograms [bins, F_i] (already denormalised) -> one waveform per input, in input order, each of
    hop * (F_i - 1) samples.  `phases` (one [K, F_i] array of uniform draws in [0, 1) per input) sets the initial Griffin-Lim phases
    exp(2 pi i u); by default they are drawn with torch.rand on the device (`generator` optional), one draw for the whole packed batch.
    The same device and numpy / torch rules as spectrogram_batch."""
    K = hp.num_fft // 2 + 1
    bins = hp.num_mels if mel else K
    b = _Batch(spectrograms, 'inverse_spectrogram_batch', 'spectrograms', dims=2)
    for i, t in enumerate(b.tensors):
        if t.shape[0] != bins:
            raise ValueError(f'spectrograms[{i}] has shape {tuple(t.shape)}; expected [{bins}, frames]')
        if t.shape[1] < 2:
            raise ValueError(f'spectrograms[{i}] has {t.shape[1]} frames; Griffin-Lim needs at least 2')
    us = None
    if phases is not None:
        if len(phases) != len(b):
            raise ValueError(f'{len(phases)} phase arrays for {len(b)} spectrograms')
        us = []
        for i, p in enumerate(phases):
            p = torch.as_tensor(np.asarray(p) if not isinstance(p, torch.Tensor) else p)
            if tuple(p.shape) != (K, b.lengths[i]):
                raise ValueError(f'phases {i} has shape {tuple(p.shape)}; expected [{K}, {b.lengths[i]}]')
            us.append(p)
    with torch.cuda.device(b.device):
        wave = _vocode(b, us, mel, generator)
    # waveform i: hop (F_i - 1) samples from hop (off_i - i)
    return b.split(wave, ms_to_frames(hp.stft_shift_ms) * (b.off - np.arange(len(b) + 1)))


def _vocode(b, us, mel, generator):
    """The library steps on the batch's device (the current CUDA device) -> the packed waveform."""
    K, device = hp.num_fft // 2 + 1, b.device
    total = int(b.off[-1])
    shape = vocoder_shape(len(b), total, mel)
    ws = F.vocoder_workspace(shape, device)
    log_spec, off = b.upload(b.off)
    if mel:
        basis, pinv_t, step = mel_tables(hp.sample_rate, hp.num_fft, hp.num_mels, device)
        S = F.spectrogram_magnitude(shape, log_spec, basis, pinv_t, step)
    else:
        S = F.spectrogram_magnitude(shape, log_spec)
    if us is None:
        u = torch.rand(total, K, device=device, dtype=torch.float64, generator=generator)
    else:
        u = torch.cat([p.to(device=device, dtype=torch.float64).t() for p in us])
    angles = torch.polar(torch.ones_like(u), 2 * np.pi * u).to(torch.complex64).contiguous()
    rebuilt = torch.zeros_like(angles)
    wave = torch.empty(shape.hop * (total - len(b)), device=device, dtype=torch.float32)
    F.griffinlim(shape, S, off, angles, rebuilt, True, int(hp.griffin_lim_iters), wave, ws)
    F.deemphasis_normalize(shape, wave, off)
    return wave


def inverse_spectrogram(s, mel=False, phases=None):
    """Convert log-magnitude spectrogram [bins, F] to waveform (reference utils/audio.py:88-97)."""
    return inverse_spectrogram_batch([s], mel, None if phases is None else [phases])[0]


def inverse_mel_spectrogram(s, phases=None):
    """Convert log-mel-spectrogram to waveform."""
    return inverse_spectrogram(s, True, phases)


def analysis_shape(B, total_samples, total_frames, mel):
    """The library shape of an analysis batch under the current hp."""
    return _lib.AnalysisShape(int(B), int(total_samples), int(total_frames), int(hp.num_fft), ms_to_frames(hp.stft_shift_ms),
                              ms_to_frames(hp.stft_window_ms), int(hp.num_mels) if mel else 0,
                              float(hp.preemphasis) if hp.use_preemphasis else 0.0)


def spectrogram_batch(waveforms, mel=False):
    """Waveforms [L_i] -> log-magnitude (mel) spectrograms [bins, F_i], F_i = 1 + L_i // hop, in input order (reference
    utils/audio.py:66-78): pre-emphasis (hp.use_preemphasis), |stft| with centre reflect padding, the mel projection when `mel`, then
    amplitude_to_db relative to each utterance's own maximum.  Waveforms are computed in fp32: a float64 input is rounded to fp32 first (16-bit
    PCM scaled by 2^-15 is exact); the transform itself runs in fp64.  The work runs on the device of the first CUDA input, or on the current
    CUDA device when no input is on one.  numpy in -> numpy out; torch in -> torch out, on that device for CUDA inputs and on the CPU for CPU
    inputs."""
    b = _Batch(waveforms, 'spectrogram_batch', 'waveforms')
    off_host = b.frame_offsets()
    with torch.cuda.device(b.device):
        shape = analysis_shape(len(b), b.off[-1], off_host[-1], mel)
        wave, soff, off = b.upload(b.off, off_host)
        basis = mel_tables(hp.sample_rate, hp.num_fft, hp.num_mels, b.device)[0] if mel else None
        S = F.stft_magnitude(shape, wave, soff, off, basis)
        F.amplitude_to_db(shape, S, off, out=S)
    return [b.out(i, S[off_host[i]:off_host[i + 1]].t().contiguous()) for i in range(len(b))]


def spectrogram(y, mel=False):
    """Convert waveform to log-magnitude spectrogram [bins, 1 + len(y) // hop] (reference utils/audio.py:66-73)."""
    return spectrogram_batch([y], mel)[0]


def mel_spectrogram(y):
    """Convert waveform to log-mel-spectrogram."""
    return spectrogram(y, True)


def _mel_batch(specs, caller, name):
    """A _Batch of log-mel spectrograms [n_mels, F_i], each with at least hp.num_mfcc bands."""
    b = _Batch(specs, caller, name, dims=2)
    for i, t in enumerate(b.tensors):
        if t.shape[0] < hp.num_mfcc:
            raise ValueError(f'{name}[{i}] has {t.shape[0]} mel bands; hp.num_mfcc = {hp.num_mfcc} needs at least as many')
    return b


def _cepstra(b):
    """A _mel_batch -> (packed cepstra [sum F, n_mfcc], int32 frame offsets) on its device (the current CUDA device)."""
    mel_db, off = b.upload(b.off)
    return F.mel_cepstrum(mel_db, hp.num_mfcc), off


def get_spectrogram_mfcc(S):
    """Compute MFCCs [hp.num_mfcc, F] of a log-mel spectrogram [n_mels, F]: librosa 0.7.0 mfcc(S=S/10), the orthonormal DCT-II over the
    mel axis, c0 included (reference utils/audio.py:117-119)."""
    b = _mel_batch([S], 'get_spectrogram_mfcc', 'S')
    with torch.cuda.device(b.device):
        cep, _ = _cepstra(b)
    return b.out(0, cep.t().contiguous())


def mel_cepstral_distortion_batch(S1s, S2s, mode='dtw'):
    """Mel cepstral distortion of each pair (S1s[i], S2s[i]) of log-mel spectrograms [n_mels, F] (reference mel_cepstral_distorision, utils/
    audio.py:127-161): MFCCs without c0, then the mean Euclidean frame distance over the frames paired by `mode`: 'cut' (the first min(F1, F2)
    frames), 'stretch' (the shorter sequence indexed at i * n // m) or 'dtw'.  'dtw' is the exact dynamic-time-warping optimum, cost / path
    length; the reference calls fastdtw with radius 1, which approximates that optimum, so the two agree when fastdtw finds the optimal path
    and may differ otherwise.  Returns float64, one value per pair: a numpy array unless the first
    input is a torch tensor (then a torch tensor on its device).  The work runs on the device of the first CUDA input of either list, else
    on the current device."""
    if mode not in _lib.MCD_MODES:
        raise ValueError(f'unknown mode {mode!r}; expected one of {sorted(_lib.MCD_MODES)}')
    a = _mel_batch(S1s, 'mel_cepstral_distortion_batch', 'S1s')
    b = _mel_batch(S2s, 'mel_cepstral_distortion_batch', 'S2s')
    if len(a) != len(b):
        raise ValueError(f'{len(a)} spectrograms against {len(b)}')
    for i, (x, y) in enumerate(zip(a.tensors, b.tensors)):
        if x.shape[0] != y.shape[0]:
            raise ValueError(f'pair {i} has {x.shape[0]} and {y.shape[0]} mel bands')
        if mode == 'dtw' and min(x.shape[1], y.shape[1]) > _lib.DTW_MAX_FRAMES:
            raise ValueError(f'pair {i} ({x.shape[1]} x {y.shape[1]} frames): dtw keeps three anti-diagonals in shared memory, so the shorter '
                             f'sequence may have at most {_lib.DTW_MAX_FRAMES} frames')
    a.device = b.device = _work_device(a.tensors + b.tensors)
    with torch.cuda.device(a.device):
        cep_a, off_a = _cepstra(a)
        cep_b, off_b = _cepstra(b)
        mcd, _ = F.mel_cepstral_distortion(cep_a, off_a, cep_b, off_b, mode)
    return a.out(0, mcd)


def mel_cepstral_distorision(S1, S2, mode):
    """Compute Mel Cepstral Distorsion between two mel spectrograms (reference spelling; see mel_cepstral_distortion_batch).

    Arguments:
        S1 and S2 -- mel spectrograms
        mode -- 'cut' to cut off frames of longer seq.
                'stretch' to stretch linearly the shorter seq.
                'dtw' to compute DTW with minimal possible MCD (exact DTW, not fastdtw's approximation)
    """
    return float(mel_cepstral_distortion_batch([S1], [S2], mode)[0])


# pYIN parameters of librosa 0.10's librosa.pyin that are fixed here
PITCH_N_THRESHOLDS = 100
PITCH_BETA = (2, 18)
PITCH_BINS_PER_SEMITONE = 10                 # resolution 0.1 semitone
PITCH_MAX_TRANSITION_RATE = 35.92            # octaves per second
PITCH_SWITCH_PROB = 0.01

_PITCH_CACHE = {}


def pitch_geometry(fmin=65.406, fmax=2093.0, frame_length=1024):
    """The derived pYIN quantities under the current hp, with librosa 0.10's numpy expressions: {sr, hop, win_length, min_period,
    max_period, n_bins, transition_width}.  Raises ValueError for parameters librosa.pyin would refuse or the kernels do not take."""
    sr, hop = hp.sample_rate, ms_to_frames(hp.stft_shift_ms)
    fmin, fmax, frame_length = float(fmin), float(fmax), int(frame_length)
    if not fmin > 0:
        raise ValueError(f'fmin = {fmin} must be positive')
    if not fmin < fmax:
        raise ValueError(f'fmin = {fmin} must be below fmax = {fmax}')
    if fmax > sr / 2:
        raise ValueError(f'fmax = {fmax} is above the Nyquist frequency {sr / 2}')
    if frame_length % 2 or not 4 <= frame_length <= _lib.PITCH_MAX_FRAME_LENGTH:
        raise ValueError(f'frame_length = {frame_length} must be even and in [4, {_lib.PITCH_MAX_FRAME_LENGTH}]')
    win = frame_length // 2
    min_period = int(np.floor(sr / fmax))
    max_period = min(int(np.ceil(sr / fmin)), frame_length - win - 1)
    if max_period <= min_period:
        raise ValueError(f'frame_length = {frame_length} leaves no lag range: max_period {max_period} <= min_period {min_period}')
    n_bins = int(np.floor(12 * PITCH_BINS_PER_SEMITONE * np.log2(fmax / fmin))) + 1
    width = round(PITCH_MAX_TRANSITION_RATE * 12 * hop / sr) * PITCH_BINS_PER_SEMITONE + 1
    if n_bins > _lib.PITCH_MAX_BINS:
        raise ValueError(f'fmin = {fmin} and fmax = {fmax} give {n_bins} pitch bins; at most {_lib.PITCH_MAX_BINS}')
    if n_bins < width:
        raise ValueError(f'fmin = {fmin} and fmax = {fmax} give {n_bins} pitch bins, fewer than the transition width {width}')
    return dict(sr=sr, hop=hop, win_length=win, min_period=min_period, max_period=max_period, n_bins=n_bins, transition_width=width)


def _pitch_log_transitions(n, width):
    """[2, W, n] float64: log(S_s T[i - h + q, i] + tiny), T librosa's transition_local(n, W, 'triangle', wrap=False) built densely with its
    own expressions, S_0 = 0.99 (same voicing) and S_1 = transition_loop(2, 0.99)'s off-diagonal."""
    import scipy.signal
    window = scipy.signal.get_window('triangle', width, fftbins=False)
    lpad = (n - width) // 2
    padded = np.pad(window, (lpad, n - width - lpad))
    local = np.zeros((n, n), dtype=np.float64)
    for i in range(n):
        row = np.roll(padded, n // 2 + i + 1)
        row[min(n, i + width // 2 + 1):] = 0
        row[:max(0, i - width // 2)] = 0
        local[i] = row
    local /= local.sum(axis=1, keepdims=True)
    tiny = np.finfo(np.float64).tiny
    h, dst = width // 2, np.arange(n)
    out = np.zeros((2, width, n), dtype=np.float64)
    for s, p in enumerate((1 - PITCH_SWITCH_PROB, (1.0 - (1 - PITCH_SWITCH_PROB)) / 1)):
        lt = np.log(p * local + tiny)
        for q in range(width):
            src = dst - h + q
            ok = (src >= 0) & (src < n)
            out[s, q, ok] = lt[src[ok], dst[ok]]
    return out


def _pitch_tables(g, fmin, device):
    """(shape fields, log transitions on `device`, f0 of every bin on `device`), built once per geometry."""
    key = (g['sr'], g['hop'], g['win_length'], g['n_bins'], g['transition_width'], float(fmin), str(device))
    if key not in _PITCH_CACHE:
        import scipy.stats
        thresholds = np.linspace(0, 1, PITCH_N_THRESHOLDS + 1)
        beta_probs = np.diff(scipy.stats.beta.cdf(thresholds, PITCH_BETA[0], PITCH_BETA[1]))
        tiny = np.finfo(np.float64).tiny
        n = g['n_bins']
        fields = dict(log_tiny=float(np.log(tiny)), log_init=float(np.log(1 / n + tiny)), thresholds=thresholds[1:], beta_probs=beta_probs)
        freqs = fmin * 2 ** (np.arange(n) / (12 * PITCH_BINS_PER_SEMITONE))
        _PITCH_CACHE[key] = (fields, torch.from_numpy(_pitch_log_transitions(n, g['transition_width'])).to(device),
                             torch.from_numpy(freqs.astype(np.float32)).to(device))
    return _PITCH_CACHE[key]


def pitch_shape(B, total_samples, total_frames, fmin=65.406, fmax=2093.0, frame_length=1024, device=None):
    """(library shape, log transitions, bin frequencies) of a pitch batch; tables on `device` (the current CUDA device by default)."""
    g = pitch_geometry(fmin, fmax, frame_length)
    device = torch.device('cuda', torch.cuda.current_device()) if device is None else device
    fields, log_trans, freqs = _pitch_tables(g, float(fmin), device)
    shape = _lib.PitchShape(int(B), int(total_samples), int(total_frames), int(frame_length), g['win_length'], g['hop'], g['min_period'],
                            g['max_period'], g['n_bins'], g['transition_width'], float(g['sr']), float(fmin), fields['log_tiny'],
                            fields['log_init'])
    shape.thresholds[:] = [float(v) for v in fields['thresholds']]
    shape.beta_probs[:] = [float(v) for v in fields['beta_probs']]
    return shape, log_trans, freqs


def pitch_batch(waveforms, fmin=65.406, fmax=2093.0, frame_length=1024):
    """F0 tracks of waveforms [L_i] by probabilistic YIN, as librosa 0.10's librosa.pyin(y, fmin=fmin, fmax=fmax, sr=hp.sample_rate,
    frame_length=frame_length, hop_length=hop) computes them with its other defaults (win_length = frame_length // 2, 100 thresholds,
    beta (2, 18), Boltzmann 2, 0.1 semitone bins, 35.92 octaves/s, switch probability 0.01, no-trough probability 0.01, center=True with
    zero padding), on the raw waveform (no pre-emphasis).  hop = ms_to_frames(hp.stft_shift_ms), so the frames are the mel frames:
    F_i = 1 + L_i // hop.  -> one (f0, voiced_prob) per input, each [F_i] float32: f0 in Hz, NaN on unvoiced frames.  The three stages
    run in the library's fp64 kernels (include/b200tts.h); waveforms are rounded to fp32 first.  The same device and numpy / torch rules as
    spectrogram_batch.  Raises ValueError on a bad input, fmin <= 0, fmin >= fmax, fmax above Nyquist, more than B200TTS_PITCH_MAX_BINS
    bins or fewer than the transition width, or a frame_length that is odd, out of range or leaves no lags."""
    b = _Batch(waveforms, 'pitch_batch', 'waveforms')
    off_host = b.frame_offsets()
    pitch_geometry(fmin, fmax, frame_length)
    with torch.cuda.device(b.device):
        shape, log_trans, freqs = pitch_shape(len(b), b.off[-1], off_host[-1], fmin, fmax, frame_length, b.device)
        wave, soff, off = b.upload(b.off, off_host)
        cmnd = F.pitch_cmnd(shape, wave, soff, off)
        obs, voiced_prob = F.pitch_observations(shape, cmnd)
        state = F.pitch_viterbi(shape, obs, voiced_prob, off, log_trans).long()
        n = shape.n_bins
        f0 = torch.where(state < n, freqs[state % n], torch.full_like(freqs[:1], float('nan')))
        vp = voiced_prob.float()
    return list(zip(b.split(f0, off_host), b.split(vp, off_host)))


def pitch(y, fmin=65.406, fmax=2093.0, frame_length=1024):
    """(f0, voiced_prob) of one waveform; see pitch_batch."""
    return pitch_batch([y], fmin, fmax, frame_length)[0]


def energy_batch(waveforms):
    """Frame energies of waveforms [L_i]: the L2 norm over frequency of each frame of the linear magnitude spectrogram spectrogram_batch
    computes before the dB scale (pre-emphasis per hp, |stft| with centre reflect padding), summed in fp64.  -> [F_i] float32 per input,
    F_i = 1 + L_i // hop; the same device and numpy / torch rules as spectrogram_batch."""
    b = _Batch(waveforms, 'energy_batch', 'waveforms')
    off_host = b.frame_offsets()
    with torch.cuda.device(b.device):
        shape = analysis_shape(len(b), b.off[-1], off_host[-1], False)
        wave, soff, off = b.upload(b.off, off_host)
        S = F.stft_magnitude(shape, wave, soff, off)
        e = S.double().square().sum(1).sqrt().float()
    return b.split(e, off_host)


def _track(x, what, frames=None, dtype=torch.float32, f0=False):
    """A per-frame track [F] (numpy or torch) -> (host numpy array of `dtype`, came as numpy, tensor).  ValueError unless it is a
    non-empty floating 1-D array, of `frames` frames when given, and with `f0` positive Hz on voiced frames (NaN marks unvoiced ones),
    checked on the `dtype` values."""
    t, is_np = _as_float_tensor(x, what, 1)
    a = t.detach().cpu().to(dtype).numpy()
    if frames is not None and len(a) != frames:
        raise ValueError(f'{what} has {len(a)} frames; its waveform has {frames} (1 + L // hop)')
    if f0 and ((a[~np.isnan(a)] <= 0).any() or np.isinf(a).any()):
        raise ValueError(f'{what} must be positive Hz on voiced frames (NaN marks unvoiced ones)')
    return a, is_np, t


def pitch_errors_batch(f0_refs, f0_gens):
    """F0 error metrics of each pair (reference, generated) of F0 tracks [F] in Hz, NaN on unvoiced frames (pitch_batch's f0), over the
    first min(F_ref, F_gen) frames in float64.  Frames voiced in both are VV; a gross error is a VV frame with |f0_gen - f0_ref| >
    0.2 f0_ref.  -> dict of float64 [B]: gpe (gross errors / VV frames), vde (frames whose voicing differs / frames), ffe ((gross errors +
    voicing errors) / frames) and f0_rmse_cents (the RMS of 1200 log2(f0_gen / f0_ref) over VV frames); gpe and f0_rmse_cents are NaN for
    a pair without VV frames.  numpy arrays, or torch tensors on the first reference's device when it is a torch tensor."""
    if not isinstance(f0_refs, (list, tuple)) or not isinstance(f0_gens, (list, tuple)) or len(f0_refs) == 0:
        raise ValueError('pitch_errors_batch expects two non-empty lists of 1-D f0 tracks')
    if len(f0_refs) != len(f0_gens):
        raise ValueError(f'{len(f0_refs)} reference tracks against {len(f0_gens)}')
    refs = [_track(x, f'f0_refs[{i}]', dtype=torch.float64, f0=True) for i, x in enumerate(f0_refs)]
    gens = [_track(x, f'f0_gens[{i}]', dtype=torch.float64, f0=True) for i, x in enumerate(f0_gens)]
    out = {k: np.empty(len(refs)) for k in ('gpe', 'vde', 'ffe', 'f0_rmse_cents')}
    for i, ((r, _, _), (g, _, _)) in enumerate(zip(refs, gens)):
        m = min(len(r), len(g))
        r, g = r[:m], g[:m]
        vr, vg = ~np.isnan(r), ~np.isnan(g)
        vv = vr & vg
        nvv = int(vv.sum())
        gross = int((np.abs(g[vv] - r[vv]) > 0.2 * r[vv]).sum())
        voicing = int((vr != vg).sum())
        out['gpe'][i] = gross / nvv if nvv else np.nan
        out['vde'][i] = voicing / m
        out['ffe'][i] = (gross + voicing) / m
        out['f0_rmse_cents'][i] = np.sqrt(np.mean((1200 * np.log2(g[vv] / r[vv])) ** 2)) if nvv else np.nan
    if refs[0][1]:
        return out
    return {k: torch.from_numpy(v).to(refs[0][2].device) for k, v in out.items()}


def _check_ratios(r, what):
    if not np.isfinite(r).all() or (r < 0.5).any() or (r > 2.0).any():
        raise ValueError(f'{what} must be finite and in [0.5, 2] (one octave each way)')


def pitch_shift_batch(waveforms, semitones=None, ratios=None, f0s=None, fmin=65.406, fmax=2093.0):
    """Pitch-shift waveforms [L_i] by TD-PSOLA, each keeping its length: grains two periods wide are taken at pitch marks placed on the F0
    track and overlap-added at marks spaced by the period over the ratio, so F0 is multiplied by the ratio while the spectral envelope
    (formants) and the duration stay.  include/b200tts.h and tests/psola_oracle.py state the rules exactly.
    Give exactly one of `semitones` (one float, or one per waveform: ratio 2^(s / 12) on every frame) and `ratios` (one [F_i] track of new
    F0 / old F0 per waveform).  Ratios must be finite and in [0.5, 2].  `f0s`: one F0 track [F_i] per waveform in Hz, NaN on unvoiced
    frames, as pitch_batch returns it; by default pitch_batch(waveforms, fmin, fmax).  Voiced F0 must give periods rint(sr / f0) in
    [2, B200TTS_PSOLA_MAX_PERIOD] samples.  Frames are the mel frames, F_i = 1 + L_i // hop, hop = ms_to_frames(hp.stft_shift_ms); unvoiced
    regions keep marks hop samples apart and are never respaced.  Only voiced grains move, so at ratio 1, or without voiced frames, the
    output equals the input.  Waveforms are rounded to fp32; marks and sums are fp64 in the library's kernels.  The same device and
    numpy / torch rules as spectrogram_batch.  Raises ValueError on a bad or non-finite waveform, both or neither of semitones and ratios,
    mismatched list or track lengths, an out-of-range ratio, or a non-positive or out-of-range F0."""
    b = _Batch(waveforms, 'pitch_shift_batch', 'waveforms', finite=True)
    off_host = b.frame_offsets()
    B = len(b)
    frames = [int(off_host[i + 1] - off_host[i]) for i in range(B)]

    def tracks(ts, what, f0=False):
        """One fp32 host track [F_i] per waveform."""
        if not isinstance(ts, (list, tuple)) or len(ts) != B:
            raise ValueError(f'{what} must be a list of {B} tracks, one per waveform')
        return [_track(t, f'{what}[{i}]', frames[i], f0=f0)[0] for i, t in enumerate(ts)]

    if (semitones is None) == (ratios is None):
        raise ValueError('give exactly one of semitones and ratios')
    if semitones is not None:
        s = [semitones] * B if np.ndim(semitones) == 0 else list(semitones)
        if len(s) != B:
            raise ValueError(f'{len(s)} semitone values for {B} waveforms')
        r = [np.full(f, 2.0 ** (float(v) / 12.0), dtype=np.float32) for v, f in zip(s, frames)]
    else:
        r = tracks(ratios, 'ratios')
    for i, a in enumerate(r):
        _check_ratios(a, f'the ratios of waveform {i}')
    if f0s is None:
        f0s = [f for f, _ in pitch_batch(waveforms, fmin, fmax)]
    f0 = tracks(f0s, 'f0s', f0=True)
    sr, hop = hp.sample_rate, ms_to_frames(hp.stft_shift_ms)
    for i, a in enumerate(f0):
        p = np.rint(sr / a[~np.isnan(a)].astype(np.float64))
        if ((p < 2) | (p > _lib.PSOLA_MAX_PERIOD)).any():
            raise ValueError(f'f0 of waveform {i} gives periods outside [2, {_lib.PSOLA_MAX_PERIOD}] samples: F0 must lie in about '
                             f'[{sr / (_lib.PSOLA_MAX_PERIOD + 0.5):.2f}, {sr / 1.5:.1f}] Hz')
    with torch.cuda.device(b.device):
        shape = _lib.PsolaShape(B, int(b.off[-1]), int(off_host[-1]), hop, hop, float(sr))
        wave, soff, off = b.upload(b.off, off_host)
        f0_d = torch.from_numpy(np.concatenate(f0)).to(b.device)
        r_d = torch.from_numpy(np.concatenate(r)).to(b.device)
        ws = F.psola_marks(shape, wave, soff, f0_d, r_d, off)
        y = F.psola_overlap_add(shape, wave, soff, ws)
    return b.split(y, b.off)


def pitch_shift(y, semitones=None, ratios=None, f0=None, fmin=65.406, fmax=2093.0):
    """One waveform pitch-shifted; `ratios` and `f0` are single [F] tracks here.  See pitch_shift_batch."""
    return pitch_shift_batch([y], semitones, None if ratios is None else [ratios], None if f0 is None else [f0], fmin, fmax)[0]


def f0_ratio(f0_target, f0_source):
    """The per-frame ratio that moves f0_source onto f0_target (both [F] in Hz, NaN unvoiced, as pitch_batch returns them), for
    pitch_shift_batch(..., ratios=[f0_ratio(target, source)], f0s=[source]): target / source clipped to [0.5, 2] on frames voiced in both,
    1 elsewhere, over the first min(F_target, F_source) frames and padded with 1 to F_source.  -> float32 [F_source], numpy for a numpy
    source, else a tensor on the source's device.  Raises ValueError on tracks that are not 1-D floating, or that hold a non-positive or
    infinite voiced F0."""
    t, _, _ = _track(f0_target, 'f0_target', dtype=torch.float64, f0=True)
    s, s_np, s_t = _track(f0_source, 'f0_source', dtype=torch.float64, f0=True)
    m = min(len(t), len(s))
    out = np.ones(len(s))
    vv = ~np.isnan(t[:m]) & ~np.isnan(s[:m])
    out[:m][vv] = np.clip(t[:m][vv] / s[:m][vv], 0.5, 2.0)
    out = out.astype(np.float32)
    return out if s_np else torch.from_numpy(out).to(s_t.device)


# time_stretch_batch's rate range: a quarter to four times the source rate
STRETCH_RATES = (0.25, 4.0)


def _stretch_length(L, rate):
    return max(1, int(round(L / rate)))


def _retime_length(L, hop, dp):
    return max(1, hop * (int(dp.sum()) - 1) + L % hop)


def _stretch_plan(L, hop, rate):
    """(L', warp tau_k = k hop rate in fp64) of a time stretch."""
    Lp = _stretch_length(L, rate)
    return Lp, np.arange((Lp - 1) // hop + 2, dtype=np.float64) * hop * rate


def _retime_plan(L, hop, d, dp):
    """(L', warp tau_k = hop phi(k)) of a retime from durations d to dp (int64 [J]).  phi maps output frame coordinates onto input ones:
    with B, B' the cumulative durations, [B'_j - 1/2, B'_{j+1} - 1/2) goes linearly onto [B_j - 1/2, B_{j+1} - 1/2), and past B'_J - 1/2
    the slope is 1.  Frame k lies in the interval of the first symbol j with B'_{j+1} > k; a symbol with d'_j = 0 has no interval."""
    Lp = _retime_length(L, hop, dp)
    K = (Lp - 1) // hop + 2
    J = len(d)
    B = np.concatenate([[0], np.cumsum(d)]).astype(np.float64)
    Bp = np.concatenate([[0], np.cumsum(dp)]).astype(np.float64)
    k = np.arange(K, dtype=np.float64)
    j = np.searchsorted(Bp[1:], k, side='right')
    inside = j < J
    jj = np.minimum(j, J - 1)
    lo_in = np.where(inside, B[jj], B[J]) - 0.5
    lo_out = np.where(inside, Bp[jj], Bp[J]) - 0.5
    num = np.where(inside, d[jj], 1).astype(np.float64)
    den = np.where(inside, dp[jj], 1).astype(np.float64)
    return Lp, hop * (lo_in + (k - lo_out) * num / den)


def _wsola_hop():
    """The hop WSOLA uses: hp.stft_shift_ms in samples, which must be in [1, WSOLA_MAX_HOP]."""
    hop = ms_to_frames(hp.stft_shift_ms)
    if not 1 <= hop <= _lib.WSOLA_MAX_HOP:
        raise ValueError(f'hop {hop} (hp.stft_shift_ms) must be in [1, {_lib.WSOLA_MAX_HOP}] samples')
    return hop


def _wsola(b, hop, ooff_host, warps):
    """Both WSOLA kernels on the packed batch b; ooff_host: host output offsets; warps: fp64 [K_i] per waveform -> the output waveforms."""
    foff_host = _offsets([len(w) for w in warps], 'frames')
    with torch.cuda.device(b.device):
        shape = _lib.WsolaShape(len(b), int(b.off[-1]), int(ooff_host[-1]), int(foff_host[-1]), hop, hop)
        wave, soff, ooff, foff = b.upload(b.off, ooff_host, foff_host)
        warp = torch.from_numpy(np.concatenate(warps)).to(b.device)
        positions = F.wsola_positions(shape, wave, soff, warp, foff)
        y = F.wsola_overlap_add(shape, wave, soff, positions, foff, ooff)
    return b.split(y, ooff_host)


def time_stretch_batch(waveforms, rate):
    """Time-stretch waveforms [L_i] by WSOLA (waveform-similarity overlap-add), keeping pitch and formants: `rate` is one float or one
    per waveform, finite and in [0.25, 4]; above 1 is faster, as in librosa.effects.time_stretch.  Output i has
    L'_i = max(1, round(L_i / rate_i)) samples.  Frames 2 hop long (hop = ms_to_frames(hp.stft_shift_ms), the mel hop) are overlap-added
    with a periodic Hann window every hop output samples; frame k is read near input sample k hop rate, shifted by up to hop samples to
    the position most similar to the natural continuation of frame k - 1.  include/b200tts.h and tests/wsola_oracle.py state the rules
    exactly.  At rate 1 the output is the input.  Waveforms are rounded to fp32; the search and the sums are fp64 in the library's kernels.
    The same device and numpy / torch rules as spectrogram_batch.  Raises ValueError on a bad or non-finite waveform, a rate count that
    does not match, a rate out of range, or more than 2^31 - 1 output samples."""
    b = _Batch(waveforms, 'time_stretch_batch', 'waveforms', finite=True, margin=_lib.WSOLA_MAX_TOLERANCE)
    hop = _wsola_hop()
    B = len(b)
    try:
        rates = np.asarray(rate).astype(np.float64)
    except (TypeError, ValueError):
        raise ValueError(f'rate must be numeric (got {rate!r})') from None
    if rates.ndim > 1 or (rates.ndim == 1 and len(rates) != B):
        raise ValueError(f'rate must be one float or one per waveform ({B})')
    rates = np.broadcast_to(rates, (B,))
    lo, hi = STRETCH_RATES
    if not np.isfinite(rates).all() or (rates < lo).any() or (rates > hi).any():
        raise ValueError(f'rate must be finite and in [{lo}, {hi}] (got {rates.tolist()})')
    ooff_host = _offsets([_stretch_length(n, float(r)) for n, r in zip(b.lengths, rates)], 'output samples')   # before any warp
    return _wsola(b, hop, ooff_host, [_stretch_plan(n, hop, float(r))[1] for n, r in zip(b.lengths, rates)])


def time_stretch(y, rate):
    """One waveform time-stretched by `rate` (above 1 is faster).  See time_stretch_batch."""
    return time_stretch_batch([y], rate)[0]


def retime_batch(waveforms, durations, new_durations):
    """Retime waveforms [L_i] by WSOLA from per-symbol durations to new ones: symbol j's frames are stretched or squeezed so that it lasts
    new_durations[i][j] mel frames instead of durations[i][j], keeping pitch and formants.  Both are int frames per symbol, one track per
    waveform, as Tacotron.align gives them for a mel made by mel_spectrogram(y) (align(...).durations[b, :L_b]): each sum(durations[i])
    must be the waveform's 1 + L_i // hop mel frames, both tracks have the same length, every entry is >= 0 and sum(new_durations[i]) >= 1.
    Output i has L'_i = max(1, hop (sum d' - 1) + L_i mod hop) samples, so spectrogram(y') has sum d' frames.  The warp is defined on frame
    coordinates: symbol j's output interval [B'_j - 1/2, B'_{j+1} - 1/2) maps linearly onto its input interval [B_j - 1/2, B_{j+1} - 1/2),
    B and B' the cumulative durations; a symbol with d'_j = 0 is dropped, one with d_j = 0 holds its boundary, and past the last boundary
    the slope is 1.  Frame k is then read near input sample hop phi(k) and placed as time_stretch_batch places it, so with
    new_durations = durations the output is the input.  Raises ValueError on a bad or non-finite waveform, counts that do not match,
    malformed durations, or more than 2^31 - 1 output samples."""
    b = _Batch(waveforms, 'retime_batch', 'waveforms', finite=True, margin=_lib.WSOLA_MAX_TOLERANCE)
    hop = _wsola_hop()
    off_host = b.frame_offsets()
    B = len(b)
    for what, t in (('durations', durations), ('new_durations', new_durations)):
        if not isinstance(t, (list, tuple)) or len(t) != B:
            raise ValueError(f'retime_batch: {what} must be a list of {B} tracks, one per waveform')
    tracks = []
    for i in range(B):
        d = F._durations_host(durations[i], f'retime_batch durations[{i}]')
        dp = F._durations_host(new_durations[i], f'retime_batch new_durations[{i}]')
        if len(d) != len(dp):
            raise ValueError(f'retime_batch: durations[{i}] has {len(d)} symbols, new_durations[{i}] {len(dp)}')
        frames = int(off_host[i + 1] - off_host[i])
        if int(d.sum()) != frames:
            raise ValueError(f'retime_batch: durations[{i}] total {int(d.sum())} frames; waveform {i} has {frames} (1 + L // hop)')
        if int(dp.sum()) < 1:
            raise ValueError(f'retime_batch: new_durations[{i}] total 0 frames')
        tracks.append((d, dp))
    ooff_host = _offsets([_retime_length(n, hop, dp) for n, (_, dp) in zip(b.lengths, tracks)], 'output samples')   # before any warp
    return _wsola(b, hop, ooff_host, [_retime_plan(n, hop, d, dp)[1] for n, (d, dp) in zip(b.lengths, tracks)])


def retime(y, durations, new_durations):
    """One waveform retimed from `durations` to `new_durations` (int frames per symbol).  See retime_batch."""
    return retime_batch([y], [durations], [new_durations])[0]


# ---- waveform front end: resampling and silence trimming ---------------------------------------------------------------------------------
_RESAMPLE_CACHE = {}


def _rate(r, what):
    if isinstance(r, (bool, np.bool_)) or not isinstance(r, (int, np.integer)) or r <= 0:
        raise ValueError(f'{what} must be a positive integer sample rate in Hz (got {r!r})')
    return int(r)


def resample_ratio(orig_sr, target_sr):
    """(up, down): target_sr / orig_sr in lowest terms."""
    g = math.gcd(orig_sr, target_sr)
    return target_sr // g, orig_sr // g


def resample_taps(up, down):
    """(polyphase table [up, T] fp64, h_len) of scipy.signal.resample_poly(x, up, down): the filter h = up firwin(2 h_len + 1, 1 / m,
    window=('kaiser', 5.0)), m = max(up, down), h_len = 10 m, built with firwin's expressions, and table[phase, i] = h[phase + i up]
    (0 past the filter), T = ceil((2 h_len + 1) / up), so that each output's taps are contiguous."""
    m = max(up, down)
    h_len = 10 * m
    n = 2 * h_len + 1
    fc = 1.0 / m
    w = fc * np.sinc(fc * (np.arange(n) - h_len)) * np.kaiser(n, 5.0)
    h = w / w.sum() * up
    T = -(-n // up)
    padded = np.zeros(up * T)
    padded[:n] = h
    return np.ascontiguousarray(padded.reshape(T, up).T), h_len


def _resample_table(up, down, device):
    """resample_taps(up, down)'s table flattened on `device`, built once per (up, down, device)."""
    key = (up, down, str(device))
    if key not in _RESAMPLE_CACHE:
        _RESAMPLE_CACHE[key] = torch.from_numpy(resample_taps(up, down)[0].ravel()).to(device)
    return _RESAMPLE_CACHE[key]


def resample_batch(waveforms, orig_sr, target_sr=None):
    """Resample waveforms [L_i] from orig_sr to target_sr (default hp.sample_rate): exactly scipy.signal.resample_poly(x, up, down) with
    its defaults (Kaiser window, beta 5, zero padding), up / down = target_sr / orig_sr in lowest terms, so output i has
    ceil(L_i up / down) samples.  `orig_sr` is one int or one per waveform, so a batch may mix source rates; `target_sr` is one int.  A
    waveform already at target_sr comes back as its fp32 copy, and no kernel runs for it.  include/b200tts.h states the rule exactly.
    Waveforms are rounded to fp32; the filter and the sums are fp64 in the library's kernel.  The same device and numpy / torch rules
    as spectrogram_batch.  Raises ValueError on a bad or non-finite waveform, a rate that is not a positive integer, an orig_sr count
    that does not match, a ratio with max(up, down) above B200TTS_RESAMPLE_MAX_FACTOR (2048; every pair of 8, 11.025, 16, 22.05, 24, 32,
    44.1, 48 and 96 kHz is within it), or more than 2^31 - 1 output samples."""
    b = _Batch(waveforms, 'resample_batch', 'waveforms', finite=True)
    B = len(b)
    target = _rate(hp.sample_rate if target_sr is None else target_sr, 'target_sr')
    srs = [orig_sr] * B if np.ndim(orig_sr) == 0 else list(orig_sr)
    if len(srs) != B:
        raise ValueError(f'orig_sr must be one rate or one per waveform ({B}); got {len(srs)}')
    ratios = []
    for i, r in enumerate(srs):
        r = _rate(r, f'orig_sr[{i}]' if np.ndim(orig_sr) else 'orig_sr')
        up, down = resample_ratio(r, target)
        if max(up, down) > _lib.RESAMPLE_MAX_FACTOR:
            raise ValueError(f'waveforms[{i}]: {r} -> {target} Hz is the ratio {up}/{down}; max(up, down) must be at most '
                             f'{_lib.RESAMPLE_MAX_FACTOR}')
        ratios.append((up, down))
    out_len = [-(-n * up // down) for n, (up, down) in zip(b.lengths, ratios)]
    _offsets(out_len, 'output samples')
    work = [i for i, r in enumerate(ratios) if r != (1, 1)]
    outs = [None] * B
    with torch.cuda.device(b.device):
        for i in set(range(B)) - set(work):
            outs[i] = b.out(i, b.tensors[i].to(device=b.device, dtype=torch.float32, copy=True))
        if work:
            pairs = sorted({ratios[i] for i in work})
            tables = [_resample_table(up, down, b.device) for up, down in pairs]
            toff = _offsets([len(t) for t in tables], 'filter taps')
            plan = np.array([[up, down, 10 * max(up, down), toff[pairs.index((up, down))]] for up, down in (ratios[i] for i in work)],
                            dtype=np.int32)
            soff = _offsets([b.lengths[i] for i in work], 'samples')
            ooff = _offsets([out_len[i] for i in work], 'output samples')
            shape = _lib.ResampleShape(len(work), int(soff[-1]), int(ooff[-1]), int(toff[-1]), max(max(p) for p in pairs))
            wave = torch.cat([b.tensors[i].to(device=b.device, dtype=torch.float32) for i in work]).contiguous()
            d_soff, d_ooff = (torch.from_numpy(o.astype(np.int32)).to(b.device) for o in (soff, ooff))
            y = F.resample(shape, wave, d_soff, d_ooff, torch.from_numpy(plan).to(b.device), torch.cat(tables))
            for j, i in enumerate(work):
                outs[i] = b.out(i, y[ooff[j]:ooff[j + 1]])
    return outs


def resample(y, orig_sr, target_sr=None):
    """One waveform resampled from orig_sr to target_sr (default hp.sample_rate).  See resample_batch."""
    return resample_batch([y], orig_sr, target_sr)[0]


def trim_silence_batch(waveforms, window_ms, hop_ms, top_db=50, margin_ms=0):
    """Trim leading and trailing silence from each waveform [L_i] as the reference's trim_silence does (librosa 0.7.0 effects.trim):
    with W, hop and M = ms_to_frames of window_ms, hop_ms and margin_ms, the waveform is cropped to x[M:L - M] when M != 0, framed at hop
    with W-sample frames after reflect padding by W // 2, and each frame's mean square is compared in dB with the loudest frame's
    (power_to_db, amin 1e-10); frames above -top_db are non-silent.  -> one (trimmed, index) per waveform: index is int64 numpy
    [start, end] in the cropped signal (a hop, min(L - 2M, (b + 1) hop) for the first and last non-silent frames a and b; [0, 0] when
    there is none, as with top_db <= 0), and trimmed is the cropped waveform's [start:end], a slice of the caller's own array or tensor.
    An all-zero waveform comes back whole.  The decision is taken on the waveform rounded to fp32, with fp64 frame powers in the
    library's kernels (include/b200tts.h); the work runs on the device of the first CUDA input, else on the current CUDA device.  Raises
    ValueError on a bad or non-finite waveform, W < 1, hop < 1, a negative margin, a margin that leaves no samples, or a non-finite
    top_db."""
    b = _Batch(waveforms, 'trim_silence_batch', 'waveforms', finite=True)
    wf, hf, mf = ms_to_frames(window_ms), ms_to_frames(hop_ms), ms_to_frames(margin_ms)
    if wf < 1 or hf < 1:
        raise ValueError(f'window_ms = {window_ms} and hop_ms = {hop_ms} give {wf} and {hf} samples; each must be at least 1')
    if mf < 0:
        raise ValueError(f'margin_ms = {margin_ms} must not be negative')
    top_db = float(top_db)
    if not math.isfinite(top_db):
        raise ValueError(f'top_db = {top_db} must be finite')
    for i, n in enumerate(b.lengths):
        if 2 * mf >= n:
            raise ValueError(f'waveforms[{i}] has {n} samples; a margin of {mf} on each side leaves none')
    cropped = [n - 2 * mf for n in b.lengths]
    foff = _offsets([1 + (n + 2 * (wf // 2) - wf) // hf for n in cropped], 'frames')
    with torch.cuda.device(b.device):
        shape = _lib.TrimShape(len(b), int(b.off[-1]) - 2 * mf * len(b), int(foff[-1]), wf, hf, top_db)
        wave = torch.cat([t[mf:n - mf].to(device=b.device, dtype=torch.float32) for t, n in zip(b.tensors, b.lengths)]).contiguous()
        soff, d_foff = (torch.from_numpy(o.astype(np.int32)).to(b.device) for o in (_offsets(cropped, 'samples'), foff))
        _, bounds = F.trim_silence(shape, wave, soff, d_foff)
        bounds = bounds.cpu().numpy().astype(np.int64)
    out = []
    for x, n, (start, end) in zip(waveforms, b.lengths, bounds):
        x = x if isinstance(x, torch.Tensor) else np.asarray(x)
        out.append((x[mf:n - mf][int(start):int(end)], np.array([start, end], dtype=np.int64)))
    return out


def trim_silence(data, window_ms, hop_ms, top_db=50, margin_ms=0):
    """Trim leading and trailing silence from an audio signal (reference utils/audio.py:30-36) -> (trimmed, index).  See
    trim_silence_batch."""
    return trim_silence_batch([data], window_ms, hop_ms, top_db, margin_ms)[0]
