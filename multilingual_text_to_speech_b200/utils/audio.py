"""Audio with the reference's names (reference utils/audio.py:49-161; librosa 0.7.0): spectrogram -> waveform (mel_to_stft + griffinlim),
waveform -> log (mel) spectrogram (stft, melspectrogram, amplitude_to_db), MFCCs and the mel cepstral distortion.

Every stage runs in the library's kernels on the GPU whatever the precision mode is.  Spectrograms go in and out as [bins, F] (numpy or
torch); a batch is packed frame-major, and each result equals what its input gives on its own.  The rest of the dataset side (loading,
trimming, duration) and writing .wav files are not provided."""
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


def vocoder_shape(B, total_frames, mel):
    """The library shape of a batch under the current hp."""
    return _lib.VocoderShape(int(B), int(total_frames), int(hp.num_fft), ms_to_frames(hp.stft_shift_ms), ms_to_frames(hp.stft_window_ms),
                             int(hp.num_mels) if mel else 0, float(hp.griffin_lim_power), MOMENTUM,
                             float(hp.preemphasis) if hp.use_preemphasis else 0.0, NNLS_ITERS)


def inverse_spectrogram_batch(spectrograms, mel=False, phases=None, generator=None):
    """Log-magnitude spectrograms [bins, F_i] (already denormalised) -> one waveform per input, in input order, each of
    hop * (F_i - 1) samples.  `phases` (one [K, F_i] array of uniform draws in [0, 1) per input) sets the initial Griffin-Lim phases
    exp(2 pi i u); by default they are drawn with torch.rand on the device (`generator` optional), one draw for the whole packed batch.
    The work runs on the device of the first CUDA input, or on the current CUDA device when no input is on one.  numpy in -> numpy out;
    torch in -> torch out, on that device for CUDA inputs and on the CPU for CPU inputs."""
    if not isinstance(spectrograms, (list, tuple)) or len(spectrograms) == 0:
        raise ValueError('inverse_spectrogram_batch expects a non-empty list of [bins, frames] spectrograms')
    K = hp.num_fft // 2 + 1
    bins = hp.num_mels if mel else K
    as_numpy = [not isinstance(s, torch.Tensor) for s in spectrograms]
    specs = []
    for i, s in enumerate(spectrograms):
        t = torch.as_tensor(np.asarray(s) if as_numpy[i] else s)
        if t.dim() != 2 or t.shape[0] != bins:
            raise ValueError(f'spectrogram {i} has shape {tuple(t.shape)}; expected [{bins}, frames]')
        if t.shape[1] < 2:
            raise ValueError(f'spectrogram {i} has {t.shape[1]} frames; Griffin-Lim needs at least 2')
        if not torch.is_floating_point(t):
            raise ValueError(f'spectrogram {i} is not floating point')
        specs.append(t)
    frames = [s.shape[1] for s in specs]
    us = None
    if phases is not None:
        if len(phases) != len(specs):
            raise ValueError(f'{len(phases)} phase arrays for {len(specs)} spectrograms')
        us = []
        for i, p in enumerate(phases):
            p = torch.as_tensor(np.asarray(p) if not isinstance(p, torch.Tensor) else p)
            if tuple(p.shape) != (K, frames[i]):
                raise ValueError(f'phases {i} has shape {tuple(p.shape)}; expected [{K}, {frames[i]}]')
            us.append(p)
    device = next((s.device for s in specs if s.is_cuda), None)
    if device is None:
        device = torch.device('cuda', torch.cuda.current_device()) if torch.cuda.is_available() else torch.device('cuda')
    with torch.cuda.device(device):
        wave, off_host = _vocode(specs, us, frames, mel, generator, device)
    hop = ms_to_frames(hp.stft_shift_ms)
    out = []
    for i, f in enumerate(frames):
        w = wave[hop * (int(off_host[i]) - i): hop * (int(off_host[i]) - i + f - 1)]
        if as_numpy[i]:
            out.append(w.cpu().numpy())
        else:
            out.append(w if spectrograms[i].is_cuda else w.cpu())
    return out


def _vocode(specs, us, frames, mel, generator, device):
    """The library steps on `device` (the current CUDA device): packed waveform and host offsets."""
    K = hp.num_fft // 2 + 1
    off_host = np.concatenate([[0], np.cumsum(frames)]).astype(np.int32)
    total = int(off_host[-1])
    shape = vocoder_shape(len(specs), total, mel)
    ws = F.vocoder_workspace(shape, device)
    log_spec = torch.cat([s.to(device=device, dtype=torch.float32).t() for s in specs]).contiguous()
    off = torch.from_numpy(off_host).to(device)
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
    wave = torch.empty(shape.hop * (total - len(specs)), device=device, dtype=torch.float32)
    F.griffinlim(shape, S, off, angles, rebuilt, True, int(hp.griffin_lim_iters), wave, ws)
    F.deemphasis_normalize(shape, wave, off)
    return wave, off_host


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


def _work_device(tensors):
    """The device of the first CUDA tensor, else the current CUDA device."""
    device = next((t.device for t in tensors if t.is_cuda), None)
    if device is None:
        device = torch.device('cuda', torch.cuda.current_device()) if torch.cuda.is_available() else torch.device('cuda')
    return device


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


def _return_like(t, is_np, src):
    if is_np:
        return t.cpu().numpy()
    return t if src.is_cuda else t.cpu()


def spectrogram_batch(waveforms, mel=False):
    """Waveforms [L_i] -> log-magnitude (mel) spectrograms [bins, F_i], F_i = 1 + L_i // hop, in input order (reference
    utils/audio.py:66-78): pre-emphasis (hp.use_preemphasis), |stft| with centre reflect padding, the mel projection when `mel`, then
    amplitude_to_db relative to each utterance's own maximum.  Waveforms are computed in fp32: a float64 input is rounded to fp32 first (16-bit
    PCM scaled by 2^-15 is exact); the transform itself runs in fp64.  The work runs on the device of the first CUDA input, or on the current
    CUDA device when no input is on one.  numpy in -> numpy out; torch in -> torch out, on that device for CUDA inputs and on the CPU for CPU
    inputs."""
    if not isinstance(waveforms, (list, tuple)) or len(waveforms) == 0:
        raise ValueError('spectrogram_batch expects a non-empty list of 1-D waveforms')
    ins = [_as_float_tensor(w, f'waveform {i}', 1) for i, w in enumerate(waveforms)]
    waves = [t for t, _ in ins]
    hop = ms_to_frames(hp.stft_shift_ms)
    lengths = [int(w.numel()) for w in waves]
    frames = [1 + n // hop for n in lengths]
    soff_host = np.concatenate([[0], np.cumsum(lengths)]).astype(np.int64)
    off_host = np.concatenate([[0], np.cumsum(frames)]).astype(np.int64)
    if soff_host[-1] >= 2 ** 31:
        raise ValueError(f'{soff_host[-1]} samples in one batch; at most 2^31 - 1')
    device = _work_device(waves)
    with torch.cuda.device(device):
        shape = analysis_shape(len(waves), soff_host[-1], off_host[-1], mel)
        wave = torch.cat([w.to(device=device, dtype=torch.float32) for w in waves]).contiguous()
        soff = torch.from_numpy(soff_host.astype(np.int32)).to(device)
        off = torch.from_numpy(off_host.astype(np.int32)).to(device)
        basis = mel_tables(hp.sample_rate, hp.num_fft, hp.num_mels, device)[0] if mel else None
        S = F.stft_magnitude(shape, wave, soff, off, basis)
        F.amplitude_to_db(shape, S, off, out=S)
    return [_return_like(S[off_host[i]:off_host[i + 1]].t().contiguous(), ins[i][1], waves[i]) for i in range(len(waves))]


def spectrogram(y, mel=False):
    """Convert waveform to log-magnitude spectrogram [bins, 1 + len(y) // hop] (reference utils/audio.py:66-73)."""
    return spectrogram_batch([y], mel)[0]


def mel_spectrogram(y):
    """Convert waveform to log-mel-spectrogram."""
    return spectrogram(y, True)


def _cepstra(specs, device):
    """[n_mels, F_i] tensors -> packed cepstra [sum F, n_mfcc] on `device` and host frame offsets."""
    off_host = np.concatenate([[0], np.cumsum([s.shape[1] for s in specs])]).astype(np.int64)
    mel_db = torch.cat([s.to(device=device, dtype=torch.float32).t() for s in specs]).contiguous()
    return F.mel_cepstrum(mel_db, hp.num_mfcc), off_host


def _check_mfcc_input(S, what):
    t, is_np = _as_float_tensor(S, what, 2)
    if t.shape[0] < hp.num_mfcc:
        raise ValueError(f'{what} has {t.shape[0]} mel bands; hp.num_mfcc = {hp.num_mfcc} needs at least as many')
    return t, is_np


def get_spectrogram_mfcc(S):
    """Compute MFCCs [hp.num_mfcc, F] of a log-mel spectrogram [n_mels, F]: librosa 0.7.0 mfcc(S=S/10), the orthonormal DCT-II over the
    mel axis, c0 included (reference utils/audio.py:117-119)."""
    t, is_np = _check_mfcc_input(S, 'spectrogram')
    device = _work_device([t])
    with torch.cuda.device(device):
        cep, _ = _cepstra([t], device)
    return _return_like(cep.t().contiguous(), is_np, t)


def mel_cepstral_distortion_batch(S1s, S2s, mode='dtw'):
    """Mel cepstral distortion of each pair (S1s[i], S2s[i]) of log-mel spectrograms [n_mels, F] (reference mel_cepstral_distorision, utils/
    audio.py:127-161): MFCCs without c0, then the mean Euclidean frame distance over the frames paired by `mode`: 'cut' (the first min(F1, F2)
    frames), 'stretch' (the shorter sequence indexed at i * n // m) or 'dtw'.  'dtw' is the exact dynamic-time-warping optimum, cost / path
    length; the reference calls fastdtw with radius 1, which approximates that optimum, so the two agree when fastdtw finds the optimal path
    and may differ otherwise.  Returns float64, one value per pair: a numpy array unless the first
    input is a torch tensor (then a torch tensor on its device).  The work runs on the device of the first CUDA input, else on the current
    device."""
    if not isinstance(S1s, (list, tuple)) or not isinstance(S2s, (list, tuple)) or len(S1s) == 0:
        raise ValueError('mel_cepstral_distortion_batch expects two non-empty lists of [n_mels, frames] spectrograms')
    if len(S1s) != len(S2s):
        raise ValueError(f'{len(S1s)} spectrograms against {len(S2s)}')
    if mode not in _lib.MCD_MODES:
        raise ValueError(f'unknown mode {mode!r}; expected one of {sorted(_lib.MCD_MODES)}')
    a = [_check_mfcc_input(s, f'S1s[{i}]') for i, s in enumerate(S1s)]
    b = [_check_mfcc_input(s, f'S2s[{i}]') for i, s in enumerate(S2s)]
    for i, ((x, _), (y, _)) in enumerate(zip(a, b)):
        if x.shape[0] != y.shape[0]:
            raise ValueError(f'pair {i} has {x.shape[0]} and {y.shape[0]} mel bands')
        if mode == 'dtw' and min(x.shape[1], y.shape[1]) > _lib.DTW_MAX_FRAMES:
            raise ValueError(f'pair {i} ({x.shape[1]} x {y.shape[1]} frames): dtw keeps three anti-diagonals in shared memory, so the shorter '
                             f'sequence may have at most {_lib.DTW_MAX_FRAMES} frames')
    xs, ys = [t for t, _ in a], [t for t, _ in b]
    device = _work_device(xs + ys)
    with torch.cuda.device(device):
        cep_a, off_a = _cepstra(xs, device)
        cep_b, off_b = _cepstra(ys, device)
        mcd, _ = F.mel_cepstral_distortion(cep_a, torch.from_numpy(off_a.astype(np.int32)).to(device), cep_b,
                                           torch.from_numpy(off_b.astype(np.int32)).to(device), mode)
    return _return_like(mcd, a[0][1], xs[0])


def mel_cepstral_distorision(S1, S2, mode):
    """Compute Mel Cepstral Distorsion between two mel spectrograms (reference spelling; see mel_cepstral_distortion_batch).

    Arguments:
        S1 and S2 -- mel spectrograms
        mode -- 'cut' to cut off frames of longer seq.
                'stretch' to stretch linearly the shorter seq.
                'dtw' to compute DTW with minimal possible MCD (exact DTW, not fastdtw's approximation)
    """
    return float(mel_cepstral_distortion_batch([S1], [S2], mode)[0])
