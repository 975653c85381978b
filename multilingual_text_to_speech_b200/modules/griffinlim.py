"""Griffin-Lim as a streaming vocoder: frame-by-frame phase reconstruction with look-ahead (RTISI-LA; Zhu, Beauregard and Wyse, IEEE TASLP
2007), specified in DESIGN ("Griffin-Lim vocoder", "Streaming").

GriffinLimVocoder has the members the streaming layer calls on a WaveRNN (generate_stream, stream_pool, lookahead), so speech_stream,
speech_streams and SpeechServer run on it with mel_transform=utils.audio.denormalize_spectrogram and preemphasis=hp.preemphasis.  The
magnitudes of each frame are the batch vocoder's (b200tts_spectrogram_magnitude: dB -> amplitude, the FISTA NNLS for mel input,
** hp.griffin_lim_power); the frame loop runs on b200tts_gl_stream_run, one CTA per stream and call.

A stream cannot know its largest sample, so unlike utils.audio.inverse_spectrogram its output is not divided by max(y): scale it
afterwards if a peak of 1 is wanted."""
import numpy as np
import torch

from .. import _lib
from .. import functional as F
from ..params.params import Params as hp
from ..utils import audio
from .stream_pool import Stream, VocoderStreamPool, generate_stream as _generate_stream


class GriffinLimVocoder:
    """Streaming Griffin-Lim under the current hp: N = hp.num_fft, hop and window from hp.stft_shift_ms / hp.stft_window_ms, input bins
    hp.num_mels (mel=True) or N/2 + 1, hp.sample_rate and hp.griffin_lim_power, all read here.  Frame m is processed once `lookahead`
    (k) frames follow it or the stream has ended, with `iters` Jacobi iterations over the look-ahead set; its audio is released once no
    later frame touches it, so a stream's latency is k frames plus half a window.  Spectrograms go in as inverse_spectrogram takes them:
    log magnitudes in dB, already denormalised.  Invalid arguments raise ValueError here, before any device work."""

    def __init__(self, mel=True, lookahead=3, iters=32):
        for name, v, lo in (('lookahead', lookahead, 0), ('iters', iters, 1)):
            if isinstance(v, bool) or not isinstance(v, (int, np.integer)) or v < lo:
                raise ValueError(f'{name} must be an int >= {lo} (got {v!r})')
        self.mel, self.k, self.iters = bool(mel), int(lookahead), int(iters)
        self.N, self.hop, self.win = int(hp.num_fft), audio.ms_to_frames(hp.stft_shift_ms), audio.ms_to_frames(hp.stft_window_ms)
        self.K = self.N // 2 + 1
        self.n_mels = int(hp.num_mels)
        self.feat_dims = self.n_mels if self.mel else self.K
        self.sample_rate, self.power = int(hp.sample_rate), float(hp.griffin_lim_power)
        F.gl_stream_workspace_bytes(self.shape(1))         # the library's checks (FFT plan, window, hop, lookahead bound), host only

    def shape(self, slots, preemphasis=0.0):
        return _lib.GLStreamShape(self.N, self.hop, self.win, self.k, self.iters, int(slots), float(preemphasis))

    def lookahead(self):
        """Frames that must follow a frame before it is processed (k)."""
        return self.k

    def _check_chunk(self, chunk, i):
        as_numpy = not isinstance(chunk, torch.Tensor)
        t = torch.as_tensor(np.asarray(chunk) if as_numpy else chunk)
        if t.dim() != 2 or t.shape[0] != self.feat_dims:
            raise ValueError(f'spectrogram chunk {i} has shape {tuple(t.shape)}; expected [{self.feat_dims}, frames]')
        if not torch.is_floating_point(t):
            raise ValueError(f'spectrogram chunk {i} is not floating point')
        return t, as_numpy

    def magnitudes(self, log_frames):
        """Log spectrogram frames [n, bins] (frame-major fp32, n >= 1, on the current CUDA device) -> magnitudes [n, N/2 + 1] by
        b200tts_spectrogram_magnitude, as inverse_spectrogram_batch computes them: its kernels treat every frame alone, so a single frame is
        computed beside a zero frame that is then dropped."""
        n = int(log_frames.shape[0])
        x = log_frames if n >= 2 else torch.cat([log_frames, torch.zeros_like(log_frames)])
        shape = _lib.VocoderShape(1, int(x.shape[0]), self.N, self.hop, self.win, self.n_mels if self.mel else 0, self.power, audio.MOMENTUM,
                                  0.0, audio.NNLS_ITERS)
        if self.mel:
            basis, pinv_t, step = audio.mel_tables(self.sample_rate, self.N, self.n_mels, x.device)
            S = F.spectrogram_magnitude(shape, x, basis, pinv_t, step)
        else:
            S = F.spectrogram_magnitude(shape, x)
        return S[:n]

    min_stream_frames = 2            # as batch Griffin-Lim
    short_stream = 'the spectrogram stream ended after {} frames; Griffin-Lim needs at least 2'

    def generate_stream(self, mel_chunks, uniforms=None, generator=None, preemphasis=0.0, target=None, overlap=None):
        """Yields the waveform of the spectrogram chunks [bins, n_k] (n_k >= 0) as it is released: their concatenation, F >= 2 frames,
        gives hop (F - 1) samples in all (inverse_spectrogram's length and alignment), bit for bit the same however the chunks are cut.
        preemphasis: de-emphasis coefficient (0 = none), carried across chunks.  No peak normalisation.  uniforms, target and overlap exist
        for the WaveRNN signature and must be None; generator is unused.  Runs through a one-stream GriffinLimStreamPool on the device of
        the first CUDA chunk, or the current CUDA device, with one run() per non-empty chunk once 2 frames are in (a run processes every
        ready frame; a shorter stream is an error, found at its end); chunks come out as the first chunk went in (numpy, CUDA or CPU
        tensors)."""
        yield from _generate_stream(self, mel_chunks, uniforms, generator, preemphasis, target, overlap, self.min_stream_frames)

    def stream_pool(self, max_streams, preemphasis=0.0, generator=None, target=None, overlap=None):
        """A GriffinLimStreamPool of up to max_streams (1 to 64) streams.  generator is unused; target and overlap must be None."""
        if target is not None or overlap is not None:
            raise ValueError('Griffin-Lim streams are not folded: target and overlap are WaveRNN arguments')
        return GriffinLimStreamPool(self, max_streams, preemphasis)


class _GLStream(Stream):
    """One stream of a GriffinLimStreamPool: its slot, the frames fed but not yet sent to the device, and the host's copy of the slot's
    counters (frames received, frames committed)."""

    def __init__(self, slot):
        super().__init__()
        self.slot = slot
        self.pending = []        # [n, bins] fp32 frame-major tensors, in feed order
        self.fed = 0
        self.sent = 0
        self.committed = 0
        self.fresh = True        # its slot has not been reset yet

    @property
    def frames(self):
        return self.fed

    def append(self, spec):
        self.pending.append(spec.t().to(torch.float32))
        self.fed += int(spec.shape[1])


class GriffinLimStreamPool(VocoderStreamPool):
    """Concurrent streaming Griffin-Lim with StreamPool's interface: up to max_streams streams, each a generate_stream, in one workspace.
    open() takes the lowest free slot (uniforms must be None; a seed is checked and unused: nothing is drawn); feed() and end() add a
    stream's frames and mark its end; run() processes every ready frame of every stream and returns {sid: waveform chunk} (CUDA tensors)
    for the streams that released samples; a stream's slot is freed when its final chunk is returned, or at once by close().  open, feed,
    end and close do no device work; a run() makes a fixed number of launches whatever the number of streams: the slot resets of newly
    opened streams, the magnitudes of the new frames of all streams, and one b200tts_gl_stream_run with a CTA per stream.  Each stream's
    concatenated chunks equal its own generate_stream bit for bit, whatever joins or leaves around it.  Runs on `device`, by default the
    CUDA device that was current when the pool was made."""

    def __init__(self, vocoder, max_streams, preemphasis=0.0, device=None):
        super().__init__(vocoder, max_streams, preemphasis, device)
        self.shape = vocoder.shape(self.rows, self.a)
        F.gl_stream_workspace_bytes(self.shape)
        self.ws = None                         # allocated by the first run()
        self.slots = [None] * self.rows        # sid of the stream in each slot

    def check_tape(self, uniforms):
        """Griffin-Lim draws nothing: only None is accepted."""
        if uniforms is not None:
            raise ValueError('Griffin-Lim draws nothing: it takes no uniform tape')

    def _open(self, sid, tape, seed):
        slot = self.slots.index(None)
        self.slots[slot] = sid
        return _GLStream(slot)

    def _drop(self, st):
        self.slots[st.slot] = None

    def _committed_after(self, st):
        """Frames committed once the next run() has processed every ready frame."""
        return st.fed if st.ended else max(st.committed, st.fed - self.v.k)

    def _released(self, st, committed):
        """Output samples released once `committed` frames are committed: those below committed hop in the untrimmed signal, or all
        hop (F - 1) once the stream has ended and its last frame is committed (with lookahead 0 that frame may have been committed in an
        earlier call, before the end was known: the rest is released by the next run())."""
        if st.ended and committed == st.fed:
            return self.v.hop * (st.fed - 1)
        return max(0, committed * self.v.hop - self.v.N // 2)

    def _pending(self, st):
        return st.fed > st.sent or self._released(st, self._committed_after(st)) > st.released

    def _busy(self):
        return any(self._pending(st) for st in self.streams.values())

    def run(self):
        """Processes every ready frame of every stream -> {sid: the waveform chunk it releases}."""
        order = sorted(self.streams, key=lambda s: self.streams[s].slot)
        resets = [self.streams[s].slot for s in order if self.streams[s].fresh]
        work = [s for s in order if self._pending(self.streams[s])]
        if not resets and not work:
            return {}
        rows, logs, spans = [], [], {}
        s_off = wave_off = 0
        for sid in work:
            st = self.streams[sid]
            m1 = self._committed_after(st)
            n = self._released(st, m1) - st.released
            rows.append(_lib.GLStreamRow(st.slot, st.fed, int(st.ended), s_off, wave_off))
            logs += st.pending
            s_off += st.fed - st.sent
            spans[sid] = (wave_off, n, m1)
            wave_off += n
        with torch.cuda.device(self.device), torch.no_grad():
            if self.ws is None:
                self.ws = F.gl_stream_workspace(self.shape, self.device)
            if resets:
                F.gl_stream_reset(self.shape, self.ws, resets)
            wave = torch.empty(max(wave_off, 1), device=self.device, dtype=torch.float32)
            if rows:
                S_new = (self.v.magnitudes(torch.cat([t.to(self.device) for t in logs]).contiguous()) if logs else
                         torch.zeros(1, self.v.K, device=self.device, dtype=torch.float32))     # no new frames: not read
                F.gl_stream_run(self.shape, rows, S_new, wave, self.ws)
        for sid in order:
            self.streams[sid].fresh = False
        out = {}
        for sid, (off, n, m1) in spans.items():
            st = self.streams[sid]
            st.pending, st.sent, st.committed = [], st.fed, m1
            st.released += n
            if n:
                out[sid] = wave[off:off + n]
            if st.ended and m1 == st.fed:
                self.close(sid)
        return out
