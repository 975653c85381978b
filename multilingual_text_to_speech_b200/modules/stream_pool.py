"""The stream contract the vocoder stream pools share (WaveRNN's StreamPool and FoldedStreamPool, GriffinLimStreamPool): open / feed / end /
run / drain / close, `streams` and `rows`, and the generate_stream driver that runs a vocoder through a one-stream pool.

VocoderStreamPool owns the argument checks, the stream ids and the errors of that contract; each pool keeps its own device policy (the
loop rows or slots a stream takes, what run() does) behind the hooks check_tape, _open, _drop, _busy and run."""
import contextlib

import numpy as np
import torch

from .. import _lib
from ..utils.audio import _return_like, _work_device


def check_preemphasis(preemphasis):
    if not -1.0 < float(preemphasis) < 1.0:
        raise ValueError(f'preemphasis {preemphasis} must lie in (-1, 1)')
    return float(preemphasis)


def check_seed(seed):
    """None, or an int in [0, 2^64) -> itself as an int (ValueError otherwise)."""
    if seed is None:
        return None
    if isinstance(seed, bool) or not isinstance(seed, (int, np.integer)) or not 0 <= int(seed) < 1 << 64:
        raise ValueError(f'a seed is an int in [0, 2^64) (got {seed!r})')
    return int(seed)


class Stream:
    """One stream's host bookkeeping: the chunks fed, the samples released and whether its input has ended.  A pool's stream type adds
    `frames` (the frames fed) and append(spec)."""

    def __init__(self):
        self.chunks = 0
        self.released = 0
        self.ended = False


class VocoderStreamPool:
    """Up to max_streams (1 to 64) concurrent streams of one vocoder.  open() checks the tape (check_tape) and seed, then hands the stream
    to the pool (_open); feed() checks a chunk with v._check_chunk (v: the vocoder) and appends it; end() needs v.min_stream_frames
    frames; close() drops a stream at once (_drop); run() is the pool's; drain() runs until no stream has work left (_busy).  Every
    check here comes before any device work.  device: by default the CUDA device that is current when the pool is made."""

    def __init__(self, vocoder, max_streams, preemphasis=0.0, device=None):
        if isinstance(max_streams, bool) or not isinstance(max_streams, (int, np.integer)) or not 1 <= max_streams <= _lib.WAVERNN_MAX_STREAMS:
            raise ValueError(f'a stream pool holds 1 to {_lib.WAVERNN_MAX_STREAMS} streams (got {max_streams!r})')
        self.v, self.a = vocoder, check_preemphasis(preemphasis)
        self.rows = int(max_streams)
        self.device = _work_device() if device is None else device
        self.streams = {}
        self.next_sid = 0

    def open(self, uniforms=None, seed=None):
        """A new stream -> its id.  uniforms: its tape as check_tape takes it, or None; seed: None or an int in [0, 2^64)."""
        tape = self.check_tape(uniforms)
        seed = check_seed(seed)
        if len(self.streams) >= self.rows:
            raise ValueError(f'the stream pool is full: {self.rows} streams are open')
        sid = self.next_sid
        self.streams[sid] = self._open(sid, tape, seed)
        self.next_sid += 1
        return sid

    def close(self, sid):
        """Drops stream sid and frees what it holds at once, whatever it has run or released."""
        st = self.streams.pop(sid, None)
        if st is None:
            raise ValueError(f'unknown or finished stream {sid}')
        self._drop(st)

    def _stream(self, sid):
        st = self.streams.get(sid)
        if st is None:
            raise ValueError(f'unknown or finished stream {sid}')
        if st.ended:
            raise ValueError(f'stream {sid} has ended')
        return st

    def feed(self, sid, chunk):
        """Appends frames [feat_dims, n] (n >= 0, as given) to stream sid."""
        st = self._stream(sid)
        spec, _ = self.v._check_chunk(chunk, st.chunks)
        st.chunks += 1
        if spec.shape[1]:
            st.append(spec)

    def end(self, sid):
        """Marks the end of stream sid's input (at least v.min_stream_frames frames)."""
        st = self._stream(sid)
        if st.frames < self.v.min_stream_frames:
            raise ValueError(self.v.short_stream.format(st.frames))
        st.ended = True

    def drain(self):
        """Runs until no stream has work left -> the non-empty {sid: chunk} results, in order."""
        out = []
        while True:
            busy = self._busy()
            r = self.run()
            if r:
                out.append(r)
            if not busy:
                return out


def generate_stream(vocoder, chunks, uniforms, generator, preemphasis, target, overlap, first_run):
    """A vocoder's generate_stream: one stream of a one-stream vocoder.stream_pool(1, preemphasis, generator, target, overlap), made on
    the device of the first chunk if it is a CUDA tensor (else the current CUDA device) and opened with `uniforms`.  Each non-empty chunk
    is fed, then, once the stream holds `first_run` frames, the pool is drained; the end is drained too.  Yields the stream's chunks as
    the first chunk went in: numpy, CUDA tensors or CPU tensors."""
    pool = sid = fmt = None
    for i, chunk in enumerate(chunks):
        spec, as_numpy = vocoder._check_chunk(chunk, i)
        if pool is None:
            fmt = (as_numpy, spec)
            with torch.cuda.device(spec.device) if spec.is_cuda else contextlib.nullcontext():
                pool = vocoder.stream_pool(1, preemphasis, generator, target, overlap)
            sid = pool.open(uniforms)
        if spec.shape[1]:
            pool.feed(sid, spec)
            if pool.streams[sid].frames >= first_run:
                for out in pool.drain():
                    yield _return_like(out[sid], *fmt)
    if pool is None:
        raise ValueError(vocoder.short_stream.format(0))
    pool.end(sid)
    for out in pool.drain():
        yield _return_like(out[sid], *fmt)
