"""Text to audio in chunks: the Tacotron decoder stream feeding the WaveRNN stream, or the streaming Griffin-Lim vocoder
(modules/griffinlim.py: GriffinLimVocoder has the members used here; pass it where `wavernn` is taken, with
mel_transform=lambda m: utils.audio.denormalize_spectrogram(m, True) and preemphasis=hp.preemphasis).

Each stage lags the one before it by a bounded number of frames, whatever the utterance length:
  * the decoder runs in chunks of `chunk_frames` frames (Tacotron.inference_stream);
  * the post-net releases a frame once `Postnet.halo()` (10) decoded frames follow it, or the stop cut is known;
  * the vocoder runs its sample loop up to `WaveRNN.lookahead()` (2 at pad 2, factors 5 x 5 x 11) frames behind the last mel frame it has;
  * it holds back the last 20 hops of samples it has run until the mel ends, because the fade-out lands on them.
With a GriffinLimVocoder the vocoder processes frame m once `lookahead()` (3) frames follow it and releases its audio once no later frame
touches it (DESIGN 8.1).  Its streams need at least 2 frames instead of 21."""
from typing import Union

from .griffinlim import GriffinLimVocoder
from .tacotron2 import MAX_STREAM_TEXTS, Tacotron, _check_batch_inputs, _plan_lists
from .wavernn import WaveRNN

Vocoder = Union[WaveRNN, GriffinLimVocoder]


def speech_stream(tacotron: Tacotron, wavernn: Vocoder, text, speaker=None, language=None, mel_transform=None, chunk_frames=None,
                  uniforms=None, generator=None, preemphasis=0.0, target=None, overlap=None, durations=None, alignment=None):
    """Yields waveform chunks of `text` as the decoder produces it: tacotron.inference_stream(text, speaker, language, chunk_frames) fed,
    through mel_transform, into wavernn.generate_stream(…, uniforms, generator, preemphasis).  mel_transform (default: none) maps a
    post-net chunk [num_mels, n] to the vocoder's input frames [feat_dims, n] frame by frame, for example
    utils.audio.denormalize_spectrogram; it must not look at neighbouring frames, since each chunk is transformed alone.  The audio equals
    wavernn.generate(mel, target=F hop, overlap=0) of the concatenated transformed mel, bit for bit given the same uniform tape.  With
    target and overlap (folded streaming, WaveRNN.generate_stream's), it equals wavernn.generate(mel, target, overlap) instead.
    `durations` or `alignment` sets the decode's attention (Tacotron.inference)."""
    mels = tacotron.inference_stream(text, speaker, language, chunk_frames, durations, alignment)
    if mel_transform is not None:
        mels = (mel_transform(m) for m in mels)
    yield from wavernn.generate_stream(mels, uniforms, generator, preemphasis, target, overlap)


def speech_streams(tacotron: Tacotron, wavernn: Vocoder, texts, speakers=None, languages=None, mel_transform=None, chunk_frames=None,
                   uniforms=None, generator=None, preemphasis=0.0, target=None, overlap=None, durations=None, alignments=None):
    """speech_stream for up to 64 texts at once: yields (i, waveform chunk) for text i.  Every text is submitted to one SpeechServer(…,
    max_streams=len(texts)) at once and the server steps until it is idle: each step runs one decoder call over the texts still decoding
    (text i reads column i of a recorded mask tape), feeds its post-net chunks (through mel_transform) into the vocoder pool and makes one
    pool.run().  uniforms: None or one tape [1, T_i, U] per text ([K_i, target + 2 overlap, U] with target and overlap).  Each text's audio equals speech_stream of that text alone, bit for bit
    given its tape, in fp32 mode (where the decoded frames of a group equal those of single texts).  A text that decodes fewer than the
    vocoder's minimum (21 frames for a WaveRNN, 2 for a GriffinLimVocoder) raises ValueError when its stream ends, as speech_stream does, and
    that ends the generator for every text of the group.  durations / alignments: as Tacotron.inference_batch takes them."""
    texts = list(texts)
    if len(texts) > MAX_STREAM_TEXTS:
        raise ValueError(f'inference_streams: at most {MAX_STREAM_TEXTS} texts decode as one group (got {len(texts)})')
    if uniforms is not None and len(uniforms) != len(texts):
        raise ValueError(f'{len(uniforms)} uniform tapes for {len(texts)} texts')
    speakers, languages = _check_batch_inputs(texts, speakers, languages)
    durations, alignments = _plan_lists(texts, durations, alignments)
    server = SpeechServer(tacotron, wavernn, len(texts), mel_transform, chunk_frames, preemphasis, generator, target, overlap)
    ids = [server.submit(text, None if speakers is None else speakers[i], None if languages is None else languages[i],
                         uniforms=None if uniforms is None else uniforms[i], durations=durations[i], alignment=alignments[i])
           for i, text in enumerate(texts)]
    text_of = {rid: i for i, rid in enumerate(ids)}
    while server.pending or server.active:
        out = server.step()
        if server.failed:
            raise ValueError(next(iter(server.failed.values())))
        for rid, chunk in out.items():
            yield text_of[rid], chunk


class _Request:
    """One request of a SpeechServer: its inputs until admission, then its decoder text id (None once its mel has ended) and its vocoder
    stream id."""

    def __init__(self, text, speaker, language, seed, masks, uniforms, plan):
        self.inputs, self.plan = (text, speaker, language, seed, masks), plan
        self.uniforms, self.seed = uniforms, seed
        self.tid = self.sid = None


class SpeechServer:
    """Continuous-batching text-to-speech: requests join the running decoder group (Tacotron.decoder_pool) and the shared sample loop
    (WaveRNN.stream_pool) at any step() and leave at their stop cut.

    submit() queues a request -> its id.  Each step() admits queued requests in FIFO order while a vocoder row is free (a request holds
    its vocoder row from admission to its last sample, which covers its decoder row's lifetime, so the vocoder pool's max_streams is the
    only limit), makes one DecoderPool.run(), feeds the post-net chunks through mel_transform into the StreamPool (a request whose decode
    ended after the previous call gets its end()), makes one pool.run() and returns {id: waveform chunk}.  A request whose mel ends under
    the vocoder's minimum (21 frames for a WaveRNN, 2 for a GriffinLimVocoder) moves to `failed` ({id: message}) and frees its rows; the others go on.  cancel() drops a queued, decoding or vocoding
    request.  `pending` lists the queued ids in order, `active` the admitted ones.

    A request's audio is speech_stream of it alone, bit for bit in fp32 mode, given the same mask tape (`masks`, as DecoderPool.open takes
    it) and uniform tape (`uniforms` [1, T, U]), whatever joins or leaves around it.  With a `seed` instead, the masks and uniforms it does
    not get from a tape are drawn from the seed alone (_lib.SEED_STREAMS), so the request gives the same bits alone, in a full server, at
    any join call and at any chunk_frames.  Without either, its masks and uniforms come from draws shared with the other such requests of
    each call.

    With target and overlap the vocoder pool is a FoldedStreamPool: each request's audio is speech_stream(…, target, overlap) of it
    alone, which equals generate(mel, target, overlap) of its mel; tapes are [K, target + 2 overlap, U].  Admission stays at most
    max_streams requests; their folds share the loop's 64 rows."""

    def __init__(self, tacotron: Tacotron, wavernn: Vocoder, max_streams=64, mel_transform=None, chunk_frames=None, preemphasis=0.0,
                 generator=None, target=None, overlap=None):
        self.decoder = tacotron.decoder_pool(max_streams, chunk_frames)
        self.pool = wavernn.stream_pool(max_streams, preemphasis, generator, target, overlap)
        self.mel_transform = mel_transform
        self.requests = {}                     # id -> _Request, queued or admitted
        self.pending, self.failed = [], {}
        self.next_id = 0

    @property
    def active(self):
        return [rid for rid in self.requests if rid not in self.pending]

    def submit(self, text, speaker=None, language=None, seed=None, masks=None, uniforms=None, durations=None, alignment=None):
        """Queues a request -> its id.  Its inputs are checked now (ValueError).  `durations` or `alignment` sets its decode's attention
        (DecoderPool.open)."""
        plan = {k: v for k, v in (('durations', durations), ('alignment', alignment)) if v is not None}
        self.decoder.check(text, speaker, language, seed, masks, **plan)
        if uniforms is not None:
            self.pool.check_tape(uniforms)
        rid = self.next_id
        self.next_id += 1
        self.requests[rid] = _Request(text, speaker, language, seed, masks, uniforms, plan)
        self.pending.append(rid)
        return rid

    def cancel(self, rid):
        """Drops a queued, decoding or vocoding request."""
        req = self.requests.pop(rid, None)
        if req is None:
            raise ValueError(f'unknown or finished request {rid}')
        if rid in self.pending:
            self.pending.remove(rid)
            return
        if req.tid is not None and req.tid in self.decoder.ids:
            self.decoder.close(req.tid)
        self.pool.close(req.sid)

    def _admit(self):
        while self.pending and len(self.active) < self.pool.rows:
            rid = self.pending.pop(0)
            req = self.requests[rid]
            req.sid = self.pool.open(req.uniforms, req.seed)
            req.tid = self.decoder.open(*req.inputs, **req.plan)
            req.inputs = req.plan = None

    def _fail(self, rid, message):
        req = self.requests.pop(rid)
        self.pool.close(req.sid)
        self.failed[rid] = message

    def step(self):
        """One decoder call and one vocoder call -> {id: waveform chunk} for the requests that released samples."""
        self._admit()
        decoding = {req.tid: rid for rid, req in self.requests.items() if req.tid is not None}
        posts = self.decoder.run() if decoding else {}
        for tid, rid in decoding.items():
            req = self.requests[rid]
            if tid in posts:
                post = posts[tid]
                self.pool.feed(req.sid, post if self.mel_transform is None else self.mel_transform(post))
            else:                              # the decoder retired it after its previous call
                req.tid = None
                try:
                    self.pool.end(req.sid)
                except ValueError as exc:
                    self._fail(rid, str(exc))
        sid_of = {req.sid: rid for rid, req in self.requests.items() if req.sid is not None}
        out = {sid_of[sid]: chunk for sid, chunk in self.pool.run().items()}
        for sid, rid in sid_of.items():
            if sid not in self.pool.streams:   # its final chunk is out
                del self.requests[rid]
        return out
