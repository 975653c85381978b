"""Text to audio in chunks: the Tacotron decoder stream feeding the WaveRNN stream.

Each stage lags the one before it by a bounded number of frames, whatever the utterance length:
  * the decoder runs in chunks of `chunk_frames` frames (Tacotron.inference_stream);
  * the post-net releases a frame once `Postnet.halo()` (10) decoded frames follow it, or the stop cut is known;
  * the vocoder runs its sample loop up to `WaveRNN.lookahead()` (2 at pad 2, factors 5 x 5 x 11) frames behind the last mel frame it has;
  * it holds back the last 20 hops of samples it has run until the mel ends, because the fade-out lands on them."""
from .tacotron2 import MAX_STREAM_TEXTS, Tacotron
from .wavernn import WaveRNN


def speech_stream(tacotron: Tacotron, wavernn: WaveRNN, text, speaker=None, language=None, mel_transform=None, chunk_frames=None,
                  uniforms=None, generator=None, preemphasis=0.0):
    """Yields waveform chunks of `text` as the decoder produces it: tacotron.inference_stream(text, speaker, language, chunk_frames) fed,
    through mel_transform, into wavernn.generate_stream(…, uniforms, generator, preemphasis).  mel_transform (default: none) maps a
    post-net chunk [num_mels, n] to the vocoder's input frames [feat_dims, n] frame by frame, for example
    utils.audio.denormalize_spectrogram; it must not look at neighbouring frames, since each chunk is transformed alone.  The audio equals
    wavernn.generate(mel, target=F hop, overlap=0) of the concatenated transformed mel, bit for bit given the same uniform tape."""
    mels = tacotron.inference_stream(text, speaker, language, chunk_frames)
    if mel_transform is not None:
        mels = (mel_transform(m) for m in mels)
    yield from wavernn.generate_stream(mels, uniforms, generator, preemphasis)


def speech_streams(tacotron: Tacotron, wavernn: WaveRNN, texts, speakers=None, languages=None, mel_transform=None, chunk_frames=None,
                   uniforms=None, generator=None, preemphasis=0.0):
    """speech_stream for up to 64 texts at once: yields (i, waveform chunk) for text i.  Each round runs one decoder call of
    tacotron.inference_streams(texts, speakers, languages, chunk_frames), feeds its post-net chunks (through mel_transform) into one
    wavernn.stream_pool(len(texts), preemphasis, generator), and makes one pool.run(); once the decoder is done, the pool runs until every
    stream has ended.  uniforms: None or one tape [1, T_i, U] per text.  Each text's audio equals speech_stream of that text alone, bit for
    bit given its tape, in fp32 mode (where the decoded frames of a group equal those of single texts).  A text that decodes fewer than
    21 frames raises ValueError when its stream ends, as speech_stream does, and that ends the generator for every text of the group."""
    texts = list(texts)
    if len(texts) > MAX_STREAM_TEXTS:
        raise ValueError(f'inference_streams: at most {MAX_STREAM_TEXTS} texts decode as one group (got {len(texts)})')
    if uniforms is not None and len(uniforms) != len(texts):
        raise ValueError(f'{len(uniforms)} uniform tapes for {len(texts)} texts')
    decoder = tacotron.inference_streams(texts, speakers, languages, chunk_frames)
    pool = wavernn.stream_pool(len(texts), preemphasis, generator)
    sids = [pool.open(None if uniforms is None else uniforms[i]) for i in range(len(texts))]
    text_of = {sid: i for i, sid in enumerate(sids)}
    ended = set()
    for posts in decoder:
        for i, post in posts.items():
            pool.feed(sids[i], post if mel_transform is None else mel_transform(post))
        for i in range(len(texts)):
            if i not in ended and i not in posts:                # the decoder retired text i after its previous call
                pool.end(sids[i])
                ended.add(i)
        for sid, chunk in pool.run().items():
            yield text_of[sid], chunk
    for i in range(len(texts)):
        if i not in ended:
            pool.end(sids[i])
    while pool.streams:
        for sid, chunk in pool.run().items():
            yield text_of[sid], chunk
