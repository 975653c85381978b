"""Text to audio in chunks: the Tacotron decoder stream feeding the WaveRNN stream.

Each stage lags the one before it by a bounded number of frames, whatever the utterance length:
  * the decoder runs in chunks of `chunk_frames` frames (Tacotron.inference_stream);
  * the post-net releases a frame once `Postnet.halo()` (10) decoded frames follow it, or the stop cut is known;
  * the vocoder runs its sample loop up to `WaveRNN.lookahead()` (2 at pad 2, factors 5 x 5 x 11) frames behind the last mel frame it has;
  * it holds back the last 20 hops of samples it has run until the mel ends, because the fade-out lands on them."""
from .tacotron2 import Tacotron
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
