"""Static hyper-parameter singleton, imported everywhere as ``hp``.

Mirrors the public surface of the reference's ``params/params.py:4-164`` (class ``Params`` with
class-level attributes, ``load``/``save``/``state_dict``/``load_state_dict``/``symbols_count``) so
that ``train.py`` / ``synthesize.py`` / checkpoints that carry ``state['parameters']`` keep working.
Attribute *names and default values* are the contract; the implementation is ours (a defaults table
installed on the class at import time).

Extra (new) attributes, all with defaults that reproduce the reference behaviour:
  * ``b200_precision``  -- "fp32" (parity mode) or "bf16" (tensor-core perf mode) for the CUDA hot path.
  * ``outputs_per_step`` -- reduction factor r: mel frames predicted per decoder step (1 = the reference's decoder).  A decode of T
    frames runs ceil(T / r) sequential steps; the alignment has one row per step.
"""
import json

_TRAINING = dict(
    version="1.0",
    epochs=300,
    batch_size=52,
    learning_rate=1e-3,
    learning_rate_decay=0.5,
    learning_rate_decay_start=15000,
    learning_rate_decay_each=15000,
    learning_rate_encoder=1e-3,
    weight_decay=1e-6,
    encoder_optimizer=False,
    max_output_length=5000,
    gradient_clipping=0.25,
    reversal_gradient_clipping=0.25,
    guided_attention_loss=True,
    guided_attention_steps=20000,
    guided_attention_toleration=0.25,
    guided_attention_gain=1.00025,
    constant_teacher_forcing=True,
    teacher_forcing=1.0,
    teacher_forcing_steps=100000,
    teacher_forcing_start_steps=50000,
    checkpoint_each_epochs=10,
    parallelization=True,
)

_DATASET = dict(
    dataset="ljspeech",
    cache_spectrograms=True,
    languages=["en-us"],
    balanced_sampling=False,
    perfect_sampling=False,
)

_TEXT = dict(
    characters="ABCDEFGHIJKLMNOPQRSTUVWXYZabcdefghijklmnopqrstuvwxyz ",
    case_sensitive=True,
    remove_multiple_wspaces=True,
    use_punctuation=True,
    punctuations_out='、。，"(),.:;¿?¡!\\',
    punctuations_in="'-",
    use_phonemes=False,
    phonemes="ɹɐpbtdkɡfvθðszʃʒhmnŋlrwjeəɪɒuːɛiaʌʊɑɜɔx ",
)

_MODEL = dict(
    embedding_dimension=512,
    encoder_type="simple",          # simple | separate | shared | convolutional | generated
    encoder_dimension=512,
    encoder_blocks=3,
    encoder_kernel_size=5,
    generator_dim=8,
    generator_bottleneck_dim=4,
    prenet_dimension=256,
    prenet_layers=2,
    attention_type="location_sensitive",
    attention_dimension=128,
    attention_kernel_size=31,
    attention_location_dimension=32,
    decoder_dimension=1024,
    decoder_regularization="dropout",   # dropout | zoneout
    zoneout_hidden=0.1,
    zoneout_cell=0.1,
    dropout_hidden=0.1,
    postnet_dimension=512,
    postnet_blocks=5,
    postnet_kernel_size=5,
    dropout=0.5,
    predict_linear=False,
    cbhg_bank_kernels=8,
    cbhg_bank_dimension=128,
    cbhg_projection_kernel_size=3,
    cbhg_projection_dimension=256,
    cbhg_highway_dimension=128,
    cbhg_rnn_dim=128,
    cbhg_dropout=0.0,
    multi_speaker=False,
    multi_language=False,
    speaker_embedding_dimension=32,
    language_embedding_dimension=4,
    input_language_embedding=4,
    reversal_classifier=False,
    reversal_classifier_type="reversal",
    reversal_classifier_dim=256,
    reversal_classifier_w=1.0,
    stop_frames=5,
    speaker_number=0,               # filled in by the training script
    language_number=0,              # filled in by the training script
)

_AUDIO = dict(
    sample_rate=22050,
    num_fft=1102,
    num_mels=80,
    num_mfcc=13,
    stft_window_ms=50,
    stft_shift_ms=12.5,
    griffin_lim_iters=60,
    griffin_lim_power=1.5,
    normalize_spectrogram=True,
    use_preemphasis=True,
    preemphasis=0.97,
)

_B200 = dict(
    b200_precision="fp32",
    outputs_per_step=1,
)

_DEFAULTS = {}
for _group in (_TRAINING, _DATASET, _TEXT, _MODEL, _AUDIO, _B200):
    _DEFAULTS.update(_group)


class Params:
    """Global mutable configuration (class attributes only; never instantiated)."""

    @staticmethod
    def reset():
        """Restore every attribute to its default (handy between tests; JSON loads are cumulative)."""
        for key, value in _DEFAULTS.items():
            setattr(Params, key, list(value) if isinstance(value, list) else value)

    @staticmethod
    def load_state_dict(d):
        for key, value in d.items():
            setattr(Params, key, value)

    @staticmethod
    def state_dict():
        names = [n for n in dir(Params) if not n.startswith("__") and not callable(getattr(Params, n))]
        return {n: getattr(Params, n) for n in names}

    @staticmethod
    def load(json_path):
        with open(json_path, "r", encoding="utf-8") as handle:
            Params.load_state_dict(json.load(handle))

    @staticmethod
    def save(json_path):
        with open(json_path, "w", encoding="utf-8") as handle:
            json.dump(Params.state_dict(), handle, indent=4)

    @staticmethod
    def symbols_count():
        count = len(Params.phonemes) if Params.use_phonemes else len(Params.characters)
        if Params.use_punctuation:
            count += len(Params.punctuations_out) + len(Params.punctuations_in)
        return count


Params.reset()
