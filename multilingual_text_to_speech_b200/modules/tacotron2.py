"""Tacotron 2 model (surface of reference modules/tacotron2.py:15-485) on the b200tts library.

Constructor signatures, attribute names (`_embedding`, `_encoder`, `_prenet`, `_attention`, `_decoder`, `_postnet`,
`_reversal_classifier`), parameter names / shapes and forward / inference signatures follow the reference so that
train.py, synthesize.py and existing checkpoints work unchanged.  All arithmetic of the hot path is inside the
library: `Decoder` is ONE fused op (forward + hand-written BPTT), encoders / postnet are fused conv-block ops.
"""
import numpy as np
import torch
from torch.nn import functional as TF
from torch.nn import Sequential, ModuleList, Linear, ReLU, Embedding

from .. import functional as F
from .. import _lib
from ..rng import MaskSource
from ..params.params import Params as hp
from ..utils import lengths_to_mask
from .layers import ZoneoutLSTMCell, DropoutLSTMCell, ConvBlock
from .attention import LocationSensitiveAttention, ForwardAttention
from .encoder import Encoder, MultiEncoder, ConditionalEncoder, ConvolutionalEncoder, GeneratedConvolutionalEncoder
from .classifier import ReversalClassifier


class Prenet(torch.nn.Module):
    """2 x (Linear -> ReLU -> dropout that stays on during inference) (tacotron2.py:15-46).

    In training the prenet over all target frames runs inside the fused decoder op; this module owns the parameters
    and offers the standalone forward used for free-running / inference frames."""

    def __init__(self, input_dim, output_dim, num_layers, dropout):
        super().__init__()
        assert num_layers > 0, 'There must be at least one layer in the pre-net.'
        self._dropout_rate = dropout
        self._activation = ReLU()
        self._layers = ModuleList([Linear(input_dim, output_dim)] + [Linear(output_dim, output_dim) for _ in range(num_layers - 1)])

    def forward(self, x):
        for j, layer in enumerate(self._layers):
            x = torch.relu(F.linear(x, layer.weight, layer.bias))
            keep = MaskSource.keep_mask(f'prenet_standalone{j}', x.shape, self._dropout_rate, x.device)
            if keep is not None:
                x = x * keep * (1.0 / (1.0 - self._dropout_rate))
        return x


class Postnet(torch.nn.Module):
    """5 x (conv5 + BN + tanh + dropout) with a residual connection (tacotron2.py:49-76)."""

    def __init__(self, input_dimension, postnet_dimension, num_blocks, kernel_size, dropout):
        super().__init__()
        assert num_blocks > 1, 'There must be at least two convolutional blocks in the post-net.'
        blocks = [ConvBlock(input_dimension, postnet_dimension, kernel_size, dropout, 'tanh')] + \
                 [ConvBlock(postnet_dimension, postnet_dimension, kernel_size, dropout, 'tanh') for _ in range(num_blocks - 2)] + \
                 [ConvBlock(postnet_dimension, input_dimension, kernel_size, dropout, 'identity')]
        for j, block in enumerate(blocks):
            block._mask_key = f'post{j}'
        self._convs = Sequential(*blocks)

    def forward(self, x, x_lengths, padded=False):
        """padded (eval only): every frame of x at or after x_lengths[b] is 0, and so is every block output there."""
        if padded:
            lengths = x_lengths.to(device=x.device, dtype=torch.int32)
            y = x.contiguous()
            for block in self._convs:
                y = block(y, lengths)
            return y + x
        return self._convs(x.contiguous()) + x


class Decoder(torch.nn.Module):
    """Attention LSTM -> location-sensitive or forward attention -> generator LSTM -> frame / stop projections
    (tacotron2.py:79-219), executed by b200tts_decoder_forward / _backward.

    With `outputs_per_step` = r > 1 each decoder step predicts r frames (row block j of the projections = frame j of the step, one stop
    logit per frame) and is fed the last frame of the previous step: T frames take ceil(T / r) sequential steps.  The alignment then has
    one row per step."""

    def __init__(self, output_dim, decoder_dim, attention, generator_rnn, attention_rnn, context_dim, prenet, prenet_dim, max_frames,
                 outputs_per_step=1):
        super().__init__()
        self._outputs_per_step = r = int(outputs_per_step)
        if r < 1:
            raise ValueError(f'outputs_per_step must be >= 1 (got {r})')
        self._prenet = prenet
        self._attention = attention
        self._output_dim = output_dim
        self._decoder_dim = decoder_dim
        self._max_frames = max_frames
        self._attention_lstm = attention_rnn
        self._generator_lstm = generator_rnn
        self._frame_prediction = Linear(context_dim + decoder_dim, r * output_dim)
        self._stop_prediction = Linear(context_dim + decoder_dim, r)
        self._speaker_embedding, self._language_embedding = None, None
        if hp.multi_speaker and hp.speaker_embedding_dimension > 0:
            self._speaker_embedding = self._get_embedding(hp.speaker_embedding_dimension, hp.speaker_number)
        if hp.multi_language and hp.language_embedding_dimension > 0:
            self._language_embedding = self._get_embedding(hp.language_embedding_dimension, len(hp.languages))

    def _get_embedding(self, embedding_dimension, size=None):
        embedding = Embedding(size, embedding_dimension)
        torch.nn.init.xavier_uniform_(embedding.weight)
        return embedding

    def _add_conditional_embedding(self, encoded, layer, condition):
        return torch.cat((encoded, F.embedding(layer.weight, condition)), dim=-1)

    def _param_list(self):
        pre, att = self._prenet._layers, self._attention
        assert len(pre) == 2, 'the fused decoder implements the 2-layer prenet used by every configuration'
        a, g = self._attention_lstm, self._generator_lstm
        # forward attention has no location weights: None selects it in the fused op
        loc, loc_features = getattr(att, '_location', None), getattr(att, '_loc_features', None)
        return [pre[0].weight, pre[0].bias, pre[1].weight, pre[1].bias,
                a.weight_ih, a.weight_hh, a.bias_ih, a.bias_hh, g.weight_ih, g.weight_hh, g.bias_ih, g.bias_hh,
                att._query.weight, att._memory.weight, loc.weight if loc is not None else None,
                loc_features.weight if loc_features is not None else None,
                att._bias, att._energy.weight, self._frame_prediction.weight, self._frame_prediction.bias,
                self._stop_prediction.weight, self._stop_prediction.bias]

    def _cell_config(self):
        cell = self._attention_lstm
        if isinstance(cell, ZoneoutLSTMCell):
            return _lib.CELL_ZONEOUT, cell.zoneout_h, cell.zoneout_c
        return _lib.CELL_DROPOUT, cell._dropout.p, 0.0

    def _steps(self, frames):
        return -(-int(frames) // self._outputs_per_step)

    def _masks(self, B, T, device, teacher):
        """Keep masks for one decode of T steps, time-major.  With a mask tape active the reference's own draws are replayed."""
        P, D = self._prenet._layers[0].weight.shape[0], self._decoder_dim
        kind, rate_h, rate_c = self._cell_config()
        masks = {}
        tape = MaskSource.tape
        for name in ('prenet0', 'prenet1'):
            if tape is not None:        # tape layout is the reference's [B, T+1, P]; row T is drawn but never consumed
                t = tape.get(name)
                if t is not None:
                    masks[name] = t[:, :T].transpose(0, 1).contiguous().to(device=device, dtype=torch.uint8)
            else:
                masks[name] = MaskSource.keep_mask(name, (T, B, P), self._prenet._dropout_rate, device)
        if teacher is not None:
            for name in ('step_prenet0', 'step_prenet1'):
                masks[name] = MaskSource.keep_mask(name, (T, B, P), self._prenet._dropout_rate, device)
        if self.training:
            names = ('att_h', 'gen_h') + (('att_c', 'gen_c') if kind == _lib.CELL_ZONEOUT else ())
            for name in names:
                rate = rate_c if name.endswith('_c') else rate_h
                masks[name] = MaskSource.keep_mask(name, (T, B, D), rate, device)
        return {k: v for k, v in masks.items() if v is not None}

    @staticmethod
    def _stop_cut(stop_logits, stop_frames):
        """Number of frames the reference's inference loop returns (tacotron2.py:201-207): the frame on which the stop
        token (sigmoid >= 0.5, i.e. logit >= 0) has fired for the (stop_frames + 1)-th time, else all frames."""
        remaining = -1
        for i, fired in enumerate((stop_logits >= 0).tolist()):
            if not fired:
                continue
            if remaining == -1:
                remaining = stop_frames
                continue
            remaining -= 1
            if remaining == 0:
                return i + 1
        return len(stop_logits)

    # frames decoded per library call in inference (rounded down to whole steps): the stop rule (one device -> host read of the chunk's stop
    # logits) runs between chunks
    inference_chunk = 128

    class _StopRule:
        """Streaming form of the reference's inference exit (tacotron2.py:201-207): returns the number of frames to keep once the stop
        token (sigmoid >= 0.5, i.e. logit >= 0) has fired for the (stop_frames + 1)-th time."""

        def __init__(self, stop_frames):
            self.stop_frames, self.remaining, self.seen, self.cut = stop_frames, -1, 0, None

        def feed(self, logits):
            for fired in (logits >= 0).tolist():
                self.seen += 1
                if self.cut is not None or not fired:
                    continue
                if self.remaining == -1:
                    self.remaining = self.stop_frames
                    continue
                self.remaining -= 1
                if self.remaining == 0:
                    self.cut = self.seen
            return self.cut

    def _memory(self, encoded_input, speaker, language):
        if hp.multi_speaker and self._speaker_embedding is not None:
            encoded_input = self._add_conditional_embedding(encoded_input, self._speaker_embedding, speaker)
        if hp.multi_language and self._language_embedding is not None:
            encoded_input = self._add_conditional_embedding(encoded_input, self._language_embedding, language)
        return encoded_input

    @staticmethod
    def _tape_part(tape, done, frames, columns):
        """Rows [done, done + frames) of a recorded step-prenet tape [steps, B_tape, P] (here `done` and `frames` count decoder steps),
        restricted to the utterances' tape columns.  A tape ends where the reference's loop stopped; steps decoded past it get all-ones rows
        and are discarded by the stop rule."""
        part = tape[done:done + frames]
        if list(columns) != list(range(tape.shape[1])):
            part = part[:, list(columns)]
        if part.shape[0] < frames:
            part = torch.cat([part, torch.ones(frames - part.shape[0], len(columns), tape.shape[2], dtype=part.dtype, device=part.device)])
        return part

    @staticmethod
    def _retire(rows, rules):
        """Positions (into `rows`, the original indices of the utterances still decoding) of the utterances whose stop cut is unknown."""
        return [j for j, r in enumerate(rows) if rules[r].cut is None]

    def _decode_inference(self, encoded_input, mask, speaker, language, att_extent=0, tape_columns=None):
        """Free-running decode in chunks with carried state and early exit (tacotron2.py:148-209 with target=None): every chunk is one
        library call; between chunks the stop rule reads the chunk's stop logits.  B == 1 reproduces the reference; B > 1 (which the
        reference cannot run: it uses the stop token as a Python bool) keeps one stop rule per utterance, and an utterance whose cut is
        known leaves the decode: the state, memory, lengths and rules are compacted to the utterances still running, and the next
        chunk runs at the smaller batch.  `att_extent` = 1 runs forward attention over each utterance's own length; `tape_columns`
        gives each utterance's column of a recorded mask tape (default: column b for utterance b).
        -> (spectrogram [B, T', N], stop [B, T'], alignment [B, ceil(T' / r), L], cuts): T' = max(cuts) frames; utterance b is zero past
        cuts[b] (its alignment past ceil(cuts[b] / r) steps).  The stop rule reads the r stop logits of each step in frame order, and
        hp.max_output_length counts frames."""
        memory = self._memory(encoded_input, speaker, language)
        B, L, M = memory.shape
        device = memory.device
        P, D, N = self._prenet._layers[0].weight.shape[0], self._decoder_dim, self._output_dim
        kind, rate_h, rate_c = self._cell_config()
        lengths = mask.sum(dim=1).to(torch.int32)
        state = F.DecoderState(B, D, M, L, N, device)
        rules = [self._StopRule(hp.stop_frames) for _ in range(B)]
        rows = list(range(B))                  # original index of every utterance still decoding
        columns = list(range(B)) if tape_columns is None else list(tape_columns)
        outs = [[] for _ in range(B)]
        done = 0                               # frames decoded (a whole number of steps)
        params = self._param_list()
        r = self._outputs_per_step
        chunk_steps = max(1, self.inference_chunk // r)
        while done < self._max_frames:
            Sc = min(chunk_steps, self._steps(self._max_frames - done))
            Tc = Sc * r
            masks = {}
            for name in ('step_prenet0', 'step_prenet1'):
                tape = MaskSource.raw(name)
                if MaskSource.tape is not None:
                    if tape is not None:
                        masks[name] = self._tape_part(tape, done // r, Sc, [columns[j] for j in rows]).to(device=device, dtype=torch.uint8).contiguous()
                else:
                    m = MaskSource.keep_mask(name, (Sc, len(rows), P), self._prenet._dropout_rate, device)
                    if m is not None:
                        masks[name] = m
            if self.training:
                for name in ('att_h', 'gen_h') + (('att_c', 'gen_c') if kind == _lib.CELL_ZONEOUT else ()):
                    m = MaskSource.keep_mask(name, (Sc, len(rows), D), rate_c if name.endswith('_c') else rate_h, device)
                    if m is not None:
                        masks[name] = m
            cfg = F.DecoderConfig(kind, self.training, rate_h, rate_c, self._prenet._dropout_rate, masks, np.zeros(Sc, dtype=np.uint8),
                                  att_extent, outputs_per_step=r)
            spec, stop, align = F.decoder_forward_chunk(cfg, memory, lengths, params, state, Tc)
            done += Tc
            host_stop = stop.float().cpu()
            for j, u in enumerate(rows):
                rules[u].feed(host_stop[j])
                outs[u].append((spec[j], stop[j], align[j]))
            keep = self._retire(rows, rules)
            if not keep:
                break
            if len(keep) < len(rows):
                idx = torch.tensor(keep, device=device)
                state.select(idx)
                memory, lengths = memory.index_select(0, idx), lengths.index_select(0, idx)
                rows = [rows[j] for j in keep]
        cuts = [min(rule.cut if rule.cut is not None else done, self._max_frames) for rule in rules]
        ends = lambda cut: (cut, cut, self._steps(cut))       # noqa: E731 -- rows kept of spectrogram, stop (frames), alignment (steps)
        if B == 1:
            spectrogram, stop, alignment = (torch.cat([o[k] for o in outs[0]], 0)[:ends(cuts[0])[k]].unsqueeze(0) for k in range(3))
            return spectrogram, stop, alignment, cuts
        T = max(cuts)
        spectrogram = torch.zeros(B, T, N, device=device)
        stop = torch.zeros(B, T, device=device)
        alignment = torch.zeros(B, self._steps(T), L, device=device)
        for b in range(B):
            for k, dst in enumerate((spectrogram, stop, alignment)):
                e = ends(cuts[b])[k]
                dst[b, :e] = torch.cat([o[k] for o in outs[b]], 0)[:e]
        return spectrogram, stop, alignment, cuts

    def _decode(self, encoded_input, mask, target, teacher_forcing_ratio, speaker, language):
        if target is None:
            return self._decode_inference(encoded_input, mask, speaker, language)[:3]
        encoded_input = self._memory(encoded_input, speaker, language)
        B, T = encoded_input.shape[0], self._steps(target.shape[2])
        device = encoded_input.device
        # one coin per decoder step, shared by the batch (tacotron2.py:171); drawn on the host: it steers the launch sequence
        tape_teacher = MaskSource.raw('teacher')
        if tape_teacher is not None:
            teacher = np.asarray(tape_teacher.cpu()).astype(np.uint8)
        else:
            teacher = (np.random.default_rng(MaskSource.seed + MaskSource.counter).random(T) > (1 - teacher_forcing_ratio)).astype(np.uint8)
            MaskSource.counter += 1
        teacher = None if teacher.all() else teacher
        kind, rate_h, rate_c = self._cell_config()
        cfg = F.DecoderConfig(kind, self.training, rate_h, rate_c, self._prenet._dropout_rate, self._masks(B, T, device, teacher), teacher,
                              outputs_per_step=self._outputs_per_step)
        lengths = mask.sum(dim=1).to(torch.int32)
        return F.decoder_forward(cfg, encoded_input, target, lengths, self._param_list())

    def forward(self, encoded_input, encoded_lenghts, target, teacher_forcing_ratio, speaker, language):
        ml = encoded_input.size(1)
        mask = lengths_to_mask(encoded_lenghts.to(encoded_input.device), max_length=ml)
        return self._decode(encoded_input, mask, target, teacher_forcing_ratio, speaker, language)

    def inference(self, encoded_input, speaker, language):
        mask = lengths_to_mask(torch.LongTensor([encoded_input.size(1)]).to(encoded_input.device))
        with torch.no_grad():
            spectrogram, _, _ = self._decode(encoded_input, mask, None, 0.0, speaker, language)
        return spectrogram


class Tacotron(torch.nn.Module):
    """Embedding -> encoder -> (adversarial classifier) -> decoder -> postnet (tacotron2.py:222-408)."""

    def __init__(self):
        super().__init__()
        other_symbols = 3  # PAD, EOS, UNK
        self._embedding = Embedding(hp.symbols_count() + other_symbols, hp.embedding_dimension, padding_idx=0)
        torch.nn.init.xavier_uniform_(self._embedding.weight)
        self._encoder = self._get_encoder(hp.encoder_type)
        if hp.reversal_classifier:
            self._reversal_classifier = self._get_adversarial_classifier(hp.reversal_classifier_type)
        self._prenet = Prenet(hp.num_mels, hp.prenet_dimension, hp.prenet_layers, hp.dropout)
        decoder_input_dimension = hp.encoder_dimension
        if hp.multi_speaker:
            decoder_input_dimension += hp.speaker_embedding_dimension
        if hp.multi_language:
            decoder_input_dimension += hp.language_embedding_dimension
        self._attention = self._get_attention(hp.attention_type, decoder_input_dimension)
        gen_cell_dimension = decoder_input_dimension + hp.decoder_dimension
        att_cell_dimension = decoder_input_dimension + hp.prenet_dimension
        if hp.decoder_regularization == 'zoneout':
            generator_rnn = ZoneoutLSTMCell(gen_cell_dimension, hp.decoder_dimension, hp.zoneout_hidden, hp.zoneout_cell)
            attention_rnn = ZoneoutLSTMCell(att_cell_dimension, hp.decoder_dimension, hp.zoneout_hidden, hp.zoneout_cell)
        else:
            generator_rnn = DropoutLSTMCell(gen_cell_dimension, hp.decoder_dimension, hp.dropout_hidden)
            attention_rnn = DropoutLSTMCell(att_cell_dimension, hp.decoder_dimension, hp.dropout_hidden)
        self._decoder = Decoder(hp.num_mels, hp.decoder_dimension, self._attention, generator_rnn, attention_rnn,
                                decoder_input_dimension, self._prenet, hp.prenet_dimension, hp.max_output_length, hp.outputs_per_step)
        self._postnet = self._get_postnet('cbhg' if hp.predict_linear else 'conv')

    def _get_encoder(self, name):
        args = (hp.embedding_dimension, hp.encoder_dimension, hp.encoder_blocks, hp.encoder_kernel_size, hp.dropout)
        ln = 1 if not hp.multi_language else hp.language_number
        if name == 'simple':
            return Encoder(*args)
        elif name == 'separate':
            return MultiEncoder(hp.language_number, args)
        elif name == 'shared':
            return ConditionalEncoder(hp.language_number, hp.input_language_embedding, args)
        elif name == 'convolutional':
            return ConvolutionalEncoder(hp.embedding_dimension, hp.encoder_dimension, 0.05, ln)
        elif name == 'generated':
            return GeneratedConvolutionalEncoder(hp.embedding_dimension, hp.encoder_dimension, 0.05, hp.generator_dim,
                                                 hp.generator_bottleneck_dim, groups=ln)
        raise ValueError(f'unknown encoder type {name}')

    def _get_adversarial_classifier(self, name):
        if name == 'reversal':
            return ReversalClassifier(hp.encoder_dimension, hp.reversal_classifier_dim, hp.speaker_number,
                                      hp.reversal_gradient_clipping)
        raise NotImplementedError('the cosine classifier is out of scope (reference: "does not converge at all")')

    def _get_attention(self, name, memory_dimension):
        if name == 'location_sensitive':
            return LocationSensitiveAttention(hp.attention_kernel_size, hp.attention_location_dimension, False,
                                              hp.attention_dimension, hp.decoder_dimension, memory_dimension)
        if name == 'forward':
            return ForwardAttention(hp.attention_dimension, hp.decoder_dimension, memory_dimension)
        if name == 'forward_transition_agent':
            raise NotImplementedError('attention type forward_transition_agent is not provided: the reference cannot run it '
                                      '(ForwardAttentionWithTransition.reset takes 3 arguments but the decoder passes 4), '
                                      'so there is no reference behaviour to match')
        raise NotImplementedError(f'attention type {name} is out of scope')

    def _get_postnet(self, name):
        if name == 'conv':
            return Postnet(hp.num_mels, hp.postnet_dimension, hp.postnet_blocks, hp.postnet_kernel_size, hp.dropout)
        raise NotImplementedError('the CBHG postnet (predict_linear) is out of scope: no shipped configuration enables it')

    def forward(self, text, text_length, target, target_length, speakers, languages, teacher_forcing_ratio=0.0):
        if speakers is not None and speakers.dim() == 1:
            speakers = speakers.unsqueeze(1).expand((-1, text.size(1)))
        if languages is not None and languages.dim() == 1:
            languages = languages.unsqueeze(1).expand((-1, text.size(1)))
        embedded = F.embedding(self._embedding.weight, text, padding_idx=0)
        encoded = self._encoder(embedded, text_length, languages)
        encoder_output = encoded
        speaker_prediction = self._reversal_classifier(encoded) if hp.reversal_classifier else None
        if languages is not None and languages.dim() == 3:
            languages = torch.argmax(languages, dim=2)
        prediction, stop_token, alignment = self._decoder(encoded, text_length, target, teacher_forcing_ratio, speakers, languages)
        pre_prediction = prediction.transpose(1, 2)
        post_prediction = self._postnet(pre_prediction, target_length)
        target_mask = lengths_to_mask(target_length.to(text.device), target.size(2))
        stop_token = stop_token.masked_fill(~target_mask, 1000)
        target_mask = target_mask.unsqueeze(1).float()
        pre_prediction = pre_prediction * target_mask
        post_prediction = post_prediction * target_mask
        return post_prediction, pre_prediction, stop_token, alignment, speaker_prediction, encoder_output

    def inference(self, text, speaker=None, language=None):
        """synthesize.py entry point (tacotron2.py:387-408): text int64 [L], speaker int64 [1] | None, language int64 [1] |
        float [1, L, G] (per-character language mixing) | None -> post-net spectrogram [num_mels, T'].  The one-utterance case of
        `inference_batch`."""
        return self.inference_batch([text], None if speaker is None else [speaker], None if language is None else [language])[0]

    def inference_batch(self, texts, speakers=None, languages=None, max_batch=64):
        """Synthesise many utterances at once: texts is a list of int64 [L_i]; speakers / languages are None or lists with one entry per
        text in the forms `inference` takes (speaker int64 [1]; language int64 [1] or float [1, L_i, G]).  -> one post-net spectrogram
        [num_mels, T_i] per text, in input order.  Texts are sorted by length and decoded in padded groups of at most max_batch (eval
        mode, no grad); each utterance's output equals `inference` of it alone given the same prenet dropout masks (a recorded tape,
        [T, len(texts), P] with one column per text).  Without a tape a batched run draws other masks than single runs do."""
        speakers, languages = _check_batch_inputs(texts, speakers, languages)
        was_training = self.training
        self.eval()
        outputs = [None] * len(texts)
        try:
            with torch.no_grad():
                for group in _batch_plan([int(t.shape[0]) for t in texts], max_batch):
                    posts = self._inference_group([texts[i] for i in group], None if speakers is None else [speakers[i] for i in group],
                                                  None if languages is None else [languages[i] for i in group], group)
                    for i, post in zip(group, posts):
                        outputs[i] = post
        finally:
            self.train(was_training)
        return outputs

    def _inference_group(self, texts, speakers, languages, tape_columns):
        device = self._embedding.weight.device
        B, Lmax = len(texts), max(int(t.shape[0]) for t in texts)
        lengths = torch.tensor([int(t.shape[0]) for t in texts], device=device)
        text = torch.zeros(B, Lmax, dtype=torch.long, device=device)
        for b, t in enumerate(texts):
            text[b, :t.shape[0]] = t.to(device)
        speaker = language = None
        if speakers is not None:
            speaker = torch.cat([s.reshape(1).to(device) for s in speakers]).unsqueeze(1).expand(-1, Lmax)
        if languages is not None:
            if languages[0].dim() == 1:
                language = torch.cat([g.reshape(1).to(device) for g in languages]).unsqueeze(1).expand(-1, Lmax)
            else:
                language = torch.zeros(B, Lmax, languages[0].shape[2], device=device)
                for b, g in enumerate(languages):
                    language[b, :g.shape[1]] = g[0].to(device=device, dtype=torch.float32)
        # padded characters embed to 0 (the padding row of the table is not zero: xavier_uniform_ ran after padding_idx was set)
        embedded = F.embedding(self._embedding.weight, text, padding_idx=0)
        embedded = embedded.masked_fill(~lengths_to_mask(lengths, Lmax).unsqueeze(2), 0.0)
        encoded = self._encoder(embedded, lengths, language, padded=True)
        if language is not None and language.dim() == 3:
            language = torch.argmax(language, dim=2)  # one-hot into indices for the decoder's language embedding
        mask = lengths_to_mask(lengths, Lmax)
        prediction, _, _, cuts = self._decoder._decode_inference(encoded, mask, speaker, language, att_extent=1, tape_columns=tape_columns)
        post = self._postnet(prediction.transpose(1, 2), torch.tensor(cuts, device=device), padded=True)
        return [post[b, :, :cuts[b]] for b in range(B)]


def _check_batch_inputs(texts, speakers, languages):
    """Validate the per-utterance arguments of Tacotron.inference_batch -> (speakers, languages) as lists or None."""
    texts = list(texts)
    if not texts:
        raise ValueError('inference_batch: no texts given')
    for t in texts:
        if not torch.is_tensor(t) or t.dim() != 1 or t.shape[0] < 1 or t.dtype != torch.int64:
            raise ValueError('inference_batch: every text must be a non-empty int64 tensor [L]')
    out = []
    for name, items in (('speakers', speakers), ('languages', languages)):
        if items is not None:
            items = list(items)
            if len(items) != len(texts):
                raise ValueError(f'inference_batch: {len(items)} {name} for {len(texts)} texts')
            if any(x is None for x in items):
                raise ValueError(f'inference_batch: {name} must be given for every text or for none')
        out.append(items)
    speakers, languages = out
    if speakers is not None and any(s.numel() != 1 or s.dtype != torch.int64 for s in speakers):
        raise ValueError('inference_batch: a speaker is an int64 tensor [1]')
    if speakers is None and hp.multi_speaker and hp.speaker_embedding_dimension > 0:
        raise ValueError('inference_batch: a multi-speaker model needs one speaker per text')
    if languages is not None:
        forms = {'index' if g.dim() == 1 else 'mix' for g in languages}
        if len(forms) > 1:
            raise ValueError('inference_batch: languages mix int64 [1] ids and float [1, L, G] weights; use one form for all texts')
        for t, g in zip(texts, languages):
            if g.dim() == 1:
                if g.numel() != 1 or g.dtype != torch.int64:
                    raise ValueError('inference_batch: a language id is an int64 tensor [1]')
            elif g.dim() != 3 or g.shape[0] != 1 or g.shape[1] != t.shape[0] or not g.is_floating_point() \
                    or g.shape[2] != languages[0].shape[2]:
                raise ValueError('inference_batch: per-character language weights are float [1, L, G] with L the text length')
    return speakers, languages


def _batch_plan(lengths, max_batch):
    """Utterance indices sorted by text length (stable), cut into consecutive groups of at most max_batch."""
    if int(max_batch) < 1:
        raise ValueError(f'inference_batch: max_batch must be >= 1 (got {max_batch})')
    order = sorted(range(len(lengths)), key=lambda i: lengths[i])
    return [order[k:k + max_batch] for k in range(0, len(order), max_batch)]


class TacotronLoss(torch.nn.Module):
    """Loss terms of the reference (tacotron2.py:411-485): 2*MSE(pre) + MSE(post) + weighted stop BCE / (mels + 2)
    [+ adversarial classifier CE] [+ guided attention].  The four Tacotron terms are ONE fused library op forward and one backward
    (csrc/loss.cu); the guided-attention weights are evaluated in closed form inside the kernels instead of the reference's
    per-utterance Python loop with meshgrid, and no [B, T, L] weight tensor is materialised."""

    def __init__(self, guided_att_steps, guided_att_variance, guided_att_gamma):
        super().__init__()
        self._g = guided_att_variance
        self._gamma = guided_att_gamma
        self._g_steps = guided_att_steps

    def load_state_dict(self, d):
        for k, v in d.items():
            setattr(self, k, v)

    def state_dict(self):
        return {'_g': self._g, '_g_steps': self._g_steps}

    def update_states(self):
        self._g *= self._gamma
        self._g_steps = max(0, self._g_steps - 1)

    def forward(self, source_length, target_length, pre_prediction, pre_target, post_prediction, post_target, stop, target_stop,
                alignment, speaker, speaker_prediction, encoder_outputs, classifier):
        guided = bool(hp.guided_attention_loss) and self._g_steps > 0
        terms = F.tacotron_loss(pre_prediction, post_prediction, stop, alignment if guided else None, pre_target, post_target,
                                target_stop, source_length, target_length, guided, self._g, 100.0, hp.outputs_per_step)
        losses = {'mel_pre': terms[0], 'mel_pos': terms[1], 'stop_token': terms[2]}
        if hp.reversal_classifier:
            losses['lang_class'] = ReversalClassifier.loss(source_length.to(stop.device), speaker, speaker_prediction)
            losses['lang_class'] = losses['lang_class'] * (hp.reversal_classifier_w / (hp.num_mels + 2))
        if hp.guided_attention_loss:
            losses['guided_att'] = terms[3] if guided else 0
        return sum(losses.values()), losses
