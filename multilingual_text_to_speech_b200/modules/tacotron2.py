"""Tacotron 2 model (surface of reference modules/tacotron2.py:15-485) on the b200tts library.

Constructor signatures, attribute names (`_embedding`, `_encoder`, `_prenet`, `_attention`, `_decoder`, `_postnet`,
`_reversal_classifier`), parameter names / shapes and forward / inference signatures follow the reference so that
train.py, synthesize.py and existing checkpoints work unchanged.  All arithmetic of the hot path is inside the
library: `Decoder` is ONE fused op (forward + hand-written BPTT), encoders / postnet are fused conv-block ops.
"""
from typing import NamedTuple

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
from .stream_pool import check_seed


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

    def halo(self):
        """Frames on each side of an output frame that it depends on: the blocks' reaches added up."""
        return sum((block._kernel - 1) * block._dilation // 2 for block in self._convs)

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

    class _PlanRule:
        """The stop rule of a forced row (a row decoding from an attention plan): a fixed cut of the plan's frames, known when the row
        opens.  The stop logits are still computed and fed, but they do not end the row."""

        def __init__(self, frames):
            self.frames, self.seen, self.cut = frames, 0, None

        def feed(self, logits):
            self.seen += len(logits)
            if self.seen >= self.frames:
                self.cut = self.frames
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

    def _inference_chunks(self, encoded_input, mask, speaker, language, att_extent=0, tape_columns=None, chunk_frames=None, att_window=None,
                          plans=None):
        """The chunk loop of free-running inference (tacotron2.py:148-209 with target=None) over a batch whose texts all open at the
        first call: every chunk is one library call of chunk_frames (default inference_chunk) frames rounded down to whole steps; after
        each it feeds the chunk's stop logits to the utterances' stop rules and yields (rows, spec [b, Tc, N], stop [b, Tc], alignment
        [b, Tc / r, L], rules, done): rows are the original indices of the b utterances the chunk decoded, rules the stop rule of every
        utterance, done the frames decoded so far.  Then an utterance whose cut is known leaves the decode (_DecodeRows.retire) and the next
        chunk runs at the smaller batch.  The loop ends when every cut is known or hp.max_output_length frames are decoded.  The rule reads
        the r stop logits of each step in frame order.  Utterance b reads column tape_columns[b] (default b) of an active mask tape.
        att_window: None or (back, ahead), windowed attention (inference_attention_window).  plans: None or one attention plan (_forced_plan)
        or None per utterance."""
        memory = self._memory(encoded_input, speaker, language)
        B = memory.shape[0]
        columns = list(range(B)) if tape_columns is None else list(tape_columns)
        rows = _DecodeRows(self, att_extent, att_window)
        rows.add(memory, [int(n) for n in mask.sum(dim=1).tolist()], list(range(B)), [('shared', c) for c in columns])
        if plans is not None:
            rows.set_plans(plans)
        rules = list(rows.rules)
        chunk_steps = max(1, (self.inference_chunk if chunk_frames is None else int(chunk_frames)) // self._outputs_per_step)
        while len(rows):
            spec, stop, align = rows.step(chunk_steps)
            yield list(rows.keys), spec, stop, align, rules, rows.done[0]
            rows.retire()

    def _decode_inference(self, encoded_input, mask, speaker, language, att_extent=0, tape_columns=None, att_window=None, plans=None):
        """Free-running decode in chunks with carried state and early exit (_inference_chunks).  B == 1 reproduces the reference; B > 1
        (which the reference cannot run: it uses the stop token as a Python bool) keeps one stop rule per utterance.  `att_extent` = 1 runs
        forward attention over each utterance's own length; `tape_columns` gives each utterance's column of a recorded mask tape (default:
        column b for utterance b); `att_window` confines each step's attention (inference_attention_window); `plans` gives utterances
        their attention (_forced_plan).
        -> (spectrogram [B, T', N], stop [B, T'], alignment [B, ceil(T' / r), L], cuts): T' = max(cuts) frames; utterance b is zero past
        cuts[b] (its alignment past ceil(cuts[b] / r) steps).  hp.max_output_length counts frames."""
        B, L = encoded_input.shape[0], encoded_input.shape[1]
        device = encoded_input.device
        N = self._output_dim
        outs = [[] for _ in range(B)]
        done = 0
        for rows, spec, stop, align, rules, done in self._inference_chunks(encoded_input, mask, speaker, language, att_extent, tape_columns,
                                                                           att_window=att_window, plans=plans):
            if align.shape[2] < L:          # the chunk ran after the longest text left: its weights past the shorter ones are zero
                align = TF.pad(align, (0, L - align.shape[2]))
            for j, u in enumerate(rows):
                outs[u].append((spec[j], stop[j], align[j]))
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

    def inference(self, text, speaker=None, language=None, durations=None, alignment=None):
        """synthesize.py entry point (tacotron2.py:387-408): text int64 [L], speaker int64 [1] | None, language int64 [1] |
        float [1, L, G] (per-character language mixing) | None -> post-net spectrogram [num_mels, T'].  The one-utterance case of
        `inference_batch`; `durations` or `alignment` sets the decode's attention as inference_batch's do."""
        return self.inference_batch([text], None if speaker is None else [speaker], None if language is None else [language],
                                    durations=None if durations is None else [durations],
                                    alignments=None if alignment is None else [alignment])[0]

    def inference_batch(self, texts, speakers=None, languages=None, max_batch=64, durations=None, alignments=None):
        """Synthesise many utterances at once: texts is a list of int64 [L_i]; speakers / languages are None or lists with one entry per
        text in the forms `inference` takes (speaker int64 [1]; language int64 [1] or float [1, L_i, G]).  -> one post-net spectrogram
        [num_mels, T_i] per text, in input order.  Texts are sorted by length and decoded in padded groups of at most max_batch (eval
        mode, no grad); each utterance's output equals `inference` of it alone given the same prenet dropout masks (a recorded tape,
        [T, len(texts), P] with one column per text).  Without a tape a batched run draws other masks than single runs do.
        hp.inference_attention_window is read once per call.

        Forced synthesis: `durations` (int [L_i] frames per symbol, each >= 0) or `alignments` (float [S_i, L_i], finite and >= 0, for
        example Tacotron.align's alignment[b, :S_b, :L_b]) is None or a list with one entry or None per text; a text with an entry decodes
        with each step's attention set by it instead of computed (functional.durations_to_alignment turns durations into one-hot rows),
        and its output has exactly sum(d_i) frames, or S_i r, whatever the stop token does.  A text takes at most one of the two.  Forced
        and free texts share groups; each output equals the text decoded alone.  ValueError before any device work for malformed
        plans (_forced_plan)."""
        speakers, languages = _check_batch_inputs(texts, speakers, languages)
        plans = _batch_plans(self._decoder, texts, durations, alignments)
        window = inference_attention_window()
        was_training = self.training
        self.eval()
        outputs = [None] * len(texts)
        try:
            with torch.no_grad():
                for group in _batch_plan([int(t.shape[0]) for t in texts], max_batch):
                    posts = self._inference_group([texts[i] for i in group], None if speakers is None else [speakers[i] for i in group],
                                                  None if languages is None else [languages[i] for i in group], group, window,
                                                  [plans[i] for i in group])
                    for i, post in zip(group, posts):
                        outputs[i] = post
        finally:
            self.train(was_training)
        return outputs

    def align(self, text, text_length, target, target_length, speakers=None, languages=None):
        """Forced alignment of a batch with its target spectrograms: `forward` in eval mode at teacher forcing 1.0 without autograd (the
        reference gta.py's call), then the monotonic alignment search (functional.monotonic_alignment) and the alignment scores on each
        utterance's steps and symbols.  Takes forward's inputs: text int [B, L], text_length [B], target [B, num_mels, T],
        target_length [B], speakers and languages in forward's forms (grouped-encoder batches in any language layout).

        With hp.outputs_per_step = r the search runs on the decoder's step grid, S_b = ceil(T_b / r) steps for T_b target frames (the
        steps the guided-attention loss weighs); a symbol's frames are its steps times r, except the last symbol's, which lose the
        S_b r - T_b frames past the target, so each utterance's frames sum to T_b.

        Prenet dropout stays on, as in the reference.  For repeatable masks replay a MaskSource tape (its 'teacher' entry is replaced by
        all ones for this call) or seed MaskSource.  -> Alignment: `alignment` [B, S, L] is forward's alignment on the same batch and
        masks, bit for bit.  ValueError before any device work for malformed inputs, lengths out of range, S_b < L_b, or a shape past
        the search's limits."""
        shapes = [('text', text, 2), ('text_length', text_length, 1), ('target', target, 3), ('target_length', target_length, 1)]
        for name, t, dims in shapes:
            if not torch.is_tensor(t) or t.dim() != dims:
                raise ValueError(f'align: {name} must be a {dims}-D tensor')
        if text.dtype.is_floating_point:
            raise ValueError(f'align: text must hold symbol ids, got {text.dtype}')
        B, L = text.shape
        if target.shape[0] != B or target.shape[1] != hp.num_mels:
            raise ValueError(f'align: target must be [B = {B}, num_mels = {hp.num_mels}, T], got {tuple(target.shape)}')
        r, T = self._decoder._outputs_per_step, target.shape[2]
        frames = F._host_lengths(target_length, B, 'target_length')
        for b, t in enumerate(frames):
            if not 1 <= t <= T:
                raise ValueError(f'align: utterance {b}: target length {t} is outside [1, {T}]')
        steps = [-(-t // r) for t in frames]
        symbols, _ = F.check_alignment_lengths(text_length, steps, B, -(-T // r), L)
        was_training, tape = self.training, MaskSource.tape
        self.eval()
        try:
            if tape is not None:
                MaskSource.use_tape({**tape, 'teacher': torch.ones(-(-T // r), dtype=torch.bool)})
            with torch.no_grad():
                alignment = self.forward(text, text_length, target, target_length, speakers, languages, teacher_forcing_ratio=1.0)[3]
        finally:
            MaskSource.use_tape(tape)
            self.train(was_training)
        step_durations, path_logp = F.monotonic_alignment(alignment, symbols, steps)
        durations = step_durations * r
        rows = torch.arange(B, device=durations.device)
        last = torch.tensor(symbols, device=durations.device) - 1
        durations[rows, last] -= torch.tensor([s * r - t for s, t in zip(steps, frames)], device=durations.device, dtype=torch.int32)
        return Alignment(alignment, durations, step_durations, path_logp, **F.alignment_scores(alignment, symbols, steps))

    def inference_stream(self, text, speaker=None, language=None, chunk_frames=None, durations=None, alignment=None):
        """Streaming `inference`: a generator of post-net spectrogram chunks [num_mels, n_k] whose concatenation is inference(text,
        speaker, language), the same stop cut and, given the same prenet dropout masks, the same decoded frames.  Takes the inputs
        `inference` takes.  The decoder runs in chunks of chunk_frames frames (default Decoder.inference_chunk, rounded down to whole
        decoder steps); after every chunk one item is yielded: the post-net over the frames that became final (stream_release), computed
        over a window with the post-net's halo of decoded frames on the left and, once the cut is known, the zeros past it on the right.
        An item may hold no frames (a chunk shorter than the halo).  The model is in eval mode, without autograd, until the generator
        ends or is closed; prenet dropout stays on, as in `inference`, and a MaskSource tape is replayed the same way.  `durations` or
        `alignment` sets the attention as in `inference`.  The one-text case of `inference_streams`."""
        for item in self._streams([text], None if speaker is None else [speaker], None if language is None else [language], chunk_frames,
                                  'inference_stream', None if durations is None else [durations], None if alignment is None else [alignment]):
            yield item[0]

    def inference_streams(self, texts, speakers=None, languages=None, chunk_frames=None, durations=None, alignments=None):
        """`inference_stream` for up to 64 texts decoded as one group: takes `inference_batch`'s inputs (text i reads column i of a
        recorded mask tape; durations and alignments as there) and yields, after every decoder call, {i: post-net chunk [num_mels, n]} for each text the call decoded (a chunk
        may hold no frames).  The frames released by one call go through the post-net as one padded batch.  Concatenated per text, the
        chunks are inference_batch's output for that text; in fp32 mode they equal inference_stream of that text alone with its tape
        column, bit for bit."""
        yield from self._streams(texts, speakers, languages, chunk_frames, 'inference_streams', durations, alignments)

    def _streams(self, texts, speakers, languages, chunk_frames, name, durations=None, alignments=None):
        speakers, languages = _check_batch_inputs(texts, speakers, languages)
        texts = list(texts)
        durations, alignments = _plan_lists(texts, durations, alignments)
        if len(texts) > MAX_STREAM_TEXTS:
            raise ValueError(f'{name}: at most {MAX_STREAM_TEXTS} texts decode as one group (got {len(texts)})')
        if chunk_frames is not None and int(chunk_frames) < 1:
            raise ValueError(f'{name}: chunk_frames must be >= 1 (got {chunk_frames})')
        pool = self.decoder_pool(len(texts), chunk_frames)
        for i, text in enumerate(texts):        # ids 0 .. B - 1: text i reads column i of a recorded mask tape
            pool.open(text, None if speakers is None else speakers[i], None if languages is None else languages[i],
                      durations=durations[i], alignment=alignments[i])
        while pool.ids:
            yield pool.run()

    def decoder_pool(self, max_texts=64, chunk_frames=None):
        """A DecoderPool of up to max_texts texts decoded in chunks of chunk_frames frames (default Decoder.inference_chunk)."""
        return DecoderPool(self, max_texts, chunk_frames)

    def _postnet_windows(self, pre, spans, halo):
        """{u: post-net output frames [t0, t1) [num_mels, t1 - t0]} for spans {u: (t0, t1, avail)} of the decoded frames pre[u] (chunks of
        [n, N], of which the first `avail` count; the rest lie past the stop cut): each run over frames [t0 - halo, t1 + halo) within
        [0, avail), zero-padded at the window's ends, all windows in one padded post-net batch."""
        N = pre[next(iter(spans))][0].shape[1]
        out, wins = {}, []
        for u, (t0, t1, avail) in spans.items():
            if t1 <= t0:
                out[u] = pre[u][0].new_zeros(N, 0)
            else:
                w0, w1 = postnet_window(t0, t1, halo, avail)
                wins.append((u, t0, t1, w0, w1))
        if wins:
            W = max(w1 - w0 for *_, w0, w1 in wins)
            x = pre[wins[0][0]][0].new_zeros(len(wins), N, W)
            for b, (u, t0, t1, w0, w1) in enumerate(wins):
                x[b, :, :w1 - w0] = torch.cat(pre[u], 0)[w0:w1].t()
            lengths = torch.tensor([w1 - w0 for *_, w0, w1 in wins], device=x.device)
            post = self._postnet(x, lengths, padded=True)
            for b, (u, t0, t1, w0, w1) in enumerate(wins):
                out[u] = post[b, :, t0 - w0:t1 - w0]
        return out

    def _encode_group(self, texts, speakers, languages):
        """Padded batch of texts -> (encoder output, mask, speaker, language) in the decoder's forms."""
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
        return encoded, lengths_to_mask(lengths, Lmax), speaker, language

    def _inference_group(self, texts, speakers, languages, tape_columns, att_window, plans=None):
        device = self._embedding.weight.device
        encoded, mask, speaker, language = self._encode_group(texts, speakers, languages)
        B = len(texts)
        prediction, _, _, cuts = self._decoder._decode_inference(encoded, mask, speaker, language, att_extent=1, tape_columns=tape_columns,
                                                                 att_window=att_window, plans=plans)
        post = self._postnet(prediction.transpose(1, 2), torch.tensor(cuts, device=device), padded=True)
        return [post[b, :, :cuts[b]] for b in range(B)]


# texts of one inference_streams group at most: the batch inference_batch decodes at once by default
MAX_STREAM_TEXTS = 64


class Alignment(NamedTuple):
    """Tacotron.align's result for B utterances of L symbols and S decoder steps (S_b = ceil(T_b / r) each)."""
    alignment: torch.Tensor         # [B, S, L] float32: Tacotron.forward's attention weights (eval mode, teacher forcing 1.0)
    durations: torch.Tensor         # [B, L] int32: frames per symbol, summing to target_length, 0 past the text
    step_durations: torch.Tensor    # [B, L] int32: decoder steps per symbol, summing to S_b, 0 past the text
    path_logp: torch.Tensor         # [B] float64: the path's sum of log max(weight, 1e-8)
    focus_rate: torch.Tensor        # [B] float32: mean over steps of the largest weight
    coverage: torch.Tensor          # [B] float32: fraction of symbols whose summed weight reaches 0.5
    max_jump: torch.Tensor          # [B] int32: largest forward move of the per-step argmax
    moves_back: torch.Tensor        # [B] bool: whether the per-step argmax ever moves backwards


def inference_attention_window():
    """hp.inference_attention_window checked -> None (off) or (back, ahead) with back >= 0, ahead >= 1.  ValueError for any other value,
    and for a window with forward attention, which already moves at most one position per step."""
    w = hp.inference_attention_window
    if w is None:
        return None
    ok = isinstance(w, (list, tuple)) and len(w) == 2 and all(isinstance(x, (int, np.integer)) and not isinstance(x, bool) for x in w)
    if not ok or int(w[0]) < 0 or int(w[1]) < 1:
        raise ValueError(f'inference_attention_window must be None or [back >= 0, ahead >= 1] of ints (got {w!r})')
    if hp.attention_type == 'forward':
        raise ValueError('inference_attention_window needs location-sensitive attention: forward attention moves at most one position a step')
    return int(w[0]), int(w[1])

PRENET_SITES = ('step_prenet0', 'step_prenet1')


class _DecodeRows:
    """The rows of a running free-running decode, one per text, and its one chunk loop (Decoder._inference_chunks, DecoderPool).  It
    holds the memory [B, L, M] and lengths of the open texts, re-padded to the longest of them (L grows when a longer text joins and
    shrinks when the longest leaves; attention weights past a text's length are exact zeros, so a row's frames do not depend on L), the
    carried DecoderState, and per row its key, stop rule, frames decoded and prenet mask source:
      * ('tape', {site: [S, P]}): the row's own recorded masks, step i of the row reading row i (all-ones past the tape's end);
      * ('seed', seed): b200tts_fill_keep_mask_rows at the row's own step count, stream _lib.SEED_STREAMS[site];
      * ('shared', column): with a MaskSource tape active, that column of it; otherwise one MaskSource draw over every shared row per
        call, as the batched decode has always drawn.
    att_window (None or (back, ahead)) goes to every call; each row's window centre is carried in the DecoderState.  A forced row also
    holds its attention plan (weights [S_i, L_i], frames T_i; _forced_plan): every call passes the plan's steps from the row's own step
    count on (zero rows past its end) to the library's forced attention step, and its stop rule is the fixed cut T_i (Decoder._PlanRule)."""

    def __init__(self, dec, att_extent, att_window=None):
        self.dec, self.att_extent, self.att_window = dec, att_extent, att_window
        self.memory = self.lengths = self.state = None
        self.keys, self.rules, self.done, self.sources, self.text_len, self.plans = [], [], [], [], [], []

    def __len__(self):
        return len(self.keys)

    def add(self, memory, lengths, keys, sources):
        """Appends texts: memory [b, Lb, M] (speaker / language columns included), lengths (host ints), one key and one mask source each.
        The memory, lengths and cum_weights are re-padded to the longest open text and the new state rows are set to a decode's initial
        state (b200tts_decoder_state_reset_rows)."""
        dec, n, b = self.dec, len(self.keys), memory.shape[0]
        L = max(list(lengths) + self.text_len)
        M, device = memory.shape[2], memory.device
        if n == 0:
            self.memory = memory[:, :L]
            self.lengths = torch.tensor(lengths, dtype=torch.int32, device=device)
            self.state = F.DecoderState(0, dec._decoder_dim, M, L, dec._output_dim, device)
        else:
            grown = memory.new_zeros(n + b, L, M)
            grown[:n, :self.memory.shape[1]] = self.memory
            grown[n:, :min(L, memory.shape[1])] = memory[:, :L]
            self.memory = grown
            self.lengths = torch.cat([self.lengths, torch.tensor(lengths, dtype=torch.int32, device=device)])
        self.state.grow(b, L)
        self.state.reset_rows(range(n, n + b), getattr(dec._attention, '_location', None) is None)
        self.state.first = False
        self.keys += list(keys)
        self.rules += [dec._StopRule(hp.stop_frames) for _ in range(b)]
        self.plans += [None] * b
        self.done += [0] * b
        self.sources += list(sources)
        self.text_len += list(lengths)

    def set_plans(self, plans):
        """Gives the last len(plans) rows added their attention plans (None: the row decodes freely) and a forced row its fixed cut."""
        n = len(self.keys) - len(plans)
        for j, p in enumerate(plans, n):
            if p is not None:
                self.plans[j], self.rules[j] = p, self.dec._PlanRule(p[1])

    def keep(self, js):
        """Keeps rows js (positions, in order); the memory and cum_weights shrink to the longest text left."""
        if len(js) == len(self.keys):
            return
        if not js:
            self.__init__(self.dec, self.att_extent, self.att_window)
            return
        idx = torch.tensor(js, device=self.memory.device)
        self.state.select(idx)
        self.memory, self.lengths = self.memory.index_select(0, idx), self.lengths.index_select(0, idx)
        for name in ('keys', 'rules', 'done', 'sources', 'text_len', 'plans'):
            setattr(self, name, [getattr(self, name)[j] for j in js])
        L = max(self.text_len)
        if L < self.memory.shape[1]:
            self.memory = self.memory[:, :L].contiguous()
            self.state.cum_weights = self.state.cum_weights[:, :L].contiguous()

    def retire(self):
        """Rows whose stop cut is known or that reached hp.max_output_length frames leave -> their keys."""
        alive = set(self.dec._retire(range(len(self.keys)), self.rules))
        js = [j for j in range(len(self.keys)) if j in alive and self.done[j] < self.dec._max_frames]
        gone = [k for j, k in enumerate(self.keys) if j not in js]
        self.keep(js)
        return gone

    def close(self, key):
        self.keep([j for j, k in enumerate(self.keys) if k != key])

    def _prenet_masks(self, Sc):
        """{site: keep masks [Sc, B, P]} for the next call (a site without masks runs without dropout)."""
        dec = self.dec
        P, rate, r = dec._prenet._layers[0].weight.shape[0], dec._prenet._dropout_rate, dec._outputs_per_step
        device, B = self.memory.device, len(self.keys)
        kinds = [src[0] for src in self.sources]
        shared = [j for j, k in enumerate(kinds) if k == 'shared']
        masks = {}
        for name in PRENET_SITES:
            part = None
            if shared:
                if MaskSource.tape is not None:
                    tape = MaskSource.raw(name)
                    if tape is not None:
                        by_done = {}
                        for j in shared:
                            by_done.setdefault(self.done[j], []).append(j)
                        if len(by_done) == 1:
                            part = dec._tape_part(tape, self.done[shared[0]] // r, Sc, [self.sources[j][1] for j in shared])
                        else:
                            part = torch.cat([dec._tape_part(tape, self.done[j] // r, Sc, [self.sources[j][1]]) for j in shared], 1)
                        part = part.to(device=device, dtype=torch.uint8).contiguous()
                else:
                    part = MaskSource.keep_mask(name, (Sc, len(shared), P), rate, device)
            if len(shared) == B:
                if part is not None:
                    masks[name] = part
                continue
            full = torch.ones(Sc, B, P, dtype=torch.uint8, device=device)
            if part is not None:
                full[:, shared] = part
            seeded = [j for j, k in enumerate(kinds) if k == 'seed']
            if seeded:
                full[:, seeded] = F.fill_keep_mask_rows(Sc, P, rate, [self.sources[j][1] for j in seeded], [self.done[j] // r for j in seeded],
                                                        _lib.SEED_STREAMS[name], device)
            for j, k in enumerate(kinds):
                if k == 'tape':
                    full[:, j] = dec._tape_part(self.sources[j][1][name].unsqueeze(1), self.done[j] // r, Sc, [0])[:, 0].to(device)
            masks[name] = full
        return masks

    def _forced(self, Sc):
        """(rows [F] int32, weights [Sc, F, L]) of the forced rows for the next Sc steps, or None: each row's plan from its own step."""
        js = [j for j, p in enumerate(self.plans) if p is not None]
        if not js:
            return None
        r, device = self.dec._outputs_per_step, self.memory.device
        weights = torch.zeros(Sc, len(js), self.memory.shape[1], device=device)
        for k, j in enumerate(js):
            part = self.plans[j][0][self.done[j] // r:self.done[j] // r + Sc]
            weights[:part.shape[0], k, :part.shape[1]] = part
        return torch.tensor(js, dtype=torch.int32, device=device), weights

    def step(self, chunk_steps):
        """One library call over every row: min(chunk_steps, the steps the furthest-from-done row has left) steps; feeds each row's stop
        rule and step count -> (spec [B, Tc, N], stop [B, Tc], alignment [B, Tc / r, L]).  A row decoded past hp.max_output_length
        discards those frames."""
        dec = self.dec
        r = dec._outputs_per_step
        ends = [dec._max_frames if p is None else p[1] for p in self.plans]
        Sc = min(chunk_steps, max(dec._steps(e - d) for e, d in zip(ends, self.done)))
        D, device = dec._decoder_dim, self.memory.device
        kind, rate_h, rate_c = dec._cell_config()
        masks = self._prenet_masks(Sc)
        if dec.training:
            for name in ('att_h', 'gen_h') + (('att_c', 'gen_c') if kind == _lib.CELL_ZONEOUT else ()):
                m = MaskSource.keep_mask(name, (Sc, len(self.keys), D), rate_c if name.endswith('_c') else rate_h, device)
                if m is not None:
                    masks[name] = m
        cfg = F.DecoderConfig(kind, dec.training, rate_h, rate_c, dec._prenet._dropout_rate, masks, np.zeros(Sc, dtype=np.uint8),
                              self.att_extent, outputs_per_step=r, att_window=self.att_window)
        args, forced = (cfg, self.memory, self.lengths, dec._param_list(), self.state, Sc * r), self._forced(Sc)
        spec, stop, align = F.decoder_forward_chunk(*args) if forced is None else F.decoder_forward_chunk(*args, forced=forced)
        host_stop = stop.float().cpu()
        for j in range(len(self.keys)):
            self.rules[j].feed(host_stop[j])
            self.done[j] += Sc * r
        return spec, stop, align


class DecoderPool:
    """Continuous-batching decode: texts join the running decoder group at any call and leave at their stop cut.  open() queues a text;
    run() encodes the texts opened since the last call as one padded group (one per form of speaker / language inputs), appends their rows
    to the running ones (_DecodeRows.add), makes one decoder call over every open text and returns {id: post-net chunk [num_mels, n]} as
    Tacotron.inference_streams does (the released frames of every text through the post-net as one padded batch).  A text's chunks,
    concatenated, are inference_stream of it alone, bit for bit in fp32 mode given the same masks, whenever it joined and whatever shares
    its calls; every text keeps its own step count, stop rule and hp.max_output_length.

    Prenet dropout masks per text: `masks` (a tape {'step_prenet0': [S, P], 'step_prenet1': [S, P]}) if given, else `seed` (draws that
    depend on the seed and the text's own steps only: its masks are one b200tts_fill_keep_mask((S, P), seed, _lib.SEED_STREAMS[site])
    call per site), else one shared MaskSource draw per call over such texts (with a MaskSource tape active: column `id` of it).  The
    model runs each call in eval mode without autograd and is restored after it.  hp.inference_attention_window is read when the pool is
    built and kept for its life.  A text opened with `durations` or `alignment` (Tacotron.inference's forms) decodes with that
    attention and ends at the plan's frame count."""

    def __init__(self, tacotron, max_texts=64, chunk_frames=None):
        if not 1 <= int(max_texts) <= MAX_STREAM_TEXTS:
            raise ValueError(f'a decoder pool holds 1 to {MAX_STREAM_TEXTS} texts (got {max_texts})')
        if chunk_frames is not None and int(chunk_frames) < 1:
            raise ValueError(f'decoder_pool: chunk_frames must be >= 1 (got {chunk_frames})')
        self.t, self.max_texts = tacotron, int(max_texts)
        dec = tacotron._decoder
        self.chunk_steps = max(1, (dec.inference_chunk if chunk_frames is None else int(chunk_frames)) // dec._outputs_per_step)
        self.rows = _DecodeRows(dec, att_extent=1, att_window=inference_attention_window())
        self.queue = []                        # (id, text, speaker, language, source) opened since the last call
        self.pre, self.released = {}, {}       # per open text: its decoded chunks [n, N], the frames its post-net chunks cover
        self.next_id = 0

    @property
    def ids(self):
        """Every open text: queued, then decoding."""
        return [q[0] for q in self.queue] + list(self.rows.keys)

    def check(self, text, speaker=None, language=None, seed=None, masks=None, durations=None, alignment=None):
        """Validates one text's inputs (ValueError) -> its mask source ('tape', {site: uint8 [S, P]}), ('seed', seed) or ('shared', None)."""
        _check_batch_inputs([text], None if speaker is None else [speaker], None if language is None else [language])
        _forced_plan(self.t._decoder, text, durations, alignment, None)
        if masks is not None:
            P = self.t._decoder._prenet._layers[0].weight.shape[0]
            if not isinstance(masks, dict) or set(masks) != set(PRENET_SITES):
                raise ValueError(f'a mask tape is a dict with exactly the keys {PRENET_SITES}')
            for k, v in masks.items():
                if not torch.is_tensor(v) or v.dim() != 2 or v.shape[0] < 1 or v.shape[1] != P:
                    raise ValueError(f'mask tape {k!r} must be a tensor [S >= 1, {P}]')
                if not bool(((v == 0) | (v == 1)).all()):
                    raise ValueError(f'mask tape {k!r} holds values other than 0 and 1')
            device = self.t._embedding.weight.device
            return 'tape', {k: v.to(device=device, dtype=torch.uint8).contiguous() for k, v in masks.items()}
        if seed is not None:
            return 'seed', check_seed(seed)
        return 'shared', None

    def open(self, text, speaker=None, language=None, seed=None, masks=None, durations=None, alignment=None):
        """Queues a text for the next run() -> its id.  Takes `inference`'s text, speaker, language, durations and alignment, and a seed
        or a mask tape."""
        source = self.check(text, speaker, language, seed, masks, durations, alignment)
        if len(self.ids) >= self.max_texts:
            raise ValueError(f'the decoder pool is full: {self.max_texts} texts are open')
        tid = self.next_id
        self.next_id += 1
        if source[0] == 'shared':
            source = ('shared', tid)
        plan = _forced_plan(self.t._decoder, text, durations, alignment, self.t._embedding.weight.device)
        self.queue.append((tid, text, speaker, language, source, plan))
        return tid

    def close(self, tid):
        """Drops an open text before its stop cut."""
        if tid in self.rows.keys:
            self.rows.close(tid)
            del self.pre[tid], self.released[tid]
        elif any(q[0] == tid for q in self.queue):
            self.queue = [q for q in self.queue if q[0] != tid]
        else:
            raise ValueError(f'unknown or finished text {tid}')

    def _admit(self):
        t, groups = self.t, {}
        for q in self.queue:
            _, _, speaker, language, _, _ = q
            form = (speaker is None, None if language is None else (language.dim(), language.shape[-1] if language.dim() == 3 else 0))
            groups.setdefault(form, []).append(q)
        self.queue = []
        for group in groups.values():
            ids, texts, speakers, languages, sources, plans = zip(*group)
            encoded, mask, speaker, language = t._encode_group(list(texts), None if speakers[0] is None else list(speakers),
                                                                None if languages[0] is None else list(languages))
            memory = t._decoder._memory(encoded, speaker, language)
            self.rows.add(memory, [int(x.shape[0]) for x in texts], ids, sources)
            self.rows.set_plans(plans)
            for i in ids:
                self.pre[i], self.released[i] = [], 0

    def run(self):
        """One decoder call over every open text -> {id: post-net chunk [num_mels, n]} (a chunk may hold no frames).  A text leaves after
        the call that finds its stop cut or reaches hp.max_output_length frames."""
        t = self.t
        if not self.queue and not len(self.rows):
            return {}
        was_training = t.training
        t.eval()
        try:
            with torch.no_grad():
                if self.queue:
                    self._admit()
                spec, _, _ = self.rows.step(self.chunk_steps)
                dec, halo, rows, spans = t._decoder, t._postnet.halo(), self.rows, {}
                for j, u in enumerate(rows.keys):
                    self.pre[u].append(spec[j])
                    done, cut = rows.done[j], rows.rules[j].cut
                    end = stream_release(done, cut, dec._max_frames, halo)
                    final = cut is not None or done >= dec._max_frames
                    spans[u] = (self.released[u], end, end if final else done)
                    self.released[u] = end
                posts = t._postnet_windows(self.pre, spans, halo)
                for u in rows.retire():
                    del self.pre[u], self.released[u]
                return posts
        finally:
            t.train(was_training)


def stream_release(done, cut, max_frames, halo):
    """Frames of a streamed utterance whose post-net output is final after `done` decoded frames: every frame up to the stop cut once it is
    known (or up to max_frames once the decode has reached it), else every frame with `halo` decoded frames to its right."""
    if cut is not None:
        return min(cut, max_frames)
    if done >= max_frames:
        return max_frames
    return max(done - halo, 0)


def postnet_window(t0, t1, halo, avail):
    """The decoded frames [w0, w1) the post-net runs over to produce its final frames [t0, t1), of `avail` decoded frames (the whole
    utterance once the cut is known): `halo` frames on each side, clipped to the decoded ones."""
    return max(t0 - halo, 0), min(t1 + halo, avail)


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


def _forced_plan(dec, text, durations, alignment, device):
    """Checks one text's attention plan -> None (a free decode), or (weights [S, L] float32 on `device`, frames): `durations` (int [L]
    frames per symbol, each >= 0; functional.durations_to_alignment at the decoder's r, sum(d) frames) or `alignment` (float [S, L], finite
    and >= 0; S r frames), L the text's length.  ValueError for both given, a wrong rank or dtype, another L, negative or non-finite values,
    0 frames, or more than hp.max_output_length frames.  device None validates only."""
    if durations is None and alignment is None:
        return None
    if durations is not None and alignment is not None:
        raise ValueError('forced synthesis: give a text durations or an alignment, not both')
    L, r = int(text.shape[0]), dec._outputs_per_step
    if durations is not None:
        d = F._durations_host(durations, 'forced synthesis')
        if d.shape[0] != L:
            raise ValueError(f'forced synthesis: {d.shape[0]} durations for a text of {L} symbols')
        frames = int(d.sum())
    else:
        if not torch.is_tensor(alignment) or alignment.dim() != 2 or not alignment.dtype.is_floating_point:
            raise ValueError('forced synthesis: an alignment is a float tensor [S, L]')
        if alignment.shape[1] != L:
            raise ValueError(f'forced synthesis: an alignment over {alignment.shape[1]} symbols for a text of {L} symbols')
        if not bool(torch.isfinite(alignment).all()) or bool((alignment < 0).any()):
            raise ValueError('forced synthesis: alignment weights must be finite and >= 0')
        frames = int(alignment.shape[0]) * r
    if frames == 0:
        raise ValueError('forced synthesis: the plan has 0 frames')
    if frames > dec._max_frames:
        raise ValueError(f'forced synthesis: the plan has {frames} frames, more than hp.max_output_length = {dec._max_frames}')
    if device is None:
        return None
    weights = F.durations_to_alignment(d, r) if durations is not None else alignment
    return weights.to(device=device, dtype=torch.float32).contiguous(), frames


def _plan_lists(texts, durations, alignments):
    """durations / alignments of a batch call (None, or one entry or None per text) -> two lists with one entry per text."""
    out = []
    for name, items in (('durations', durations), ('alignments', alignments)):
        items = [None] * len(texts) if items is None else list(items)
        if len(items) != len(texts):
            raise ValueError(f'forced synthesis: {len(items)} {name} for {len(texts)} texts')
        out.append(items)
    return out


def _batch_plans(dec, texts, durations, alignments):
    """Every text's plan checked first (ValueError), then built on the model's device -> one plan or None per text."""
    durations, alignments = _plan_lists(texts, durations, alignments)
    for t, d, a in zip(texts, durations, alignments):
        _forced_plan(dec, t, d, a, None)
    device = dec._prenet._layers[0].weight.device
    return [_forced_plan(dec, t, d, a, device) for t, d, a in zip(texts, durations, alignments)]


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
