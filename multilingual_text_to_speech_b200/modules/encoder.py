"""Encoders (surface of reference modules/encoder.py:9-221) on the b200tts library ops."""
import torch
from torch.nn import Sequential, ModuleList, LSTM, Embedding

from .. import functional as F
from .. import _lib
from .layers import ConvBlock, HighwayConvBlock, ConvBlockGenerated, HighwayConvBlockGenerated
from ..params.params import Params as hp  # noqa: F401  (kept for parity with the reference module surface)


class Encoder(torch.nn.Module):
    """Vanilla Tacotron 2 encoder: 3 x (conv5 + BN + ReLU + dropout) -> packed bi-LSTM (encoder.py:9-45)."""

    def __init__(self, input_dim, output_dim, num_blocks, kernel_size, dropout, generated=False):
        super().__init__()
        assert num_blocks > 0, 'There must be at least one convolutional block in the encoder.'
        assert output_dim % 2 == 0, 'Bidirectional LSTM output dimension must be divisible by 2.'
        convs = [ConvBlock(input_dim, output_dim, kernel_size, dropout, 'relu')] + \
                [ConvBlock(output_dim, output_dim, kernel_size, dropout, 'relu') for _ in range(num_blocks - 1)]
        for j, block in enumerate(convs):
            block._mask_key = f'enc{j}'
        self._convs = Sequential(*convs)
        self._lstm = LSTM(output_dim, output_dim // 2, batch_first=True, bidirectional=True)   # parameter container

    def forward(self, x, x_lenghts, x_langs=None, padded=False):
        """padded (eval only): x is a zero-padded batch of utterances of lengths x_lenghts; each is encoded as if it were alone."""
        x = x.transpose(1, 2).contiguous()
        x = _run_blocks(self._convs, x, x_lenghts if padded else None)
        x = x.transpose(1, 2).contiguous()
        params = [getattr(self._lstm, name + '_l0' + suffix) for suffix in ('', '_reverse')
                  for name in ('weight_ih', 'weight_hh', 'bias_ih', 'bias_hh')]
        return F.bilstm(x, x_lenghts.to(x.device), params)


class ConditionalEncoder(torch.nn.Module):
    """Encoder with a language embedding concatenated to every input character (encoder.py:48-71)."""

    def __init__(self, num_langs, langs_embedding_dim, encoder_args):
        super().__init__()
        self._language_embedding = Embedding(num_langs, langs_embedding_dim)
        encoder_args = list(encoder_args)
        encoder_args[0] += langs_embedding_dim
        self._encoder = Encoder(*encoder_args)

    def forward(self, x, x_lenghts, x_langs, padded=False):
        x_langs = torch.argmax(x_langs, dim=2)
        l = F.embedding(self._language_embedding.weight, x_langs)
        x = torch.cat((x, l), dim=-1)
        if padded:
            x = _zero_padding(x, x_lenghts)
        return self._encoder(x, x_lenghts, padded=padded)


class MultiEncoder(torch.nn.Module):
    """One vanilla encoder per language, outputs mixed by the language weights (encoder.py:74-97)."""

    def __init__(self, num_langs, encoder_args):
        super().__init__()
        self._num_langs = num_langs
        self._encoders = ModuleList([Encoder(*encoder_args) for _ in range(num_langs)])

    def forward(self, x, x_lenghts, x_langs, padded=False):
        """x_langs [B, L, G]: per-character language weights.  The reference divides by `x_langs.sum(2, keepdim=True)[0]`
        (encoder.py:88): the weight sums of utterance 0, broadcast over the batch.  A padded batch (eval) normalises every utterance by
        its own sums instead, as when it is encoded alone; its padded positions get weight 0."""
        share = _language_share(x_langs) if padded else x_langs / x_langs.sum(dim=2, keepdim=True)[0].unsqueeze(0)     # [B, L, G]
        mixed = None
        for lang, encoder in enumerate(self._encoders):
            w = share[..., lang:lang + 1]
            if not bool((w != 0).any()):
                continue                                  # languages that are not requested are not encoded at all
            part = w * encoder(x, x_lenghts, padded=padded)
            mixed = part if mixed is None else mixed + part
        return mixed


def _zero_padding(x, lengths):
    """x [B, L, ...] with every position l >= lengths[b] set to 0."""
    keep = torch.arange(x.shape[1], device=x.device).unsqueeze(0) < lengths.to(x.device).unsqueeze(1)
    return x.masked_fill(~keep.view(*keep.shape, *([1] * (x.dim() - 2))), 0.0)


def _language_share(x_langs):
    """Per-character language weights [B, L, G] normalised by their own sums; all-zero rows (padding) stay 0."""
    total = x_langs.sum(dim=2, keepdim=True)
    return torch.where(total != 0, x_langs / torch.where(total != 0, total, torch.ones_like(total)), torch.zeros_like(x_langs))


def _run_blocks(blocks, x, lengths):
    """A Sequential of conv blocks; with `lengths` (a zero-padded eval batch) every block zeroes the positions past them."""
    if lengths is None:
        return blocks(x)
    if isinstance(x, tuple):                 # generated blocks pass (generator embedding, x)
        e, x = x
        lengths = lengths.to(device=x.device, dtype=torch.int32)
        for block in blocks:
            _, x = block((e, x), lengths)
        return e, x
    lengths = lengths.to(device=x.device, dtype=torch.int32)
    for block in blocks:
        x = block(x, lengths)
    return x


def _mix_languages(per_language, x_langs):
    """Code-switching / accent blending at inference (encoder.py:213-219): `per_language` [B*G, L, E] holds every utterance encoded by
    every language's generated weights (row b*G + g), `x_langs` [B, L, G] the per-character language weights; each character takes
    the convex combination given by its own normalised weights, summed over the languages in order as the reference does."""
    G = x_langs.shape[2]
    per_language = per_language.reshape(x_langs.shape[0], G, *per_language.shape[1:])
    share = _language_share(x_langs)
    mixed = share[:, :, 0:1] * per_language[:, 0]
    for g in range(1, G):
        mixed = mixed + share[:, :, g:g + 1] * per_language[:, g]
    return mixed


def _expand_groups(x, x_langs, padded, groups):
    """Inference input of a grouped encoder: one utterance (the reference's batch-1 branch) or a padded batch is repeated for every
    language, row b*G + g = utterance b under language g, so that sample row b of the grouped layout is utterance b."""
    mixing = x_langs is not None and (padded or x_langs.shape[0] == 1)
    if mixing:
        x = x.repeat_interleave(groups, dim=0)
    return x, mixing


class ConvolutionalEncoder(torch.nn.Module):
    """Fully convolutional grouped encoder with plain weights (encoder.py:100-156).

    Input [B, L, F] with B divisible by the number of languages and sample b belonging to language b % groups."""

    def __init__(self, input_dim, output_dim, dropout, groups=1):
        super().__init__()
        self._groups, self._input_dim, self._output_dim = groups, input_dim, output_dim
        input_dim *= groups
        output_dim *= groups
        layers = [ConvBlock(input_dim, output_dim, 1, dropout, activation='relu', groups=groups),
                  ConvBlock(output_dim, output_dim, 1, dropout, groups=groups)] + \
                 [HighwayConvBlock(output_dim, output_dim, 3, dropout, dilation=3 ** i, groups=groups) for i in range(4)] + \
                 [HighwayConvBlock(output_dim, output_dim, 3, dropout, dilation=3 ** i, groups=groups) for i in range(4)] + \
                 [HighwayConvBlock(output_dim, output_dim, 3, dropout, dilation=1, groups=groups) for _ in range(2)] + \
                 [HighwayConvBlock(output_dim, output_dim, 1, dropout, dilation=1, groups=groups) for _ in range(2)]
        for j, block in enumerate(layers):
            block._mask_key = f'enc{j}'
        self._layers = Sequential(*layers)

    def forward(self, x, x_lenghts=None, x_langs=None, padded=False):
        x, mixing = _expand_groups(x, x_langs, padded, self._groups)
        bs = x.shape[0]
        if bs % self._groups != 0:
            raise _lib.B200TTSError(f'batch size {bs} must be divisible by the number of languages {self._groups}')
        x = x.transpose(1, 2).reshape(bs // self._groups, self._groups * self._input_dim, -1).contiguous()
        x = _run_blocks(self._layers, x, x_lenghts if padded else None)
        x = x.reshape(bs, self._output_dim, -1).transpose(1, 2)
        return _mix_languages(x, x_langs) if mixing else x


class GeneratedConvolutionalEncoder(torch.nn.Module):
    """Grouped convolutional encoder whose weights are generated from language embeddings (encoder.py:159-221)."""

    def __init__(self, input_dim, output_dim, dropout, embedding_dim, bottleneck_dim, groups=1):
        super().__init__()
        self._groups, self._input_dim, self._output_dim = groups, input_dim, output_dim
        input_dim *= groups
        output_dim *= groups
        gen = (embedding_dim, bottleneck_dim)
        layers = [ConvBlockGenerated(*gen, input_dim, output_dim, 1, dropout=dropout, activation='relu', groups=groups),
                  ConvBlockGenerated(*gen, output_dim, output_dim, 1, dropout=dropout, groups=groups)] + \
                 [HighwayConvBlockGenerated(*gen, output_dim, output_dim, 3, dropout=dropout, dilation=3 ** i, groups=groups)
                  for i in range(4)] + \
                 [HighwayConvBlockGenerated(*gen, output_dim, output_dim, 3, dropout=dropout, dilation=3 ** i, groups=groups)
                  for i in range(4)] + \
                 [HighwayConvBlockGenerated(*gen, output_dim, output_dim, 3, dropout=dropout, dilation=1, groups=groups)
                  for _ in range(2)] + \
                 [HighwayConvBlockGenerated(*gen, output_dim, output_dim, 1, dropout=dropout, dilation=1, groups=groups)
                  for _ in range(2)]
        for j, block in enumerate(layers):
            block._mask_key = f'enc{j}'
        self._layers = Sequential(*layers)
        self._embedding = Embedding(groups, embedding_dim)

    def forward(self, x, x_lenghts=None, x_langs=None, padded=False):
        x, mixing = _expand_groups(x, x_langs, padded, self._groups)
        e = self._embedding.weight                       # Embedding(arange(groups)) == the table itself
        bs = x.shape[0]
        if bs % self._groups != 0:
            raise _lib.B200TTSError(f'batch size {bs} must be divisible by the number of languages {self._groups}')
        x = x.transpose(1, 2).reshape(bs // self._groups, self._groups * self._input_dim, -1).contiguous()
        _, x = _run_blocks(self._layers, (e, x), x_lenghts if padded else None)
        x = x.reshape(bs, self._output_dim, -1).transpose(1, 2)
        return _mix_languages(x, x_langs) if mixing else x
