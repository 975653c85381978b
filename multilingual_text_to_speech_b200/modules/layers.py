"""Building blocks (surface of reference modules/layers.py:18-178) on top of the b200tts library ops."""
import torch
from torch.nn import Sequential, ReLU, Sigmoid, Tanh, Identity, Dropout, Conv1d, ConstantPad1d, BatchNorm1d

from .. import functional as F
from ..rng import MaskSource
from .generated import Conv1dGenerated, BatchNorm1dGenerated


def get_activation(name):
    return {'relu': ReLU(), 'sigmoid': Sigmoid(), 'tanh': Tanh(), 'identity': Identity()}[name]


def _require_eval(block):
    """The length-masked block normalises with the running statistics and applies no dropout: it exists for eval mode only."""
    if block.training:
        raise RuntimeError('conv block: per-sample lengths (a zero-padded batch) are supported in eval mode only; call .eval() first')


class ZoneoutLSTMCell(torch.nn.LSTMCell):
    """LSTM cell with zoneout (layers.py:18-34).  Inside `Decoder` the recurrence runs in the fused decoder op, which reads the
    parameters and `zoneout_h` / `zoneout_c` from here; the standalone `forward` is one library cell step (with autograd)."""

    def __init__(self, input_size, hidden_size, zoneout_rate_hidden, zoneout_rate_cell, bias=True):
        super().__init__(input_size, hidden_size, bias)
        self.zoneout_c = zoneout_rate_cell
        self.zoneout_h = zoneout_rate_hidden

    def forward(self, cell_input, h, c):
        mh = mc = None
        if self.training:
            mh = MaskSource.keep_mask('cell_h', h.shape, self.zoneout_h, h.device)
            mc = MaskSource.keep_mask('cell_c', c.shape, self.zoneout_c, c.device)
        from .. import _lib
        return F.lstm_cell(cell_input, h, c, self.weight_ih, self.weight_hh, self.bias_ih, self.bias_hh, _lib.CELL_ZONEOUT, self.training,
                           self.zoneout_h, self.zoneout_c, mh, mc)


class DropoutLSTMCell(torch.nn.LSTMCell):
    """LSTM cell with dropout on the hidden state (layers.py:37-47); fused inside `Decoder`, standalone `forward` = one library step."""

    def __init__(self, input_size, hidden_size, dropout_rate, bias=True):
        super().__init__(input_size, hidden_size, bias)
        self._dropout = Dropout(dropout_rate)

    def forward(self, cell_input, h, c):
        mh = MaskSource.keep_mask('cell_h', h.shape, self._dropout.p, h.device) if self.training else None
        from .. import _lib
        return F.lstm_cell(cell_input, h, c, self.weight_ih, self.weight_hh, self.bias_ih, self.bias_hh, _lib.CELL_DROPOUT, self.training,
                           self._dropout.p, 0.0, mh, None)


class ConvBlock(torch.nn.Module):
    """pad -> Conv1d(no bias) -> BatchNorm1d -> activation -> Dropout, channel-first (layers.py:50-86).

    The torch sub-modules inside `_block` only carry parameters / buffers (names `_block.1.weight`,
    `_block.2.*` as in the reference); the computation is one fused library op.
    """

    def __init__(self, input_channels, output_channels, kernel, dropout=0.0, activation='identity', dilation=1, groups=1,
                 batch_norm=True):
        super().__init__()
        assert batch_norm, 'every reference call site uses batch_norm=True'
        assert kernel % 2 == 1, 'even kernels are not used on the hot path'
        self._groups, self._kernel, self._dilation = groups, kernel, dilation
        self._activation_name, self._dropout_rate = activation, dropout
        p = (kernel - 1) * dilation // 2
        layers = [ConstantPad1d(p, 0.0),
                  Conv1d(input_channels, output_channels, kernel, padding=0, dilation=dilation, groups=groups, bias=False),
                  BatchNorm1d(output_channels), get_activation(activation), Dropout(dropout)]
        self._block = Sequential(*layers)
        self._mask_key = None
        self._highway = False

    def _run(self, x, counts=None):
        conv, bn = self._block[1], self._block[2]
        G = self._groups
        cout = conv.weight.shape[0] // G
        keep = None
        if self.training and self._dropout_rate > 0.0:
            keep = MaskSource.keep_mask(self._mask_key, (x.shape[0], conv.weight.shape[0], x.shape[2]), self._dropout_rate, x.device)
        out = F.conv_block(x, conv.weight, bn.weight, bn.bias, bn.running_mean, bn.running_var, keep, G, self._kernel,
                           self._dilation, self._activation_name, self._highway, self.training, bn.eps, bn.momentum,
                           self._dropout_rate if keep is not None else 0.0, cout, counts=counts)
        if self.training:
            bn.num_batches_tracked += 1
        return out

    def forward(self, x, lengths=None, counts=None):
        """lengths (eval only): per-sample lengths of a zero-padded batch; outputs past each length are 0.
        counts: int32 [groups] on the device, the utterances in each channel block (rows past them are vacant, see F.conv_block)."""
        if lengths is not None:
            _require_eval(self)
            conv, bn = self._block[1], self._block[2]
            return F.conv_block_masked(x, lengths, conv.weight, bn.weight, bn.bias, bn.running_mean, bn.running_var, self._groups,
                                       self._kernel, self._dilation, self._activation_name, self._highway, bn.eps,
                                       conv.weight.shape[0] // self._groups)
        return self._run(x, counts)


class HighwayConvBlock(ConvBlock):
    """Gated convolution: out = h2 * sigmoid(h1) + x * (1 - sigmoid(h1)) (layers.py:134-153)."""

    def __init__(self, input_channels, output_channels, kernel, dropout=0.0, activation='identity', dilation=1, groups=1,
                 batch_norm=True):
        super().__init__(input_channels, 2 * output_channels, kernel, dropout, activation, dilation, groups, batch_norm)
        self._gate = Sigmoid()
        self._highway = True


class ConvBlockGenerated(torch.nn.Module):
    """Conv block whose kernel and batch-norm affine are generated per language (layers.py:89-131).
    Takes and returns the tuple (generator_embedding, x)."""

    def __init__(self, embedding_dim, bottleneck_dim, input_channels, output_channels, kernel, dropout=0.0,
                 activation='identity', dilation=1, groups=1, batch_norm=True):
        super().__init__()
        assert batch_norm and kernel % 2 == 1
        self._groups, self._kernel, self._dilation = groups, kernel, dilation
        self._activation_name, self._dropout_rate = activation, dropout
        p = (kernel - 1) * dilation // 2
        self._padding = ConstantPad1d(p, 0.0)
        self._convolution = Conv1dGenerated(embedding_dim, bottleneck_dim, input_channels, output_channels, kernel, padding=0,
                                            dilation=dilation, groups=groups, bias=False)
        self._regularizer = BatchNorm1dGenerated(embedding_dim, bottleneck_dim, output_channels, groups=groups)
        self._activation = Sequential(get_activation(activation), Dropout(dropout))
        self._mask_key = None
        self._highway = False

    def forward(self, x, lengths=None, counts=None):
        """lengths (eval only): per-sample lengths of a zero-padded batch; outputs past each length are 0.
        counts: int32 [groups] on the device, the utterances in each channel block (rows past them are vacant, see F.conv_block)."""
        if lengths is not None:
            _require_eval(self)
        e, x = x
        bn = self._regularizer
        G = self._groups
        kernel = self._convolution.generate(e)                 # [G*Cout, Cin, k]
        affine = bn.generate(e)                                # [G, 2*Cout]
        cout = kernel.shape[0] // G
        if lengths is not None:
            return e, F.conv_block_masked(x, lengths, kernel, affine[:, :cout], affine[:, cout:], bn.running_mean, bn.running_var, G,
                                          self._kernel, self._dilation, self._activation_name, self._highway, bn._eps, 2 * cout)
        keep = None
        if self.training and self._dropout_rate > 0.0:
            keep = MaskSource.keep_mask(self._mask_key, (x.shape[0], kernel.shape[0], x.shape[2]), self._dropout_rate, x.device)
        out = F.conv_block(x, kernel, affine[:, :cout], affine[:, cout:], bn.running_mean, bn.running_var, keep, G,
                           self._kernel, self._dilation, self._activation_name, self._highway, self.training, bn._eps,
                           bn._momentum, self._dropout_rate if keep is not None else 0.0, 2 * cout, counts=counts)
        if self.training:
            bn.num_batches_tracked += 1
        return e, out


class HighwayConvBlockGenerated(ConvBlockGenerated):
    """Gated convolution with generated weights (layers.py:156-178)."""

    def __init__(self, embedding_dim, bottleneck_dim, input_channels, output_channels, kernel, dropout=0.0,
                 activation='identity', dilation=1, groups=1, batch_norm=True):
        super().__init__(embedding_dim, bottleneck_dim, input_channels, 2 * output_channels, kernel, dropout, activation,
                         dilation, groups, batch_norm)
        self._gate = Sigmoid()
        self._highway = True
