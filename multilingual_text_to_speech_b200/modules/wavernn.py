"""WaveRNN vocoder, the fatchord architecture (github.com/fatchord/WaveRNN, models/fatchord_version.py) as the reference's published samples
use it: log-mel spectrogram -> waveform on the GPU.

Submodule and parameter names follow fatchord, so its state_dict (or one of a fork with the same architecture) loads with load_state_dict.
Batched (folded) generation (generate_batch) and teacher-forced training (forward, wavernn_loss, vocoder_batch) are provided.  Mels go
in as given: any normalisation a generation script applies before the vocoder is the caller's business.

Stages of generate_batch (all on the library's kernels):
  * upsampling network: MelResNet on the convolution-block op (eval-mode batch norm) and the GEMM, the mel path's stretch + FIR layers on
    b200tts_wavernn_upsample_layer (the last one evaluated inside the fold kernel, with the `indent` cut);
  * per chunk of loop steps: the folded features (b200tts_wavernn_fold), the products that do not depend on the previous sample on the GEMM,
    then the persistent sample loop (b200tts_wavernn_run);
  * b200tts_wavernn_unfold: mu-law decode (RAW), cross-fade, overlap-add, cut to (F - 1) hop samples and the 20-hop fade-out.

Stages of forward (training, with autograd):
  * MelResNet on the convolution-block op (train-mode batch norm updates the running statistics like nn.BatchNorm1d): conv_in as its
    convolution-only stage over the mel window (the 'same'-padded op's middle outputs are the unpadded convolution), then its batch-norm
    stage; conv_out and every linear layer on the library GEMM; the aux stretch and the mel path's layers with their library adjoints;
  * both GRUs on the persistent fp32 sequence loops (b200tts_gru_seq_forward / _backward);
  * wavernn_loss: one fused kernel per mode writes the loss and d logits."""
import collections
import contextlib

import numpy as np
import torch
from torch import nn

from .. import _lib
from .. import functional as F
from ..utils.audio import _return_like, _work_device
from .stream_pool import Stream, VocoderStreamPool, check_preemphasis, generate_stream as _generate_stream

# fp32 bytes of the conditioning products and folded features held at once: bounds the chunk of loop steps
COND_BYTES = 512 << 20
# loop steps per StreamPool.run at most, in hops (then bounded by COND_BYTES): 16 hops are 0.2 s of audio at 22050 Hz, so a stream's chunks
# come at least that often while it is behind, and the host work around each loop call is spread over 4400 steps
POOL_CALL_HOPS = 16
LOG_SCALE_MIN = float(np.log(1e-14))
# training windows the sequence loops take: at most this many hops of samples, at most 64 of them
MAX_TRAIN_HOPS = 16
MAX_TRAIN_BATCH = 64


# ---- labels and training windows (fatchord's utils/distribution.py, utils/dsp.py and collate_vocoder) ----
def label_2_float(x, bits):
    """2 x / (2^bits - 1) - 1, in fp32 like fatchord's torch expression."""
    return 2 * torch.as_tensor(x).float() / (2 ** bits - 1.) - 1.


def float_2_label(x, bits):
    """trunc(clip((x + 1) (2^bits - 1) / 2, 0, 2^bits - 1)) as int64: fatchord's MOL labels of a waveform in [-1, 1]."""
    x = np.asarray(x, dtype=np.float64)
    if x.size and np.abs(x).max() > 1.0:
        raise ValueError('float_2_label expects samples in [-1, 1]')
    return np.clip((x + 1.) * (2 ** bits - 1) / 2, 0, 2 ** bits - 1).astype(np.int64)


def encode_mu_law(x, mu):
    """fatchord's encode_mu_law(x, mu = 2^bits): floor((sign(x) log(1 + m|x|) / log(1 + m) + 1) / 2 m + 0.5) with m = mu - 1, int64."""
    m = mu - 1
    x = np.asarray(x, dtype=np.float64)
    fx = np.sign(x) * np.log(1 + m * np.abs(x)) / np.log(1 + m)
    return np.floor((fx + 1) / 2 * m + 0.5).astype(np.int64)


def mel_window(seq_len, hop, pad):
    """Frames of one training window's mel: seq_len / hop + 2 pad."""
    if seq_len < hop or seq_len % hop:
        raise ValueError(f'seq_len {seq_len} must be a positive multiple of the hop {hop}')
    return seq_len // hop + 2 * pad


def draw_offsets(frames, seq_len, hop, pad, rng=None):
    """One mel offset per utterance of `frames` frames, uniform in [0, F - 2 - (mel_win + 2 pad)) as fatchord's collate_vocoder draws them."""
    rng = np.random.default_rng() if rng is None else rng
    win = mel_window(seq_len, hop, pad)
    hi = [int(f) - 2 - (win + 2 * pad) for f in frames]
    if min(hi) < 1:
        raise ValueError(f'an utterance of {min(frames)} frames is too short for a window of {win} frames')
    return [int(rng.integers(0, h)) for h in hi]


def vocoder_batch(mels, labels, offsets, mode, bits, seq_len, pad, hop):
    """fatchord's collate_vocoder with explicit offsets: host mels [feat, F_i], integer labels [samples_i] and mel offsets o_i ->
    (x [B, seq_len] fp32, y [B, seq_len] (RAW int64 labels, MOL fp32 in [-1, 1]), m [B, feat, mel_win] fp32) on the CPU.  m = mel[:, o:o +
    mel_win]; the labels window starts at (o + pad) hop and holds seq_len + 1 labels; x = label_2_float(labels[:seq_len], 16 for MOL, else
    bits), y = labels[1:] (MOL: label_2_float(y, 16))."""
    if mode not in _lib.WAVERNN_MODES:
        raise ValueError(f'unknown mode {mode!r}; expected RAW or MOL')
    if not (len(mels) == len(labels) == len(offsets)) or len(mels) == 0:
        raise ValueError(f'{len(mels)} mels, {len(labels)} label sequences and {len(offsets)} offsets: need as many of each, at least one')
    win = mel_window(seq_len, hop, pad)
    ms, ls = [], []
    for i, (mel, lab, o) in enumerate(zip(mels, labels, offsets)):
        mel, lab, o = np.asarray(mel), np.asarray(lab), int(o)
        s0 = (o + pad) * hop
        if o < 0 or o + win > mel.shape[-1] or s0 + seq_len + 1 > lab.shape[0]:
            raise ValueError(f'offset {o} of item {i} leaves its window outside the mel ({mel.shape[-1]} frames) or the labels '
                             f'({lab.shape[0]})')
        ms.append(mel[:, o:o + win])
        ls.append(lab[s0:s0 + seq_len + 1])
    m = torch.tensor(np.stack(ms).astype(np.float32))
    lab = torch.tensor(np.stack(ls).astype(np.int64))
    b = 16 if mode == 'MOL' else bits
    x = label_2_float(lab[:, :seq_len], b)
    y = lab[:, 1:]
    if mode == 'MOL':
        y = label_2_float(y, b)
    return x, y, m


class VocoderCorpus:
    """A WaveRNN training corpus packed into one GPU's memory once, from which each batch's windows are cut on the device in one launch
    (b200tts_wavernn_cut_windows): `batch(ids, offsets)` returns vocoder_batch's (x, y, m) for the same utterances and offsets, bit for bit,
    without host slicing or a host-to-device copy of the windows.

    mels: host mels [feat, F_i]; labels: integer labels [N_i] (RAW labels of `bits` bits, or MOL's 16-bit labels), in [0, 2^16).  Device
    footprint: 2 bytes per sample plus 4 feat bytes per frame; a corpus larger than one GPU's memory is the caller's to shard or subset.
    The lengths stay on the host, so `batch` validates its table (ids, offsets, the utterances' labels) from host data alone and raises
    ValueError before any device work; an utterance whose labels lie outside [0, 2^16) is stored as zeros and refused by `batch`."""

    def __init__(self, mels, labels, mode, bits, seq_len, pad, hop, device):
        if mode not in _lib.WAVERNN_MODES:
            raise ValueError(f'unknown mode {mode!r}; expected RAW or MOL')
        if len(mels) != len(labels) or len(mels) == 0:
            raise ValueError(f'{len(mels)} mels and {len(labels)} label sequences: need as many of each, at least one')
        if not 1 <= int(bits) <= 16:
            raise ValueError(f'bits {bits} outside [1, 16]')
        self.win = mel_window(seq_len, hop, pad)
        if seq_len // hop > MAX_TRAIN_HOPS:
            raise ValueError(f'seq_len {seq_len}: at most {MAX_TRAIN_HOPS} hops of {hop}')
        self.mode, self.bits, self.seq_len, self.pad, self.hop = mode, int(bits), int(seq_len), int(pad), int(hop)
        self.device = torch.device(device)
        mels = [np.asarray(m, dtype=np.float32) for m in mels]
        self.feat = mels[0].shape[0] if mels[0].ndim == 2 else -1
        for i, m in enumerate(mels):
            if m.ndim != 2 or m.shape[0] != self.feat or m.shape[1] < 1:
                raise ValueError(f'mel {i} of shape {m.shape}: expected [{self.feat}, frames >= 1]')
        packed, self.labels_ok = [], []
        for i, lab in enumerate(labels):
            lab = np.asarray(lab)
            if lab.ndim != 1 or not (np.issubdtype(lab.dtype, np.integer) or lab.size == 0):
                raise ValueError(f'labels {i} of shape {lab.shape} and dtype {lab.dtype}: expected one integer sequence')
            ok = lab.size == 0 or (int(lab.min()) >= 0 and int(lab.max()) < 1 << 16)
            self.labels_ok.append(ok)
            packed.append(lab.astype(np.uint16) if ok else np.zeros(lab.shape, np.uint16))
        self.frames = [m.shape[1] for m in mels]
        self.samples = [p.shape[0] for p in packed]
        self.frame_start = np.concatenate(([0], np.cumsum(self.frames)[:-1])).astype(np.int64)
        self.sample_start = np.concatenate(([0], np.cumsum(self.samples)[:-1])).astype(np.int64)
        dev = self.device
        self.mels = torch.from_numpy(np.concatenate(mels, axis=1)).to(dev)
        # uint16 labels held in an int16 tensor (the kernel reads the bits as uint16)
        self.labels = torch.from_numpy(np.concatenate(packed).view(np.int16)).to(dev)
        self.frame_start_dev = torch.from_numpy(self.frame_start).to(dev)
        self.sample_start_dev = torch.from_numpy(self.sample_start).to(dev)

    def __len__(self):
        return len(self.frames)

    @property
    def nbytes(self):
        return 2 * sum(self.samples) + 4 * self.feat * sum(self.frames)

    def _check_ids(self, ids):
        for i, u in enumerate(ids):
            if not 0 <= int(u) < len(self.frames):
                raise ValueError(f'utterance id {u} of item {i} outside [0, {len(self.frames)})')

    def draw_offsets(self, ids, rng=None):
        """draw_offsets for the utterances `ids`: the same draws from the same numpy generator."""
        self._check_ids(ids)
        return draw_offsets([self.frames[int(u)] for u in ids], self.seq_len, self.hop, self.pad, rng)

    def table(self, ids, offsets):
        """The host table int32 [B, 2] of (utterance, mel offset), validated as vocoder_batch validates its windows: ValueError for B outside
        1 to 64, an id out of range, a window outside its utterance's mel or labels, or an utterance whose labels lie outside [0, 2^16)."""
        ids, offsets = list(ids), list(offsets)
        if len(ids) != len(offsets) or len(ids) == 0:
            raise ValueError(f'{len(ids)} utterance ids and {len(offsets)} offsets: need as many of each, at least one')
        if len(ids) > MAX_TRAIN_BATCH:
            raise ValueError(f'a batch of {len(ids)} windows: need 1 to {MAX_TRAIN_BATCH}')
        self._check_ids(ids)
        for i, (u, o) in enumerate(zip(ids, offsets)):
            u, o = int(u), int(o)
            if o < 0 or o + self.win > self.frames[u] or (o + self.pad) * self.hop + self.seq_len + 1 > self.samples[u]:
                raise ValueError(f'offset {o} of item {i} leaves its window outside the mel ({self.frames[u]} frames) or the labels '
                                 f'({self.samples[u]})')
            if not self.labels_ok[u]:
                raise ValueError(f'labels of utterance {u} (item {i}) lie outside [0, 65536)')
        return np.array([[int(u), int(o)] for u, o in zip(ids, offsets)], dtype=np.int32)

    def cut(self, table, out=None):
        """(x, y, m) of the device table int32 [B, 2], which is not checked (see `table`); written into `out` when given."""
        return F.wavernn_cut_windows(self.mode, self.bits, self.seq_len, self.pad, self.hop, self.mels, self.frame_start_dev, self.labels,
                                     self.sample_start_dev, table, out)

    def batch(self, ids, offsets):
        """vocoder_batch(mels[ids], labels[ids], offsets, ...) on the device: (x [B, seq_len] fp32, y [B, seq_len] (RAW int64, MOL fp32),
        m [B, feat, mel_win] fp32).  The table is validated on the host, then copied in with one pinned host-to-device copy."""
        host = torch.from_numpy(self.table(ids, offsets))
        if self.device.type == 'cuda':
            host = host.pin_memory()
        return self.cut(host.to(self.device, non_blocking=True))


def wavernn_loss(logits, y, mode):
    """fatchord's training loss of forward's logits [B, T, n_classes] against y [B, T]: RAW F.cross_entropy against the labels, MOL
    discretized_mix_logistic_loss (65536 classes, log scales clamped at log 1e-14); the mean over B T, with autograd."""
    if mode not in _lib.WAVERNN_MODES:
        raise ValueError(f'unknown mode {mode!r}; expected RAW or MOL')
    n = logits.shape[-1]
    if tuple(y.shape) != tuple(logits.shape[:-1]):
        raise ValueError(f'targets of shape {tuple(y.shape)} for logits of shape {tuple(logits.shape)}')
    return F.wavernn_loss_rows(logits.reshape(-1, n), y.reshape(-1).to(logits.device), mode)


class ResBlock(nn.Module):
    def __init__(self, dims):
        super().__init__()
        self.conv1 = nn.Conv1d(dims, dims, kernel_size=1, bias=False)
        self.conv2 = nn.Conv1d(dims, dims, kernel_size=1, bias=False)
        self.batch_norm1 = nn.BatchNorm1d(dims)
        self.batch_norm2 = nn.BatchNorm1d(dims)


class MelResNet(nn.Module):
    def __init__(self, res_blocks, in_dims, compute_dims, res_out_dims, pad):
        super().__init__()
        self.conv_in = nn.Conv1d(in_dims, compute_dims, kernel_size=2 * pad + 1, bias=False)
        self.batch_norm = nn.BatchNorm1d(compute_dims)
        self.layers = nn.ModuleList([ResBlock(compute_dims) for _ in range(res_blocks)])
        self.conv_out = nn.Conv1d(compute_dims, res_out_dims, kernel_size=1)


class Stretch2d(nn.Module):
    def __init__(self, x_scale, y_scale):
        super().__init__()
        self.x_scale, self.y_scale = x_scale, y_scale


class UpsampleNetwork(nn.Module):
    def __init__(self, feat_dims, upsample_scales, compute_dims, res_blocks, res_out_dims, pad):
        super().__init__()
        total_scale = int(np.prod(upsample_scales))
        self.indent = pad * total_scale
        self.resnet = MelResNet(res_blocks, feat_dims, compute_dims, res_out_dims, pad)
        self.resnet_stretch = Stretch2d(total_scale, 1)
        self.up_layers = nn.ModuleList()
        for scale in upsample_scales:
            k = scale * 2 + 1
            conv = nn.Conv2d(1, 1, kernel_size=(1, k), padding=(0, scale), bias=False)
            conv.weight.data.fill_(1.0 / k)
            self.up_layers.append(Stretch2d(scale, 1))
            self.up_layers.append(conv)


def fold_count(total_len, target, overlap):
    """Folds of fold_with_overlap for a sequence of total_len samples."""
    n = (total_len - overlap) // (target + overlap)
    if total_len - (n * (overlap + target) + overlap) != 0:
        n += 1
    return n


class WaveRNN(nn.Module):
    def __init__(self, rnn_dims, fc_dims, bits, pad, upsample_factors, feat_dims, compute_dims, res_out_dims, res_blocks, hop_length,
                 sample_rate, mode='RAW'):
        super().__init__()
        if mode not in _lib.WAVERNN_MODES:
            raise ValueError(f'unknown mode {mode!r}; expected RAW or MOL')
        if int(np.prod(upsample_factors)) != hop_length:
            raise ValueError(f'hop_length {hop_length} must equal the product of upsample_factors {tuple(upsample_factors)}')
        if res_out_dims % 4:
            raise ValueError(f'res_out_dims {res_out_dims} must be divisible by 4')
        self.mode = mode
        self.pad = pad
        self.n_classes = 2 ** bits if mode == 'RAW' else 30
        self.rnn_dims, self.fc_dims, self.feat_dims = rnn_dims, fc_dims, feat_dims
        self.aux_dims = res_out_dims // 4
        self.hop_length, self.sample_rate = hop_length, sample_rate
        self.upsample_factors = tuple(int(s) for s in upsample_factors)
        self.upsample = UpsampleNetwork(feat_dims, upsample_factors, compute_dims, res_blocks, res_out_dims, pad)
        self.I = nn.Linear(feat_dims + self.aux_dims + 1, rnn_dims)
        self.rnn1 = nn.GRU(rnn_dims, rnn_dims, batch_first=True)
        self.rnn2 = nn.GRU(rnn_dims + self.aux_dims, rnn_dims, batch_first=True)
        self.fc1 = nn.Linear(rnn_dims + self.aux_dims, fc_dims)
        self.fc2 = nn.Linear(fc_dims + self.aux_dims, fc_dims)
        self.fc3 = nn.Linear(fc_dims, self.n_classes)
        self.register_buffer('step', torch.zeros(1, dtype=torch.long))
        # the loop's shape limits, checked here rather than at the first call
        shape = _lib.WaveRNNShape(1, rnn_dims, fc_dims, self.n_classes, _lib.WAVERNN_MODES[mode], 1)
        if _lib.load().b200tts_wavernn_workspace_bytes(shape) == 0:
            raise ValueError(_lib.load().b200tts_last_error().decode())

    # ---- shapes ----
    def uniforms_per_step(self):
        return 1 if self.mode == 'RAW' else self.n_classes // 3 + 1

    def tape_shape(self, frames, target=11000, overlap=550):
        """Shape of one mel's uniform tape: (folds, target + 2 overlap, uniforms per step)."""
        return fold_count(frames * self.hop_length, target, overlap), target + 2 * overlap, self.uniforms_per_step()

    # ---- training ----
    def forward(self, x, mels, trace=None):
        """fatchord's teacher-forced WaveRNN.forward: x [B, T] (the previous samples as floats), mels [B, feat_dims, T / hop + 2 pad] ->
        logits [B, T, n_classes], with autograd; increments the `step` buffer.  T a multiple of the hop, at most 16 hops; B at most 64.
        Batch norm uses batch statistics (and updates the running ones) in training mode, the running statistics in eval mode.  The GRUs run
        in fp32; the rest follows the library's precision mode.  A grid-barrier timeout of a GRU loop raises B200TTSError after the backward's
        last loop, after the forward when no backward can follow, or at the next call when a backward could follow but did not run.
        trace (a dict or None, tests): receives 'rnn1' / 'rnn2' loop traces and the last hidden layer 'y2'."""
        dev = self.I.weight.device
        x, mels = x.to(dev, torch.float32), mels.to(dev, torch.float32)
        B, T = x.shape
        hop, p = self.hop_length, self.pad
        if T < hop or T % hop or T // hop > MAX_TRAIN_HOPS or not 1 <= B <= MAX_TRAIN_BATCH:
            raise ValueError(f'x of shape {tuple(x.shape)}: need 1 to {MAX_TRAIN_BATCH} windows of a multiple of the hop {hop}, at most '
                             f'{MAX_TRAIN_HOPS} hops')
        if tuple(mels.shape) != (B, self.feat_dims, T // hop + 2 * p):
            raise ValueError(f'mels of shape {tuple(mels.shape)}; expected {(B, self.feat_dims, T // hop + 2 * p)}')
        # under CUDA-graph capture no flag is read (a read synchronises): the loops' guard goes to `_graph_guard`, whose flag the captured
        # step (graph.GraphedVocoderStep) reads after each replay
        capturing = dev.type == 'cuda' and torch.cuda.is_current_stream_capturing()
        pending = getattr(self, '_pending_guard', None)
        if pending is not None and not pending.checked and not capturing:
            pending.check()          # the previous call's loops were never followed by a backward: read their abort flag now
        self._pending_guard = None
        self.step += 1
        mel_up, aux = self.upsample_train(mels)
        A = self.aux_dims
        a1, a2, a3, a4 = (aux[:, :, A * i:A * (i + 1)] for i in range(4))
        tr = (lambda k: trace.setdefault(k, {})) if trace is not None else (lambda k: None)
        x1 = F.linear(torch.cat([x.unsqueeze(-1), mel_up, a1], dim=2), self.I.weight, self.I.bias)
        r1, r2 = self.rnn1, self.rnn2
        # both GRUs share one loop workspace, whose abort flag is read once per call: after GRU1's reverse loop (the last loop of the
        # backward), or after GRU2's forward loop when no backward follows
        guard = F.GRUSeqGuard(F.gru_seq_shape(B, T, self.rnn_dims), dev)
        grads = torch.is_grad_enabled() and any(p.requires_grad for p in self.parameters())
        x2 = x1 + F.gru_seq(x1, r1.weight_ih_l0, r1.weight_hh_l0, r1.bias_ih_l0, r1.bias_hh_l0, tr('rnn1'), guard, False,
                            grads and not capturing)
        x3 = x2 + F.gru_seq(torch.cat([x2, a2], dim=2), r2.weight_ih_l0, r2.weight_hh_l0, r2.bias_ih_l0, r2.bias_hh_l0, tr('rnn2'), guard,
                            not grads and not capturing, False)
        if capturing:
            self._graph_guard = guard
        elif grads:
            self._pending_guard = guard
        y1 = torch.relu(F.linear(torch.cat([x3, a3], dim=2), self.fc1.weight, self.fc1.bias))
        y2 = torch.relu(F.linear(torch.cat([y1, a4], dim=2), self.fc2.weight, self.fc2.bias))
        if trace is not None:
            trace['y2'] = y2
        return F.linear(y2, self.fc3.weight, self.fc3.bias)

    def upsample_train(self, mels):
        """UpsampleNetwork.forward with autograd: mels [B, feat, W] -> (mel path [B, (W - 2 pad) hop, feat], aux [B, (W - 2 pad) hop, res_out])."""
        B, _, W = mels.shape
        p, hop, tr = self.pad, self.hop_length, self.training
        rn = self.upsample.resnet
        k = rn.conv_in.kernel_size[0]

        def bn_stage(h, bn, activation, conv=None):
            if tr:
                bn.num_batches_tracked += 1
            if conv is None:
                return F.conv_block(h, None, bn.weight, bn.bias, bn.running_mean, bn.running_var, None, 1, 1, 1, activation, False, tr, bn.eps,
                                    bn.momentum, 0.0, bn.weight.shape[0], stage=2)
            return F.conv_block(h, conv.weight, bn.weight, bn.bias, bn.running_mean, bn.running_var, None, 1, conv.kernel_size[0], 1, activation,
                                False, tr, bn.eps, bn.momentum, 0.0, bn.weight.shape[0])
        # conv_in is unpadded: the middle W - 2 pad outputs of the 'same'-padded convolution
        h = F.conv_block(mels, rn.conv_in.weight, None, None, None, None, None, 1, k, 1, 'identity', False, tr, 0.0, 0.0, 0.0, 0, stage=1)
        h = bn_stage(h[:, :, p:W - p].contiguous(), rn.batch_norm, 'relu')
        for layer in rn.layers:
            y = bn_stage(h, layer.batch_norm1, 'relu', layer.conv1)
            h = h + bn_stage(y, layer.batch_norm2, 'identity', layer.conv2)
        co = rn.conv_out
        aux = F.linear(h.transpose(1, 2), co.weight.view(co.out_channels, co.in_channels), co.bias)
        aux = F.wavernn_stretch(aux, hop)
        m = mels.reshape(B * self.feat_dims, W)
        for j, scale in enumerate(self.upsample_factors):
            m = F.wavernn_upsample_layer_train(m, self.upsample.up_layers[2 * j + 1].weight, scale)
        m = m[:, p * hop:(W - p) * hop].reshape(B, self.feat_dims, -1).transpose(1, 2)
        return m, aux

    # ---- public API ----
    def generate(self, mel, target=11000, overlap=550, uniforms=None, generator=None, preemphasis=0.0):
        """One mel [feat_dims, F]: generate_batch([mel])[0]."""
        return self.generate_batch([mel], target, overlap, None if uniforms is None else [uniforms], generator, preemphasis)[0]

    def generate_batch(self, mels, target=11000, overlap=550, uniforms=None, generator=None, preemphasis=0.0):
        """Mels [feat_dims, F_i] (F_i >= 21, as given: no normalisation is applied) -> one waveform of (F_i - 1) hop samples per mel, in input
        order.  `uniforms`: one tape per mel of tape_shape(F_i, target, overlap), values in [0, 1); by default drawn with torch.rand on the
        device (`generator` optional).  preemphasis (default 0 = off): each fold is de-emphasised, lfilter([1], [1, -preemphasis]), after
        the mu-law decode and before the cross-fade; nothing is normalised.  Every stage runs in fp32 (the library's precision mode is set to
        fp32 for the call and restored after it), except the loop's recurrent products (bf16 operands, fp32 accumulation).  The same device and
        numpy / torch rules as utils.audio.spectrogram_batch."""
        specs, as_numpy = self._check_mels(mels)
        frames = [int(s.shape[1]) for s in specs]
        tapes = self._check_uniforms(uniforms, frames, target, overlap)
        preemphasis = check_preemphasis(preemphasis)
        device = _work_device(specs)
        with _fp32_context(device):
            wave, wave_off = self._generate(specs, frames, tapes, target, overlap, generator, device, preemphasis=preemphasis)
        return [_return_like(wave[int(wave_off[i]): int(wave_off[i]) + (f - 1) * self.hop_length], as_numpy[i], specs[i])
                for i, f in enumerate(frames)]

    # ---- streaming ----
    min_stream_frames = 21          # the 20-hop fade-out
    short_stream = 'the mel stream ended after {} frames; the 20-hop fade-out needs at least 21'

    def generate_stream(self, mel_chunks, uniforms=None, generator=None, preemphasis=0.0, target=None, overlap=None):
        """Streaming form of generate(mel, target=F hop, overlap=0), fatchord's unbatched generation: mel_chunks is an iterable of
        [feat_dims, n_k] mels (n_k >= 0, as given: no normalisation), whose concatenation is the mel of F >= 21 frames; yields waveform
        chunks whose concatenation is that call's (F - 1) hop samples, bit for bit given the same uniform tape.  A sample's loop features are
        final once lookahead() frames follow its frame, so the loop runs up to there after each input chunk; the last 20 hops it has run are
        held back until the input ends, because the fade-out lands on them.  uniforms: the tape [1, T, U] of generate (step t reads
        uniforms[0, t]; T >= (F - 1) hop), by default drawn with torch.rand per call of the loop (`generator` optional).  preemphasis as in
        generate_batch, de-emphasised sequentially across chunks: within fp32 roundings of the one-shot call, not bit for bit.  Runs through
        a one-stream StreamPool on the device of the first CUDA chunk, or the current CUDA device, in fp32 (the precision mode is set for
        each stretch of work and restored before every yield).  Chunks come out as the first chunk went in: numpy, CUDA tensors, or CPU
        tensors.

        With target and overlap: the streaming form of generate(mel, target, overlap), fatchord's folded generation, through a one-stream
        FoldedStreamPool (its folds run as rows of one loop): the chunks concatenate to that call's samples bit for bit given the same tape
        uniforms [folds, target + 2 overlap, U] (fold k step j reads uniforms[k, j]); preemphasis de-emphasises each fold from a zero state,
        within generate_batch's bound."""
        if target is None and overlap is None:
            self._check_stream_tape(uniforms)          # before the pool's device work
        yield from _generate_stream(self, mel_chunks, uniforms, generator, preemphasis, target, overlap, 0)

    def stream_pool(self, max_streams, preemphasis=0.0, generator=None, target=None, overlap=None):
        """A StreamPool of up to max_streams (1 to 64) concurrent generate_stream-like streams sharing one sample loop; with target and
        overlap, a FoldedStreamPool of up to max_streams folded streams on the loop's 64 rows."""
        if target is None and overlap is None:
            return StreamPool(self, max_streams, preemphasis, generator)
        return FoldedStreamPool(self, max_streams, target, overlap, preemphasis, generator)

    def lookahead(self):
        """Frames past a sample's own frame that its loop features read: `pad` for conv_in (the rest of the MelResNet is pointwise) or the
        reach of the mel path's stretch + FIR layers, whichever is larger."""
        return max(self.pad, self._mel_path_reads(0, self.hop_length)[-1][1] - self.pad)

    def _mel_path_reads(self, s0, s1):
        """Inclusive index ranges that the features of sample positions [s0, s1) read, layer by layer from the last mel-path layer's input
        down to the padded mel's frames: a stretch + FIR layer of scale s reads its input at (i + k) // s for |k| <= s."""
        lo, hi = s0 + self.pad * self.hop_length, s1 - 1 + self.pad * self.hop_length
        out = []
        for scale in reversed(self.upsample_factors):
            lo, hi = lo // scale - 1, hi // scale + 1
            out.append((lo, hi))
        return out

    def window_plan(self, s0, s1, known, final):
        """The windows the features of sample positions [s0, s1) are computed from, with `known` mel frames arrived (`final`: the whole
        mel): the padded-mel frames [P0, P1) the mel path runs over, the mel frames [r0, r1) the MelResNet runs over, and the aux frames
        [a0, a1) the features read.  Outside the mel's ends both run on the zero padding the whole-mel computation sees; elsewhere each
        window reaches as far as the reads do, so the values read equal the whole mel's."""
        p, hop = self.pad, self.hop_length
        P0, P1 = self._mel_path_reads(s0, s1)[-1]
        P0, P1 = max(P0, 0), P1 + 1
        a0, a1 = s0 // hop, (s1 - 1) // hop + 1
        r0, r1 = max(a0 - p, 0), a1 + p
        if final:
            P1, r1 = min(P1, known + 2 * p), min(r1, known)
        elif P1 - p > known or r1 > known:
            raise ValueError(f'positions [{s0}, {s1}) read mel frames past the {known} that have arrived')
        return (P0, P1), (r0, r1), (a0, a1)

    def _check_chunk(self, chunk, i):
        as_numpy = not isinstance(chunk, torch.Tensor)
        t = torch.as_tensor(np.asarray(chunk) if as_numpy else chunk)
        if t.dim() != 2 or t.shape[0] != self.feat_dims:
            raise ValueError(f'mel chunk {i} has shape {tuple(t.shape)}; expected [{self.feat_dims}, frames]')
        if not torch.is_floating_point(t):
            raise ValueError(f'mel chunk {i} is not floating point')
        if not bool(torch.isfinite(t).all()):
            raise ValueError(f'mel chunk {i} has non-finite values')
        return t, as_numpy

    def _check_stream_tape(self, uniforms, fold_len=None):
        """A stream's uniform tape as a tensor, or None: [1, steps, U], or with fold_len (a folded stream) [folds, fold_len, U]."""
        if uniforms is None:
            return None
        u = torch.as_tensor(np.asarray(uniforms) if not isinstance(uniforms, torch.Tensor) else uniforms)
        U = self.uniforms_per_step()
        if fold_len is not None:
            if u.dim() != 3 or u.shape[0] < 1 or u.shape[1] != fold_len or u.shape[2] != U:
                raise ValueError(f'uniform tape of shape {tuple(u.shape)}; expected [folds, {fold_len}, {U}] (target + 2 overlap = {fold_len})')
        elif u.dim() != 3 or u.shape[0] != 1 or u.shape[2] != U:
            raise ValueError(f'uniform tape of shape {tuple(u.shape)}; expected [1, steps, {U}]')
        if not torch.is_floating_point(u):
            raise ValueError('uniform tape is not floating point')
        if u.numel() and (bool((u < 0).any()) or bool((u >= 1).any()) or bool(torch.isnan(u).any())):
            raise ValueError('uniform tape has values outside [0, 1)')
        return u

    # ---- checks ----
    def _check_mels(self, mels):
        if not isinstance(mels, (list, tuple)) or len(mels) == 0:
            raise ValueError('generate_batch expects a non-empty list of [feat_dims, frames] mels')
        as_numpy = [not isinstance(m, torch.Tensor) for m in mels]
        specs = []
        for i, m in enumerate(mels):
            t = torch.as_tensor(np.asarray(m) if as_numpy[i] else m)
            if t.dim() != 2 or t.shape[0] != self.feat_dims:
                raise ValueError(f'mel {i} has shape {tuple(t.shape)}; expected [{self.feat_dims}, frames]')
            if t.shape[1] < 21:
                raise ValueError(f'mel {i} has {t.shape[1]} frames; the 20-hop fade-out needs at least 21')
            if not torch.is_floating_point(t):
                raise ValueError(f'mel {i} is not floating point')
            if not bool(torch.isfinite(t).all()):
                raise ValueError(f'mel {i} has non-finite values')
            specs.append(t)
        return specs, as_numpy

    def _check_uniforms(self, uniforms, frames, target, overlap):
        if target < 1 or overlap < 0:
            raise ValueError(f'target {target} must be positive and overlap {overlap} non-negative')
        if uniforms is None:
            return None
        if len(uniforms) != len(frames):
            raise ValueError(f'{len(uniforms)} uniform tapes for {len(frames)} mels')
        tapes = []
        for i, u in enumerate(uniforms):
            u = torch.as_tensor(np.asarray(u) if not isinstance(u, torch.Tensor) else u)
            want = self.tape_shape(frames[i], target, overlap)
            if tuple(u.shape) != want:
                raise ValueError(f'uniform tape {i} has shape {tuple(u.shape)}; expected {want}')
            if not torch.is_floating_point(u):
                raise ValueError(f'uniform tape {i} is not floating point')
            if u.numel() and (bool((u < 0).any()) or bool((u >= 1).any()) or bool(torch.isnan(u).any())):
                raise ValueError(f'uniform tape {i} has values outside [0, 1)')
            tapes.append(u)
        return tapes

    # ---- stages ----
    def fold_plan(self, frames, target, overlap):
        """(row_utt, row_fold, row_off) host int32 arrays of the fold rows of utterances with these frame counts."""
        n = [fold_count(f * self.hop_length, target, overlap) for f in frames]
        row_utt = np.repeat(np.arange(len(frames)), n).astype(np.int32)
        row_fold = np.concatenate([np.arange(k) for k in n]).astype(np.int32)
        row_off = np.concatenate([[0], np.cumsum(n)]).astype(np.int32)
        return row_utt, row_fold, row_off

    def upsample_batch(self, specs, device):
        """(mel_up, mel_off, aux): the mel path up to its penultimate layer, packed per utterance as [feat_dims, (F + 2 pad) hop / s_last]
        at element offset mel_off[b], and the MelResNet output aux [B, max F, res_out_dims]."""
        frames = [int(s.shape[1]) for s in specs]
        B, Fm, p = len(specs), max(frames), self.pad
        x = torch.zeros(B, self.feat_dims, Fm, device=device, dtype=torch.float32)
        for i, s in enumerate(specs):
            x[i, :, :frames[i]] = s.to(device=device, dtype=torch.float32)
        aux = self._resnet(x, frames, device)
        ups = []
        for i, s in enumerate(specs):
            m = torch.zeros(self.feat_dims, frames[i] + 2 * p, device=device, dtype=torch.float32)
            m[:, p:p + frames[i]] = s.to(device=device, dtype=torch.float32)
            ups.append(self._mel_path(m, device).reshape(-1))
        mel_off = np.concatenate([[0], np.cumsum([u.numel() for u in ups])[:-1]]).astype(np.int64)
        return torch.cat(ups), mel_off, aux

    def _resnet(self, x, frames, device):
        """The MelResNet of a zero-padded batch x [B, feat_dims, W] whose mel b has frames[b] frames -> aux [B, W, res_out_dims]."""
        rn = self.upsample.resnet
        d = lambda t: t.detach().to(device=device, dtype=torch.float32).contiguous()
        lengths = torch.tensor(frames, device=device, dtype=torch.int32)

        def block(inp, conv, bn, activation):
            return F.conv_block_masked(inp, lengths, d(conv.weight), d(bn.weight), d(bn.bias), d(bn.running_mean), d(bn.running_var), 1,
                                       conv.kernel_size[0], 1, activation, False, bn.eps, bn.weight.shape[0])
        # conv_in has no padding but reads the mel padded by `pad` zero frames: the same as a zero-padded convolution of the mel itself
        h = block(x, rn.conv_in, rn.batch_norm, 'relu')
        for layer in rn.layers:
            y = block(h, layer.conv1, layer.batch_norm1, 'relu')
            h = h + block(y, layer.conv2, layer.batch_norm2, 'identity')
        w_out, b_out = d(rn.conv_out.weight.reshape(rn.conv_out.out_channels, -1)), d(rn.conv_out.bias)
        return F.gemm_tn_batched(h, w_out, b_out)

    def _mel_path(self, m, device):
        """Every mel-path layer but the last over frames of the padded mel m [feat_dims, W] (zero beyond them) -> [feat_dims, W hop / s_last]."""
        for j, scale in enumerate(self.upsample_factors[:-1]):
            fir = self.upsample.up_layers[2 * j + 1].weight.detach().reshape(-1).to(device=device, dtype=torch.float32).contiguous()
            m = F.wavernn_upsample_layer(m, fir, scale)
        return m

    def loop_weights(self, device):
        """fp32 contiguous tensors on `device` of the loop parameters (_lib.WAVERNN_PARAM_FIELDS) and of the conditioning products."""
        R, Fc, A = self.rnn_dims, self.fc_dims, self.aux_dims
        f = lambda t: t.detach().to(device=device, dtype=torch.float32).contiguous()
        w = {
            'w_hh1': f(self.rnn1.weight_hh_l0), 'b_hh1': f(self.rnn1.bias_hh_l0),
            'w_prev': f(self.I.weight[:, 0]),
            'w_ih2x': f(self.rnn2.weight_ih_l0[:, :R]), 'w_hh2': f(self.rnn2.weight_hh_l0), 'b_hh2': f(self.rnn2.bias_hh_l0),
            'w_fc1x': f(self.fc1.weight[:, :R]), 'w_fc2x': f(self.fc2.weight[:, :Fc]), 'w_fc3': f(self.fc3.weight), 'b_fc3': f(self.fc3.bias),
            # conditioning
            'w_I': f(self.I.weight[:, 1:]), 'b_I': f(self.I.bias), 'w_ih1': f(self.rnn1.weight_ih_l0), 'b_ih1': f(self.rnn1.bias_ih_l0),
            'w_ih2a': f(self.rnn2.weight_ih_l0[:, R:]), 'b_ih2': f(self.rnn2.bias_ih_l0),
            'w_fc1a': f(self.fc1.weight[:, R:]), 'b_fc1': f(self.fc1.bias), 'w_fc2a': f(self.fc2.weight[:, Fc:]), 'b_fc2': f(self.fc2.bias),
        }
        assert w['w_fc1x'].shape[1] == R and w['w_fc2a'].shape[1] == A
        w['u1'] = F.gemm(w['w_ih1'], w['w_prev'].reshape(-1, 1)).reshape(-1).contiguous()
        return w

    def conditioning(self, w, feat):
        """The loop's inputs that do not depend on the previous sample, from feat [S, rows, n_mels + aux_dims]: (c, g1, c2, p1, p2)."""
        S, rows, D = feat.shape
        nm, A = self.feat_dims, self.aux_dims
        X = feat.reshape(S * rows, D)
        c = F.gemm(X[:, :nm + A], w['w_I'], trans_b=True, bias=w['b_I'])
        g1 = F.gemm(c, w['w_ih1'], trans_b=True, bias=w['b_ih1'])
        c2 = F.gemm(X[:, nm + A:nm + 2 * A], w['w_ih2a'], trans_b=True, bias=w['b_ih2'])
        p1 = F.gemm(X[:, nm + 2 * A:nm + 3 * A], w['w_fc1a'], trans_b=True, bias=w['b_fc1'])
        p2 = F.gemm(X[:, nm + 3 * A:nm + 4 * A], w['w_fc2a'], trans_b=True, bias=w['b_fc2'])
        return tuple(t.reshape(S, rows, -1) for t in (c, g1, c2, p1, p2))

    def chunk_steps(self, rows, fold_len):
        # floats per step and row: the features, c, g1, c2, p1 and p2
        per_step = rows * 4 * (self.feat_dims + 4 * self.aux_dims + 7 * self.rnn_dims + 2 * self.fc_dims)
        return int(max(1, min(fold_len, COND_BYTES // per_step)))

    def _generate(self, specs, frames, tapes, target, overlap, generator, device, trace=None, preemphasis=0.0):
        """(packed waveform, host offsets).  trace (a dict, tests): receives the stage inputs and outputs; trace['dbg'], if given, is the
        loop's debug buffer [fold_len, rows, 4 R + 2 fc + n_out]."""
        row_utt, row_fold, row_off = self.fold_plan(frames, target, overlap)
        rows, L, hop = int(row_off[-1]), target + 2 * overlap, self.hop_length
        mel_up, mel_off, aux = self.upsample_batch(specs, device)
        dev = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(device)
        frames_d, row_utt_d, row_fold_d, row_off_d, mel_off_d = dev(np.asarray(frames, np.int32)), dev(row_utt), dev(row_fold), dev(row_off), \
            dev(mel_off)
        fshape = _lib.WaveRNNFoldShape(len(frames), rows, self.feat_dims, 4 * self.aux_dims, hop, self.pad, self.upsample_factors[-1], target,
                                       overlap, max(frames))
        U = self.uniforms_per_step()
        if tapes is None:
            uni = torch.rand(rows, L, U, device=device, dtype=torch.float32, generator=generator)
        else:
            uni = torch.cat([t.to(device=device, dtype=torch.float32) for t in tapes]).contiguous()
        loop = _SampleLoop(self, rows, L, device)
        y = torch.empty(rows, L, device=device, dtype=torch.float32)
        S = self.chunk_steps(rows, L)
        for t0 in range(0, L, S):
            n = min(S, L - t0)
            feat = F.wavernn_fold(fshape, mel_up, mel_off_d, frames_d, row_utt_d, row_fold_d, loop.firs[-1], aux, t0, n)
            cond = self.conditioning(loop.w, feat)
            dbg = None if trace is None or trace.get('dbg') is None else trace['dbg'][t0:t0 + n]
            F.wavernn_run(loop.shape, loop.params, cond, t0, n, uni, y, loop.ws, dbg)
            if trace is not None and t0 == 0:
                trace.update(feat=feat, cond=cond, chunk=n)
        _check_loop(loop.shape, loop.ws)
        wave, wave_off = self.postprocess(y, frames, target, overlap, preemphasis)
        if trace is not None:
            trace.update(folded=y, uniforms=uni, weights=loop.w, row_off=row_off, wave_off=wave_off, mel_up=mel_up, mel_off=mel_off, aux=aux)
        return wave, wave_off

    def postprocess(self, y, frames, target, overlap, preemphasis=0.0):
        """The loop's folded samples y [rows, target + 2 overlap] (CUDA) -> (packed waveform, host offsets): mu-law decode (RAW), optional
        de-emphasis of each fold, cross-fade and overlap-add, cut to (F - 1) hop samples, 20-hop fade-out.  y is not modified."""
        hop, device = self.hop_length, y.device
        _, _, row_off = self.fold_plan(frames, target, overlap)
        dev = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(device)
        wave_off = np.concatenate([[0], np.cumsum([(f - 1) * hop for f in frames])]).astype(np.int64)
        mu = self.n_classes - 1 if self.mode == 'RAW' else 0
        if preemphasis:
            y = F.wavernn_deemphasis(y.clone(), mu, preemphasis)          # decodes the mu-law first
            mu = 0
        wave = F.wavernn_unfold(y, dev(np.asarray(frames, np.int32)), dev(row_off), dev(wave_off), int(wave_off[-1]), hop, target, overlap, mu)
        return wave, wave_off


@contextlib.contextmanager
def _fp32_context(device):
    """The sample loop's context: fp32 precision mode (restored after), `device` current, no autograd."""
    precision = _lib.get_precision()
    try:
        _lib.set_precision('fp32')
        with torch.cuda.device(device), torch.no_grad():
            yield
    finally:
        _lib.set_precision(precision)


def _check_loop(shape, ws):
    """Reads a sample loop's abort flag (a synchronising read)."""
    if F.wavernn_aborted(shape, ws):
        raise _lib.B200TTSError('wavernn: the sample loop timed out at a grid barrier')


def _upload(a, device):
    return torch.from_numpy(np.ascontiguousarray(a)).to(device)


# One row of a loop call: its loop row `slot`, the mel of its stream (`ended`: the whole mel), the n sample positions [t, t + n) it runs,
# the steps it has run (the loop's per-row parity), and its uniforms: uni [n, U] from a tape, else draws from `seed` at draw0, else None
# (drawn for the call)
_Row = collections.namedtuple('_Row', 'slot mel ended t n steps uni seed draw0')


class _SampleLoop:
    """WaveRNN's sample loop on `device`: the loop weights, shape, workspace and parameters of `rows` rows of up to `steps` steps per call,
    the mel-path FIRs, and, with preemphasis, each row's last de-emphasised sample.  generate_batch runs it over its fold rows with
    b200tts_wavernn_run, then _check_loop; the stream pools through step_rows, which computes each row's windowed features itself."""

    def __init__(self, model, rows, steps, device, preemphasis=0.0, generator=None):
        self.m, self.device, self.a, self.generator = model, device, preemphasis, generator
        self.mu = model.n_classes - 1 if model.mode == 'RAW' else 0
        self.out_mu = 0 if preemphasis else self.mu          # the mu-law step_rows' samples still carry: the de-emphasis decodes it
        self.w = model.loop_weights(device)
        self.shape = _lib.WaveRNNShape(rows, model.rnn_dims, model.fc_dims, model.n_classes, _lib.WAVERNN_MODES[model.mode], steps)
        self.ws = F.wavernn_workspace(self.shape, device)
        self.params = F.wavernn_params(self.w)
        F.wavernn_prepare(self.shape, self.params, self.ws)
        self.firs = [c.weight.detach().reshape(-1).to(device, torch.float32).contiguous() for c in model.upsample.up_layers[1::2]]
        self.last = torch.zeros(rows, device=device, dtype=torch.float32) if preemphasis else None

    def reset(self, slots):
        """Resets loop rows `slots` for new rows."""
        F.wavernn_reset_rows(self.shape, self.ws, slots)
        if self.a:
            self.last[_upload(np.array(slots, np.int64), self.device)] = 0.0

    def step_rows(self, rows):
        """One loop call over `rows` (_Row, sorted by slot) -> (y [active, nmax], de-emphasised with preemphasis, active, nmax)."""
        m, dev, U = self.m, self.device, self.m.uniforms_per_step()
        active = rows[-1].slot + 1
        nmax = max(r.n for r in rows)
        feat = self.features(rows, active, nmax)
        cond = m.conditioning(self.w, feat)
        slot = np.array([r.slot for r in rows], np.int64)
        n = np.array([r.n for r in rows], np.int64)
        # uniforms: the taped rows' steps gathered from their tapes (source 0 is a zero) and the seeded rows' from one seeded draw, in one
        # gather; the other rows' drawn for the call
        taped = [r for r in rows if r.uni is not None]
        seeded = [r for r in rows if r.uni is None and r.seed is not None]
        if taped or seeded:
            parts = [torch.zeros(1, device=dev)] + [r.uni.reshape(-1) for r in taped]
            if seeded:
                parts.append(F.fill_uniform_rows(nmax, U, [r.seed for r in seeded], [r.draw0 for r in seeded], _lib.SEED_STREAMS['vocoder'],
                                                 dev).reshape(-1))
            src = torch.cat(parts)
            idx = np.zeros((active, nmax, U), np.int64)
            off = 1
            i = np.arange(nmax)[:, None] * U + np.arange(U)[None, :]
            for r in taped:
                idx[r.slot, :r.n] = off + i[:r.n]
                off += r.n * U
            for r in seeded:
                idx[r.slot, :r.n] = off + i[:r.n]
                off += nmax * U
            uni = src[_upload(idx, dev)]
        if len(taped) + len(seeded) < len(rows):
            drawn = torch.rand(active, nmax, U, device=dev, dtype=torch.float32, generator=self.generator)
            if taped or seeded:
                has = np.zeros((active, 1, 1), bool)
                has[[r.slot for r in taped + seeded]] = True
                uni = torch.where(_upload(has, dev), uni, drawn)
            else:
                uni = drawn
        y = torch.zeros(active, nmax, device=dev, dtype=torch.float32)
        if self.shape.rows == 1:
            # a one-row loop: the loop without per-row budgets runs row 0 bit for bit as run_rows does (it runs every row of the shape,
            # so it serves only a loop of one row)
            F.wavernn_run_stream(self.shape, self.params, cond, rows[0].steps, nmax, uni, y, self.ws)
        else:
            row_t, row_n = np.zeros(active, np.int64), np.zeros(active, np.int32)
            row_t[slot], row_n[slot] = [r.steps for r in rows], n
            F.wavernn_run_rows(self.shape, self.params, cond, _upload(row_t, dev), _upload(row_n, dev), nmax, uni, y, self.ws)
        if self.a:
            if self.mu:
                y = F.wavernn_deemphasis(y, self.mu, 0.0)                    # a = 0: the mu-law decode only
            y = F.wavernn_deemphasis(torch.cat([self.last[:active, None], y], 1).contiguous(), 0, self.a)[:, 1:]
            sl = _upload(slot, dev)
            self.last[sl] = y[sl, _upload(n - 1, dev)]
        return y, active, nmax

    def window_layout(self, rows):
        """The host side of features: (sources [(row index, frame0, frame1)] packed side by side, then a zero column; the gather index of
        the packed mel-path windows followed by the padded MelResNet batch; window lengths; MelResNet widths and batch width; window-row
        descriptors without the aux width, as (slot, frames or 0, m0, mel_len, a0, aux_len, s0, mel_off, aux_off / aux width, n))."""
        m = self.m
        p, hop, s_last, C = m.pad, m.hop_length, m.upsample_factors[-1], m.feat_dims
        srcs, wins, res = [], [], []
        for b, r in enumerate(rows):
            frames = int(r.mel.shape[1])
            (P0, P1), (r0, r1), _ = m.window_plan(r.t, r.t + r.n, frames, r.ended)
            lo, hi = max(P0, p), min(P1, frames + p)
            wins.append((P0, P1, lo, hi))
            res.append((r0, r1))
            srcs.append((b, lo - p, max(hi, lo) - p))
        srcs += [(b, r0, r1) for b, (r0, r1) in enumerate(res)]
        off = np.concatenate([[0], np.cumsum([c - a for _, a, c in srcs])])
        Wt = int(off[-1]) + 1                       # the last column is zero
        c = np.arange(C)[:, None] * Wt
        parts, lens, desc, mel_off = [], [], [], 0
        for b, (P0, P1, lo, hi) in enumerate(wins):
            P = np.arange(P0, P1)
            col = np.where((P >= lo) & (P < hi), off[b] + P - lo, Wt - 1)
            parts.append((c + col[None, :]).reshape(-1))
            lens.append(P1 - P0)
        widths = [r1 - r0 for r0, r1 in res]
        W = max(widths)
        w = np.arange(W)[None, :]
        col = np.where(w < np.array(widths)[:, None], off[len(rows):-1, None] + w, Wt - 1)
        parts.append((c[None, :, :] + col[:, None, :]).reshape(-1))
        scale = int(np.prod(m.upsample_factors[:-1]))
        for b, r in enumerate(rows):
            P0, r0 = wins[b][0], res[b][0]
            desc.append((r.slot, int(r.mel.shape[1]) if r.ended else 0, P0 * (hop // s_last), lens[b] * scale, r0, widths[b], r.t, mel_off,
                         b * W, r.n))
            mel_off += C * lens[b] * scale
        return srcs, np.concatenate(parts), lens, widths, W, desc

    def features(self, rows, active, nmax):
        """Loop features [nmax, active, feat_dims + res_out_dims] of every row's positions, in a fixed number of launches: one gather of
        every window, the mel-path layers on the packed windows, the MelResNet over the padded batch of windows, one window-rows launch."""
        m, dev = self.m, self.device
        p, hop, s_last, C = m.pad, m.hop_length, m.upsample_factors[-1], m.feat_dims
        srcs, idx, lens, widths, W, desc = self.window_layout(rows)
        packed = torch.cat([rows[b].mel[:, a:c] for b, a, c in srcs] + [torch.zeros(C, 1, device=dev)], dim=1)
        g = packed.reshape(-1)[_upload(idx, dev)]
        nw = C * sum(lens)
        x, batch = g[:nw], g[nw:].view(len(rows), C, W)
        for j, scale in enumerate(m.upsample_factors[:-1]):
            x = F.wavernn_upsample_segments(x, lens, self.firs[j], scale)
            lens = [ln * scale for ln in lens]
        aux = m._resnet(batch, widths, dev)
        A = aux.shape[2]
        blank = _lib.WaveRNNWindowShape(C, A, hop, p, s_last, 0, 0, 1, 0, 0)
        win = [_lib.WaveRNNWindowRow(blank, 0, 0, 0, 0) for _ in range(active)]
        for slot, frames, m0, mel_len, a0, aux_len, s0, mel_off, aux_row, n in desc:
            shape = _lib.WaveRNNWindowShape(C, A, hop, p, s_last, frames, m0, mel_len, a0, aux_len)
            win[slot] = _lib.WaveRNNWindowRow(shape, s0, mel_off, aux_row * A, n)
        return F.wavernn_window_rows(win, nmax, x, self.firs[-1], aux)


class _MelStream(Stream):
    """One WaveRNN stream: the mel frames that have arrived (fp32 on the pool's device), its uniform tape (fp32 on the device, or None)
    and its seed (or None)."""

    def __init__(self, device, feat_dims, tape, seed):
        super().__init__()
        self.mel = torch.zeros(feat_dims, 0, device=device, dtype=torch.float32)
        self.tape, self.seed = tape, seed

    @property
    def frames(self):
        return int(self.mel.shape[1])

    def append(self, spec):
        self.mel = torch.cat([self.mel, spec.to(device=self.mel.device, dtype=torch.float32)], dim=1)


class _PoolStream(_MelStream):
    """One stream of a StreamPool: its loop row and the steps it has run.  Its run but unreleased samples [released, steps) sit in the
    pool's per-row ring buffer."""

    def __init__(self, slot, device, feat_dims, tape, seed=None):
        super().__init__(device, feat_dims, tape, seed)
        self.slot = slot
        self.steps = 0


class StreamPool(VocoderStreamPool):
    """Concurrent streaming generation: up to max_streams streams, each a generate_stream, advance together in one sample loop whose rows
    run independently (b200tts_wavernn_run_rows; a one-stream pool, whose loop has one row, runs b200tts_wavernn_run_stream, the loop
    without per-row budgets, bit for bit the same).  open() takes the lowest free row and resets it; feed() and end() add a stream's mel
    frames and mark its end; run() makes one loop call over every stream with samples ready, under generate_stream's rule (lookahead()
    frames after a sample's frame, the last 20 hops held back until end()), at most POOL_CALL_HOPS hops per call in a pool of more than one
    stream, and returns {sid: waveform chunk} (CUDA tensors) for the streams that released samples.  A stream's row is freed when its final
    chunk is returned, or at once by close().

    For each stream the concatenated chunks equal generate_stream of the same mel with the same uniform tape, bit for bit, whenever it
    joined, whatever else shares the loop and however its mel was chunked.  With preemphasis the stream is de-emphasised across calls and
    stays within generate_batch's bound.  Without a tape the uniforms are drawn with torch.rand (`generator` optional) once per call for all
    rows, so they differ from a solo run's draws; a stream opened with a seed draws its own (b200tts_fill_uniform_rows at its own step count,
    stream _lib.SEED_STREAMS['vocoder']), which depend on the seed alone: its tape is one fill_uniform_rows row over [0, T).  Every call runs
    in fp32 (the precision mode is set for the call and restored after it) on the CUDA device that was current when the pool was made; each
    run() reads the loop's abort flag once.  The device work of a run() is a fixed number of launches whatever the number of streams: the
    per-stream windows, tapes and samples are gathered and scattered with indices built on the host."""

    def __init__(self, model, max_streams, preemphasis=0.0, generator=None):
        super().__init__(model, max_streams, preemphasis)
        self.hop, self.lookahead = model.hop_length, model.lookahead()
        self.slots = [None] * self.rows          # sid of the stream on each row
        # a lone stream runs all its ready steps in one call (up to COND_BYTES): each call costs 3 to 4 ms outside the loop, and no other
        # stream waits on it
        S = model.chunk_steps(self.rows, 1 << 30)
        self.S = S if self.rows == 1 else min(POOL_CALL_HOPS * self.hop, S)
        # per-row ring of the samples run but not released: at most 20 held-back hops, the partial hop and one call's steps
        self.P = self.S + 22 * self.hop
        with self._fp32():
            self.loop = _SampleLoop(model, self.rows, self.S, self.device, self.a, generator)
            self.ring = torch.zeros(self.rows * self.P + 2, device=self.device, dtype=torch.float32)   # + a write sink and a zero
        self.shape, self.ws = self.loop.shape, self.loop.ws          # read by the abort check after each run()

    def _fp32(self):
        return _fp32_context(self.device)

    def check_tape(self, uniforms):
        """A stream's tape [1, T, U] as for generate_stream, or None."""
        return self.v._check_stream_tape(uniforms)

    def _open(self, sid, tape, seed):
        slot = self.slots.index(None)
        with self._fp32():
            self.loop.reset([slot])
            if tape is not None:
                tape = tape[0].to(device=self.device, dtype=torch.float32).contiguous()
        self.slots[slot] = sid
        return _PoolStream(slot, self.device, self.v.feat_dims, tape, seed)

    def _drop(self, st):
        self.slots[st.slot] = None

    def plan(self):
        """{sid: (steps run, steps of the next call)} for every stream with ready samples."""
        out = {}
        for sid, st in self.streams.items():
            F_ = st.frames
            end = (F_ - 1) * self.hop if st.ended else max(min(F_ - self.lookahead, F_ - 1), 0) * self.hop
            n = min(self.S, end - st.steps)
            if n > 0:
                out[sid] = (st.steps, n)
        return out

    def release_plan(self):
        """[(sid, samples, frames)] of every stream with samples to release: the final chunk once the stream has ended and run all its
        (F - 1) hop steps (frames: the utterance length left, so that the unfold places the fade-out), else the whole hops run more than 20
        hops ago (frames: 21 hops more than it writes, so that no fade lands on them)."""
        hop, rel = self.hop, []
        for sid, st in self.streams.items():
            F_ = st.frames
            if st.ended and st.steps == (F_ - 1) * hop:
                n, frames = (F_ - 1) * hop - st.released, F_ - st.released // hop
            else:
                n = (st.steps - 20 * hop) // hop * hop - st.released
                frames = n // hop + 21
            if n > 0:
                rel.append((sid, n, frames))
        return rel

    def run(self):
        """One loop call over every stream with ready samples -> {sid: the waveform chunk it releases}."""
        plan = self.plan()
        for sid, (t, n) in plan.items():
            tape = self.streams[sid].tape
            if tape is not None and tape.shape[0] < t + n:
                raise ValueError(f'the uniform tape holds {tape.shape[0]} steps; the stream needs at least {t + n}')
        with self._fp32():
            if plan:
                self._loop(plan)
            released = self._release()
            _check_loop(self.shape, self.ws)
        for sid in released:
            st = self.streams[sid]
            if st.ended and st.released == (st.frames - 1) * self.hop:
                self.close(sid)
        return released

    def _busy(self):
        return bool(self.plan())

    def _loop_rows(self, plan):
        """The loop rows of the streams in plan, by slot."""
        rows = []
        for sid in sorted(plan, key=lambda s: self.streams[s].slot):
            st, (t, n) = self.streams[sid], plan[sid]
            rows.append(_Row(st.slot, st.mel, st.ended, t, n, t, None if st.tape is None else st.tape[t:t + n], st.seed, t))
        return rows

    def _loop(self, plan):
        rows = self._loop_rows(plan)
        y, active, nmax = self.loop.step_rows(rows)
        row_t, row_n = np.zeros(active, np.int64), np.zeros(active, np.int32)
        row_t[[r.slot for r in rows]] = [r.t for r in rows]
        row_n[[r.slot for r in rows]] = [r.n for r in rows]
        # into the ring: row r's step i at slot r P + (row_t + i) mod P; steps past a row's budget go to the sink
        i = np.arange(nmax)[None, :]
        dst = np.where(i < row_n[:, None], np.arange(active)[:, None] * self.P + (row_t[:, None] + i) % self.P, self.rows * self.P)
        self.ring.index_put_((_upload(dst.reshape(-1), self.device),), y.reshape(-1))
        for sid, (_, n) in plan.items():
            self.streams[sid].steps += n

    def _release(self):
        """Every stream's releasable samples, gathered from the ring, through one b200tts_wavernn_unfold, each stream one fold of one
        utterance -> {sid: chunk}."""
        rel = self.release_plan()
        if not rel:
            return {}
        L = max(n for _, n, _ in rel)
        i = np.arange(L)[None, :]
        slot = np.array([self.streams[sid].slot for sid, _, _ in rel])[:, None]
        start = np.array([self.streams[sid].released for sid, _, _ in rel])[:, None]
        n = np.array([n for _, n, _ in rel])[:, None]
        src = np.where(i < n, slot * self.P + (start + i) % self.P, self.rows * self.P + 1)
        y = self.ring[_upload(src, self.device)]
        for sid, k, _ in rel:
            self.streams[sid].released += k
        wave_off = np.concatenate([[0], np.cumsum(n[:, 0])])
        meta = _upload(np.concatenate([[f for *_, f in rel], np.arange(len(rel) + 1), wave_off]).astype(np.int64), self.device)
        B = len(rel)
        wave = F.wavernn_unfold(y, meta[:B].int(), meta[B:2 * B + 1].int(), meta[2 * B + 1:], int(wave_off[-1]), self.hop, L, 0,
                                self.loop.out_mu)
        return {sid: wave[int(wave_off[b]):int(wave_off[b + 1])] for b, (sid, *_) in enumerate(rel)}


class _Fold:
    """Fold k of a folded stream st: sample positions [start, start + fold_len) with start = k (target + overlap), its loop row (None before
    its grant and once it has run every step it needs), its storage slot (None once its samples are all released) and the steps it has
    run."""

    def __init__(self, st, k, start):
        self.st, self.k, self.start = st, k, start
        self.slot = self.store = None
        self.steps = 0
        self.done = False


class _FoldedStream(_MelStream):
    """One stream of a FoldedStreamPool, which has no loop row of its own: `folds` lists the folds opened so far, fold k at index k."""

    def __init__(self, sid, device, feat_dims, tape, seed=None):
        super().__init__(device, feat_dims, tape, seed)
        self.sid = sid
        self.folds = []


class FoldedStreamPool(VocoderStreamPool):
    """Folded streaming generation: up to max_streams streams, each the streaming form of generate(mel, target, overlap) (fatchord's
    folded generation, the library's default), whose folds run as rows of one 64-row sample loop (b200tts_wavernn_run_rows).  The
    interface is StreamPool's: open / feed / end / run / drain / close / streams.

    Fold geometry is fold_count's: with L = target + 2 overlap, fold k covers positions [k (target + overlap), k (target + overlap) + L) and
    exists iff k (target + overlap) + overlap < F hop.  While the mel arrives, fold k opens only once its existence is certain (it exists
    for the frames that have arrived).  It runs up to generate_stream's readiness rule (lookahead() frames after a sample's frame), and
    once F is known up to min(L, (F - 1) hop - k (target + overlap)) steps: samples at or past the cut are never needed.  Fold k step j
    reads tape[k, j] (tape [K, L, U], K at least the folds the stream ends up running), or, seeded, draw (k L + j) U + u of the vocoder
    stream (b200tts_fill_uniform_rows at t0 = k L + j): its tape is one seeded row of K L steps reshaped to [K, L, U].  De-emphasis runs
    per fold from a zero state, as postprocess does per fold row.

    Rows: each run() grants free loop rows to the waiting folds in order of k (target + overlap) minus the samples their stream has
    released (ties by stream id), so the fold whose audio is needed soonest goes first; a new stream's fold 0 is not starved by old
    streams' later folds.  A fold's row is freed as soon as it has run every step it needs; its unreleased samples wait in pool-owned
    storage of L samples per fold.  The storage holds 64 folds plus, per stream, the finished folds that can wait on the release: those
    within 21 hops + L of its release point, so that a row never waits for storage.  Each run() runs at most POOL_CALL_HOPS hops, bounded
    by COND_BYTES at the rows it runs.

    Release: position q is final when every existing fold covering it has run step q - k (target + overlap); a fold whose existence is
    still undecided blocks the positions it would cover.  Before end() the final positions are released in whole hops, 20 hops behind
    (the fade-out may land there); after it, every final position.  Each run() writes every stream's chunk with one
    b200tts_wavernn_unfold_streams launch, whose arithmetic is b200tts_wavernn_unfold's: a stream's chunks concatenate to generate(mel,
    target, overlap, uniforms=tape) bit for bit, whatever joins or leaves the pool and however its mel is chunked.  With preemphasis each
    fold is de-emphasised across calls, within generate_batch's bound.  close() frees every row and all storage of a stream at once."""

    def __init__(self, model, max_streams, target, overlap, preemphasis=0.0, generator=None):
        self._layout(model, max_streams, target, overlap, _lib.WAVERNN_MAX_STREAMS)
        self.a = check_preemphasis(preemphasis)
        with self._fp32():
            self.loop = _SampleLoop(model, len(self.slots), self.S, self.device, self.a, generator)
            self.store = torch.zeros(self.nstore * self.fold_len + 1, device=self.device, dtype=torch.float32)     # + a write sink
        self.shape, self.ws = self.loop.shape, self.loop.ws          # read by the abort check after each run()

    def _fp32(self):
        return _fp32_context(self.device)

    def _layout(self, model, max_streams, target, overlap, nrows):
        """The host state of a pool with nrows loop rows: the checks but preemphasis, geometry, rows, streams and storage slots
        (ValueError past COND_BYTES)."""
        super().__init__(model, max_streams)
        if target is None or overlap is None or int(target) != target or int(overlap) != overlap or target < 1 or overlap < 0:
            raise ValueError(f'a folded stream pool needs an integer target >= 1 and overlap >= 0 (got {target!r}, {overlap!r})')
        self.target, self.overlap = int(target), int(overlap)
        self.step, self.fold_len = self.target + self.overlap, self.target + 2 * self.overlap
        self.hop, self.lookahead = model.hop_length, model.lookahead()
        self.S = POOL_CALL_HOPS * self.hop
        self.slots = [None] * nrows                          # the fold on each loop row
        self.hold = -(-(21 * self.hop + self.fold_len) // self.step) + 1      # finished folds of one stream that can wait on its release
        self.nstore = nrows + self.rows * self.hold
        if self.nstore * self.fold_len * 4 > COND_BYTES:
            raise ValueError(f'target {target} and overlap {overlap}: the fold storage of {self.nstore} folds of {self.fold_len} samples '
                             f'exceeds {COND_BYTES >> 20} MiB')
        self.free_store = list(range(self.nstore))

    # ---- streams ----
    def check_tape(self, uniforms):
        """A stream's tape [K, target + 2 overlap, U], or None."""
        return self.v._check_stream_tape(uniforms, self.fold_len)

    def _open(self, sid, tape, seed):
        """No loop row is taken until the stream's first fold is granted one."""
        if tape is not None:
            tape = tape.to(device=self.device, dtype=torch.float32).contiguous()
        return _FoldedStream(sid, self.device, self.v.feat_dims, tape, seed)

    def _drop(self, st):
        for f in st.folds:
            if f.slot is not None:
                self.slots[f.slot] = None
                f.slot = None
            if f.store is not None:
                self.free_store.append(f.store)
                f.store = None

    # ---- geometry ----
    def folds_known(self, st):
        """Folds of stream st whose existence is certain: fold_count of the samples of the frames that have arrived (all of them once it
        has ended)."""
        return fold_count(st.frames * self.hop, self.target, self.overlap)

    def ready(self, st):
        """The positions below which st's samples can run: generate_stream's readiness rule, (F - 1) hop once it has ended."""
        F_ = st.frames
        return (F_ - 1) * self.hop if st.ended else max(min(F_ - self.lookahead, F_ - 1), 0) * self.hop

    def needed(self, st, k):
        """Steps fold k of st can run so far: up to the ready positions, at most the fold length (<= 0: none)."""
        return min(self.fold_len, self.ready(st) - k * self.step)

    def final(self, st):
        """The end of st's final positions: every position below it has been run by every existing fold that covers it."""
        P = (st.frames - 1) * self.hop if st.ended else 1 << 62
        for f in st.folds:
            if not f.done:
                P = min(P, f.start + f.steps)
        # the first fold without a grant blocks the positions it covers while its existence is undecided, or while it exists and has
        # steps to run
        n = len(st.folds)
        if not st.ended or (n < self.folds_known(st) and self.needed(st, n) > 0):
            P = min(P, n * self.step)
        return P

    # ---- one call ----
    def grants(self):
        """[(stream, k)] of the folds granted a row in the next run(), in grant order: the folds whose existence is certain and that have
        steps to run, by k (target + overlap) minus their stream's released samples, then stream id, while a row and storage are free."""
        wait = []
        for sid, st in self.streams.items():
            for k in range(len(st.folds), self.folds_known(st)):
                if self.needed(st, k) <= 0:
                    break
                wait.append((k * self.step - st.released, sid, k))
        wait.sort()
        n = min(self.slots.count(None), len(self.free_store), len(wait))
        return [(self.streams[sid], k) for _, sid, k in wait[:n]]

    def plan(self):
        """{fold: (position, steps of the next call)} for every fold on a row with steps to run.  The call's budget: POOL_CALL_HOPS hops,
        bounded by COND_BYTES at the rows it runs."""
        work = {f: self.needed(f.st, f.k) - f.steps for f in self.slots if f is not None}
        work = {f: n for f, n in work.items() if n > 0}
        if not work:
            return {}
        S = min(self.S, self.v.chunk_steps(max(f.slot for f in work) + 1, 1 << 30))
        return {f: (f.start + f.steps, min(S, n)) for f, n in work.items()}

    def release_plan(self):
        """[(sid, q0, q1, frames)] of every stream with positions to release: [released, final) once it has ended (frames F), else the whole
        hops of it more than 20 hops behind (frames 0: no fade-out)."""
        rel = []
        for sid, st in self.streams.items():
            P = self.final(st)
            q1 = P if st.ended else (P - 20 * self.hop) // self.hop * self.hop
            if q1 > st.released:
                rel.append((sid, st.released, q1, st.frames if st.ended else 0))
        return rel

    def _busy(self):
        return bool(self.grants() or self.plan())

    def run(self):
        """Grants rows, makes one loop call over every fold with steps to run and releases the final positions -> {sid: the waveform chunk
        it releases}.  A fold beyond a stream's tape raises ValueError before any device work."""
        self._retire()
        grants = self.grants()
        for st, k in grants:
            if st.tape is not None and k >= st.tape.shape[0]:
                raise ValueError(f'the uniform tape holds {st.tape.shape[0]} folds; stream {st.sid} needs fold {k}')
        with self._fp32():
            if grants:
                self._reset(self._grant(grants))
            plan = self.plan()
            if plan:
                self._loop(plan)
            rel = self.release_plan()
            released = self._release(rel) if rel else {}
            _check_loop(self.shape, self.ws)
        for sid in list(self.streams):
            st = self.streams[sid]
            if st.ended and st.released == (st.frames - 1) * self.hop:
                self.close(sid)
        return released

    # ---- host bookkeeping ----
    def _grant(self, grants):
        """Opens the granted folds on the lowest free rows, each with a storage slot -> the rows."""
        free = [r for r, f in enumerate(self.slots) if f is None]
        for (st, k), slot in zip(grants, free):
            f = _Fold(st, k, k * self.step)
            f.slot, f.store = slot, self.free_store.pop()
            st.folds.append(f)
            self.slots[slot] = f
        return free[:len(grants)]

    def _advance(self, plan):
        for f, (_, n) in plan.items():
            f.steps += n
        self._retire()

    def _retire(self):
        """Frees the row of every fold that has run every step it needs: its fold length, or up to the cut once the mel has ended."""
        for f in self.slots:
            if f is not None and (f.steps == self.fold_len or f.st.ended and f.steps == self.needed(f.st, f.k)):
                f.done = True
                self.slots[f.slot] = None
                f.slot = None

    def _mark_released(self, rel):
        """Advances each stream's released samples and frees the storage of its finished folds whose samples are all released."""
        for sid, _, q1, _ in rel:
            st = self.streams[sid]
            st.released = q1
            for f in st.folds:
                if f.done and f.store is not None and f.start + f.steps <= q1:
                    self.free_store.append(f.store)
                    f.store = None

    # ---- device work ----
    def _reset(self, slots):
        self.loop.reset(slots)

    def _loop(self, plan):
        L = self.fold_len
        live = sorted(plan, key=lambda f: f.slot)
        rows = [_Row(f.slot, f.st.mel, f.st.ended, plan[f][0], plan[f][1], f.steps,
                     None if f.st.tape is None else f.st.tape[f.k, f.steps:f.steps + plan[f][1]], f.st.seed, f.k * L + f.steps) for f in live]
        y, active, nmax = self.loop.step_rows(rows)
        # into the storage: fold f's step s at f.store L + s; steps past a row's budget go to the sink
        base, row_n = np.full(active, self.nstore * L, np.int64), np.zeros(active, np.int64)
        for f in live:
            base[f.slot], row_n[f.slot] = f.store * L + f.steps, plan[f][1]
        i = np.arange(nmax)[None, :]
        dst = np.where(i < row_n[:, None], base[:, None] + i, self.nstore * L)
        self.store.index_put_((_upload(dst.reshape(-1), self.device),), y.reshape(-1))
        self._advance(plan)

    def unfold_layout(self, rel):
        """The host side of _release: (b200tts_wavernn_unfold_streams descriptors, the storage base of each fold source entry or -1 for a
        fold that does not exist)."""
        L, descs, base, off = self.fold_len, [], [], 0
        for sid, q0, q1, frames in rel:
            st = self.streams[sid]
            f0 = (q0 - L) // self.step + 1 if q0 >= L else 0
            f1 = (q1 - 1) // self.step
            descs.append(_lib.WaveRNNUnfoldStream(q0, q1, off, frames, f0, f1 - f0 + 1, len(base)))
            # a fold that covers a final position has been opened if it exists
            base += [st.folds[k].store * L if k < len(st.folds) else -1 for k in range(f0, f1 + 1)]
            off += q1 - q0
        return descs, base

    def _release(self, rel):
        """Every stream's final positions through one b200tts_wavernn_unfold_streams launch -> {sid: chunk}."""
        descs, base = self.unfold_layout(rel)
        b = _upload(np.array(base, np.int64), self.device)
        wave = F.wavernn_unfold_streams(self.store, descs, b, torch.full_like(b, self.fold_len, dtype=torch.int32), self.hop, self.target,
                                        self.overlap, self.loop.out_mu)
        self._mark_released(rel)
        return {sid: wave[d.wave_off:d.wave_off + q1 - q0] for d, (sid, q0, q1, _) in zip(descs, rel)}
