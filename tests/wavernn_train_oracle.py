"""fp64 restatement of fatchord's teacher-forced WaveRNN.forward and of both training losses, built over a double copy of the model's own
submodules (plain torch: nn.Conv1d, nn.BatchNorm1d, nn.GRU, nn.Linear, nn.Conv2d); torch autograd gives the gradients."""
import copy

import numpy as np
import torch
import torch.nn.functional as tF

LOG_SCALE_MIN = float(np.log(1e-14))


def double_copy(model, device='cpu'):
    """A float64 copy of `model` on `device`, in the same training / eval mode."""
    return copy.deepcopy(model).to(device=device, dtype=torch.float64)


def _stretch(x, s):
    """Stretch2d(s, 1): nearest repeat x s along the last dimension."""
    return x.repeat_interleave(s, dim=-1)


def upsample(m, mels):
    """UpsampleNetwork.forward: mels [B, feat, W] -> (mel path [B, (W - 2 pad) hop, feat], aux [B, (W - 2 pad) hop, res_out])."""
    up, rn = m.upsample, m.upsample.resnet
    x = torch.relu(rn.batch_norm(rn.conv_in(mels)))
    for layer in rn.layers:
        x = x + layer.batch_norm2(layer.conv2(torch.relu(layer.batch_norm1(layer.conv1(x)))))
    aux = _stretch(rn.conv_out(x), m.hop_length)
    mm = mels.unsqueeze(1)
    for j, s in enumerate(m.upsample_factors):
        mm = up.up_layers[2 * j + 1](_stretch(mm, s))
    mm = mm.squeeze(1)[:, :, up.indent:-up.indent]
    return mm.transpose(1, 2), aux.transpose(1, 2)


def forward(m, x, mels):
    """fatchord's WaveRNN.forward on the fp64 copy m (increments its step buffer): x [B, T], mels [B, feat, T / hop + 2 pad] -> logits
    [B, T, n_classes]."""
    B = x.shape[0]
    m.step += 1
    mel_up, aux = upsample(m, mels)
    A = m.aux_dims
    a1, a2, a3, a4 = (aux[:, :, A * i:A * (i + 1)] for i in range(4))
    h0 = torch.zeros(1, B, m.rnn_dims, dtype=x.dtype, device=x.device)
    h = m.I(torch.cat([x.unsqueeze(-1), mel_up, a1], dim=2))
    h = h + m.rnn1(h, h0)[0]
    h = h + m.rnn2(torch.cat([h, a2], dim=2), h0)[0]
    h = torch.relu(m.fc1(torch.cat([h, a3], dim=2)))
    h = torch.relu(m.fc2(torch.cat([h, a4], dim=2)))
    return m.fc3(h)


def raw_loss(logits, y):
    return tF.cross_entropy(logits.reshape(-1, logits.shape[-1]), y.reshape(-1))


def _log_sum_exp(x):
    m, _ = torch.max(x, dim=-1)
    m2, _ = torch.max(x, dim=-1, keepdim=True)
    return m + torch.log(torch.sum(torch.exp(x - m2), dim=-1))


def mol_loss(logits, y, num_classes=65536, log_scale_min=LOG_SCALE_MIN):
    """fatchord's discretized_mix_logistic_loss (reduce=True) of logits [B, T, 3 nr] against y [B, T] in [-1, 1]."""
    nr = logits.shape[-1] // 3
    logit_probs = logits[..., :nr]
    means = logits[..., nr:2 * nr]
    log_scales = torch.clamp(logits[..., 2 * nr:3 * nr], min=log_scale_min)
    y = y.unsqueeze(-1).expand_as(means)
    centered_y = y - means
    inv_stdv = torch.exp(-log_scales)
    plus_in = inv_stdv * (centered_y + 1. / (num_classes - 1))
    cdf_plus = torch.sigmoid(plus_in)
    min_in = inv_stdv * (centered_y - 1. / (num_classes - 1))
    cdf_min = torch.sigmoid(min_in)
    log_cdf_plus = plus_in - tF.softplus(plus_in)
    log_one_minus_cdf_min = -tF.softplus(min_in)
    cdf_delta = cdf_plus - cdf_min
    mid_in = inv_stdv * centered_y
    log_pdf_mid = mid_in - log_scales - 2. * tF.softplus(mid_in)
    inner_inner_cond = (cdf_delta > 1e-5).to(logits.dtype)
    inner_inner_out = inner_inner_cond * torch.log(torch.clamp(cdf_delta, min=1e-12)) + \
        (1. - inner_inner_cond) * (log_pdf_mid - np.log((num_classes - 1) / 2))
    inner_cond = (y > 0.999).to(logits.dtype)
    inner_out = inner_cond * log_one_minus_cdf_min + (1. - inner_cond) * inner_inner_out
    cond = (y < -0.999).to(logits.dtype)
    log_probs = cond * log_cdf_plus + (1. - cond) * inner_out
    log_probs = log_probs + tF.log_softmax(logit_probs, -1)
    return -torch.mean(_log_sum_exp(log_probs))


def loss(logits, y, mode):
    return raw_loss(logits, y) if mode == 'RAW' else mol_loss(logits, y)


def train_step(m, x, y, mels, mode):
    """One forward + loss + backward on the fp64 copy m (its .grad accumulate): -> (logits, loss)."""
    logits = forward(m, x, mels)
    lo = loss(logits, y, mode)
    lo.backward()
    return logits.detach(), lo.detach()
