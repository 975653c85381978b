"""fp64 numpy restatement of fatchord's WaveRNN generation (models/fatchord_version.py): upsampling network, fold_with_overlap /
xfade_and_unfold, the per-sample step with explicit GRU math, the RAW / MOL samplers on an explicit uniform tape, mu-law decoding and the
final fade-out.  `quantised=True` rounds the loop's recurrent weights and the operands of its products to bf16 (round to nearest even), as
the persistent loop does."""
import numpy as np
import torch

LOG_SCALE_MIN = np.log(1e-14)


def bf16(x):
    """Round to bf16 (nearest even) and back to fp64."""
    return torch.from_numpy(np.asarray(x, dtype=np.float32)).to(torch.bfloat16).to(torch.float64).numpy()


def sigmoid(x):
    return 1.0 / (1.0 + np.exp(-x))


def gru_cell(x, h, w_ih, w_hh, b_ih, b_hh):
    """torch.nn.GRU's cell, gate order r, z, n: x [..., in], h [..., H]."""
    H = h.shape[-1]
    gi = x @ w_ih.T + b_ih
    gh = h @ w_hh.T + b_hh
    r = sigmoid(gi[..., :H] + gh[..., :H])
    z = sigmoid(gi[..., H:2 * H] + gh[..., H:2 * H])
    n = np.tanh(gi[..., 2 * H:] + r * gh[..., 2 * H:])
    return (1 - z) * n + z * h


def sd64(model):
    return {k: v.detach().double().cpu().numpy() for k, v in model.state_dict().items()}


def _bn(x, p, name, eps=1e-5):
    return (x - p[name + '.running_mean'][:, None]) / np.sqrt(p[name + '.running_var'][:, None] + eps) * p[name + '.weight'][:, None] + \
        p[name + '.bias'][:, None]


def upsample(p, mel, factors, pad, res_blocks):
    """mel [feat, F] -> (m [F hop, feat], aux [F hop, res_out]) of UpsampleNetwork on the padded mel."""
    F = mel.shape[1]
    hop = int(np.prod(factors))
    m = np.pad(mel, ((0, 0), (pad, pad)))
    w = p['upsample.resnet.conv_in.weight']            # [C, feat, k]
    k = w.shape[2]
    x = sum(np.einsum('cf,ft->ct', w[:, :, j], m[:, j:j + F]) for j in range(k))
    x = np.maximum(_bn(x, p, 'upsample.resnet.batch_norm'), 0)
    for i in range(res_blocks):
        q = f'upsample.resnet.layers.{i}.'
        y = np.maximum(_bn(p[q + 'conv1.weight'][:, :, 0] @ x, p, q + 'batch_norm1'), 0)
        x = x + _bn(p[q + 'conv2.weight'][:, :, 0] @ y, p, q + 'batch_norm2')
    aux = p['upsample.resnet.conv_out.weight'][:, :, 0] @ x + p['upsample.resnet.conv_out.bias'][:, None]
    aux = np.repeat(aux, hop, axis=1)
    for i, s in enumerate(factors):
        fir = p[f'upsample.up_layers.{2 * i + 1}.weight'].reshape(-1)
        st = np.repeat(m, s, axis=1)
        sp = np.pad(st, ((0, 0), (s, s)))
        m = sum(fir[j] * sp[:, j:j + st.shape[1]] for j in range(2 * s + 1))
    indent = pad * hop
    m = m[:, indent:-indent]
    return m.T, aux.T


def fold_with_overlap(x, target, overlap):
    """x [T, C] -> [folds, target + 2 overlap, C] (fatchord fold_with_overlap)."""
    total_len = x.shape[0]
    num_folds = (total_len - overlap) // (target + overlap)
    extended_len = num_folds * (overlap + target) + overlap
    remaining = total_len - extended_len
    if remaining != 0:
        num_folds += 1
        padding = target + 2 * overlap - remaining
        x = np.concatenate([x, np.zeros((padding,) + x.shape[1:])])
    out = np.zeros((num_folds, target + 2 * overlap) + x.shape[1:])
    for i in range(num_folds):
        start = i * (target + overlap)
        out[i] = x[start:start + target + 2 * overlap]
    return out


def xfade_and_unfold(y, target, overlap):
    y = np.array(y, dtype=np.float64)
    num_folds, length = y.shape
    target = length - 2 * overlap
    total_len = num_folds * (target + overlap) + overlap
    silence_len = overlap // 2
    fade_len = overlap - silence_len
    silence = np.zeros(silence_len, dtype=np.float64)
    t = np.linspace(-1, 1, fade_len, dtype=np.float64)
    fade_in = np.concatenate([silence, np.sqrt(0.5 * (1 + t))])
    fade_out = np.concatenate([np.sqrt(0.5 * (1 - t)), silence])
    y[:, :overlap] *= fade_in
    y[:, -overlap:] *= fade_out
    unfolded = np.zeros(total_len, dtype=np.float64)
    for i in range(num_folds):
        start = i * (target + overlap)
        unfolded[start:start + target + 2 * overlap] += y[i]
    return unfolded


def decode_mu_law(y, mu):
    mu = mu - 1
    return np.sign(y) / mu * ((1 + mu) ** np.abs(y) - 1)


def postprocess(folded, frames, hop, target, overlap, n_classes=None, preemphasis=0.0):
    """Folded samples of one utterance -> its waveform: mu-law decode (RAW: n_classes), de-emphasis of each fold (lfilter([1], [1, -a]),
    when preemphasis != 0), unfold, cut, fade-out."""
    out = np.asarray(folded, dtype=np.float64)
    if n_classes is not None:
        out = decode_mu_law(out, n_classes)
    if preemphasis:
        from scipy.signal import lfilter
        out = lfilter([1.0], [1.0, -preemphasis], out, axis=1)
    out = xfade_and_unfold(out, target, overlap)
    out = out[:(frames - 1) * hop]
    out[-20 * hop:] *= np.linspace(1, 0, 20 * hop)
    return out


def raw_sample(logits, u):
    """(class, margin): the smallest k whose softmax CDF exceeds u, and the distance of u to the nearest CDF boundary around it."""
    z = np.exp(logits - logits.max())
    cdf = np.cumsum(z / z.sum())
    k = int(np.searchsorted(cdf, u, side='right'))
    k = min(k, len(cdf) - 1)
    lo = cdf[k - 1] if k > 0 else 0.0
    return k, min(abs(cdf[k] - u), abs(u - lo))


def mol_sample(logits, u):
    """(sample, margin): Gumbel-argmax component and the logistic draw; margin = gap between the best two Gumbel scores."""
    nr = len(logits) // 3
    uu = 1e-5 + (1 - 2e-5) * np.asarray(u, dtype=np.float64)
    score = logits[:nr] - np.log(-np.log(uu[:nr]))
    order = np.argsort(-score, kind='stable')
    j = int(order[0])
    margin = score[order[0]] - score[order[1]]
    ls = max(logits[2 * nr + j], LOG_SCALE_MIN)
    x = logits[nr + j] + np.exp(ls) * (np.log(uu[nr]) - np.log(1 - uu[nr]))
    return float(np.clip(x, -1, 1)), margin, j


def loop_weights(p, R, Fc, quantised):
    q = bf16 if quantised else (lambda a: a)
    return {
        'w_hh1': q(p['rnn1.weight_hh_l0']), 'b_hh1': p['rnn1.bias_hh_l0'], 'w_ih1': p['rnn1.weight_ih_l0'], 'b_ih1': p['rnn1.bias_ih_l0'],
        'w_I': p['I.weight'], 'b_I': p['I.bias'],
        'w_ih2x': q(p['rnn2.weight_ih_l0'][:, :R]), 'w_ih2a': p['rnn2.weight_ih_l0'][:, R:], 'b_ih2': p['rnn2.bias_ih_l0'],
        'w_hh2': q(p['rnn2.weight_hh_l0']), 'b_hh2': p['rnn2.bias_hh_l0'],
        'w_fc1x': q(p['fc1.weight'][:, :R]), 'w_fc1a': p['fc1.weight'][:, R:], 'b_fc1': p['fc1.bias'],
        'w_fc2x': q(p['fc2.weight'][:, :Fc]), 'w_fc2a': p['fc2.weight'][:, Fc:], 'b_fc2': p['fc2.bias'],
        'w_fc3': q(p['fc3.weight']), 'b_fc3': p['fc3.bias'],
    }


def conditioning(w, feat, n_mels, A):
    """feat [..., n_mels + 4 A] -> (c, g1, c2, p1, p2), the loop inputs that do not depend on the previous sample."""
    c = feat[..., :n_mels + A] @ w['w_I'][:, 1:].T + w['b_I']
    g1 = c @ w['w_ih1'].T + w['b_ih1']
    c2 = feat[..., n_mels + A:n_mels + 2 * A] @ w['w_ih2a'].T + w['b_ih2']
    p1 = feat[..., n_mels + 2 * A:n_mels + 3 * A] @ w['w_fc1a'].T + w['b_fc1']
    p2 = feat[..., n_mels + 3 * A:] @ w['w_fc2a'].T + w['b_fc2']
    return c, g1, c2, p1, p2


def step(w, cond_t, prev, h1, h2, quantised):
    """One step of all rows from (prev [rows], h1, h2): (h1, h2, logits).  With quantised, the products' operands are rounded to bf16."""
    q = bf16 if quantised else (lambda a: a)
    c, g1, c2, p1, p2 = cond_t
    R = h1.shape[-1]
    wp = w['w_I'][:, 0]
    u1 = w['w_ih1'] @ wp
    gi1 = g1 + u1 * prev[:, None]
    gh1 = q(h1) @ w['w_hh1'].T + w['b_hh1']
    h1n = _gru_from_gates(gi1, gh1, h1, R)
    x = c + wp * prev[:, None] + h1n
    gi2 = q(x) @ w['w_ih2x'].T + c2
    gh2 = q(h2) @ w['w_hh2'].T + w['b_hh2']
    h2n = _gru_from_gates(gi2, gh2, h2, R)
    x = x + h2n
    y1 = np.maximum(q(x) @ w['w_fc1x'].T + p1, 0)
    y2 = np.maximum(q(y1) @ w['w_fc2x'].T + p2, 0)
    logits = q(y2) @ w['w_fc3'].T + w['b_fc3']
    return h1n, h2n, logits


def _gru_from_gates(gi, gh, h, H):
    r = sigmoid(gi[..., :H] + gh[..., :H])
    z = sigmoid(gi[..., H:2 * H] + gh[..., H:2 * H])
    n = np.tanh(gi[..., 2 * H:] + r * gh[..., 2 * H:])
    return (1 - z) * n + z * h
