"""fp64 oracle of a routed grouped encoder: each language's utterances run on their own, as a batch of that language alone (G = 1)
with that language's weights, batch-norm affine, running statistics and dropout masks, composed from oracle/tacotron_oracle.py's
pieces.  Both encoder types (ConvolutionalEncoder, GeneratedConvolutionalEncoder) share the block structure O.GENERATED_BLOCKS.

Dropout masks are read from a mask tape in the routed layout: language g's utterances, in batch order, are rows 0 .. n_g - 1 of
channel block g of the tape entry 'enc{j}' [n_max, G*C, L]."""
import torch

from oracle import tacotron_oracle as O


def block_channels(enc):
    """Per-language output channels of each conv block (before the highway gate halves them)."""
    out = []
    for blk in enc._layers:
        rows = blk._block[1].weight.shape[0] if hasattr(blk, '_block') else blk._regularizer.running_mean.shape[0]
        out.append(rows // enc._groups)
    return out


def encode(enc, x, ids, tape=None, training=True, dout=None, device=None):
    """x [B, L, F]; ids: the language of each utterance.  Returns (out [B, L, E], {parameter name: gradient of sum(out * dout)} or
    None, {buffer name: value after the call}), all fp64, for the encoder module `enc` (read, not modified)."""
    gen = hasattr(enc, '_embedding')
    dev = device or x.device
    P = {k: v.detach().to(dev, torch.float64).clone().requires_grad_(dout is not None) for k, v in enc.named_parameters()}
    bufs = {k: v.detach().to(dev, torch.float64).clone() for k, v in enc.named_buffers() if 'running' in k}
    G = enc._groups
    B, L, _ = x.shape
    x = x.detach().to(dev, torch.float64)
    outs, total = [None] * B, None
    for g in range(G):
        idx = [b for b in range(B) if int(ids[b]) == g]
        if not idx:
            continue
        n = len(idx)
        h = x[idx].transpose(1, 2)
        for j, (k, dil, act, highway) in enumerate(O.GENERATED_BLOCKS):
            blk, pre = enc._layers[j], f'_layers.{j}'
            Cin = h.shape[1]
            if gen:
                e = P['_embedding.weight'][g:g + 1]
                kern = O.generated_kernel(P, f'{pre}._convolution', e)
                C = kern.shape[1] // (Cin * k)
                w = kern[0].view(C, Cin, k)
                eb = O._linear(e, P[f'{pre}._regularizer._bottleneck.weight'], P[f'{pre}._regularizer._bottleneck.bias'])
                aff = O._linear(eb, P[f'{pre}._regularizer._affine.weight'], P[f'{pre}._regularizer._affine.bias'])
                gamma, beta = aff[0, :C], aff[0, C:]
                rmk, rvk = f'{pre}._regularizer.running_mean', f'{pre}._regularizer.running_var'
                eps, mom = blk._regularizer._eps, blk._regularizer._momentum
            else:
                C = P[f'{pre}._block.1.weight'].shape[0] // G
                sl = slice(g * C, (g + 1) * C)
                w = P[f'{pre}._block.1.weight'][sl]
                gamma, beta = P[f'{pre}._block.2.weight'][sl], P[f'{pre}._block.2.bias'][sl]
                rmk, rvk = f'{pre}._block.2.running_mean', f'{pre}._block.2.running_var'
                eps, mom = blk._block[2].eps, blk._block[2].momentum
            sl = slice(g * C, (g + 1) * C)
            y = O.conv1d_same(h, w, dil)
            if training:
                y, mean, var = O.batch_norm_train(y, gamma, beta, eps)
                rm, rv = O.running_stats_update(bufs[rmk][sl], bufs[rvk][sl], mean.detach().reshape(-1), var.detach().reshape(-1),
                                                n * L, mom)
                bufs[rmk][sl], bufs[rvk][sl] = rm, rv
            else:
                y = O.batch_norm_eval(y, gamma, beta, bufs[rmk][sl], bufs[rvk][sl], eps)
            y = O._act(act, y)
            if training and tape is not None and tape.get(f'enc{j}') is not None:
                keep = tape[f'enc{j}'][:n, sl].to(dev, torch.float64)
                y = O.apply_dropout(y, keep, blk._dropout_rate)
            if highway:
                half = C // 2
                gate = O._sigmoid(y[:, :half])
                h = y[:, half:] * gate + h * (1.0 - gate)
            else:
                h = y
        o = h.transpose(1, 2)
        for r, b in enumerate(idx):
            outs[b] = o[r]
        if dout is not None:
            term = (o * dout[idx].to(dev, torch.float64)).sum()
            total = term if total is None else total + term
    out = torch.stack(outs)
    grads = None
    if dout is not None:
        total.backward()
        grads = {k: (p.grad if p.grad is not None else torch.zeros_like(p)) for k, p in P.items()}
    return out.detach(), grads, bufs


def routed_tape(enc, ids, L, p, generator):
    """Random keep masks 'enc{j}' in the routed layout [n_max, G*C_j, L] of the batch with languages ids."""
    G = enc._groups
    n_max = max(sum(1 for i in ids if int(i) == g) for g in range(G))
    return {f'enc{j}': (torch.rand(n_max, G * C, L, generator=generator) >= p).to(torch.uint8)
            for j, C in enumerate(block_channels(enc))}
