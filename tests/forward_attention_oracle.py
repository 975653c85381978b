"""CPU oracle of forward attention (reference modules/attention.py:23-45, 89-124) -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.

Elementary torch arithmetic (float32 or float64), pinned against tests/golden/fwd_*.npz (tests/golden/make_golden_forward_attention.py,
the unmodified reference).  The decoder, model and loss are the location-sensitive oracle's own (oracle/tacotron_oracle.py);
`forward_attention()` swaps its two attention functions for the ones below while a decode runs, so both attention types share
one restatement of Decoder._decode.
"""
import contextlib

import torch

from oracle import tacotron_oracle as O


def attention_reset(sd, prefix, memory):
    """ForwardAttention.reset: memT = memory . Wm^T; alpha = one-hot at position 0; context = 0."""
    B, L, M = memory.shape
    memT = O._linear(memory, sd[f'{prefix}._memory.weight'])      # the per-step kernels keep the projection in fp32
    alpha = torch.zeros(B, L, dtype=memory.dtype)
    alpha[:, 0] = 1
    return memT, alpha, torch.zeros(B, M, dtype=memory.dtype)


def attention_step(sd, prefix, query, memory, memT, alpha, mask):
    """One ForwardAttention.forward call.  Returns (context, weights, new alpha = weights)."""
    Wq = sd[f'{prefix}._query.weight']                 # [A, D]
    bias = sd[f'{prefix}._bias']                       # [1, A]
    v = sd[f'{prefix}._energy.weight']                 # [1, A]
    q = query @ Wq.transpose(0, 1)                     # [B, A]  (fp32 in both precision modes)
    e = (torch.tanh(q[:, None, :] + memT + bias.view(1, 1, -1)) * v.view(1, 1, -1)).sum(dim=2)    # [B, L]
    ex = torch.exp(e - e.max(dim=1, keepdim=True).values)
    s = ex / ex.sum(dim=1, keepdim=True)               # softmax over every position, padding included
    shifted = torch.cat((torch.zeros_like(alpha[:, :1]), alpha[:, :-1]), dim=1)
    a = (alpha + shifted) * s
    a = torch.where(mask, a, torch.zeros_like(a))      # energies[~mask] = 0 (in place in the reference: no gradient there)
    c = torch.clamp(a, min=1e-6)
    w = c / c.sum(dim=1, keepdim=True).clamp(min=1e-12)     # F.normalize(p=1)
    ctx = (w[:, :, None] * memory).sum(dim=1)          # over every position, padding included
    return ctx, w, w


@contextlib.contextmanager
def forward_attention():
    """Run O.decoder_forward / O.tacotron_forward with forward attention."""
    saved = O.attention_reset, O.attention_step
    O.attention_reset, O.attention_step = attention_reset, attention_step
    try:
        yield
    finally:
        O.attention_reset, O.attention_step = saved


def for_hp(hp):
    """The attention of `hp` (hp.attention_type, default location_sensitive) as a context manager."""
    return forward_attention() if getattr(hp, 'attention_type', 'location_sensitive') == 'forward' else contextlib.nullcontext()
