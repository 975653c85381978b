"""CPU oracle of windowed synthesis (hp.inference_attention_window) -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.

Step i of utterance b gives energies only to positions [c_b - back, c_b + ahead] within its length: those positions join the padding
mask of oracle/tacotron_oracle.py's attention_step, whose softmax, cumulative weights and context are used as they are.  c_b is 0 before
step 0 and then torch.argmax of the step's weights (the first maximum).  `windowed()` switches O's attention functions, which
O.decoder_forward and outputs_per_step_oracle.decoder_forward look up at call time, so both decode with the window.
"""
import contextlib

import torch

from oracle import tacotron_oracle as O

_attention_step = O.attention_step      # windowed() replaces O's; the window narrows the mask of this one


def window_mask(centre, L, window):
    """[B, L] bool: positions [centre - back, centre + ahead] of each row."""
    back, ahead = window
    pos = torch.arange(L)[None]
    c = centre.long()[:, None]
    return (pos >= c - back) & (pos <= c + ahead)


def attention_step(sd, prefix, query, memory, memT, cum, mask, centre, window=None):
    """One windowed LocationSensitiveAttention step -> (context, weights, new cum, new centre).  window None: O.attention_step."""
    if window is not None:
        mask = mask & window_mask(centre, cum.shape[1], window)
    ctx, w, cum = _attention_step(sd, prefix, query, memory, memT, cum, mask)
    return ctx, w, cum, torch.argmax(w, dim=1)


@contextlib.contextmanager
def windowed(window):
    """Inside: every decode of the oracle attends through the window; yields {'centre': the centres after the last step}."""
    saved = O.attention_reset, O.attention_step
    track = {}

    def reset(sd, prefix, memory):
        track['centre'] = torch.zeros(memory.shape[0], dtype=torch.long)
        return saved[0](sd, prefix, memory)

    def step(sd, prefix, query, memory, memT, cum, mask):
        ctx, w, cum, track['centre'] = attention_step(sd, prefix, query, memory, memT, cum, mask, track['centre'], window)
        return ctx, w, cum

    O.attention_reset, O.attention_step = reset, step
    try:
        yield track
    finally:
        O.attention_reset, O.attention_step = saved


def check_window_property(align, lengths, window, atol=1e-5):
    """align [B, S, L] from a decode: every row's non-zero weights lie in the window of the previous row's first argmax (0 for row 0)
    and within the utterance's length, and every row sums to 1 within atol.  Rows of all zeros (past an utterance's cut) are skipped."""
    align = align.double().cpu()
    B, S, L = align.shape
    for b in range(B):
        c = torch.zeros(1, dtype=torch.long)
        for i in range(S):
            row = align[b, i]
            if not bool((row != 0).any()):
                break
            allowed = window_mask(c, L, window)[0] & (torch.arange(L) < int(lengths[b]))
            assert not bool((row[~allowed] != 0).any()), (b, i, int(c), torch.nonzero(row).flatten().tolist())
            assert abs(float(row.sum()) - 1.0) <= atol, (b, i, float(row.sum()))
            c = torch.argmax(row).reshape(1)
