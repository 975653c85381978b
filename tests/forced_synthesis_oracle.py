"""CPU oracle of forced synthesis (durations= / alignments=) -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.

`forced(rows)` replaces oracle/tacotron_oracle.py's attention step with one that returns the plan's row for the current step: the
context is that row times the memory, the cumulative weights add it, and no energy is computed.  O.decoder_forward and
outputs_per_step_oracle.decoder_forward look the step up at call time, so both decode from the plan.  `brute_rows` is
durations_to_alignment written frame by frame.
"""
import contextlib

import numpy as np
import torch

from oracle import tacotron_oracle as O


def brute_rows(durations, r):
    """One-hot rows [S, L] (float64): step s attends the symbol that owns frame s r, walking the frames one by one."""
    owner = [j for j, d in enumerate(durations) for _ in range(int(d))]
    S = -(-len(owner) // r)
    rows = np.zeros((S, len(durations)))
    for s in range(S):
        rows[s, owner[s * r]] = 1.0
    return rows


def forced_step(memory, cum, w, mask):
    """One forced attention step -> (context, weights, new cum); weights past the length are zero."""
    w = torch.where(mask, w.to(cum.dtype), torch.zeros_like(cum))
    return (w[:, :, None] * O._q(memory)).sum(dim=1), w, cum + w


@contextlib.contextmanager
def forced(rows):
    """Inside: every oracle decode attends with rows [S, B, L] (step i reads rows[i]; zero rows past S)."""
    saved = O.attention_reset, O.attention_step
    track = {}

    def reset(sd, prefix, memory):
        track['i'] = 0
        return saved[0](sd, prefix, memory)

    def step(sd, prefix, query, memory, memT, cum, mask):
        i = track['i']
        track['i'] += 1
        w = rows[i] if i < rows.shape[0] else torch.zeros_like(cum)
        return forced_step(memory, cum, w, mask)

    O.attention_reset, O.attention_step = reset, step
    try:
        yield track
    finally:
        O.attention_reset, O.attention_step = saved
