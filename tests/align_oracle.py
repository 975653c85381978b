"""fp64 numpy oracles of the forced-alignment kernels (include/b200tts.h): the monotonic alignment search with its tie rule, a brute-force
search for tiny grids, and the alignment scores."""
import itertools

import numpy as np


def log_weights(P):
    return np.log(np.maximum(np.asarray(P, dtype=np.float32).astype(np.float64), 1e-8))


def mas(P, n_text, n_steps):
    """One utterance: P [>= n_steps, >= n_text] -> (durations int [n_text], path_logp, path int [n_steps]).  Q[s][l] = lp[s, l] +
    max(Q[s-1][l], Q[s-1][l-1]); the path advances to l only when Q[s-1][l-1] > Q[s-1][l] (stays on equal values)."""
    assert 1 <= n_text <= n_steps
    lp = log_weights(np.asarray(P)[:n_steps, :n_text])
    Q = np.full(n_text, -np.inf)
    Q[0] = lp[0, 0]
    adv = np.zeros((n_steps, n_text), dtype=bool)
    for s in range(1, n_steps):
        diag = np.concatenate(([-np.inf], Q[:-1]))
        adv[s] = diag > Q
        Q = lp[s] + np.where(adv[s], diag, Q)
    path = np.empty(n_steps, dtype=np.int64)
    l = n_text - 1
    for s in range(n_steps - 1, -1, -1):
        path[s] = l
        if s > 0 and adv[s, l]:
            l -= 1
    assert l == 0
    return np.bincount(path, minlength=n_text), float(Q[n_text - 1]), path


def mas_batch(P, text_lengths, step_lengths):
    """P [B, S, L] -> (durations int [B, L] zero past L_b, path_logp [B], path int [B, S] -1 past S_b)."""
    B, S, L = P.shape
    dur, logp, path = np.zeros((B, L), np.int64), np.zeros(B), np.full((B, S), -1, np.int64)
    for b in range(B):
        d, v, p = mas(P[b], int(text_lengths[b]), int(step_lengths[b]))
        dur[b, :len(d)], logp[b], path[b, :len(p)] = d, v, p
    return dur, logp, path


def monotonic_paths(n_text, n_steps):
    """Every path from symbol 0 to n_text - 1 over n_steps steps moving by 0 or 1: choose the n_text - 1 steps that advance."""
    for moves in itertools.combinations(range(1, n_steps), n_text - 1):
        path = np.zeros(n_steps, np.int64)
        for s in moves:
            path[s:] += 1
        yield path


def brute_force_best(P, n_text, n_steps):
    """The largest path sum over all monotonic paths, each summed in step order as the DP does."""
    lp = log_weights(np.asarray(P)[:n_steps, :n_text])
    best = -np.inf
    for path in monotonic_paths(n_text, n_steps):
        v = 0.0
        for s, l in enumerate(path):
            v = lp[s, l] if s == 0 else v + lp[s, l]
        best = max(best, v)
    return best


def scores(P, n_text, n_steps):
    """(focus rate, coverage, largest forward argmax move, moves back) over the valid steps and symbols, in fp64."""
    W = np.asarray(P, dtype=np.float64)[:n_steps, :n_text]
    am = W.argmax(1)
    moves = np.diff(am)
    return (float(W.max(1).mean()), float((W.sum(0) >= 0.5).mean()), int(max(0, moves.max(initial=0))), bool((moves < 0).any()),
            W.sum(0))
