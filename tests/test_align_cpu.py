"""Forced alignment on the host: the fp64 oracle of the monotonic alignment search against brute force and its tie rule, the limits the
header states, and every ValueError of functional.monotonic_alignment and Tacotron.align (raised before any device work)."""
import os
import re

import numpy as np
import pytest
import torch

import align_oracle as A
import model_cases
from helpers import Golden, ROOT


def _random(rng, S, L):
    return rng.dirichlet(np.ones(L) * 0.3, size=S).astype(np.float32)


@pytest.mark.parametrize('seed', range(40))
def test_oracle_path_is_monotonic_and_covers_every_symbol(seed):
    rng = np.random.default_rng(seed)
    L = int(rng.integers(1, 12))
    S = L + int(rng.integers(0, 30))
    P = _random(rng, S + 2, L + 3)                       # padding past the lengths is never read
    dur, logp, path = A.mas(P, L, S)
    assert path[0] == 0 and path[-1] == L - 1
    assert set(np.diff(path).tolist()) <= {0, 1}
    assert (dur >= 1).all() and dur.sum() == S
    assert np.array_equal(dur, np.bincount(path, minlength=L))
    lp = A.log_weights(P)
    assert logp == pytest.approx(sum(lp[s, l] for s, l in enumerate(path)), rel=1e-13)


@pytest.mark.parametrize('L,S', [(1, 1), (1, 5), (2, 2), (3, 7), (4, 8), (5, 9), (6, 10)])
def test_oracle_reaches_the_brute_force_maximum(L, S):
    rng = np.random.default_rng(L * 100 + S)
    for _ in range(5):
        P = _random(rng, S, L)
        dur, logp, path = A.mas(P, L, S)
        assert logp == A.brute_force_best(P, L, S)


def test_oracle_tie_rule_stays_on_the_symbol():
    # uniform weights: every path ties, and at every cell the search keeps the same symbol, so the walk back from the last symbol stays
    # there until the diagonal forces it down: one step for each earlier symbol, the rest on the last
    S, L = 9, 4
    dur, _, path = A.mas(np.full((S, L), 0.25, np.float32), L, S)
    assert dur.tolist() == [1, 1, 1, 6] and path.tolist() == [0, 1, 2, 3, 3, 3, 3, 3, 3]
    # weights equal along each step: every path has the same value, summed in the same order
    row = np.random.default_rng(3).random(S).astype(np.float32)
    assert A.mas(np.repeat(row[:, None], L, 1), L, S)[0].tolist() == [1, 1, 1, 6]
    # below 1e-8 every weight clamps to the same value
    assert A.mas(np.full((S, L), 1e-12, np.float32), L, S)[0].tolist() == [1, 1, 1, 6]


def test_oracle_scores():
    P = np.zeros((5, 3), np.float32)
    for s, l in enumerate([0, 0, 2, 1, 2]):
        P[s, l] = 0.75
        P[s, (l + 1) % 3] = 0.25
    focus, coverage, jump, back, _ = A.scores(P, 3, 5)
    assert focus == 0.75 and jump == 2 and back
    assert coverage == 1.0                                  # column sums 1.5, 1.0, 1.75


def test_header_limits_follow_from_shared_memory():
    from multilingual_text_to_speech_b200 import _lib
    h = open(os.path.join(ROOT, 'include', 'b200tts.h')).read()
    assert re.search(rf'#define B200TTS_ALIGN_MAX_SYMBOLS {_lib.ALIGN_MAX_SYMBOLS}\b', h)
    assert re.search(rf'#define B200TTS_ALIGN_MAX_CELLS {_lib.ALIGN_MAX_CELLS}\b', h)
    # two fp64 rows of the longest text plus one bit per cell fill the 227 KB an sm_90 CTA may have
    assert 16 * _lib.ALIGN_MAX_SYMBOLS + _lib.ALIGN_MAX_CELLS // 8 == 227 * 1024
    assert _lib.ALIGN_MAX_CELLS == 1688 * 1024 and 1200 * 300 // 8 == 45000


def _weights(B=2, S=6, L=4):
    return torch.full((B, S, L), 0.25)


@pytest.mark.parametrize('args,message', [
    ((torch.full((6, 4), 0.25), [4], [6]), r'weights must be a \[B, S, L\] tensor'),
    ((_weights().double(), [4, 4], [6, 6]), 'weights must be float32'),
    ((_weights(S=0), [4, 4], [6, 6]), 'weights must be non-empty'),
    ((_weights(), [4], [6, 6]), r'text_lengths must hold one length per utterance \(2\)'),
    ((_weights(), [4, 4], torch.tensor([6.0, 6.0])), 'step_lengths must be integers'),
    ((_weights(), [0, 4], [6, 6]), r'utterance 0: text length 0 is outside \[1, 4\]'),
    ((_weights(), [4, 5], [6, 6]), r'utterance 1: text length 5 is outside \[1, 4\]'),
    ((_weights(), [4, 4], [6, 7]), r'utterance 1: step count 7 is outside \[1, 6\]'),
    ((_weights(), [4, 4], [6, 3]), 'utterance 1: 3 steps cannot cover 4 symbols'),
    ((torch.full((1, 1100, 1025), 1e-3), [1025], [1100]), 'utterance 0: 1025 symbols exceed the 1024'),
    ((torch.full((1, 1689, 1024), 1e-3), [1024], [1689]), r'utterance 0: 1689 steps x 1024 symbols = 1729536 cells exceed the 1728512'),
])
def test_monotonic_alignment_value_errors(args, message):
    from multilingual_text_to_speech_b200 import functional as F
    with pytest.raises(ValueError, match=message):
        F.monotonic_alignment(*args)
    with pytest.raises(ValueError, match=message):
        F.alignment_scores(*args)


@pytest.mark.parametrize('bad', [float('nan'), float('inf'), -float('inf')])
def test_monotonic_alignment_rejects_non_finite_weights(bad):
    from multilingual_text_to_speech_b200 import functional as F
    w = _weights()
    w[1, 2, 3] = bad
    with pytest.raises(ValueError, match='weights must be finite'):
        F.monotonic_alignment(w, [4, 4], [6, 6])


def test_largest_accepted_shape_passes_the_host_checks():
    from multilingual_text_to_speech_b200 import functional as F
    assert F.check_alignment_lengths([1024, 300], [1688, 5761], 2, 5761, 1024) == ([1024, 300], [1688, 5761])


@pytest.fixture(scope='module')
def model():
    g = Golden('lj_eval_free')
    m = model_cases.build_model(g)
    return m, g


def _align_inputs(g):
    i = g.inputs
    return [i['text'], i['text_length'], i['target'], i['target_length']]


def _replace(args, k, v):
    args = list(args)
    args[k] = v
    return args


@pytest.mark.parametrize('edit,message', [
    (lambda a: _replace(a, 0, a[0][0]), 'align: text must be a 2-D tensor'),
    (lambda a: _replace(a, 1, a[1].unsqueeze(0)), 'align: text_length must be a 1-D tensor'),
    (lambda a: _replace(a, 2, a[2][0]), 'align: target must be a 3-D tensor'),
    (lambda a: _replace(a, 3, [10, 10, 10]), 'align: target_length must be a 1-D tensor'),
    (lambda a: _replace(a, 0, a[0].float()), 'align: text must hold symbol ids'),
    (lambda a: _replace(a, 2, a[2][:, :6]), r'align: target must be \[B = 3, num_mels = 12, T\]'),
    (lambda a: _replace(a, 3, torch.tensor([10, 0, 10])), r'align: utterance 1: target length 0 is outside \[1, 10\]'),
    (lambda a: _replace(a, 3, torch.tensor([10, 11, 10])), r'align: utterance 1: target length 11 is outside \[1, 10\]'),
    (lambda a: _replace(a, 3, torch.tensor([10, 10, 3])), r'utterance 2: \d steps cannot cover \d symbols'),
    (lambda a: _replace(a, 1, torch.tensor([9, 10, 5])), r'utterance 1: text length 10 is outside \[1, 9\]'),
    (lambda a: _replace(a, 1, torch.tensor([9, 7])), r'text_lengths must hold one length per utterance \(3\)'),
])
def test_align_value_errors(model, edit, message):
    m, g = model
    with pytest.raises(ValueError, match=message):
        m.align(*edit(_align_inputs(g)))


def test_align_value_error_on_the_step_grid(model):
    """At r = 2 the search has ceil(T_b / 2) steps: 9 symbols need at least 17 frames."""
    m, g = model
    r = m._decoder._outputs_per_step
    try:
        m._decoder._outputs_per_step = 2
        args = _align_inputs(g)
        args[1] = torch.tensor([9, 5, 5])
        args[3] = torch.tensor([10, 10, 10])
        with pytest.raises(ValueError, match='utterance 0: 5 steps cannot cover 9 symbols'):
            m.align(*args)
    finally:
        m._decoder._outputs_per_step = r
