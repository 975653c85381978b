"""Forced alignment on the H100: the monotonic alignment search kernel against the fp64 oracle (tests/align_oracle.py), the scores kernel
against fp64, and Tacotron.align on the golden batches at r = 1 and r = 2 in both precision modes."""
import numpy as np
import pytest
import torch

import align_oracle as A
import model_cases
import outputs_per_step_oracle as R
from helpers import Golden

pytestmark = pytest.mark.gpu


@pytest.fixture(scope='module', autouse=True)
def _built():
    import __graft_entry__ as entry
    entry.build()
    assert torch.cuda.is_available(), 'GPU tests need a CUDA device'


def _dirichlet(rng, S, L, alpha=0.3):
    return rng.dirichlet(np.ones(L) * alpha, size=S).astype(np.float32)


def _diagonal(rng, S, L, width=1.5):
    """Sharp weights around the line from (0, 0) to (S - 1, L - 1), renormalised per step."""
    centre = np.linspace(0, L - 1, S)[:, None] + rng.normal(0, 0.3, (S, 1))
    w = np.exp(-0.5 * ((np.arange(L)[None, :] - centre) / width) ** 2) + 1e-12
    return (w / w.sum(1, keepdims=True)).astype(np.float32)


def _batch(items, pad_s=0, pad_l=0, fill=0.0):
    """Pack [(P_b [S_b, L_b])] into a padded [B, S, L] batch filled with `fill`."""
    S = max(p.shape[0] for p in items) + pad_s
    L = max(p.shape[1] for p in items) + pad_l
    out = np.full((len(items), S, L), fill, np.float32)
    for b, p in enumerate(items):
        out[b, :p.shape[0], :p.shape[1]] = p
    return out, [p.shape[1] for p in items], [p.shape[0] for p in items]


def _check(P, tl, sl, noncontiguous=False):
    from multilingual_text_to_speech_b200 import functional as F
    w = torch.from_numpy(P).cuda()
    if noncontiguous:      # a row stride larger than L and a batch stride larger than S ld
        big = torch.full((P.shape[0], P.shape[1] + 3, P.shape[2] + 5), 0.5, device='cuda')
        big[:, :P.shape[1], :P.shape[2]] = w
        w = big[:, :P.shape[1], :P.shape[2]]
    dur, logp, path = F.monotonic_alignment(w, torch.tensor(tl), torch.tensor(sl), return_path=True)
    torch.cuda.synchronize()
    want_d, want_v, want_p = A.mas_batch(P, tl, sl)
    assert dur.dtype == torch.int32 and logp.dtype == torch.float64 and path.dtype == torch.int32
    assert np.array_equal(dur.cpu().numpy(), want_d), 'durations'
    assert np.array_equal(path.cpu().numpy(), want_p), 'path'
    np.testing.assert_allclose(logp.cpu().numpy(), want_v, rtol=1e-12, atol=0)
    d2, v2 = F.monotonic_alignment(w, tl, sl)
    assert torch.equal(d2, dur) and torch.equal(v2, logp)
    return dur, logp


@pytest.mark.parametrize('kind', ['random', 'diagonal'])
@pytest.mark.parametrize('L,S', [(1, 1), (1, 37), (7, 7), (40, 40), (33, 95), (180, 900), (300, 1200), (5, 3000), (1024, 1100)])
def test_kernel_matches_the_oracle(kind, L, S):
    rng = np.random.default_rng(L * 7919 + S)
    make = _dirichlet if kind == 'random' else _diagonal
    P, tl, sl = _batch([make(rng, S, L), make(rng, max(L, S // 2), max(1, L // 2))], pad_s=2, pad_l=3, fill=0.7)
    _check(P, tl, sl)


def test_kernel_reads_strided_weights():
    rng = np.random.default_rng(5)
    P, tl, sl = _batch([_dirichlet(rng, 60, 20), _diagonal(rng, 41, 17)])
    _check(P, tl, sl, noncontiguous=True)


@pytest.mark.parametrize('B', [1, 7, 64])
def test_ragged_batches_at_the_largest_accepted_shape(B):
    from multilingual_text_to_speech_b200 import _lib
    rng = np.random.default_rng(B)
    items = [_diagonal(rng, 1688, 1024), _dirichlet(rng, _lib.ALIGN_MAX_CELLS // 300, 300)]
    while len(items) < B:
        L = int(rng.integers(1, 400))
        S = int(rng.integers(L, min(3000, _lib.ALIGN_MAX_CELLS // L) + 1))
        items.append((_diagonal if rng.random() < 0.5 else _dirichlet)(rng, S, L))
    items = items[:B]
    P, tl, sl = _batch(items)
    assert max(s * n for s, n in zip(sl, tl)) <= _lib.ALIGN_MAX_CELLS
    dur, _ = _check(P, tl, sl)
    # each utterance alone gives the same integers: the result does not depend on the batch
    b = B - 1
    alone = _batch([items[b]])
    from multilingual_text_to_speech_b200 import functional as F
    d1, _ = F.monotonic_alignment(torch.from_numpy(alone[0]).cuda(), alone[1], alone[2])
    assert torch.equal(d1[0, :tl[b]], dur[b, :tl[b]])


@pytest.mark.parametrize('case', ['uniform', 'equal_per_step', 'clamped', 'blocks'])
def test_exact_ties_follow_the_tie_rule(case):
    rng = np.random.default_rng(11)
    S, L = 300, 70
    if case == 'uniform':
        P = np.full((S, L), 1.0 / L, np.float32)
    elif case == 'equal_per_step':
        P = np.repeat(rng.random((S, 1)).astype(np.float32), L, 1)
    elif case == 'clamped':
        P = np.full((S, L), 1e-20, np.float32)
    else:   # two-valued blocks: many paths share their sums exactly
        P = np.where(rng.random((S, L)) < 0.5, 0.5, 0.25).astype(np.float32)
    dur, _ = _check(P[None], [L], [S])
    if case != 'blocks':
        assert dur[0].tolist() == [1] * (L - 1) + [S - L + 1]


@pytest.mark.parametrize('seed', range(4))
def test_scores_match_fp64(seed):
    from multilingual_text_to_speech_b200 import functional as F
    rng = np.random.default_rng(100 + seed)
    items = []
    for b in range(9):
        L = int(rng.integers(1, 200))
        S = int(rng.integers(L, L + 1000))
        items.append((_diagonal if b % 2 else _dirichlet)(rng, S, L))
    items.append(np.eye(5, dtype=np.float32)[[0, 1, 1, 4, 2, 3, 4]])     # jump of 3 and moves back
    P, tl, sl = _batch(items, pad_s=3, pad_l=2, fill=0.9)
    got = {k: v.cpu().numpy() for k, v in F.alignment_scores(torch.from_numpy(P).cuda(), tl, sl).items()}
    for b in range(len(items)):
        focus, coverage, jump, back, colsum = A.scores(P[b], tl[b], sl[b])
        assert abs(float(got['focus_rate'][b]) - focus) <= 2 ** -23 * focus + 1e-12, b
        near = np.abs(colsum - 0.5) < 1e-6                  # the fp64 sum order may decide a column exactly at 0.5
        assert abs(float(got['coverage'][b]) - coverage) <= near.sum() / tl[b] + 1e-7, b
        assert int(got['max_jump'][b]) == jump and bool(got['moves_back'][b]) == back, b
    assert int(got['max_jump'][-1]) == 3 and bool(got['moves_back'][-1])


# ---- Tacotron.align ----

def _golden_model(name, r, dev):
    """The golden's model and batch on the device; at r = 2 a seeded model of the golden's configuration with every target frame
    repeated twice (so that each utterance keeps at least as many steps as symbols), with the tape cut to the step grid."""
    from multilingual_text_to_speech_b200.modules.tacotron2 import Tacotron
    from multilingual_text_to_speech_b200.params.params import Params as hp
    g = Golden(name)
    batch = {k: v.to(dev) for k, v in g.inputs.items()}
    if r == 1:
        model = model_cases.build_model(g, dev)
    else:
        model_cases.configure_hp(g)
        hp.outputs_per_step = r
        torch.manual_seed(0)
        model = Tacotron().to(dev)
        batch['target'] = R.repeat_frames(batch['target'], r, 2)
        batch['target_length'] = batch['target_length'] * r - 1          # not a multiple of r: the last step's last frame is cut
    S = R.steps(batch['target'].shape[2], r)
    tape = {}
    for k, v in g.tape.items():
        if k in ('prenet0', 'prenet1'):
            tape[k] = v[:, :S + 1].contiguous().to(dev)
    return model, batch, tape, S


def _forward_alignment(model, batch, tape, S):
    from multilingual_text_to_speech_b200.rng import MaskSource
    was = model.training
    model.eval()
    MaskSource.use_tape({**tape, 'teacher': torch.ones(S, dtype=torch.bool)})
    try:
        with torch.no_grad():
            return model(batch['text'], batch['text_length'], batch['target'], batch['target_length'], batch.get('speakers'),
                         batch.get('languages'), 1.0)[3]
    finally:
        MaskSource.use_tape(None)
        model.train(was)


@pytest.mark.parametrize('precision', ['fp32', 'bf16'])
@pytest.mark.parametrize('name,r', [('lj_eval_free', 1), ('generated_training', 1), ('fwd_lj_eval_free', 1), ('lj_eval_free', 2),
                                    ('generated_training', 2), ('generated_switching', 1)])
def test_tacotron_align_on_the_goldens(name, r, precision):
    from multilingual_text_to_speech_b200 import _lib
    from multilingual_text_to_speech_b200.params.params import Params as hp
    from multilingual_text_to_speech_b200.rng import MaskSource
    dev = torch.device('cuda:0')
    try:
        model, batch, tape, S = _golden_model(name, r, dev)
        was_training = model.training
        _lib.set_precision(precision)
        want = _forward_alignment(model, batch, tape, S)
        MaskSource.use_tape(tape)
        try:
            got = model.align(batch['text'], batch['text_length'], batch['target'], batch['target_length'], batch.get('speakers'),
                              batch.get('languages'))
        finally:
            MaskSource.use_tape(None)
        torch.cuda.synchronize()
        assert model.training == was_training and MaskSource.tape is None
        assert torch.equal(got.alignment, want), 'alignment is not forward\'s bit for bit'
        tl = batch['text_length'].tolist()
        frames = batch['target_length'].tolist()
        steps = [-(-t // r) for t in frames]
        assert want.shape[1] == S
        d, v, _ = A.mas_batch(want.cpu().numpy(), tl, steps)
        assert np.array_equal(got.step_durations.cpu().numpy(), d)
        np.testing.assert_allclose(got.path_logp.cpu().numpy(), v, rtol=1e-12, atol=0)
        dur = got.durations.cpu().numpy()
        assert dur.sum(1).tolist() == frames
        for b in range(len(tl)):
            assert (dur[b, :tl[b]] >= 1).all() and (dur[b, tl[b]:] == 0).all()
            assert np.array_equal(dur[b, :tl[b] - 1], d[b, :tl[b] - 1] * r)
            focus, coverage, jump, back, _ = A.scores(want[b].cpu().numpy(), tl[b], steps[b])
            assert abs(float(got.focus_rate[b]) - focus) <= 1e-6 * focus
            assert int(got.max_jump[b]) == jump and bool(got.moves_back[b]) == back
    finally:
        _lib.set_precision('fp32')
        hp.reset()


def test_tacotron_align_on_a_language_sorted_grouped_batch():
    """generated_training's batch with its utterances sorted by language (the other layout the grouped encoder routes)."""
    from multilingual_text_to_speech_b200.params.params import Params as hp
    from multilingual_text_to_speech_b200.rng import MaskSource
    dev = torch.device('cuda:0')
    try:
        model, batch, tape, S = _golden_model('generated_training', 1, dev)
        order = torch.argsort(batch['languages'].cpu(), stable=True).to(dev)
        batch = {k: v[order] for k, v in batch.items()}
        tape = {k: v[order] for k, v in tape.items()}
        want = _forward_alignment(model, batch, tape, S)
        MaskSource.use_tape(tape)
        try:
            got = model.align(batch['text'], batch['text_length'], batch['target'], batch['target_length'], None, batch['languages'])
        finally:
            MaskSource.use_tape(None)
        assert torch.equal(got.alignment, want)
        d, _, _ = A.mas_batch(want.cpu().numpy(), batch['text_length'].tolist(), batch['target_length'].tolist())
        assert np.array_equal(got.durations.cpu().numpy(), d)
    finally:
        hp.reset()


def test_export_alignments_writes_one_file_per_utterance(tmp_path):
    import importlib.util
    import os
    from helpers import ROOT
    from multilingual_text_to_speech_b200.params.params import Params as hp
    spec = importlib.util.spec_from_file_location('export_alignments', os.path.join(ROOT, 'tools', 'export_alignments.py'))
    tool = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(tool)
    try:
        g = Golden('generated_training')
        model = model_cases.build_model(g, torch.device('cuda:0'))
        i = g.inputs
        items = [(0, int(i['languages'][b]), i['text'][b, :int(i['text_length'][b])].tolist(),
                  i['target'][b, :, :int(i['target_length'][b])].numpy(), None) for b in range(g.B)]
        ids = [f'utt{b:03}' for b in range(g.B)]
        tool.export(model, tool.ItemDataset(items), ids, str(tmp_path), batch_size=4)
        for b, uid in enumerate(ids):
            dur = np.load(os.path.join(tmp_path, f'{uid}.durations.npy'))
            sc = np.load(os.path.join(tmp_path, f'{uid}.scores.npy'))
            assert dur.shape == (len(items[b][2]),) and dur.sum() == items[b][3].shape[1] and (dur >= 1).all()
            assert sc.shape == (5,) and 0 < sc[0] <= 1 and 0 <= sc[1] <= 1
    finally:
        hp.reset()
