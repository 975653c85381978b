"""The bi-LSTM step checker (tests/bilstm_check.py) on synthetic saved states, without a GPU.

A synthetic state is the recurrence of both directions in fp64, rounded to fp32 where the kernels store, with unsorted ragged lengths.
The checker must pass on it in both precision modes on both paths, and must flag each of a set of kernel-style mistakes at the
stage (and step) where it was made.  Also: the GPU case list takes the path each case names and covers the edges of the cluster
kernel, through the library's layout query (host arithmetic, no device needed).
"""
import os

import pytest
import torch

import bilstm_check as C

PATHS = [('fp32', True, 1, 1), ('bf16', True, 1, 1), ('fp32', False, 3, 2), ('bf16', False, 3, 2)]
FORWARD = {'xp', 'bsum', 'gates', 'c', 'h', 'frozen', 'zero_start', 'out', 'out_pad'}
BACKWARD = {'dg', 'dg_frozen', 'dW_ih', 'dW_hh', 'db_ih', 'db_hh', 'dx', 'dx_pad'}


def _run(precision='fp32', persist=True, split=1, split_b=1, fault=None):
    s = C.synthetic(precision=precision, persist=persist, split=split, split_b=split_b, fault=fault)
    return s, C.check_synthetic(s, precision, persist, split, split_b)


@pytest.mark.parametrize('precision,persist,split,split_b', PATHS)
def test_checker_passes_on_a_consistent_trajectory(precision, persist, split, split_b):
    s, rep = _run(precision, persist, split, split_b)
    assert rep.failures() == {}, '\n'.join(rep.lines())
    assert set(rep.worst) == FORWARD | BACKWARD | ({'xproj'} if persist else set())
    lens = s['lengths']
    assert not bool((lens[1:] <= lens[:-1]).all()) and int(lens.min()) == 1 and int(lens.max()) == s['v']['gates'].shape[1]


def _flags(rep, stage, step=None, only=None, carried=False):
    """flagged at `stage` (at `step` alone when given); only: the stages allowed to fail.  carried: the mistake also changed the
    d c carry the reference scans itself, so the steps after it in the backward sweep (j < step) may fail as well"""
    bad = rep.failures()
    assert stage in bad, ('not flagged', stage, bad)
    if step is not None:
        assert (max(bad[stage]) if carried else bad[stage]) == (step if carried else [step]), (stage, step, bad)
    assert set(bad) <= (only or {stage}), bad


@pytest.mark.parametrize('persist', (True, False))
def test_moved_gate_is_flagged(persist):
    """one gate element of the reverse direction 4x its bound off; the cell goes on from it, as a kernel's would"""
    _, rep = _run(persist=persist, fault=('gate', 1, 7, 6, 3 * 16 + 2))
    _flags(rep, 'gates', 7)


@pytest.mark.parametrize('precision', ('fp32', 'bf16'))
def test_dropped_recurrent_dh_is_flagged(precision):
    """step 5 of the forward direction took no W_hh^T . dg_6 (dh_rec never refilled)"""
    _, rep = _run(precision, fault=('dh_rec', 0, 5))
    _flags(rep, 'dg', 5, carried=True)


def test_lost_dc_carry_is_flagged():
    _, rep = _run(fault=('dc', 1, 6))
    _flags(rep, 'dg', 6, carried=True)


def test_reverse_direction_from_a_nonzero_state_is_flagged():
    """utterance 3's reverse direction starts from a nonzero state instead of zeros at its own last token"""
    _, rep = _run(fault=('rev_start', 3))
    _flags(rep, 'zero_start')


def test_nonzero_output_at_a_frozen_position_is_flagged():
    """utterance 1 has length 1: forward step 4 is frozen"""
    _, rep = _run(fault=('out_pad', 0, 4, 1))
    _flags(rep, 'out_pad', 4)


def test_nonzero_dg_at_a_frozen_step_is_flagged():
    """a frozen step's gate gradient leaks into the closing products as well: dx is then nonzero at that padded position"""
    _, rep = _run(fault=('dg_frozen', 0, 4, 1))
    _flags(rep, 'dg_frozen', 4, only={'dg_frozen', 'dx_pad'})


@pytest.mark.parametrize('name,stage', [('w_hh', 'dW_hh'), ('w_ih_reverse', 'dW_ih'), ('b_hh_reverse', 'db_hh')])
def test_one_parameter_gradient_element_off_is_flagged(name, stage):
    s, _ = _run()
    d = int(name.endswith('_reverse'))
    base = name.replace('_reverse', '')
    bound = [b for n, dd, _, b in C.closing_products(s['v'], s['prm'], 'fp32') if n == base and dd == d][0]
    idx = (5, 3) if bound.dim() == 2 else (5,)
    s['grads'][name][idx] += float(4 * bound[idx] + 4 * 2.0 ** -24 * s['grads'][name][idx].abs())
    _flags(C.check_synthetic(s), stage, 0)


def test_prefill_not_accumulated_is_flagged():
    """dW_hh overwritten instead of accumulated onto its prefill"""
    s, _ = _run()
    s['grads']['w_hh'] -= s['prefill']['w_hh']
    _flags(C.check_synthetic(s), 'dW_hh', 0)


def _layout(B, L, E, H, chain=False):
    old = os.environ.pop('B200TTS_BILSTM_CHAIN', None)
    if chain:
        os.environ['B200TTS_BILSTM_CHAIN'] = '1'
    try:
        return C.layout(B, L, E, H)
    finally:
        os.environ.pop('B200TTS_BILSTM_CHAIN', None)
        if old is not None:
            os.environ['B200TTS_BILSTM_CHAIN'] = old


@pytest.fixture(scope='module')
def lib():
    from multilingual_text_to_speech_b200 import _lib
    return _lib.load()


def test_gpu_cases_take_their_path_and_cover_the_edges(lib):
    cluster_sizes = set()
    for B, L, E, H, lengths, path in C.GPU_CASES:
        lay = _layout(B, L, E, H)
        assert lay['persist'] == (path == 'persist'), (B, L, E, H, lay)
        assert not _layout(B, L, E, H, chain=True)['persist']
        if path == 'persist':
            cluster_sizes.add(H // 32)
        lens = C.gpu_lengths(B, L, lengths, seed=B * 131 + L)
        assert int(lens.min()) >= 1 and int(lens.max()) == L
        if B > 1:
            assert int(lens.min()) == 1
    assert {1, 4, 7, 8} <= cluster_sizes
    assert any(B % 8 for B, *_ in C.GPU_CASES) and any(B == 1 for B, *_ in C.GPU_CASES) and any(L == 1 for _, L, *_ in C.GPU_CASES)
    assert {(B, L, E, H) for B, L, E, H, *_ in C.GPU_CASES} >= {(16, 180, 512, 256), (64, 180, 512, 256), (64, 180, 256, 128)}
    # unsorted lengths: some group of 8 ends far earlier than a neighbour, in a case the persistent kernel runs
    unsorted = [c for c in C.GPU_CASES if c[4] == 'unsorted']
    assert unsorted and unsorted[0][5] == 'persist'
    B, L = unsorted[0][:2]
    lens = C.gpu_lengths(B, L, 'unsorted', seed=B * 131 + L)
    gmax = [int(lens[q:q + 8].max()) for q in range(0, B, 8)]
    assert any(b <= L // 6 and a == L for a, b in zip(gmax[1:], gmax)), gmax
    assert not bool((lens[1:] <= lens[:-1]).all())


def test_layout_query_matches_the_buffer_sizes(lib):
    """the views lie inside the buffers the size queries give, in the documented order, and a rejected shape gives 0"""
    import ctypes
    from multilingual_text_to_speech_b200 import _lib
    for B, L, E, H, *_ in C.GPU_CASES:
        lay = _layout(B, L, E, H)
        sh = ctypes.byref(_lib.BiLSTMShape(B, L, E, H))
        saved, ws = lib.b200tts_bilstm_saved_bytes(sh), lib.b200tts_bilstm_workspace_bytes(sh)
        sizes = {'xp': 2 * L * B * E, 'gates': 2 * L * B * 4 * H, 'hs': 2 * (L + 1) * B * H, 'cs': 2 * (L + 1) * B * H, 'bsum': 8 * H}
        order = ['xp', 'gates', 'hs', 'cs', 'bsum']
        for a, b in zip(order, order[1:]):
            assert lay[a] + 4 * sizes[a] <= lay[b]
        assert lay['bsum'] + 4 * sizes['bsum'] <= saved
        assert lay['dg'] + 4 * 2 * L * B * 4 * H <= lay['dxp'] and lay['dxp'] + 4 * 2 * L * B * E <= ws
        assert 1 <= lay['split'] <= 8 and 1 <= lay['split_b'] <= 8
    out = (ctypes.c_size_t * 10)()
    assert lib.b200tts_debug_bilstm_layout(ctypes.byref(_lib.BiLSTMShape(0, 5, 8, 32)), out, 10) == 0
    assert lib.b200tts_debug_bilstm_layout(ctypes.byref(_lib.BiLSTMShape(4, 5, 8, 32)), out, 3) == 3


def test_synthetic_lengths_are_unsorted():
    s = C.synthetic()
    assert sorted(s['lengths'].tolist(), reverse=True) != s['lengths'].tolist()
    assert torch.equal(C.valid_steps(s['lengths'], 11, 'cpu')[0].sum(0), s['lengths'])
