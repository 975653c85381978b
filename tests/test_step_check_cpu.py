"""The step-local fp64 checker (tests/step_check.py) on synthetic workspaces, without a GPU.

A synthetic workspace is an fp64 trajectory with the kernels' rounding points, stored in the decoder's view layout.  The checker
must pass on it in every rounding mode, cell kind and train / eval, and must flag each of a set of small kernel-style mistakes at
the step and stage where it was made.  Also: the GPU step-check shape list covers the edges the wgmma loops accept.
"""
import ctypes

import pytest
import torch

import step_check as S


def _synthetic(**kw):
    return S.synthetic(**kw)


def _check(v, prm, masks, cfg, lengths, memory, align, aux, mode='persist'):
    return S.check_all(v, prm, masks, cfg, lengths, memory, align, aux, mode)


@pytest.mark.parametrize('mode', S.MODES)
@pytest.mark.parametrize('kind', (0, 1))
@pytest.mark.parametrize('training', (True, False))
def test_checker_passes_on_a_consistent_trajectory(mode, kind, training):
    args = _synthetic(kind=kind, training=training, mode=mode)
    rep = _check(*args, mode=mode)
    assert rep.failures() == {}, '\n'.join(rep.lines())
    expected = {'ga', 'c_att', 'h_att', 'q', 'align', 'align_pad', 'ctx', 'cum', 'gg', 'c_gen', 'h_gen', 'fs', 'dgg', 'dga',
                'dctxt', 'dq', 'dmemT', 'gen_w_hh', 'gen_w_ih', 'att_w_hh', 'att_w_ih[0:32]', 'att_w_ih[32:96]', 'frame_w', 'stop_w',
                'attn_query', 'attn_memory', 'gen_b_ih', 'gen_b_hh', 'att_b_ih', 'att_b_hh', 'attn_bias', 'frame_b', 'stop_b', 'memory'}
    if mode == 'persist':
        expected |= {'aib_rn', 'hgb_rn', 'aib_row0', 'hgb_row0', 'dggb_rn', 'dgab_rn'}
    assert set(rep.worst) == expected


def _flags(rep, stage, step):
    """the mutation is flagged at (stage, step) and nowhere else in that stage"""
    bad = rep.failures()
    assert stage in bad, ('not flagged', stage, step, bad)
    assert bad[stage] == [step], (stage, step, bad)


def test_stale_h_operand_is_flagged():
    """the generator product of step i used one utterance's h row of step i-1"""
    v, prm, masks, cfg, lengths, memory, align, aux = args = _synthetic()
    i, b = 3, 5
    h = S.gen_operand(v, i, i + 1, 'persist').clone()
    h[0, b] = S.gen_operand(v, i - 1, i, 'persist')[0, b]
    z, _ = S.gen_preact(v, prm, S.att_operand(v, i + 1, i + 2, 'persist'), h, 'persist')
    v['gg'][i, b] = S.activate(z, 'persist')[0][0, b].float()
    _flags(_check(*args), 'gg', i)


def test_dropped_k_block_is_flagged():
    """one 64-column k-block (the first h block) missing from one gate row of the attention-LSTM product"""
    v, prm, masks, cfg, lengths, memory, align, aux = args = _synthetic()
    i, b, row = 2, 3, 70
    a = S.att_operand(v, i, i + 1, 'persist').clone()
    a[..., :64] = 0
    z, _ = S.att_preact(v, prm, a, i, i + 1, 'persist')
    v['ga'][i, b, row] = S.activate(z, 'persist')[0][0, b, row].float()
    _flags(_check(*args), 'ga', i)


def test_ignored_keep_mask_bit_is_flagged():
    i = 2
    _, _, masks, *_ = _synthetic()
    b, u = [int(x) for x in torch.nonzero(masks['att_h'][i] == 0)[0]]
    km = {k: t.clone() for k, t in masks.items()}
    km['att_h'][i, b, u] = 1
    args = _synthetic(kernel_masks=km)
    _flags(_check(*args), 'h_att', i)


def test_swapped_batch_halves_in_the_context_are_flagged():
    """utterances b and b + 32 (the two batch halves of the loops) exchanged in one step's context"""
    v, prm, masks, cfg, lengths, memory, align, aux = args = _synthetic()
    i, b = 4, 0
    M = memory.shape[2]
    row = v['ai'][i + 1, :, :M]
    row[[b, b + 32]] = row[[b + 32, b]].clone()
    _flags(_check(*args), 'ctx', i)


@pytest.mark.parametrize('mode', S.MODES)
def test_alignment_weight_off_by_one_percent_is_flagged(mode):
    """With accurate tanhf the weight's own stage sees 1 %.  The persistent loops' energies use tanh.approx, whose documented worst case
    (2^-11 relative on each of the A terms) admits a few percent on a weight: there the context and the cumulative weights, which are
    checked against the weights the kernel wrote, flag it."""
    v, prm, masks, cfg, lengths, memory, align, aux = args = _synthetic(mode=mode)
    i, b = 3, 0
    align[b, i, int(align[b, i].argmax())] *= 1.01
    rep = _check(*args, mode=mode)
    for stage in (('ctx', 'cum') if mode == 'persist' else ('align', 'ctx', 'cum')):
        _flags(rep, stage, i)


def test_gate_gradient_row_from_the_wrong_step_is_flagged():
    v, prm, masks, cfg, lengths, memory, align, aux = args = _synthetic()
    i, b = 2, 7
    v['dgg'][i, b] = v['dgg'][i + 1, b]
    _flags(_check(*args), 'dgg', i)


def test_query_gradient_row_from_the_wrong_step_is_flagged():
    v, prm, masks, cfg, lengths, memory, align, aux = args = _synthetic()
    i, b = 2, 4
    v['dq'][i, b] = v['dq'][i + 1, b]
    bad = _check(*args).failures()
    assert bad.get('dq') == [i], bad


@pytest.mark.parametrize('mode', S.MODES)
def test_lost_dcum_carry_is_flagged(mode):
    """the attention reverse loop loses the d cum carry on entry to step i: its query gradient is the first one off"""
    i = 3
    args = _synthetic(lose_dcum_carry_at=i, mode=mode)
    bad = _check(*args, mode=mode).failures()
    assert 'dq' in bad and max(bad['dq']) == i, bad


def test_recurrent_context_gradient_from_the_wrong_step_is_flagged():
    """d context total of step i built from the gate gradients of step i + 2 instead of i + 1"""
    v, prm, masks, cfg, lengths, memory, align, aux = args = _synthetic()
    i, P = 2, v['p1'].shape[2]
    W = S.rn(prm['att_w_ih'][:, P:])
    v['dctxt'][i] = (v['dctxs'][i].double() + v['dgab'][i + 2].double() @ W).float()
    _flags(_check(*args), 'dctxt', i)


@pytest.mark.parametrize('wiring', ('rows 1..T for gen_w_hh', 'ctx columns for att_w_hh'))
def test_weight_gradient_operand_wiring_is_flagged(wiring):
    """an in-place bf16 operand read one row block off, or at the wrong column offset into aib"""
    v, prm, masks, cfg, lengths, memory, align, aux = args = _synthetic()
    T, B, D = v['dggb'].shape[0], v['dggb'].shape[1], v['dggb'].shape[2] // 4
    flat = lambda x: x.double().reshape(T * B, -1)     # noqa: E731
    if wiring.startswith('rows'):
        aux['grads']['gen_w_hh'] = (flat(v['dggb']).t() @ flat(v['hgb'][1:, :, :D])).float()
        _flags(_check(*args), 'gen_w_hh', 0)
    else:
        aux['grads']['att_w_hh'] = (flat(v['dgab']).t() @ flat(v['aib'][:T, :, D:2 * D])).float()
        _flags(_check(*args), 'att_w_hh', 0)


def test_cumulative_weights_not_updated_at_the_last_step_are_flagged():
    v, prm, masks, cfg, lengths, memory, align, aux = args = _synthetic()
    T = v['ga'].shape[0]
    v['cum'][T] = v['cum'][T - 1]
    _flags(_check(*args), 'cum', T - 1)


def test_gpu_shape_list_covers_the_accepted_edges():
    """tests/test_gpu_persist_steps.py runs the step checker on S.GPU_SHAPES: every one must run on all three wgmma loops, and
    together they must include B = 1, an odd B, B = 64, L = 1 and 15 (mod 16), L = 300, M = 512, a D other than 1024 (the path
    query accepts D = 512, not 960, 1152 or 1280 for a training step) and T = 1, 2."""
    import __graft_entry__ as entry
    from multilingual_text_to_speech_b200 import _lib
    entry.build()
    lib = _lib.load()

    def path(B, L, T, M, D, kind=1):
        s = _lib.DecoderShape(B, L, T, M, D, 256, 128, 32, 31, 80, kind, 1, 0.1, 0.1, 0.5)
        return lib.b200tts_decoder_path(ctypes.byref(s))
    for sh in S.GPU_SHAPES:
        B, L, T, M, D = sh
        for kind in (0, 1):
            assert path(B, L, T, M, D, kind) == 0b111111, (sh, kind, bin(path(B, L, T, M, D, kind)))
    Bs, Ls, Ts, Ms, Ds = zip(*S.GPU_SHAPES)
    assert 1 in Bs and 64 in Bs and any(b % 2 for b in Bs if b > 1)
    assert any(L % 16 == 1 for L in Ls) and any(L % 16 == 15 for L in Ls) and 300 in Ls
    assert 512 in Ms and 1 in Ts and 2 in Ts
    assert path(8, 100, 6, 288, 512) == 0b111111 and 512 in Ds
    for D in (960, 1152, 1280):
        assert path(8, 100, 6, 288, D) != 0b111111, D


def test_view_offsets_follow_the_library_layout():
    """the views are where the workspace sizes say they can be: every view inside its workspace, the forward views disjoint"""
    import __graft_entry__ as entry
    import decoder_workspace as W
    from multilingual_text_to_speech_b200 import _lib
    entry.build()
    lib = _lib.load()
    for B, L, T, M, D in S.GPU_SHAPES + [(60, 180, 900, 288, 1024)]:
        s = _lib.DecoderShape(B, L, T, M, D, 256, 128, 32, 31, 80, 1, 1, 0.1, 0.1, 0.5)
        off = W.offsets(s)
        shapes = W.view_shapes(s, off['Kp_att'], off['Kp_gen'])
        assert off['Kp_att'] % 64 == 0 and off['Kp_att'] >= D + M and off['Kp_gen'] % 64 == 0 and off['Kp_gen'] >= D
        for group, total in ((W.FWD, lib.b200tts_decoder_workspace_bytes(ctypes.byref(s))),
                             (W.BWD, lib.b200tts_decoder_bwd_workspace_bytes(ctypes.byref(s)))):
            spans = []
            for name in group:
                dtype, dims = shapes[name]
                n = torch.Size(dims).numel() * (torch.finfo(dtype).bits // 8)
                assert off[name] + n <= total, (name, off[name], n, total)
                spans.append((off[name], off[name] + n, name))
            spans.sort()
            for (a0, a1, na), (b0, b1, nb) in zip(spans, spans[1:]):
                assert a1 <= b0, (na, nb)
