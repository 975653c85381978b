"""The step-local fp64 checker (tests/step_check.py) on synthetic workspaces, without a GPU.

A synthetic workspace is an fp64 trajectory with the kernels' rounding points, stored in the decoder's view layout.  The checker
must pass on it in every rounding mode, cell kind and train / eval and at 1, 2 and 3 frames per step, must check every parameter
gradient, and must flag each of a set of small kernel-style mistakes at the step and stage where it was made.  Also: the GPU
step-check shape list covers the edges the wgmma loops accept, and the workspace views follow the library's layout.
"""
import ctypes

import pytest
import torch

import step_check as S


def _synthetic(**kw):
    return S.synthetic(**kw)


def _check(v, prm, masks, cfg, lengths, memory, align, aux, mode='persist'):
    return S.check_all(v, prm, masks, cfg, lengths, memory, align, aux, mode)


def _expected_stages(mode):
    out = {'ga', 'c_att', 'h_att', 'q', 'align', 'align_pad', 'ctx', 'cum', 'gg', 'c_gen', 'h_gen', 'fs', 'dgg', 'dga',
           'dctxt', 'dq', 'dmemT', 'gen_w_hh', 'gen_w_ih', 'att_w_hh', 'att_w_ih[0:32]', 'att_w_ih[32:96]', 'frame_w', 'stop_w',
           'attn_query', 'attn_memory', 'gen_b_ih', 'gen_b_hh', 'att_b_ih', 'att_b_hh', 'attn_bias', 'frame_b', 'stop_b', 'memory',
           'xtm', 'p0', 'p1', 'spec', 'stop', 'dfs', 'dhgd', 'dctxs', 'dp1', 'dp0', 'prenet_w1', 'prenet_b1', 'prenet_w0', 'prenet_b0',
           'attn_energy', 'attn_location', 'attn_loc_features'}
    if mode == 'persist':
        out |= {'aib_rn', 'hgb_rn', 'aib_row0', 'hgb_row0', 'dggb_rn', 'dgab_rn'}
    return out


@pytest.mark.parametrize('mode', S.MODES)
@pytest.mark.parametrize('kind', (0, 1))
@pytest.mark.parametrize('training', (True, False))
def test_checker_passes_on_a_consistent_trajectory(mode, kind, training):
    args = _synthetic(kind=kind, training=training, mode=mode)
    rep = _check(*args, mode=mode)
    assert rep.failures() == {}, '\n'.join(rep.lines())
    assert set(rep.worst) == _expected_stages(mode)


@pytest.mark.parametrize('mode', S.MODES)
@pytest.mark.parametrize('R', (2, 3))
def test_checker_passes_at_several_frames_per_step(mode, R):
    """R frames per step, the last step's last frame not emitted: the views carry S rows, fs / dfs are R (N + 1) wide"""
    v, prm, masks, cfg, lengths, memory, align, aux = args = _synthetic(R=R, mode=mode, T=5)
    N = prm['frame_w'].shape[0] // R
    assert v['fs'].shape == v['dfs'].shape == (5, 34, R * (N + 1)) and v['xtm'].shape == (5, 34, N)
    assert aux['target'].shape[2] == aux['spec'].shape[1] == 5 * R - 1
    rep = _check(*args, mode=mode)
    assert rep.failures() == {}, '\n'.join(rep.lines())
    assert set(rep.worst) == _expected_stages(mode)


@pytest.mark.parametrize('mode', S.MODES)
def test_every_parameter_gradient_has_a_closing_stage(mode):
    """check_all checks each of the decoder's parameter gradients and d memory: a parameter added to the library without a stage
    fails here"""
    from multilingual_text_to_speech_b200._lib import DECODER_PARAM_FIELDS
    assert len(DECODER_PARAM_FIELDS) == 22
    rep = _check(*_synthetic(mode=mode, T=3), mode=mode)
    checked = {stage.split('[')[0] for stage in rep.worst}
    missing = (set(DECODER_PARAM_FIELDS) | {'memory'}) - checked
    assert not missing, missing
    assert {'att_w_ih[0:32]', 'att_w_ih[32:96]'} <= set(rep.worst)      # both column blocks of the one split gradient


def _flags(rep, stage, step):
    """the mutation is flagged at (stage, step) and nowhere else in that stage"""
    bad = rep.failures()
    assert stage in bad, ('not flagged', stage, step, bad)
    assert bad[stage] == [step], (stage, step, bad)


def test_mixed_plan_checks_each_recurrence_under_the_loop_that_ran_it():
    """A training step whose plan runs only the generator reverse loop persistent (forward and attention reverse on the bf16 chains): the
    generator reverse is checked from its bf16 history under the persistent loop's model, everything else under the chains' model."""
    mixed = ('chain_bf16', 'persist', 'chain_bf16')
    v, prm, masks, cfg, lengths, memory, align, aux = args = _synthetic(mode='chain_bf16')
    v['dggb'] = v['dgg'].to(torch.bfloat16)
    rep = _check(*args, mode=mixed)
    assert rep.failures() == {}, '\n'.join(rep.lines())
    assert 'dggb_rn' in rep.worst and not {'aib_rn', 'hgb_rn', 'dgab_rn'} & set(rep.worst)
    i = 3
    v['dggb'][i, 2, 5] = (v['dgg'][i, 2, 5] * 1.01).to(torch.bfloat16)      # the history the next reverse step multiplied is off
    _flags(_check(*args, mode=mixed), 'dggb_rn', i)
    with pytest.raises(AssertionError):                                    # no plan runs the forward loops without the attention reverse loop
        _check(*args, mode=('persist', 'persist', 'chain_bf16'))


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
    """the views are where the workspace sizes say they can be: every view inside its workspace, the views of each workspace
    disjoint, at R = 1, 2 and 3 frames per step with a frame count T that is a multiple of R and one that is not
    (S = ceil(T / R) step rows)"""
    import __graft_entry__ as entry
    import decoder_workspace as W
    from multilingual_text_to_speech_b200 import _lib
    entry.build()
    lib = _lib.load()
    cases = [(B, L, T * R - j, M, D, R) for R in (1, 2, 3) for B, L, T, M, D in S.GPU_SHAPES + [(60, 180, 900, 288, 1024)]
             for j in sorted({0, R - 1})]
    for B, L, T, M, D, R in cases:
        s = _lib.DecoderShape(B, L, T, M, D, 256, 128, 32, 31, 80, 1, 1, 0.1, 0.1, 0.5)
        s.R = R
        off = W.offsets(s)
        shapes = W.view_shapes(s, off['Kp_att'], off['Kp_gen'])
        Sn = -(-T // R)
        assert shapes['ga'][1][0] == Sn and shapes['fs'][1] == shapes['dfs'][1] == (Sn, B, R * 81), (T, R, shapes['fs'])
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


def _only(rep, expected):
    """the checker flags exactly these {stage: [steps]}"""
    bad = rep.failures()
    assert bad == expected, (bad, expected)


def test_teacher_frame_off_by_one_is_flagged():
    """every step i >= 1 fed target frame i R instead of i R - 1: the prenet input is off, everything after it is consistent"""
    T, R = 5, 2
    _only(_check(*_synthetic(R=R, T=T, faults=('teacher_frame',))), {'xtm': list(range(1, T))})


def test_swapped_stop_slots_are_flagged():
    """the two stop logits of one step emitted in the wrong frame order at R = 2"""
    v, prm, masks, cfg, lengths, memory, align, aux = args = _synthetic(R=2, T=5)
    i = 2
    aux['stop'][:, [2 * i, 2 * i + 1]] = aux['stop'][:, [2 * i + 1, 2 * i]].clone()
    _only(_check(*args), {'stop': [i]})


def test_ignored_prenet_keep_bit_is_flagged():
    """the first prenet layer keeps one unit its mask dropped"""
    i = 3
    v, prm, masks, *_ = _synthetic()
    z = v['xtm'][i].double() @ S.rn(prm['prenet_w0']).t() + prm['prenet_b0'].double()
    b, u = [int(x) for x in torch.nonzero((masks['prenet0'][i] == 0) & (z > 0.1))[0]]
    km = {k: t.clone() for k, t in masks.items()}
    km['prenet0'][i, b, u] = 1
    _only(_check(*_synthetic(kernel_masks=km)), {'p0': [i]})


def test_frame_gradient_past_the_last_frame_is_flagged():
    """the gather writes a gradient into the frame slot past T of the last step (R = 2, T = 2 S - 1) instead of 0"""
    T = 5
    _only(_check(*_synthetic(R=2, T=T, faults=('dfs_past_T',))), {'dfs': [T - 1]})


def _attention_fault(mode, drop=None, wloc_transposed=False, min_length=1):
    """aux['grads'] of the attention parameters formed from the synthetic trajectory's own terms with one kernel-style mistake:
    drop(step, field) -> a [B, L] mask of the positions whose terms that field's sum leaves out.  Three steps: the bounds of these
    sums carry the d cum carry's, which widens with every reverse step (step_check.AttentionReverse)."""
    v, prm, masks, cfg, lengths, memory, align, aux = args = _synthetic(mode=mode, L=20, T=3, min_length=min_length)
    terms = S.attention_terms(v, prm, lengths, memory, align, aux['dalign'], mode)
    for field in ('attn_energy', 'attn_location', 'attn_loc_features'):
        kept = terms
        if drop is not None:
            kept = []
            for i, ds, unf, de, t in terms:
                keep = ~drop(i, field)
                kept.append((i, ds * keep[..., None], unf, de * keep, t))
        wloc = prm['attn_location'].reshape(prm['attn_location'].shape[1], -1).t() if wloc_transposed else None
        aux['grads'][field].copy_(S.attention_grads_of_terms(prm, kept, mode, wloc)[field])
    return _check(*args, mode=mode)


@pytest.mark.parametrize('mode', S.MODES)
def test_attention_gradients_of_the_trajectory_pass(mode):
    """the terms the fault tests below edit sum to gradients the checker passes"""
    _only(_attention_fault(mode), {})


@pytest.mark.parametrize('mode', S.MODES)
def test_dropped_partial_position_tile_is_flagged(mode):
    """L = 20, every text 17 to 20 long: positions 16..19 (the last, partial 16-position tile of the post pass) missing from d v
    and d Wcomb"""
    rep = _attention_fault(mode, drop=lambda i, f: (torch.arange(20) >= 16)[None, :].expand(34, 20), min_length=17)
    _only(rep, {'attn_energy': [0], 'attn_location': [0], 'attn_loc_features': [0]})


@pytest.mark.parametrize('mode', S.MODES)
def test_step_missing_from_the_location_gradients_is_flagged(mode):
    """one decoder step's terms missing from d Wcomb (d Wloc and d Wc), d v complete"""
    step = 1
    rep = _attention_fault(mode, drop=lambda i, f: torch.full((34, 20), i == step and f != 'attn_energy'))
    _only(rep, {'attn_location': [0], 'attn_loc_features': [0]})


@pytest.mark.parametrize('mode', S.MODES)
def test_location_feature_gradient_with_transposed_wloc_is_flagged(mode):
    """d Wc = Wloc^T . d Wcomb read with Wloc's two indices exchanged ([C, A] storage order)"""
    _only(_attention_fault(mode, wloc_transposed=True), {'attn_loc_features': [0]})
