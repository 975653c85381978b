"""Every step of the persistent decoder loops against an fp64 step computed from the loop's own saved state (tests/step_check.py),
with the frame edges around them (prenet input and layers, frame split and gather, prenet backward) and every parameter gradient,
at 1, 2 and 3 frames per step; and bit-reproducibility of a bf16 training decode.  Run with -s to see the worst err / bound ratio
of every stage."""
import time

import pytest
import torch

import decoder_cases
import decoder_workspace
import outputs_per_step_oracle as R
import persist_geometry as G
import step_check as S
from multilingual_text_to_speech_b200._lib import DECODER_PARAM_FIELDS

pytestmark = pytest.mark.gpu


def _decode(B, L, T, M, D, kind='zoneout', precision='bf16', seed=0, backward=True, training=True, keep_views=True, r=1):
    """One teacher-forced decode of T steps (ragged lengths including a length-1 utterance, dropout / zoneout masks in training),
    forward and (training) backward with random output gradients.  r > 1: r frames per step with untied random projections and a
    target of T r - 1 frames, so that the last step's last frame is not emitted.  -> dict: shape, views (keep_views), params, cfg,
    lengths, memory, target, align, dalign, dspec, dstop, outputs, grads"""
    from multilingual_text_to_speech_b200 import functional as F, _lib
    c = decoder_cases.full_dim_case(B=B, L=L, T=T, M=M, D=D, kind=kind, seed=seed, ragged=True, training=training)
    if r > 1:
        c = R.untie(c, r, T * r - 1, seed)
    if B > 1:
        c.lengths[-1] = 1
    dev = torch.device('cuda:0')
    cfg, params, memory = decoder_cases._cuda_inputs(c, dev, r)
    lengths, target = c.lengths.to(dev), c.target.to(dev)
    out = {'cfg': cfg, 'params': params, 'lengths': lengths, 'memory': memory, 'target': target, 'dalign': None, 'dspec': None,
           'dstop': None, 'grads': None, 'views': None}
    _lib.set_precision(precision)
    F.PROFILE['keep_ws'] = keep_views
    try:
        spec, stop, align = F.decoder_forward(cfg, memory, target, lengths, params)
        if backward:
            g = torch.Generator(device=dev).manual_seed(99)
            d_spec, d_stop = torch.randn(spec.shape, generator=g, device=dev), torch.randn(stop.shape, generator=g, device=dev)
            d_align = torch.randn(align.shape, generator=g, device=dev)
            ((spec * d_spec).sum() + (stop * d_stop).sum() + (align * d_align).sum()).backward()
            out['dalign'], out['dspec'], out['dstop'] = d_align, d_spec, d_stop
            out['grads'] = dict(zip(DECODER_PARAM_FIELDS, [p.grad for p in params]))
            out['grads']['memory'] = memory.grad
        torch.cuda.synchronize()
        if keep_views:
            out['shape'] = F.PROFILE['last_shape']
            out['views'] = decoder_workspace.last_views()
            if not backward:
                out['views'] = {k: t for k, t in out['views'].items() if k not in decoder_workspace.BWD}
    finally:
        # the views hold what they need; the kept workspaces are released with them
        for key in ('keep_ws', 'last_ws', 'last_bws', 'last_shape'):
            F.PROFILE.pop(key, None)
        _lib.set_precision('fp32')
    out['align'] = align.detach()
    out['outputs'] = (spec.detach(), stop.detach(), align.detach())
    return out


def _mode(shape, precision):
    """The rounding model of the decode: one mode, or (forward, generator reverse, attention reverse) for a training step whose plan
    runs only the generator reverse loop persistent (step_check.modes_of)"""
    import ctypes
    from multilingual_text_to_speech_b200 import _lib
    if precision == 'fp32':
        return 'fp32'
    bits = _lib.load().b200tts_decoder_path(ctypes.byref(shape))
    if not shape.training:          # evaluation: the forward loops only
        bits &= 0b11
    return G.mode_of(bits)


def _mode_of(dims):
    from multilingual_text_to_speech_b200 import _lib
    B, L, T, M, D = dims
    return _mode(_lib.DecoderShape(B, L, T, M, D, 256, 128, 32, 31, 80, _lib.CELL_ZONEOUT, 1, 0.1, 0.1, 0.5), 'bf16')


# every stage a training step reports in every mode; persist adds the checks of its bf16 operand rows and histories
TRAIN_STAGES = {'ga', 'c_att', 'h_att', 'q', 'align', 'align_pad', 'ctx', 'cum', 'gg', 'c_gen', 'h_gen', 'fs', 'xtm', 'p0', 'p1', 'spec',
                'stop', 'dfs', 'dhgd', 'dctxs', 'dgg', 'dga', 'dctxt', 'dq', 'dmemT', 'dp1', 'dp0', 'memory'} | set(DECODER_PARAM_FIELDS)


def _step_check(B, L, T, M, D, kind='zoneout', precision='bf16', expect_mode=None, training=True, key=None, r=1):
    """key: the loop geometry key (persist_geometry.py) the shape must still have.  T: decoder steps (of r frames)."""
    if key is not None:
        assert G.key_of(B, L, M, D, training) == key, (G.key_of(B, L, M, D, training), key)
    t0 = time.perf_counter()
    res = _decode(B, L, T, M, D, kind, precision, backward=training, training=training, r=r)
    mode = _mode(res['shape'], precision)
    if expect_mode:
        assert mode == expect_mode, (mode, expect_mode)
    assert res['shape'].R == r and res['views']['fs'].shape[0] == T, (res['shape'].R, tuple(res['views']['fs'].shape))
    v, cfg = res['views'], res['cfg']
    prm = {f: p.detach() for f, p in zip(DECODER_PARAM_FIELDS, res['params'])}
    scfg = S.Config(cfg.cell_kind, cfg.training, cfg.rate_h, cfg.rate_c, cfg.prenet_rate)
    memory = res['memory'].detach()
    spec, stop, _ = res['outputs']
    t1 = time.perf_counter()
    if training:
        aux = {'dalign': res['dalign'], 'grads': res['grads'], 'target': res['target'], 'spec': spec, 'stop': stop,
               'dspec': res['dspec'], 'dstop': res['dstop']}
        rep = S.check_all(v, prm, cfg.masks, scfg, res['lengths'], memory, res['align'], aux, mode)
        stages = {s.split('[')[0] for s in rep.worst}
        assert TRAIN_STAGES <= stages, TRAIN_STAGES - stages
    else:
        rep = S.check_forward(v, prm, cfg.masks, scfg, res['lengths'], memory, res['align'], mode)
        S.check_frames_forward(v, prm, cfg.masks, cfg.prenet_rate, res['target'], spec, stop, mode, rep)
        assert {'xtm', 'p0', 'p1', 'spec', 'stop'} <= set(rep.worst)
    title = f'[B{B} L{L} T{T} r{r} M{M} D{D} {kind} {"train" if training else "eval"} {precision} {mode}] '
    print()
    print('\n'.join(rep.lines(title)))
    print(f'{title}key {key}: worst err/bound {rep.max_ratio():.3e} over {len(rep.worst)} stages, decode {t1 - t0:.1f} s, '
          f'check {time.perf_counter() - t1:.1f} s')
    assert rep.failures() == {}, (title, rep.failures())
    return rep


@pytest.mark.parametrize('shape', S.GPU_SHAPES, ids=lambda s: 'B{}_L{}_T{}_M{}_D{}'.format(*s))
@pytest.mark.parametrize('kind', ('zoneout', 'dropout'))
def test_persistent_loop_steps_within_bounds(shape, kind):
    _step_check(*shape, kind=kind, expect_mode='persist')


@pytest.mark.parametrize('kind', ('zoneout', 'dropout'))
def test_persistent_forward_loop_steps_within_bounds_eval(kind):
    """evaluation mode (no keep masks; zoneout blends with the expected keep rate) on the persistent forward loops"""
    _step_check(16, 77, 12, 288, 1024, kind=kind, expect_mode='persist', training=False)


def _case_id(c):
    B, L, T, M, D, training = c
    return f'B{B}_L{L}_T{T}_M{M}_D{D}_{"train" if training else "eval"}'


@pytest.mark.parametrize('case', sorted(G.REPRESENTATIVES), ids=_case_id)
def test_every_loop_geometry_steps_within_bounds(case):
    """One representative per geometry key the plan can produce (persist_geometry.py): evaluation decodes through check_forward, training
    steps forward and backward through check_all, each recurrence under the rounding model of the loop that ran it."""
    B, L, T, M, D, training = case
    key = G.REPRESENTATIVES[case]
    kind = ('zoneout', 'dropout')[sorted(G.REPRESENTATIVES).index(case) % 2]
    _step_check(B, L, T, M, D, kind, expect_mode=G.mode_of(key[1]), training=bool(training), key=key)


@pytest.mark.parametrize('case', sorted(G.PAST_LIMITS), ids=_case_id)
def test_steps_past_the_loop_limits_within_bounds(case):
    B, L, T, M, D, training = case
    _step_check(B, L, T, M, D, 'zoneout', expect_mode=G.mode_of(G.PAST_LIMITS[case]), training=bool(training))


def test_alignment_sized_eval_decode_steps_within_bounds():
    B, L, T, M, D, training = G.ALIGNMENT_SIZED
    key = G.key_of(B, L, M, D, training)
    assert key in G.REPRESENTATIVES.values(), key
    _step_check(B, L, T, M, D, 'zoneout', expect_mode='persist', training=False, key=key)


def test_persistent_loop_steps_within_bounds_benchmark_shape():
    """generated_training dims, B = 60, L = 180, T = 900, zoneout, train, forward and backward"""
    _step_check(60, 180, 900, 288, 1024, 'zoneout', expect_mode='persist')


def test_step_checker_on_the_fp32_per_step_chains():
    _step_check(8, 40, 12, 288, 1024, 'zoneout', precision='fp32', expect_mode='fp32')


def test_step_checker_on_the_fp32_per_step_chains_two_attention_chunks():
    """L = 300: the decoder's per-step attention backward runs each utterance's positions in two chunks (LC = 172)"""
    from multilingual_text_to_speech_b200 import _lib
    LC = _lib.load().b200tts_debug_attention_backward_chunk(300, 288, 128, 32, 31)
    assert -(-300 // LC) == 2, LC
    _step_check(8, 300, 6, 288, 1024, 'zoneout', precision='fp32', expect_mode='fp32')


def test_step_checker_on_the_bf16_per_step_chains_d1280():
    _step_check(8, 60, 10, 288, 1280, 'zoneout', expect_mode='chain_bf16')


# ---- several frames per step (hp.outputs_per_step): T r - 1 frames, the last step's last frame not emitted ----

@pytest.mark.parametrize('r', (2, 3))
@pytest.mark.parametrize('kind', ('zoneout', 'dropout'))
@pytest.mark.parametrize('training', (True, False), ids=('train', 'eval'))
def test_persistent_loop_steps_within_bounds_frames_per_step(r, kind, training):
    _step_check(33, 47, 8, 288, 1024, kind, expect_mode='persist', training=training, r=r)


def test_step_checker_on_the_fp32_per_step_chains_r2():
    _step_check(8, 40, 12, 288, 1024, 'zoneout', precision='fp32', expect_mode='fp32', r=2)


def test_step_checker_on_the_bf16_per_step_chains_d1280_r3():
    _step_check(8, 60, 10, 288, 1280, 'dropout', expect_mode='chain_bf16', r=3)


@pytest.mark.parametrize('shape', [(60, 180, 900, 288, 1024), (64, 300, 400, 288, 1024)], ids=('benchmark', 'B64_L300'))
def test_bf16_training_decode_is_bit_reproducible(shape):
    """Two identical training decodes, forward + backward: outputs, every parameter gradient and d memory bitwise equal."""
    runs = []
    for _ in range(2):
        r = _decode(*shape, kind='zoneout', keep_views=False)
        assert _mode_of(shape) == 'persist'
        g = r['grads']
        runs.append([t.clone() for t in r['outputs']] + [g['memory'].clone()] + [g[f].clone() for f in DECODER_PARAM_FIELDS])
        del r, g
        torch.cuda.empty_cache()
    names = ['spec', 'stop', 'align', 'd_memory'] + ['d_' + f for f, _ in decoder_cases.PARAM_KEYS]
    for name, a, b in zip(names, *runs):
        assert torch.equal(a, b), (name, float((a - b).abs().max()), int((a != b).sum()))
