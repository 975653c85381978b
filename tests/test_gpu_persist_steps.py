"""Every step of the persistent decoder loops against an fp64 step computed from the loop's own saved state (tests/step_check.py),
and bit-reproducibility of a bf16 training decode.  Run with -s to see the worst err / bound ratio of every stage."""
import pytest
import torch

import decoder_cases
import decoder_workspace
import step_check as S
from multilingual_text_to_speech_b200._lib import DECODER_PARAM_FIELDS

pytestmark = pytest.mark.gpu


def _decode(B, L, T, M, D, kind='zoneout', precision='bf16', seed=0, backward=True, training=True, keep_views=True):
    """One teacher-forced decode (ragged lengths including a length-1 utterance, dropout / zoneout masks in training), forward and
    (training) backward with random output gradients.  -> dict: shape, views (keep_views), params, cfg, lengths, memory, align, dalign,
    outputs, grads"""
    from multilingual_text_to_speech_b200 import functional as F, _lib
    c = decoder_cases.full_dim_case(B=B, L=L, T=T, M=M, D=D, kind=kind, seed=seed, ragged=True, training=training)
    if B > 1:
        c.lengths[-1] = 1
    dev = torch.device('cuda:0')
    cfg, params, memory = decoder_cases._cuda_inputs(c, dev)
    lengths, target = c.lengths.to(dev), c.target.to(dev)
    out = {'cfg': cfg, 'params': params, 'lengths': lengths, 'memory': memory, 'dalign': None, 'grads': None, 'views': None}
    _lib.set_precision(precision)
    F.PROFILE['keep_ws'] = keep_views
    try:
        spec, stop, align = F.decoder_forward(cfg, memory, target, lengths, params)
        if backward:
            g = torch.Generator(device=dev).manual_seed(99)
            d_spec, d_stop = torch.randn(spec.shape, generator=g, device=dev), torch.randn(stop.shape, generator=g, device=dev)
            d_align = torch.randn(align.shape, generator=g, device=dev)
            ((spec * d_spec).sum() + (stop * d_stop).sum() + (align * d_align).sum()).backward()
            out['dalign'] = d_align
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
    import ctypes
    from multilingual_text_to_speech_b200 import _lib
    if precision == 'fp32':
        return 'fp32'
    bits = _lib.load().b200tts_decoder_path(ctypes.byref(shape))
    if not shape.training:          # evaluation: the forward loops only
        bits &= 0b11
        assert bits in (0, 0b11), bin(bits)
    else:
        assert bits in (0, 0b111111), bin(bits)
    return 'persist' if bits else 'chain_bf16'


def _mode_of(dims):
    from multilingual_text_to_speech_b200 import _lib
    B, L, T, M, D = dims
    return _mode(_lib.DecoderShape(B, L, T, M, D, 256, 128, 32, 31, 80, _lib.CELL_ZONEOUT, 1, 0.1, 0.1, 0.5), 'bf16')


def _step_check(B, L, T, M, D, kind='zoneout', precision='bf16', expect_mode=None, training=True):
    r = _decode(B, L, T, M, D, kind, precision, backward=training, training=training)
    mode = _mode(r['shape'], precision)
    if expect_mode:
        assert mode == expect_mode, (mode, expect_mode)
    v, cfg = r['views'], r['cfg']
    prm = {f: p.detach() for f, p in zip(DECODER_PARAM_FIELDS, r['params'])}
    scfg = S.Config(cfg.cell_kind, cfg.training, cfg.rate_h, cfg.rate_c)
    memory = r['memory'].detach()
    if training:
        rep = S.check_all(v, prm, cfg.masks, scfg, r['lengths'], memory, r['align'], {'dalign': r['dalign'], 'grads': r['grads']}, mode)
    else:
        rep = S.check_forward(v, prm, cfg.masks, scfg, r['lengths'], memory, r['align'], mode)
    title = f'[B{B} L{L} T{T} M{M} D{D} {kind} {"train" if training else "eval"} {precision} {mode}] '
    print()
    print('\n'.join(rep.lines(title)))
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


def test_persistent_loop_steps_within_bounds_benchmark_shape():
    """generated_training dims, B = 60, L = 180, T = 900, zoneout, train, forward and backward"""
    _step_check(60, 180, 900, 288, 1024, 'zoneout', expect_mode='persist')


def test_step_checker_on_the_fp32_per_step_chains():
    _step_check(8, 40, 12, 288, 1024, 'zoneout', precision='fp32', expect_mode='fp32')


def test_step_checker_on_the_bf16_per_step_chains_d1280():
    _step_check(8, 60, 10, 288, 1280, 'zoneout', expect_mode='chain_bf16')


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
