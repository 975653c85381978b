"""Several mel frames per decoder step (hp.outputs_per_step = r) without a GPU: the parameter surface, the r-frames oracle tied back to
the reference-pinned r = 1 oracle, and the step shape the library derives from a frame count."""
import ctypes
import json

import pytest
import torch

import decoder_cases as DC
import forward_attention_oracle as FA
import outputs_per_step_oracle as R
from oracle import tacotron_oracle as O


def test_default_is_one_and_reference_configs_load_without_it(tmp_path):
    """The reference's JSON files have no outputs_per_step key: a file of the reference's keys (each named configuration, which restates
    one of them) loads as r = 1."""
    from multilingual_text_to_speech_b200 import configs
    from multilingual_text_to_speech_b200.params.params import Params as hp
    hp.reset()
    assert hp.outputs_per_step == 1
    for name, overlay in configs.CONFIGS.items():
        path = tmp_path / f'{name}.json'
        path.write_text(json.dumps(overlay))
        hp.outputs_per_step = 3
        hp.reset()
        hp.load(str(path))
        assert hp.outputs_per_step == 1, name
    hp.reset()


def _model(r, **kw):
    from multilingual_text_to_speech_b200.params.params import Params as hp
    from multilingual_text_to_speech_b200.modules.tacotron2 import Tacotron
    hp.reset()
    for k, v in kw.items():
        setattr(hp, k, v)
    hp.outputs_per_step = r
    try:
        torch.manual_seed(0)
        return Tacotron()
    finally:
        hp.reset()


@pytest.mark.parametrize('r', [2, 3])
def test_projection_shapes_and_state_dict(r):
    base, model = _model(1), _model(r)
    dec = model._decoder
    DM = dec._frame_prediction.weight.shape[1]
    assert tuple(dec._frame_prediction.weight.shape) == (r * 80, DM)
    assert tuple(dec._frame_prediction.bias.shape) == (r * 80,)
    assert tuple(dec._stop_prediction.weight.shape) == (r, DM)
    assert tuple(dec._stop_prediction.bias.shape) == (r,)
    assert list(model.state_dict().keys()) == list(base.state_dict().keys())
    changed = {k for k, v in model.state_dict().items() if v.shape != base.state_dict()[k].shape}
    assert changed == set(R.PROJECTION_KEYS)
    model.load_state_dict(model.state_dict(), strict=True)


def test_outputs_per_step_below_one_is_rejected():
    with pytest.raises(ValueError):
        _model(0)


def _small(att, tf, kind='zoneout', T=7, seed=0):
    c = DC.full_dim_case(B=3, L=9, T=T, M=24, D=32, P=16, A=8, C=4, K=5, N=6, kind=kind, seed=seed, tf=tf)
    if att == 'forward':
        c.hp.attention_type = 'forward'
        for k in ('_attention._location.weight', '_attention._loc_features.weight',
                  '_decoder._attention._location.weight', '_decoder._attention._loc_features.weight'):
            c.sd.pop(k, None)
    return c


@pytest.mark.parametrize('tf', [1.0, 0.5])
@pytest.mark.parametrize('att', ['location_sensitive', 'forward'])
def test_r1_is_the_reference_pinned_oracle(att, tf):
    c = _small(att, tf)
    _, _, spec, stop, align = R.run(c, 1, with_grad=False)
    sd = {k: v.double() if v.is_floating_point() else v for k, v in c.sd.items()}
    with FA.for_hp(c.hp):
        ref = O.decoder_forward(sd, c.hp, c.memory.double(), O.lengths_to_mask(c.lengths, 9), c.target.double(), None, None,
                                {k: (v if k == 'teacher' else v.double()) for k, v in c.tape.items()}, training=c.training)
    for got, want in zip((spec, stop, align), ref):
        assert torch.equal(got, want)


@pytest.mark.parametrize('tf', [1.0, 0.5])
@pytest.mark.parametrize('att', ['location_sensitive', 'forward'])
@pytest.mark.parametrize('r', [2, 3])
def test_tied_weights_identity(r, att, tf):
    """r copies of the r = 1 projection fed a target with every frame repeated r times: each r = 1 frame comes out r times, the
    alignment is the r = 1 alignment, and the gradients are the r = 1 gradients (projections: summed over the r row blocks) for the
    upstream gradient g_1[t] = sum_j g_r[t*r + j]."""
    c1 = _small(att, tf)
    cr = _small(att, tf)
    cr.sd = R.tie(cr.sd, r)
    cr.target = R.repeat_frames(cr.target, r, 2)
    sd1, mem1, spec1, stop1, align1 = R.run(c1, 1)
    sdr, memr, specr, stopr, alignr = R.run(cr, r)
    T = c1.target.shape[2]
    assert specr.shape == (3, T * r, 6) and alignr.shape == align1.shape
    assert torch.allclose(specr, R.repeat_frames(spec1, r, 1), rtol=1e-12, atol=1e-12)
    assert torch.allclose(stopr, R.repeat_frames(stop1, r, 1), rtol=1e-12, atol=1e-12)
    assert torch.allclose(alignr, align1, rtol=1e-12, atol=1e-12)

    g = torch.Generator().manual_seed(5)
    gs, gt, ga = (torch.randn(t.shape, generator=g, dtype=torch.float64) for t in (specr, stopr, alignr))
    ((specr * gs).sum() + (stopr * gt).sum() + (alignr * ga).sum()).backward()
    g1s = gs.reshape(3, T, r, 6).sum(2)
    g1t = gt.reshape(3, T, r).sum(2)
    ((spec1 * g1s).sum() + (stop1 * g1t).sum() + (align1 * ga).sum()).backward()
    assert torch.allclose(memr.grad, mem1.grad, rtol=1e-9, atol=1e-12)
    for k, p in sd1.items():
        if not torch.is_tensor(p) or p.grad is None or k.startswith('_decoder._prenet.') or k.startswith('_decoder._attention.'):
            continue
        got = sdr[k].grad
        if k in R.PROJECTION_KEYS:
            got = R.block_sum(got, r)
        assert torch.allclose(got, p.grad, rtol=1e-9, atol=1e-12), k


@pytest.mark.parametrize('r', [2, 3])
def test_target_length_not_a_multiple_of_r(r):
    T = 37
    S = R.steps(T, r)
    c = R.untie(_small('location_sensitive', 1.0, T=S), r, T)
    _, _, spec, stop, align = R.run(c, r, with_grad=False)
    assert spec.shape == (3, T, 6) and stop.shape == (3, T) and align.shape == (3, S, 9)


def test_guided_loss_on_the_step_grid_is_the_reference_term_at_r1():
    g = torch.Generator().manual_seed(0)
    align = torch.rand(2, 11, 7, generator=g, dtype=torch.float64)
    il, tl = torch.tensor([7, 5]), torch.tensor([11, 8])
    assert float(R.guided_attention_loss(align, il, tl, 0.2, 1)) == float(O.guided_attention_loss(align, il, tl, 0.2))
    a2 = align[:, :6]
    assert float(R.guided_attention_loss(a2, il, torch.tensor([11, 7]), 0.2, 2)) == \
        float(O.guided_attention_loss(a2, il, torch.tensor([6, 4]), 0.2))


def _shape(T, R_, B=60, L=300):
    from multilingual_text_to_speech_b200 import _lib
    s = _lib.DecoderShape(B, L, T, 288, 1024, 256, 128, 32, 31, 80, _lib.CELL_ZONEOUT, 1, 0.1, 0.1, 0.5)
    s.R = R_
    return s


def test_decoder_path_sees_the_step_shape():
    from multilingual_text_to_speech_b200 import _lib
    lib = _lib.load()
    r2 = lib.b200tts_decoder_path(ctypes.byref(_shape(1200, 2)))
    assert r2 == lib.b200tts_decoder_path(ctypes.byref(_shape(600, 1))) == 0b111111
    assert lib.b200tts_decoder_path(ctypes.byref(_shape(1200, 0))) == lib.b200tts_decoder_path(ctypes.byref(_shape(1200, 1)))
    for q in ('b200tts_decoder_workspace_bytes', 'b200tts_decoder_bwd_workspace_bytes'):
        fn = getattr(lib, q)
        assert fn(ctypes.byref(_shape(1200, 2))) > 0
        assert fn(ctypes.byref(_shape(1199, 2))) == fn(ctypes.byref(_shape(1200, 2)))
    assert lib.b200tts_decoder_path(ctypes.byref(_shape(1200, -1))) == 0
    assert lib.b200tts_decoder_workspace_bytes(ctypes.byref(_shape(1200, -1))) == 0
    assert b'frames per step' in lib.b200tts_last_error()
