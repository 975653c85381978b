"""Module-level forwards of the boundary (SURVEY 8b) against golden vectors of the UNMODIFIED reference classes (CPU, fp32;
tests/golden/make_golden_modules.py -> tests/golden/modules.npz): ZoneoutLSTMCell / DropoutLSTMCell (modules/layers.py:18-47),
Conv1dGenerated / BatchNorm1dGenerated (modules/generated.py:7-96), LocationSensitiveAttention (modules/attention.py:6-86),
forward values and gradients through the library ops.  The cases themselves are in tests/module_cases.py."""
import os
import numpy as np
import pytest
import torch

import module_cases as C
from helpers import assert_close, GOLDEN_DIR

pytestmark = pytest.mark.gpu


@pytest.fixture(scope='module', autouse=True)
def _built():
    import __graft_entry__ as entry
    entry.build()
    assert torch.cuda.is_available()


@pytest.fixture(scope='module')
def golden():
    return np.load(os.path.join(GOLDEN_DIR, 'modules.npz'))


def _check(golden, prefix, result, tol):
    """tol(key) -> (rtol, atol relative to the reference tensor's largest magnitude, absolute atol floor)."""
    for key, t in result.items():
        got, ref, amax = C.unpack_like(golden, prefix, key, t)
        rtol, atol_rel, atol_abs = tol(key)
        assert_close(got, ref, rtol, atol_rel * amax + atol_abs, f'{prefix}.{key}')


def test_zoneout_cell_train_mode_with_masks():
    """Training mode: h = (1 - z) * dropout(h' - h, z) + h with explicit keep masks (reference layers.py:29-30 with F.dropout's mask)."""
    from multilingual_text_to_speech_b200.modules.layers import ZoneoutLSTMCell
    from multilingual_text_to_speech_b200.rng import MaskSource
    torch.manual_seed(4)
    I, H, B, z = 96, 128, 5, 0.1
    cell = ZoneoutLSTMCell(I, H, z, z).train()
    x, h, c = torch.randn(B, I), torch.randn(B, H), torch.randn(B, H)
    mh, mc = (torch.rand(B, H) >= z).float(), (torch.rand(B, H) >= z).float()
    xr, hr, cr = (t.clone().double().requires_grad_(True) for t in (x, h, c))
    w = {k: v.detach().double() for k, v in cell.state_dict().items()}
    g = xr @ w['weight_ih'].t() + w['bias_ih'] + hr @ w['weight_hh'].t() + w['bias_hh']
    i_, f_, g_, o_ = g.chunk(4, 1)
    cn = torch.sigmoid(f_) * cr + torch.sigmoid(i_) * torch.tanh(g_)
    hn = torch.sigmoid(o_) * torch.tanh(cn)
    h1 = (1 - z) * (mh.double() * (hn - hr) / (1 - z)) + hr
    c1 = (1 - z) * (mc.double() * (cn - cr) / (1 - z)) + cr
    cell = cell.cuda()
    xo, ho, co = (t.cuda().requires_grad_(True) for t in (x, h, c))
    MaskSource.use_tape({'cell_h': mh, 'cell_c': mc})
    try:
        h2, c2 = cell(xo, ho, co)
    finally:
        MaskSource.use_tape(None)
    assert_close(h2, h1, 1e-3, 1e-5, 'h'); assert_close(c2, c1, 1e-3, 1e-5, 'c')
    gh, gc = torch.randn(B, H), torch.randn(B, H)
    ((h1 * gh.double()).sum() + (c1 * gc.double()).sum()).backward()
    ((h2 * gh.cuda()).sum() + (c2 * gc.cuda()).sum()).backward()
    for name, a, b in (('dx', xo, xr), ('dh', ho, hr), ('dc', co, cr)):
        assert_close(a.grad, b.grad, 2e-3, 1e-5, name)


@pytest.mark.parametrize('kind', ['zoneout', 'dropout'])
def test_lstm_cells_match_reference_eval_mode(kind, golden):
    from multilingual_text_to_speech_b200.modules.layers import ZoneoutLSTMCell, DropoutLSTMCell
    I, H = 544, 1024
    own = ZoneoutLSTMCell(I, H, 0.1, 0.1) if kind == 'zoneout' else DropoutLSTMCell(I, H, 0.1)
    res = C.lstm_case(kind, own, 'cuda')
    _check(golden, f'lstm_{kind}', res,
           lambda k: (1e-3, 0.0, 1e-5) if k in ('h', 'c') else (2e-3, 0.0, 1e-5) if k in ('dx', 'dh', 'dc') else (2e-3, 1e-4, 0.0))


@pytest.mark.parametrize('train', [True, False])
def test_generated_conv_and_batchnorm_match_reference(train, golden):
    from multilingual_text_to_speech_b200.modules.generated import Conv1dGenerated, BatchNorm1dGenerated
    G, gd, bn, Cin, Cout, k, dil = 3, 6, 4, 8, 12, 3, 2
    oc = Conv1dGenerated(gd, bn, G * Cin, G * Cout, k, padding=0, dilation=dil, groups=G, bias=False)
    ob = BatchNorm1dGenerated(gd, bn, G * Cout, groups=G)
    res = C.conv_case(train, oc, ob, 'cuda')
    assert res['y'].shape[2] == 21                           # un-padded ("valid") convolution, as in the reference
    if not train:
        for key in ('running_mean', 'running_var', 'num_batches_tracked'):
            res.pop(key)
    else:
        assert int(res['num_batches_tracked']) == 1

    def tol(key):
        if key == 'y':
            return 1e-3, 0.0, 1e-5
        if key == 'z':
            return 1e-3, 0.0, 1e-4
        if key in ('running_mean', 'running_var', 'num_batches_tracked'):
            return 1e-3, 0.0, 1e-6
        if key in ('de', 'dx'):
            return 3e-3, 1e-4, 0.0
        return 3e-3, 2e-4, 1e-9
    _check(golden, f'conv_train{int(train)}', res, tol)


def test_attention_module_forward_and_autograd_match_reference(golden):
    """LocationSensitiveAttention.reset + three forward steps (attention.py:23-28, 39-45, 67-86) with gradients through the carried
    cumulative weights, against the reference module."""
    from multilingual_text_to_speech_b200.modules.attention import LocationSensitiveAttention
    d = C.ATT_DIMS
    res = C.attention_case(LocationSensitiveAttention(d['K'], d['C'], False, d['A'], d['D'], d['M']), 'cuda')

    def tol(key):
        if key.startswith('weights'):
            return 1e-3, 0.0, 1e-6
        if key.startswith('context'):
            return 1e-3, 0.0, 1e-5
        if key == 'dmemory' or key.startswith('dquery'):
            return 3e-3, 1e-4, 0.0
        return 3e-3, 2e-4, 0.0
    _check(golden, 'attention', res, tol)
