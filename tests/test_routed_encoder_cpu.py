"""Routed grouped encoders without a GPU: the layout helper (modules/encoder.py GroupLayout / encoder_layout), the argument checks of
b200tts_convblock_forward_counts / _backward_counts, GraphedTrainStep's refusal of a routed example batch, the per-language oracle
against the reference-layout oracle, and the registers and spills of the kernels the counts touch."""
import ctypes
import os
import re
import subprocess

import pytest
import torch

import routed_encoder_oracle as RO
from oracle import tacotron_oracle as O
from multilingual_text_to_speech_b200 import _lib, build
from multilingual_text_to_speech_b200.modules.encoder import GroupLayout, encoder_layout, language_ids, reference_layout


def test_layout_ranks_counts_and_rows():
    lay = GroupLayout([2, 0, 0, 3, 2, 2, 0], 4)
    assert lay.counts == [3, 0, 3, 1]
    assert lay.ranks == [0, 0, 1, 0, 1, 2, 2]
    assert lay.n_max == 3
    assert lay.rows() == [2, 0, 4, 3, 6, 10, 8]
    assert not lay.reference


def test_reference_layout_is_detected():
    assert GroupLayout([0, 1, 2, 0, 1, 2], 3).reference
    assert GroupLayout([0, 1, 2, 0, 1, 2], 3).rows() == list(range(6))
    assert not GroupLayout([0, 1, 2, 0, 2, 1], 3).reference        # B % G == 0 but the labels do not follow b % G
    assert not GroupLayout([0, 1, 2, 0], 3).reference               # B % G != 0
    langs = torch.arange(64) % 10
    assert encoder_layout(langs, 64, 10).counts == [7, 7, 7, 7, 6, 6, 6, 6, 6, 6]
    assert encoder_layout(torch.arange(60) % 10, 60, 10) is None


def test_layout_decision_skips_mixing_labels_and_one_language():
    ids = torch.tensor([1, 0, 1])
    assert encoder_layout(None, 3, 2) is None                       # no labels: positions decide, as before
    assert encoder_layout(ids, 3, 1) is None                        # one language
    assert encoder_layout(ids[:1], 1, 2) is None                    # batch of one: the inference mixing branch
    assert encoder_layout(ids, 3, 2, padded=True) is None           # padded inference batch: the mixing branch
    assert encoder_layout(ids, 3, 2) is not None
    with reference_layout():
        assert encoder_layout(ids, 3, 2) is None
    with pytest.raises(ValueError, match='labels for 3 utterances given for a batch of 4'):
        encoder_layout(ids, 4, 2)


def test_language_ids_of_every_label_form():
    assert language_ids(torch.tensor([2, 0, 1])) == [2, 0, 1]
    assert language_ids(torch.tensor([[2, 2], [0, 0]])) == [2, 0]
    w = torch.zeros(2, 4, 3)
    w[0, :, 1] = 1
    w[1, :, 2] = 1
    assert language_ids(w) == [1, 2]
    with pytest.raises(ValueError, match='language ids'):
        GroupLayout([0, 3], 3)


def test_cpu_labels_are_read_without_a_device_copy(monkeypatch):
    """CPU labels are read in place: no .cpu() / .to() copy, hence no device synchronisation."""
    def forbidden(*a, **k):
        raise AssertionError('the layout decision copied the labels')
    monkeypatch.setattr(torch.Tensor, 'cpu', forbidden)
    monkeypatch.setattr(torch.Tensor, 'to', forbidden)
    monkeypatch.setattr(torch.Tensor, 'item', forbidden)
    lay = encoder_layout(torch.tensor([[1, 1], [0, 0], [1, 1]]), 3, 2)
    assert lay.counts == [1, 2]


def test_graphed_train_step_refuses_a_routed_example_batch():
    from multilingual_text_to_speech_b200 import configs
    from multilingual_text_to_speech_b200.graph import GraphedTrainStep
    from multilingual_text_to_speech_b200.modules.tacotron2 import Tacotron
    hp = configs.apply('generated_training', decoder_regularization='zoneout')
    G = hp.language_number
    model = Tacotron()
    batch = {'text': torch.ones(G + 1, 5, dtype=torch.long), 'languages': torch.arange(G + 1) % G}
    with pytest.raises(ValueError, match='reference layout'):
        GraphedTrainStep(model, None, None, batch)
    batch = {'text': torch.ones(G, 5, dtype=torch.long), 'languages': torch.arange(G).flip(0)}
    with pytest.raises(ValueError, match='reference layout'):
        GraphedTrainStep(model, None, None, batch)


@pytest.mark.parametrize('kind', ['generated', 'convolutional'])
def test_per_language_oracle_equals_reference_oracle_on_a_reference_batch(kind):
    """On a batch in the reference layout, running each language alone is the reference's grouped computation (fp64)."""
    from multilingual_text_to_speech_b200.modules.encoder import ConvolutionalEncoder, GeneratedConvolutionalEncoder
    torch.manual_seed(0)
    G, F_in, E, L, B = 3, 8, 6, 7, 6
    enc = GeneratedConvolutionalEncoder(F_in, E, 0.05, 4, 2, groups=G) if kind == 'generated' else ConvolutionalEncoder(F_in, E, 0.05, groups=G)
    g = torch.Generator().manual_seed(1)
    x = torch.randn(B, L, F_in, generator=g, dtype=torch.float64)
    ids = [b % G for b in range(B)]
    tape = RO.routed_tape(enc, ids, L, 0.05, g)
    out, _, bufs = RO.encode(enc, x, ids, tape, True, None, device='cpu')
    if kind == 'generated':
        sd = {k: v.detach().double() for k, v in enc.state_dict().items()}
        sd = {('_encoder.' + k): v for k, v in sd.items()}
        stats = {}
        ref = O.generated_encoder(sd, None, x, tape, True, stats=stats)
        torch.testing.assert_close(out, ref, rtol=1e-12, atol=1e-12)
        for j in range(len(O.GENERATED_BLOCKS)):
            mean, var, n = stats[f'_encoder._layers.{j}']
            rm, rv = O.running_stats_update(sd[f'_encoder._layers.{j}._regularizer.running_mean'],
                                            sd[f'_encoder._layers.{j}._regularizer.running_var'], mean.reshape(-1), var.reshape(-1), n)
            torch.testing.assert_close(bufs[f'_layers.{j}._regularizer.running_mean'], rm, rtol=1e-12, atol=1e-12)
            torch.testing.assert_close(bufs[f'_layers.{j}._regularizer.running_var'], rv, rtol=1e-12, atol=1e-12)
    else:
        assert out.shape == (B, L, E) and bool(torch.isfinite(out).all())


def _shape(G=2, NB=3):
    return _lib.ConvBlockShape(NB, G, 4, 8, 16, 1, 1, 1, 0, 1, 1e-5, 0.1, 0.0, 0)


def test_counts_abi_argument_errors():
    lib = _lib.load()
    p = ctypes.c_void_p(16)
    sh = _shape()
    cases = [
        ('forward', lambda: lib.b200tts_convblock_forward_counts(ctypes.byref(sh), None, 2, 3, p, p, p, p, 8, p, p, None, p, p, p, None), 'null argument'),
        ('forward', lambda: lib.b200tts_convblock_forward_counts(ctypes.byref(sh), p, 3, 3, p, p, p, p, 8, p, p, None, p, p, p, None), 'counts are for G=3'),
        ('forward', lambda: lib.b200tts_convblock_forward_counts(ctypes.byref(sh), p, 2, 4, p, p, p, p, 8, p, p, None, p, p, p, None), 'NB=4'),
        ('forward', lambda: lib.b200tts_convblock_forward_counts(ctypes.byref(sh), p, 2, 3, p, None, p, p, 8, p, p, None, p, p, p, None), 'null parameter'),
        ('backward', lambda: lib.b200tts_convblock_backward_counts(ctypes.byref(sh), None, 2, 3, p, p, p, p, 8, None, p, p, p, p, p, p, p, None), 'null argument'),
        ('backward', lambda: lib.b200tts_convblock_backward_counts(ctypes.byref(sh), p, 1, 3, p, p, p, p, 8, None, p, p, p, p, p, p, p, None), 'counts are for G=1'),
        ('backward', lambda: lib.b200tts_convblock_backward_counts(ctypes.byref(sh), p, 2, 2, p, p, p, p, 8, None, p, p, p, p, p, p, p, None), 'NB=2'),
    ]
    for what, call, msg in cases:
        rc = call()
        assert rc != 0, what
        err = lib.b200tts_last_error().decode()
        assert msg in err, (what, err)


# measured (CUDA 12.9, sm_90a): bn_stats 38, block_fwd 40 / 40 (scalar / float4), block_bwd_prep 32 / 40, bn_bwd_reduce 63,
# bn_bwd_apply 34 / 32, zero_vacant 26 registers; no spills
REG_BOUND = {'bn_stats_kernel': 40, 'block_fwd_kernel': 48, 'block_fwd_vec4_kernel': 48, 'block_bwd_prep_kernel': 40,
             'block_bwd_prep_vec4_kernel': 48, 'bn_bwd_reduce_kernel': 64, 'bn_bwd_apply_kernel': 40, 'bn_bwd_apply_vec4_kernel': 40,
             'zero_vacant_kernel': 32}


def test_touched_kernels_registers_and_spills(tmp_path):
    from test_wavernn_cpu import _nvcc
    nvcc = _nvcc()
    if nvcc is None:
        pytest.skip('nvcc not available')
    src = os.path.join(build.CSRC, 'encoder.cu')
    cmd = [nvcc] + build.NVCC_FLAGS + ['-I', os.path.join(build.ROOT, 'include'), '-Xptxas', '-v', '-cubin', src, '-o',
                                       str(tmp_path / 'encoder.cubin')]
    res = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    assert res.returncode == 0, res.stdout
    found = re.findall(r'Function properties for (\S+)\n\s*(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads\n'
                       r'[^\n]*Used (\d+) registers', res.stdout)
    seen = set()
    for mangled, _, st, ld, regs in found:
        for name, bound in REG_BOUND.items():
            if re.search(r'\d' + name + r'E', mangled):
                seen.add(name)
                assert int(st) == 0 and int(ld) == 0, f'{name} spills {st} / {ld} bytes'
                assert int(regs) <= bound, f'{name}: {regs} registers > {bound}'
    assert seen == set(REG_BOUND), set(REG_BOUND) - seen

