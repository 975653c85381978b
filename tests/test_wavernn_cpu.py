"""WaveRNN without a GPU: the fp64 oracle against torch, the fold / unfold identities, the samplers' distributions, the state-dict surface,
the loop kernel's registers and the argument checks."""
import ctypes
import os
import re
import shutil
import subprocess

import numpy as np
import pytest
import torch
from scipy import stats

import wavernn_oracle as O
from multilingual_text_to_speech_b200 import _lib, build
from multilingual_text_to_speech_b200.modules.wavernn import WaveRNN, fold_count

REAL = dict(rnn_dims=512, fc_dims=512, bits=9, pad=2, upsample_factors=(5, 5, 11), feat_dims=80, compute_dims=128, res_out_dims=128,
            res_blocks=10, hop_length=275, sample_rate=22050)


def test_oracle_gru_cell_matches_torch():
    torch.manual_seed(0)
    gru = torch.nn.GRU(24, 16, batch_first=True).double()
    x = torch.randn(5, 1, 24, dtype=torch.float64)
    h = torch.randn(1, 5, 16, dtype=torch.float64)
    ref = gru(x, h)[1][0].detach().numpy()
    got = O.gru_cell(x[:, 0].numpy(), h[0].numpy(), *(getattr(gru, n).detach().numpy() for n in
                                                      ('weight_ih_l0', 'weight_hh_l0', 'bias_ih_l0', 'bias_hh_l0')))
    np.testing.assert_allclose(got, ref, rtol=1e-12, atol=1e-14)


def test_upsampling_lengths_and_indent_cut():
    torch.manual_seed(1)
    m = WaveRNN(**dict(REAL, res_blocks=1))
    p = O.sd64(m)
    F = 7
    mel = np.random.default_rng(0).standard_normal((80, F))
    mu, aux = O.upsample(p, mel, (5, 5, 11), 2, 1)
    assert mu.shape == (F * 275, 80) and aux.shape == (F * 275, 128)
    assert m.upsample.indent == 2 * 275
    # with the default FIR (box filters) a constant mel stays constant away from the ends of the padded sequence
    mu1, _ = O.upsample(p, np.ones((80, 30)), (5, 5, 11), 2, 1)
    np.testing.assert_allclose(mu1[600:-600], 1.0, rtol=1e-6)     # the taps are fp32 roundings of 1 / k


def test_fold_unfold_constant_signal():
    target, overlap = 100, 20
    x = np.ones((777, 1))
    folded = O.fold_with_overlap(x, target, overlap)[..., 0]
    assert folded.shape[0] == fold_count(777, target, overlap)
    y = O.xfade_and_unfold(folded, target, overlap)
    sil = overlap // 2
    # fade_in^2 + fade_out^2 = 1, so the cross-faded regions keep the energy of a constant signal: fade_in + fade_out >= 1
    t = np.linspace(-1, 1, overlap - sil)
    np.testing.assert_allclose(np.sqrt(0.5 * (1 + t)) ** 2 + np.sqrt(0.5 * (1 - t)) ** 2, 1.0, rtol=1e-15)
    # away from the overlaps every sample of the signal (not of the tail padding) is exactly 1
    for i in range(folded.shape[0]):
        s = i * (target + overlap)
        np.testing.assert_array_equal(y[s + overlap:min(777, s + target + overlap)], 1.0)
    assert np.all(y[777:] == 0)
    assert np.all(y[:sil] == 0)


def test_raw_sampler_distribution():
    rng = np.random.default_rng(3)
    logits = rng.standard_normal(16) * 2
    p = np.exp(logits - logits.max())
    p /= p.sum()
    u = rng.random(20000)
    ks = np.array([O.raw_sample(logits, v)[0] for v in u])
    counts = np.bincount(ks, minlength=16)
    chi2 = stats.chisquare(counts, p * len(u))
    assert chi2.pvalue > 1e-3, chi2


def test_mol_sampler_distribution():
    rng = np.random.default_rng(4)
    nr = 10
    logits = np.concatenate([rng.standard_normal(nr), rng.uniform(-0.5, 0.5, nr), np.full(nr, np.log(0.05))])
    n = 20000
    us = rng.random((n, nr + 1))
    draws = [O.mol_sample(logits, u) for u in us]
    comps = np.bincount([d[2] for d in draws], minlength=nr)
    w = np.exp(logits[:nr] - logits[:nr].max())
    w /= w.sum()
    assert stats.chisquare(comps, w * n).pvalue > 1e-3
    # one component: the sample is a logistic with that mean and scale (the clamp to [-1, 1] is far in the tails here)
    j = int(np.argmax(comps))
    xs = np.array([d[0] for d in draws if d[2] == j])
    ks = stats.kstest(xs, stats.logistic(loc=logits[nr + j], scale=0.05).cdf)
    assert ks.pvalue > 1e-3, ks


# fatchord's names and shapes at the reference's dimensions
def _expected_keys():
    keys = [('step', (1,)), ('upsample.resnet.conv_in.weight', (128, 80, 5))]
    bn = lambda n, c: [(f'{n}.weight', (c,)), (f'{n}.bias', (c,)), (f'{n}.running_mean', (c,)), (f'{n}.running_var', (c,)),
                       (f'{n}.num_batches_tracked', ())]
    keys += bn('upsample.resnet.batch_norm', 128)
    for i in range(10):
        q = f'upsample.resnet.layers.{i}.'
        keys += [(q + 'conv1.weight', (128, 128, 1)), (q + 'conv2.weight', (128, 128, 1))] + bn(q + 'batch_norm1', 128) + bn(q + 'batch_norm2', 128)
    keys += [('upsample.resnet.conv_out.weight', (128, 128, 1)), ('upsample.resnet.conv_out.bias', (128,))]
    keys += [('upsample.up_layers.1.weight', (1, 1, 1, 11)), ('upsample.up_layers.3.weight', (1, 1, 1, 11)),
             ('upsample.up_layers.5.weight', (1, 1, 1, 23))]
    keys += [('I.weight', (512, 113)), ('I.bias', (512,))]
    keys += [('rnn1.weight_ih_l0', (1536, 512)), ('rnn1.weight_hh_l0', (1536, 512)), ('rnn1.bias_ih_l0', (1536,)), ('rnn1.bias_hh_l0', (1536,))]
    keys += [('rnn2.weight_ih_l0', (1536, 544)), ('rnn2.weight_hh_l0', (1536, 512)), ('rnn2.bias_ih_l0', (1536,)), ('rnn2.bias_hh_l0', (1536,))]
    keys += [('fc1.weight', (512, 544)), ('fc1.bias', (512,)), ('fc2.weight', (512, 544)), ('fc2.bias', (512,)),
             ('fc3.weight', (512, 512)), ('fc3.bias', (512,))]
    return keys


def test_state_dict_keys_and_shapes():
    sd = WaveRNN(**REAL).state_dict()
    assert [(k, tuple(v.shape)) for k, v in sd.items()] == _expected_keys()
    mol = WaveRNN(**dict(REAL, mode='MOL')).state_dict()
    assert tuple(mol['fc3.weight'].shape) == (30, 512)
    # a state dict of that layout loads
    WaveRNN(**REAL).load_state_dict({k: torch.randn(v.shape) if v.dtype.is_floating_point else v for k, v in sd.items()})


def test_bad_hop_length_and_mode():
    with pytest.raises(ValueError, match='hop_length'):
        WaveRNN(**dict(REAL, hop_length=256))
    with pytest.raises(ValueError, match='mode'):
        WaveRNN(**dict(REAL, mode='MU'))
    with pytest.raises(ValueError, match='rnn_dims'):
        WaveRNN(**dict(REAL, rnn_dims=500))


def test_bad_mels_and_tapes():
    m = WaveRNN(**REAL)
    with pytest.raises(ValueError, match='expected \\[80, frames\\]'):
        m.generate_batch([np.zeros((40, 30), np.float32)])
    with pytest.raises(ValueError, match='at least 21'):
        m.generate_batch([np.zeros((80, 20), np.float32)])
    with pytest.raises(ValueError, match='non-empty'):
        m.generate_batch([])
    mel = np.zeros((80, 30), np.float32)
    shape = m.tape_shape(30, 1000, 100)
    with pytest.raises(ValueError, match='expected'):
        m.generate_batch([mel], 1000, 100, uniforms=[np.zeros(shape[:2], np.float32)])
    with pytest.raises(ValueError, match='outside \\[0, 1\\)'):
        m.generate_batch([mel], 1000, 100, uniforms=[np.ones(shape, np.float32)])
    with pytest.raises(ValueError, match='tapes for'):
        m.generate_batch([mel, mel], 1000, 100, uniforms=[np.zeros(shape, np.float32)])


def test_abi_rejects_bad_shapes_without_a_device():
    lib = _lib.load()
    assert lib.b200tts_wavernn_workspace_bytes(ctypes.byref(_lib.WaveRNNShape(4, 512, 512, 512, 0, 700))) > 0
    for bad, msg in [((0, 512, 512, 512, 0, 700), b'fold row'), ((4, 500, 512, 512, 0, 700), b'rnn_dims'),
                     ((4, 512, 512, 31, 1, 700), b'MOL'), ((4, 512, 512, 512, 2, 700), b'mode'), ((4, 512, 512, 512, 0, 0), b'fold length')]:
        assert lib.b200tts_wavernn_workspace_bytes(ctypes.byref(_lib.WaveRNNShape(*bad))) == 0
        assert msg in lib.b200tts_last_error(), (bad, lib.b200tts_last_error())
    fs = _lib.WaveRNNFoldShape(1, 1, 80, 128, 275, 2, 7, 1000, 100, 30)      # 275 is not a multiple of 7
    one = ctypes.c_void_p(16)
    st = lib.b200tts_wavernn_fold(ctypes.byref(fs), one, one, one, one, one, one, one, 0, 10, one, None)
    assert st == -1 and b'multiple of the last upsampling factor' in lib.b200tts_last_error()
    assert lib.b200tts_wavernn_upsample_layer(80, 0, 5, one, one, one, None) == -1


def _nvcc():
    for cand in (os.environ.get('NVCC'), '/usr/local/cuda/bin/nvcc', shutil.which('nvcc')):
        if cand and os.path.exists(cand):
            return cand
    return None


# measured: 156 registers, no stack, no spills (CUDA 12.9, sm_90a); __launch_bounds__(256, 1) allows 255
REG_BOUND = 200


def test_loop_kernel_registers_and_spills(tmp_path):
    nvcc = _nvcc()
    if nvcc is None:
        pytest.skip('nvcc not available')
    cmd = [nvcc] + build.NVCC_FLAGS + ['-I', os.path.join(build.ROOT, 'include'), '-Xptxas', '-v', '-cubin',
                                       os.path.join(build.CSRC, 'wavernn.cu'), '-o', str(tmp_path / 'wavernn.cubin')]
    res = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    assert res.returncode == 0, res.stdout
    m = re.search(r'Function properties for \S*wavernn_loop_kernel\S*\n\s*(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill '
                  r'loads\n[^\n]*Used (\d+) registers', res.stdout)
    assert m, res.stdout
    stack, st, ld, regs = map(int, m.groups())
    assert st == 0 and ld == 0 and stack == 0, m.group(0)
    assert regs <= REG_BOUND, regs


def test_non_finite_mels_and_bad_preemphasis_are_rejected():
    m = WaveRNN(**REAL)
    for bad in (np.nan, np.inf, -np.inf):
        mel = np.zeros((80, 30), np.float32)
        mel[3, 7] = bad
        with pytest.raises(ValueError, match='non-finite'):
            m.generate_batch([np.zeros((80, 30), np.float32), mel])
        with pytest.raises(ValueError, match='non-finite'):
            m.generate(torch.from_numpy(mel))
    with pytest.raises(ValueError, match='preemphasis'):
        m.generate(np.zeros((80, 30), np.float32), preemphasis=1.0)
    lib = _lib.load()
    one = ctypes.c_void_p(16)
    assert lib.b200tts_wavernn_deemphasis(4, 100, 511, ctypes.c_float(1.5), one, None) == -1
    assert b'(-1, 1)' in lib.b200tts_last_error()
    assert lib.b200tts_wavernn_deemphasis(0, 100, 511, ctypes.c_float(0.9), one, None) == -1


def test_oracle_deemphasis_is_the_recurrence():
    rng = np.random.default_rng(9)
    folded = rng.uniform(-1, 1, (3, 140))
    out = O.postprocess(folded, 30, 10, 100, 20, None, 0.9)
    y = folded.copy()
    for r in range(3):
        for i in range(1, 140):
            y[r, i] += 0.9 * y[r, i - 1]
    ref = O.postprocess(y, 30, 10, 100, 20, None, 0.0)
    np.testing.assert_allclose(out, ref, rtol=1e-12, atol=1e-12)
