"""WaveRNN training without a GPU: the fp64 oracle's MOL loss against finite differences in every branch, the oracle's upsampling against
the generation oracle, vocoder_batch and the label functions against hand-computed windows and the mu-law round trip, the new kernels'
registers and spills, and the argument checks."""
import ctypes
import os
import re
import subprocess

import numpy as np
import pytest
import torch

import wavernn_oracle as O
import wavernn_train_oracle as TO
from multilingual_text_to_speech_b200 import _lib, build
from multilingual_text_to_speech_b200.modules.wavernn import (WaveRNN, draw_offsets, encode_mu_law, float_2_label, label_2_float, mel_window,
                                                              vocoder_batch, wavernn_loss)
from test_wavernn_cpu import REAL, _nvcc


def _mol_case(y, means, log_scales, seed=0):
    g = torch.Generator().manual_seed(seed)
    nr = len(means)
    lp = torch.randn(1, 1, nr, generator=g, dtype=torch.float64)
    logits = torch.cat([lp, torch.tensor(means, dtype=torch.float64).view(1, 1, nr),
                        torch.tensor(log_scales, dtype=torch.float64).view(1, 1, nr)], dim=2).requires_grad_(True)
    return logits, torch.tensor([[y]], dtype=torch.float64)


# (y, means, log scales): each branch of the per-mixture log probability, and a log scale below the clamp
MOL_BRANCHES = {
    'y_at_minus_one': (-1.0, [-0.99, -0.9, 0.2], [-4.0, -3.0, -2.0]),
    'y_at_plus_one': (1.0, [0.99, 0.9, -0.2], [-4.0, -3.0, -2.0]),
    'cdf_delta': (0.3, [0.3001, 0.2995, 0.3003], [-9.0, -7.0, -8.0]),
    'tiny_cdf_delta': (0.3, [0.1, -0.5, 0.8], [3.0, 4.0, 2.5]),
    'below_clamp': (0.3, [0.3, 0.31, 0.3002], [-40.0, -35.0, -9.0]),
}


@pytest.mark.parametrize('branch', sorted(MOL_BRANCHES))
def test_mol_loss_oracle_against_finite_differences(branch):
    y, means, scales = MOL_BRANCHES[branch]
    logits, yt = _mol_case(y, means, scales)
    assert torch.autograd.gradcheck(lambda lg: TO.mol_loss(lg, yt), (logits,), eps=1e-7, atol=1e-6, rtol=1e-5)
    g, = torch.autograd.grad(TO.mol_loss(logits, yt), logits)
    if branch == 'below_clamp':       # no gradient through the clamp of the log scales
        assert g[0, 0, 6] == 0 and g[0, 0, 7] == 0 and g[0, 0, 8] != 0


def test_mol_loss_oracle_selects_each_branch():
    nr, q = 3, 1. / 65535
    for branch, (y, means, scales) in MOL_BRANCHES.items():
        logits, yt = _mol_case(y, means, scales)
        mu, ls = torch.tensor(means, dtype=torch.float64), torch.clamp(torch.tensor(scales, dtype=torch.float64), min=TO.LOG_SCALE_MIN)
        inv = torch.exp(-ls)
        plus, mn, mid = inv * (y - mu + q), inv * (y - mu - q), inv * (y - mu)
        cd = torch.sigmoid(plus) - torch.sigmoid(mn)
        if y < -0.999:
            lp = torch.log(torch.sigmoid(plus))
        elif y > 0.999:
            lp = torch.log(1 - torch.sigmoid(mn))
        else:
            lp = torch.where(cd > 1e-5, torch.log(cd), mid - ls - 2 * torch.nn.functional.softplus(mid) - np.log(65535 / 2))
        if branch == 'tiny_cdf_delta':
            assert bool((cd <= 1e-5).all())
        if branch == 'cdf_delta':
            assert bool((cd > 1e-5).all())
        lp = lp + torch.log_softmax(logits[0, 0, :nr].detach(), -1)
        ref = -torch.logsumexp(lp, 0)
        torch.testing.assert_close(TO.mol_loss(logits.detach(), yt), ref, rtol=1e-10, atol=1e-10)


def test_raw_loss_oracle_is_cross_entropy():
    g = torch.Generator().manual_seed(3)
    logits = torch.randn(2, 5, 16, generator=g, dtype=torch.float64)
    y = torch.randint(0, 16, (2, 5), generator=g)
    ref = -torch.log_softmax(logits, -1).gather(-1, y.unsqueeze(-1)).mean()
    torch.testing.assert_close(TO.raw_loss(logits, y), ref, rtol=1e-12, atol=1e-12)


def test_oracle_upsampling_equals_the_generation_oracle():
    torch.manual_seed(4)
    m = WaveRNN(**dict(REAL, res_blocks=2)).eval()
    with torch.no_grad():
        for name, b in m.named_buffers():
            if name.endswith('running_var'):
                b.uniform_(0.8, 1.2)
    m64 = TO.double_copy(m)
    mel = np.random.default_rng(5).standard_normal((80, 9))
    padded = torch.from_numpy(np.pad(mel, ((0, 0), (2, 2))))[None]
    with torch.no_grad():
        mu, aux = TO.upsample(m64, padded)
    ref_mu, ref_aux = O.upsample(O.sd64(m), mel, (5, 5, 11), 2, 2)
    np.testing.assert_allclose(mu[0].numpy(), ref_mu, rtol=1e-10, atol=1e-12)
    np.testing.assert_allclose(aux[0].numpy(), ref_aux, rtol=1e-10, atol=1e-12)


def test_label_functions():
    assert label_2_float(np.array([0, 511]), 9).tolist() == [-1.0, 1.0]
    assert float(label_2_float(np.array([32767]), 16)) == pytest.approx(2 * 32767 / 65535 - 1, abs=1e-7)
    assert float_2_label(np.array([-1.0, 1.0, 0.0]), 16).tolist() == [0, 65535, 32767]
    with pytest.raises(ValueError):
        float_2_label(np.array([1.5]), 16)
    # mu-law: the generation path's decode of label_2_float(encode(w)) returns w within half a quantisation step of the companded value
    w = np.linspace(-1, 1, 2001)
    for bits in (8, 9, 10):
        lab = encode_mu_law(w, 2 ** bits)
        assert lab.min() == 0 and lab.max() == 2 ** bits - 1 and lab.dtype == np.int64
        back = O.decode_mu_law(label_2_float(lab, bits).double().numpy(), 2 ** bits)
        m = 2 ** bits - 1
        comp = np.sign(w) * np.log1p(m * np.abs(w)) / np.log1p(m)
        comp_back = np.sign(back) * np.log1p(m * np.abs(back)) / np.log1p(m)
        assert np.abs(comp - comp_back).max() <= 1.0 / m + 1e-6
    assert encode_mu_law(np.array([0.0]), 512).tolist() == [256]


def test_vocoder_batch_windows():
    hop, pad, seq_len = 5, 2, 10
    rng = np.random.default_rng(6)
    mels = [rng.standard_normal((3, 12)).astype(np.float32), rng.standard_normal((3, 15)).astype(np.float32)]
    labels = [np.arange(12 * hop) % 512, (np.arange(15 * hop) * 7) % 512]
    offsets = [1, 4]
    assert mel_window(seq_len, hop, pad) == 6
    x, y, m = vocoder_batch(mels, labels, offsets, 'RAW', 9, seq_len, pad, hop)
    assert x.shape == (2, 10) and y.shape == (2, 10) and m.shape == (2, 3, 6)
    assert x.dtype == torch.float32 and y.dtype == torch.int64
    np.testing.assert_array_equal(m[0].numpy(), mels[0][:, 1:7])
    np.testing.assert_array_equal(m[1].numpy(), mels[1][:, 4:10])
    # item 0: the labels window starts at (1 + 2) 5 = 15; item 1 at (4 + 2) 5 = 30
    assert y[0].tolist() == list(range(16, 26)) and y[1].tolist() == [(i * 7) % 512 for i in range(31, 41)]
    np.testing.assert_array_equal(x[0].numpy(), (2 * np.arange(15, 25, dtype=np.float32) / np.float32(511) - 1).astype(np.float32))
    xm, ym, _ = vocoder_batch(mels, labels, offsets, 'MOL', 9, seq_len, pad, hop)
    assert ym.dtype == torch.float32
    np.testing.assert_allclose(xm[0].numpy(), 2 * np.arange(15, 25) / 65535 - 1, rtol=1e-6)
    np.testing.assert_allclose(ym[0].numpy(), 2 * np.arange(16, 26) / 65535 - 1, rtol=1e-6)
    with pytest.raises(ValueError, match='outside'):
        vocoder_batch(mels, labels, [7, 4], 'RAW', 9, seq_len, pad, hop)
    with pytest.raises(ValueError, match='multiple of the hop'):
        vocoder_batch(mels, labels, offsets, 'RAW', 9, 12, pad, hop)
    with pytest.raises(ValueError, match='mode'):
        vocoder_batch(mels, labels, offsets, 'MU', 9, seq_len, pad, hop)


def test_draw_offsets_range():
    rng = np.random.default_rng(7)
    offs = [draw_offsets([40], 1375, 275, 2, rng)[0] for _ in range(2000)]
    win = mel_window(1375, 275, 2)
    assert min(offs) == 0 and max(offs) == 40 - 2 - (win + 4) - 1
    with pytest.raises(ValueError, match='too short'):
        draw_offsets([15], 1375, 275, 2, rng)


def test_abi_rejects_bad_shapes_without_a_device():
    lib = _lib.load()
    ok = _lib.GRUSeqShape(32, 1375, 512)
    assert lib.b200tts_gru_seq_workspace_bytes(ctypes.byref(ok)) > 0
    assert lib.b200tts_gru_seq_saved_bytes(ctypes.byref(ok)) == 32 * 1375 * 4 * 512 * 4
    for bad, msg in [((0, 10, 512), b'batch'), ((65, 10, 512), b'batch'), ((4, 10, 500), b'hidden size'), ((4, 10, 768), b'hidden size'),
                     ((4, 0, 512), b'steps'), ((4, 4401, 512), b'steps')]:
        assert lib.b200tts_gru_seq_workspace_bytes(ctypes.byref(_lib.GRUSeqShape(*bad))) == 0
        assert msg in lib.b200tts_last_error(), (bad, lib.b200tts_last_error())
    one = ctypes.c_void_p(256)
    assert lib.b200tts_gru_seq_forward(ctypes.byref(_lib.GRUSeqShape(4, 10, 512)), one, one, one, one, one, one, 16, None) == -1
    assert b'workspace' in lib.b200tts_last_error()
    assert lib.b200tts_wavernn_loss(2, 10, 30, one, one, one, one, one, 64, None) == -1
    assert b'mode' in lib.b200tts_last_error()
    assert lib.b200tts_wavernn_loss(1, 10, 31, one, one, one, one, one, 64, None) == -1
    assert lib.b200tts_wavernn_stretch_backward(1, 0, 128, 275, one, one, None) == -1
    assert lib.b200tts_wavernn_upsample_layer_backward(80, 0, 5, one, one, one, one, one, one, 1024, None) == -1
    assert lib.b200tts_wavernn_upsample_layer_backward_workspace_bytes(80, 9, 11) == 23 * 64 * 4
    assert lib.b200tts_column_sum(0, 1536, one, one, one, 1 << 20, None) == -1 and b'column_sum' in lib.b200tts_last_error()
    assert lib.b200tts_column_sum(100, 1536, None, one, one, 1 << 20, None) == -1
    assert lib.b200tts_column_sum_workspace_bytes(1536) == 64 * 1536 * 4


def test_forward_and_loss_argument_errors():
    m = WaveRNN(**REAL)
    with pytest.raises(ValueError, match='multiple of the hop'):
        m(torch.zeros(2, 300), torch.zeros(2, 80, 6))
    with pytest.raises(ValueError, match='16 hops'):
        m(torch.zeros(2, 17 * 275), torch.zeros(2, 80, 21))
    with pytest.raises(ValueError, match='mels of shape'):
        m(torch.zeros(2, 550), torch.zeros(2, 80, 5))
    with pytest.raises(ValueError, match='targets'):
        wavernn_loss(torch.zeros(2, 5, 512), torch.zeros(2, 4, dtype=torch.long), 'RAW')
    with pytest.raises(ValueError, match='mode'):
        wavernn_loss(torch.zeros(2, 5, 30), torch.zeros(2, 5), 'MU')


# measured (CUDA 12.9, sm_90a): GRU loops 48-80 registers, the other new kernels at most 36; none spills
REG_BOUND = {'gru_seq_fwd_kernel': 128, 'gru_seq_bwd_kernel': 96, 'wavernn_': 64, 'column_sum_': 64}


def test_new_kernels_registers_and_spills(tmp_path):
    nvcc = _nvcc()
    if nvcc is None:
        pytest.skip('nvcc not available')
    cmd = [nvcc] + build.NVCC_FLAGS + ['-I', os.path.join(build.ROOT, 'include'), '-Xptxas', '-v', '-cubin',
                                       os.path.join(build.CSRC, 'wavernn_train.cu'), '-o', str(tmp_path / 'wavernn_train.cubin')]
    res = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    assert res.returncode == 0, res.stdout
    found = re.findall(r'Function properties for (\S+)\n\s*(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads\n'
                       r'[^\n]*Used (\d+) registers', res.stdout)
    names = [f[0] for f in found]
    assert sum('gru_seq_fwd_kernel' in n for n in names) == 5 and sum('gru_seq_bwd_kernel' in n for n in names) == 5, names
    assert len(found) == 19, names
    for name, stack, st, ld, regs in found:
        assert int(stack) == 0 and int(st) == 0 and int(ld) == 0, name
        bound = next(v for k, v in REG_BOUND.items() if k in name)
        assert int(regs) <= bound, (name, regs)
