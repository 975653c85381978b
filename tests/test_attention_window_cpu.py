"""Windowed synthesis (hp.inference_attention_window) without a GPU: the ValueErrors of the setting, the library's argument checks,
the CPU oracle's own consistency (a window covering every position is no window; a windowed decode keeps the window property), the
registers of attn_fwd_kernel<true> and the unchanged SASS of attn_fwd_kernel<false>."""
import ctypes
import hashlib
import os
import re
import subprocess

import numpy as np
import pytest
import torch

import attention_window_oracle as AW
import decoder_cases as DC
from oracle import tacotron_oracle as O
from multilingual_text_to_speech_b200 import _lib, build
from multilingual_text_to_speech_b200.params.params import Params as hp
from multilingual_text_to_speech_b200.modules import tacotron2 as T
from test_wavernn_cpu import _nvcc


@pytest.fixture
def params():
    hp.reset()
    yield hp
    hp.reset()


@pytest.mark.parametrize('value', [[1], [1, 2, 3], (0, 0), [-1, 3], [2, 0], [1.0, 3], [True, 3], '1,3', 3, [1, '3']])
def test_bad_window_values_raise(params, value):
    hp.inference_attention_window = value
    with pytest.raises(ValueError, match='inference_attention_window'):
        T.inference_attention_window()


def test_window_values(params):
    assert T.inference_attention_window() is None
    hp.inference_attention_window = [0, 1]
    assert T.inference_attention_window() == (0, 1)
    hp.inference_attention_window = (np.int64(4), 7)
    assert T.inference_attention_window() == (4, 7)


def test_window_with_forward_attention_raises(params):
    hp.inference_attention_window = [1, 3]
    hp.attention_type = 'forward'
    with pytest.raises(ValueError, match='forward attention'):
        T.inference_attention_window()


def test_entry_points_check_the_setting(params):
    """inference_batch and a decoder pool read the setting before they decode anything, so a bad value fails on any device."""
    model = T.Tacotron()
    hp.inference_attention_window = [1, 0]
    with pytest.raises(ValueError, match='inference_attention_window'):
        model.inference_batch([torch.tensor([1, 2, 3])])
    with pytest.raises(ValueError, match='inference_attention_window'):
        model.decoder_pool()
    with pytest.raises(ValueError, match='inference_attention_window'):
        next(model.inference_stream(torch.tensor([1, 2, 3])))


def _shape(**kw):
    s = _lib.DecoderShape(2, 12, 8, 16, 24, 8, 8, 4, 5, 6, 0, 0, 0.1, 0.0, 0.5)
    for k, v in kw.items():
        setattr(s, k, v)
    return s


def test_library_argument_checks():
    lib = _lib.load()
    ws = lambda s: lib.b200tts_decoder_workspace_bytes(ctypes.byref(s))        # noqa: E731 -- validates the shape, no device needed
    assert ws(_shape()) > 0 and ws(_shape(att_window_back=2, att_window_ahead=3)) > 0 and ws(_shape(att_window_ahead=1)) > 0
    for bad in (dict(att_window_back=-1, att_window_ahead=3), dict(att_window_back=2, att_window_ahead=0), dict(att_window_ahead=-2)):
        assert ws(_shape(**bad)) == 0 and b'bad attention window' in lib.b200tts_last_error(), bad
    assert ws(_shape(att_kind=_lib.ATT_FORWARD, att_window_back=1, att_window_ahead=3)) == 0
    assert b'forward attention' in lib.b200tts_last_error()
    win = _shape(att_window_back=1, att_window_ahead=3)
    one = ctypes.c_void_p(16)
    P, I, O_ = _lib.DecoderParams(), _lib.DecoderInputs(), _lib.DecoderOutputs()
    assert lib.b200tts_decoder_forward(ctypes.byref(win), ctypes.byref(P), ctypes.byref(I), ctypes.byref(O_), one, 1, None) == -1
    assert b'decoder_forward: an attention window is for synthesis only' in lib.b200tts_last_error()
    G = _lib.DecoderOutputGrads()
    assert lib.b200tts_decoder_backward(ctypes.byref(win), ctypes.byref(P), ctypes.byref(I), ctypes.byref(O_), ctypes.byref(G), one, one,
                                        1, ctypes.byref(P), None, None) == -1
    assert b'decoder_backward: an attention window is for synthesis only' in lib.b200tts_last_error()
    st = _lib.DecoderState(*([one] * 7))
    assert lib.b200tts_decoder_forward_chunk(ctypes.byref(win), ctypes.byref(P), ctypes.byref(I), ctypes.byref(O_), ctypes.byref(st), 1,
                                             one, 1, None) == -1
    assert b'needs state->attended' in lib.b200tts_last_error()


def _decode(window, L=14, frames=24, seed=3):
    c = DC.full_dim_case(B=1, L=L, T=frames, M=16, D=24, P=8, A=8, C=4, K=5, N=6, seed=seed, training=False, tf=0.0, ragged=False)
    sd = {k: v.double() for k, v in c.sd.items()}
    tape = {k: (v if k == 'teacher' else v.double()) for k, v in c.tape.items()}
    mask = O.lengths_to_mask(c.lengths, L)
    hp_ = c.hp
    hp_.stop_frames = 10 ** 6           # decode every frame
    if window is None:
        return O.decoder_forward(sd, hp_, c.memory.double(), mask, None, None, None, tape, training=False)
    with AW.windowed(window):
        return O.decoder_forward(sd, hp_, c.memory.double(), mask, None, None, None, tape, training=False)


def test_oracle_full_window_is_no_window():
    ref = _decode(None)
    for window in ((14, 14), (100, 20)):
        out = _decode(window)
        for a, b in zip(out, ref):
            assert torch.equal(a, b)


def test_oracle_window_property():
    free = _decode(None)
    for window in ((0, 1), (1, 3), (2, 2)):
        spec, stop, align = _decode(window)
        AW.check_window_property(align, [14], window, atol=1e-12)
        assert not torch.equal(align, free[2])          # the window changed the decode
    with pytest.raises(AssertionError):                 # and the check notices weights outside a window
        AW.check_window_property(free[2], [14], (0, 1), atol=1e-12)


# measured (CUDA 12.9, sm_90a): attn_fwd_kernel<true> 60 registers, no spills (attn_fwd_kernel<false>: 64 registers, 8 bytes of spills,
# as before the window existed)
WINDOW_REG_BOUND = 64
# sha256 of attn_fwd_kernel's SASS instructions (addresses stripped) as the parent commit built them with CUDA 12.9 for sm_90a
ATTN_SASS_SHA256 = 'f9c9b15c51daeca11fe750c4548b85be4ac0bbe2bd4f9e9bc06f0a3648be7f9f'


@pytest.fixture(scope='module')
def compiled(tmp_path_factory):
    nvcc = _nvcc()
    if nvcc is None:
        pytest.skip('nvcc not available')
    cubin = tmp_path_factory.mktemp('attn') / 'decoder_fwd.cubin'
    cmd = [nvcc] + build.NVCC_FLAGS + ['-I', os.path.join(build.ROOT, 'include'), '-Xptxas', '-v', '-cubin',
                                       os.path.join(build.CSRC, 'decoder_fwd.cu'), '-o', str(cubin)]
    res = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    assert res.returncode == 0, res.stdout
    return nvcc, cubin, res.stdout


def test_windowed_kernel_registers_and_spills(compiled):
    _, _, log = compiled
    m = re.search(r'Function properties for \S*attn_fwd_kernelILb1E\S*\n\s*(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes '
                  r'spill loads\n[^\n]*Used (\d+) registers', log)
    assert m, log
    stack, st, ld, regs = map(int, m.groups())
    assert st == 0 and ld == 0 and stack == 0, m.group(0)
    assert regs <= WINDOW_REG_BOUND, regs


def test_unwindowed_kernel_sass_unchanged(compiled):
    """attn_fwd_kernel<false>, which training and every decode without a window run, is the parent's kernel instruction for instruction."""
    nvcc, cubin, _ = compiled
    version = subprocess.run([nvcc, '--version'], stdout=subprocess.PIPE, text=True).stdout
    if 'release 12.9' not in version:
        pytest.skip('the recorded SASS is CUDA 12.9\'s')
    cuobjdump = os.path.join(os.path.dirname(nvcc), 'cuobjdump')
    out = subprocess.run([cuobjdump, '-sass', str(cubin)], stdout=subprocess.PIPE, text=True).stdout
    funcs = [f for f in re.split(r'\n\s*Function : ', out) if '15attn_fwd_kernelILb0E' in f.split('\n', 1)[0]]
    assert len(funcs) == 1
    ins = [re.sub(r'/\*[0-9a-f]{4}\*/', '', line).split(';')[0].strip() for line in funcs[0].split('\n')[1:]
           if re.match(r'\s*/\*[0-9a-f]{4}\*/', line)]
    assert hashlib.sha256('\n'.join(ins).encode()).hexdigest() == ATTN_SASS_SHA256
