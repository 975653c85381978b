"""Every step of the packed bi-LSTM (csrc/rnn.cu, csrc/bilstm_persist.cu), forward and backward, both directions, against an fp64
step computed from the kernel's own saved state (tests/bilstm_check.py), in fp32 and bf16 mode, on the persistent cluster kernel and
on the per-step chain (B200TTS_BILSTM_CHAIN=1).  Run with -s to see the worst err / bound ratio of every stage.

Each call goes through the C ABI with buffers the test owns: out, d x, saved and both workspaces are NaN-poisoned and carved from
larger buffers whose sentinel bands must be intact afterwards; the parameter gradients start from random prefills they must be
accumulated onto; the inputs must come back unchanged; the kernels that ran must be the path the layout query announces; and a
second identical call must give bitwise the same results.
"""
import ctypes
import os

import pytest
import torch

import bilstm_check as C

pytestmark = pytest.mark.gpu

SENT = 0x7fa1b2c3          # a NaN bit pattern no kernel writes
HEAD, TAIL = 256, 4096


@pytest.fixture(scope='module', autouse=True)
def _built():
    import __graft_entry__ as entry
    entry.build()
    assert torch.cuda.is_available()


class Guarded:
    """n 4-byte elements between sentinel bands; filled from init, or NaN-poisoned"""

    def __init__(self, n, init=None, dtype=torch.float32):
        self.buf = torch.full((HEAD + n + TAIL,), SENT, dtype=torch.int32, device='cuda')
        self.t = self.buf[HEAD:HEAD + n].view(dtype)
        if init is not None:
            self.t.copy_(init.reshape(-1))
        else:
            self.t.fill_(float('nan'))

    def intact(self):
        return bool((self.buf[:HEAD] == SENT).all()) and bool((self.buf[HEAD + self.t.numel():] == SENT).all())


def _inputs(B, L, E, H, lengths, seed):
    g = torch.Generator().manual_seed(seed)
    k = 2.0 / H ** 0.5                        # twice PyTorch's init range: a livelier recurrence
    prm = {}
    for n in C.PARAMS:
        shape = {'w_ih': (4 * H, E), 'w_hh': (4 * H, H)}.get(n.replace('_reverse', ''), (4 * H,))
        prm[n] = (torch.rand(*shape, generator=g) * 2 - 1) * k
    return dict(x=torch.randn(B, L, E, generator=g), lengths=C.gpu_lengths(B, L, lengths, seed), prm=prm,
                dout=torch.randn(B, L, 2 * H, generator=g), prefill={n: 0.1 * torch.randn(*p.shape, generator=g) for n, p in prm.items()})


def _call(B, L, E, H, inp, precision):
    """forward + backward through the C ABI -> (results on the device, kernel names that ran)"""
    from multilingual_text_to_speech_b200 import _lib, functional as F
    lib = _lib.load()
    shape = _lib.BiLSTMShape(B, L, E, H)
    sh, st = ctypes.byref(shape), F._stream()
    nsaved, nws = lib.b200tts_bilstm_saved_bytes(sh) // 4, lib.b200tts_bilstm_workspace_bytes(sh) // 4
    b = {'x': Guarded(B * L * E, inp['x']), 'lengths': Guarded(B, inp['lengths'].int(), torch.int32),
         'dout': Guarded(B * L * 2 * H, inp['dout']), 'out': Guarded(B * L * 2 * H), 'dx': Guarded(B * L * E),
         'saved': Guarded(nsaved), 'ws_fwd': Guarded(nws), 'ws_bwd': Guarded(nws)}
    for n in C.PARAMS:
        b[n] = Guarded(inp['prm'][n].numel(), inp['prm'][n])
        b['d' + n] = Guarded(inp['prm'][n].numel(), inp['prefill'][n])
    params = _lib.BiLSTMParams(*[F.ptr(b[n].t) for n in C.PARAMS])
    grads = _lib.BiLSTMParams(*[F.ptr(b['d' + n].t) for n in C.PARAMS])
    _lib.set_precision(precision)
    _lib.kernel_timing(True)
    try:
        F.check(lib.b200tts_bilstm_forward(sh, ctypes.byref(params), F.ptr(b['x'].t), F.ptr(b['lengths'].t), F.ptr(b['out'].t),
                                           F.ptr(b['saved'].t), F.ptr(b['ws_fwd'].t), st), 'b200tts_bilstm_forward')
        F.check(lib.b200tts_bilstm_backward(sh, ctypes.byref(params), F.ptr(b['lengths'].t), F.ptr(b['saved'].t), F.ptr(b['dout'].t),
                                            F.ptr(b['dx'].t), ctypes.byref(grads), F.ptr(b['ws_bwd'].t), st), 'b200tts_bilstm_backward')
        torch.cuda.synchronize()
        ran = set(_lib.kernel_timing_read())
    finally:
        _lib.kernel_timing(False)
        _lib.set_precision('fp32')
    intact = {k: g.intact() for k, g in b.items()}
    assert all(intact.values()), intact
    for k in ('x', 'dout', 'lengths'):
        assert torch.equal(b[k].t.cpu(), inp[k].reshape(-1).to(b[k].t.dtype)), f'{k} changed'
    for n in C.PARAMS:
        assert torch.equal(b[n].t.cpu(), inp['prm'][n].reshape(-1)), f'{n} changed'
    res = {'out': b['out'].t.view(B, L, 2 * H), 'dx': b['dx'].t.view(B, L, E), 'saved': b['saved'].t, 'ws': b['ws_bwd'].t}
    res.update({'d' + n: b['d' + n].t.view(inp['prm'][n].shape) for n in C.PARAMS})
    return res, ran


def _step_check(B, L, E, H, lengths, precision, chain, seed=0):
    old = os.environ.pop('B200TTS_BILSTM_CHAIN', None)
    if chain:
        os.environ['B200TTS_BILSTM_CHAIN'] = '1'
    try:
        lay = C.layout(B, L, E, H)
        assert lay['persist'] == (not chain), lay
        inp = _inputs(B, L, E, H, lengths, seed=B * 131 + L + seed)
        runs = [_call(B, L, E, H, inp, precision) for _ in range(2)]
    finally:
        os.environ.pop('B200TTS_BILSTM_CHAIN', None)
        if old is not None:
            os.environ['B200TTS_BILSTM_CHAIN'] = old
    (res, ran), (res2, _) = runs
    persistent = {'bilstm_fwd_loop_kernel', 'bilstm_bwd_loop_kernel'}
    assert (persistent <= ran) if lay['persist'] else not (persistent & ran), ran
    v = C.views(res['saved'].view(torch.uint8), res['ws'].view(torch.uint8), B, L, E, H, lay)
    v2 = C.views(res2['saved'].view(torch.uint8), res2['ws'].view(torch.uint8), B, L, E, H, lay)
    for k in C.VIEWS:                 # what the checker reads came back finite, and bitwise equal on the second call
        assert bool(torch.isfinite(v[k]).all()), k
        assert torch.equal(v[k], v2[k]), k
    for k in ['out', 'dx'] + ['d' + n for n in C.PARAMS]:
        assert bool(torch.isfinite(res[k]).all()), k
        assert torch.equal(res[k], res2[k]), k
    dev = torch.device('cuda:0')
    prm = {n: p.to(dev) for n, p in inp['prm'].items()}
    grads = {n: res['d' + n] for n in C.PARAMS}
    prefill = {n: p.to(dev) for n, p in inp['prefill'].items()}
    rep = C.check_all(v, prm, inp['x'].to(dev), inp['lengths'].to(dev), res['out'], inp['dout'].to(dev), grads, prefill, res['dx'],
                      precision, lay['persist'], lay['split'], lay['split_b'])
    title = f'[B{B} L{L} E{E} H{H} {precision} {"persist" if lay["persist"] else "chain"}] '
    print()
    print('\n'.join(rep.lines(title)))
    assert rep.failures() == {}, (title, rep.failures())
    return rep


def _cases(path):
    out = []
    for B, L, E, H, lengths, p in C.GPU_CASES:
        if path == 'chain' or p == 'persist':
            out.append(pytest.param(B, L, E, H, lengths, id=f'B{B}_L{L}_E{E}_H{H}' + ('_unsorted' if lengths == 'unsorted' else '')))
    return out


@pytest.mark.parametrize('precision', ('fp32', 'bf16'))
@pytest.mark.parametrize('B,L,E,H,lengths', _cases('persist'))
def test_bilstm_persistent_kernel_steps_within_bounds(B, L, E, H, lengths, precision):
    _step_check(B, L, E, H, lengths, precision, chain=False)


@pytest.mark.parametrize('precision', ('fp32', 'bf16'))
@pytest.mark.parametrize('B,L,E,H,lengths', _cases('chain'))
def test_bilstm_per_step_chain_steps_within_bounds(B, L, E, H, lengths, precision):
    _step_check(B, L, E, H, lengths, precision, chain=True)
