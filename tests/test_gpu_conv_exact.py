"""The encoder / postnet convolution (stage 1 of the conv block: the grouped Conv1d alone, no batch norm) against an fp64 conv1d with
the same zero padding and groups, at the generated_training encoder's real shapes, the postnet's, and the edges where a tiled
kernel goes wrong; and the parameter generator's backward against fp64 autograd of (e . Wb^T + bb) . Wk^T + bk.

bf16 mode compares with fp64 on bf16-rounded x, w and d out (what the kernels multiply, accumulating in fp32), so the bounds are
those of the wgmma GEMM test: rtol 1e-4, atol 2e-4 sqrt(K) with K the reduction length (Cin k for the output, Cout k for dx,
NB L for dw).  fp32 mode (im2col + fp32 GEMM) compares with fp64 on the unrounded operands.

Every case asserts which kernel path ran, from the launches each call makes (`_lib.launch_count`) and the wgmma GEMM launches among
them (kernel timer "gemm_tc_kernel"); forward, input gradient and weight gradient are separate library calls:
- 'implicit': gemm_tc_conv, the TMA row-shift convolution (forward and input gradient of k > 1): 2 packs + 1 GEMM.
- 'fused' / 'fused+splitK': gemm_tc_conv_dw (weight gradient of k > 1): 2 packs + 1 GEMM (+ the split-K reduction when G == 1).
- 'two-level': the batched weight-gradient GEMM whose K runs over (sample row, position), taken when the fused product does not
  apply and NB > 1 (k == 1 blocks here; the pack cache that also makes gemm_tc_conv_dw decline is only open inside the decoder's
  backward, where no convolution runs): 2 packs + 1 GEMM.
- 'per-row': one GEMM per sample row (NB == 1).
- 'gemm': a k == 1 forward / input gradient, a plain GEMM on the input.
"""
import ctypes

import pytest
import torch

from helpers import assert_close

pytestmark = pytest.mark.gpu


@pytest.fixture(scope='module', autouse=True)
def _built():
    import __graft_entry__ as entry
    entry.build()
    assert torch.cuda.is_available()


def _call(fn):
    """Run fn(); return (library launches, wgmma GEMM launches) it made."""
    from multilingual_text_to_speech_b200 import _lib
    torch.cuda.synchronize()
    _lib.kernel_timing(True)
    n0 = _lib.launch_count()
    try:
        fn()
        torch.cuda.synchronize()
        n = _lib.launch_count() - n0
        tc = _lib.kernel_timing_read().get('gemm_tc_kernel', (0.0, 0))[1]
    finally:
        _lib.kernel_timing(False)
    return n, tc


def _path(what, c, launches, tc):
    if what in ('out', 'dx'):
        if c['k'] > 1 and (launches, tc) == (3, 1):
            return 'implicit'
        if c['k'] == 1 and tc <= 1:
            return 'gemm'
    else:
        if c['k'] > 1 and (launches, tc) == (3, 1):
            return 'fused'
        if c['k'] > 1 and (launches, tc) == (4, 1):
            return 'fused+splitK'
        if c['k'] == 1 and c['NB'] > 1 and (launches, tc) in ((3, 1), (4, 1)):
            return 'two-level'
        if c['NB'] == 1 and tc <= 1:
            return 'per-row'
    return f'unexpected ({launches} launches, {tc} wgmma)'


def _conv_lib(c, x, w, dout):
    """Stage-1 forward, input-gradient-only and weight-gradient-only calls through the C ABI:
    (out, dx, dw, {what: (launches, wgmma launches)})."""
    from multilingual_text_to_speech_b200 import _lib, functional as F
    NB, G, Cin, Cout, L, k, dil = (c[n] for n in ('NB', 'G', 'Cin', 'Cout', 'L', 'k', 'dil'))
    shape = _lib.ConvBlockShape(NB, G, Cin, Cout, L, k, dil, 0, 0, 1, 1e-5, 0.1, 0.0, 1)
    lib = _lib.load()
    sh = ctypes.byref(shape)
    saved = F._bytes(lib.b200tts_convblock_saved_bytes(sh), x.device)
    ws = F._bytes(lib.b200tts_convblock_workspace_bytes(sh), x.device)
    out = torch.empty(NB, G * Cout, L, device=x.device)
    dx = torch.empty_like(x)
    dw = torch.zeros_like(w)            # the weight gradient accumulates
    st = F._stream()
    counts = {}
    calls = {
        'out': lambda: F.check(lib.b200tts_convblock_forward(sh, F.ptr(x), F.ptr(w), None, None, Cout, None, None, None, F.ptr(out),
                                                             F.ptr(saved), F.ptr(ws), st), 'b200tts_convblock_forward'),
        'dx': lambda: F.check(lib.b200tts_convblock_backward(sh, F.ptr(x), F.ptr(w), None, None, Cout, None, F.ptr(saved), F.ptr(dout),
                                                             F.ptr(dx), None, None, None, F.ptr(ws), st), 'b200tts_convblock_backward'),
        'dw': lambda: F.check(lib.b200tts_convblock_backward(sh, F.ptr(x), F.ptr(w), None, None, Cout, None, F.ptr(saved), F.ptr(dout),
                                                             None, F.ptr(dw), None, None, F.ptr(ws), st), 'b200tts_convblock_backward'),
    }
    for what, fn in calls.items():
        counts[what] = _call(fn)
    return out, dx, dw, counts


def _reference(c, x, w, dout):
    """fp64 conv1d (zero padding (k - 1) dil / 2 on both sides, G groups) and its gradients, on the GPU."""
    x = x.double().requires_grad_(True)
    w = w.double().requires_grad_(True)
    out = torch.nn.functional.conv1d(x, w, None, 1, (c['k'] - 1) * c['dil'] // 2, c['dil'], c['G'])
    out.backward(dout.double())
    return out.detach(), x.grad, w.grad


ENC = dict(NB=6, G=10, L=180)        # generated_training at the benchmark batch: B = 60 utterances over 10 languages, L = 180
POST = dict(NB=8, G=1, L=900, k=5, dil=1)
CASES = {
    # GeneratedConvolutionalEncoder (encoder_dimension 256, embedding 512): per-group channels
    'enc_in_k1': (dict(ENC, Cin=512, Cout=256, k=1, dil=1), dict(out='gemm', dx='gemm', dw='two-level')),
    'enc_k1': (dict(ENC, Cin=256, Cout=256, k=1, dil=1), dict(out='gemm', dx='gemm', dw='two-level')),
    'enc_highway_k1': (dict(ENC, Cin=256, Cout=512, k=1, dil=1), dict(out='gemm', dx='gemm', dw='two-level')),
    **{f'enc_highway_k3_dil{d}': (dict(ENC, Cin=256, Cout=512, k=3, dil=d), dict(out='implicit', dx='implicit', dw='fused'))
       for d in (1, 3, 9, 27)},
    # postnet at T = 900: the 80 mel channels zero-pad the k-blocks of the forward (Cin) or the input gradient (Cout)
    'post_in': (dict(POST, Cin=80, Cout=512), dict(out='implicit', dx='implicit', dw='fused+splitK')),
    'post_mid': (dict(POST, Cin=512, Cout=512), dict(out='implicit', dx='implicit', dw='fused+splitK')),
    'post_out': (dict(POST, Cin=512, Cout=80), dict(out='implicit', dx='implicit', dw='fused+splitK')),
    # edges
    'L64': (dict(NB=3, G=2, Cin=64, Cout=128, L=64, k=3, dil=1), dict(out='implicit', dx='implicit', dw='fused')),
    'L65': (dict(NB=3, G=2, Cin=64, Cout=128, L=65, k=3, dil=3), dict(out='implicit', dx='implicit', dw='fused')),
    'L100_NB4': (dict(NB=4, G=2, Cin=128, Cout=64, L=100, k=5, dil=2), dict(out='implicit', dx='implicit', dw='fused')),
    'pad_over_quarter_L': (dict(NB=2, G=2, Cin=64, Cout=128, L=80, k=3, dil=27), dict(out='implicit', dx='implicit', dw='fused')),
    'NB1': (dict(NB=1, G=10, Cin=256, Cout=512, L=180, k=3, dil=9), dict(out='implicit', dx='implicit', dw='fused')),
    'NB1_k1': (dict(NB=1, G=10, Cin=256, Cout=512, L=180, k=1, dil=1), dict(out='gemm', dx='gemm', dw='per-row')),
    # x of sample `big` and d out of the next 100x their neighbours': a row shift that reads across a sample boundary shows as a
    # large error
    'big_sample_dil27': (dict(ENC, Cin=256, Cout=512, k=3, dil=27, big=3), dict(out='implicit', dx='implicit', dw='fused')),
    'big_sample_L65': (dict(NB=3, G=2, Cin=64, Cout=128, L=65, k=3, dil=9, big=1), dict(out='implicit', dx='implicit', dw='fused')),
    'big_sample_post': (dict(POST, NB=6, Cin=512, Cout=512, big=2), dict(out='implicit', dx='implicit', dw='fused+splitK')),
}


def _operands(c, seed):
    g = torch.Generator().manual_seed(seed)
    NB, G, Cin, Cout, L, k = (c[n] for n in ('NB', 'G', 'Cin', 'Cout', 'L', 'k'))
    x = torch.randn(NB, G * Cin, L, generator=g)
    w = torch.randn(G * Cout, Cin, k, generator=g)
    dout = torch.randn(NB, G * Cout, L, generator=g)
    # magnitude of each sample's terms, by which the comparison divides: out [NB, 1, 1], dx [NB, 1, 1], dw scalar
    mag = dict(out=torch.ones(NB, 1, 1), dx=torch.ones(NB, 1, 1), dw=1.0)
    if 'big' in c:            # x of sample `big` and d out of the next sample are 100x: every product of the weight gradient <= 100x
        x[c['big']] *= 100.0
        dout[(c['big'] + 1) % NB] *= 100.0
        mag['out'][c['big']] = 100.0
        mag['dx'][(c['big'] + 1) % NB] = 100.0
        mag['dw'] = 100.0
    return x, w, dout, mag


def _compare(name, mode, c, got, ref, mag, atol_per_sqrt_k):
    """rtol 1e-4 and atol atol_per_sqrt_k * sqrt(K), both relative to the magnitude of the element's operands."""
    K = dict(out=c['Cin'] * c['k'], dx=c['Cout'] * c['k'], dw=c['NB'] * c['L'])
    errs = {}
    for n in ('out', 'dx', 'dw'):
        m = mag[n].cuda() if torch.is_tensor(mag[n]) else mag[n]
        a, r = got[n].double() / m, ref[n] / m
        errs[n] = float(((a - r).abs() - 1e-4 * r.abs()).max() / K[n] ** 0.5)
        got[n], ref[n] = a, r
    print(name, mode, {n: f'{e:.2e}' for n, e in errs.items()}, '(max |diff| - 1e-4 |ref|, over sqrt K)')
    for n in ('out', 'dx', 'dw'):
        assert_close(got[n], ref[n], 1e-4, atol_per_sqrt_k * K[n] ** 0.5, f'{name} {mode} {n}')


@pytest.mark.parametrize('name', list(CASES))
def test_conv_bf16_matches_fp64(name):
    from multilingual_text_to_speech_b200 import _lib
    c, expected = CASES[name]
    x, w, dout, mag = _operands(c, sum(map(ord, name)))
    x, w, dout = (t.bfloat16().float().cuda() for t in (x, w, dout))       # what the kernels multiply
    _lib.set_precision('bf16')
    try:
        out, dx, dw, calls = _conv_lib(c, x, w, dout)
    finally:
        _lib.set_precision('fp32')
    paths = {what: _path(what, c, *calls[what]) for what in calls}
    print(name, paths)
    assert paths == expected, (paths, expected)
    r_out, r_dx, r_dw = _reference(c, x, w, dout)
    # measured on an H100 80GB HBM3: at most 6e-6 sqrt(K) beyond the rtol term, over 30x inside the bound
    _compare(name, 'bf16', c, dict(out=out, dx=dx, dw=dw), dict(out=r_out, dx=r_dx, dw=r_dw), mag, 2e-4)


@pytest.mark.parametrize('name', ['enc_in_k1', 'enc_highway_k3_dil27', 'post_in', 'post_out', 'L65', 'NB1', 'big_sample_L65'])
def test_conv_fp32_matches_fp64(name):
    from multilingual_text_to_speech_b200 import _lib
    c, _ = CASES[name]
    x, w, dout, mag = _operands(c, sum(map(ord, name)))
    x, w, dout = (t.cuda() for t in (x, w, dout))
    assert _lib.get_precision() == 'fp32'
    out, dx, dw, calls = _conv_lib(c, x, w, dout)
    assert all(tc == 0 for _, tc in calls.values()), calls         # im2col + fp32 GEMM: no bf16 wgmma product
    r_out, r_dx, r_dw = _reference(c, x, w, dout)
    # measured on an H100 80GB HBM3: at most 3.3e-6 sqrt(K) beyond the rtol term
    _compare(name, 'fp32', c, dict(out=out, dx=dx, dw=dw), dict(out=r_out, dx=r_dx, dw=r_dw), mag, 2e-5)


@pytest.mark.parametrize('G,gd,bn,R,path', [
    (10, 20, 8, 512 * 256 * 3, 'fused'),        # generated_training's k = 3 highway kernel: 264 deb partials
    (10, 20, 8, 256 * 512, 'fused'),            # its first block (512 -> 256, k = 1)
    (10, 20, 8, 1 << 21, 'fused'),
    (5, 10, 4, 512 * 256 * 3, 'unfused'),       # generated_switching (bottleneck 4)
    (5, 10, 4, 256 * 256 + 7, 'unfused'),       # R not a multiple of the 256-wide chunk
])
def test_generator_backward_matches_fp64(G, gd, bn, R, path):
    from multilingual_text_to_speech_b200 import functional as F
    g = torch.Generator().manual_seed(G * 7 + bn + R % 1000)
    e, Wb, bb = torch.randn(G, gd, generator=g), torch.randn(bn, gd, generator=g) / gd ** 0.5, torch.randn(bn, generator=g)
    Wk, bk = torch.randn(R, bn, generator=g) / bn ** 0.5, torch.randn(R, generator=g)
    dout = torch.randn(G, R, generator=g)
    dev = torch.device('cuda:0')
    leaves = [t.to(dev).requires_grad_(True) for t in (e, Wb, bb, Wk, bk)]
    out = F.GeneratorFunction.apply(*leaves)
    launches, _ = _call(lambda: out.backward(dout.to(dev)))
    ref = [t.to(dev).double().requires_grad_(True) for t in (e, Wb, bb, Wk, bk)]
    r_out = (ref[0] @ ref[1].t() + ref[2]) @ ref[3].t() + ref[4]
    r_out.backward(dout.to(dev).double())
    # the library's launches only: fused = one pass over dout / Wk + the tail; unfused = dWk / dbk, deb partials, their reduction,
    # then dWb, dbb and de one launch each
    print(G, gd, bn, R, path, f'{launches} launches')
    assert_close(out, r_out, 1e-5, 1e-5 * float(r_out.abs().max()), 'generator forward')
    # K: R for de / dWb / dbb (through deb = dout . Wk), G for dWk / dbk
    for n, got, r, K in zip(('de', 'dWb', 'dbb', 'dWk', 'dbk'), leaves, ref, (R, R, R, G, G)):
        scale = float(r.grad.abs().max())
        assert_close(got.grad, r.grad, 1e-5, 2e-7 * K ** 0.5 * scale, f'generator {n} (G={G}, bn={bn}, R={R})')
    assert launches == {'fused': 2, 'unfused': 6}[path], launches
