"""bf16 perf-mode convolution paths of the conv block (implicit wgmma convolution forward / input gradient, fused weight
gradient) against the library's own fp32 parity path (itself pinned to the reference by the golden model tests)."""
import pytest
import torch

pytestmark = pytest.mark.gpu


@pytest.fixture(scope='module', autouse=True)
def _built():
    import __graft_entry__ as entry
    entry.build()
    assert torch.cuda.is_available()


def _rel(a, b):
    return float((a.double() - b.double()).abs().sum() / b.double().abs().sum().clamp_min(1e-30))


@pytest.mark.parametrize('cfg', [
    dict(NB=3, G=2, Cin=64, Cout=128, L=100, k=5, dil=1, highway=True, act='tanh'),      # grouped, highway (Cout = 2 Cin)
    dict(NB=2, G=1, Cin=128, Cout=128, L=77, k=3, dil=2, highway=False, act='relu'),     # dilated
    dict(NB=4, G=1, Cin=64, Cout=80, L=130, k=5, dil=1, highway=False, act='identity'),  # Cout % 64 != 0 (postnet's last layer): zero-padded k-blocks in the input gradient
    dict(NB=3, G=1, Cin=80, Cout=128, L=150, k=5, dil=1, highway=False, act='tanh'),     # Cin % 64 != 0 (postnet's first layer): zero-padded k-blocks in the forward
    dict(NB=6, G=10, Cin=64, Cout=128, L=64, k=3, dil=4, highway=True, act='relu'),      # 10 language groups
])
def test_convblock_bf16_paths_match_fp32(cfg):
    from multilingual_text_to_speech_b200 import functional as F, _lib
    NB, G, Cin, Cout, L, k, dil = (cfg[n] for n in ('NB', 'G', 'Cin', 'Cout', 'L', 'k', 'dil'))
    g = torch.Generator().manual_seed(NB * 1000 + L)
    dev = torch.device('cuda:0')
    x0 = torch.randn(NB, G * Cin, L, generator=g).to(dev)
    w0 = (torch.randn(G * Cout, Cin, k, generator=g) / (Cin * k) ** 0.5).to(dev)
    gamma0 = (1.0 + 0.1 * torch.randn(G * Cout, generator=g)).to(dev)
    beta0 = (0.1 * torch.randn(G * Cout, generator=g)).to(dev)
    Cf = Cout // 2 if cfg['highway'] else Cout
    probe = torch.randn(NB, G * Cf, L, generator=g).to(dev)
    res = {}
    for mode in ('fp32', 'bf16'):
        _lib.set_precision(mode)
        try:
            x, w = x0.clone().requires_grad_(True), w0.clone().requires_grad_(True)
            gamma, beta = gamma0.clone().requires_grad_(True), beta0.clone().requires_grad_(True)
            rm, rv = torch.zeros(G * Cout, device=dev), torch.ones(G * Cout, device=dev)
            out = F.conv_block(x, w, gamma, beta, rm, rv, None, G, k, dil, cfg['act'], cfg['highway'], True, 1e-5, 0.1, 0.0, Cout)
            (out * probe).sum().backward()
            res[mode] = dict(out=out.detach(), dx=x.grad, dw=w.grad, dgamma=gamma.grad, dbeta=beta.grad, rm=rm, rv=rv)
        finally:
            _lib.set_precision('fp32')
    errs = {n: _rel(res['bf16'][n], res['fp32'][n]) for n in res['fp32']}
    print(cfg, errs)
    # bf16 operands (8 mantissa bits), fp32 accumulation: the block output differs norm-wise by a few 1e-3; the gradients pass through
    # the batch-norm backward (differences of nearly equal sums), which amplifies the operand rounding to the percent level
    assert errs['out'] < 1e-2, errs
    for n in ('dx', 'dw', 'dgamma', 'dbeta'):
        assert errs[n] < 6e-2, (n, errs)
    assert errs['rm'] < 1e-2 and errs['rv'] < 1e-2, errs
