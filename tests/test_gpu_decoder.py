"""GPU parity tests (run on an H100): GEMM, attention step and the fused decoder fwd/bwd through the C ABI
against the CPU oracle / golden vectors of the unmodified reference.  Tolerance: rtol 1e-3, atol 1e-4 (north_star),
alignment argmax bit-exact."""
import pytest
import torch

import decoder_cases as dc
from helpers import GOLDEN_CASES, assert_close
from oracle import tacotron_oracle as O

pytestmark = pytest.mark.gpu


@pytest.fixture(scope='module', autouse=True)
def _built():
    import __graft_entry__ as entry
    entry.build()
    assert torch.cuda.is_available(), 'GPU tests need a CUDA device'


@pytest.mark.parametrize('M,N,K,ta,tb,splitk', [
    (64, 4096, 1312, False, True, 2), (57, 130, 77, False, True, 1), (300, 260, 513, False, False, 1),
    (81, 1024, 2000, True, False, 4), (128, 128, 16, True, True, 1), (1, 1, 1, False, True, 1),
    (200, 81, 1312, False, True, 1), (4096, 288, 640, True, False, 3), (65, 65, 65, False, False, 8),
])
def test_gemm_matches_fp64(M, N, K, ta, tb, splitk):
    from multilingual_text_to_speech_b200 import functional as F
    g = torch.Generator().manual_seed(M * 7 + N * 3 + K)
    a = torch.randn((K, M) if ta else (M, K), generator=g)
    b = torch.randn((N, K) if tb else (K, N), generator=g)
    bias = torch.randn(N, generator=g)
    c0 = torch.randn(M, N, generator=g)
    ref = (a.double().t() if ta else a.double()) @ (b.double().t() if tb else b.double()) * 0.5 + bias.double() + 0.25 * c0.double()
    out = c0.cuda().clone()
    F.gemm(a.cuda(), b.cuda(), ta, tb, bias=bias.cuda(), out=out, beta=0.25, alpha=0.5, splitk=splitk)
    assert_close(out, ref, 1e-4, 1e-4 * (K ** 0.5), f'gemm {M}x{N}x{K}')


def test_gemm_strided_views():
    from multilingual_text_to_speech_b200 import functional as F
    g = torch.Generator().manual_seed(5)
    big_a = torch.randn(100, 300, generator=g).cuda()
    big_b = torch.randn(90, 300, generator=g).cuda()
    a, b = big_a[:, 20:148], big_b[:, 31:159]          # unaligned column offset on b -> scalar path
    out = F.gemm(a, b, False, True)
    assert_close(out, a.double().cpu() @ b.double().cpu().t(), 1e-4, 1e-3, 'strided gemm')


@pytest.mark.parametrize('B,L,M', [(1, 1, 256), (3, 31, 288), (60, 180, 288), (64, 180, 292), (5, 300, 512), (80, 77, 256)])
def test_attention_step_matches_oracle(B, L, M):
    from multilingual_text_to_speech_b200 import functional as F
    D, A, C, K = 1024, 128, 32, 31
    g = torch.Generator().manual_seed(B * 1000 + L)
    rn = lambda *s, scale=1.0: torch.randn(*s, generator=g) * scale   # noqa: E731
    sd = {'a._query.weight': rn(A, D, scale=0.1), 'a._loc_features.weight': rn(C, 1, K, scale=0.3),
          'a._location.weight': rn(A, C, scale=0.3), 'a._bias': rn(1, A, scale=0.1), 'a._energy.weight': rn(1, A, scale=1.5),
          'a._memory.weight': rn(A, M, scale=0.1)}
    memory, query = rn(B, L, M), rn(B, D)
    lens = torch.randint(1, L + 1, (B,), generator=g); lens[0] = L
    mask = O.lengths_to_mask(lens, L)
    cum = torch.rand(B, L, generator=g) * mask
    memT = memory @ sd['a._memory.weight'].t()
    ctx_o, w_o, cum_o = O.attention_step({k: v.double() for k, v in sd.items()}, 'a', query.double(), memory.double(),
                                         memT.double(), cum.double(), mask)
    cum_d = cum.cuda().contiguous()
    ctx, w = F.attention_step(query.cuda(), memory.cuda(), memT.cuda(), lens.cuda(), sd['a._query.weight'].cuda(),
                              sd['a._location.weight'].cuda(), sd['a._loc_features.weight'].cuda(), sd['a._bias'].cuda(),
                              sd['a._energy.weight'].cuda(), cum_d)
    assert_close(w, w_o, 1e-3, 1e-5, 'weights')
    assert_close(ctx, ctx_o, 1e-3, 1e-4, 'context')
    assert_close(cum_d, cum_o, 1e-3, 1e-5, 'cumulative weights')
    assert torch.equal(w.cpu().argmax(1), w_o.argmax(1))
    assert float(w.cpu()[~mask].abs().max() if (~mask).any() else 0.0) == 0.0
    assert_close(w.sum(1), torch.ones(B), 1e-5, 1e-5, 'rows sum to one')


@pytest.mark.parametrize('name', GOLDEN_CASES)
def test_decoder_golden(name):
    dc.run_case(dc.golden_case(name), check_grads=True, verbose=True)


@pytest.mark.parametrize('kw', [
    dict(B=8, L=40, T=30, kind='dropout'),
    dict(B=8, L=40, T=30, kind='zoneout', seed=1),
    dict(B=5, L=33, T=21, M=292, kind='dropout', seed=2),
    dict(B=4, L=50, T=16, M=512, kind='dropout', seed=3, dropout=False),
    dict(B=3, L=20, T=12, kind='dropout', seed=4, tf=0.5),
    dict(B=2, L=20, T=10, kind='zoneout', seed=5, tf=0.0, training=False),
])
def test_decoder_full_dims(kw):
    dc.run_case(dc.full_dim_case(**kw), check_grads=True, verbose=True)


def test_decoder_baseline_shape_properties():
    """BASELINE shape (B=64, L=180, T=900 is too slow for the fp64 oracle): size-independent properties."""
    from multilingual_text_to_speech_b200 import functional as F
    c = dc.full_dim_case(B=64, L=180, T=120, seed=11)
    dev = torch.device('cuda:0')
    cfg, params, memory = dc._cuda_inputs(c, dev)
    with torch.no_grad():
        s1, t1, a1 = F.decoder_forward(cfg, memory, c.target.to(dev), c.lengths.to(dev), params)
        s2, t2, a2 = F.decoder_forward(cfg, memory, c.target.to(dev), c.lengths.to(dev), params)
    assert torch.equal(s1, s2) and torch.equal(a1, a2) and torch.equal(t1, t2), 'decode is not bit-reproducible'
    assert_close(a1.sum(2), torch.ones(64, 120), 1e-5, 1e-5, 'alignment rows sum to one')
    mask = O.lengths_to_mask(c.lengths, 180)
    assert float(a1.cpu()[~mask[:, None, :].expand(-1, 120, -1)].abs().max()) == 0.0
    # causality: the first 60 frames do not depend on later targets
    c2 = dc.full_dim_case(B=64, L=180, T=120, seed=11)
    tgt = c.target.clone(); tgt[:, :, 60:] = 0
    with torch.no_grad():
        s3, _, a3 = F.decoder_forward(cfg, memory, tgt.to(dev), c.lengths.to(dev), params)
    assert torch.equal(s1[:, :60], s3[:, :60]) and torch.equal(a1[:, :60], a3[:, :60])


@pytest.mark.parametrize('M,N,K,ta,tb,splitk', [
    (300, 260, 513, False, True, 1), (256, 4096, 1312, False, True, 1), (81, 1024, 2000, True, False, 4),
    (4096, 288, 640, True, False, 3), (65, 65, 65, False, False, 2), (130, 77, 40, True, True, 1), (1, 7, 3, False, True, 1),
])
def test_gemm_bf16_mode(M, N, K, ta, tb, splitk):
    """bf16 tensor-core mode: exact up to fp32 accumulation order once the operands are rounded to bf16."""
    from multilingual_text_to_speech_b200 import functional as F, _lib
    g = torch.Generator().manual_seed(M + N + K)
    a = torch.randn((K, M) if ta else (M, K), generator=g)
    b = torch.randn((N, K) if tb else (K, N), generator=g)
    bias = torch.randn(N, generator=g)
    ar, br = a.bfloat16().double(), b.bfloat16().double()
    ref = (ar.t() if ta else ar) @ (br.t() if tb else br) + bias.double()
    _lib.set_precision('bf16')
    try:
        # route through the library's dispatching GEMM entry (same C ABI call; the mode selects the kernel)
        out = F.gemm(a.cuda(), b.cuda(), ta, tb, bias=bias.cuda(), splitk=splitk)
    finally:
        _lib.set_precision('fp32')
    assert_close(out, ref, 1e-4, 2e-4 * (K ** 0.5), f'bf16 gemm {M}x{N}x{K}')


@pytest.mark.parametrize('kw', [
    dict(B=8, L=40, T=30, kind='dropout'),
    dict(B=40, L=64, T=24, kind='zoneout', seed=1),
    dict(B=5, L=33, T=21, M=292, kind='dropout', seed=2),
    dict(B=60, L=180, T=16, kind='zoneout', seed=6),
    dict(B=12, L=300, T=12, kind='zoneout', seed=7),            # BASELINE configs[4]: texts up to 300 on the persistent kernels
    dict(B=80, L=50, T=10, kind='dropout', seed=8),             # B > 64 (configs[3..4] run 65 / 80 per GPU): decoded as two slices
    dict(B=65, L=44, T=9, M=292, kind='zoneout', seed=9),
    # memory dim 512 (monolingual default, BASELINE configs[0]): accumulator staging aliased onto the TMA slot, ctx part in several TMA
    # instructions (forward), wgmma N = 96 n-blocks (attention reverse product)
    dict(B=16, L=60, T=14, M=512, kind='zoneout', seed=10),
    dict(B=52, L=300, T=8, M=512, kind='dropout', seed=11),
    dict(B=9, L=37, T=11, M=384, kind='dropout', seed=12),
    dict(B=4, L=40, T=12, D=1280, kind='zoneout', seed=13),      # D = 1280: off the persistent loops, per-step chains in bf16
])
def test_decoder_bf16_perf_mode(kw):
    """bf16 perf mode: persistent weight-stationary TMA + wgmma loops (decoder_persist_tc.cu, decoder_persist_bwd_tc.cu,
    decoder_persist_bwd.cu) + bf16 tensor-core GEMMs; shapes off those loops run the per-step chains in bf16."""
    dc.run_case_bf16(dc.full_dim_case(**kw), check_grads=True, verbose=True)


@pytest.mark.parametrize('M,N,K,ta,tb', [
    (256, 256, 256, False, True), (256, 384, 512, False, True), (300, 260, 513, False, True), (1000, 4096, 1312, False, True),
    (4096, 288, 640, True, False), (513, 130, 2000, True, True), (200, 1000, 96, False, False),
    (128, 1024, 20000, True, False), (81, 1312, 9000, True, False),        # few tiles, long K: split-K over the idle SMs (+ reduction launch)
])
def test_gemm_tcgen05_path(M, N, K, ta, tb):
    """wgmma / TMA GEMM (gemm_tc.cu) against fp64 on bf16-rounded operands, and against the mma.sync kernel."""
    from multilingual_text_to_speech_b200 import functional as F, _lib
    g = torch.Generator().manual_seed(M + 3 * N + 7 * K)
    a = torch.randn((K, M) if ta else (M, K), generator=g)
    b = torch.randn((N, K) if tb else (K, N), generator=g)
    bias = torch.randn(N, generator=g)
    c0 = torch.randn(M, N, generator=g)
    ar, br = a.bfloat16().double(), b.bfloat16().double()
    ref = 0.5 * ((ar.t() if ta else ar) @ (br.t() if tb else br)) + bias.double() + 0.25 * c0.double()
    _lib.set_precision('bf16')
    try:
        n0 = _lib.launch_count()
        out = c0.cuda().clone()
        F.gemm(a.cuda(), b.cuda(), ta, tb, bias=bias.cuda(), out=out, alpha=0.5, beta=0.25)
        used = _lib.launch_count() - n0
        _lib.set_tensor_core_gemm(False)
        out2 = c0.cuda().clone()
        F.gemm(a.cuda(), b.cuda(), ta, tb, bias=bias.cuda(), out=out2, alpha=0.5, beta=0.25)
    finally:
        _lib.set_tensor_core_gemm(True)
        _lib.set_precision('fp32')
    assert used in (3, 4), f'expected pack + pack + wgmma kernel (+ split-K reduction), saw {used} launches'
    assert_close(out, ref, 1e-4, 2e-4 * (K ** 0.5), f'wgmma gemm {M}x{N}x{K}')
    assert_close(out, out2, 1e-4, 2e-4 * (K ** 0.5), 'wgmma vs mma.sync')
