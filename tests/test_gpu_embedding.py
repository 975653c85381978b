"""The embedding gather / scatter (`embedding_fwd_kernel`, `embedding_bwd_kernel` in csrc/encoder.cu) through the C ABI.

Forward: bitwise table[ids]; with a row stride ldo > E the columns past E are left untouched.
Backward: dtable[v] += the sum of d out over the tokens with id v.  The kernel compacts each 1024-token tile's hits in token order
(4 tokens per thread) and adds them serially into one fp32 register per column, then once into dtable, so each element is
within (hits - 1) 2^-24 sum |terms| of the fp64 index_add_, plus one rounding of the final +=.  Covered: one and several tiles
(ntok up to 10,800 = the benchmark's 60 x 180 tokens), E across the 256-column and 4-columns-per-thread edges, a row hit 2,500 times
over three tiles, ldo != E, every token padding, accumulation into an existing gradient, bitwise reproducibility and the E > 1024
refusal.
"""
import pytest
import torch

from step_check import U

pytestmark = pytest.mark.gpu

SENT = 0x7fa1b2c3          # a NaN bit pattern no kernel writes


@pytest.fixture(scope='module', autouse=True)
def _built():
    import __graft_entry__ as entry
    entry.build()
    assert torch.cuda.is_available()


def _fwd(out, ldo, table, ids, E):
    from multilingual_text_to_speech_b200 import _lib, functional as F
    F.check(_lib.load().b200tts_embedding_forward(F.ptr(out), ldo, F.ptr(table), F.ptr(ids), ids.numel(), E, F._stream()),
            'b200tts_embedding_forward')


def _bwd(dtable, V, dout, ldo, ids, E, padding_idx):
    from multilingual_text_to_speech_b200 import _lib, functional as F
    F.check(_lib.load().b200tts_embedding_backward(F.ptr(dtable), V, F.ptr(dout), ldo, F.ptr(ids), ids.numel(), E, padding_idx,
                                                   F._stream()), 'b200tts_embedding_backward')


def _ids(ntok, V, seed, heavy=None):
    g = torch.Generator().manual_seed(seed)
    ids = torch.randint(0, V, (ntok,), generator=g, dtype=torch.int32)
    if heavy is not None:
        v, hits = heavy
        ids[ids == v] = (v + 1) % V
        ids[torch.randperm(ntok, generator=g)[:hits]] = v
    return ids


def _check_backward(dtable, d0, dout, ids, V, E, padding_idx, what):
    """dtable (kernel) against d0 + fp64 index_add_ of the tokens' rows, each element within its serial-sum bound."""
    ids64 = ids.long().cuda()
    rows = dout.double()
    keep = ids64 != padding_idx
    ref = d0.double().index_add(0, ids64[keep], rows[keep])
    mag = torch.zeros_like(ref).index_add_(0, ids64[keep], rows[keep].abs())
    hits = torch.zeros(V, dtype=torch.float64, device='cuda').index_add_(0, ids64[keep], torch.ones_like(ids64[keep], dtype=torch.float64))
    bound = ((hits - 1).clamp(min=0)[:, None] * U * mag + U * (d0.double().abs() + mag)) * 1.01
    err = (dtable.double() - ref).abs()
    ratio = torch.where(err == 0, torch.zeros_like(err), err / bound)
    print(f'{what}: worst err/bound {float(ratio.max()):.3e}, most hits {int(hits.max())}')
    assert float(ratio.max()) <= 1.0, what
    if padding_idx >= 0:
        assert torch.equal(dtable[padding_idx], d0[padding_idx]), f'{what}: the padding row changed'
    return hits


@pytest.mark.parametrize('E', [1, 255, 256, 257, 512, 1024])
@pytest.mark.parametrize('ntok', [1, 1023, 1024, 1025, 10800])
def test_embedding_matches_fp64(ntok, E):
    V, pad = 70, 0
    ldo = E + 7 if ntok in (1, 1025) else E
    g = torch.Generator().manual_seed(ntok * 31 + E)
    table = torch.randn(V, E, generator=g).cuda()
    ids = _ids(ntok, V, ntok + E).cuda()
    # forward: bitwise gather; the 7 columns past E of every output row keep their sentinel
    buf = torch.full((ntok, E + 7), SENT, dtype=torch.int32, device='cuda')
    _fwd(buf.view(torch.float32), E + 7, table, ids, E)
    torch.cuda.synchronize()
    assert torch.equal(buf[:, :E].view(torch.float32), table[ids.long()])
    assert bool((buf[:, E:] == SENT).all()), 'forward wrote past E'
    # backward into an existing gradient, twice: the second run must be bitwise equal
    dout = torch.randn(ntok, ldo, generator=g).cuda()
    d0 = torch.randn(V, E, generator=g).cuda()
    results = []
    for _ in range(2):
        dtable = d0.clone()
        _bwd(dtable, V, dout, ldo, ids, E, pad)
        torch.cuda.synchronize()
        results.append(dtable)
    assert torch.equal(results[0], results[1]), 'embedding backward is not reproducible'
    _check_backward(results[0], d0, dout[:, :E], ids, V, E, pad, f'ntok {ntok} E {E} ldo {ldo}')


@pytest.mark.parametrize('E', [256, 257, 1024])
def test_embedding_backward_row_hit_2500_times(E):
    """One id hit 2,500 times among 10,800 tokens: its hits span at least three 1024-token tiles, in per-tile counts that are not
    all multiples of 4."""
    V, pad, ntok, heavy = 70, 0, 10800, 5
    ids = _ids(ntok, V, 17, heavy=(heavy, 2500))
    per_tile = torch.bincount(torch.nonzero(ids == heavy).flatten() // 1024)
    assert int((ids == heavy).sum()) == 2500 and int((per_tile > 0).sum()) >= 3 and bool((per_tile % 4 != 0).any())
    g = torch.Generator().manual_seed(E)
    dout = torch.randn(ntok, E, generator=g).cuda()
    dtable = torch.zeros(V, E, device='cuda')
    _bwd(dtable, V, dout, E, ids.cuda(), E, pad)
    torch.cuda.synchronize()
    hits = _check_backward(dtable, torch.zeros_like(dtable), dout, ids, V, E, pad, f'2,500 hits E {E}')
    assert int(hits[heavy]) == 2500


def test_embedding_backward_all_padding():
    V, E, ntok, pad = 70, 257, 3000, 3
    ids = torch.full((ntok,), pad, dtype=torch.int32, device='cuda')
    d0 = torch.randn(V, E, device='cuda')
    dtable = d0.clone()
    _bwd(dtable, V, torch.randn(ntok, E, device='cuda'), E, ids, E, pad)
    torch.cuda.synchronize()
    assert torch.equal(dtable, d0)


def test_embedding_function_accumulates_into_grad():
    """Through autograd: an existing .grad of the table is accumulated into (+=); the padding row gets nothing."""
    from multilingual_text_to_speech_b200 import functional as F
    V, E, pad = 70, 512, 0
    g = torch.Generator().manual_seed(4)
    table = torch.randn(V, E, generator=g).cuda().requires_grad_(True)
    g0 = torch.randn(V, E, generator=g).cuda()
    table.grad = g0.clone()
    ids = _ids(60 * 180, V, 5).cuda().view(60, 180)
    dout = torch.randn(60, 180, E, generator=g).cuda()
    out = F.embedding(table, ids, padding_idx=pad)
    assert torch.equal(out, table.detach()[ids.long()])
    out.backward(dout)
    torch.cuda.synchronize()
    _check_backward(table.grad, g0, dout.view(-1, E), ids.view(-1), V, E, pad, 'autograd += into .grad')


def test_embedding_backward_refuses_e_over_1024():
    from multilingual_text_to_speech_b200 import _lib
    V, E, ntok = 8, 1025, 16
    buf = torch.full((V * E,), SENT, dtype=torch.int32, device='cuda')
    ids = torch.zeros(ntok, dtype=torch.int32, device='cuda')
    with pytest.raises(_lib.B200TTSError, match='embedding dimension 1025 > 1024'):
        _bwd(buf.view(torch.float32), V, torch.ones(ntok, E, device='cuda'), E, ids, E, -1)
    torch.cuda.synchronize()
    assert bool((buf == SENT).all()), 'dtable changed'
