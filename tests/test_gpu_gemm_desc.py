"""The GEMM descriptor (GemmDesc) on every kernel path against the fp64 oracle of tests/gemm_cases.py, through
b200tts_debug_gemm: batches with strides and gaps, a_batch_mod, bf16 operands read in place (A16 K-major and MN-major, B16),
two-level K, explicit split-K with kept partials, the wgmma split-K and its scratch limits, the pack cache, gemm_run_auto.

Each call asserts the path that ran (library launches and wgmma GEMM launches, as tests/test_gpu_conv_exact.py does), that a
second identical call is bit-identical (the library uses no atomics), and that nothing stale is read: C is NaN when beta == 0,
every element the descriptor does not cover is NaN, the wgmma scratch is filled with 0xFF bytes (bf16 NaN) before every call made
outside a pack-cache scope and the partial buffer with NaN; the result must be finite, and C outside the output untouched.
"""
import ctypes
from types import SimpleNamespace

import pytest
import torch

import gemm_cases as gc
from helpers import assert_close

pytestmark = pytest.mark.gpu

ERR_INVALID = -1


@pytest.fixture(scope='module', autouse=True)
def _built():
    import __graft_entry__ as entry
    entry.build()
    assert torch.cuda.is_available()


def _L():
    from multilingual_text_to_speech_b200 import _lib
    return _lib


def _scratch():
    """(1024-aligned base, bytes) of the full library scratch."""
    s = _L().ensure_scratch()
    return (s.data_ptr() + 1023) // 1024 * 1024, s.numel() - 1024


def _set_scratch(nbytes):
    L = _L()
    L.check(L.load().b200tts_set_scratch(ctypes.c_void_p(_scratch()[0]), nbytes), 'b200tts_set_scratch')


def _pack_cache(open_):
    L = _L()
    L.check(L.load().b200tts_debug_gemm_pack_cache(int(open_)), 'b200tts_debug_gemm_pack_cache')


@pytest.fixture(autouse=True)
def _library_state():
    """Whatever a test changes, the next one starts from fp32, tensor-core GEMM on, the full scratch and the pack cache closed."""
    L = _L()
    L.ensure_scratch()
    try:
        yield
    finally:
        torch.cuda.synchronize()
        L.kernel_timing(False)
        _pack_cache(False)
        _set_scratch(_scratch()[1])
        L.set_tensor_core_gemm(True)
        L.set_precision('fp32')


def _route(route):
    L = _L()
    L.set_precision('fp32' if route in ('f32', 'auto_f32') else 'bf16')
    L.set_tensor_core_gemm(route != 'mma')


def _dev(ops):
    cu = lambda t: None if t is None else t.cuda()      # noqa: E731
    return SimpleNamespace(A=cu(ops.A), B=cu(ops.B), C0=cu(ops.C0), bias=cu(ops.bias), A16=cu(ops.A16), B16=cu(ops.B16))


def _desc(c, d, C, partial):
    L = _L()
    g = L.GemmDesc()
    ptr = lambda t: None if t is None else t.data_ptr()      # noqa: E731
    g.A, g.B, g.C, g.bias, g.partial = ptr(d.A), ptr(d.B), ptr(C), ptr(d.bias), ptr(partial)
    g.A16, g.B16 = ptr(d.A16) if c.a16 else None, ptr(d.B16) if c.b16 else None
    for f in ('M', 'N', 'K', 'lda', 'ldb', 'ldc', 'batch', 'strideA', 'strideB', 'strideC', 'a_batch_mod', 'splitk', 'keep_partials',
              'lda16', 'ldb16', 'kin', 'kosA', 'kosB'):
        setattr(g, f, getattr(c, f))
    g.transA, g.transB, g.alpha, g.beta = c.ta, c.tb, c.alpha, c.beta
    return g


def _call(c, route, d, C, partial=None, poison=True):
    """One b200tts_debug_gemm call: (status, library launches, wgmma GEMM launches)."""
    L = _L()
    lib = L.load()
    if poison:
        L._scratch.fill_(0xFF)
    if partial is not None:
        partial.fill_(float('nan'))
    auto = route.startswith('auto')
    g = _desc(c, d, C, None if auto else partial)
    torch.cuda.synchronize()
    L.kernel_timing(True)
    n0 = L.launch_count()
    try:
        st = lib.b200tts_debug_gemm(ctypes.byref(g), int(auto), ctypes.c_void_p(partial.data_ptr()) if auto and partial is not None else None,
                                    partial.numel() if auto and partial is not None else 0, None)
        torch.cuda.synchronize()
        n = L.launch_count() - n0
        tc = L.kernel_timing_read().get('gemm_tc_kernel', (0.0, 0))[1]
    finally:
        L.kernel_timing(False)
    return st, n, tc


def _bits(t):
    return t.view(torch.int32) if t.dtype == torch.float32 else t.view(torch.int16)


def _assert_matches(actual, expected, rtol, atol, what):
    assert bool(torch.isfinite(actual).all()), f'{what}: {int((~torch.isfinite(actual)).sum())} non-finite values (a stale or out-of-range read)'
    assert_close(actual, expected, rtol, atol, what)


def _check(c, route, ops, C, C0, partial, what):
    """C (and the kept partials) against the oracle; C outside the output untouched."""
    bf16 = route in gc.BF16_ROUTES
    rtol, atol = gc.tolerance(c, route)
    idx = torch.from_numpy(gc.c_index(c).reshape(-1)).cuda()
    outside = torch.ones(C.numel(), dtype=torch.bool, device=C.device)
    outside[idx] = False
    assert torch.equal(_bits(C)[outside], _bits(C0)[outside]), f'{what}: wrote outside the output'
    if c.keep_partials:
        assert torch.equal(_bits(C), _bits(C0)), f'{what}: keep_partials changed C'
        p = partial.view(c.splitk, c.batch, c.M, c.N)
        want = gc.partials(c, ops, bf16, gc.kchunk(c, route))
        for s in range(c.splitk):
            _assert_matches(p[s], want[s], rtol, atol, f'{what}: partial {s}')
        _assert_matches(p.double().sum(0), gc.reference(c, ops, bf16), rtol, atol, f'{what}: sum of the partials')
    else:
        _assert_matches(C[idx].view(c.batch, c.M, c.N), gc.reference(c, ops, bf16), rtol, atol, what)


def _run_checked(c, route, ops, d, want, partial_elems=0, poison=True, explicit_partial=True, want_again=None):
    """Run c, assert the launches `want` = (library, wgmma), check against the oracle, repeat bit-identically (expecting
    `want_again` launches the second time, when a pack-cache scope holds the operands by then); return C."""
    elems = c.splitk * c.batch * c.M * c.N if (explicit_partial and c.splitk > 1) else partial_elems
    runs = []
    for want in (want, want_again or want):
        C = d.C0.clone()
        partial = torch.empty(elems, device='cuda') if elems else None
        st, n, tc = _call(c, route, d, C, partial, poison)
        _L().check(st, f'{c.name} on {route}')
        assert (n, tc) == want, f'{c.name} on {route}: expected {want[0]} launches / {want[1]} wgmma, saw {n} / {tc}'
        _check(c, route, ops, C, d.C0, partial, f'{c.name} on {route}')
        runs.append((C, partial))
    (c1, p1), (c2, p2) = runs
    assert torch.equal(_bits(c1), _bits(c2)), f'{c.name} on {route}: not bit-reproducible'
    if c.keep_partials:
        assert torch.equal(_bits(p1), _bits(p2)), f'{c.name} on {route}: partials not bit-reproducible'
    return c1


@pytest.mark.parametrize('name,route', [(c.name, r) for c in gc.CASES for r in c.routes if not r.startswith('auto')])
def test_descriptor_on_each_path(name, route):
    c = gc.BY_NAME[name]
    ops = gc.operands(c)
    _route(route)
    d = _dev(ops)
    path, launches, tc = gc.expected_path(c, route, _scratch()[1])
    print(f'{name} on {route}: {path}')
    if path == 'rejected':
        C = d.C0.clone()
        st, n, ntc = _call(c, route, d, C)
        assert st == ERR_INVALID and (n, ntc) == (0, 0), f'{name} on {route}: status {st}, {n} launches: two-level K not refused'
        assert b'two-level K' in _L().load().b200tts_last_error()
        assert torch.equal(_bits(C), _bits(d.C0))
        return
    _run_checked(c, route, ops, d, (launches, tc))


@pytest.mark.parametrize('size', ['none', 'preferred', 'short'])
@pytest.mark.parametrize('name,route', [(c.name, r) for c in gc.CASES for r in c.routes if r.startswith('auto')])
def test_auto_split(name, route, size):
    """gemm_run_auto without a partial buffer, with one that holds its preferred split, and with one that forces half of it."""
    c = gc.BY_NAME[name]
    ops = gc.operands(c)
    _route(route)
    d = _dev(ops)
    pref = gc.auto_split(c, route == 'auto_bf16', 1 << 40)
    elems = {'none': 0, 'preferred': pref, 'short': pref // 2}[size] * c.batch * c.M * c.N
    path, launches, tc = gc.expected_path(c, route, _scratch()[1], elems)
    print(f'{name} on {route}, {size} partial buffer: {path}')
    if size == 'short' and tc == 0:
        assert 1 < gc.auto_split(c, route == 'auto_bf16', elems) < pref
    _run_checked(c, route, ops, d, (launches, tc), partial_elems=elems, explicit_partial=False)


def test_tc_splitk_scratch_limits():
    """The wgmma split-K product; the same with a scratch that holds the packs but not the partials (un-split: one launch fewer);
    and with one too small for the packs (mma.sync, no wgmma launch).  All three match the oracle."""
    c = gc.BY_NAME['tc_splitk']
    ops = gc.operands(c)
    _route('wgmma')
    d = _dev(ops)
    full = _scratch()[1]
    plan = gc.tc_plan(c, full)
    assert plan.ksplit > 1
    packs = int(plan.pack_a) + int(plan.pack_b)
    out = {}
    for label, nbytes, want in (('split', full, (packs + 2, 1)), ('packs only', plan.a_bytes + plan.b_bytes + 1024, (packs + 1, 1)),
                                ('no room for the packs', plan.a_bytes + plan.b_bytes - 1024, (1, 0))):
        _set_scratch(nbytes)
        assert gc.expected_path(c, 'wgmma', nbytes)[1:] == want
        print(f'tc_splitk, {label}: {gc.expected_path(c, "wgmma", nbytes)[0]}')
        out[label] = _run_checked(c, 'wgmma', ops, d, want)
    rtol, atol = gc.tolerance(c, 'wgmma')
    _assert_matches(out['packs only'], out['split'], rtol, atol, 'un-split vs split')


def _shared_a_cases():
    M, K = 250, 700
    cases = [gc.make(f'shared_a_{i}', M, N, K, 1, 0, beta=0.5, seed=40 + i) for i, N in enumerate((130, 200, 100))]
    ops = [gc.operands(x) for x in cases]
    for o in ops[1:]:
        o.A = ops[0].A
    return cases, ops


def test_pack_cache_shares_one_transposed_operand():
    """Three weight-gradient products of one transA operand (the decoder backward's pattern): inside a scope only the first packs it,
    and each product is bit-identical to the same product with the scope closed."""
    _route('wgmma')
    cases, ops = _shared_a_cases()
    devs = [_dev(o) for o in ops]
    for d in devs[1:]:
        d.A = devs[0].A
    closed = []
    for c, o, d in zip(cases, ops, devs):
        path, n, tc = gc.expected_path(c, 'wgmma', _scratch()[1])
        assert (n, tc) == (3, 1), path                # pack A, pack B, GEMM; no split-K
        closed.append(_run_checked(c, 'wgmma', o, d, (n, tc)))
    _L()._scratch.fill_(0xFF)
    _pack_cache(True)
    try:
        for i, (c, o, d) in enumerate(zip(cases, ops, devs)):
            C = _run_checked(c, 'wgmma', o, d, (3, 1) if i == 0 else (2, 1), poison=False, want_again=(1, 1))
            assert torch.equal(_bits(C), _bits(closed[i])), f'{c.name}: cached pack differs from a fresh one'
    finally:
        _pack_cache(False)


def test_pack_cache_views_of_one_pointer():
    """Views of one buffer with another row stride or another K inside one scope are distinct cache entries."""
    _route('wgmma')
    g = torch.Generator().manual_seed(77)
    X, Y = torch.randn(200 * 330 + 100, generator=g), torch.randn(330 * 300, generator=g)
    views = [gc.make('view_ld320', 200, 330, 300, 0, 1, lda=320, ldb=300), gc.make('view_ld330', 200, 330, 300, 0, 1, lda=330, ldb=300),
             gc.make('view_k256', 200, 330, 256, 0, 1, lda=320, ldb=300)]
    dX, dY = X.cuda(), Y.cuda()
    _L()._scratch.fill_(0xFF)
    _pack_cache(True)
    try:
        first = None
        for c, want in zip(views + views[:1], ((3, 1), (2, 1), (3, 1), (1, 1))):
            ops = SimpleNamespace(A=X, B=Y, C0=torch.full((c.M * c.ldc,), float('nan')), bias=None, A16=None, B16=None)
            d = SimpleNamespace(A=dX, B=dY, C0=ops.C0.cuda(), bias=None, A16=None, B16=None)
            C = _run_checked(c, 'wgmma', ops, d, want, poison=False, want_again=(1, 1))
            if first is None:
                first = C
        assert torch.equal(_bits(C), _bits(first))
    finally:
        _pack_cache(False)


def test_pack_cache_beyond_its_entries():
    """More operands than the cache has entries (MAX_CACHE) in one scope: every product stays correct, the early ones stay cached."""
    _route('wgmma')
    n = gc.MAX_CACHE // 2 + 2
    cases = [gc.make(f'many_{i}', 72, 80, 3000, 0, 1, bias=True, seed=100 + i) for i in range(n)]
    ops = [gc.operands(c) for c in cases]
    devs = [_dev(o) for o in ops]
    assert gc.expected_path(cases[0], 'wgmma')[1:] == (3, 1)
    _L()._scratch.fill_(0xFF)
    _pack_cache(True)
    try:
        # the first MAX_CACHE / 2 products fill the cache (their repeat finds both operands there); the rest are packed every time
        first = [_run_checked(c, 'wgmma', o, d, (3, 1), poison=False, want_again=(1, 1) if i < gc.MAX_CACHE // 2 else (3, 1))
                 for i, (c, o, d) in enumerate(zip(cases, ops, devs))]
        again0 = _run_checked(cases[0], 'wgmma', ops[0], devs[0], (1, 1), poison=False)
        again_last = _run_checked(cases[-1], 'wgmma', ops[-1], devs[-1], (3, 1), poison=False)
        assert torch.equal(_bits(again0), _bits(first[0])) and torch.equal(_bits(again_last), _bits(first[-1]))
    finally:
        _pack_cache(False)
