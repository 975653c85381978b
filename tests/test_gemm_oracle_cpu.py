"""CPU checks of the fp64 GEMM-descriptor oracle (tests/gemm_cases.py) that tests/test_gpu_gemm_desc.py compares every kernel path
with: the oracle agrees with torch on strided views, the two-level K is the sum of its slabs, a_batch_mod is a per-batch loop, the
split-K partials sum to the product; and each case's tolerance is tight enough that a subtly wrong kernel (a k-block dropped, the
wrong A group, a kin slab at the wrong offset, bias left out, beta on the wrong C) would fail it."""
import math

import pytest
import torch

import gemm_cases as gc


def _view_a(c, A, group, q=None):
    """op(A) of one group [M, K] (or of slab q [M, kin]) as a torch strided view of the flat buffer."""
    off = group * c.strideA
    if q is not None:
        return torch.as_strided(A, (c.M, c.kin), (c.lda, 1), off + q * c.kosA)
    return torch.as_strided(A, (c.K, c.M), (c.lda, 1), off).t() if c.ta else torch.as_strided(A, (c.M, c.K), (c.lda, 1), off)


def _view_b(c, B, bz, q=None):
    off = bz * c.strideB
    if q is not None:
        return torch.as_strided(B, (c.N, c.kin), (c.ldb, 1), off + q * c.kosB).t()
    return torch.as_strided(B, (c.N, c.K), (c.ldb, 1), off).t() if c.tb else torch.as_strided(B, (c.K, c.N), (c.ldb, 1), off)


def _epilogue(c, ops, prod):
    out = c.alpha * prod
    if c.bias:
        out = out + ops.bias.double()
    if c.beta != 0:
        out = out + c.beta * torch.as_strided(ops.C0, (c.batch, c.M, c.N), (c.strideC, c.ldc, 1)).double()
    return out


@pytest.mark.parametrize('name', [c.name for c in gc.CASES if not c.kin and not c.a_batch_mod])
@pytest.mark.parametrize('bf16', [False, True])
def test_oracle_matches_torch_views(name, bf16):
    c = gc.BY_NAME[name]
    ops = gc.operands(c)
    cast = (lambda t: t.bfloat16().double()) if bf16 else (lambda t: t.double())       # noqa: E731
    a = torch.stack([cast(_view_a(c, ops.A, z)) for z in range(c.batch)])
    b = torch.stack([cast(_view_b(c, ops.B, z)) for z in range(c.batch)])
    want = _epilogue(c, ops, torch.einsum('zmk,zkn->zmn', a, b))
    got = gc.reference(c, ops, bf16)
    assert torch.allclose(got, want, rtol=1e-12, atol=1e-10)
    assert bool(torch.isfinite(got).all())


@pytest.mark.parametrize('name', [c.name for c in gc.CASES if c.kin])
def test_two_level_k_is_the_sum_of_its_slabs(name):
    c = gc.BY_NAME[name]
    ops = gc.operands(c)
    prod = torch.zeros(c.batch, c.M, c.N, dtype=torch.float64)
    for z in range(c.batch):
        for q in range(c.kouter):
            prod[z] += _view_a(c, ops.A, z, q).double() @ _view_b(c, ops.B, z, q).double()
    assert torch.allclose(gc.reference(c, ops, False), _epilogue(c, ops, prod), rtol=1e-12, atol=1e-9)


@pytest.mark.parametrize('name', [c.name for c in gc.CASES if c.a_batch_mod])
def test_a_batch_mod_is_a_per_batch_loop(name):
    c = gc.BY_NAME[name]
    ops = gc.operands(c)
    prod = torch.stack([_view_a(c, ops.A, z % c.a_batch_mod).double() @ _view_b(c, ops.B, z).double() for z in range(c.batch)])
    assert torch.allclose(gc.reference(c, ops, False), _epilogue(c, ops, prod), rtol=1e-12, atol=1e-10)


@pytest.mark.parametrize('name', [c.name for c in gc.CASES if c.splitk > 1])
def test_split_partials_sum_to_the_product(name):
    c = gc.BY_NAME[name]
    ops = gc.operands(c)
    for route in c.routes:
        bf16 = route in gc.BF16_ROUTES
        chunk = gc.kchunk(c, route)
        assert chunk % gc.KBLOCK[route] == 0 and (c.splitk - 1) * chunk < c.K <= c.splitk * chunk
        p = gc.partials(c, ops, bf16, chunk)
        assert torch.allclose(_epilogue(c, ops, p.sum(0)), gc.reference(c, ops, bf16), rtol=1e-12, atol=1e-10)


@pytest.mark.parametrize('name', [c.name for c in gc.CASES])
def test_mutations_fall_outside_the_gpu_tolerance(name):
    """The suite's teeth: on the case's own operands, every applicable one-off mistake of the oracle is outside the tolerance the GPU
    test uses on each of the case's routes, while the exact oracle is inside it."""
    c = gc.BY_NAME[name]
    ops = gc.operands(c)
    checked = 0
    for route in c.routes:
        bf16 = route in gc.BF16_ROUTES
        rtol, atol = gc.tolerance(c, route)
        exact = gc.reference(c, ops, bf16)
        assert gc.within(exact, exact, rtol, atol)
        for mutation in gc.MUTATIONS:
            if not gc.applicable(c, mutation):
                continue
            wrong = gc.reference(c, ops, bf16, mutation, kblock=gc.route_kblock(c, route))
            assert not gc.within(wrong, exact, rtol, atol), f'{route}: mutation {mutation} is inside the tolerance'
            checked += 1
    assert checked >= 1


def test_case_table_meets_the_preconditions():
    """Every descriptor the GPU test sends meets the documented preconditions, sits off the tile multiples, and reaches the path
    it is meant for: wgmma cases clear that path's limits (taken with the full scratch), two-level K is refused by f32 / mma.sync."""
    for c in gc.CASES:
        assert c.M % 64 and c.N % 64, c.name
        assert (c.lda >= (c.M if c.ta else (c.kin or c.K))) and c.ldb >= (c.kin or (c.K if c.tb else c.N)) and c.ldc >= c.N, c.name
        if c.a16:
            assert c.batch == 1 and c.lda16 % 8 == 0 and c.lda16 >= (c.M if c.ta else c.K), c.name
            if c.ta:
                assert c.lda16 % 64 == 0 and c.M % 64 != 0, c.name
        if c.b16:
            assert c.batch == 1 and not c.tb and c.ldb16 == gc.cdiv(c.N, 64) * 64 and c.N % 64 != 0, c.name
        if c.kin:
            assert c.kin % 64 and c.K % c.kin == 0 and not c.ta and c.tb, c.name
            # slabs do not overlap, and a gap separates them
            assert c.kosA > (c.a_groups - 1) * c.strideA + c.M * c.lda and c.kosB > (c.batch - 1) * c.strideB + c.N * c.ldb, c.name
        for route in c.routes:
            path, launches, tc = gc.expected_path(c, route)
            if route == 'wgmma':
                assert tc == 1, f'{c.name}: the wgmma path declines it ({path})'
            if c.kin and route in ('f32', 'mma'):
                assert path == 'rejected'
    assert any(c.K % 8 for c in gc.CASES if 'wgmma' in c.routes)
    kin = gc.BY_NAME['kin_splitk']
    assert kin.K >= 4096 and gc.tc_plan(kin, gc.SCRATCH_BYTES).ksplit > 1      # two-level K and wgmma split-K together
    assert gc.tc_plan(gc.BY_NAME['tc_splitk'], gc.SCRATCH_BYTES).ksplit > 1
    assert gc.expected_path(gc.BY_NAME['a16_b16'], 'wgmma')[1:] == (1, 1)      # A16 + B16: the GEMM alone


def test_bf16_operands_round_to_nearest_even():
    """The oracle's bf16 rounding is round-to-nearest-even, the rounding of the kernels' cvt.rn.bf16."""
    x = torch.tensor([1.0 + 2.0 ** -8, 1.0 + 3 * 2.0 ** -8, -(1.0 + 2.0 ** -8), 1.0 + 2.0 ** -8 + 2.0 ** -20])
    assert x.bfloat16().double().tolist() == [1.0, 1.0 + 2.0 ** -6, -1.0, 1.0 + 2.0 ** -7]
    assert math.isnan(float(torch.tensor(float('nan')).bfloat16()))
