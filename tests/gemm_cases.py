"""fp64 oracle of the GEMM descriptor contract (GemmDesc, csrc/common.cuh) and the case table shared by the CPU checks of the
oracle (tests/test_gemm_oracle_cpu.py) and the GPU tests of every kernel path (tests/test_gpu_gemm_desc.py).

The contract, per batch index bz:
    C[bz] = alpha * op(A)[g(bz)] . op(B)[bz] + beta * C[bz] + bias[n]       g(bz) = bz % a_batch_mod (a_batch_mod > 0) else bz
    op(A)(m, k) = transA ? A[g * strideA + k * lda + m] : A[g * strideA + m * lda + k]
    op(B)(k, n) = transB ? B[bz * strideB + n * ldb + k] : B[bz * strideB + k * ldb + n]
    C(m, n)     = C[bz * strideC + m * ldc + n]
    two-level K (kin > 0, !transA, transB): k = q * kin + l, op(A)(m, k) = A[g * strideA + q * kosA + m * lda + l] (B likewise, kosB)
    explicit split-K s of splitk: raw sums over k in [s * kchunk, (s + 1) * kchunk) in partial[s][bz][m][n] (dense)
The oracle evaluates it with explicit index arithmetic on the flat operand buffers.  Every element a descriptor does not cover
(row padding beyond the row, gaps between batches and between kin slabs) is NaN, so a kernel that reads outside its operand
returns NaN; so is all of C when beta == 0, and the bf16 columns the wgmma path reads but never stores.

Routes (one kernel path each):
    f32       fp32 mode, gemm_run                    -> gemm_f32 (SIMT, k-block 16)
    mma       bf16 mode, tensor-core GEMM off        -> gemm_bf16_kernel (mma.sync, k-block 32)
    wgmma     bf16 mode, tensor-core GEMM on         -> gemm_tc_try (TMA + wgmma, k-block 64), mma.sync when it declines
    auto_f32  fp32 mode, gemm_run_auto               -> gemm_f32 with its own split-K factor
    auto_bf16 bf16 mode, gemm_run_auto               -> wgmma un-split, else mma.sync with its own split-K factor
bf16 routes multiply the operands rounded to bf16 (round to nearest even); the oracle does the same and accumulates in fp64.
"""
import math
from dataclasses import dataclass, replace
from types import SimpleNamespace

import numpy as np
import torch

NUM_SMS = 132
TC_TILE, TC_KBLOCK = 128, 64
SCRATCH_BYTES = 3 << 29                 # _lib.ensure_scratch()'s default
MAX_CACHE = 32                          # pack-cache entries of gemm_tc.cu
KBLOCK = {'f32': 16, 'mma': 32, 'wgmma': 64}
BF16_ROUTES = ('mma', 'wgmma', 'auto_bf16')


def cdiv(a, b):
    return -(-a // b)


@dataclass(frozen=True)
class Case:
    name: str
    M: int
    N: int
    K: int
    ta: int = 0
    tb: int = 0
    batch: int = 1
    lda: int = 0
    ldb: int = 0
    ldc: int = 0
    strideA: int = 0
    strideB: int = 0
    strideC: int = 0
    a_batch_mod: int = 0
    alpha: float = 1.0
    beta: float = 0.0
    bias: bool = False
    kin: int = 0
    kosA: int = 0
    kosB: int = 0
    splitk: int = 1
    keep_partials: int = 0
    a16: int = 0            # A also given as bf16 (A16, row stride lda16): [M, lda16] rows, or [K, lda16] rows when ta
    lda16: int = 0
    b16: int = 0            # B also given as bf16 (B16): [K, ldb16] rows
    ldb16: int = 0
    routes: tuple = ('f32', 'mma', 'wgmma')
    seed: int = 0

    @property
    def a_groups(self):
        return self.a_batch_mod if self.a_batch_mod > 0 else self.batch

    @property
    def kouter(self):
        return self.K // self.kin if self.kin else 1


def make(name, M, N, K, ta=0, tb=0, batch=1, pad=0, gap=0, kin=0, **kw):
    """Case with padded rows (`pad` elements past each row) and `gap` elements between batches (and between kin slabs)."""
    groups = kw.get('a_batch_mod') or batch
    if kin:
        lda, ldb = kin + pad, kin + pad
        sa, sb = M * lda + gap, N * ldb + gap
        kw.setdefault('kosA', groups * sa + gap)
        kw.setdefault('kosB', batch * sb + gap)
    else:
        lda = (M if ta else K) + pad
        ldb = (K if tb else N) + pad
        sa = (K if ta else M) * lda + gap
        sb = (N if tb else K) * ldb + gap
    ldc = N + pad
    kw.setdefault('lda', lda)
    kw.setdefault('ldb', ldb)
    kw.setdefault('ldc', ldc)
    kw.setdefault('strideA', sa if groups > 1 else 0)
    kw.setdefault('strideB', sb if batch > 1 else 0)
    kw.setdefault('strideC', M * kw['ldc'] + gap if batch > 1 else 0)
    return Case(name, M, N, K, ta=ta, tb=tb, batch=batch, kin=kin, **kw)


# ---------------------------------------------------------------------------------------------------------------------------
# the case table.  Shapes sit off the tile multiples (64 / 128 for M and N, 16 / 32 / 64 for K, K % 8 != 0 where the packer pads);
# the wgmma cases clear that path's limits (M, N >= 64, K >= 32, M N K batch >= 2^24).
# ---------------------------------------------------------------------------------------------------------------------------
CASES = [
    # 1. batched, strided, padded: all four (transA, transB); the odd pads / gaps take the scalar loads, the others the vector loads
    make('batched_nn', 200, 136, 157, 0, 0, batch=4, pad=3, gap=5, alpha=0.5, beta=0.25, bias=True, seed=1),
    make('batched_nt', 130, 200, 172, 0, 1, batch=5, pad=4, gap=8, seed=2),
    make('batched_tn', 190, 132, 141, 1, 0, batch=5, pad=4, gap=12, alpha=-1.5, bias=True, seed=3),
    make('batched_tt', 152, 170, 222, 1, 1, batch=3, pad=1, gap=7, beta=1.0, seed=4),
    # the decoder's d memory = align^T . d ctx per utterance: B interleaved across the batch (ldb = B * M, strideB = M)
    Case('decoder_dmemory', 180, 288, 120, ta=1, tb=0, batch=8, lda=180, ldb=8 * 288, ldc=288, strideA=120 * 180, strideB=288,
         strideC=180 * 288, seed=5),
    # 2. a_batch_mod: the grouped convolution's forward (A = weights [G][Cout][Cin k]) and input gradient (A^T), NB = 2 rows, G = 3
    make('conv_fwd_groups', 96, 150, 200, 0, 0, batch=6, a_batch_mod=3, seed=6),
    make('conv_dx_groups', 200, 150, 96, 1, 0, batch=6, a_batch_mod=3, pad=2, gap=3, beta=0.5, seed=7),
    # 3. A16 K-major (lda16 > K): no A pack on wgmma
    make('a16_kmajor', 200, 150, 600, 0, 1, pad=5, a16=1, lda16=616, bias=True, seed=8),
    # 4. A16 with transA: [K, lda16] bf16 rows, lda16 % 64 == 0, M % 64 != 0, columns [M, lda16) NaN
    make('a16_mn', 150, 170, 700, 1, 0, a16=1, lda16=192, beta=0.5, seed=9),
    # 5. B16 (ldb16 = ceil64(N) exactly, columns [N, ldb16) NaN); A16 and B16 together: the GEMM alone
    make('b16', 160, 170, 644, 0, 0, pad=3, b16=1, ldb16=192, seed=10),
    make('a16_b16', 150, 170, 700, 1, 0, a16=1, lda16=192, b16=1, ldb16=192, bias=True, seed=11),
    make('a16k_b16', 200, 100, 900, 0, 0, a16=1, lda16=904, b16=1, ldb16=128, alpha=2.0, seed=12),
    # 6. two-level K, kin no multiple of 64 (k-blocks straddle slabs), gaps between slabs: f32 / mma.sync must refuse it
    make('kin_groups', 136, 200, 600, 0, 1, batch=3, kin=100, pad=4, gap=24, beta=1.0, seed=13),
    make('kin_splitk', 250, 330, 7200, 0, 1, kin=900, pad=4, gap=40, alpha=0.5, bias=True, seed=14),
    # 7. explicit split-K, batch > 1: raw partials kept for the consumer, and reduced in place
    make('split_keep', 96, 130, 700, 0, 1, batch=3, pad=2, gap=3, splitk=4, keep_partials=1, routes=('f32', 'mma'), seed=15),
    make('split_reduce', 70, 90, 1000, 1, 0, batch=2, pad=1, gap=9, splitk=5, alpha=0.75, beta=-0.5, bias=True,
         routes=('f32', 'mma'), seed=16),
    # 8. wgmma split-K: 4 output tiles, K = 5000
    make('tc_splitk', 200, 136, 5000, 1, 0, alpha=0.5, beta=0.25, bias=True, routes=('wgmma',), seed=17),
    # 10. gemm_run_auto: a product the wgmma path declines (M < 64, split by the auto factor in both modes), and one it takes in bf16
    make('auto_small', 48, 100, 3000, 0, 0, pad=1, bias=True, beta=0.5, routes=('auto_f32', 'auto_bf16'), seed=18),
    make('auto_tc', 200, 136, 5000, 0, 1, alpha=0.5, routes=('auto_f32', 'auto_bf16'), seed=19),
]
BY_NAME = {c.name: c for c in CASES}


# ---------------------------------------------------------------------------------------------------------------------------
# operands
# ---------------------------------------------------------------------------------------------------------------------------
def a_index(c):
    """[a_groups, M, K] flat indices of op(A) in A."""
    g = np.arange(c.a_groups, dtype=np.int64)[:, None, None] * c.strideA
    m = np.arange(c.M, dtype=np.int64)[None, :, None]
    k = np.arange(c.K, dtype=np.int64)[None, None, :]
    if c.kin:
        return g + (k // c.kin) * c.kosA + m * c.lda + k % c.kin
    return g + (k * c.lda + m if c.ta else m * c.lda + k)


def b_index(c):
    """[batch, K, N] flat indices of op(B) in B."""
    z = np.arange(c.batch, dtype=np.int64)[:, None, None] * c.strideB
    k = np.arange(c.K, dtype=np.int64)[None, :, None]
    n = np.arange(c.N, dtype=np.int64)[None, None, :]
    if c.kin:
        return z + (k // c.kin) * c.kosB + n * c.ldb + k % c.kin
    return z + (n * c.ldb + k if c.tb else k * c.ldb + n)


def c_index(c):
    """[batch, M, N] flat indices of the output in C."""
    z = np.arange(c.batch, dtype=np.int64)[:, None, None] * c.strideC
    return z + np.arange(c.M, dtype=np.int64)[None, :, None] * c.ldc + np.arange(c.N, dtype=np.int64)[None, None, :]


def a_group_of(c):
    return [bz % c.a_batch_mod if c.a_batch_mod > 0 else bz for bz in range(c.batch)]


def _fill(index, gen, bf16_exact):
    idx = torch.from_numpy(index.reshape(-1))
    buf = torch.full((int(idx.max()) + 1,), float('nan'))
    buf[idx] = torch.randn(idx.numel(), generator=gen)
    return buf.bfloat16().float() if bf16_exact else buf


def operands(c, seed=None):
    """Seeded flat CPU buffers for case c: A, B, C0 (fp32), bias, A16 / B16 (bf16) or None.  A / B hold bf16-exact values when
    they are also given as bf16, so that every route multiplies the same numbers."""
    gen = torch.Generator().manual_seed(c.seed if seed is None else seed)
    A = _fill(a_index(c), gen, c.a16)
    B = _fill(b_index(c), gen, c.b16)
    ci = torch.from_numpy(c_index(c).reshape(-1))
    C0 = torch.full((int(ci.max()) + 1,), float('nan'))
    if c.beta != 0:
        C0[ci] = torch.randn(ci.numel(), generator=gen)
    bias = torch.randn(c.N, generator=gen) if c.bias else None
    A16 = B16 = None
    if c.a16:
        assert c.batch == 1
        opa = A[torch.from_numpy(a_index(c))][0]                      # [M, K]
        if c.ta:
            A16 = torch.full((c.K, c.lda16), float('nan'))
            A16[:, :c.M] = opa.t()
        else:
            A16 = torch.full((c.M, c.lda16), float('nan'))
            A16[:, :c.K] = opa
        A16 = A16.bfloat16().reshape(-1)
    if c.b16:
        assert c.batch == 1 and not c.tb
        B16 = torch.full((c.K, c.ldb16), float('nan'))
        B16[:, :c.N] = B[torch.from_numpy(b_index(c))][0]
        B16 = B16.bfloat16().reshape(-1)
    return SimpleNamespace(A=A, B=B, C0=C0, bias=bias, A16=A16, B16=B16)


# ---------------------------------------------------------------------------------------------------------------------------
# the oracle
# ---------------------------------------------------------------------------------------------------------------------------
MUTATIONS = ('drop_kblock', 'a_group', 'kin_offset', 'no_bias', 'beta_wrong_c')


def applicable(c, mutation):
    return {'drop_kblock': True, 'a_group': c.a_batch_mod > 0 and c.a_groups > 1, 'kin_offset': c.kin > 0 and c.kouter > 1,
            'no_bias': c.bias, 'beta_wrong_c': c.beta != 0}[mutation]


def _logical(c, ops, bf16):
    a = ops.A[torch.from_numpy(a_index(c))]
    b = ops.B[torch.from_numpy(b_index(c))]
    if bf16:
        a, b = a.bfloat16(), b.bfloat16()
    return a.double(), b.double()


def reference(c, ops, bf16, mutation=None, kblock=64):
    """[batch, M, N] fp64 result of the descriptor on ops.  `mutation` makes one deliberate mistake (see MUTATIONS):
    drop_kblock   the k-block of width `kblock` that holds k = K / 2 is left out
    a_group       the last batch multiplies the next group's A instead of group bz % a_batch_mod
    kin_offset    the last kin slab of A is read at the previous slab's offset
    no_bias       bias left out
    beta_wrong_c  beta scales the C of the next batch (one row down when batch == 1)"""
    a, b = _logical(c, ops, bf16)
    grp = a_group_of(c)
    if mutation == 'drop_kblock':
        k0 = (c.K // 2) // kblock * kblock
        a = a.clone()
        a[:, :, k0:k0 + kblock] = 0
    elif mutation == 'a_group':
        grp[-1] = (grp[-1] + 1) % c.a_groups
    elif mutation == 'kin_offset':
        a = a.clone()
        q = c.kouter - 1
        a[:, :, q * c.kin:] = a[:, :, (q - 1) * c.kin:q * c.kin]
    out = c.alpha * torch.matmul(a[grp], b)
    if c.bias and mutation != 'no_bias':
        out = out + ops.bias.double()
    if c.beta != 0:
        c0 = ops.C0[torch.from_numpy(c_index(c))].double()
        if mutation == 'beta_wrong_c':
            c0 = torch.roll(c0, 1, dims=0) if c.batch > 1 else torch.roll(c0, 1, dims=1)
        out = out + c.beta * c0
    return out


def kchunk(c, route):
    """k range of one explicit split on the f32 / mma.sync kernels: ceil(K / splitk) rounded up to the kernel's k-block."""
    bk = KBLOCK[route]
    return cdiv(cdiv(c.K, c.splitk), bk) * bk


def partials(c, ops, bf16, chunk):
    """[splitk, batch, M, N] fp64 raw partial sums (no alpha, bias or beta) of the explicit split-K layout."""
    a, b = _logical(c, ops, bf16)
    a = a[a_group_of(c)]
    out = torch.zeros(c.splitk, c.batch, c.M, c.N, dtype=torch.float64)
    for s in range(c.splitk):
        k0, k1 = s * chunk, min(c.K, (s + 1) * chunk)
        if k1 > k0:
            out[s] = torch.matmul(a[:, :, k0:k1], b[:, k0:k1])
    return out


def tolerance(c, route):
    """(rtol, atol) of the existing GEMM tests: fp32 1e-4 / 1e-4 sqrt(K); bf16 routes against the bf16-rounded oracle 1e-4 / 2e-4 sqrt(K)."""
    return 1e-4, (2e-4 if route in BF16_ROUTES else 1e-4) * math.sqrt(c.K)


def within(actual, expected, rtol, atol):
    actual, expected = actual.double().cpu(), expected.double().cpu()
    if not bool(torch.isfinite(actual).all()) or not bool(torch.isfinite(expected).all()):
        return False
    return bool(((actual - expected).abs() <= atol + rtol * expected.abs()).all())


# ---------------------------------------------------------------------------------------------------------------------------
# which kernels a route launches (host decisions of gemm_tc.cu / gemm.cu, mirrored)
# ---------------------------------------------------------------------------------------------------------------------------
def tc_plan(c, scratch_bytes, used0=0):
    """What gemm_tc_try does with c and a scratch of `scratch_bytes` whose first `used0` bytes hold cached packs (nothing cached for
    this product): None when it declines, else SimpleNamespace(pack_a, pack_b, a_bytes, b_bytes, ksplit)."""
    if c.splitk != 1 or c.keep_partials:
        return None
    if c.kin and (c.ta or not c.tb or c.K % c.kin or c.a16):
        return None
    if c.M < 64 or c.N < 64 or c.K < 32 or c.M * c.N * c.K * c.batch < (1 << 24):
        return None
    Kp = cdiv(c.K, 8) * 8
    a16ok = c.a16 and c.batch == 1 and c.lda16 % 8 == 0
    a_mn_ready = a16ok and c.ta and not c.kin and c.lda16 % 64 == 0
    a_ready = (a16ok and not c.ta) or a_mn_ready
    a_mn = c.ta and not a_ready and c.batch == 1 and not c.kin
    b_mn = not c.tb and c.batch == 1 and not c.kin
    b_ready = b_mn and c.b16 and c.ldb16 % 64 == 0
    Mp64, Np64 = cdiv(c.M, 64) * 64, cdiv(c.N, 64) * 64
    r1k = lambda x: cdiv(x, 1024) * 1024                           # noqa: E731
    a_bytes = 0 if a_ready else r1k(c.K * Mp64 * 2) if a_mn else r1k(c.a_groups * c.M * Kp * 2)
    b_bytes = 0 if b_ready else r1k(c.K * Np64 * 2) if b_mn else r1k(c.batch * c.N * Kp * 2)
    if used0 + a_bytes + b_bytes > scratch_bytes:
        return None
    ksplit = 1
    tiles, nk = cdiv(c.N, TC_TILE) * cdiv(c.M, TC_TILE), cdiv(c.K, TC_KBLOCK)
    if c.batch == 1 and tiles <= NUM_SMS and nk >= 64:
        want = min(2 * NUM_SMS // tiles, nk // 16, 32)
        if want >= 2:
            kper = cdiv(nk, want)
            splits = cdiv(nk, kper)
            if splits >= 2 and used0 + a_bytes + b_bytes + splits * c.M * c.N * 4 + 1024 <= scratch_bytes:
                ksplit = splits
    return SimpleNamespace(pack_a=not a_ready, pack_b=not b_ready, a_bytes=a_bytes, b_bytes=b_bytes, ksplit=ksplit)


def auto_split(c, bf16, partial_elems):
    """Split-K factor gemm_run_auto picks for the f32 / mma.sync kernel with a partial buffer of `partial_elems` floats (0 = none)."""
    big = bf16 or (c.M > 64 and c.N > 64)
    tiles = (cdiv(c.M, 128) * cdiv(c.N, 128) if big else cdiv(c.M, 64) * cdiv(c.N, 64)) * c.batch
    s = 1
    if tiles < NUM_SMS and partial_elems > 0:
        s = max(1, min(cdiv(2 * NUM_SMS, tiles), cdiv(c.K, 128), 160))
        while s > 1 and s * c.batch * c.M * c.N > partial_elems:
            s -= 1
    return s


def expected_path(c, route, scratch_bytes=SCRATCH_BYTES, partial_elems=0):
    """(path name, library launches, wgmma GEMM launches) of c on `route`; ('rejected', 0, 0) when the library refuses it."""
    if route in ('wgmma', 'auto_bf16'):
        p = tc_plan(replace(c, splitk=1, keep_partials=0) if route == 'auto_bf16' else c, scratch_bytes)
        if p is not None:
            packs = int(p.pack_a) + int(p.pack_b)
            name = f'wgmma, {packs} pack(s)' + (f', split-K {p.ksplit}' if p.ksplit > 1 else '')
            return name, packs + 1 + (p.ksplit > 1), 1
    if c.kin:
        return 'rejected', 0, 0
    kernel = 'f32' if route in ('f32', 'auto_f32') else 'mma.sync'
    if route in ('auto_f32', 'auto_bf16'):
        s = auto_split(c, route == 'auto_bf16', partial_elems)
        return f'{kernel}' + (f', auto split-K {s}' if s > 1 else ''), 1 + (s > 1), 0
    split = c.splitk > 1
    return (f'{kernel}' + (f', split-K {c.splitk}' if split else '') + (' (partials kept)' if c.keep_partials else ''),
            1 + (split and not c.keep_partials), 0)


def route_kblock(c, route):
    """k-block of the kernel a route runs c on."""
    if route == 'auto_f32':
        return KBLOCK['f32']
    if route in ('wgmma', 'auto_bf16') and expected_path(c, route)[2] == 1:
        return KBLOCK['wgmma']
    return KBLOCK['f32'] if route == 'f32' else KBLOCK['mma']
