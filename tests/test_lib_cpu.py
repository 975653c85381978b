"""CPU-side checks of the C-ABI library: it loads, exports every symbol include/b200tts.h declares, sizes
workspaces, and FAILS LOUDLY when asked to compute without a GPU (no CPU fallback)."""
import ctypes
import os
import re

import pytest
import torch

import __graft_entry__ as entry
from multilingual_text_to_speech_b200 import _lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope='module')
def lib():
    entry.build()
    return _lib.load()


# C scalar types of the header -> the ctypes type SIGNATURES must use (ctypes aliases size_t / uint64_t and long long / int64_t on LP64)
_C_SCALARS = {'int': ctypes.c_int, 'float': ctypes.c_float, 'double': ctypes.c_double, 'size_t': ctypes.c_size_t,
              'long long': ctypes.c_longlong, 'int64_t': ctypes.c_int64, 'uint64_t': ctypes.c_uint64,
              'unsigned long long': ctypes.c_ulonglong}


def _is_pointer(t):
    return t in (ctypes.c_void_p, ctypes.c_char_p) or issubclass(t, ctypes._Pointer)


def _c_type(decl, named):
    """ctypes type of one C declaration ('const float* x', 'size_t'), or 'ptr' for any pointer."""
    if '*' in decl:
        return 'ptr'
    words = decl.replace('const ', '').split()
    return _C_SCALARS[' '.join(words[:-1] if named else words)]


def test_header_symbols_exported(lib):
    header = open(os.path.join(ROOT, 'include', 'b200tts.h')).read()
    declared = set(re.findall(r'\b(b200tts_[a-z0-9_]+)\s*\(', header))
    assert declared, 'no declarations parsed'
    for name in sorted(declared):
        assert hasattr(lib, name), f'{name} declared in include/b200tts.h but not exported'
    assert declared == set(_lib.SIGNATURES), declared ^ set(_lib.SIGNATURES)

    # every prototype's return type, argument count and argument types agree with SIGNATURES (any pointer stands for any pointer)
    code = re.sub(r'//[^\n]*', '', re.sub(r'/\*.*?\*/', '', header, flags=re.S))
    protos = re.findall(r'([A-Za-z_][\w \t*]*?)\s*\b(b200tts_\w+)\s*\(([^)]*)\)\s*;', code)
    assert {name for _, name, _ in protos} == declared
    for ret, name, args in protos:
        restype, argtypes = _lib.SIGNATURES[name]
        want = _c_type(ret, named=False)
        assert (want == 'ptr' and _is_pointer(restype)) or restype is want, f'{name}: returns {ret.strip()}, SIGNATURES has {restype}'
        params = [] if args.strip() in ('', 'void') else [p.strip() for p in args.split(',')]
        assert len(params) == len(argtypes), f'{name}: {len(params)} arguments in the header, {len(argtypes)} in SIGNATURES'
        for i, (p, t) in enumerate(zip(params, argtypes)):
            want = _c_type(p, named=True)
            assert (want == 'ptr' and _is_pointer(t)) or t is want, f'{name}: argument {i} is `{p}`, SIGNATURES has {t}'


def test_workspace_queries_are_host_only(lib):
    shape = _lib.DecoderShape(64, 180, 900, 288, 1024, 256, 128, 32, 31, 80, 0, 1, 0.1, 0.0, 0.5)
    fwd = lib.b200tts_decoder_workspace_bytes(ctypes.byref(shape))
    bwd = lib.b200tts_decoder_bwd_workspace_bytes(ctypes.byref(shape))
    assert 2e9 < fwd < 6e9 and 2e9 < bwd < 6e9, (fwd, bwd)
    bad = _lib.DecoderShape(64, 180, 900, 288, 1024, 256, 129, 32, 31, 80, 0, 1, 0.1, 0.0, 0.5)
    assert lib.b200tts_decoder_workspace_bytes(ctypes.byref(bad)) == 0
    assert b'attention dimension' in lib.b200tts_last_error()


@pytest.mark.skipif(torch.cuda.is_available(), reason='checks the no-GPU failure mode')
def test_compute_without_gpu_fails_loudly(lib):
    a = torch.zeros(4, 4)
    st = lib.b200tts_gemm_f32(0, 0, 4, 4, 4, 1.0, _lib.ptr(a), 4, _lib.ptr(a), 4, 0.0, _lib.ptr(a), 4, None, 1, 0, 0, 0, 1,
                              None, None)
    assert st != 0
    assert b'no CPU fallback' in lib.b200tts_last_error() or b'CUDA' in lib.b200tts_last_error()
    from multilingual_text_to_speech_b200 import functional as F
    with pytest.raises(_lib.B200TTSError):
        F.gemm(a, a)


def test_fused_adam_needs_gpu():
    """The optimizer step has no CPU fallback either."""
    import pytest
    import torch
    from multilingual_text_to_speech_b200 import _lib
    from multilingual_text_to_speech_b200.optim import FlatParams, FusedAdam
    from multilingual_text_to_speech_b200.distributed import GradBucket
    model = torch.nn.Linear(4, 3)
    flat, bucket = FlatParams(model), GradBucket(model, 1)
    assert model.weight.data_ptr() == flat.flat.data_ptr() and model.weight.grad.data_ptr() == bucket.flat.data_ptr()
    opt = FusedAdam(flat, bucket, lr=1e-3, lr_decay_every=10, lr_decay=0.5)
    assert opt.current_lr() == 1e-3
    with pytest.raises(_lib.B200TTSError):
        opt.step()


def test_decoder_path_covers_baseline_configs(lib):
    """BASELINE configs[1..4] run on the persistent wgmma kernels in every pass (host-side path query, no GPU needed): memory
    dims 288 (generated_training / generated_switching) and 292 (shared_switching), per-GPU batches up to 64, texts up to 300.
    The monolingual default (memory dim 512, configs[0]) fits too (accumulator staging aliased onto the TMA slot, wider n-blocks)."""
    def path(B, L, T, M, kind=1, training=1):
        s = _lib.DecoderShape(B, L, T, M, 1024, 256, 128, 32, 31, 80, kind, training, 0.1, 0.1, 0.5)
        return lib.b200tts_decoder_path(ctypes.byref(s))
    for M in (288, 292):
        for B in (16, 50, 60, 64):
            for L, T in ((180, 900), (300, 1200)):
                for kind in (0, 1):
                    assert path(B, L, T, M, kind) == 0b111111, (B, L, T, M, kind, bin(path(B, L, T, M, kind)))
    assert path(64, 180, 900, 288, training=0) & 0b11 == 0b11          # inference / evaluation: forward loops on wgmma
    for B, L in ((16, 180), (52, 180), (64, 300)):
        assert path(B, L, 900, 512) == 0b111111, (B, L, bin(path(B, L, 900, 512)))


def _decoder_path(lib, B, L, M, D, training):
    s = _lib.DecoderShape(B, L, 900, M, D, 256, 128, 32, 31, 80, 1, training, 0.1, 0.1, 0.5)
    return lib.b200tts_decoder_path(ctypes.byref(s))


def test_decoder_path_variant_bits_pair_with_loop_bits(lib):
    """Every persistent loop is a TMA + wgmma kernel: each variant bit (1, 3, 5) is set exactly when its loop bit (0, 2, 4) is."""
    for D in (512, 960, 1024, 1040, 1152, 1280, 2048):
        for M in (128, 288, 512):
            for B in (1, 8, 33, 64):
                for training in (0, 1):
                    bits = _decoder_path(lib, B, 180, M, D, training)
                    for loop in (0, 2, 4):
                        assert (bits >> loop) & 1 == (bits >> (loop + 1)) & 1, (D, M, B, training, bin(bits))


def test_decoder_path_off_the_wgmma_loops_is_the_per_step_chains(lib):
    """Shapes no wgmma loop accepts run every such pass on the per-step chains (no mma.sync persistent loops)."""
    assert _decoder_path(lib, 8, 180, 288, 1280, 1) == 0          # D = 1280 training: the generator reverse loop included
    assert _decoder_path(lib, 8, 180, 288, 1040, 0) & 0b11 == 0   # no-grad forward with D % 64 != 0


def test_grad_targets_accumulate_in_place_only_into_bound_leaf_gradients():
    """functional._grad_targets: a leaf parameter whose .grad is a dense fp32 tensor of its own shape (the GradBucket views) is the
    accumulation target itself and autograd gets None; anything else gets a fresh zero tensor that autograd accumulates as usual."""
    from multilingual_text_to_speech_b200 import functional as F
    bound = torch.nn.Parameter(torch.ones(3, 4))
    bound.grad = torch.full((3, 4), 2.0)
    fresh = torch.nn.Parameter(torch.ones(5))
    non_leaf = bound * 2.0
    strided = torch.nn.Parameter(torch.ones(4, 6))
    strided.grad = torch.zeros(6, 4).t()                      # not contiguous: must not be written through a flat pointer
    targets, returned = F._grad_targets((bound, fresh, non_leaf, None, strided))
    assert targets[0] is bound.grad and returned[0] is None
    assert returned[1] is targets[1] and float(targets[1].abs().sum()) == 0.0 and targets[1].shape == fresh.shape
    assert returned[2] is targets[2] and targets[2].shape == non_leaf.shape
    assert targets[3] is None and returned[3] is None
    assert returned[4] is targets[4] and targets[4].is_contiguous()
