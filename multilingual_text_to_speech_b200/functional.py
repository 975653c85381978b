"""Host-side op layer: torch.autograd.Functions and thin wrappers that call the C ABI (libb200tts.so).

PyTorch is plumbing here (device memory, streams, autograd glue between the fused ops); all arithmetic
of the hot path happens inside the library.
"""
import ctypes
import numpy as np
import torch

from . import _lib
from ._lib import (DecoderShape, DecoderParams, DecoderInputs, DecoderOutputs, DecoderOutputGrads,
                   DECODER_PARAM_FIELDS, check, ptr)


# Optional in-band timing of the dominant ops (bench.py): when PROFILE['enabled'] is set, CUDA events are recorded on
# the launching stream around the library call and appended as (start, end) pairs under the op's name.
PROFILE = {}


class _Timed:
    def __init__(self, name):
        self.name = name

    def __enter__(self):
        self.on = bool(PROFILE.get('enabled'))
        if self.on:
            self.start = torch.cuda.Event(enable_timing=True)
            self.end = torch.cuda.Event(enable_timing=True)
            self.start.record()
        return self

    def __exit__(self, *exc):
        if self.on:
            self.end.record()
            PROFILE.setdefault(self.name, []).append((self.start, self.end))
        return False


def _stream():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def _require_cuda(*tensors):
    for t in tensors:
        if t is not None and not t.is_cuda:
            raise _lib.B200TTSError('b200tts ops need CUDA tensors (there is no CPU fallback)')


def _f32c(t):
    if t.dtype != torch.float32:
        t = t.float()
    return t.contiguous()


# ------------------------------------------------------------------------------------------------
# generic GEMM
# ------------------------------------------------------------------------------------------------
def gemm(a, b, trans_a=False, trans_b=False, bias=None, out=None, beta=0.0, alpha=1.0, splitk=1):
    """out = alpha * op(a) @ op(b) + beta * out + bias  on 2-D fp32 CUDA tensors (row-major, any row stride)."""
    _require_cuda(a, b)
    assert a.dim() == 2 and b.dim() == 2 and a.stride(1) == 1 and b.stride(1) == 1
    M, K = (a.shape[1], a.shape[0]) if trans_a else a.shape
    K2, N = (b.shape[1], b.shape[0]) if trans_b else b.shape
    assert K == K2, (a.shape, b.shape, trans_a, trans_b)
    if out is None:
        out = torch.empty(M, N, device=a.device, dtype=torch.float32)
    ws = torch.empty(splitk * M * N, device=a.device, dtype=torch.float32) if splitk > 1 else None
    lib = _lib.load()
    check(lib.b200tts_gemm_f32(int(trans_a), int(trans_b), M, N, K, float(alpha), ptr(a), a.stride(0), ptr(b), b.stride(0),
                               float(beta), ptr(out), out.stride(0), ptr(bias), 1, 0, 0, 0, splitk, ptr(ws), _stream()),
          'b200tts_gemm_f32')
    return out


# ------------------------------------------------------------------------------------------------
# dropout keep-masks
# ------------------------------------------------------------------------------------------------
def fill_keep_mask(shape, rate, seed, stream_id, device):
    """uint8 keep mask (1 = keep) with P(keep) = 1 - rate from the library's counter-based generator."""
    mask = torch.empty(shape, dtype=torch.uint8, device=device)
    check(_lib.load().b200tts_fill_keep_mask(ptr(mask), mask.numel(), float(rate), int(seed) & (2 ** 64 - 1), int(stream_id),
                                            _stream()), 'b200tts_fill_keep_mask')
    return mask


# ------------------------------------------------------------------------------------------------
# single attention step (module-level API of LocationSensitiveAttention)
# ------------------------------------------------------------------------------------------------
def attention_step(query, memory, memory_transform, text_lengths, w_query, w_location, w_loc_features, bias, w_energy,
                   cum_weights):
    """One LocationSensitiveAttention.forward (reference modules/attention.py:39-45, 67-86).

    Updates `cum_weights` in place; returns (context [B, M], weights [B, L]).
    """
    _require_cuda(query, memory, memory_transform, cum_weights)
    B, L, M = memory.shape
    D = query.shape[1]
    A = w_query.shape[0]
    C, _, K = w_loc_features.shape
    lib = _lib.load()
    ws = torch.empty(lib.b200tts_attention_step_workspace_elems(B, L, A), device=query.device, dtype=torch.float32)
    ctx = torch.empty(B, M, device=query.device, dtype=torch.float32)
    weights = torch.empty(B, L, device=query.device, dtype=torch.float32)
    args = [_f32c(query), _f32c(memory), _f32c(memory_transform), text_lengths.to(torch.int32).contiguous(),
            _f32c(w_query), _f32c(w_location), _f32c(w_loc_features), _f32c(bias), _f32c(w_energy)]
    assert cum_weights.is_contiguous() and cum_weights.dtype == torch.float32
    check(lib.b200tts_attention_step(B, L, M, D, A, C, K, *[ptr(t) for t in args], ptr(cum_weights), ptr(ctx),
                                     ptr(weights), ptr(ws), _stream()), 'b200tts_attention_step')
    return ctx, weights


class AttentionStepFunction(torch.autograd.Function):
    """One LocationSensitiveAttention step WITH autograd (reference modules/attention.py:39-45, 67-86): returns
    (context, weights, updated cumulative weights); the backward is the library's single-step attention backward."""

    @staticmethod
    def forward(ctx, query, memory, memT, cum_prev, text_lengths, w_query, w_location, w_loc_features, bias, w_energy):
        _require_cuda(query, memory, memT, cum_prev)
        query, memory, memT = _f32c(query), _f32c(memory), _f32c(memT)
        ws_args = [_f32c(t) for t in (w_query, w_location, w_loc_features, bias, w_energy)]
        lengths = text_lengths.to(torch.int32).contiguous()
        B, L, M = memory.shape
        D, A = query.shape[1], ws_args[0].shape[0]
        C, _, K = ws_args[2].shape
        lib = _lib.load()
        ws = torch.empty(lib.b200tts_attention_step_workspace_elems(B, L, A), device=query.device, dtype=torch.float32)
        context = torch.empty(B, M, device=query.device, dtype=torch.float32)
        weights = torch.empty(B, L, device=query.device, dtype=torch.float32)
        cum_next = _f32c(cum_prev).clone()
        check(lib.b200tts_attention_step(B, L, M, D, A, C, K, ptr(query), ptr(memory), ptr(memT), ptr(lengths), *[ptr(t) for t in ws_args],
                                         ptr(cum_next), ptr(context), ptr(weights), ptr(ws), _stream()), 'b200tts_attention_step')
        q = ws[:B * A].view(B, A).clone()              # the forward left q = query . Wq^T at the head of its workspace
        ctx.dims = (B, L, M, D, A, C, K)
        ctx.save_for_backward(query, memory, memT, _f32c(cum_prev), lengths, q, weights, *ws_args)
        return context, weights, cum_next

    @staticmethod
    def backward(ctx, d_context, d_weights, d_cum_next):
        query, memory, memT, cum_prev, lengths, q, weights, w_query, w_location, w_loc_features, bias, w_energy = ctx.saved_tensors
        B, L, M, D, A, C, K = ctx.dims
        dev = query.device
        z = lambda *shape: torch.zeros(*shape, device=dev, dtype=torch.float32)   # noqa: E731
        d_context = _f32c(d_context) if d_context is not None else z(B, M)
        d_weights = _f32c(d_weights) if d_weights is not None else None
        d_cum = _f32c(d_cum_next).clone() if d_cum_next is not None else z(B, L)
        d_q, d_memT, d_wloc, d_wc, d_v = z(B, A), z(B, L, A), torch.zeros_like(w_location), torch.zeros_like(w_loc_features), torch.zeros_like(w_energy)
        lib = _lib.load()
        ws = torch.empty(lib.b200tts_attention_step_backward_workspace_elems(B, M, A, C, K), device=dev, dtype=torch.float32)
        check(lib.b200tts_attention_step_backward(B, L, M, A, C, K, ptr(q), ptr(memory), ptr(memT), ptr(lengths), ptr(w_location),
                                                  ptr(w_loc_features), ptr(bias), ptr(w_energy), ptr(cum_prev), ptr(weights), ptr(d_context),
                                                  ptr(d_weights), ptr(d_cum), ptr(d_q), ptr(d_memT), ptr(d_wloc), ptr(d_wc), ptr(d_v), ptr(ws),
                                                  _stream()), 'b200tts_attention_step_backward')
        d_query = gemm(d_q, w_query, False, False)                       # [B, A] . [A, D]
        d_wq = gemm(d_q, query, True, False)                             # [A, B] . [B, D]
        d_bias = d_q.sum(0, keepdim=True).view_as(bias)
        d_memory = weights.unsqueeze(2) * d_context.unsqueeze(1)         # context = weights . memory
        return d_query, d_memory, d_memT, d_cum, None, d_wq, d_wloc, d_wc, d_bias, d_v


class ForwardAttentionStepFunction(torch.autograd.Function):
    """One ForwardAttention step WITH autograd (reference modules/attention.py:23-45, 89-124): returns (context, weights); the weights
    are also the next alpha.  Forward and backward are the library's single-step forward-attention ops."""

    @staticmethod
    def forward(ctx, query, memory, memT, alpha_prev, text_lengths, w_query, bias, w_energy):
        _require_cuda(query, memory, memT, alpha_prev)
        query, memory, memT, alpha_prev = _f32c(query), _f32c(memory), _f32c(memT), _f32c(alpha_prev)
        w_query, bias, w_energy = _f32c(w_query), _f32c(bias), _f32c(w_energy)
        lengths = text_lengths.to(torch.int32).contiguous()
        B, L, M = memory.shape
        D, A = query.shape[1], w_query.shape[0]
        lib = _lib.load()
        ws = torch.empty(lib.b200tts_forward_attention_step_workspace_elems(B, L, A), device=query.device, dtype=torch.float32)
        context = torch.empty(B, M, device=query.device, dtype=torch.float32)
        weights = torch.empty(B, L, device=query.device, dtype=torch.float32)
        alpha = alpha_prev.clone()
        check(lib.b200tts_forward_attention_step(B, L, M, D, A, ptr(query), ptr(memory), ptr(memT), ptr(lengths), ptr(w_query), ptr(bias),
                                                 ptr(w_energy), ptr(alpha), ptr(context), ptr(weights), ptr(ws), _stream()),
              'b200tts_forward_attention_step')
        q = ws[:B * A].view(B, A).clone()              # the forward left q = query . Wq^T at the head of its workspace
        ctx.dims = (B, L, M, D, A)
        ctx.save_for_backward(query, memory, memT, alpha_prev, lengths, q, weights, w_query, bias, w_energy)
        return context, weights

    @staticmethod
    def backward(ctx, d_context, d_weights):
        query, memory, memT, alpha_prev, lengths, q, weights, w_query, bias, w_energy = ctx.saved_tensors
        B, L, M, D, A = ctx.dims
        dev = query.device
        z = lambda *shape: torch.zeros(*shape, device=dev, dtype=torch.float32)   # noqa: E731
        d_context = _f32c(d_context) if d_context is not None else z(B, M)
        d_weights = _f32c(d_weights) if d_weights is not None else None
        d_alpha = z(B, L)           # in: no gradient beyond the weights themselves; out: gradient of alpha_prev
        d_q, d_memT, d_v = z(B, A), z(B, L, A), torch.zeros_like(w_energy)
        lib = _lib.load()
        ws = torch.empty(lib.b200tts_forward_attention_step_backward_workspace_elems(B, M, A), device=dev, dtype=torch.float32)
        check(lib.b200tts_forward_attention_step_backward(B, L, M, A, ptr(q), ptr(memory), ptr(memT), ptr(lengths), ptr(bias), ptr(w_energy),
                                                          ptr(alpha_prev), ptr(weights), ptr(d_context), ptr(d_weights), ptr(d_alpha),
                                                          ptr(d_q), ptr(d_memT), ptr(d_v), ptr(ws), _stream()),
              'b200tts_forward_attention_step_backward')
        d_query = gemm(d_q, w_query, False, False)                       # [B, A] . [A, D]
        d_wq = gemm(d_q, query, True, False)                             # [A, B] . [B, D]
        d_bias = d_q.sum(0, keepdim=True).view_as(bias)
        d_memory = weights.unsqueeze(2) * d_context.unsqueeze(1)         # context = weights . memory
        return d_query, d_memory, d_memT, d_alpha, None, d_wq, d_bias, d_v


# ------------------------------------------------------------------------------------------------
# fused decoder
# ------------------------------------------------------------------------------------------------
class DecoderConfig:
    """Non-tensor arguments of one decode: shapes, regulariser settings, dropout masks, teacher-forcing coins.  With r frames per
    step (outputs_per_step) a decode of T frames runs S = ceil(T / r) steps: masks and coins have one row per step."""

    MASK_NAMES = ('prenet0', 'prenet1', 'att_h', 'att_c', 'gen_h', 'gen_c', 'step_prenet0', 'step_prenet1')

    def __init__(self, cell_kind, training, rate_h, rate_c, prenet_rate, masks=None, teacher=None, att_extent=0, outputs_per_step=1):
        self.att_extent = int(att_extent)    # 1: forward attention over each utterance's own length (inference of padded batches)
        self.cell_kind = int(cell_kind)
        self.training = bool(training)
        self.rate_h, self.rate_c, self.prenet_rate = float(rate_h), float(rate_c), float(prenet_rate)
        self.masks = dict(masks or {})       # name -> uint8 CUDA tensor, time-major ([S, B, P] / [S, B, D])
        self.teacher = teacher               # None (all teacher forced) or host bool/uint8 array [S]
        self.outputs_per_step = int(outputs_per_step)

    def steps(self, frames):
        """Decoder steps of a decode of `frames` frames."""
        return -(-int(frames) // self.outputs_per_step)


def _attention_dims(byname):
    """(att_kind, C, K): forward attention is the parameter set without location weights (both None)."""
    if byname['attn_location'] is None and byname['attn_loc_features'] is None:
        return _lib.ATT_FORWARD, 0, 0
    return _lib.ATT_LOCATION, byname['attn_loc_features'].shape[0], byname['attn_loc_features'].shape[-1]


def _decoder_structs(cfg, shape_dims, params, memory, text_lengths, target):
    B, L, T, M, D, P, A, C, K, N = shape_dims
    S = cfg.steps(T)
    att_kind = _attention_dims(dict(zip(DECODER_PARAM_FIELDS, params)))[0]
    shape = DecoderShape(B, L, T, M, D, P, A, C, K, N, cfg.cell_kind, int(cfg.training), cfg.rate_h, cfg.rate_c,
                         cfg.prenet_rate, att_kind, cfg.att_extent, cfg.outputs_per_step)
    pstruct = DecoderParams(*[ptr(p) for p in params])
    teacher_np = None
    if cfg.teacher is not None:
        teacher_np = np.ascontiguousarray(np.asarray(cfg.teacher).astype(np.uint8))
        assert teacher_np.shape == (S,)
    expect = {'prenet0': (S, B, P), 'prenet1': (S, B, P), 'step_prenet0': (S, B, P), 'step_prenet1': (S, B, P),
              'att_h': (S, B, D), 'att_c': (S, B, D), 'gen_h': (S, B, D), 'gen_c': (S, B, D)}
    mp = {}
    for name in DecoderConfig.MASK_NAMES:
        m = cfg.masks.get(name)
        if m is not None:
            assert m.dtype == torch.uint8 and m.is_cuda and m.is_contiguous() and tuple(m.shape) == expect[name], \
                (name, m.dtype, tuple(m.shape), expect[name])
        mp[name] = ptr(m)
    inputs = DecoderInputs(ptr(memory), ptr(text_lengths), ptr(target),
                           ctypes.c_void_p(teacher_np.ctypes.data) if teacher_np is not None else None,
                           mp['prenet0'], mp['prenet1'], mp['att_h'], mp['att_c'], mp['gen_h'], mp['gen_c'],
                           mp['step_prenet0'], mp['step_prenet1'])
    return shape, pstruct, inputs, teacher_np


class DecoderFunction(torch.autograd.Function):
    """Decoder._decode (reference modules/tacotron2.py:148-209) as one fused op with a hand-written backward.  Returns spectrogram
    [B, T, N] and stop logits [B, T] per frame, and the alignment [B, S, L] per decoder step."""

    @staticmethod
    def forward(ctx, cfg, memory, target, text_lengths, *params):
        assert len(params) == len(DECODER_PARAM_FIELDS)
        _require_cuda(memory, target, text_lengths, *params)
        memory, target = _f32c(memory), _f32c(target)
        params = [None if p is None else _f32c(p) for p in params]
        text_lengths = text_lengths.to(torch.int32).contiguous()
        byname = dict(zip(DECODER_PARAM_FIELDS, params))
        B, L, M = memory.shape
        N, T = target.shape[1], target.shape[2]
        D = byname['att_w_hh'].shape[1]
        P = byname['prenet_w1'].shape[0]
        A = byname['attn_query'].shape[0]
        _, C, K = _attention_dims(byname)
        assert byname['att_w_ih'].shape == (4 * D, P + M) and byname['gen_w_ih'].shape == (4 * D, D + M)
        dims = (B, L, T, M, D, P, A, C, K, N)
        shape, pstruct, inputs, teacher_np = _decoder_structs(cfg, dims, params, memory, text_lengths, target)
        lib = _lib.load()
        nbytes = lib.b200tts_decoder_workspace_bytes(ctypes.byref(shape))
        if nbytes == 0:
            raise _lib.B200TTSError('decoder shape rejected: ' + lib.b200tts_last_error().decode())
        ws = torch.empty(nbytes, dtype=torch.uint8, device=memory.device)
        spec = torch.empty(B, T, N, device=memory.device, dtype=torch.float32)
        stop = torch.empty(B, T, device=memory.device, dtype=torch.float32)
        align = torch.empty(B, cfg.steps(T), L, device=memory.device, dtype=torch.float32)
        outs = DecoderOutputs(ptr(spec), ptr(stop), ptr(align))
        with _Timed('decoder_fwd'):
            check(lib.b200tts_decoder_forward(ctypes.byref(shape), ctypes.byref(pstruct), ctypes.byref(inputs),
                                              ctypes.byref(outs), ptr(ws), nbytes, _stream()), 'b200tts_decoder_forward')
        ctx.cfg, ctx.dims, ctx.ws = cfg, dims, ws
        if PROFILE.get('keep_ws'):
            PROFILE['last_ws'], PROFILE['last_shape'] = ws, shape
        ctx.save_for_backward(memory, target, text_lengths, align, *params)
        ctx.set_materialize_grads(False)
        return spec, stop, align

    @staticmethod
    def backward(ctx, d_spec, d_stop, d_align):
        memory, target, text_lengths, align, *params = ctx.saved_tensors
        cfg, dims = ctx.cfg, ctx.dims
        shape, pstruct, inputs, teacher_np = _decoder_structs(cfg, dims, params, memory, text_lengths, target)
        lib = _lib.load()
        nbytes = lib.b200tts_decoder_bwd_workspace_bytes(ctypes.byref(shape))
        bws = torch.empty(nbytes, dtype=torch.uint8, device=memory.device)
        if PROFILE.get('keep_ws'):
            PROFILE['last_bws'] = bws
        grads, returned = _grad_targets(params)
        gstruct = DecoderParams(*[ptr(g) for g in grads])
        d_memory = torch.empty_like(memory) if ctx.needs_input_grad[1] else None
        d_spec, d_stop, d_align = [None if t is None else _f32c(t) for t in (d_spec, d_stop, d_align)]
        douts = DecoderOutputGrads(ptr(d_spec), ptr(d_stop), ptr(d_align))
        fouts = DecoderOutputs(None, None, ptr(align))
        with _Timed('decoder_bwd'):
            check(lib.b200tts_decoder_backward(ctypes.byref(shape), ctypes.byref(pstruct), ctypes.byref(inputs),
                                               ctypes.byref(fouts), ctypes.byref(douts), ptr(ctx.ws), ptr(bws), nbytes,
                                               ctypes.byref(gstruct), ptr(d_memory), _stream()), 'b200tts_decoder_backward')
        return (None, d_memory, None, None, *returned)


class DecoderState:
    """Device buffers of the decoder state carried between the chunks of one free-running decode (b200tts_decoder_state)."""

    def __init__(self, B, D, M, L, N, device):
        z = lambda *shape: torch.zeros(*shape, device=device, dtype=torch.float32)   # noqa: E731
        self.att_h, self.att_c, self.gen_h, self.gen_c = z(B, D), z(B, D), z(B, D), z(B, D)
        self.context, self.cum_weights, self.frame = z(B, M), z(B, L), z(B, N)
        self.first = True

    def select(self, rows):
        """Keep only the utterances `rows` (a device index tensor), in that order: a finished utterance leaves the decode."""
        for name in ('att_h', 'att_c', 'gen_h', 'gen_c', 'context', 'cum_weights', 'frame'):
            setattr(self, name, getattr(self, name).index_select(0, rows).contiguous())

    def struct(self):
        return _lib.DecoderState(*[ptr(t) for t in (self.att_h, self.att_c, self.gen_h, self.gen_c, self.context, self.cum_weights, self.frame)])


def decoder_forward_chunk(cfg, memory, text_lengths, params, state, frames):
    """`frames` free-running frames (frames / r decoder steps; a multiple of r) continuing from `state` (updated in place); no autograd
    (inference).  -> spectrogram [B, frames, N], stop [B, frames], alignment [B, frames / r, L]."""
    _require_cuda(memory, text_lengths, *params)
    with torch.no_grad():
        memory = _f32c(memory)
        params = [None if p is None else _f32c(p) for p in params]
        text_lengths = text_lengths.to(torch.int32).contiguous()
        byname = dict(zip(DECODER_PARAM_FIELDS, params))
        B, L, M = memory.shape
        D, P, A = byname['att_w_hh'].shape[1], byname['prenet_w1'].shape[0], byname['attn_query'].shape[0]
        _, C, K = _attention_dims(byname)
        N = byname['frame_w'].shape[0] // cfg.outputs_per_step
        T = int(frames)
        target = torch.zeros(B, N, T, device=memory.device, dtype=torch.float32)
        shape, pstruct, inputs, teacher_np = _decoder_structs(cfg, (B, L, T, M, D, P, A, C, K, N), params, memory, text_lengths, target)
        lib = _lib.load()
        nbytes = lib.b200tts_decoder_workspace_bytes(ctypes.byref(shape))
        if nbytes == 0:
            raise _lib.B200TTSError('decoder shape rejected: ' + lib.b200tts_last_error().decode())
        ws = torch.empty(nbytes, dtype=torch.uint8, device=memory.device)
        spec = torch.empty(B, T, N, device=memory.device, dtype=torch.float32)
        stop = torch.empty(B, T, device=memory.device, dtype=torch.float32)
        align = torch.empty(B, cfg.steps(T), L, device=memory.device, dtype=torch.float32)
        outs = DecoderOutputs(ptr(spec), ptr(stop), ptr(align))
        st = state.struct()
        check(lib.b200tts_decoder_forward_chunk(ctypes.byref(shape), ctypes.byref(pstruct), ctypes.byref(inputs), ctypes.byref(outs),
                                                ctypes.byref(st), int(state.first), ptr(ws), nbytes, _stream()), 'b200tts_decoder_forward_chunk')
        state.first = False
    return spec, stop, align


# the persistent loop kernels of the bf16 mode hold the whole batch in one MMA tile (<= 64 utterances)
MAX_PERSIST_BATCH = 64


def decoder_forward(cfg, memory, target, text_lengths, params):
    """params: list of the 22 decoder parameter tensors in DECODER_PARAM_FIELDS order; forward attention (ForwardAttention) passes None
    for the two location weights (attn_location, attn_loc_features), which selects B200TTS_ATT_FORWARD.

    Utterances are independent inside the decoder (only the weights are shared), so a batch larger than the persistent kernels' tile
    (B > 64: BASELINE configs[3..4] run 65 / 80 per GPU) is decoded as ceil(B / 64) equal slices through the same fused op instead of
    dropping to the per-step kernel chains; parameter gradients of the slices add up in autograd."""
    B = memory.shape[0]
    if B <= MAX_PERSIST_BATCH or _lib.get_precision() != 'bf16':
        return DecoderFunction.apply(cfg, memory, target, text_lengths, *params)
    nslice = -(-B // MAX_PERSIST_BATCH)
    bounds = [round(k * B / nslice) for k in range(nslice + 1)]
    outs = []
    for lo, hi in zip(bounds[:-1], bounds[1:]):
        masks = {k: v[:, lo:hi].contiguous() for k, v in cfg.masks.items()}
        sub = DecoderConfig(cfg.cell_kind, cfg.training, cfg.rate_h, cfg.rate_c, cfg.prenet_rate, masks, cfg.teacher,
                            outputs_per_step=cfg.outputs_per_step)
        outs.append(DecoderFunction.apply(sub, memory[lo:hi], target[lo:hi], text_lengths[lo:hi], *params))
    return tuple(torch.cat([o[j] for o in outs], dim=0) for j in range(3))


# ------------------------------------------------------------------------------------------------
# encoder-side ops
# ------------------------------------------------------------------------------------------------
ACTIVATIONS = {'identity': 0, 'relu': 1, 'tanh': 2}


def _bytes(n, device):
    return torch.empty(max(int(n), 16), dtype=torch.uint8, device=device)


class ConvBlockFunction(torch.autograd.Function):
    """pad -> grouped conv -> batch norm -> activation -> dropout (-> highway) (reference modules/layers.py:50-178).

    x [NB, G*Cin, L]; weight [G*Cout, Cin, k]; gamma/beta: flat tensors addressed (g, o) -> [g*gstride + o]
    (a [G, 2*Cout] generated affine passes gamma = aff, beta = aff[:, Cout:] views with gstride = 2*Cout).
    """

    @staticmethod
    def forward(ctx, x, weight, gamma, beta, running_mean, running_var, keep, meta):
        (G, k, dilation, activation, highway, training, eps, momentum, dropout, gstride, stage) = meta
        _require_cuda(x, weight, gamma, beta)
        x = _f32c(x)
        NB, GC, L = x.shape
        Cin = GC // G
        if stage == 2:          # batch norm only
            Cout = Cin
        else:
            weight = _f32c(weight)
            Cout = weight.shape[0] // G
            assert weight.shape[1] == Cin and weight.shape[2] == k, (weight.shape, Cin, k)
        if stage != 1:
            assert gamma.stride(-1) == 1 and beta.stride(-1) == 1
        shape = _lib.ConvBlockShape(NB, G, Cin, Cout, L, k, dilation, ACTIVATIONS[activation], int(highway), int(training),
                                    eps, momentum, dropout, stage)
        lib = _lib.load()
        saved = _bytes(lib.b200tts_convblock_saved_bytes(ctypes.byref(shape)), x.device)
        ws = _bytes(lib.b200tts_convblock_workspace_bytes(ctypes.byref(shape)), x.device)
        Cf = Cout // 2 if highway else Cout
        out = torch.empty(NB, G * Cf, L, device=x.device, dtype=torch.float32)
        if keep is not None:
            assert keep.dtype == torch.uint8 and keep.is_contiguous() and tuple(keep.shape) == (NB, G * Cout, L)
        check(lib.b200tts_convblock_forward(ctypes.byref(shape), ptr(x), ptr(weight), ptr(gamma), ptr(beta), gstride,
                                            ptr(running_mean), ptr(running_var), ptr(keep), ptr(out), ptr(saved), ptr(ws), _stream()),
              'b200tts_convblock_forward')
        ctx.shape, ctx.gstride, ctx.saved_buf, ctx.keep = shape, gstride, saved, keep
        ctx.save_for_backward(x, weight, gamma, beta)
        return out

    @staticmethod
    def backward(ctx, dout):
        x, weight, gamma, beta = ctx.saved_tensors
        shape = ctx.shape
        lib = _lib.load()
        ws = _bytes(lib.b200tts_convblock_workspace_bytes(ctypes.byref(shape)), x.device)
        dout = _f32c(dout)
        dx = torch.empty_like(x)
        (dweight,), (r_weight,) = _grad_targets((weight,))           # leaf convolution weights accumulate straight into .grad
        # gamma / beta may be strided views of one generated-affine tensor: produce gradients in the same geometry
        G, Cout, gs = shape.G, shape.Cout, ctx.gstride
        if shape.stage == 1:    # convolution only: no affine parameters
            check(lib.b200tts_convblock_backward(ctypes.byref(shape), ptr(x), ptr(weight), None, None, gs, None, ptr(ctx.saved_buf), ptr(dout),
                                                 ptr(dx), ptr(dweight), None, None, ptr(ws), _stream()), 'b200tts_convblock_backward')
            return dx, r_weight, None, None, None, None, None, None
        if gs == Cout:      # plain batch norm: separate dense gamma / beta (leaf parameters accumulate straight into .grad)
            (dgamma, dbeta), (g_gamma, g_beta) = _grad_targets((gamma, beta))
            dgb = None
        else:               # generated affine [G, 2*Cout]: gamma = [:, :Cout], beta = [:, Cout:]
            dgb = torch.zeros(2 * G * Cout, device=x.device, dtype=torch.float32)
            dgamma, dbeta = dgb, dgb[Cout:]
        check(lib.b200tts_convblock_backward(ctypes.byref(shape), ptr(x), ptr(weight), ptr(gamma), ptr(beta), gs, ptr(ctx.keep),
                                             ptr(ctx.saved_buf), ptr(dout), ptr(dx), ptr(dweight), ptr(dgamma), ptr(dbeta),
                                             ptr(ws), _stream()), 'b200tts_convblock_backward')
        if dgb is not None:
            full = dgb.view(G, gs)
            g_gamma, g_beta = full[:, :Cout], full[:, Cout:]
        return dx, r_weight, g_gamma, g_beta, None, None, None, None


def conv_block_masked(x, lengths, weight, gamma, beta, running_mean, running_var, groups, kernel, dilation, activation, highway, eps,
                      gstride):
    """Eval-mode whole block over a zero-padded batch (no autograd): sample n keeps its first lengths[n] positions and every output
    past them is 0, so each sample's output equals running the block on it alone."""
    _require_cuda(x, weight, gamma, beta, lengths)
    with torch.no_grad():
        x, weight = _f32c(x), _f32c(weight)
        NB, GC, L = x.shape
        G = groups
        Cin, Cout = GC // G, weight.shape[0] // G
        assert weight.shape[1] == Cin and weight.shape[2] == kernel, (weight.shape, Cin, kernel)
        assert gamma.stride(-1) == 1 and beta.stride(-1) == 1
        lengths = lengths.to(device=x.device, dtype=torch.int32).contiguous()
        assert tuple(lengths.shape) == (NB,), (tuple(lengths.shape), NB)
        shape = _lib.ConvBlockShape(NB, G, Cin, Cout, L, kernel, dilation, ACTIVATIONS[activation], int(highway), 0, eps, 0.0, 0.0, 0)
        lib = _lib.load()
        saved = _bytes(lib.b200tts_convblock_saved_bytes(ctypes.byref(shape)), x.device)
        ws = _bytes(lib.b200tts_convblock_workspace_bytes(ctypes.byref(shape)), x.device)
        out = torch.empty(NB, G * (Cout // 2 if highway else Cout), L, device=x.device, dtype=torch.float32)
        check(lib.b200tts_convblock_forward_masked(ctypes.byref(shape), ptr(lengths), ptr(x), ptr(weight), ptr(gamma), ptr(beta), gstride,
                                                   ptr(running_mean), ptr(running_var), None, ptr(out), ptr(saved), ptr(ws), _stream()),
              'b200tts_convblock_forward_masked')
    return out


def conv_block(x, weight, gamma, beta, running_mean, running_var, keep, groups, kernel, dilation, activation, highway,
               training, eps, momentum, dropout, gstride, stage=0):
    """stage 0: the whole block; 1: grouped convolution only (gamma / beta None); 2: batch norm (+ activation / dropout) only (weight None)."""
    meta = (groups, kernel, dilation, activation, highway, training, eps, momentum, dropout, gstride, stage)
    return ConvBlockFunction.apply(x, weight, gamma, beta, running_mean, running_var, keep, meta)


# ------------------------------------------------------------------------------------------------
# one LSTM cell step (module-level API of ZoneoutLSTMCell / DropoutLSTMCell)
# ------------------------------------------------------------------------------------------------
class LSTMCellFunction(torch.autograd.Function):
    """(h, c) = cell(gates_pre, h_prev, c_prev) with the regulariser of the cell kind (reference modules/layers.py:26-34, 44-47);
    gates_pre = x . W_ih^T + b_ih + h . W_hh^T + b_hh comes from the library GEMM."""

    @staticmethod
    def forward(ctx, gates_pre, h_prev, c_prev, mask_h, mask_c, meta):
        kind, training, rate_h, rate_c = meta
        _require_cuda(gates_pre, h_prev, c_prev)
        gates = _f32c(gates_pre).clone()
        h_prev, c_prev = _f32c(h_prev), _f32c(c_prev)
        B, D = h_prev.shape
        h, c = torch.empty_like(h_prev), torch.empty_like(c_prev)
        check(_lib.load().b200tts_lstm_cell_forward(B, D, kind, int(training), rate_h, rate_c, ptr(gates), ptr(h_prev), ptr(c_prev), ptr(mask_h),
                                                    ptr(mask_c), ptr(h), ptr(c), _stream()), 'b200tts_lstm_cell_forward')
        ctx.meta, ctx.masks = meta, (mask_h, mask_c)
        ctx.save_for_backward(gates, c_prev)
        return h, c

    @staticmethod
    def backward(ctx, dh, dc):
        gates, c_prev = ctx.saved_tensors
        kind, training, rate_h, rate_c = ctx.meta
        B, D = c_prev.shape
        dh = _f32c(dh) if dh is not None else torch.zeros_like(c_prev)
        dc_io = _f32c(dc).clone() if dc is not None else torch.zeros_like(c_prev)
        dh_prev, dgates = torch.empty_like(c_prev), torch.empty_like(gates)
        check(_lib.load().b200tts_lstm_cell_backward(B, D, kind, int(training), rate_h, rate_c, ptr(gates), ptr(c_prev), ptr(ctx.masks[0]),
                                                     ptr(ctx.masks[1]), ptr(dh), ptr(dc_io), ptr(dh_prev), ptr(dgates), _stream()),
              'b200tts_lstm_cell_backward')
        return dgates, dh_prev, dc_io, None, None, None


def lstm_cell(cell_input, h, c, w_ih, w_hh, b_ih, b_hh, kind, training, rate_h, rate_c, mask_h=None, mask_c=None):
    gates = linear(cell_input, w_ih, b_ih) + linear(h, w_hh, b_hh)
    return LSTMCellFunction.apply(gates, h, c, mask_h, mask_c, (int(kind), bool(training), float(rate_h), float(rate_c)))


class GeneratorFunction(torch.autograd.Function):
    """out[g] = (e[g] . Wb^T + bb) . Wk^T + bk   (reference modules/generated.py:38-39, 81-82)."""

    @staticmethod
    def forward(ctx, e, Wb, bb, Wk, bk):
        _require_cuda(e, Wb, bb, Wk, bk)
        e, Wb, bb, Wk, bk = [_f32c(t) for t in (e, Wb, bb, Wk, bk)]
        G, gd = e.shape
        bn, R = Wb.shape[0], Wk.shape[0]
        eb = torch.empty(G, bn, device=e.device, dtype=torch.float32)
        out = torch.empty(G, R, device=e.device, dtype=torch.float32)
        check(_lib.load().b200tts_generator_forward(G, gd, bn, R, ptr(e), ptr(Wb), ptr(bb), ptr(Wk), ptr(bk), ptr(eb), ptr(out),
                                                    _stream()), 'b200tts_generator_forward')
        ctx.save_for_backward(e, Wb, Wk, eb, bb, bk)
        return out

    @staticmethod
    def backward(ctx, dout):
        e, Wb, Wk, eb, bb, bk = ctx.saved_tensors
        G, gd = e.shape
        bn, R = Wb.shape[0], Wk.shape[0]
        lib = _lib.load()
        dout = _f32c(dout)
        (de, dWb, dbb, dWk, dbk), returned = _grad_targets((e, Wb, bb, Wk, bk))       # all accumulated (+=) by the library
        ws = _bytes(lib.b200tts_generator_workspace_bytes(G, bn), e.device)
        check(lib.b200tts_generator_backward(G, gd, bn, R, ptr(e), ptr(Wb), ptr(Wk), ptr(eb), ptr(dout), ptr(de), ptr(dWb),
                                             ptr(dbb), ptr(dWk), ptr(dbk), ptr(ws), _stream()), 'b200tts_generator_backward')
        return tuple(returned)


def _grad_targets(params):
    """Where the library accumulates (+=) the gradients of `params` (the saved inputs of a Function).  A leaf parameter whose `.grad` already
    exists as a dense fp32 tensor of its own shape (the flat gradient bucket of distributed.GradBucket binds such views) is accumulated INTO
    directly and reported to autograd as None: no zero-filled temporary, no AccumulateGrad add per parameter (~2 launches and 3x the
    parameter bytes per tensor and step).  Everything else gets a fresh zero tensor that autograd accumulates as usual.
    -> (targets, returned)"""
    targets, returned = [], []
    for q in params:
        g = q.grad if (q is not None and q.is_leaf and q.requires_grad) else None
        if g is not None and g.dtype == torch.float32 and g.is_contiguous() and g.shape == q.shape and g.device == q.device:
            targets.append(g); returned.append(None)
        else:
            t = None if q is None else torch.zeros_like(q, dtype=torch.float32)
            targets.append(t); returned.append(t)
    return targets, returned


class EmbeddingFunction(torch.autograd.Function):
    """table[ids] with optional padding row (nn.Embedding, reference modules/tacotron2.py:237-239, 121-124)."""

    @staticmethod
    def forward(ctx, table, ids, padding_idx):
        _require_cuda(table, ids)
        table = _f32c(table)
        ids32 = ids.to(torch.int32).contiguous()
        E = table.shape[1]
        out = torch.empty(*ids.shape, E, device=table.device, dtype=torch.float32)
        check(_lib.load().b200tts_embedding_forward(ptr(out), E, ptr(table), ptr(ids32), ids32.numel(), E, _stream()),
              'b200tts_embedding_forward')
        ctx.save_for_backward(ids32)
        ctx.table_ref = table          # the parameter itself (not saved for its values): its .grad may be the accumulation target
        ctx.V, ctx.E, ctx.padding_idx = table.shape[0], E, -1 if padding_idx is None else int(padding_idx)
        return out

    @staticmethod
    def backward(ctx, dout):
        (ids32,) = ctx.saved_tensors
        dout = _f32c(dout)
        table = ctx.table_ref
        if table is not None and table.dtype == torch.float32 and table.is_contiguous():
            (dtable,), (ret,) = _grad_targets((table,))
        else:
            dtable = ret = torch.zeros(ctx.V, ctx.E, device=dout.device, dtype=torch.float32)
        check(_lib.load().b200tts_embedding_backward(ptr(dtable), ctx.V, ptr(dout), ctx.E, ptr(ids32), ids32.numel(), ctx.E,
                                                     ctx.padding_idx, _stream()), 'b200tts_embedding_backward')
        return ret, None, None


def embedding(table, ids, padding_idx=None):
    return EmbeddingFunction.apply(table, ids, padding_idx)


class BiLSTMFunction(torch.autograd.Function):
    """Packed bidirectional LSTM (reference modules/encoder.py:41-44)."""

    @staticmethod
    def forward(ctx, x, lengths, *params):
        _require_cuda(x, lengths, *params)
        x = _f32c(x)
        params = [_f32c(p) for p in params]
        lengths32 = lengths.to(torch.int32).contiguous()
        B, L, E = x.shape
        H = params[1].shape[1]
        shape = _lib.BiLSTMShape(B, L, E, H)
        lib = _lib.load()
        saved = _bytes(lib.b200tts_bilstm_saved_bytes(ctypes.byref(shape)), x.device)
        ws = _bytes(lib.b200tts_bilstm_workspace_bytes(ctypes.byref(shape)), x.device)
        out = torch.empty(B, L, 2 * H, device=x.device, dtype=torch.float32)
        pstruct = _lib.BiLSTMParams(*[ptr(p) for p in params])
        check(lib.b200tts_bilstm_forward(ctypes.byref(shape), ctypes.byref(pstruct), ptr(x), ptr(lengths32), ptr(out), ptr(saved),
                                         ptr(ws), _stream()), 'b200tts_bilstm_forward')
        ctx.shape, ctx.saved_buf = shape, saved
        ctx.save_for_backward(lengths32, *params)
        return out

    @staticmethod
    def backward(ctx, dout):
        lengths32, *params = ctx.saved_tensors
        shape = ctx.shape
        lib = _lib.load()
        dout = _f32c(dout)
        ws = _bytes(lib.b200tts_bilstm_workspace_bytes(ctypes.byref(shape)), dout.device)
        dx = torch.empty(shape.B, shape.L, shape.E, device=dout.device, dtype=torch.float32)
        grads, returned = _grad_targets(params)
        pstruct = _lib.BiLSTMParams(*[ptr(p) for p in params])
        gstruct = _lib.BiLSTMParams(*[ptr(g) for g in grads])
        check(lib.b200tts_bilstm_backward(ctypes.byref(shape), ctypes.byref(pstruct), ptr(lengths32), ptr(ctx.saved_buf), ptr(dout),
                                          ptr(dx), ctypes.byref(gstruct), ptr(ws), _stream()), 'b200tts_bilstm_backward')
        return (dx, None, *returned)


def bilstm(x, lengths, params):
    """params: 8 tensors in _lib.BILSTM_PARAM_FIELDS order."""
    return BiLSTMFunction.apply(x, lengths, *params)


class LinearFunction(torch.autograd.Function):
    """y = x . W^T + b on the library GEMM (used by the small dense layers outside the fused decoder)."""

    @staticmethod
    def forward(ctx, x, weight, bias):
        _require_cuda(x, weight)
        x2 = _f32c(x).reshape(-1, x.shape[-1])
        weight = _f32c(weight)
        out = gemm(x2, weight, False, True, bias=None if bias is None else _f32c(bias))
        ctx.save_for_backward(x2, weight)
        ctx.has_bias, ctx.xshape = bias is not None, x.shape
        return out.reshape(*x.shape[:-1], weight.shape[0])

    @staticmethod
    def backward(ctx, dout):
        x2, weight = ctx.saved_tensors
        d2 = _f32c(dout).reshape(-1, weight.shape[0])
        dx = gemm(d2, weight, False, False).reshape(ctx.xshape) if ctx.needs_input_grad[0] else None
        dw = gemm(d2, x2, True, False, splitk=8 if x2.shape[0] > 4096 else 1)
        db = d2.sum(0) if ctx.has_bias else None
        return dx, dw, db


def linear(x, weight, bias=None):
    return LinearFunction.apply(x, weight, bias)


# ------------------------------------------------------------------------------------------------
# fused loss
# ------------------------------------------------------------------------------------------------
class TacotronLossFunction(torch.autograd.Function):
    """[2*MSE(pre), MSE(post), stop BCE / (N + 2), guided attention] as ONE library op each way (reference modules/tacotron2.py:439-485);
    the guided-attention weights are evaluated in closed form inside the kernels (no [B, T, L] weight tensor, no Python loop)."""

    @staticmethod
    def forward(ctx, pre, post, stop, align, pre_target, post_target, stop_target, text_lengths, target_lengths, meta):
        guided, g, pos_weight, r = meta
        _require_cuda(pre, post, stop, pre_target, post_target, stop_target)
        pre, post, stop, pre_target, post_target, stop_target = [_f32c(t) for t in (pre, post, stop, pre_target, post_target, stop_target)]
        align = _f32c(align) if align is not None else None
        B, N, T = pre.shape
        L = align.shape[2] if align is not None else 1
        dev = pre.device
        tl = text_lengths.to(device=dev, dtype=torch.int32).contiguous()
        ml = target_lengths.to(device=dev, dtype=torch.int32).contiguous()
        shape = _lib.LossShape(B, N, T, L, int(bool(guided) and align is not None), float(g), float(pos_weight), int(r))
        lib = _lib.load()
        ws = _bytes(lib.b200tts_loss_workspace_bytes(), dev)
        losses = torch.empty(4, device=dev, dtype=torch.float32)
        check(lib.b200tts_tacotron_loss_forward(ctypes.byref(shape), ptr(pre), ptr(pre_target), ptr(post), ptr(post_target), ptr(stop),
                                                ptr(stop_target), ptr(align), ptr(tl), ptr(ml), ptr(losses), ptr(ws), _stream()),
              'b200tts_tacotron_loss_forward')
        ctx.shape = shape
        ctx.has_align = align is not None
        ctx.align_shape = None if align is None else tuple(align.shape)
        ctx.save_for_backward(pre, post, stop, pre_target, post_target, stop_target, tl, ml)
        return losses

    @staticmethod
    def backward(ctx, g):
        pre, post, stop, pre_target, post_target, stop_target, tl, ml = ctx.saved_tensors
        need = ctx.needs_input_grad
        g = _f32c(g)
        d_pre = torch.empty_like(pre) if need[0] else None
        d_post = torch.empty_like(post) if need[1] else None
        d_stop = torch.empty_like(stop) if need[2] else None
        d_align = torch.empty(ctx.align_shape, device=pre.device, dtype=torch.float32) if (need[3] and ctx.has_align) else None
        check(_lib.load().b200tts_tacotron_loss_backward(ctypes.byref(ctx.shape), ptr(pre), ptr(pre_target), ptr(post), ptr(post_target),
                                                         ptr(stop), ptr(stop_target), ptr(tl), ptr(ml), ptr(g), ptr(d_pre), ptr(d_post),
                                                         ptr(d_stop), ptr(d_align), _stream()), 'b200tts_tacotron_loss_backward')
        return d_pre, d_post, d_stop, d_align, None, None, None, None, None, None


def tacotron_loss(pre, post, stop, align, pre_target, post_target, stop_target, text_lengths, target_lengths, guided, g, pos_weight=100.0,
                  outputs_per_step=1):
    """-> tensor [4]: mel_pre, mel_pos, stop_token, guided_att (0 when `guided` is false).  align [B, ceil(T / r), L] has one row per decoder
    step; the guided term uses each utterance's step count ceil(target_length / r) in place of its frame count."""
    return TacotronLossFunction.apply(pre, post, stop, align, pre_target, post_target, stop_target, text_lengths, target_lengths,
                                      (guided, g, pos_weight, outputs_per_step))
