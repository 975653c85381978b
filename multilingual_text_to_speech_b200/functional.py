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


def gemm_tn_batched(a, b, bias=None):
    """out[i] = a[i]^T b^T + bias for a [B, K, M], b [N, K] -> [B, M, N] in one launch, each out[i] equal to gemm(a[i], b, trans_a=True,
    trans_b=True, bias=bias)."""
    _require_cuda(a, b)
    a, b = a.contiguous(), b.contiguous()
    B, K, M = a.shape
    N = b.shape[0]
    out = torch.empty(B, M, N, device=a.device, dtype=torch.float32)
    check(_lib.load().b200tts_gemm_f32(1, 1, M, N, K, 1.0, ptr(a), M, ptr(b), K, 0.0, ptr(out), N, ptr(bias), B, K * M, 0, M * N, 1, None,
                                       _stream()), 'b200tts_gemm_f32')
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


def _seed_tensor(seeds, device):
    """Request seeds (ints in [0, 2^64)) as a device int64 tensor holding their uint64 bits."""
    return torch.tensor([int(s) - (1 << 64) if int(s) >= 1 << 63 else int(s) for s in seeds], dtype=torch.int64, device=device)


def fill_keep_mask_rows(steps, width, rate, seeds, step0, stream_id, device):
    """Seeded keep masks [steps, len(seeds), width] (b200tts_fill_keep_mask_rows): row r continues, from step step0[r], the stream of
    fill_keep_mask((S, width), rate, seeds[r], stream_id)."""
    mask = torch.empty(int(steps), len(seeds), int(width), dtype=torch.uint8, device=device)
    s, t = _seed_tensor(seeds, device), torch.tensor([int(v) for v in step0], dtype=torch.int64, device=device)
    check(_lib.load().b200tts_fill_keep_mask_rows(ptr(mask), int(steps), len(seeds), int(width), float(rate), ptr(s), ptr(t), int(stream_id),
                                                 _stream()), 'b200tts_fill_keep_mask_rows')
    return mask


def fill_uniform_rows(nsteps, width, seeds, t0, stream_id, device):
    """Seeded uniforms in [0, 1), [len(seeds), nsteps, width] (b200tts_fill_uniform_rows): row r holds draws [t0[r] width, (t0[r] +
    nsteps) width) of the stream keyed by (seeds[r], stream_id)."""
    out = torch.empty(len(seeds), int(nsteps), int(width), dtype=torch.float32, device=device)
    s, t = _seed_tensor(seeds, device), torch.tensor([int(v) for v in t0], dtype=torch.int64, device=device)
    check(_lib.load().b200tts_fill_uniform_rows(ptr(out), len(seeds), int(nsteps), int(width), ptr(s), ptr(t), int(stream_id), _stream()),
          'b200tts_fill_uniform_rows')
    return out


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

    def __init__(self, cell_kind, training, rate_h, rate_c, prenet_rate, masks=None, teacher=None, att_extent=0, outputs_per_step=1,
                 att_window=None):
        self.att_extent = int(att_extent)    # 1: forward attention over each utterance's own length (inference of padded batches)
        # (back, ahead) or None: windowed location-sensitive attention, decoder_forward_chunk only (b200tts_decoder_shape.att_window_*)
        self.att_window = None if att_window is None else (int(att_window[0]), int(att_window[1]))
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
                         cfg.prenet_rate, att_kind, cfg.att_extent, cfg.outputs_per_step, *(cfg.att_window or (0, 0)))
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
        self.attended = torch.zeros(B, device=device, dtype=torch.int32)     # window centres (read only with a window)
        self.first = True

    def select(self, rows):
        """Keep only the utterances `rows` (a device index tensor), in that order: a finished utterance leaves the decode."""
        for name in ('att_h', 'att_c', 'gen_h', 'gen_c', 'context', 'cum_weights', 'frame', 'attended'):
            setattr(self, name, getattr(self, name).index_select(0, rows).contiguous())

    def grow(self, b, L):
        """Appends b rows (their values unset until reset_rows) and re-pads cum_weights to L positions: zeros past a row's old width
        (attention weights past a text's length are zero), or the first L positions when L is smaller."""
        for name in ('att_h', 'att_c', 'gen_h', 'gen_c', 'context', 'frame'):
            t = getattr(self, name)
            setattr(self, name, torch.cat([t, t.new_empty(b, t.shape[1])]) if b else t)
        if b:
            self.attended = torch.cat([self.attended, self.attended.new_empty(b)])
        cum = self.cum_weights
        out = cum.new_zeros(cum.shape[0] + b, L)
        w = min(L, cum.shape[1])
        out[:cum.shape[0], :w] = cum[:, :w]
        self.cum_weights = out

    def reset_rows(self, rows, forward_attention):
        """The initial state of a decode in `rows` (host ints; b200tts_decoder_state_reset_rows); other rows are untouched."""
        B, L = self.cum_weights.shape
        shape = DecoderShape(B=B, L=L, M=self.context.shape[1], D=self.att_h.shape[1], N=self.frame.shape[1],
                             att_kind=_lib.ATT_FORWARD if forward_attention else _lib.ATT_LOCATION)
        rows = [int(r) for r in rows]
        st = self.struct()
        check(_lib.load().b200tts_decoder_state_reset_rows(ctypes.byref(shape), ctypes.byref(st), (ctypes.c_int * len(rows))(*rows), len(rows),
                                                           _stream()), 'b200tts_decoder_state_reset_rows')

    def struct(self):
        return _lib.DecoderState(*[ptr(t) for t in (self.att_h, self.att_c, self.gen_h, self.gen_c, self.context, self.cum_weights, self.frame,
                                                    self.attended)])


def decoder_forward_chunk(cfg, memory, text_lengths, params, state, frames, forced=None):
    """`frames` free-running frames (frames / r decoder steps; a multiple of r) continuing from `state` (updated in place); no autograd
    (inference).  cfg.att_window, if set, confines each step's attention to the window around state.attended, which the call advances.
    forced: None, or (rows, weights) with rows a device int32 tensor [F] of distinct rows and weights a device float32 tensor
    [frames / r, F, L] whose row [i, k] is the attention of step i of utterance rows[k] (b200tts_decoder_inputs.forced_*).
    -> spectrogram [B, frames, N], stop [B, frames], alignment [B, frames / r, L]."""
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
        if forced is not None:
            rows, weights = forced
            assert rows.dtype == torch.int32 and rows.is_cuda and rows.is_contiguous() and rows.dim() == 1, rows
            assert weights.dtype == torch.float32 and weights.is_cuda and weights.is_contiguous() and \
                tuple(weights.shape) == (cfg.steps(T), rows.shape[0], L), tuple(weights.shape)
            inputs.forced_rows, inputs.forced_count, inputs.forced_alignment = ptr(rows), rows.shape[0], ptr(weights)
        st = state.struct()
        check(lib.b200tts_decoder_forward_chunk(ctypes.byref(shape), ctypes.byref(pstruct), ctypes.byref(inputs), ctypes.byref(outs),
                                                ctypes.byref(st), int(state.first), ptr(ws), nbytes, _stream()), 'b200tts_decoder_forward_chunk')
        state.first = False
    return spec, stop, align


def _durations_host(durations, name):
    d = np.asarray(durations.detach().cpu() if torch.is_tensor(durations) else durations)
    if d.ndim != 1 or d.shape[0] < 1 or not np.issubdtype(d.dtype, np.integer):
        raise ValueError(f'{name}: durations must be a non-empty 1-D integer array [L], got shape {d.shape} of {d.dtype}')
    if (d < 0).any():
        raise ValueError(f'{name}: durations must be >= 0')
    return d.astype(np.int64)


def durations_to_alignment(durations, r=1):
    """Frames per symbol (int [L], each >= 0) -> the one-hot attention rows [S, L] float32 of a decode with r frames per step that gives
    each symbol its frames: S = ceil(sum(d) / r), and step s attends the symbol whose frame range [C_{j-1}, C_j) (C the cumulative
    frames) holds frame s r.  A symbol with no frames is never attended.  For Alignment.durations from Tacotron.align these are the
    one-hot rows of the monotonic path (Alignment.step_durations).  On the durations' device (the host for arrays and lists)."""
    d = _durations_host(durations, 'durations_to_alignment')
    r = int(r)
    if r < 1:
        raise ValueError(f'durations_to_alignment: r must be >= 1 (got {r})')
    total = int(d.sum())
    if total == 0:
        raise ValueError('durations_to_alignment: the durations total 0 frames')
    S = -(-total // r)
    sym = np.searchsorted(np.cumsum(d), np.arange(S) * r, side='right')
    rows = np.zeros((S, d.shape[0]), dtype=np.float32)
    rows[np.arange(S), sym] = 1.0
    return torch.from_numpy(rows).to(durations.device if torch.is_tensor(durations) else 'cpu')


def scale_durations(durations, factor):
    """Speaking-rate control: frames per symbol (int [L], each >= 0) stretched by `factor` (> 1 slower, < 1 faster) -> int [L] of the
    input's type.  The new symbol boundaries are B_j = floor(factor C_j + 0.5) in float64 (C the cumulative frames) and each new
    duration is B_j - B_{j-1}, so the total is the rounded scaled total and no rounding error accumulates.  At strong speed-ups a short
    symbol can get 0 frames, and then it is not attended (durations_to_alignment).  ValueError for a factor that is not finite or
    is <= 0, and for a result of 0 frames."""
    d = _durations_host(durations, 'scale_durations')
    f = float(factor)
    if not np.isfinite(f) or f <= 0:
        raise ValueError(f'scale_durations: factor must be finite and > 0 (got {factor!r})')
    bounds = np.floor(f * np.cumsum(d).astype(np.float64) + 0.5).astype(np.int64)
    out = np.diff(bounds, prepend=0)
    if int(bounds[-1]) == 0:
        raise ValueError(f'scale_durations: {int(d.sum())} frames scaled by {f} total 0 frames')
    if torch.is_tensor(durations):
        return torch.from_numpy(out).to(device=durations.device, dtype=durations.dtype)
    return out.astype(np.asarray(durations).dtype)


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


def _aligned_bytes(n, device, align=256):
    buf = torch.empty(int(n) + align, dtype=torch.uint8, device=device)
    off = (-buf.data_ptr()) % align
    return buf[off:off + int(n)]


def _workspace(bytes_fn, shape, device, alloc=_bytes):
    """The workspace that bytes_fn (a b200tts_*_workspace_bytes entry point) sizes for `shape`, allocated by `alloc`; raises B200TTSError
    with the library's message when bytes_fn rejects the shape."""
    n = bytes_fn(ctypes.byref(shape))
    if n == 0:
        raise _lib.B200TTSError(f'{bytes_fn.__name__}: {_lib.load().b200tts_last_error().decode()}')
    return alloc(n, device)


class ConvBlockFunction(torch.autograd.Function):
    """pad -> grouped conv -> batch norm -> activation -> dropout (-> highway) (reference modules/layers.py:50-178).

    x [NB, G*Cin, L]; weight [G*Cout, Cin, k]; gamma/beta: flat tensors addressed (g, o) -> [g*gstride + o]
    (a [G, 2*Cout] generated affine passes gamma = aff, beta = aff[:, Cout:] views with gstride = 2*Cout).
    counts (or None): int32 [G] on the device, the occupied rows of each channel block (b200tts_convblock_forward_counts); rows
    nb >= counts[g] of block g are vacant and their outputs and gradients are 0.
    """

    @staticmethod
    def forward(ctx, x, weight, gamma, beta, running_mean, running_var, keep, counts, meta):
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
        if counts is None:
            check(lib.b200tts_convblock_forward(ctypes.byref(shape), ptr(x), ptr(weight), ptr(gamma), ptr(beta), gstride,
                                                ptr(running_mean), ptr(running_var), ptr(keep), ptr(out), ptr(saved), ptr(ws), _stream()),
                  'b200tts_convblock_forward')
        else:
            assert counts.dtype == torch.int32 and counts.is_cuda and tuple(counts.shape) == (G,), (counts.dtype, tuple(counts.shape), G)
            check(lib.b200tts_convblock_forward_counts(ctypes.byref(shape), ptr(counts), G, NB, ptr(x), ptr(weight), ptr(gamma), ptr(beta),
                                                       gstride, ptr(running_mean), ptr(running_var), ptr(keep), ptr(out), ptr(saved), ptr(ws),
                                                       _stream()), 'b200tts_convblock_forward_counts')
        ctx.shape, ctx.gstride, ctx.saved_buf, ctx.keep, ctx.counts = shape, gstride, saved, keep, counts
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

        def run(weight, gamma, beta, keep, dgamma, dbeta):
            if ctx.counts is None:
                check(lib.b200tts_convblock_backward(ctypes.byref(shape), ptr(x), ptr(weight), ptr(gamma), ptr(beta), gs, ptr(keep),
                                                     ptr(ctx.saved_buf), ptr(dout), ptr(dx), ptr(dweight), ptr(dgamma), ptr(dbeta),
                                                     ptr(ws), _stream()), 'b200tts_convblock_backward')
            else:
                check(lib.b200tts_convblock_backward_counts(ctypes.byref(shape), ptr(ctx.counts), G, shape.NB, ptr(x), ptr(weight), ptr(gamma),
                                                            ptr(beta), gs, ptr(keep), ptr(ctx.saved_buf), ptr(dout), ptr(dx), ptr(dweight),
                                                            ptr(dgamma), ptr(dbeta), ptr(ws), _stream()), 'b200tts_convblock_backward_counts')

        if shape.stage == 1:    # convolution only: no affine parameters
            run(weight, None, None, None, None, None)
            return dx, r_weight, None, None, None, None, None, None, None
        if gs == Cout:      # plain batch norm: separate dense gamma / beta (leaf parameters accumulate straight into .grad)
            (dgamma, dbeta), (g_gamma, g_beta) = _grad_targets((gamma, beta))
            dgb = None
        else:               # generated affine [G, 2*Cout]: gamma = [:, :Cout], beta = [:, Cout:]
            dgb = torch.zeros(2 * G * Cout, device=x.device, dtype=torch.float32)
            dgamma, dbeta = dgb, dgb[Cout:]
        run(weight, gamma, beta, ctx.keep, dgamma, dbeta)
        if dgb is not None:
            full = dgb.view(G, gs)
            g_gamma, g_beta = full[:, :Cout], full[:, Cout:]
        return dx, r_weight, g_gamma, g_beta, None, None, None, None, None


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
               training, eps, momentum, dropout, gstride, stage=0, counts=None):
    """stage 0: the whole block; 1: grouped convolution only (gamma / beta None); 2: batch norm (+ activation / dropout) only (weight None).
    counts: None (every row of every channel block is an utterance) or int32 [groups] on the device, the occupied rows per block."""
    meta = (groups, kernel, dilation, activation, highway, training, eps, momentum, dropout, gstride, stage)
    return ConvBlockFunction.apply(x, weight, gamma, beta, running_mean, running_var, keep, counts, meta)


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


# ------------------------------------------------------------------------------------------------
# Griffin-Lim vocoder (packed ragged layout: utterance b owns frames off[b]:off[b+1])
# ------------------------------------------------------------------------------------------------
def vocoder_workspace(shape, device):
    """Workspace of b200tts_griffinlim for `shape` (a _lib.VocoderShape); raises on an invalid shape."""
    return _workspace(_lib.load().b200tts_vocoder_workspace_bytes, shape, device)


def spectrogram_magnitude(shape, log_spec, mel_basis=None, mel_pinv_t=None, nnls_step=0.0):
    """log_spec [total_frames, n_mels or K] -> magnitudes [total_frames, K] = db_to_amplitude, then (mel) NNLS, then ** power."""
    _require_cuda(log_spec, mel_basis, mel_pinv_t)
    for t in (mel_basis, mel_pinv_t):
        if t is not None and not (t.dtype == torch.float32 and t.is_contiguous()):
            raise ValueError('the mel basis and its transposed pseudo-inverse must be contiguous fp32 [n_mels, K] tensors')
    log_spec = _f32c(log_spec)
    S = torch.empty(shape.total_frames, shape.N // 2 + 1, device=log_spec.device, dtype=torch.float32)
    check(_lib.load().b200tts_spectrogram_magnitude(ctypes.byref(shape), ptr(log_spec), ptr(mel_basis), ptr(mel_pinv_t), float(nnls_step),
                                                    ptr(S), _stream()), 'b200tts_spectrogram_magnitude')
    return S


def griffinlim(shape, S, off, angles, rebuilt, first, iters, wave=None, workspace=None):
    """`iters` Griffin-Lim iterations on the state (angles, rebuilt), both complex64 [total_frames, K], updated in place; then the inverse
    into `wave` (fp32 [hop * (total_frames - B)]) when it is given."""
    _require_cuda(S, off, angles, rebuilt, wave)
    assert angles.dtype == torch.complex64 and rebuilt.dtype == torch.complex64 and angles.is_contiguous() and rebuilt.is_contiguous()
    assert off.dtype == torch.int32 and S.dtype == torch.float32 and S.is_contiguous()
    ws = vocoder_workspace(shape, S.device) if workspace is None else workspace
    check(_lib.load().b200tts_griffinlim(ctypes.byref(shape), ptr(S), ptr(off), ptr(angles), ptr(rebuilt), int(bool(first)), int(iters),
                                         ptr(wave), ptr(ws), ws.numel(), _stream()), 'b200tts_griffinlim')
    return wave


def deemphasis_normalize(shape, wave, off):
    """In place per utterance: de-emphasis (when shape.preemphasis != 0), then division by the largest sample."""
    _require_cuda(wave, off)
    check(_lib.load().b200tts_deemphasis_normalize(ctypes.byref(shape), ptr(wave), ptr(off), _stream()), 'b200tts_deemphasis_normalize')
    return wave


def gl_stream_workspace_bytes(shape):
    """Bytes of the streaming Griffin-Lim workspace for `shape` (a _lib.GLStreamShape), host only; raises ValueError on an invalid shape."""
    n = _lib.load().b200tts_gl_stream_workspace_bytes(ctypes.byref(shape))
    if n == 0:
        raise ValueError(_lib.load().b200tts_last_error().decode())
    return n


def gl_stream_workspace(shape, device):
    """A 256-byte aligned workspace of b200tts_gl_stream_run for `shape`."""
    return _aligned_bytes(gl_stream_workspace_bytes(shape), device)


def gl_stream_reset(shape, ws, slots):
    """Reset the listed slots (host ints) to empty streams and write the FFT tables."""
    n = len(slots)
    check(_lib.load().b200tts_gl_stream_reset(ctypes.byref(shape), ptr(ws), ws.numel(), (ctypes.c_int * n)(*slots), n, _stream()),
          'b200tts_gl_stream_reset')


def gl_stream_run(shape, rows, S_new, wave, ws):
    """One call over `rows` (a list of _lib.GLStreamRow): new magnitudes S_new [rows, K] fp32, released samples into `wave`."""
    _require_cuda(S_new, wave, ws)
    assert wave.dtype == torch.float32 and wave.is_contiguous()
    assert S_new.dtype == torch.float32 and S_new.is_contiguous()
    n = len(rows)
    check(_lib.load().b200tts_gl_stream_run(ctypes.byref(shape), (_lib.GLStreamRow * n)(*rows), n, ptr(S_new), ptr(wave), ptr(ws), ws.numel(),
                                            _stream()), 'b200tts_gl_stream_run')
    return wave


# ------------------------------------------------------------------------------------------------
# audio analysis (packed ragged layout: utterance b owns samples soff[b]:soff[b+1] and frames off[b]:off[b+1])
# ------------------------------------------------------------------------------------------------
def analysis_workspace(shape, device):
    """Workspace of b200tts_stft_magnitude for `shape` (a _lib.AnalysisShape); raises on an invalid shape."""
    return _workspace(_lib.load().b200tts_analysis_workspace_bytes, shape, device)


def stft_magnitude(shape, wave, soff, off, mel_basis=None, workspace=None):
    """wave fp32 [total_samples] -> |STFT| [total_frames, K], or mel_basis . |STFT| [total_frames, n_mels] when shape.n_mels > 0."""
    _require_cuda(wave, soff, off, mel_basis)
    if mel_basis is not None and not (mel_basis.dtype == torch.float32 and mel_basis.is_contiguous()):
        raise ValueError('the mel basis must be a contiguous fp32 [n_mels, K] tensor')
    assert soff.dtype == torch.int32 and off.dtype == torch.int32 and wave.dtype == torch.float32 and wave.is_contiguous()
    ws = analysis_workspace(shape, wave.device) if workspace is None else workspace
    out = torch.empty(shape.total_frames, shape.n_mels or shape.N // 2 + 1, device=wave.device, dtype=torch.float32)
    check(_lib.load().b200tts_stft_magnitude(ctypes.byref(shape), ptr(wave), ptr(soff), ptr(off), ptr(mel_basis), ptr(out), ptr(ws),
                                             ws.numel(), _stream()), 'b200tts_stft_magnitude')
    return out


def amplitude_to_db(shape, S, off, out=None):
    """Per utterance amplitude_to_db(ref=max): S [total_frames, bins] -> dB, into `out` (may be S; new tensor when None)."""
    _require_cuda(S, off, out)
    assert S.dtype == torch.float32 and S.is_contiguous() and off.dtype == torch.int32
    out = torch.empty_like(S) if out is None else out
    check(_lib.load().b200tts_amplitude_to_db(ctypes.byref(shape), ptr(S), ptr(off), ptr(out), _stream()), 'b200tts_amplitude_to_db')
    return out


def mel_cepstrum(mel_db, n_mfcc):
    """mel_db [total_frames, n_mels] -> DCT-II (ortho) of mel_db / 10, first n_mfcc coefficients [total_frames, n_mfcc]."""
    _require_cuda(mel_db)
    mel_db = _f32c(mel_db)
    out = torch.empty(mel_db.shape[0], n_mfcc, device=mel_db.device, dtype=torch.float32)
    check(_lib.load().b200tts_mel_cepstrum(mel_db.shape[0], mel_db.shape[1], int(n_mfcc), ptr(mel_db), ptr(out), _stream()),
          'b200tts_mel_cepstrum')
    return out


def mel_cepstral_distortion(cep_a, off_a, cep_b, off_b, mode):
    """Packed cepstra [frames, n_mfcc] of B pairs -> (mcd float64 [B], path length int32 [B]); mode 'cut', 'stretch' or 'dtw'."""
    _require_cuda(cep_a, off_a, cep_b, off_b)
    if mode not in _lib.MCD_MODES:
        raise ValueError(f'unknown mode {mode!r}; expected one of {sorted(_lib.MCD_MODES)}')
    assert off_a.dtype == torch.int32 and off_b.dtype == torch.int32 and cep_a.shape[1] == cep_b.shape[1]
    cep_a, cep_b = _f32c(cep_a), _f32c(cep_b)
    B = off_a.numel() - 1
    mcd = torch.empty(B, device=cep_a.device, dtype=torch.float64)
    plen = torch.empty(B, device=cep_a.device, dtype=torch.int32)
    check(_lib.load().b200tts_mel_cepstral_distortion(B, cep_a.shape[1], _lib.MCD_MODES[mode], ptr(cep_a), ptr(off_a), ptr(cep_b), ptr(off_b),
                                                      ptr(mcd), ptr(plen), _stream()), 'b200tts_mel_cepstral_distortion')
    return mcd, plen


# ------------------------------------------------------------------------------------------------
# pitch analysis (probabilistic YIN in three stages, include/b200tts.h; the same packed ragged layout)
# ------------------------------------------------------------------------------------------------
def pitch_cmnd(shape, wave, soff, off):
    """wave fp32 [total_samples] -> the cumulative mean normalised difference d' float64 [total_frames, K] (a _lib.PitchShape)."""
    _require_cuda(wave, soff, off)
    assert soff.dtype == torch.int32 and off.dtype == torch.int32 and wave.dtype == torch.float32 and wave.is_contiguous()
    out = torch.empty(shape.total_frames, shape.max_period - shape.min_period + 1, device=wave.device, dtype=torch.float64)
    check(_lib.load().b200tts_pitch_cmnd(ctypes.byref(shape), ptr(wave), ptr(soff), ptr(off), ptr(out), _stream()), 'b200tts_pitch_cmnd')
    return out


def pitch_observations(shape, cmnd):
    """d' [total_frames, K] -> (voiced-bin probabilities float64 [total_frames, n_bins], voiced_prob float64 [total_frames])."""
    _require_cuda(cmnd)
    assert cmnd.dtype == torch.float64 and cmnd.is_contiguous() and tuple(cmnd.shape) == (shape.total_frames,
                                                                                          shape.max_period - shape.min_period + 1)
    obs = torch.empty(shape.total_frames, shape.n_bins, device=cmnd.device, dtype=torch.float64)
    voiced_prob = torch.empty(shape.total_frames, device=cmnd.device, dtype=torch.float64)
    check(_lib.load().b200tts_pitch_observations(ctypes.byref(shape), ptr(cmnd), ptr(obs), ptr(voiced_prob), _stream()),
          'b200tts_pitch_observations')
    return obs, voiced_prob


def pitch_viterbi(shape, obs, voiced_prob, off, log_trans):
    """Viterbi decode of each utterance -> state int32 [total_frames] (voiced bin i when < n_bins, else unvoiced bin state - n_bins).
    log_trans: float64 [2, W, n_bins] (include/b200tts.h)."""
    _require_cuda(obs, voiced_prob, off, log_trans)
    assert obs.dtype == torch.float64 and voiced_prob.dtype == torch.float64 and log_trans.dtype == torch.float64 and off.dtype == torch.int32
    assert tuple(log_trans.shape) == (2, shape.transition_width, shape.n_bins) and log_trans.is_contiguous()
    ws = _workspace(_lib.load().b200tts_pitch_workspace_bytes, shape, obs.device)
    state = torch.empty(shape.total_frames, device=obs.device, dtype=torch.int32)
    check(_lib.load().b200tts_pitch_viterbi(ctypes.byref(shape), ptr(obs), ptr(voiced_prob), ptr(off), ptr(log_trans), ptr(state), ptr(ws),
                                            ws.numel(), _stream()), 'b200tts_pitch_viterbi')
    return state


# ------------------------------------------------------------------------------------------------
# pitch modification (TD-PSOLA in two stages, include/b200tts.h; the same packed ragged layout)
# ------------------------------------------------------------------------------------------------
def psola_workspace(shape, device):
    """The uint8 workspace of a pitch-shift batch (a _lib.PsolaShape) on `device`."""
    return _workspace(_lib.load().b200tts_psola_workspace_bytes, shape, device)


def psola_marks(shape, wave, soff, f0, ratio, off, ws=None):
    """Analysis and synthesis pitch marks of each utterance from wave fp32 [total_samples], f0 and ratio fp32 [total_frames] -> the
    workspace (include/b200tts.h describes its layout; psola_workspace_views reads it)."""
    _require_cuda(wave, soff, f0, ratio, off)
    assert soff.dtype == torch.int32 and off.dtype == torch.int32 and wave.dtype == torch.float32 and wave.is_contiguous()
    assert f0.dtype == torch.float32 and ratio.dtype == torch.float32 and f0.is_contiguous() and ratio.is_contiguous()
    assert f0.numel() == ratio.numel() == shape.total_frames and wave.numel() == shape.total_samples
    ws = psola_workspace(shape, wave.device) if ws is None else ws
    check(_lib.load().b200tts_psola_marks(ctypes.byref(shape), ptr(wave), ptr(soff), ptr(f0), ptr(ratio), ptr(off), ptr(ws), ws.numel(),
                                          _stream()), 'b200tts_psola_marks')
    return ws


def psola_workspace_views(shape, ws):
    """(info int32 [B, 4], marks, spacings, centres, nearest marks int32 [total_samples], voiced uint8 [total_samples]) viewing `ws`."""
    B, N = shape.B, shape.total_samples
    ints = ws[:(4 * B + 4 * N) * 4].view(torch.int32)
    info = ints[:4 * B].view(B, 4)
    marks, spacing, centre, nearest = (ints[4 * B + i * N:4 * B + (i + 1) * N] for i in range(4))
    return info, marks, spacing, centre, nearest, ws[(4 * B + 4 * N) * 4:(4 * B + 4 * N) * 4 + N]


def psola_overlap_add(shape, wave, soff, ws):
    """The grains overlap-added from the marks psola_marks wrote to `ws` -> fp32 [total_samples]."""
    _require_cuda(wave, soff, ws)
    assert soff.dtype == torch.int32 and wave.dtype == torch.float32 and wave.is_contiguous() and wave.numel() == shape.total_samples
    out = torch.empty_like(wave)
    check(_lib.load().b200tts_psola_overlap_add(ctypes.byref(shape), ptr(wave), ptr(soff), ptr(ws), ws.numel(), ptr(out), _stream()),
          'b200tts_psola_overlap_add')
    return out


# ------------------------------------------------------------------------------------------------
# time-scale modification (WSOLA in two stages, include/b200tts.h; the same packed ragged layout)
# ------------------------------------------------------------------------------------------------
def wsola_positions(shape, wave, soff, warp, foff):
    """The input position of every synthesis frame (a _lib.WsolaShape batch) from wave fp32 [total_samples] and the warp fp64
    [total_frames] -> int32 [total_frames]."""
    _require_cuda(wave, soff, warp, foff)
    assert soff.dtype == torch.int32 and foff.dtype == torch.int32 and wave.dtype == torch.float32 and wave.is_contiguous()
    assert warp.dtype == torch.float64 and warp.is_contiguous() and warp.numel() == shape.total_frames
    assert wave.numel() == shape.total_samples
    positions = torch.empty(shape.total_frames, dtype=torch.int32, device=wave.device)
    check(_lib.load().b200tts_wsola_positions(ctypes.byref(shape), ptr(wave), ptr(soff), ptr(warp), ptr(foff), ptr(positions),
                                              _stream()), 'b200tts_wsola_positions')
    return positions


def wsola_overlap_add(shape, wave, soff, positions, foff, ooff):
    """The frames at `positions` (wsola_positions) overlap-added with the periodic Hann window -> fp32 [total_out_samples]."""
    _require_cuda(wave, soff, positions, foff, ooff)
    assert soff.dtype == torch.int32 and foff.dtype == torch.int32 and ooff.dtype == torch.int32 and positions.dtype == torch.int32
    assert wave.dtype == torch.float32 and wave.is_contiguous() and wave.numel() == shape.total_samples
    assert positions.is_contiguous() and positions.numel() == shape.total_frames
    out = torch.empty(shape.total_out_samples, dtype=torch.float32, device=wave.device)
    check(_lib.load().b200tts_wsola_overlap_add(ctypes.byref(shape), ptr(wave), ptr(soff), ptr(positions), ptr(foff), ptr(ooff), ptr(out),
                                                _stream()), 'b200tts_wsola_overlap_add')
    return out


# ------------------------------------------------------------------------------------------------
# waveform front end: polyphase resampling and silence trimming (include/b200tts.h; the same packed ragged layout)
# ------------------------------------------------------------------------------------------------
def resample(shape, wave, soff, ooff, plan, taps):
    """Each utterance of a _lib.ResampleShape batch resampled by its plan row (up, down, h_len, table offset) with the packed polyphase
    taps fp64 -> fp32 [total_out_samples]."""
    _require_cuda(wave, soff, ooff, plan, taps)
    assert soff.dtype == torch.int32 and ooff.dtype == torch.int32 and plan.dtype == torch.int32 and plan.is_contiguous()
    assert wave.dtype == torch.float32 and wave.is_contiguous() and wave.numel() == shape.total_samples and plan.numel() == 4 * shape.B
    assert taps.dtype == torch.float64 and taps.is_contiguous() and taps.numel() == shape.total_taps
    out = torch.empty(shape.total_out_samples, dtype=torch.float32, device=wave.device)
    check(_lib.load().b200tts_resample(ctypes.byref(shape), ptr(wave), ptr(soff), ptr(ooff), ptr(plan), ptr(taps), ptr(out), _stream()),
          'b200tts_resample')
    return out


def trim_silence(shape, wave, soff, foff):
    """The frame powers and the non-silent bounds of a _lib.TrimShape batch -> (fp64 [total_frames], int32 [B, 2] (start, end))."""
    _require_cuda(wave, soff, foff)
    assert soff.dtype == torch.int32 and foff.dtype == torch.int32
    assert wave.dtype == torch.float32 and wave.is_contiguous() and wave.numel() == shape.total_samples
    power = torch.empty(shape.total_frames, dtype=torch.float64, device=wave.device)
    bounds = torch.empty(shape.B, 2, dtype=torch.int32, device=wave.device)
    check(_lib.load().b200tts_trim_silence(ctypes.byref(shape), ptr(wave), ptr(soff), ptr(foff), ptr(power), ptr(bounds), _stream()),
          'b200tts_trim_silence')
    return power, bounds


def symbol_average(track, durations, voiced=None):
    """Per-symbol means of a frame track [B, T] over each symbol's frames: symbol l of row b owns frames [C_{l-1}, C_l), C the cumulative
    sum of durations [B, L] (frames past C_{L-1} belong to no symbol).  Summed in frame order in float64; with `voiced` [B, T] (bool) only
    voiced frames count, as FastPitch averages pitch.  A symbol with no counted frames gets 0.  -> float64 [B, L] on track's device.
    Raises ValueError on wrong shapes, negative durations or durations summing past T."""
    if not torch.is_tensor(track) or track.dim() != 2 or not track.dtype.is_floating_point:
        raise ValueError(f'track must be a floating [B, T] tensor, got {tuple(track.shape) if torch.is_tensor(track) else type(track)}')
    if not torch.is_tensor(durations) or durations.dim() != 2 or durations.dtype.is_floating_point or durations.dtype == torch.bool:
        raise ValueError('durations must be an integer [B, L] tensor')
    B, T = track.shape
    if durations.shape[0] != B:
        raise ValueError(f'durations has {durations.shape[0]} rows for {B} tracks')
    d = durations.detach().cpu().long()
    if bool((d < 0).any()):
        raise ValueError('durations must be non-negative')
    ends = d.cumsum(1)
    if ends.shape[1] and int(ends[:, -1].max()) > T:
        raise ValueError(f'durations sum to {int(ends[:, -1].max())} frames; the track has {T}')
    x = track.detach().cpu().double()
    w = torch.ones(B, T, dtype=torch.float64)
    if voiced is not None:
        if not torch.is_tensor(voiced) or tuple(voiced.shape) != (B, T) or voiced.dtype != torch.bool:
            raise ValueError(f'voiced must be a bool [{B}, {T}] tensor')
        w = voiced.detach().cpu().double()
        x = torch.where(voiced.cpu(), x, torch.zeros_like(x))
    L = d.shape[1]
    # symbol of every frame (L for frames past the last symbol): one CPU index_add per row sums the frames of each symbol in frame order
    owner = torch.searchsorted(ends, torch.arange(T).expand(B, T).contiguous(), right=True)
    sums = torch.zeros(B, L + 1, dtype=torch.float64)
    counts = torch.zeros(B, L + 1, dtype=torch.float64)
    for b in range(B):
        sums[b].index_add_(0, owner[b], x[b])
        counts[b].index_add_(0, owner[b], w[b])
    mean = torch.where(counts > 0, sums / counts.clamp(min=1), torch.zeros_like(sums))[:, :L]
    return mean.to(track.device)


# ------------------------------------------------------------------------------------------------
# forced alignment (monotonic alignment search over attention probabilities, include/b200tts.h)
# ------------------------------------------------------------------------------------------------
def _host_lengths(x, B, what):
    if torch.is_tensor(x):
        if x.dtype.is_floating_point or x.dtype in (torch.bool, torch.complex64, torch.complex128):
            raise ValueError(f'{what} must be integers, got {x.dtype}')
        x = x.tolist()
    x = np.asarray(x)
    if x.ndim != 1 or x.shape[0] != B:
        raise ValueError(f'{what} must hold one length per utterance ({B}), got shape {tuple(x.shape)}')
    if x.dtype.kind not in 'iu':
        raise ValueError(f'{what} must be integers, got {x.dtype}')
    return [int(v) for v in x]


def check_alignment_inputs(weights, text_lengths, step_lengths):
    """The host checks of monotonic_alignment, made before any device work.  -> (text lengths, step lengths) as lists of ints."""
    if not torch.is_tensor(weights) or weights.dim() != 3:
        raise ValueError(f'weights must be a [B, S, L] tensor, got {tuple(weights.shape) if torch.is_tensor(weights) else type(weights)}')
    if weights.dtype != torch.float32:
        raise ValueError(f'weights must be float32, got {weights.dtype}')
    B, S, L = weights.shape
    if B < 1 or S < 1 or L < 1:
        raise ValueError(f'weights must be non-empty, got shape {tuple(weights.shape)}')
    tl, sl = check_alignment_lengths(text_lengths, step_lengths, B, S, L)
    if not bool(torch.isfinite(weights).all()):
        raise ValueError('weights must be finite')
    return tl, sl


def check_alignment_lengths(text_lengths, step_lengths, B, S, L):
    """Host checks of B utterances' text lengths and step counts against a padded [B, S, L] grid and the search's shared-memory limits.
    -> both as lists of ints."""
    tl, sl = _host_lengths(text_lengths, B, 'text_lengths'), _host_lengths(step_lengths, B, 'step_lengths')
    for b, (n, s) in enumerate(zip(tl, sl)):
        if not 1 <= n <= L:
            raise ValueError(f'utterance {b}: text length {n} is outside [1, {L}]')
        if not 1 <= s <= S:
            raise ValueError(f'utterance {b}: step count {s} is outside [1, {S}]')
        if s < n:
            raise ValueError(f'utterance {b}: {s} steps cannot cover {n} symbols (a monotonic path needs at least one step per symbol)')
        if n > _lib.ALIGN_MAX_SYMBOLS:
            raise ValueError(f'utterance {b}: {n} symbols exceed the {_lib.ALIGN_MAX_SYMBOLS} the search keeps in shared memory')
        if s * n > _lib.ALIGN_MAX_CELLS:
            raise ValueError(f'utterance {b}: {s} steps x {n} symbols = {s * n} cells exceed the {_lib.ALIGN_MAX_CELLS} back-pointer bits '
                             'the search keeps in shared memory')
    return tl, sl


def _align_args(weights, tl, sl):
    """Library view of the checked weights, cut to the longest lengths, and the lengths on its device."""
    _require_cuda(weights)
    w = weights[:, :max(sl), :max(tl)]
    if w.stride(2) != 1:
        w = w.contiguous()
    shape = _lib.AlignShape(w.shape[0], w.shape[1], w.shape[2], w.stride(1), w.stride(0))
    lengths = torch.tensor([tl, sl], dtype=torch.int32).to(w.device)
    return shape, w, lengths[0], lengths[1]


def monotonic_alignment(weights, text_lengths, step_lengths, return_path=False):
    """Monotonic alignment search (Glow-TTS MAS) over attention probabilities weights [B, S, L] (fp32, CUDA; forward attention's,
    windowed decoding's or any other): per utterance b, over steps s < step_lengths[b] and symbols l < text_lengths[b], the path from
    symbol 0 to symbol L_b - 1 that advances by 0 or 1 symbol per step and maximises sum log(max(w, 1e-8)) in fp64; on equal values it
    stays on the same symbol (include/b200tts.h states the rule).  Lengths: int tensors or sequences, 1 <= L_b <= S_b.
    -> (durations int32 [B, L]: steps per symbol, each >= 1, summing to S_b, 0 past L_b; path_logp float64 [B]) and, with return_path,
    path int32 [B, S]: the symbol of every step, -1 past S_b.  Raises ValueError before any device work on a wrong rank or dtype,
    lengths out of range, S_b < L_b, a shape past B200TTS_ALIGN_MAX_SYMBOLS / _MAX_CELLS, or non-finite weights."""
    tl, sl = check_alignment_inputs(weights, text_lengths, step_lengths)
    B, S, L = weights.shape
    shape, w, d_tl, d_sl = _align_args(weights, tl, sl)
    durations = torch.empty(B, shape.L, device=w.device, dtype=torch.int32)
    path_logp = torch.empty(B, device=w.device, dtype=torch.float64)
    path = torch.empty(B, shape.S, device=w.device, dtype=torch.int32) if return_path else None
    check(_lib.load().b200tts_monotonic_alignment(ctypes.byref(shape), ptr(w), ptr(d_tl), ptr(d_sl), ptr(durations), ptr(path_logp),
                                                  ptr(path), _stream()), 'b200tts_monotonic_alignment')
    durations = torch.nn.functional.pad(durations, (0, L - shape.L))
    if not return_path:
        return durations, path_logp
    return durations, path_logp, torch.nn.functional.pad(path, (0, S - shape.S), value=-1)


def alignment_scores(weights, text_lengths, step_lengths):
    """Alignment quality per utterance of weights [B, S, L] over its valid steps and symbols (the checks of monotonic_alignment apply).
    -> dict of focus_rate (float32 [B], the mean over steps of the step's largest weight), coverage (float32 [B], the fraction of
    symbols whose summed weight reaches 0.5), max_jump (int32 [B], the largest forward move of the per-step argmax) and moves_back
    (bool [B], whether the argmax ever moves backwards)."""
    tl, sl = check_alignment_inputs(weights, text_lengths, step_lengths)
    shape, w, d_tl, d_sl = _align_args(weights, tl, sl)
    B = w.shape[0]
    out = {k: torch.empty(B, device=w.device, dtype=dt) for k, dt in (('focus_rate', torch.float32), ('coverage', torch.float32),
                                                                      ('max_jump', torch.int32), ('moves_back', torch.int32))}
    check(_lib.load().b200tts_alignment_scores(ctypes.byref(shape), ptr(w), ptr(d_tl), ptr(d_sl), *(ptr(v) for v in out.values()), _stream()),
          'b200tts_alignment_scores')
    out['moves_back'] = out['moves_back'].bool()
    return out


# ------------------------------------------------------------------------------------------------
# WaveRNN vocoder (fold rows: see include/b200tts.h)
# ------------------------------------------------------------------------------------------------
def wavernn_upsample_layer(x, fir, scale):
    """x [C, len] -> [C, len * scale]: nearest stretch x scale, then the FIR fir [2 scale + 1] with zero padding scale."""
    _require_cuda(x, fir)
    x, fir = _f32c(x), _f32c(fir)
    out = torch.empty(x.shape[0], x.shape[1] * scale, device=x.device, dtype=torch.float32)
    check(_lib.load().b200tts_wavernn_upsample_layer(x.shape[0], x.shape[1], int(scale), ptr(fir), ptr(x), ptr(out), _stream()),
          'b200tts_wavernn_upsample_layer')
    return out


def wavernn_fold(shape, mel_up, mel_off, frames, row_utt, row_fold, fir, aux, t0, nsteps, out=None):
    """feat [nsteps, rows, n_mels + aux_dims] of the loop steps [t0, t0 + nsteps) (shape: a _lib.WaveRNNFoldShape)."""
    _require_cuda(mel_up, mel_off, frames, row_utt, row_fold, fir, aux)
    if out is None:
        out = torch.empty(nsteps, shape.rows, shape.n_mels + shape.aux_dims, device=mel_up.device, dtype=torch.float32)
    check(_lib.load().b200tts_wavernn_fold(ctypes.byref(shape), ptr(mel_up), ptr(mel_off), ptr(frames), ptr(row_utt), ptr(row_fold), ptr(fir),
                                           ptr(aux), int(t0), int(nsteps), ptr(out), _stream()), 'b200tts_wavernn_fold')
    return out


def wavernn_upsample_segments(x, lens, fir, scale):
    """wavernn_upsample_layer over packed segments: x holds [C, lens[g]] for each g one after another (flat) -> the same packing of
    [C, lens[g] scale], each segment equal to its own wavernn_upsample_layer."""
    _require_cuda(x, fir)
    x, fir = _f32c(x), _f32c(fir)
    n = len(lens)
    C = x.numel() // max(sum(lens), 1)
    out = torch.empty(x.numel() * scale, device=x.device, dtype=torch.float32)
    check(_lib.load().b200tts_wavernn_upsample_segments(C, n, (ctypes.c_int * n)(*lens), int(scale), ptr(fir), ptr(x), ptr(out), _stream()),
          'b200tts_wavernn_upsample_segments')
    return out


def wavernn_window_rows(rows, nsteps, mel, fir, aux):
    """feat [nsteps, len(rows), n_mels + aux_dims] of many rows' positions (rows: _lib.WaveRNNWindowRow descriptors) from the packed mel and
    aux windows."""
    _require_cuda(mel, fir, aux)
    n = len(rows)
    w0 = rows[0].w
    out = torch.empty(int(nsteps), n, w0.n_mels + w0.aux_dims, device=mel.device, dtype=torch.float32)
    check(_lib.load().b200tts_wavernn_window_rows((_lib.WaveRNNWindowRow * n)(*rows), n, int(nsteps), ptr(_f32c(mel)), ptr(_f32c(fir)),
                                                  ptr(_f32c(aux)), ptr(out), _stream()), 'b200tts_wavernn_window_rows')
    return out


def wavernn_workspace(shape, device):
    """256-byte aligned workspace of the sample loop for `shape` (a _lib.WaveRNNShape); raises on an invalid shape."""
    return _workspace(_lib.load().b200tts_wavernn_workspace_bytes, shape, device, _aligned_bytes)


def wavernn_params(weights):
    """_lib.WaveRNNParams from a dict of fp32 contiguous CUDA tensors named as its fields (the caller keeps them alive)."""
    return _lib.WaveRNNParams(*[ptr(weights[n]) for n in _lib.WAVERNN_PARAM_FIELDS])


def wavernn_prepare(shape, params, ws):
    check(_lib.load().b200tts_wavernn_prepare(ctypes.byref(shape), ctypes.byref(params), ptr(ws), ws.numel(), _stream()),
          'b200tts_wavernn_prepare')


def wavernn_run(shape, params, cond, t0, nsteps, uniforms, out, ws, dbg=None):
    """Loop steps [t0, t0 + nsteps); cond: (c, g1, c2, p1, p2) [nsteps, rows, width] fp32 CUDA tensors."""
    cs = _lib.WaveRNNCond(*[ptr(t) for t in cond])
    check(_lib.load().b200tts_wavernn_run(ctypes.byref(shape), ctypes.byref(params), ctypes.byref(cs), int(t0), int(nsteps), ptr(uniforms),
                                          ptr(out), ptr(dbg), ptr(ws), ws.numel(), _stream()), 'b200tts_wavernn_run')


def wavernn_run_stream(shape, params, cond, t, nsteps, uniforms, out, ws):
    """nsteps more loop steps after the t run since the last prepare; uniforms [rows, nsteps, U] and out [rows, nsteps] hold this call's
    steps only."""
    cs = _lib.WaveRNNCond(*[ptr(t_) for t_ in cond])
    check(_lib.load().b200tts_wavernn_run_stream(ctypes.byref(shape), ctypes.byref(params), ctypes.byref(cs), int(t), int(nsteps), ptr(uniforms),
                                                 ptr(out), ptr(ws), ws.numel(), _stream()), 'b200tts_wavernn_run_stream')


def wavernn_run_rows(shape, params, cond, row_t, row_n, nsteps, uniforms, out, ws):
    """Up to nsteps more steps of each of the first len(row_t) rows: row r has run row_t[r] steps (int64, device) and runs row_n[r] (int32,
    device); cond [nsteps, rows, width], uniforms [rows, nsteps, U], out [rows, nsteps]."""
    cs = _lib.WaveRNNCond(*[ptr(t_) for t_ in cond])
    check(_lib.load().b200tts_wavernn_run_rows(ctypes.byref(shape), ctypes.byref(params), ctypes.byref(cs), ptr(row_t), ptr(row_n),
                                               int(row_t.numel()), int(nsteps), ptr(uniforms), ptr(out), ptr(ws), ws.numel(), _stream()),
          'b200tts_wavernn_run_rows')


def wavernn_reset_rows(shape, ws, rows):
    """Zero the recurrent state of the listed rows (host ints)."""
    n = len(rows)
    check(_lib.load().b200tts_wavernn_reset_rows(ctypes.byref(shape), ptr(ws), ws.numel(), (ctypes.c_int * n)(*rows), n, _stream()),
          'b200tts_wavernn_reset_rows')


def wavernn_aborted(shape, ws):
    flag = ctypes.c_int(0)
    check(_lib.load().b200tts_wavernn_aborted(ctypes.byref(shape), ptr(ws), ws.numel(), ctypes.byref(flag), _stream()), 'b200tts_wavernn_aborted')
    return flag.value != 0


def wavernn_deemphasis(y, mu, a):
    """In place on the folded samples y [rows, len]: mu-law decode (mu > 0), then lfilter([1], [1, -a]) along each row."""
    _require_cuda(y)
    assert y.dtype == torch.float32 and y.is_contiguous() and y.dim() == 2
    check(_lib.load().b200tts_wavernn_deemphasis(y.shape[0], y.shape[1], int(mu), float(a), ptr(y), _stream()), 'b200tts_wavernn_deemphasis')
    return y


def wavernn_unfold(y, frames, row_off, wave_off, total, hop, target, overlap, mu):
    """Folded samples y [rows, target + 2 overlap] -> the packed waveform [total] (mu-law decoded when mu > 0)."""
    _require_cuda(y, frames, row_off, wave_off)
    wave = torch.empty(max(int(total), 1), device=y.device, dtype=torch.float32)
    check(_lib.load().b200tts_wavernn_unfold(frames.numel(), int(hop), int(target), int(overlap), int(mu), ptr(frames), ptr(row_off),
                                             ptr(wave_off), int(total), ptr(_f32c(y)), ptr(wave), _stream()), 'b200tts_wavernn_unfold')
    return wave[:int(total)]


def wavernn_unfold_streams(y, streams, base, period, hop, target, overlap, mu):
    """Positions [q0, q1) of each folded stream (streams: _lib.WaveRNNUnfoldStream descriptors) from fold samples in the storage y, fold
    source e at y[base[e] + j mod period[e]] (base int64 and period int32 on the device) -> the packed waveform [sum q1 - q0]."""
    _require_cuda(y, base, period)
    n = len(streams)
    total = sum(int(s.q1 - s.q0) for s in streams)
    wave = torch.empty(max(total, 1), device=y.device, dtype=torch.float32)
    check(_lib.load().b200tts_wavernn_unfold_streams(n, int(hop), int(target), int(overlap), int(mu), (_lib.WaveRNNUnfoldStream * n)(*streams),
                                                     ptr(base), ptr(period), base.numel(), total, ptr(_f32c(y)), ptr(wave), _stream()),
          'b200tts_wavernn_unfold_streams')
    return wave[:total]


# ------------------------------------------------------------------------------------------------
# WaveRNN training
# ------------------------------------------------------------------------------------------------
def gru_seq_shape(B, T, R):
    """_lib.GRUSeqShape; raises on a shape the loops do not take."""
    shape = _lib.GRUSeqShape(int(B), int(T), int(R))
    if _lib.load().b200tts_gru_seq_workspace_bytes(ctypes.byref(shape)) == 0:
        raise _lib.B200TTSError(f'b200tts_gru_seq: {_lib.load().b200tts_last_error().decode()}')
    return shape


def gru_seq_aborted(shape, ws):
    flag = ctypes.c_int(0)
    check(_lib.load().b200tts_gru_seq_aborted(ctypes.byref(shape), ptr(ws), ws.numel(), ctypes.byref(flag), _stream()), 'b200tts_gru_seq_aborted')
    return flag.value != 0


class GRUSeqGuard:
    """One zeroed loop workspace for GRU loops of one shape (both GRUs of a training step, forward and reverse, in stream order) and its
    abort flag, which collects a grid-barrier timeout of any of them.  check() synchronises, reads the flag once and raises if it is set."""

    def __init__(self, shape, device):
        self.shape = shape
        self.ws = _aligned_bytes(_lib.load().b200tts_gru_seq_workspace_bytes(ctypes.byref(shape)), device)
        self.ws.zero_()
        self.checked = False

    def check(self):
        self.checked = True
        if gru_seq_aborted(self.shape, self.ws):
            raise _lib.B200TTSError('gru_seq: a GRU loop timed out at a grid barrier')


def column_sum(x, out):
    """out += x.sum(0) for x [rows, cols] (fp32, fixed order)."""
    rows, cols = x.shape
    ws = _bytes(_lib.load().b200tts_column_sum_workspace_bytes(cols), x.device)
    check(_lib.load().b200tts_column_sum(rows, cols, ptr(x), ptr(out), ptr(ws), ws.numel(), _stream()), 'b200tts_column_sum')
    return out


class GRUSeqFunction(torch.autograd.Function):
    """torch.nn.GRU (batch_first, one layer, h0 = 0) on the persistent fp32 sequence loops: x [B, T, in] -> every step's output [B, T, R].
    gi = x W_ih^T + b_ih runs on the library GEMM before the loop; the backward's weight and input gradients are GEMMs over the loop's
    dgi / dgh histories, the bias gradients fixed-order column sums.  The loops run on `guard`'s workspace; check_fwd / check_bwd read its
    abort flag after the forward / reverse loop.  `trace` (a dict or None, tests): receives the input, gi, the outputs, the saved state and,
    after the backward, dgi, dgh and every step's total dh."""

    @staticmethod
    def forward(ctx, x, w_ih, w_hh, b_ih, b_hh, trace, guard, check_fwd, check_bwd):
        _require_cuda(x, w_ih, w_hh, b_ih, b_hh)
        B, T, In = x.shape
        R = w_hh.shape[1]
        shape = guard.shape
        assert (shape.B, shape.T, shape.R) == (B, T, R), ((shape.B, shape.T, shape.R), (B, T, R))
        w_ih, w_hh, b_ih, b_hh = _f32c(w_ih), _f32c(w_hh), _f32c(b_ih), _f32c(b_hh)
        x2 = _f32c(x).reshape(B * T, In)
        gi = gemm(x2, w_ih, trans_b=True, bias=b_ih)
        lib = _lib.load()
        h = torch.empty(B, T, R, device=x.device, dtype=torch.float32)
        saved = torch.empty(B, T, 4 * R, device=x.device, dtype=torch.float32)
        with _Timed('gru_seq_fwd'):
            check(lib.b200tts_gru_seq_forward(ctypes.byref(shape), ptr(gi), ptr(w_hh), ptr(b_hh), ptr(h), ptr(saved), ptr(guard.ws),
                                              guard.ws.numel(), _stream()), 'b200tts_gru_seq_forward')
        if check_fwd:
            guard.check()
        if trace is not None:
            trace.update(x=x2, gi=gi.view(B, T, 3 * R), h=h, saved=saved)
        ctx.guard, ctx.check_bwd, ctx.trace = guard, check_bwd, trace
        ctx.save_for_backward(x2, w_ih, w_hh, b_ih, b_hh, h, saved)
        return h

    @staticmethod
    def backward(ctx, dh):
        x2, w_ih, w_hh, b_ih, b_hh, h, saved = ctx.saved_tensors
        guard, trace = ctx.guard, ctx.trace
        shape = guard.shape
        B, T, R = shape.B, shape.T, shape.R
        dh = _f32c(dh)
        dgi = torch.empty(B, T, 3 * R, device=dh.device, dtype=torch.float32)
        dgh = torch.empty_like(dgi)
        dh_dbg = torch.empty(B, T, R, device=dh.device, dtype=torch.float32) if trace is not None else None
        lib = _lib.load()
        with _Timed('gru_seq_bwd'):
            check(lib.b200tts_gru_seq_backward(ctypes.byref(shape), ptr(w_hh), ptr(h), ptr(saved), ptr(dh), ptr(dgi), ptr(dgh), ptr(dh_dbg),
                                               ptr(guard.ws), guard.ws.numel(), _stream()), 'b200tts_gru_seq_backward')
        if ctx.check_bwd:
            guard.check()
        if trace is not None:
            trace.update(dgi=dgi, dgh=dgh, dh=dh_dbg, dh_ext=dh)
        dgi2, dgh2, h2 = dgi.view(B * T, 3 * R), dgh.view(B * T, 3 * R), h.view(B * T, R)
        (dw_ih, dw_hh, db_ih, db_hh), returned = _grad_targets(ctx.saved_tensors[1:5])
        sk = 8 if B * T > 4096 else 1
        gemm(dgi2, x2, True, False, out=dw_ih, beta=1.0, splitk=sk)
        # d W_hh = sum over b and t >= 1 of dgh[b, t]^T h[b, t - 1]: the flat rows shifted by one pair every dgh row but the first with the
        # h row before it, which for t = 0 of utterance b >= 1 is h[b - 1, T - 1]; those B - 1 products are taken back out
        gemm(dgh2[1:], h2[:-1], True, False, out=dw_hh, beta=1.0, splitk=sk)
        if B > 1:
            gemm(dgh[1:, 0], h[:-1, T - 1], True, False, out=dw_hh, beta=1.0, alpha=-1.0)
        column_sum(dgi2, db_ih)
        column_sum(dgh2, db_hh)
        dx = gemm(dgi2, w_ih).view(B, T, -1) if ctx.needs_input_grad[0] else None
        return (dx, *returned, None, None, None, None)


def gru_seq(x, w_ih, w_hh, b_ih, b_hh, trace=None, guard=None, check_fwd=None, check_bwd=None):
    """One GRU on the sequence loops.  Without a guard the call owns a fresh one and reads its abort flag once: after the reverse loop when
    a backward will run, else after the forward loop."""
    if guard is None:
        guard = GRUSeqGuard(gru_seq_shape(x.shape[0], x.shape[1], w_hh.shape[1]), x.device)
        grads = torch.is_grad_enabled() and any(t.requires_grad for t in (x, w_ih, w_hh, b_ih, b_hh))
        check_fwd, check_bwd = not grads, grads
    return GRUSeqFunction.apply(x, w_ih, w_hh, b_ih, b_hh, trace, guard, bool(check_fwd), bool(check_bwd))


class WaveRNNUpsampleLayerFunction(torch.autograd.Function):
    """One upsampling layer pair (nearest stretch x scale, FIR of 2 scale + 1 taps, zero padding scale) of every row of x [C, len] ->
    [C, len scale]; the backward is the library's adjoint (d fir accumulated into its .grad view when there is one)."""

    @staticmethod
    def forward(ctx, x, fir, scale):
        _require_cuda(x, fir)
        x, f = _f32c(x), _f32c(fir).reshape(-1)
        out = torch.empty(x.shape[0], x.shape[1] * scale, device=x.device, dtype=torch.float32)
        check(_lib.load().b200tts_wavernn_upsample_layer(x.shape[0], x.shape[1], int(scale), ptr(f), ptr(x), ptr(out), _stream()),
              'b200tts_wavernn_upsample_layer')
        ctx.scale = int(scale)
        ctx.save_for_backward(x, fir)
        return out

    @staticmethod
    def backward(ctx, dout):
        x, fir = ctx.saved_tensors
        C, L = x.shape
        lib = _lib.load()
        dout = _f32c(dout)
        din = torch.empty_like(x) if ctx.needs_input_grad[0] else None
        (dfir,), (ret,) = _grad_targets((fir,))
        ws = _bytes(lib.b200tts_wavernn_upsample_layer_backward_workspace_bytes(C, L, ctx.scale), x.device)
        check(lib.b200tts_wavernn_upsample_layer_backward(C, L, ctx.scale, ptr(_f32c(fir).reshape(-1)), ptr(x), ptr(dout), ptr(din), ptr(dfir),
                                                          ptr(ws), ws.numel(), _stream()), 'b200tts_wavernn_upsample_layer_backward')
        return din, ret, None


def wavernn_upsample_layer_train(x, fir, scale):
    return WaveRNNUpsampleLayerFunction.apply(x, fir, scale)


class WaveRNNStretchFunction(torch.autograd.Function):
    """aux [B, F, C] -> [B, F hop, C], each frame repeated hop times; the backward sums each frame's hop positions on the library."""

    @staticmethod
    def forward(ctx, aux, hop):
        _require_cuda(aux)
        ctx.hop, ctx.dims = int(hop), tuple(aux.shape)
        return _f32c(aux).repeat_interleave(int(hop), dim=1)

    @staticmethod
    def backward(ctx, dup):
        B, Fr, C = ctx.dims
        dup = _f32c(dup)
        daux = torch.empty(B, Fr, C, device=dup.device, dtype=torch.float32)
        check(_lib.load().b200tts_wavernn_stretch_backward(B, Fr, C, ctx.hop, ptr(dup), ptr(daux), _stream()), 'b200tts_wavernn_stretch_backward')
        return daux, None


def wavernn_stretch(aux, hop):
    return WaveRNNStretchFunction.apply(aux, hop)


class WaveRNNLossFunction(torch.autograd.Function):
    """Mean RAW cross entropy / MOL discretized-logistic loss of logits [N, n_out] (one fused kernel writes the loss and d logits)."""

    @staticmethod
    def forward(ctx, logits, target, mode):
        _require_cuda(logits, target)
        logits = _f32c(logits)
        N, n = logits.shape
        lib = _lib.load()
        if mode == 'RAW':
            target = target.to(torch.int32).contiguous()
        else:
            target = _f32c(target)
        if target.numel() != N:
            raise ValueError(f'{target.numel()} targets for {N} rows of logits')
        loss = torch.empty((), device=logits.device, dtype=torch.float32)
        dlogits = torch.empty_like(logits)
        ws = _bytes(lib.b200tts_wavernn_loss_workspace_bytes(N), logits.device)
        with _Timed('wavernn_loss'):
            check(lib.b200tts_wavernn_loss(_lib.WAVERNN_MODES[mode], N, n, ptr(logits), ptr(target), ptr(loss), ptr(dlogits), ptr(ws), ws.numel(),
                                           _stream()), 'b200tts_wavernn_loss')
        ctx.save_for_backward(dlogits)
        return loss

    @staticmethod
    def backward(ctx, g):
        (dlogits,) = ctx.saved_tensors
        return dlogits * g, None, None


def wavernn_loss_rows(logits, target, mode):
    return WaveRNNLossFunction.apply(logits, target, mode)


def wavernn_cut_windows(mode, bits, seq_len, pad, hop, mels, frame_start, labels, sample_start, table, out=None):
    """Training windows of the device corpus (mels fp32 [feat, total frames], labels uint16, int64 frame / sample starts per utterance) for
    the device table int32 [B, 2] of (utterance, mel offset): (x [B, seq_len] fp32, y [B, seq_len] (RAW int64, MOL fp32), m [B, feat,
    mel_win] fp32), written into `out` when given.  The table is not checked (modules/wavernn.py VocoderCorpus validates it on the host)."""
    _require_cuda(mels, frame_start, labels, sample_start, table)
    B, feat = table.shape[0], mels.shape[0]
    if out is None:
        win = seq_len // hop + 2 * pad
        out = (torch.empty(B, seq_len, device=mels.device, dtype=torch.float32),
               torch.empty(B, seq_len, device=mels.device, dtype=torch.float32 if mode == 'MOL' else torch.int64),
               torch.empty(B, feat, win, device=mels.device, dtype=torch.float32))
    x, y, m = out
    check(_lib.load().b200tts_wavernn_cut_windows(_lib.WAVERNN_MODES[mode], int(bits), B, feat, int(seq_len), int(pad), int(hop), ptr(mels),
                                                  mels.shape[1], ptr(frame_start), ptr(labels), ptr(sample_start), ptr(table), ptr(x), ptr(y),
                                                  ptr(m), _stream()), 'b200tts_wavernn_cut_windows')
    return x, y, m


def gru_seq_abort_flag_copy(guard, dst):
    """Enqueue a copy of `guard`'s abort flag into dst (one int32, pinned host or device) on the current stream, without synchronising."""
    check(_lib.load().b200tts_gru_seq_abort_flag_copy(ctypes.byref(guard.shape), ptr(guard.ws), guard.ws.numel(), ptr(dst), _stream()),
          'b200tts_gru_seq_abort_flag_copy')
