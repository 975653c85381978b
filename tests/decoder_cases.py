"""Decoder parity cases: the CUDA decoder (through the C ABI) against the CPU oracle, forward and backward.

Used by tests/test_gpu_decoder.py and by __graft_entry__.smoke().
"""
import types
import numpy as np
import torch

from helpers import Golden, assert_close
from oracle import tacotron_oracle as O

PARAM_KEYS = [
    ('prenet_w0', '_prenet._layers.0.weight'), ('prenet_b0', '_prenet._layers.0.bias'),
    ('prenet_w1', '_prenet._layers.1.weight'), ('prenet_b1', '_prenet._layers.1.bias'),
    ('att_w_ih', '_decoder._attention_lstm.weight_ih'), ('att_w_hh', '_decoder._attention_lstm.weight_hh'),
    ('att_b_ih', '_decoder._attention_lstm.bias_ih'), ('att_b_hh', '_decoder._attention_lstm.bias_hh'),
    ('gen_w_ih', '_decoder._generator_lstm.weight_ih'), ('gen_w_hh', '_decoder._generator_lstm.weight_hh'),
    ('gen_b_ih', '_decoder._generator_lstm.bias_ih'), ('gen_b_hh', '_decoder._generator_lstm.bias_hh'),
    ('attn_query', '_attention._query.weight'), ('attn_memory', '_attention._memory.weight'),
    ('attn_location', '_attention._location.weight'), ('attn_loc_features', '_attention._loc_features.weight'),
    ('attn_bias', '_attention._bias'), ('attn_energy', '_attention._energy.weight'),
    ('frame_w', '_decoder._frame_prediction.weight'), ('frame_b', '_decoder._frame_prediction.bias'),
    ('stop_w', '_decoder._stop_prediction.weight'), ('stop_b', '_decoder._stop_prediction.bias'),
]


# bf16 perf-mode gradient gates (relative L2 error vs the operand-quantised oracle), see run_case_bf16
GRAD_REL_BOUND = 4e-2
GRAD_REL_BOUND_ATT = 8e-2


class Case:
    """hp (namespace), sd (fp32 CPU state dict, reference names), memory [B,L,M], lengths, target [B,N,T], tape."""
    pass


def _decoder_sd_alias(sd):
    for k in list(sd):
        if k.startswith('_prenet.') or k.startswith('_attention.'):
            sd['_decoder.' + k] = sd[k]
    return sd


def full_dim_case(B=8, L=40, T=30, M=288, D=1024, P=256, A=128, C=32, K=31, N=80, kind='dropout', seed=0, ragged=True,
                  training=True, tf=1.0, dropout=True):
    g = torch.Generator().manual_seed(seed)
    rn = lambda *s, scale=1.0: torch.randn(*s, generator=g) * scale   # noqa: E731
    hp = types.SimpleNamespace(num_mels=N, decoder_dimension=D, decoder_regularization=kind, zoneout_hidden=0.1,
                               zoneout_cell=0.1, dropout_hidden=0.1, dropout=0.5, multi_speaker=False, multi_language=False,
                               max_output_length=T, stop_frames=5, prenet_dimension=P)
    s_in = lambda n: 1.0 / np.sqrt(n)   # noqa: E731
    sd = {
        '_prenet._layers.0.weight': rn(P, N, scale=s_in(N)), '_prenet._layers.0.bias': rn(P, scale=0.1),
        '_prenet._layers.1.weight': rn(P, P, scale=s_in(P)), '_prenet._layers.1.bias': rn(P, scale=0.1),
        '_decoder._attention_lstm.weight_ih': rn(4 * D, P + M, scale=2 * s_in(D)),
        '_decoder._attention_lstm.weight_hh': rn(4 * D, D, scale=2 * s_in(D)),
        '_decoder._attention_lstm.bias_ih': rn(4 * D, scale=0.1), '_decoder._attention_lstm.bias_hh': rn(4 * D, scale=0.1),
        '_decoder._generator_lstm.weight_ih': rn(4 * D, D + M, scale=s_in(D)),
        '_decoder._generator_lstm.weight_hh': rn(4 * D, D, scale=s_in(D)),
        '_decoder._generator_lstm.bias_ih': rn(4 * D, scale=0.1), '_decoder._generator_lstm.bias_hh': rn(4 * D, scale=0.1),
        '_attention._query.weight': rn(A, D, scale=3 * s_in(D)), '_attention._memory.weight': rn(A, M, scale=3 * s_in(M)),
        '_attention._location.weight': rn(A, C, scale=s_in(C)), '_attention._loc_features.weight': rn(C, 1, K, scale=s_in(K)),
        '_attention._bias': rn(1, A, scale=0.1), '_attention._energy.weight': rn(1, A, scale=6 * s_in(A)),
        '_decoder._frame_prediction.weight': rn(N, D + M, scale=s_in(D + M)), '_decoder._frame_prediction.bias': rn(N, scale=0.1),
        '_decoder._stop_prediction.weight': rn(1, D + M, scale=s_in(D + M)), '_decoder._stop_prediction.bias': rn(1, scale=0.1),
    }
    c = Case()
    c.hp, c.sd = hp, _decoder_sd_alias(sd)
    c.memory = rn(B, L, M)
    if ragged:
        lens = torch.sort(torch.randint(max(1, L // 2), L + 1, (B,), generator=g), descending=True).values
        lens[0] = L
    else:
        lens = torch.full((B,), L)
    c.lengths = lens
    c.target = rn(B, N, T)
    c.training = training
    keep = lambda shape, p: (torch.rand(*shape, generator=g) >= p).float()   # noqa: E731
    tape = {'teacher': torch.rand(T, generator=g) > (1 - tf)}
    if dropout:
        tape.update(prenet0=keep((B, T + 1, P), 0.5), prenet1=keep((B, T + 1, P), 0.5),
                    step_prenet0=keep((T, B, P), 0.5), step_prenet1=keep((T, B, P), 0.5))
        if training:
            tape.update(att_h=keep((T, B, D), 0.1), gen_h=keep((T, B, D), 0.1))
            if kind == 'zoneout':
                tape.update(att_c=keep((T, B, D), 0.1), gen_c=keep((T, B, D), 0.1))
    c.tape = tape
    c.name = f'full B{B} L{L} T{T} M{M} {kind} tf{tf}'
    return c


def golden_case(name):
    """Decoder inputs taken from a golden fixture (encoder output of the unmodified reference as memory source)."""
    gld = Golden(name)
    c = Case()
    c.hp = gld.hp
    c.sd = gld.cast_sd(torch.float32)
    i = gld.inputs
    L = gld.L
    spk = i['speakers'][:, None].expand(-1, L) if 'speakers' in i else None
    lang = i['languages'][:, None].expand(-1, L) if 'languages' in i else None
    c.memory = O.decoder_memory(c.sd, c.hp, gld.out['enc'], spk, lang)
    c.lengths = i['text_length']
    c.target = i['target']
    c.training = gld.train
    c.tape = gld.tape
    c.name = 'golden ' + name
    c.golden = gld
    return c


def _oracle_run(c, dtype, with_grad):
    sd = {k: (v.to(dtype).clone().requires_grad_(with_grad) if v.is_floating_point() else v) for k, v in c.sd.items()
          if not (k.startswith('_decoder._prenet.') or k.startswith('_decoder._attention.'))}
    _decoder_sd_alias(sd)
    memory = c.memory.to(dtype).clone().requires_grad_(with_grad)
    tape = {k: (v if k == 'teacher' else v.to(dtype)) for k, v in c.tape.items()}
    hp = types.SimpleNamespace(**vars(c.hp))
    hp.multi_speaker = hp.multi_language = False        # memory already carries the embeddings
    mask = O.lengths_to_mask(c.lengths, c.memory.shape[1])
    spec, stop, align = O.decoder_forward(sd, hp, memory, mask, c.target.to(dtype), None, None, tape, training=c.training)
    return sd, memory, spec, stop, align


def _cuda_inputs(c, device, r=1):
    """Library config / parameters / memory of case `c`; at r frames per step (outputs_per_step_oracle.untie) its tape has one row per
    decoder step, S = ceil(T / r)."""
    from multilingual_text_to_speech_b200 import functional as F
    from multilingual_text_to_speech_b200 import _lib
    hp = c.hp
    kind = _lib.CELL_ZONEOUT if hp.decoder_regularization == 'zoneout' else _lib.CELL_DROPOUT
    rates = (hp.zoneout_hidden, hp.zoneout_cell) if kind == _lib.CELL_ZONEOUT else (hp.dropout_hidden, 0.0)
    S = -(-c.target.shape[2] // r)
    masks = {}
    for name in ('prenet0', 'prenet1'):
        if name in c.tape:          # tape layout [B, S+1, P] -> time-major [S, B, P] (row S is never consumed)
            masks[name] = c.tape[name][:, :S].transpose(0, 1).contiguous().to(torch.uint8).to(device)
    for name in ('att_h', 'att_c', 'gen_h', 'gen_c', 'step_prenet0', 'step_prenet1'):
        if name in c.tape:
            masks[name] = c.tape[name][:S].contiguous().to(torch.uint8).to(device)
    teacher = c.tape['teacher'][:S].numpy().astype(np.uint8)
    cfg = F.DecoderConfig(kind, c.training, rates[0], rates[1], hp.dropout, masks, None if teacher.all() else teacher, outputs_per_step=r)
    params = [c.sd[key].to(device).clone().requires_grad_(True) for _, key in PARAM_KEYS]
    memory = c.memory.to(device).clone().requires_grad_(True)
    return cfg, params, memory


def run_case_bf16(c, check_grads=True, verbose=False):
    """bf16 perf mode (tensor-core operands, fp32 state): gate = mel L1 < 1e-3 against the fp64 oracle (north_star)."""
    from multilingual_text_to_speech_b200 import functional as F, _lib
    device = torch.device('cuda:0')
    cfg, params, memory = _cuda_inputs(c, device)
    _lib.set_precision('bf16')
    try:
        spec, stop, align = F.decoder_forward(cfg, memory, c.target.to(device), c.lengths.to(device), params)
        torch.cuda.synchronize()
        with_grad = check_grads and bool(c.tape['teacher'].all())
        report = {}
        assert torch.isfinite(spec).all() and torch.isfinite(align).all()
        # (1) against the oracle with the SAME operand rounding (bf16 operands, wide accumulation): isolates kernel bugs from
        #     the trajectory divergence bf16 causes.  Its autograd (straight-through casts) is the gradient reference too.
        O.QUANT = O.bf16_round
        try:
            sd, mem_o, spec_q, stop_q, align_q = _oracle_run(c, torch.float64, with_grad)
        finally:
            O.QUANT = None
        for name, got, ref in (('spec', spec, spec_q), ('stop', stop, stop_q), ('align', align, align_q)):
            d = (got.detach().cpu().double() - ref.detach()).abs()
            report[name + '_q_l1'], report[name + '_q_max'] = float(d.mean()), float(d.max())
        scale = float(spec_q.detach().abs().mean())
        # residual = bf16 rounding decisions flipping on 1-ulp fp32 differences (measured 2e-4 .. 1.4e-3), not accumulation error
        assert report['spec_q_l1'] < 3e-3 * max(scale, 1.0), report
        assert report['align_q_l1'] < 5e-4, report
        # (2) against the exact fp64 oracle: the cost of bf16 operands (informational + loose relative bound)
        with torch.no_grad():
            _, _, spec_o, stop_o, align_o = _oracle_run(c, torch.float64, False)
        for name, got, ref in (('spec', spec, spec_o), ('stop', stop, stop_o), ('align', align, align_o)):
            d = (got.detach().cpu().double() - ref.detach()).abs()
            report[name + '_l1'], report[name + '_max'] = float(d.mean()), float(d.max())
        report['spec_rel_l1'] = report['spec_l1'] / float(spec_o.detach().abs().mean())
        assert report['spec_rel_l1'] < 2e-2, report
        agree = float((align.detach().cpu().argmax(2) == align_o.detach().argmax(2)).float().mean())
        report['argmax_agree'] = agree
        assert agree > 0.95, report
        if with_grad:
            g = torch.Generator().manual_seed(99)
            r_spec = torch.randn(spec_q.shape, generator=g, dtype=torch.float64)
            r_stop = torch.randn(stop_q.shape, generator=g, dtype=torch.float64)
            r_align = torch.randn(align_q.shape, generator=g, dtype=torch.float64)
            ((spec_q * r_spec).sum() + (stop_q * r_stop).sum() + (align_q * r_align).sum()).backward()
            ((spec * r_spec.float().to(device)).sum() + (stop * r_stop.float().to(device)).sum() +
             (align * r_align.float().to(device)).sum()).backward()
            torch.cuda.synchronize()
            pairs = [('memory', memory.grad, mem_o.grad)] + [(f, p.grad, sd[k].grad) for (f, k), p in zip(PARAM_KEYS, params)]
            for name, got, ref in pairs:
                got = got.detach().cpu().double()
                ref = ref if ref is not None else torch.zeros_like(got)
                rel = float((got - ref).norm() / (ref.norm() + 1e-12))
                cos = float((got * ref).sum() / (got.norm() * ref.norm() + 1e-30))
                report['d_' + name] = rel
                # relative L2 error against the gradient of the operand-quantised oracle (same bf16 operands, wide accumulation):
                # what remains is the kernels' own arithmetic (fp32 accumulation order, tanh.approx / ex2 gate math, bf16 rounding of the
                # gate GRADIENTS in the recurrent products).  Bounds: measured values (<= 2e-2 everywhere, attention parameters up to
                # ~4e-2 on the sharpened synthetic attention) with ~2x margin; a wrong block or a 30 % error fails.
                bound = GRAD_REL_BOUND_ATT if name.startswith('attn_') or name in ('memory',) else GRAD_REL_BOUND
                assert rel < bound and cos > 0.995, (c.name, name, rel, cos, bound)
    finally:
        _lib.set_precision('fp32')
    if verbose:
        print(c.name, '[bf16]', {k: f'{v:.2e}' for k, v in report.items()})
    return report


def run_case(c, check_grads=True, verbose=False, rtol=1e-3, atol=1e-4):
    """Run the CUDA decoder on `c`, compare with the fp64 oracle.  Returns a dict of max abs differences."""
    from multilingual_text_to_speech_b200 import functional as F
    device = torch.device('cuda:0')
    cfg, params, memory = _cuda_inputs(c, device)
    spec, stop, align = F.decoder_forward(cfg, memory, c.target.to(device), c.lengths.to(device), params)
    torch.cuda.synchronize()
    teacher_all = bool(c.tape['teacher'].all())
    with_grad = check_grads and teacher_all
    sd, mem_o, spec_o, stop_o, align_o = _oracle_run(c, torch.float64, with_grad)
    report = {}
    for name, got, ref in (('spec', spec, spec_o), ('stop', stop, stop_o), ('align', align, align_o)):
        report[name] = float((got.detach().cpu().double() - ref.detach()).abs().max())
        assert_close(got, ref, rtol, atol, f'{c.name}: {name}')
    # bit-exact discrete decisions
    assert torch.equal(align.detach().cpu().argmax(2), align_o.detach().argmax(2)), f'{c.name}: alignment argmax differs'
    margin = stop_o.detach().abs() > 1e-4
    assert torch.equal((stop.detach().cpu() > 0)[margin], (stop_o.detach() > 0)[margin]), f'{c.name}: stop sign differs'
    if with_grad:
        g = torch.Generator().manual_seed(99)
        r_spec = torch.randn(spec_o.shape, generator=g, dtype=torch.float64)
        r_stop = torch.randn(stop_o.shape, generator=g, dtype=torch.float64)
        r_align = torch.randn(align_o.shape, generator=g, dtype=torch.float64)
        loss_o = (spec_o * r_spec).sum() + (stop_o * r_stop).sum() + (align_o * r_align).sum()
        loss_o.backward()
        loss = (spec * r_spec.float().to(device)).sum() + (stop * r_stop.float().to(device)).sum() + \
               (align * r_align.float().to(device)).sum()
        loss.backward()
        torch.cuda.synchronize()
        pairs = [('memory', memory.grad, mem_o.grad)]
        for (field, key), p in zip(PARAM_KEYS, params):
            ref = sd[key].grad
            pairs.append((field, p.grad, ref if ref is not None else torch.zeros_like(sd[key])))
        for name, got, ref in pairs:
            scale = float(ref.abs().max()) + 1e-12
            report['d_' + name] = float((got.detach().cpu().double() - ref).abs().max()) / scale
            assert_close(got, ref, 2e-3, 2e-4 * scale, f'{c.name}: grad {name}')
    if verbose:
        print(c.name, {k: f'{v:.2e}' for k, v in report.items()})
    return report
