"""Forward attention (hp.attention_type = "forward", reference modules/attention.py:89-124) on the GPU: the module step, the fused
decoder forward / backward (per-step forward-attention kernels) against the reference goldens and the oracle, bf16 mode, chunked
inference, the whole model with its loss, and run-to-run reproducibility."""
import json
import os

import numpy as np
import pytest
import torch

import decoder_cases as DC
import forward_attention_oracle as FA
import model_cases
import module_cases as C
from helpers import GOLDEN_DIR, assert_close
from oracle import tacotron_oracle as O

pytestmark = pytest.mark.gpu

LOCATION_FIELDS = ('attn_location', 'attn_loc_features')


@pytest.fixture(scope='module', autouse=True)
def _built():
    import __graft_entry__ as entry
    entry.build()
    assert torch.cuda.is_available()


def test_module_step_forward_and_autograd_match_reference():
    """ForwardAttention.reset + three forward steps with gradients through the carried alpha, against the reference module."""
    from multilingual_text_to_speech_b200.modules.attention import ForwardAttention
    stored = np.load(os.path.join(GOLDEN_DIR, 'fwd_attention_module.npz'))
    d = C.ATT_DIMS
    res = C.attention_case(ForwardAttention(d['A'], d['D'], d['M']), 'cuda')
    for key, t in res.items():
        got, ref, absmax = C.unpack_like(stored, 'forward_attention', key, t)
        if key.startswith('weights'):
            rtol, atol = 1e-3, 1e-7
        elif key.startswith('context'):
            rtol, atol = 1e-3, 1e-5
        else:
            rtol, atol = 3e-3, 2e-4 * absmax
        assert_close(got, ref, rtol, atol, key)


def _strip_location(c):
    for k in [k for k in c.sd if '_location.' in k or '_loc_features.' in k]:
        del c.sd[k]
    c.hp.attention_type = 'forward'
    return c


def _cuda_run(c, device, seed=99):
    """The fused decoder on case `c` (forward attention: None location weights); returns outputs and, when every step is teacher
    forced, the gradients of <outputs, r> for seeded r."""
    from multilingual_text_to_speech_b200 import functional as F
    from multilingual_text_to_speech_b200 import _lib
    hp = c.hp
    kind = _lib.CELL_ZONEOUT if hp.decoder_regularization == 'zoneout' else _lib.CELL_DROPOUT
    rates = (hp.zoneout_hidden, hp.zoneout_cell) if kind == _lib.CELL_ZONEOUT else (hp.dropout_hidden, 0.0)
    T = c.target.shape[2]
    masks = {}
    for name in ('prenet0', 'prenet1'):
        if name in c.tape:
            masks[name] = c.tape[name][:, :T].transpose(0, 1).contiguous().to(torch.uint8).to(device)
    for name in ('att_h', 'att_c', 'gen_h', 'gen_c', 'step_prenet0', 'step_prenet1'):
        if name in c.tape:
            masks[name] = c.tape[name].contiguous().to(torch.uint8).to(device)
    teacher = c.tape['teacher'].numpy().astype(np.uint8)
    cfg = F.DecoderConfig(kind, c.training, rates[0], rates[1], hp.dropout, masks, None if teacher.all() else teacher)
    params = [None if f in LOCATION_FIELDS else c.sd[k].to(device).clone().requires_grad_(True) for f, k in DC.PARAM_KEYS]
    memory = c.memory.to(device).clone().requires_grad_(True)
    spec, stop, align = F.decoder_forward(cfg, memory, c.target.to(device), c.lengths.to(device), params)
    grads = None
    if bool(c.tape['teacher'].all()):
        g = torch.Generator().manual_seed(seed)
        rs = [torch.randn(t.shape, generator=g, dtype=torch.float64) for t in (spec, stop, align)]
        sum((t * r.float().to(device)).sum() for t, r in zip((spec, stop, align), rs)).backward()
        grads = [('memory', memory.grad)] + [(f, p.grad) for (f, _), p in zip(DC.PARAM_KEYS, params) if p is not None]
    torch.cuda.synchronize()
    return spec, stop, align, grads


def _oracle(c, dtype, with_grad, seed=99):
    with FA.forward_attention():
        sd, mem_o, spec, stop, align = DC._oracle_run(c, dtype, with_grad)
    if with_grad:
        g = torch.Generator().manual_seed(seed)
        rs = [torch.randn(t.shape, generator=g, dtype=torch.float64) for t in (spec, stop, align)]
        sum((t * r.to(dtype)).sum() for t, r in zip((spec, stop, align), rs)).backward()
    return sd, mem_o, spec, stop, align


def _check_fp32(c, rtol=1e-3, atol=1e-4, grad_rtol=2e-3, grad_atol=2e-4):
    dev = torch.device('cuda:0')
    spec, stop, align, grads = _cuda_run(c, dev)
    sd, mem_o, spec_o, stop_o, align_o = _oracle(c, torch.float64, grads is not None)
    for name, got, ref in (('spec', spec, spec_o), ('stop', stop, stop_o), ('align', align, align_o)):
        assert_close(got, ref, rtol, atol, f'{c.name}: {name}')
    assert torch.equal(align.detach().cpu().argmax(2), align_o.detach().argmax(2)), f'{c.name}: alignment argmax differs'
    margin = stop_o.detach().abs() > 1e-4
    assert torch.equal((stop.detach().cpu() > 0)[margin], (stop_o.detach() > 0)[margin]), f'{c.name}: stop sign differs'
    rows = align.detach().sum(2)
    assert float((rows - 1).abs().max()) < 1e-5, 'alignment rows must sum to one'
    if grads is not None:
        keys = dict(DC.PARAM_KEYS)
        for name, got in grads:
            ref = mem_o.grad if name == 'memory' else sd[keys[name]].grad
            ref = torch.zeros_like(got.cpu().double()) if ref is None else ref
            scale = float(ref.abs().max()) + 1e-12
            assert_close(got, ref, grad_rtol, grad_atol * scale, f'{c.name}: grad {name}')


@pytest.mark.parametrize('name', ['fwd_lj_dropout', 'fwd_lj_zoneout_tf05', 'fwd_lj_eval_free', 'fwd_generated_ragged'])
def test_fused_decoder_matches_golden_cases(name):
    """Forward on every golden; backward where every step is teacher forced (the fused backward covers teacher-forced decodes)."""
    _check_fp32(DC.golden_case(name))


@pytest.mark.parametrize('kind', ['dropout', 'zoneout'])
def test_fused_decoder_real_dimensions(kind):
    """D = 1024, A = 128, M = 288, L = 180, ragged lengths, T = 200: forward and backward against the fp64 oracle.  Over 200 steps of
    the multiplicative alpha recurrence the fp32 rounding of the kernels drifts by up to ~5e-4 absolute in the frames (measured on the
    dropout case), so the absolute tolerances are 1e-3 here; the discrete decisions stay exact."""
    c = _strip_location(DC.full_dim_case(B=4, L=180, T=200, kind=kind, seed=5))
    _check_fp32(c, atol=1e-3, grad_rtol=5e-3, grad_atol=1e-3)


def test_fused_decoder_bf16_mode_against_quantised_oracle():
    """bf16 GEMM operands on the per-step chains.  Bounds: mean |spec - oracle with bf16 operands| below 3e-3 of the spectrogram
    scale, alignments within 5e-4 mean absolute, alignment argmax agreement above 95 % with the exact fp64 oracle, and gradients
    within 8e-2 relative L2 of the operand-quantised oracle's with cosine similarity above 0.995."""
    from multilingual_text_to_speech_b200 import _lib
    c = _strip_location(DC.full_dim_case(B=4, L=180, T=120, kind='dropout', seed=6))
    dev = torch.device('cuda:0')
    _lib.set_precision('bf16')
    try:
        spec, stop, align, grads = _cuda_run(c, dev)
    finally:
        _lib.set_precision('fp32')
    O.QUANT = O.bf16_round
    try:
        sd, mem_o, spec_q, stop_q, align_q = _oracle(c, torch.float64, True)
    finally:
        O.QUANT = None
    scale = float(spec_q.detach().abs().mean())
    spec_l1 = float((spec.detach().cpu().double() - spec_q.detach()).abs().mean())
    align_l1 = float((align.detach().cpu().double() - align_q.detach()).abs().mean())
    assert spec_l1 < 3e-3 * max(scale, 1.0), (spec_l1, scale)
    assert align_l1 < 5e-4, align_l1
    with torch.no_grad():
        align_o = _oracle(c, torch.float64, False)[4]
    agree = float((align.detach().cpu().argmax(2) == align_o.argmax(2)).float().mean())
    assert agree > 0.95, agree
    keys = dict(DC.PARAM_KEYS)
    for name, got in grads:
        ref = mem_o.grad if name == 'memory' else sd[keys[name]].grad
        got = got.detach().cpu().double()
        rel = float((got - ref).norm() / (ref.norm() + 1e-12))
        cos = float((got * ref).sum() / (got.norm() * ref.norm() + 1e-30))
        assert rel < 8e-2 and cos > 0.995, (name, rel, cos)


def test_fused_decoder_is_bit_reproducible():
    c = _strip_location(DC.full_dim_case(B=4, L=60, T=40, kind='zoneout', seed=7))
    dev = torch.device('cuda:0')
    a = _cuda_run(c, dev)
    b = _cuda_run(c, dev)
    for x, y in zip(a[:3], b[:3]):
        assert torch.equal(x, y)
    for (n, x), (_, y) in zip(a[3], b[3]):
        assert torch.equal(x, y), n


@pytest.mark.parametrize('chunk', [4, 128])
def test_chunked_inference_matches_reference(chunk):
    """Tacotron.inference with forward attention: the carried alpha crosses chunk boundaries (chunk 4 splits the decode)."""
    from multilingual_text_to_speech_b200.params.params import Params as hp
    from multilingual_text_to_speech_b200.modules.tacotron2 import Tacotron, Decoder
    from multilingual_text_to_speech_b200.rng import MaskSource
    z = np.load(os.path.join(GOLDEN_DIR, 'fwd_inf_lj.npz'))
    meta = json.loads(bytes(z['meta']).decode())
    sd = {k[3:]: torch.from_numpy(z[k]) for k in z.files if k.startswith('sd.')}
    tape = {k[5:]: torch.from_numpy(z[k]) for k in z.files if k.startswith('tape.')}
    hp.reset()
    hp.load_state_dict(meta['hp'])
    model = Tacotron()
    model.load_state_dict(sd, strict=True)
    dev = torch.device('cuda:0')
    model = model.to(dev).eval()
    old_chunk = Decoder.inference_chunk
    Decoder.inference_chunk = chunk
    MaskSource.use_tape(tape)
    try:
        out = model.inference(torch.from_numpy(z['in.text']).to(dev), speaker=None, language=None)
    finally:
        MaskSource.use_tape(None)
        Decoder.inference_chunk = old_chunk
    ref = torch.from_numpy(z['out.post'])
    assert tuple(out.shape) == tuple(ref.shape) == (hp.num_mels, meta['T'])
    assert_close(out, ref, 1e-3, 1e-4, 'fwd_inf_lj: inference spectrogram')


@pytest.mark.parametrize('name', ['fwd_lj_dropout', 'fwd_lj_eval_free', 'fwd_generated_ragged'])
def test_whole_model_forward_loss_backward_match_reference(name):
    """Tacotron.forward + TacotronLoss (guided-attention term on) + backward against the reference, strict checkpoint load."""
    from multilingual_text_to_speech_b200.params.params import Params as hp
    model_cases.run_golden(name)
    assert hp.attention_type == 'forward' and hp.guided_attention_loss
