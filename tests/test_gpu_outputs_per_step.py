"""Several mel frames per decoder step (hp.outputs_per_step = r) on the H100: tied weights against the reference goldens, untied
decodes against the r-frames oracle (tests/outputs_per_step_oracle.py) in both precision modes, the guided loss on the step grid, the
graphed training step, synthesis and the training example."""
import ctypes
import os
import subprocess
import sys
import types

import numpy as np
import pytest
import torch

import decoder_cases as DC
import outputs_per_step_oracle as R
from helpers import assert_close
from oracle import tacotron_oracle as O

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope='module', autouse=True)
def _built():
    import __graft_entry__ as entry
    entry.build()
    assert torch.cuda.is_available(), 'GPU tests need a CUDA device'


def _cuda_inputs(c, r, dev):
    """Library config / parameters / memory of case `c` at r frames per step (its tape has one row per step)."""
    from multilingual_text_to_speech_b200 import functional as F, _lib
    hp = c.hp
    kind = _lib.CELL_ZONEOUT if hp.decoder_regularization == 'zoneout' else _lib.CELL_DROPOUT
    rates = (hp.zoneout_hidden, hp.zoneout_cell) if kind == _lib.CELL_ZONEOUT else (hp.dropout_hidden, 0.0)
    S = R.steps(c.target.shape[2], r)
    masks = {}
    for name in ('prenet0', 'prenet1'):
        if name in c.tape:
            masks[name] = c.tape[name][:, :S].transpose(0, 1).contiguous().to(torch.uint8).to(dev)
    for name in ('att_h', 'att_c', 'gen_h', 'gen_c', 'step_prenet0', 'step_prenet1'):
        if name in c.tape:
            masks[name] = c.tape[name][:S].contiguous().to(torch.uint8).to(dev)
    teacher = c.tape['teacher'][:S].numpy().astype(np.uint8)
    cfg = F.DecoderConfig(kind, c.training, rates[0], rates[1], hp.dropout, masks, None if teacher.all() else teacher, outputs_per_step=r)
    params = [None if key not in c.sd else c.sd[key].to(dev).clone().requires_grad_(True) for _, key in DC.PARAM_KEYS]
    memory = c.memory.to(dev).clone().requires_grad_(True)
    return cfg, params, memory


def _library(c, r, precision='fp32', upstream=None):
    """Decode `c` on the library at r; with `upstream` (d spec, d stop, d align on the host) also the backward.
    -> (spec, stop, align, {name: grad} or None)"""
    from multilingual_text_to_speech_b200 import functional as F, _lib
    dev = torch.device('cuda:0')
    cfg, params, memory = _cuda_inputs(c, r, dev)
    _lib.set_precision(precision)
    try:
        spec, stop, align = F.decoder_forward(cfg, memory, c.target.to(dev), c.lengths.to(dev), params)
        grads = None
        if upstream is not None:
            sum((t * u.float().to(dev)).sum() for t, u in zip((spec, stop, align), upstream)).backward()
            grads = {'memory': memory.grad.cpu()}
            grads.update({f: p.grad.cpu() for (f, _), p in zip(DC.PARAM_KEYS, params) if p is not None})
        torch.cuda.synchronize()
    finally:
        _lib.set_precision('fp32')
    return spec.detach().cpu(), stop.detach().cpu(), align.detach().cpu(), grads


PROJ_FIELDS = ('frame_w', 'frame_b', 'stop_w', 'stop_b')


# ---- 1. tied weights against the reference goldens ----

@pytest.mark.parametrize('name', ['lj_dropout', 'lj_zoneout', 'lj_mixed_tf', 'lj_eval_free', 'fwd_lj_dropout', 'fwd_lj_zoneout_tf05'])
def test_tied_r2_reproduces_the_golden_decode(name):
    r = 2
    c1, cr = DC.golden_case(name), DC.golden_case(name)
    cr.sd = R.tie(cr.sd, r)
    cr.target = R.repeat_frames(cr.target, r, 2)
    gold = c1.golden
    B, N, T = c1.target.shape
    tmask = O.lengths_to_mask(gold.inputs['target_length'], T)
    g = torch.Generator().manual_seed(7)
    up_r = [torch.randn(B, T * r, N, generator=g), torch.randn(B, T * r, generator=g), torch.randn(B, T, gold.L, generator=g)]
    up_1 = [up_r[0].reshape(B, T, r, N).sum(2), up_r[1].reshape(B, T, r).sum(2), up_r[2]]
    train = c1.training
    spec, stop, align, grads = _library(cr, r, upstream=up_r if train else None)
    assert spec.shape == (B, T * r, N) and align.shape == (B, T, gold.L)
    # every frame of the golden decode, r times (the golden pre / stop are masked past each target length)
    for j in range(r):
        sj, tj = spec[:, j::r], stop[:, j::r]
        assert_close(sj.transpose(1, 2) * tmask[:, None, :], gold.out['pre'], 1e-3, 1e-4, f'{name}: frames of slot {j}')
        assert_close(tj[tmask], gold.out['stop'][tmask], 1e-3, 1e-4, f'{name}: stop logits of slot {j}')
        assert torch.equal(tj[tmask] > 0, gold.out['stop'][tmask] > 0), f'{name}: stop decision of slot {j}'
    assert_close(align, gold.out['align'], 1e-3, 1e-4, f'{name}: alignment')
    assert torch.equal(align.argmax(2), gold.out['align'].argmax(2)), f'{name}: alignment argmax'
    spec1, stop1, align1, grads1 = _library(c1, 1, upstream=up_1 if train else None)
    if train:
        for f, g1 in grads1.items():
            got = R.block_sum(grads[f], r) if f in PROJ_FIELDS else grads[f]
            scale = float(g1.abs().max()) + 1e-12
            assert_close(got, g1, 2e-3, 2e-4 * scale, f'{name}: grad {f}')
    if bool(c1.tape['teacher'].all()):
        # teacher-forced: the recurrences see bit-identical operands at r = 2 and r = 1, in both precision modes
        assert torch.equal(align, align1), name
        assert torch.equal(_library(cr, r, 'bf16')[2], _library(c1, 1, 'bf16')[2]), name


# ---- 2. untied decodes against the r-frames oracle ----

def _untied(r, att, kind, tf, S=7, B=4, L=24, seed=0, **kw):
    c = DC.full_dim_case(B=B, L=L, T=S, kind=kind, seed=seed, tf=tf, **kw)
    if att == 'forward':
        c.hp.attention_type = 'forward'
        for k in [k for k in c.sd if k.endswith('_location.weight') or k.endswith('_loc_features.weight')]:
            c.sd.pop(k)
    return R.untie(c, r, S * r - 1, seed)        # T not a multiple of r: the last step's last frame is dropped


@pytest.mark.parametrize('tf', [1.0, 0.5])
@pytest.mark.parametrize('kind', ['dropout', 'zoneout'])
@pytest.mark.parametrize('att', ['location_sensitive', 'forward'])
@pytest.mark.parametrize('r', [2, 3])
def test_untied_fp32_matches_the_oracle(r, att, kind, tf):
    c = _untied(r, att, kind, tf)
    sd, mem_o, spec_o, stop_o, align_o = R.run(c, r)
    g = torch.Generator().manual_seed(99)
    up = [torch.randn(t.shape, generator=g, dtype=torch.float64) for t in (spec_o, stop_o, align_o)]
    spec, stop, align, grads = _library(c, r, upstream=up)
    assert spec.shape == spec_o.shape and align.shape == align_o.shape
    for what, got, ref in (('spec', spec, spec_o), ('stop', stop, stop_o), ('align', align, align_o)):
        assert_close(got, ref.detach(), 1e-3, 1e-4, f'{c.name}: {what}')
    assert torch.equal(align.argmax(2), align_o.detach().argmax(2)), f'{c.name}: alignment argmax'
    margin = stop_o.detach().abs() > 1e-4
    assert torch.equal((stop > 0)[margin], (stop_o.detach() > 0)[margin]), f'{c.name}: stop sign'
    sum((t * u).sum() for t, u in zip((spec_o, stop_o, align_o), up)).backward()
    refs = {'memory': mem_o.grad}
    refs.update({f: sd[k].grad for f, k in DC.PARAM_KEYS if k in sd})
    for f, got in grads.items():
        ref = refs[f] if refs[f] is not None else torch.zeros_like(got, dtype=torch.float64)
        scale = float(ref.abs().max()) + 1e-12
        assert_close(got, ref, 2e-3, 2e-4 * scale, f'{c.name}: grad {f}')


def _path(c, r):
    from multilingual_text_to_speech_b200 import _lib
    B, L, M = c.memory.shape
    kind = _lib.CELL_ZONEOUT if c.hp.decoder_regularization == 'zoneout' else _lib.CELL_DROPOUT
    s = _lib.DecoderShape(B, L, c.target.shape[2], M, c.hp.decoder_dimension, c.hp.prenet_dimension, 128, 32, 31, c.hp.num_mels, kind, 1,
                          0.1, 0.1, 0.5)
    s.R = r
    return _lib.load().b200tts_decoder_path(ctypes.byref(s))


@pytest.mark.parametrize('kind', ['dropout', 'zoneout'])
def test_untied_bf16_on_the_persistent_loops(kind):
    """bf16 perf mode at r = 2 on a shape whose S = 30 steps run the persistent loops, against the operand-quantised oracle."""
    r = 2
    c = _untied(r, 'location_sensitive', kind, 1.0, S=30, B=8, L=40)
    assert _path(c, r) == 0b111111
    O.QUANT = O.bf16_round
    try:
        sd, mem_o, spec_q, stop_q, align_q = R.run(c, r)
    finally:
        O.QUANT = None
    g = torch.Generator().manual_seed(99)
    up = [torch.randn(t.shape, generator=g, dtype=torch.float64) for t in (spec_q, stop_q, align_q)]
    spec, stop, align, grads = _library(c, r, 'bf16', upstream=up)
    scale = float(spec_q.detach().abs().mean())
    spec_l1 = float((spec.double() - spec_q.detach()).abs().mean())
    align_l1 = float((align.double() - align_q.detach()).abs().mean())
    assert spec_l1 < 3e-3 * max(scale, 1.0), spec_l1
    assert align_l1 < 5e-4, align_l1
    sum((t * u).sum() for t, u in zip((spec_q, stop_q, align_q), up)).backward()
    refs = {'memory': mem_o.grad}
    refs.update({f: sd[k].grad for f, k in DC.PARAM_KEYS if k in sd})
    for f, got in grads.items():
        got, ref = got.double(), refs[f]
        rel = float((got - ref).norm() / (ref.norm() + 1e-12))
        cos = float((got * ref).sum() / (got.norm() * ref.norm() + 1e-30))
        bound = DC.GRAD_REL_BOUND_ATT if f.startswith('attn_') or f == 'memory' else DC.GRAD_REL_BOUND
        assert rel < bound and cos > 0.995, (f, rel, cos)


# ---- 4. the guided-attention loss on the step grid ----

def test_loss_r2_guided_on_the_step_grid():
    from multilingual_text_to_speech_b200 import functional as F
    r, B, N, T, L = 2, 4, 80, 37, 20
    S = R.steps(T, r)
    g = torch.Generator().manual_seed(3)
    pre, post, tgt = (torch.randn(B, N, T, generator=g) for _ in range(3))
    stop, stop_t = torch.randn(B, T, generator=g), (torch.rand(B, T, generator=g) > 0.8).float()
    align = torch.softmax(torch.randn(B, S, L, generator=g), 2)
    tlen, mlen = torch.tensor([20, 17, 13, 6]), torch.tensor([37, 30, 25, 11])
    hp = types.SimpleNamespace(num_mels=N, reversal_classifier=False, guided_attention_loss=True)
    a_o = align.double().requires_grad_(True)
    _, parts = O.tacotron_loss(hp, 0.2, tlen, mlen, pre.double(), tgt.double(), post.double(), tgt.double(), stop.double(), stop_t.double(),
                               None, guided=False)
    guided = R.guided_attention_loss(a_o, tlen, mlen, 0.2, r)
    guided.backward()
    dev = torch.device('cuda:0')
    a_c = align.to(dev).requires_grad_(True)
    terms = F.tacotron_loss(pre.to(dev), post.to(dev), stop.to(dev), a_c, tgt.to(dev), tgt.to(dev), stop_t.to(dev), tlen.to(dev),
                            mlen.to(dev), True, 0.2, 100.0, outputs_per_step=r)
    terms[3].backward()
    got = terms.detach().cpu().double()
    for k, (name, want) in enumerate((('mel_pre', parts['mel_pre']), ('mel_pos', parts['mel_pos']), ('stop_token', parts['stop_token']),
                                       ('guided_att', guided))):
        assert abs(float(got[k]) - float(want.detach())) < 1e-5 * max(1.0, abs(float(want))), (name, float(got[k]), float(want))
    assert_close(a_c.grad, a_o.grad, 1e-4, 1e-8, 'd alignment')


# ---- 5. graph, synthesis, training ----

def test_graphed_train_step_r2_equals_eager():
    import model_cases
    from helpers import Golden
    from multilingual_text_to_speech_b200.distributed import GradBucket
    from multilingual_text_to_speech_b200.graph import GraphedTrainStep
    from multilingual_text_to_speech_b200.modules.tacotron2 import Tacotron, TacotronLoss
    from multilingual_text_to_speech_b200.rng import MaskSource
    from multilingual_text_to_speech_b200.params.params import Params as hp
    r = 2
    gld = Golden('generated_training')
    dev = torch.device('cuda:0')
    model_cases.configure_hp(gld)
    hp.outputs_per_step = r
    try:
        torch.manual_seed(0)
        model = Tacotron().to(dev).train()
        bucket = GradBucket(model, 1)
        crit = TacotronLoss(hp.guided_attention_steps, gld.meta['guided_g'], hp.guided_attention_gain)
        batch = {k: v.to(dev) for k, v in gld.inputs.items()}
        batch.setdefault('speakers', None); batch.setdefault('languages', None)
        S = R.steps(batch['target'].shape[2], r)
        step_rows = {'teacher', 'att_h', 'att_c', 'gen_h', 'gen_c', 'step_prenet0', 'step_prenet1'}
        tape = {}
        for k, v in gld.tape.items():
            if k in ('prenet0', 'prenet1'):
                v = v[:, :S + 1].contiguous()
            elif k in step_rows:
                v = v[:S].contiguous()
            tape[k] = v if k == 'teacher' else v.to(dev)
        MaskSource.use_tape(tape)
        step = None
        try:
            step = GraphedTrainStep(model, crit, bucket, batch, teacher_forcing=1.0, warmup=2)
            got = []
            for _ in range(2):
                loss_g = step(batch)
                torch.cuda.synchronize()
                got.append((float(loss_g), bucket.flat.clone()))
            step.close(); step = None
            bucket.zero()
            post, pre, stop, align, spk, enc = model(batch['text'], batch['text_length'], batch['target'], batch['target_length'],
                                                     batch['speakers'], batch['languages'], 1.0)
            assert align.shape[1] == S
            loss, _ = crit(batch['text_length'], batch['target_length'], pre, batch['target'], post, batch['target'], stop,
                           batch['stop_target'], align, batch['speakers'], spk, enc, None)
            loss.backward()
            want_loss, want_grad = float(loss), bucket.flat.clone()
            for got_loss, got_grad in got:
                assert abs(got_loss - want_loss) < 1e-6 * max(1.0, abs(want_loss))
                assert torch.allclose(got_grad, want_grad, rtol=1e-5, atol=1e-8)
        finally:
            MaskSource.use_tape(None)
            if step is not None:
                step.close()
    finally:
        hp.reset()


def _synthesis_model(r, dev):
    from multilingual_text_to_speech_b200.modules.tacotron2 import Tacotron
    from multilingual_text_to_speech_b200.params.params import Params as hp
    hp.reset()
    hp.outputs_per_step = r
    hp.max_output_length = 60
    torch.manual_seed(0)
    model = Tacotron().to(dev).eval()
    with torch.no_grad():       # the stop token fires on the first frame of every step only: the cut (the 6th firing frame) is mid-step
        model._decoder._stop_prediction.weight.zero_()
        model._decoder._stop_prediction.bias.fill_(-100.0)
        model._decoder._stop_prediction.bias[0] = 100.0
    return model, types.SimpleNamespace(**hp.state_dict())


def test_inference_r2_matches_the_oracle_cut_included():
    from multilingual_text_to_speech_b200.rng import MaskSource
    from multilingual_text_to_speech_b200.params.params import Params as hp
    r, L, dev = 2, 17, torch.device('cuda:0')
    try:
        model, ohp = _synthesis_model(r, dev)
        g = torch.Generator().manual_seed(4)
        S = R.steps(ohp.max_output_length, r)
        P = ohp.prenet_dimension
        tape = {k: (torch.rand(S, 1, P, generator=g) >= 0.5).float() for k in ('step_prenet0', 'step_prenet1')}
        encoded = torch.randn(1, L, ohp.encoder_dimension, generator=g)
        mask = O.lengths_to_mask(torch.tensor([L]), L)
        MaskSource.use_tape({k: v.to(dev) for k, v in tape.items()})
        try:
            spec, stop, align, cuts = model._decoder._decode_inference(encoded.to(dev), mask.to(dev), None, None)
        finally:
            MaskSource.use_tape(None)
        sd = {k: v.detach().cpu().double() for k, v in model.state_dict().items() if v.is_floating_point()}
        DC._decoder_sd_alias(sd)
        spec_o, stop_o, align_o = R.decoder_forward(sd, ohp, encoded.double(), mask, None, None, None,
                                                    {k: v.double() for k, v in tape.items()}, training=False)
        assert cuts[0] == spec_o.shape[1] == r * ohp.stop_frames + 1, (cuts, spec_o.shape)
        assert align.shape[1] == align_o.shape[1] == R.steps(cuts[0], r)
        assert_close(spec.cpu(), spec_o, 1e-3, 1e-4, 'inference spectrogram')
        assert_close(align.cpu(), align_o, 1e-3, 1e-4, 'inference alignment')
    finally:
        hp.reset()


def test_inference_batch_r2_equals_single_utterances():
    from multilingual_text_to_speech_b200.rng import MaskSource
    from multilingual_text_to_speech_b200.params.params import Params as hp
    r, dev = 2, torch.device('cuda:0')
    try:
        model, ohp = _synthesis_model(r, dev)
        g = torch.Generator().manual_seed(6)
        texts = [torch.randint(1, hp.symbols_count() + 3, (n,), generator=g) for n in (23, 9, 17, 30, 12)]
        S = R.steps(ohp.max_output_length, r)
        tape = {k: (torch.rand(S, len(texts), ohp.prenet_dimension, generator=g) >= 0.5).to(dev) for k in ('step_prenet0', 'step_prenet1')}
        MaskSource.use_tape(tape)
        try:
            batched = model.inference_batch(texts)
        finally:
            MaskSource.use_tape(None)
        for i, t in enumerate(texts):
            MaskSource.use_tape({k: v[:, i:i + 1] for k, v in tape.items()})
            try:
                single = model.inference(t)
            finally:
                MaskSource.use_tape(None)
            assert torch.equal(batched[i], single), (i, batched[i].shape, single.shape)
    finally:
        hp.reset()


def test_training_example_runs_at_r2():
    env = dict(os.environ, PYTHONPATH=ROOT)
    res = subprocess.run([sys.executable, os.path.join(ROOT, 'examples', 'train_synthetic.py'), '--steps', '5', '--batch', '10',
                          '--outputs-per-step', '2'], cwd=ROOT, env=env, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True,
                         timeout=900)
    assert res.returncode == 0, res.stdout[-4000:]
    losses = [float(line.split('loss')[1].split()[0]) for line in res.stdout.splitlines() if line.startswith('step ')]
    assert losses and all(np.isfinite(losses)), res.stdout[-2000:]
