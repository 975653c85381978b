""""train.py calls into it unchanged" (north_star, SURVEY 8b): the reference's training procedure (train.py:29-95: model.train,
zero_grad, forward, TacotronLoss, adversarial classifier accuracy, backward, clip_grad_norm_, Adam step, criterion.update_states)
driving THIS package for two optimisation steps, against the golden record of the UNMODIFIED reference's own `train()` on its own
modules (tests/golden/make_golden_train.py -> tests/golden/reference_train.npz; case definition in tests/train_case.py).  Each step
replays the dropout masks the reference drew at that step.
Checks, for both steps: the seeded weights are the reference's; the loss terms, gradient norm and classifier accuracy match what the
reference logged; every parameter's gradient matches the reference's; every parameter's change over the two Adam updates matches;
and update_states ran once per step.
"""
import pytest
import torch

import train_case as TC
from helpers import assert_close

pytestmark = pytest.mark.gpu


@pytest.fixture(scope='module', autouse=True)
def _built():
    import __graft_entry__ as entry
    entry.build()
    assert torch.cuda.is_available()


def _train(hp, data, tapes, model, criterion, optimizer):
    """train.py:29-95 on this package, step s replaying tapes[s]; returns what the reference's Logger.training receives
    (losses, gradient norm, accuracy) and each step's gradients before clipping, in sorted parameter-name order."""
    from multilingual_text_to_speech_b200.rng import MaskSource
    from multilingual_text_to_speech_b200.utils import lengths_to_mask, to_gpu
    logged, grads = [], []
    named = sorted(model.named_parameters())
    model.train()
    for batch, tape in zip(data, tapes):
        optimizer.zero_grad()
        src, src_len, trg_mel, trg_lin, trg_len, stop_trg, spkrs, langs = map(to_gpu, batch)
        MaskSource.use_tape(tape)
        try:
            post_pred, pre_pred, stop_pred, alignment, spkrs_pred, enc_output = model(src, src_len, trg_mel, trg_len, spkrs, langs,
                                                                                      hp.teacher_forcing)
        finally:
            MaskSource.use_tape(None)
        classifier = model._reversal_classifier if hp.reversal_classifier else None
        loss, batch_losses = criterion(src_len, trg_len, pre_pred, trg_mel, post_pred, trg_mel, stop_pred, stop_trg, alignment,
                                       spkrs, spkrs_pred, enc_output, classifier)
        cla = 0.0
        if hp.reversal_classifier:
            input_mask = lengths_to_mask(src_len)
            trg_spkrs = torch.zeros_like(input_mask, dtype=torch.int64)
            for s in range(hp.speaker_number):
                trg_spkrs[spkrs == s] = s
            matches = trg_spkrs == torch.argmax(torch.softmax(spkrs_pred, dim=-1), dim=-1)
            matches[~input_mask] = False
            cla = matches.sum().item() / input_mask.sum().item()
        loss.backward()
        grads.append({n: p.grad.detach().double().cpu() for n, p in named})
        gradient = torch.nn.utils.clip_grad_norm_(model.parameters(), hp.gradient_clipping)
        optimizer.step()
        logged.append(({k: float(v) for k, v in batch_losses.items()}, float(gradient), cla))
        criterion.update_states()
    return logged, grads


# fp32 parity mode against the reference's CPU fp32.  Largest deviations measured on an H100 80GB HBM3 (700 W), over both configs,
# step 0 / step 1: loss terms 1.3e-7 / 2.2e-7 relative, gradient norm 3.0e-7 / 1.4e-7 relative, gradients 2.0e-5 / 9.0e-5 of their
# tensor's max (abs), conditioned updates 9.8e-7 absolute.  Step 1 came out no worse than step 0, so both steps share the bounds.
LOSS_RTOL = (5e-7, 5e-7)
NORM_RTOL = (6e-7, 6e-7)
GRAD_TOL = ((3e-3, 3e-4), (3e-3, 3e-4))        # (rtol, atol as a fraction of the reference tensor's max), as model_cases.run_golden
UPDATE_ATOL = 2e-6


@pytest.mark.parametrize('config', TC.CONFIGS)
def test_reference_train_function_runs_on_this_package(config):
    from multilingual_text_to_speech_b200 import configs, _lib
    from multilingual_text_to_speech_b200.modules.tacotron2 import Tacotron, TacotronLoss
    fx = TC.Fixture(config)
    hp = configs.apply(config, speakers=TC.SPEAKERS, **TC.overrides(config))
    torch.manual_seed(0)
    model = Tacotron()
    assert torch.equal(TC.param_sums(model), torch.from_numpy(fx.param_sums)), 'seeded weights differ from the reference'
    assert [n for n, _ in sorted(model.named_parameters())] == fx.names
    model = model.cuda()
    optimizer = torch.optim.Adam(model.parameters(), lr=hp.learning_rate, weight_decay=hp.weight_decay)
    criterion = TacotronLoss(hp.guided_attention_steps, hp.guided_attention_toleration, hp.guided_attention_gain)
    batch = TC.make_batch(hp)
    before = {n: p.detach().double().cpu() for n, p in sorted(model.named_parameters())}
    g_before = criterion._g
    previous = _lib.get_precision()
    _lib.set_precision('fp32')                # the reference arithmetic: the fp32 parity mode
    try:
        logged, grads = _train(hp, [batch, batch], [fx.tape(0), fx.tape(1)], model, criterion, optimizer)
    finally:
        _lib.set_precision(previous)
    assert len(logged) == 2
    bad, report = [], {}
    for step, (losses, grad, cla) in enumerate(logged):
        assert sorted(losses) == fx.loss_keys, (sorted(losses), fx.loss_keys)
        for k, r in zip(fx.loss_keys, fx.losses[step]):
            report[f'{step} {k}'] = abs(losses[k] - r) / abs(r)
            if not abs(losses[k] - r) <= LOSS_RTOL[step] * abs(r):
                bad.append(f'step {step} {k}: {losses[k]} vs reference {r}')
        rg = float(fx.gradient[step])
        report[f'{step} norm'] = abs(grad - rg) / rg
        if not abs(grad - rg) <= NORM_RTOL[step] * rg:
            bad.append(f'step {step} gradient norm: {grad} vs reference {rg}')
        if cla != float(fx.classifier[step]):        # the same masks: the same count of matching positions
            bad.append(f'step {step} classifier accuracy: {cla} vs reference {float(fx.classifier[step])}')
        ref = fx.grad(step)
        rtol, atol = GRAD_TOL[step]
        for n in fx.names:
            scale = float(ref[n].abs().max()) + 1e-12
            report[f'{step} d{n}'] = float((grads[step][n] - ref[n]).abs().max()) / scale
            try:
                assert_close(grads[step][n], ref[n], rtol, atol * scale + 1e-12, f'step {step} grad {n}')
            except AssertionError as exc:
                bad.append(str(exc))
    after = {n: p.detach().double().cpu() for n, p in sorted(model.named_parameters())}
    ref, cond = fx.update(), fx.conditioned()
    for n in fx.names:
        got = after[n] - before[n]
        report[f'update {n}'] = float((got - ref[n])[cond[n]].abs().max()) if bool(cond[n].any()) else 0.0
        assert not torch.equal(after[n], before[n]), f'{n} was not updated'
        try:
            assert_close(got[cond[n]], ref[n][cond[n]], 0.0, UPDATE_ATOL, f'update {n}')
        except AssertionError as exc:
            bad.append(str(exc))
    for step in '01':
        losses = [v for k, v in report.items() if k.startswith(step) and k[2:] in fx.loss_keys]
        grads = max((kv for kv in report.items() if kv[0].startswith(step + ' d')), key=lambda kv: kv[1])
        print(config, f'step {step}: loss terms {max(losses):.2e}, norm {report[step + " norm"]:.2e}, worst gradient {grads}')
    print(config, 'worst update', max((kv for kv in report.items() if kv[0].startswith('update')), key=lambda kv: kv[1]))
    assert not bad, '; '.join(bad[:12])
    assert logged[0][0]['mel_pre'] != logged[1][0]['mel_pre']                   # the optimiser step changed the model
    assert criterion._g == g_before * hp.guided_attention_gain ** 2          # update_states ran once per step
