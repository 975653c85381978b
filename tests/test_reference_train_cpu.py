"""Pin the training-loop golden (tests/golden/reference_train.npz, tests/train_case.py) on the CPU, before any kernel is judged against
it: step 0 of the reference's train() replayed through the fp64 oracle with the recorded dropout tape reproduces the logged loss terms,
the gradient norm and every parameter gradient, and Adam applied in fp64 to the recorded gradients reproduces the recorded updates.
A golden that drew randomness it did not record fails here.
"""
import pytest
import torch

import train_case as TC
from helpers import assert_close
from oracle import tacotron_oracle as O


def _seeded(config):
    from multilingual_text_to_speech_b200 import configs
    from multilingual_text_to_speech_b200.modules.tacotron2 import Tacotron
    hp = configs.apply(config, speakers=TC.SPEAKERS, **TC.overrides(config))
    torch.manual_seed(0)
    model = Tacotron()
    return hp, model


def oracle_step0(config, fx, tape):
    """Step 0 through the fp64 oracle: (loss terms, {name: gradient}, gradient norm)."""
    from multilingual_text_to_speech_b200 import configs
    hp, model = _seeded(config)
    assert torch.equal(TC.param_sums(model), torch.from_numpy(fx.param_sums)), 'seeded weights differ from the reference'
    assert [n for n, _ in sorted(model.named_parameters())] == fx.names
    sd = {k: v.detach().double().clone().requires_grad_(v.is_floating_point()) for k, v in model.state_dict().items()}
    for k in list(sd):          # prenet and attention are registered twice (top level and under _decoder): one tensor each
        if k.startswith('_decoder._prenet.') or k.startswith('_decoder._attention.'):
            sd[k] = sd[k[len('_decoder.'):]]
    text, lens, mel, _, tlens, stop_t, spk, lang = TC.make_batch(hp)
    mel = mel.double()
    tape = {k: (v if k == 'teacher' else v.double()) for k, v in tape.items()}
    ohp = configs.as_namespace()
    post, pre, stop, align, spk_pred, _ = O.tacotron_forward(sd, ohp, text, lens, mel, tlens, spk, lang, tape, training=True)
    loss, parts = O.tacotron_loss(ohp, hp.guided_attention_toleration, lens, tlens, pre, mel, post, mel, stop, stop_t, align, spk,
                                  spk_pred)
    loss.backward()
    grads = {}
    for name in fx.names:
        g = sd[name].grad.clone()
        if name == '_embedding.weight':
            g[0] = 0            # Embedding(padding_idx=0): row 0 receives no gradient (tacotron2.py:237-238)
        grads[name] = g
    norm = float(torch.cat([g.reshape(-1) for g in grads.values()]).norm())
    return {k: float(v.detach()) for k, v in parts.items()}, grads, norm


@pytest.mark.parametrize('config', TC.CONFIGS)
def test_fixture_step0_replays_through_oracle(config):
    fx = TC.Fixture(config)
    parts, grads, norm = oracle_step0(config, fx, fx.tape(0))
    assert sorted(parts) == fx.loss_keys
    bad = [f'{k}: oracle {parts[k]:.7g} vs reference {r:.7g}' for k, r in zip(fx.loss_keys, fx.losses[0])
           if not abs(parts[k] - r) <= 1e-5 * abs(r) + 1e-8]
    assert not bad, '; '.join(bad)
    assert abs(norm - fx.gradient[0]) <= 1e-5 * fx.gradient[0], (norm, fx.gradient[0])
    ref = fx.grad(0)
    for name in fx.names:
        scale = float(ref[name].abs().max()) + 1e-12
        assert_close(grads[name], ref[name], 0.0, 1e-4 * scale + 1e-12, f'{config}: grad {name}')


@pytest.mark.parametrize('config', TC.CONFIGS)
def test_fixture_updates_are_adam_of_the_recorded_gradients(config):
    """train(): clip_grad_norm_(gradient_clipping) then Adam(lr, weight_decay), twice; in fp64 from the recorded gradients."""
    fx = TC.Fixture(config)
    hp, model = _seeded(config)
    params = [p.detach().double().clone().requires_grad_(True) for _, p in sorted(model.named_parameters())]
    start = [p.detach().clone() for p in params]
    opt = torch.optim.Adam(params, lr=hp.learning_rate, weight_decay=hp.weight_decay)
    for step in range(2):
        g = fx.grad(step)
        norm = float(torch.cat([g[n].reshape(-1) for n in fx.names]).norm())
        assert abs(norm - fx.gradient[step]) <= 1e-4 * fx.gradient[step], (step, norm, fx.gradient[step])
        coef = min(1.0, hp.gradient_clipping / (fx.gradient[step] + 1e-6))
        for p, n in zip(params, fx.names):
            p.grad = g[n] * coef
        opt.step()
    ref, cond = fx.update(), fx.conditioned()
    for p, p0, n in zip(params, start, fx.names):
        # float16 storage of a change of ~2 * lr: measured at most 1.3e-6 off on the conditioned elements
        assert_close((p.detach() - p0)[cond[n]], ref[n][cond[n]], 0.0, 3e-6, f'{config}: update {n}')
