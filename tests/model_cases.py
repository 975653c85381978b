"""Whole-model parity: this package's Tacotron (host modules + library) against golden vectors of the unmodified reference."""
import torch

from helpers import Golden, assert_close


def configure_hp(g):
    from multilingual_text_to_speech_b200.params.params import Params as hp
    hp.reset()
    hp.load_state_dict(g.meta['hp'])
    return hp


def build_model(g, device=None):
    from multilingual_text_to_speech_b200.modules.tacotron2 import Tacotron
    configure_hp(g)
    model = Tacotron()
    model.load_state_dict(g.sd, strict=True)
    model.train(g.train)
    return model.to(device) if device is not None else model


def run_golden(name, check_grads=True, verbose=False):
    from multilingual_text_to_speech_b200.modules.tacotron2 import TacotronLoss
    from multilingual_text_to_speech_b200.rng import MaskSource
    from multilingual_text_to_speech_b200.params.params import Params as hp
    g = Golden(name)
    dev = torch.device('cuda:0')
    model = build_model(g, dev)
    i = {k: v.to(dev) for k, v in g.inputs.items()}
    MaskSource.use_tape(g.tape)
    try:
        with torch.set_grad_enabled(g.train):
            post, pre, stop, align, spk, enc = model(i['text'], i['text_length'], i['target'], i['target_length'],
                                                     i.get('speakers'), i.get('languages'), g.tf)
    finally:
        MaskSource.use_tape(None)
    report = {}
    for key, got in (('enc', enc), ('align', align), ('pre', pre), ('stop', stop), ('post', post), ('spk_pred', spk)):
        if got is None:
            continue
        report[key] = float((got.detach().cpu() - g.out[key]).abs().max())
        assert_close(got, g.out[key], 1e-3, 1e-4, f'{name}: {key}')
    assert torch.equal(align.detach().cpu().argmax(2), g.out['align'].argmax(2)), 'alignment argmax differs'
    assert torch.equal(stop.detach().cpu() > 0, g.out['stop'] > 0), 'stop-token decision differs'
    # running statistics after one training forward
    if g.train:
        sd_after = model.state_dict()
        for k, ref in g.sd_after.items():
            if 'num_batches' in k:
                assert int(sd_after[k]) == int(ref), k
            else:
                assert_close(sd_after[k], ref, 1e-3, 1e-5, f'{name}: {k}')
    if check_grads and g.train and bool(g.tape['teacher'].all()):
        crit = TacotronLoss(hp.guided_attention_steps, g.meta['guided_g'], hp.guided_attention_gain)
        loss, parts = crit(i['text_length'], i['target_length'], pre, i['target'], post, i['target'], stop, i['stop_target'],
                           align, i.get('speakers'), spk, enc, None)
        for k, v in parts.items():
            assert abs(float(v) - g.losses[k]) < 2e-4 * max(1.0, abs(g.losses[k])), (k, float(v), g.losses[k])
        loss.backward()
        torch.cuda.synchronize()
        for k, prm in model.named_parameters():
            ref = g.grad[k]
            got = prm.grad if prm.grad is not None else torch.zeros_like(prm)
            scale = float(ref.abs().max()) + 1e-12
            report['d' + k] = float((got.detach().cpu() - ref).abs().max()) / scale
            assert_close(got, ref, 3e-3, 3e-4 * scale + 1e-9, f'{name}: grad {k}')
    if verbose:
        worst = sorted(report.items(), key=lambda kv: -kv[1])[:6]
        print(name, {k: f'{v:.2e}' for k, v in worst})
    return report
