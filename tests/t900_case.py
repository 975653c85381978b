"""The real-dimension, benchmarked-shape parity case: `generated_training` (10 languages, generated encoder, M = 288,
D = 1024, A = 128), zoneout cells, B = 10, L = 180, T = 900, teacher forcing 1.0, train mode, default initialisation.

Everything that can be regenerated from a seed is NOT stored in the fixture (tests/golden/t900_generated_training.npz):
* weights    = `torch.manual_seed(WEIGHT_SEED); Tacotron()` -- the host classes construct their parameters in the reference's
               order, so the values are bit-identical to the reference's own `Tacotron()` (checked when the fixture is made and,
               through a checksum, every time it is used);
* inputs     = `build_inputs` (seeded);
* mask tape  = `replay_tape`: the dropout masks / teacher-forcing coins the reference drew, in its call order
               (SURVEY.md appendix A.7), regenerated from TAPE_SEED by replaying the same sequence of `torch.rand` calls.
tests/golden/make_golden_t900.py (run in the build container, imports the UNMODIFIED reference) asserts that these regenerated
tensors are exactly what the reference consumed, and stores their checksums next to the reference's outputs / gradients.
"""
import hashlib
import numpy as np
import torch

NAME = 't900_generated_training'
CONFIG = 'generated_training'
B, L, T = 10, 180, 900
WEIGHT_SEED, INPUT_SEED, TAPE_SEED = 0, 1234, 4321
HP_OVERRIDES = dict(decoder_regularization='zoneout')
# encoder block list of GeneratedConvolutionalEncoder (reference modules/encoder.py:180-191): conv output channels per group
ENC_COUT = [256, 256] + [512] * 10 + [512, 512]


def digest(t):
    t = t.detach().cpu().contiguous()
    return hashlib.sha256(t.numpy().tobytes()).hexdigest()[:16]


def state_digest(sd):
    h = hashlib.sha256()
    for k in sorted(sd):
        h.update(k.encode())
        h.update(sd[k].detach().cpu().contiguous().numpy().tobytes())
    return h.hexdigest()[:16]


def build_inputs(symbols, num_mels, stop_frames, G):
    """Seeded synthetic batch in the layout of SURVEY section 8d, ragged (lengths exercise the masks), language b % G."""
    g = torch.Generator().manual_seed(INPUT_SEED)
    lens = torch.randint(L // 2, L + 1, (B,), generator=g)
    lens[0] = L
    text = torch.randint(1, symbols, (B, L), generator=g)
    for b in range(B):
        text[b, lens[b]:] = 0
    tlens = torch.clamp(lens * 5, max=T)
    tlens[0] = T
    target = torch.randn(B, num_mels, T, generator=g)
    stop_target = torch.zeros(B, T)
    for b in range(B):
        stop_target[b, int(tlens[b]) - stop_frames:] = 1.0
    return {'text': text, 'text_length': lens, 'target': target, 'target_length': tlens, 'stop_target': stop_target,
            'languages': torch.arange(B) % G}


def draw_plan(G, P, D, N, postnet_dim, postnet_blocks, zoneout=True):
    """The sequence of random draws of one training forward (tf = 1.0): [(name, kind, p, shape)], reference call order."""
    plan = []
    for j, c in enumerate(ENC_COUT):
        plan.append((f'enc{j}', 'mask', 0.05, (B // G, G * c, L)))
    plan.append(('prenet0', 'mask', 0.5, (B, T + 1, P)))
    plan.append(('prenet1', 'mask', 0.5, (B, T + 1, P)))
    plan.append(('teacher', 'rand', None, (T,)))
    for i in range(T):
        for cell in ('att', 'gen'):
            plan.append((f'{cell}_h/{i}', 'mask', 0.1, (B, D)))
            if zoneout:
                plan.append((f'{cell}_c/{i}', 'mask', 0.1, (B, D)))
    for j in range(postnet_blocks):
        plan.append((f'post{j}', 'mask', 0.5, (B, N if j == postnet_blocks - 1 else postnet_dim, T)))
    return plan


def replay_tape(G, P, D, N, postnet_dim, postnet_blocks, frames=T):
    """Regenerate the named mask tape (uint8 keep masks, teacher bools).  Always replays ALL draws (the random stream must stay
    aligned); `frames` < T only truncates what is returned (for the CPU oracle check on a prefix of the frames)."""
    torch.manual_seed(TAPE_SEED)
    tape = {}
    per = {k: torch.ones(T, B, D, dtype=torch.uint8) for k in ('att_h', 'att_c', 'gen_h', 'gen_c')}
    for name, kind, p, shape in draw_plan(G, P, D, N, postnet_dim, postnet_blocks):
        r = torch.rand(shape)
        if kind == 'rand':
            tape[name] = r > 0.0                        # teacher forcing 1.0: rand > 1 - tf
        elif '/' in name:
            key, i = name.split('/')
            per[key][int(i)] = (r >= p).to(torch.uint8)
        else:
            tape[name] = (r >= p).to(torch.uint8)
    tape.update(per)
    tape['step_prenet0'] = torch.ones(T, B, P, dtype=torch.uint8)
    tape['step_prenet1'] = torch.ones(T, B, P, dtype=torch.uint8)
    if frames < T:
        for k in ('att_h', 'att_c', 'gen_h', 'gen_c', 'step_prenet0', 'step_prenet1'):
            tape[k] = tape[k][:frames]
        tape['teacher'] = tape['teacher'][:frames]
        tape['prenet0'], tape['prenet1'] = tape['prenet0'][:, :frames + 1], tape['prenet1'][:, :frames + 1]
        for j in range(postnet_blocks):
            tape[f'post{j}'] = tape[f'post{j}'][:, :, :frames]
    return tape


def tape_digest(tape):
    h = hashlib.sha256()
    for k in sorted(tape):
        h.update(k.encode())
        h.update(tape[k].to(torch.uint8).contiguous().numpy().tobytes())
    return h.hexdigest()[:16]


# parameters whose full gradient is stored (everything up to this many elements); larger ones: norm, sum, strided sample
FULL_GRAD_LIMIT = 200_000
SAMPLE_STRIDE = 997


def grad_summary(g):
    g = g.detach().double().flatten()
    return np.array([float(g.norm()), float(g.sum()), float(g.abs().max())]), g[::SAMPLE_STRIDE].float().numpy()


# ------------------------------------------------------------------------------------------------------------------
# fixture access + the GPU run shared by tests/test_gpu_t900.py and __graft_entry__.smoke()
# ------------------------------------------------------------------------------------------------------------------
class Fixture:
    def __init__(self):
        import json
        import os
        here = os.path.dirname(os.path.abspath(__file__))
        z = np.load(os.path.join(here, 'golden', NAME + '.npz'))
        self.meta = json.loads(bytes(z['meta']).decode())
        self.out, self.grad, self.gsum, self.gsample, self.sd_after = {}, {}, {}, {}, {}
        for key in z.files:
            if key == 'meta':
                continue
            group, _, rest = key.partition('.')
            {'out': self.out, 'grad': self.grad, 'gsum': self.gsum, 'gsample': self.gsample,
             'sd_after': self.sd_after}[group][rest] = torch.from_numpy(z[key])
        self.losses = self.meta['losses']


def configure():
    """hp of the case, the seeded model (bit-identical to the reference's seeded `Tacotron()`), inputs, tape."""
    from multilingual_text_to_speech_b200 import configs
    from multilingual_text_to_speech_b200.modules.tacotron2 import Tacotron
    hp = configs.apply(CONFIG, **HP_OVERRIDES)
    torch.manual_seed(WEIGHT_SEED)
    model = Tacotron().train()
    inp = build_inputs(hp.symbols_count() + 3, hp.num_mels, hp.stop_frames, hp.language_number)
    return hp, model, inp


def tape_for(hp, frames=T):
    return replay_tape(hp.language_number, hp.prenet_dimension, hp.decoder_dimension, hp.num_mels, hp.postnet_dimension,
                       hp.postnet_blocks, frames)


def run_gpu(mode, fx=None, with_grads=True, verbose=True):
    """This package's path (host modules + libb200tts.so) on the fixture's inputs in precision `mode`; returns a report of errors
    against the UNMODIFIED reference's recorded results.  Asserts nothing: the callers hold the gates."""
    from multilingual_text_to_speech_b200 import _lib
    from multilingual_text_to_speech_b200.modules.tacotron2 import TacotronLoss
    from multilingual_text_to_speech_b200.rng import MaskSource
    fx = fx or Fixture()
    hp, model, inp = configure()
    assert state_digest(model.state_dict()) == fx.meta['weight_digest'], 'seeded weights differ from the reference fixture'
    tape = tape_for(hp)
    assert tape_digest(tape) == fx.meta['tape_digest'], 'replayed mask tape differs from what the reference consumed'
    dev = torch.device('cuda:0')
    model = model.to(dev)
    i = {k: v.to(dev) for k, v in inp.items()}
    _lib.set_precision(mode)
    MaskSource.use_tape(tape)
    try:
        post, pre, stop, align, _, enc = model(i['text'], i['text_length'], i['target'], i['target_length'], None, i['languages'], 1.0)
        rep = {}
        ref = fx.out
        for name, got in (('enc', enc), ('pre', pre), ('post', post), ('stop', stop)):
            d = (got.detach().cpu().double() - ref[name].double()).abs()
            r = ref[name].double().abs()
            rep[name + '_l1'], rep[name + '_max'] = float(d.mean()), float(d.max())
            rep[name + '_viol'] = float((d > 1e-4 + 1e-3 * r).float().mean())          # fraction outside rtol 1e-3 / atol 1e-4
        rep['pre_scale'] = float(ref['pre'].abs().mean())
        al = align.detach().cpu()
        rows = al[:, ::30]
        d = (rows.double() - ref['align_rows'].double()).abs()
        rep['align_max'], rep['align_viol'] = float(d.max()), float((d > 1e-4 + 1e-3 * ref['align_rows'].double().abs()).float().mean())
        rep['align_rowsum_max'] = float((al.sum(2) - ref['align_rowsum']).abs().max())
        idx = ref['align_top2_idx'].long()
        margin = ref['align_top2_val'][..., 0] - ref['align_top2_val'][..., 1]
        same = al.argmax(2) == idx[..., 0]
        rep['argmax_agree'] = float(same.float().mean())
        for eps in (0.0, 1e-7, 1e-6):
            clear = margin > eps
            rep[f'argmax_mismatch_margin>{eps:g}'] = int((~same & clear).sum())
        rep['argmax_tie_steps<=1e-7'] = int((margin <= 1e-7).sum())
        # stop decision: sign of the logit on the real frames (padding is filled with 1000)
        rs = ref['stop']
        real = rs < 999.0
        rep['stop_sign_mismatch'] = int(((stop.detach().cpu() > 0) != (rs > 0))[real & (rs.abs() > 1e-5)].sum())
        rep['stop_sign_mismatch_margin>2e-3'] = int(((stop.detach().cpu() > 0) != (rs > 0))[real & (rs.abs() > 2e-3)].sum())
        if with_grads:
            crit = TacotronLoss(hp.guided_attention_steps, fx.meta['guided_g'], hp.guided_attention_gain)
            loss, parts = crit(i['text_length'], i['target_length'], pre, i['target'], post, i['target'], stop, i['stop_target'],
                               align, None, None, enc, None)
            rep['losses'] = {k: float(v) for k, v in parts.items()}
            rep['losses']['total'] = float(loss)
            loss.backward()
            torch.cuda.synchronize()
            grel = {}
            for k, prm in model.named_parameters():
                g = (prm.grad if prm.grad is not None else torch.zeros_like(prm)).detach().cpu()
                if k in fx.grad:
                    refg = fx.grad[k].double()
                    grel[k] = float((g.double() - refg).norm() / (refg.norm() + 1e-30))
                else:
                    refs = fx.gsample[k].double()
                    gs = g.double().flatten()[::SAMPLE_STRIDE]
                    grel[k] = float((gs - refs).norm() / (refs.norm() + 1e-30))
                    nrm = float(g.double().norm())
                    grel[k + '#norm'] = abs(nrm - float(fx.gsum[k][0])) / (float(fx.gsum[k][0]) + 1e-30)
            rep['grad_rel'] = grel
            sd_after = model.state_dict()
            rep['running_stat_max'] = max(float((sd_after[k].cpu().double() - v.double()).abs().max() / (v.double().abs().max() + 1e-12))
                                          for k, v in fx.sd_after.items() if 'num_batches' not in k)
    finally:
        MaskSource.use_tape(None)
        _lib.set_precision('fp32')
    if verbose:
        flat = {k: v for k, v in rep.items() if not isinstance(v, dict)}
        print(f'[t900 {mode}]', {k: (f'{v:.3e}' if isinstance(v, float) else v) for k, v in flat.items()})
        if 'grad_rel' in rep:
            worst = sorted(rep['grad_rel'].items(), key=lambda kv: -kv[1])[:8]
            print(f'[t900 {mode}] losses', rep['losses'], 'reference', fx.losses)
            print(f'[t900 {mode}] worst gradient relative errors', {k: f'{v:.2e}' for k, v in worst})
    return rep
