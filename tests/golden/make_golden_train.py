"""Golden record of the UNMODIFIED reference's own `train()` (train.py:29-95) for two optimisation steps (tests/train_case.py):
the losses, gradient norms and classifier accuracies it logs, checksums of the seeded initial weights, every dropout mask it draws,
every parameter's gradient at both steps and every parameter's change over the two Adam updates.

    python tests/golden/make_golden_train.py          # needs the reference checkout at REF; writes tests/golden/reference_train.npz

The reference runs on its own modules on the CPU; only the modules train.py imports for data loading and logging (corpus readers,
samplers, audio / text front end, TensorBoard) are replaced by stubs, as they are not on the training path.  As in make_golden.py,
`torch.nn.functional.dropout` and `torch.rand` are wrapped (the reference code itself is not edited) so that the masks of the generated
encoder, whose dropout rate is fixed at 0.05 (tacotron2.py:300-302), and the teacher-forcing coins are recorded in call order.
`torch.nn.utils.clip_grad_norm_` is wrapped to take each step's gradients before they are clipped.  The layout of the arrays is
described by train_case.Fixture.
"""
import importlib.util
import json
import os
import sys
import types
import zipfile

import numpy as np

REF = '/root/reference'
HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))


def main():
    sys.path.insert(0, REF)
    sys.dont_write_bytecode = True
    import torch
    import torch.nn.functional as F
    import utils  # noqa: F401  (must precede modules.tacotron2: circular import in the reference)
    from params.params import Params as hp
    from modules.tacotron2 import Tacotron, TacotronLoss
    import train_case as TC

    logged = []

    class Logger:
        @staticmethod
        def training(train_step, losses, gradient, learning_rate, duration, classifier):
            logged.append(({k: float(v) for k, v in losses.items()}, float(gradient), float(classifier)))

    def stub(name, **attrs):
        m = types.ModuleType(name)
        m.__dict__.update(attrs)
        return m
    sys.modules['utils.logging'] = stub('utils.logging', Logger=Logger)
    for name in ('audio', 'text'):           # DSP / text front end: third-party dependencies, not on the training path
        sys.modules[f'utils.{name}'] = stub(f'utils.{name}')
        setattr(utils, name, sys.modules[f'utils.{name}'])
    sys.modules['utils.samplers'] = stub('utils.samplers', RandomImbalancedSampler=object, PerfectBatchSampler=object)
    sys.modules['dataset'] = stub('dataset', __path__=[])
    sys.modules['dataset.dataset'] = stub('dataset.dataset', TextToSpeechDatasetCollection=object, TextToSpeechCollate=object)
    spec = importlib.util.spec_from_file_location('reference_train_py', os.path.join(REF, 'train.py'))
    train_py = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(train_py)

    real_dropout, real_rand, real_clip = F.dropout, torch.rand, torch.nn.utils.clip_grad_norm_
    masks, rands, steps = [], [], []

    def taped_dropout(input, p=0.5, training=True, inplace=False):
        if not training or p == 0.0:
            return input
        keep = (torch.rand_like(input) >= p).to(input.dtype)
        masks.append((float(p), keep.detach().clone()))
        return input * keep * (1.0 / (1.0 - p))

    def taped_rand(*a, **k):
        r = real_rand(*a, **k)
        rands.append(r.detach().clone())
        return r

    def taped_clip(parameters, *a, **k):
        parameters = list(parameters)
        steps.append(dict(masks=list(masks), rands=list(rands), grads={id(p): p.grad.detach().clone() for p in parameters}))
        masks.clear(); rands.clear()
        return real_clip(parameters, *a, **k)

    defaults = dict(hp.state_dict())
    jsons = {'generated_switching': 'generated_switching.json', 'ljspeech': None}
    out, meta = {}, {}
    for config in TC.CONFIGS:
        hp.load_state_dict(defaults)
        if jsons[config]:
            hp.load(os.path.join(REF, 'params', jsons[config]))
        hp.load_state_dict(TC.overrides(config))
        hp.language_number = len(hp.languages) if hp.multi_language else 0      # train.py:239-240
        hp.speaker_number = TC.SPEAKERS if hp.multi_speaker else 0
        torch.manual_seed(0)
        model = Tacotron()
        named = sorted(model.named_parameters())
        out[f'{config}.param_sums'] = TC.param_sums(model).numpy()
        before = [p.detach().clone() for _, p in named]
        optimizer = torch.optim.Adam(model.parameters(), lr=hp.learning_rate, weight_decay=hp.weight_decay)
        criterion = TacotronLoss(hp.guided_attention_steps, hp.guided_attention_toleration, hp.guided_attention_gain)
        batch = TC.make_batch(hp)
        logged.clear(); steps.clear()
        F.dropout, torch.rand, torch.nn.utils.clip_grad_norm_ = taped_dropout, taped_rand, taped_clip
        try:
            train_py.train(0, 0, [batch, batch], model, criterion, optimizer)
        finally:
            F.dropout, torch.rand, torch.nn.utils.clip_grad_norm_ = real_dropout, real_rand, real_clip
        assert len(steps) == len(logged) == 2

        keys = sorted(logged[0][0])
        n_enc = 14 if hp.encoder_type == 'generated' else hp.encoder_blocks
        tapes, mask_shapes = [], []
        for s, rec in enumerate(steps):
            # with DETERMINISTIC rates only the generated encoder's fixed 0.05 draws masks, one per block in block order
            expected = n_enc if hp.encoder_type == 'generated' else 0
            assert len(rec['masks']) == expected and all(p == 0.05 for p, _ in rec['masks']), (config, s, len(rec['masks']))
            assert len(rec['rands']) == 1 and bool((rec['rands'][0] > 1 - hp.teacher_forcing).all())
            tapes.append(np.concatenate([m.numpy().astype(np.uint8).ravel() for _, m in rec['masks']] + [np.zeros(0, np.uint8)]))
            mask_shapes = [list(m.shape) for _, m in rec['masks']]
        grads = [[rec['grads'][id(p)] for _, p in named] for rec in steps]
        update = [p.detach() - b for (_, p), b in zip(named, before)]
        meta[config] = dict(loss_keys=keys, params=[[k, list(p.shape)] for k, p in named], masks=mask_shapes)
        out[f'{config}.losses'] = np.array([[step[0][k] for k in keys] for step in logged], dtype=np.float64)
        out[f'{config}.gradient'] = np.array([step[1] for step in logged], dtype=np.float64)
        out[f'{config}.classifier'] = np.array([step[2] for step in logged], dtype=np.float64)
        out[f'{config}.tape'] = np.stack(tapes)
        q = [TC.quantise(g) for g in grads]
        out[f'{config}.grad'] = np.stack([a for a, _ in q])
        out[f'{config}.grad_scale'] = np.stack([sc for _, sc in q])
        out[f'{config}.update'] = torch.cat([u.reshape(-1) for u in update]).numpy().astype(np.float16)
        print(config, keys, out[f'{config}.losses'].tolist(), out[f'{config}.gradient'].tolist(), out[f'{config}.classifier'].tolist(),
              f'{sum(p.numel() for _, p in named)} parameter elements, {len(mask_shapes)} masks')
    out['meta'] = np.frombuffer(json.dumps(meta).encode(), dtype=np.uint8)
    path = os.path.join(HERE, 'reference_train.npz')
    # np.savez_compressed stamps each member with the current time; fixed stamps make a rerun reproduce the file byte for byte
    with zipfile.ZipFile(path, 'w') as zf:
        for key, arr in out.items():
            info = zipfile.ZipInfo(key + '.npy', date_time=(1980, 1, 1, 0, 0, 0))
            info.compress_type = zipfile.ZIP_DEFLATED
            with zf.open(info, 'w') as f:
                np.lib.format.write_array(f, np.asanyarray(arr), allow_pickle=False)
    print(path, os.path.getsize(path), 'bytes')


if __name__ == '__main__':
    main()
