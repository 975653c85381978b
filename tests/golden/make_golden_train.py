"""Golden record of the UNMODIFIED reference's own `train()` (train.py:29-95) for two optimisation steps (tests/train_case.py):
the losses, gradient norms and classifier accuracies it logs, and checksums of the seeded initial weights.

    python tests/golden/make_golden_train.py          # needs the reference checkout at REF; writes tests/golden/reference_train.npz

The reference runs on its own modules on the CPU; only the modules train.py imports for data loading and logging (corpus readers,
samplers, audio / text front end, TensorBoard) are replaced by stubs, as they are not on the training path.
"""
import importlib.util
import json
import os
import sys
import types

import numpy as np

REF = '/root/reference'
HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))


def main():
    sys.path.insert(0, REF)
    sys.dont_write_bytecode = True
    import torch
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
        out[f'{config}.param_sums'] = TC.param_sums(model).numpy()
        optimizer = torch.optim.Adam(model.parameters(), lr=hp.learning_rate, weight_decay=hp.weight_decay)
        criterion = TacotronLoss(hp.guided_attention_steps, hp.guided_attention_toleration, hp.guided_attention_gain)
        batch = TC.make_batch(hp)
        logged.clear()
        train_py.train(0, 0, [batch, batch], model, criterion, optimizer)
        keys = sorted(logged[0][0])
        meta[config] = {'loss_keys': keys}
        out[f'{config}.losses'] = np.array([[step[0][k] for k in keys] for step in logged], dtype=np.float64)
        out[f'{config}.gradient'] = np.array([step[1] for step in logged], dtype=np.float64)
        out[f'{config}.classifier'] = np.array([step[2] for step in logged], dtype=np.float64)
        print(config, keys, out[f'{config}.losses'].tolist(), out[f'{config}.gradient'].tolist(), out[f'{config}.classifier'].tolist())
    out['meta'] = np.frombuffer(json.dumps(meta).encode(), dtype=np.uint8)
    path = os.path.join(HERE, 'reference_train.npz')
    np.savez_compressed(path, **out)
    print(path, os.path.getsize(path), 'bytes')


if __name__ == '__main__':
    main()
