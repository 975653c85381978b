"""Golden vectors of forward attention (hp.attention_type = "forward", reference modules/attention.py:89-124) from the UNMODIFIED
reference (build container only):

    PYTHONDONTWRITEBYTECODE=1 python tests/golden/make_golden_forward_attention.py

Reuses the recipes of make_golden.py (training / evaluation: Tacotron.forward + TacotronLoss + backward with the recorded mask tape)
and make_golden_inference.py (Tacotron.inference with early exit) on new case names, and the module case of module_cases.py.  Writes
only new files:
  fwd_lj_dropout          LJ-like, dropout cells, teacher forcing 1.0, training
  fwd_lj_zoneout_tf05     LJ-like, zoneout cells, teacher forcing 0.5, training (free-running steps inside the backward)
  fwd_lj_eval_free        LJ-like, evaluation mode, teacher forcing 0.0 (what train.py evaluates every epoch)
  fwd_generated_ragged    generated encoder, three languages, ragged text lengths (softmax over padded positions)
  fwd_inf_lj              Tacotron.inference
  fwd_attention_module    ForwardAttention.reset + three forward steps with the gradients of every input and parameter
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))
import make_golden              # noqa: E402
import make_golden_inference    # noqa: E402

FWD = dict(attention_type='forward')
TRAIN_CASES = {
    # name: (hp overrides, B, L, T, teacher_forcing, train_mode)
    'fwd_lj_dropout': (dict(FWD), 5, 11, 17, 1.0, True),
    'fwd_lj_zoneout_tf05': (dict(FWD, decoder_regularization='zoneout'), 5, 11, 17, 0.5, True),
    'fwd_lj_eval_free': (dict(FWD), 3, 9, 10, 0.0, False),
    # narrower encoder and decoder than the other cases: the 14 generated encoder blocks would otherwise make this the largest fixture
    'fwd_generated_ragged': (dict(FWD, encoder_type='generated', multi_language=True, languages=['a', 'b', 'c'], embedding_dimension=8,
                                  encoder_dimension=8, decoder_dimension=32, language_embedding_dimension=6, generator_dim=5,
                                  generator_bottleneck_dim=2), 6, 11, 17, 1.0, True),
}
INFERENCE_CASES = {
    'fwd_inf_lj': (dict(FWD, max_output_length=60), 9, 0.0),
}


def module_golden():
    sys.path.insert(0, make_golden.REF)
    import torch
    import utils  # noqa: F401  (must precede the modules: circular import in the reference)
    from modules.attention import ForwardAttention
    import module_cases as C
    torch.manual_seed(0)
    d = C.ATT_DIMS
    out = C.pack('forward_attention', C.attention_case(ForwardAttention(d['A'], d['D'], d['M']), 'cpu'))
    path = os.path.join(HERE, 'fwd_attention_module.npz')
    np.savez_compressed(path, **out)
    print(path, os.path.getsize(path), 'bytes,', len(out), 'arrays')


def main():
    sys.path.insert(0, make_golden.REF)
    import utils  # noqa: F401  (must precede the modules: circular import in the reference)
    from params.params import Params as hp
    defaults = dict(hp.state_dict())
    make_golden.CASES = TRAIN_CASES
    make_golden.main()
    hp.load_state_dict(defaults)        # make_golden_inference takes its defaults from the current Params
    make_golden_inference.CASES = INFERENCE_CASES
    make_golden_inference.main()
    module_golden()


if __name__ == '__main__':
    main()
