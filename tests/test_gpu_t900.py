"""Parity at the BENCHMARKED shape against the unmodified reference: generated_training, zoneout cells, D = 1024, A = 128,
M = 288, G = 10, L = 180, T = 900 teacher-forced frames (B = 10: one utterance per language), fixture recorded by
tests/golden/make_golden_t900.py.  The reference modules replaced: modules/tacotron2.py:148-209,355-385,439-485.

fp32 mode  : north_star gate -- rtol 1e-3 / atol 1e-4 on every output, alignment argmax bit-exact on all 900 steps (steps whose
             reference top-1 / top-2 margin is below 1e-7, i.e. below fp32 resolution of the softmax, are counted and excluded),
             stop decision bit-exact, loss terms, every parameter gradient.
bf16 mode  : the benchmarked mode -- mel L1 < 1e-3 against the REFERENCE (north_star), alignment-argmax agreement and gradient
             relative errors reported and bounded.
"""
import pytest
import torch

import t900_case as C

pytestmark = pytest.mark.gpu


@pytest.fixture(scope='module', autouse=True)
def _built():
    import __graft_entry__ as entry
    entry.build()
    assert torch.cuda.is_available()


@pytest.fixture(scope='module')
def fx():
    return C.Fixture()


def test_t900_fp32_mode_meets_the_parity_gate(fx):
    rep = C.run_gpu('fp32', fx)
    for name in ('enc', 'pre', 'post', 'stop'):
        assert rep[name + '_viol'] == 0.0, (name, rep[name + '_max'], rep[name + '_viol'])
    assert rep['align_viol'] == 0.0 and rep['align_rowsum_max'] < 1e-5, rep
    assert rep['argmax_mismatch_margin>1e-07'] == 0, rep
    assert rep['stop_sign_mismatch'] == 0, rep
    for k, v in fx.losses.items():
        assert abs(rep['losses'][k] - v) < 2e-4 * max(1.0, abs(v)), (k, rep['losses'][k], v)
    bad = {k: v for k, v in rep['grad_rel'].items() if v > 2e-3}
    assert not bad, bad
    assert rep['running_stat_max'] < 1e-4, rep['running_stat_max']


def test_t900_bf16_mode_meets_the_mel_gate(fx):
    rep = C.run_gpu('bf16', fx)
    # north_star: mel L1 vs reference < 1e-3 (decoder output = `pre`; mean |pre| of the reference is 4.4e-2)
    assert rep['pre_l1'] < 1e-3, rep
    # `post` passes 5 train-mode BatchNorm layers that amplify any input difference (SURVEY 7.3); bounded relative to mean |post| = 0.66
    assert rep['post_l1'] < 2e-2, rep
    assert rep['enc_l1'] < 4e-3, rep
    # argmax disagreements come from steps whose reference top-1 / top-2 margin is within the bf16 operand rounding of the attention weights
    assert rep['argmax_agree'] > 0.975, rep
    assert rep['align_max'] < 1e-4, rep
    # the stop decision can only flip where the reference logit is within the bf16 error (max |d stop| 5.3e-4) of zero
    assert rep['stop_sign_mismatch_margin>2e-3'] == 0 and rep['stop_sign_mismatch'] <= 20, rep
    for k, v in fx.losses.items():
        assert abs(rep['losses'][k] - v) < 1e-2 * max(1.0, abs(v)), (k, rep['losses'][k], v)
    # gradients against the reference's fp32 gradients: bf16 operand rounding over a 900-step recurrence
    grel = rep['grad_rel']
    worst = max(grel.values())
    print('bf16 gradient relative errors: max', worst)
    bad = {k: v for k, v in grel.items() if v > 0.1}
    assert not bad, bad
