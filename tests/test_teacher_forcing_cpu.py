"""Teacher forcing below 1.0 on the host side: the example's schedule restates train.py:58-60, and a graphed training step refuses a
ratio below 1.0 up front (the coins it would capture decide the launch sequence)."""
import importlib.util
import math
import os

import pytest

from helpers import ROOT


def _example():
    spec = importlib.util.spec_from_file_location('train_synthetic', os.path.join(ROOT, 'examples', 'train_synthetic.py'))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def test_example_schedule_follows_the_reference():
    ex = _example()
    hp = type('hp', (), dict(constant_teacher_forcing=True, teacher_forcing=0.7, teacher_forcing_start_steps=50000,
                             teacher_forcing_steps=100000))
    assert ex.teacher_forcing_ratio(hp, 0) == 0.7 and ex.teacher_forcing_ratio(hp, 10 ** 6) == 0.7
    hp.constant_teacher_forcing = False
    assert ex.teacher_forcing_ratio(hp, 0) == 1.0
    assert ex.teacher_forcing_ratio(hp, 50000) == 1.0
    assert math.isclose(ex.teacher_forcing_ratio(hp, 100000), 0.5, abs_tol=1e-12)
    assert math.isclose(ex.teacher_forcing_ratio(hp, 75000), 0.5 * (1 + math.cos(math.pi / 4)), abs_tol=1e-12)
    assert math.isclose(ex.teacher_forcing_ratio(hp, 150000), 0.0, abs_tol=1e-12)
    assert math.isclose(ex.teacher_forcing_ratio(hp, 10 ** 6), 0.0, abs_tol=1e-12)
    assert ex.teacher_forcing_ratio(hp, 50001) < 1.0


@pytest.mark.parametrize('tf', [0.99, 0.5, 0.0])
def test_graphed_step_refuses_teacher_forcing_below_one(tf):
    from multilingual_text_to_speech_b200.graph import GraphedTrainStep
    with pytest.raises(ValueError, match='teacher_forcing'):
        GraphedTrainStep(None, None, None, {}, teacher_forcing=tf)
