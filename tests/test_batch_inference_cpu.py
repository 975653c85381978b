"""Host logic of Tacotron.inference_batch without a GPU: argument validation, sorting / grouping / order restoration, the mask-tape
columns of utterances that leave the decode, and the library's refusal of a masked conv block outside eval mode."""
import ctypes

import pytest
import torch

from multilingual_text_to_speech_b200.modules import tacotron2 as T
from multilingual_text_to_speech_b200.modules.tacotron2 import Decoder
from multilingual_text_to_speech_b200.params.params import Params as hp


@pytest.fixture(autouse=True)
def _hp():
    hp.reset()
    yield
    hp.reset()


def _texts(*lengths):
    return [torch.ones(L, dtype=torch.long) for L in lengths]


def test_validation():
    with pytest.raises(ValueError, match='no texts'):
        T._check_batch_inputs([], None, None)
    with pytest.raises(ValueError, match='int64'):
        T._check_batch_inputs([torch.ones(3)], None, None)
    with pytest.raises(ValueError, match='1 speakers for 2 texts'):
        T._check_batch_inputs(_texts(3, 4), [torch.LongTensor([0])], None)
    with pytest.raises(ValueError, match='every text or for none'):
        T._check_batch_inputs(_texts(3, 4), None, [torch.LongTensor([0]), None])
    mixed = [torch.LongTensor([0]), torch.zeros(1, 4, 3)]
    with pytest.raises(ValueError, match='one form'):
        T._check_batch_inputs(_texts(3, 4), None, mixed)
    with pytest.raises(ValueError, match='L the text length'):
        T._check_batch_inputs(_texts(3), None, [torch.zeros(1, 4, 3)])
    hp.multi_speaker = True
    with pytest.raises(ValueError, match='multi-speaker'):
        T._check_batch_inputs(_texts(3), None, None)
    speakers, languages = T._check_batch_inputs(_texts(3, 4), [torch.LongTensor([1]), torch.LongTensor([0])],
                                                [torch.zeros(1, 3, 2), torch.zeros(1, 4, 2)])
    assert len(speakers) == len(languages) == 2


def test_sorting_grouping_and_order():
    lengths = [9, 3, 7, 3, 12, 1, 8]
    plan = T._batch_plan(lengths, 3)
    assert plan == [[5, 1, 3], [2, 6, 0], [4]]
    assert sorted(i for g in plan for i in g) == list(range(len(lengths)))
    assert all(len(g) <= 3 for g in plan)
    flat = [lengths[i] for g in plan for i in g]
    assert flat == sorted(flat)
    assert T._batch_plan(lengths, 64) == [sorted(range(7), key=lambda i: lengths[i])]
    with pytest.raises(ValueError):
        T._batch_plan(lengths, 0)


def test_tape_columns_follow_retired_utterances():
    """Three utterances whose tape columns are 4, 0 and 2 of a shared tape; the second stops in the first chunk, so the second chunk
    must read the columns of the first and third only."""
    Tt, P, chunk = 10, 3, 4
    tape = torch.arange(Tt * 5 * P, dtype=torch.int64).reshape(Tt, 5, P)
    columns = [4, 0, 2]
    rows = [0, 1, 2]
    rules = [Decoder._StopRule(1) for _ in rows]
    part = Decoder._tape_part(tape, 0, chunk, [columns[r] for r in rows])
    assert torch.equal(part, tape[:chunk][:, columns])
    logits = {0: [-1.0] * chunk, 1: [-1.0, 1.0, 1.0, -1.0], 2: [-1.0] * chunk}
    for r in rows:
        rules[r].feed(torch.tensor(logits[r]))
    keep = Decoder._retire(rows, rules)
    assert keep == [0, 2] and rules[1].cut == 3
    rows = [rows[j] for j in keep]
    part = Decoder._tape_part(tape, chunk, chunk, [columns[r] for r in rows])
    assert torch.equal(part, tape[chunk:2 * chunk][:, [4, 2]])
    # past the end of the recorded tape: all-ones rows for every utterance still decoding
    part = Decoder._tape_part(tape, 8, chunk, [columns[r] for r in rows])
    assert torch.equal(part[:2], tape[8:][:, [4, 2]]) and bool((part[2:] == 1).all()) and part.shape == (chunk, 2, P)


def test_masked_conv_block_rejected_outside_eval():
    from multilingual_text_to_speech_b200 import _lib
    lib = _lib.load()
    fake = ctypes.c_void_p(256)        # never dereferenced: the shape is refused before any device work
    for training, stage in ((1, 0), (0, 1), (0, 2)):
        shape = _lib.ConvBlockShape(1, 1, 4, 4, 8, 1 if stage == 2 else 3, 1, 0, 0, training, 1e-5, 0.1, 0.0, stage)
        status = lib.b200tts_convblock_forward_masked(ctypes.byref(shape), fake, fake, fake, fake, fake, 4, None, None, None, fake, fake,
                                                      fake, None)
        assert status != 0
        assert b'eval mode' in lib.b200tts_last_error()


def test_masked_block_module_refuses_training_mode():
    from multilingual_text_to_speech_b200.modules.layers import ConvBlock, ConvBlockGenerated
    block = ConvBlock(4, 4, 3, activation='relu')
    gen = ConvBlockGenerated(2, 2, 4, 4, 3)
    lengths = torch.tensor([3], dtype=torch.int32)
    x = torch.zeros(1, 4, 5)
    with pytest.raises(RuntimeError, match='eval mode only'):
        block(x, lengths)
    with pytest.raises(RuntimeError, match='eval mode only'):
        gen((torch.zeros(1, 2), x), lengths)
