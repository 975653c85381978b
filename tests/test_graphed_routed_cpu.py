"""Graph-captured routed steps without a GPU: GroupLayout with a capacity (modules/encoder.py), the given-layout scope, and the host
side of graph.GraphedTrainStep's routed replays (graph.StaticRouting): the layout read from each batch's labels, the capacity and
batch-size checks made before any static buffer is written, and the counts / rows that one copy puts into the static buffer."""
import pytest
import torch

from multilingual_text_to_speech_b200.graph import GraphedTrainStep, StaticRouting
from multilingual_text_to_speech_b200.modules.encoder import GroupLayout, encoder_layout, given_layout, reference_layout


IDS = [2, 0, 0, 3, 2, 2, 0]          # G = 4: language 1 absent, n_max = 3


def test_capacity_layout_rows_counts_and_vacancy():
    lay = GroupLayout(IDS, 4, capacity=5)
    assert lay.counts == [3, 0, 3, 1]
    assert lay.ranks == [0, 0, 1, 0, 1, 2, 2]
    assert lay.n_max == 3 and lay.capacity == 5 and lay.nb == 5
    assert lay.rows() == [2, 0, 4, 3, 6, 10, 8]          # rank * G + language: independent of the capacity
    occupied = set(lay.rows())
    vacant = [q * 4 + g for g in range(4) for q in range(lay.counts[g], lay.nb)]
    assert len(vacant) == lay.nb * 4 - len(IDS) and not occupied & set(vacant)
    assert all(r < lay.nb * 4 for r in lay.rows())


def test_capacity_equal_to_n_max_is_todays_layout():
    for ids, G in ((IDS, 4), ([b % 10 for b in range(64)], 10), ([0, 1, 2, 0, 1, 2], 3)):
        plain, capped = GroupLayout(ids, G), GroupLayout(ids, G, capacity=GroupLayout(ids, G).n_max)
        assert plain.capacity is None and plain.nb == plain.n_max
        assert (capped.counts, capped.ranks, capped.rows(), capped.nb, capped.reference) == \
               (plain.counts, plain.ranks, plain.rows(), plain.nb, plain.reference)


def test_over_capacity_names_the_language_its_count_and_the_capacity():
    with pytest.raises(ValueError, match='language 0 has 3 utterances .* capacity of 2'):
        GroupLayout(IDS, 4, capacity=2)
    GroupLayout(IDS, 4, capacity=3)                      # exactly at capacity


def test_given_layout_scope():
    ids = torch.tensor([1, 0, 1])
    routing = (torch.zeros(2, dtype=torch.int32), torch.zeros(3, dtype=torch.int64), 4)
    with given_layout(routing):
        assert encoder_layout(ids, 3, 2) is routing
        with reference_layout():                         # the innermost scope decides
            assert encoder_layout(ids, 3, 2) is None
        assert encoder_layout(ids, 3, 2) is routing
        assert encoder_layout(ids, 3, 1) is None          # one language, the mixing branch: never routed
        assert encoder_layout(ids[:1], 1, 2) is None
        assert encoder_layout(ids, 3, 2, padded=True) is None
    assert isinstance(encoder_layout(ids, 3, 2), GroupLayout)


def _unpacked(r):
    return r.counts.tolist(), r.rows.tolist()


def test_static_routing_fills_counts_and_rows_from_cpu_labels_without_a_device_copy(monkeypatch):
    r = StaticRouting(4, len(IDS), 3, 'cpu')
    assert r.buffer.dtype == torch.int32 and r.counts.dtype == torch.int32 and r.rows.dtype == torch.int64
    assert r.rows.data_ptr() % 8 == 0
    labels = [torch.tensor(IDS), torch.tensor(IDS).unsqueeze(1).expand(-1, 5)]
    real_to = torch.Tensor.to

    def forbidden(*a, **k):
        raise AssertionError('the labels were copied')
    monkeypatch.setattr(torch.Tensor, 'cpu', forbidden)
    monkeypatch.setattr(torch.Tensor, 'to', forbidden)
    monkeypatch.setattr(torch.Tensor, 'item', forbidden)
    layouts = [r.layout(lab) for lab in labels]
    monkeypatch.setattr(torch.Tensor, 'to', real_to)
    for lay in layouts:
        r.load(lay)
        assert _unpacked(r) == ([3, 0, 3, 1], [2, 0, 4, 3, 6, 10, 8])
    other = [1, 1, 3, 3, 3, 0, 1]                        # a new pattern, language 2 absent
    r.load(r.layout(torch.tensor(other)))
    assert _unpacked(r) == (GroupLayout(other, 4).counts, GroupLayout(other, 4).rows())


def test_static_routing_checks_before_writing():
    r = StaticRouting(5, 6, 2, 'cpu')                    # odd G: the rows start after one pad word
    r.load(r.layout(torch.tensor([0, 1, 2, 3, 4, 0])))
    before = r.buffer.clone()
    with pytest.raises(ValueError, match='language 4 has 3 utterances .* capacity of 2'):
        r.layout(torch.tensor([4, 1, 4, 3, 4, 0]))
    with pytest.raises(ValueError, match='labels for 5 utterances given for a graph captured at a batch of 6'):
        r.layout(torch.tensor([0, 1, 2, 3, 4]))
    with pytest.raises(ValueError, match='language ids'):
        r.layout(torch.tensor([0, 1, 2, 3, 5, 0]))
    assert torch.equal(r.buffer, before)
    assert _unpacked(r) == ([2, 1, 1, 1, 1], [0, 1, 2, 3, 4, 5])


def test_graphed_train_step_refuses_an_over_capacity_example_batch():
    """The example batch meets the same capacity check as every later batch, before anything is allocated or captured; a routed
    example batch without a capacity is refused with the capacity it would need."""
    from multilingual_text_to_speech_b200 import configs
    from multilingual_text_to_speech_b200.modules.tacotron2 import Tacotron
    hp = configs.apply('generated_training', decoder_regularization='zoneout')
    G = hp.language_number
    model = Tacotron()
    batch = {'text': torch.ones(G + 3, 5, dtype=torch.long), 'languages': torch.arange(G + 3) % G}     # languages 0..2 twice
    with pytest.raises(ValueError, match='language 0 has 2 utterances .* capacity of 1'):
        GraphedTrainStep(model, None, None, batch, max_per_language=1)
    with pytest.raises(ValueError, match=r'pass max_per_language.*the example batch has 2'):                   # no capacity given
        GraphedTrainStep(model, None, None, batch)
    batch = {'text': torch.ones(G, 5, dtype=torch.long), 'languages': torch.arange(G) % G}             # reference layout
    with pytest.raises(ValueError, match='max_per_language must be at least 1'):
        GraphedTrainStep(model, None, None, batch, max_per_language=0)
