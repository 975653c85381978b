"""GraphedTrainStep on routed grouped-encoder batches (graph.StaticRouting, modules/encoder.py given_layout): one CUDA graph captured
at a fixed capacity of rows per language, replayed across changing language layouts.

1. Every replay (balanced, imbalanced with an absent language, languages at capacity, the reference layout) gives bitwise the loss,
   loss terms, gradient bucket and model state of an eager step run in the same capacity layout at the same mask epoch; an absent
   language gets exactly zero gradients and keeps its running statistics.
2. One replay's encoder output, gradients and running statistics meet the fp64 per-language oracle of tests/routed_encoder_oracle.py
   under its bounds, with the masks that replay drew.
3. Over-capacity batches raise ValueError before any static buffer is written, with CPU and with CUDA labels.
4. CUDA labels rewritten in place between calls are read again.
5. A reference-layout example without max_per_language captures exactly the reference step (the plain body under reference_layout()):
   the same number of graph nodes and the same bits."""
import ctypes

import pytest
import torch

import routed_encoder_oracle as RO
from test_gpu_routed_encoder import _compare

pytestmark = pytest.mark.gpu

SMALL = dict(embedding_dimension=32, encoder_dimension=32, decoder_dimension=48, prenet_dimension=24, attention_dimension=16,
             attention_location_dimension=8, postnet_dimension=32, generator_dim=5, generator_bottleneck_dim=3,
             language_embedding_dimension=6, languages=['a', 'b', 'c', 'd'])


def _shuffled(counts, seed):
    ids = [g for g, n in enumerate(counts) for _ in range(n)]
    return [ids[i] for i in torch.randperm(len(ids), generator=torch.Generator().manual_seed(seed)).tolist()]


# name -> (hp overrides, capacity, L, T, patterns (the first is the example batch), the pattern checked against the oracle)
CASES = {
    # benchmark widths, G = 10, B = 64: the smallest capacity (7) puts at least four languages at capacity
    'B64_cap7': ({}, 7, 48, 24, {'balanced_7_6': [b % 10 for b in range(64)],
                                  'imbalanced': _shuffled([7, 7, 3, 7, 7, 7, 7, 7, 7, 5], 1),
                                  'sorted': sorted(b % 10 for b in range(64))}, 'imbalanced'),
    # B = 60 at capacity 9: the imbalanced sampler batch (language 2 absent, language 1 alone, language 0 at capacity) and a
    # reference-layout batch on the same graph
    'B60_cap9': ({}, 9, 48, 24, {'imbalanced_absent': _shuffled([9, 1, 0, 8, 7, 6, 8, 7, 6, 8], 9),
                                  'reference': [b % 10 for b in range(60)],
                                  'other_absent': _shuffled([9, 9, 9, 9, 9, 0, 6, 0, 0, 9], 3)}, 'imbalanced_absent'),
    'small_cap4': (SMALL, 4, 16, 12, {'reference': [b % 4 for b in range(12)],
                                       'absent': _shuffled([4, 4, 4, 0], 5),
                                       'imbalanced': _shuffled([4, 1, 3, 4], 6)}, 'absent'),
}


@pytest.fixture(scope='module', autouse=True)
def _built():
    import __graft_entry__ as entry
    entry.build()
    assert torch.cuda.is_available()


def _setup(kind, overrides):
    from multilingual_text_to_speech_b200 import configs
    from multilingual_text_to_speech_b200.distributed import GradBucket
    from multilingual_text_to_speech_b200.modules.tacotron2 import Tacotron, TacotronLoss
    hp = configs.apply('generated_training', decoder_regularization='zoneout', encoder_type=kind, **overrides)
    torch.manual_seed(0)
    model = Tacotron().cuda().train()
    crit = TacotronLoss(hp.guided_attention_steps, hp.guided_attention_toleration, hp.guided_attention_gain)
    return hp, model, crit, GradBucket(model, 1)


def _batch(hp, B, L, T, seed):
    g = torch.Generator().manual_seed(seed)
    text = torch.randint(1, hp.symbols_count() + 3, (B, L), generator=g)
    lens = torch.randint(L // 2, L + 1, (B,), generator=g)
    lens[0] = L
    for i in range(B):
        text[i, lens[i]:] = 0
    stop = torch.zeros(B, T)
    stop[:, T - hp.stop_frames:] = 1.0
    return {k: v.cuda() for k, v in dict(text=text, text_length=lens, target=torch.randn(B, hp.num_mels, T, generator=g),
                                          target_length=torch.full((B,), T), stop_target=stop).items()}


def _fill(static, src, lab, ids):
    """Rewrites the batch tensors `static` and the CUDA labels `lab` in place."""
    for k, v in src.items():
        static[k].copy_(v)
    lab.copy_(torch.tensor(ids))


class _Masks:
    """Records the encoder masks an eager step draws."""

    def __enter__(self):
        from multilingual_text_to_speech_b200.rng import MaskSource
        self.drawn, self.orig = {}, MaskSource.keep_mask.__func__

        def keep_mask(cls, key, shape, rate, device):
            m = self.orig(cls, key, shape, rate, device)
            if key.startswith('enc') and m is not None:
                self.drawn[key] = m.clone()
            return m
        MaskSource.keep_mask = classmethod(keep_mask)
        return self

    def __exit__(self, *exc):
        from multilingual_text_to_speech_b200.rng import MaskSource
        MaskSource.keep_mask = classmethod(self.orig)


def _eager(model, crit, bucket, b, ids, G, capacity):
    """One eager step in the [capacity, G*F, L] layout of `ids`, on the capture stream, inside given_layout."""
    from multilingual_text_to_speech_b200.graph import capture_stream
    from multilingual_text_to_speech_b200.modules.encoder import GroupLayout, given_layout
    counts, rows = GroupLayout(ids, G, capacity).device_tensors('cuda')
    side = capture_stream(torch.device('cuda:0'))
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side), given_layout((counts, rows, capacity)):
        bucket.zero()
        post, pre, stop, align, spk, enc = model(b['text'], b['text_length'], b['target'], b['target_length'], None, b['languages'], 1.0)
        loss, parts = crit(b['text_length'], b['target_length'], pre, b['target'], post, b['target'], stop, b['stop_target'], align,
                           None, spk, enc, None)
        loss.backward()
    torch.cuda.current_stream().wait_stream(side)
    torch.cuda.synchronize()
    return _snapshot(model, loss, parts, bucket)


def _snapshot(model, loss, parts, bucket):
    return {'loss': loss.detach().clone(), 'parts': {k: v.detach().clone() for k, v in parts.items()}, 'flat': bucket.flat.clone(),
            'state': {k: v.detach().clone() for k, v in model.state_dict().items()}}


def _assert_bitwise(got, want, what):
    assert torch.equal(got['loss'], want['loss']), f'{what}: loss {float(got["loss"])} != {float(want["loss"])}'
    assert got['parts'].keys() == want['parts'].keys()
    for k in want['parts']:
        assert torch.equal(got['parts'][k], want['parts'][k]), f'{what}: loss term {k}'
    diff = (got['flat'] != want['flat']).sum()
    assert int(diff) == 0, f'{what}: {int(diff)} gradient elements differ'
    for k in want['state']:
        assert torch.equal(got['state'][k], want['state'][k]), f'{what}: {k}'


def _assert_absent_untouched(model, before, ids, G, what):
    enc = model._encoder
    absent = [g for g in range(G) if g not in set(ids)]
    for name, p in enc.named_parameters():
        if name == '_embedding.weight':
            for g in absent:
                assert bool((p.grad[g] == 0).all()), f'{what}: absent language {g} has an embedding gradient'
        elif not hasattr(enc, '_embedding'):
            C = p.shape[0] // G
            for g in absent:
                assert bool((p.grad[g * C:(g + 1) * C] == 0).all()), f'{what}: absent language {g} has a gradient in {name}'
    for name, buf in enc.named_buffers():
        if 'running' in name:
            C = buf.shape[0] // G
            for g in absent:
                assert torch.equal(buf[g * C:(g + 1) * C], before['_encoder.' + name][g * C:(g + 1) * C]), \
                    f'{what}: running statistics {name} of absent language {g} moved'


@pytest.mark.parametrize('mode', ['fp32', 'bf16'])
@pytest.mark.parametrize('kind', ['generated', 'convolutional'])
@pytest.mark.parametrize('case', list(CASES))
def test_routed_replays_equal_eager_steps(case, kind, mode):
    from multilingual_text_to_speech_b200 import _lib
    from multilingual_text_to_speech_b200.graph import GraphedTrainStep
    from multilingual_text_to_speech_b200.rng import MaskSource
    overrides, capacity, L, T, patterns, oracle_pattern = CASES[case]
    hp, model, crit, bucket = _setup(kind, overrides)
    G = hp.language_number
    names = list(patterns)
    B = len(patterns[names[0]])
    src = {name: _batch(hp, B, L, T, 10 + j) for j, name in enumerate(names)}
    lab = torch.tensor(patterns[names[0]], device='cuda')
    static = {k: v.clone() for k, v in src[names[0]].items()}
    batch = dict(static, languages=lab, speakers=None)
    enc = model._encoder
    captured = {}

    def hook(mod, inp, out):          # at capture: static copies of the encoder's input, output and output gradient in the graph
        captured['x'] = inp[0].detach().clone()
        captured['out'] = out.detach().clone()
        out.register_hook(lambda gr: captured.__setitem__('dout', gr.detach().clone()))

    _lib.set_precision(mode)
    MaskSource.manual_seed(77)
    step = None
    try:
        handle = enc.register_forward_hook(hook)
        try:
            c0 = MaskSource.counter
            step = GraphedTrainStep(model, crit, bucket, batch, teacher_forcing=1.0, warmup=2, max_per_language=capacity)
        finally:
            handle.remove()
        assert step.routing is not None and step.routing.capacity == capacity
        per_body, rem = divmod(MaskSource.counter - c0, 3)          # 2 warm-up bodies + the capture
        assert rem == 0 and per_body > 0
        counter_at_capture = MaskSource.counter - per_body
        for j, name in enumerate(names):
            ids = patterns[name]
            cpu_labels = j == 0
            if cpu_labels:
                batch['languages'] = torch.tensor(ids)                  # CPU labels: read in place
            else:
                _fill(static, src[name], lab, ids)                      # CUDA labels rewritten in place: read again
                batch['languages'] = lab
            if j == 1:                                                  # over capacity, CPU and CUDA labels: refused before any write
                over = [0] * (capacity + 1) + [1 + g % (G - 1) for g in range(B - capacity - 1)]
                routing_before = step.routing.buffer.clone()
                static_before = {k: v.clone() for k, v in step.static.items() if v is not None}
                for labels in (torch.tensor(over), torch.tensor(over, device='cuda')):
                    with pytest.raises(ValueError, match=f'language 0 has {capacity + 1} utterances'):
                        step(dict(batch, languages=labels))
                torch.cuda.synchronize()
                assert torch.equal(step.routing.buffer, routing_before)
                for k, v in static_before.items():
                    assert torch.equal(step.static[k], v), k
            before = {k: v.detach().clone() for k, v in model.state_dict().items()}
            loss = step(batch)
            torch.cuda.synchronize()
            got = _snapshot(model, loss, step.parts, bucket)
            enc_grads = {k: p.grad.detach().clone() for k, p in enc.named_parameters()}
            _assert_absent_untouched(model, before, ids, G, f'{case} {kind} {mode} {name}')
            if name == oracle_pattern:
                x, out, dout = captured['x'].clone(), captured['out'].clone(), captured['dout'].clone()
            # the eager step from the same state, at the replay's mask counters and epoch
            with torch.no_grad():
                model.load_state_dict(before)
            if name == oracle_pattern:
                enc_before = {k: v.detach().cpu().clone() for k, v in enc.named_buffers()}
            epoch = int(step.epoch)
            MaskSource.counter = counter_at_capture
            step.epoch.fill_(epoch)
            with _Masks() as masks:
                want = _eager(model, crit, bucket, dict(batch, languages=torch.tensor(ids, device='cuda')), ids, G, capacity)
            _assert_bitwise(got, want, f'{case} {kind} {mode} {name}')
            assert all(m.shape[0] == capacity for m in masks.drawn.values())
            if name == oracle_pattern:
                with torch.no_grad():
                    for k, v in enc.named_buffers():
                        v.copy_(enc_before[k])
                oracle = RO.encode(enc, x, ids, {k: v.cpu() for k, v in masks.drawn.items()}, True, dout, device='cuda')
                with torch.no_grad():
                    for k, v in enc.named_buffers():
                        v.copy_(got['state']['_encoder.' + k])
                worst = _compare(enc, out, enc_grads, enc_before, *oracle, ids, mode, f'{case} {kind} {mode} {name} vs oracle')
                print(case, kind, mode, name, f'worst relative encoder gradient error {worst:.3e}')
            print(case, kind, mode, name, f'loss {float(got["loss"]):.6f} bitwise equal to the eager step')
    finally:
        _lib.set_precision('fp32')
        if step is not None:
            step.close()


def _graph_nodes(graph):
    cuda = ctypes.CDLL('libcuda.so.1')
    n = ctypes.c_size_t(0)
    assert cuda.cuGraphGetNodes(ctypes.c_void_p(graph.raw_cuda_graph()), None, ctypes.byref(n)) == 0
    return n.value


@pytest.mark.parametrize('mode', ['fp32', 'bf16'])
@pytest.mark.parametrize('kind', ['generated', 'convolutional'])
def test_reference_layout_capture_is_the_reference_step(kind, mode, monkeypatch):
    """A reference-layout example without max_per_language: no routing, and the captured graph is the step body captured under
    reference_layout() (what GraphedTrainStep captured before routed graphs existed): as many nodes, and the same bits."""
    from multilingual_text_to_speech_b200 import _lib
    from multilingual_text_to_speech_b200.graph import GraphedTrainStep, capture_stream
    from multilingual_text_to_speech_b200.modules.encoder import reference_layout
    from multilingual_text_to_speech_b200.rng import MaskSource
    hp, model, crit, bucket = _setup(kind, SMALL)
    real_graph = torch.cuda.CUDAGraph
    G, B = hp.language_number, 12
    batch = dict(_batch(hp, B, 16, 12, 3), languages=torch.tensor([b % G for b in range(B)], device='cuda'), speakers=None)
    _lib.set_precision(mode)
    MaskSource.manual_seed(5)
    step = None
    try:
        c0 = MaskSource.counter
        with monkeypatch.context() as m:         # keep the captured cudaGraph_t to count its nodes (instantiated at the first replay)
            m.setattr(torch.cuda, 'CUDAGraph', lambda: real_graph(keep_graph=True))
            step = GraphedTrainStep(model, crit, bucket, batch, teacher_forcing=1.0, warmup=2)
        assert step.routing is None
        counter_at_capture = MaskSource.counter - (MaskSource.counter - c0) // 3
        before = {k: v.detach().clone() for k, v in model.state_dict().items()}
        loss = step(batch)
        torch.cuda.synchronize()
        got = _snapshot(model, loss, step.parts, bucket)
        epoch = int(step.epoch)
        graph = step.graph
        plain = torch.cuda.CUDAGraph(keep_graph=True)
        side = capture_stream(torch.device('cuda:0'))
        MaskSource.counter = counter_at_capture
        with torch.cuda.graph(plain, stream=side), reference_layout():
            step._body()
        torch.cuda.synchronize()
        assert _graph_nodes(graph) == _graph_nodes(plain), (_graph_nodes(graph), _graph_nodes(plain))
        with torch.no_grad():
            model.load_state_dict(before)
        step.epoch.fill_(epoch - 1)
        plain.replay()
        torch.cuda.synchronize()
        _assert_bitwise(got, _snapshot(model, step.loss, step.parts, bucket), f'{kind} {mode} reference layout')
        print(kind, mode, f'reference-layout capture: {_graph_nodes(graph)} graph nodes')
    finally:
        _lib.set_precision('fp32')
        if step is not None:
            step.close()
