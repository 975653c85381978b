"""WaveRNN training from a device-resident corpus on the GPU:
  1. VocoderCorpus.batch against vocoder_batch moved to the device, bit for bit (x, y, m): RAW at 9 and 16 bits and MOL, ragged utterances
     (one just long enough for a window), offsets 0 and the largest allowed, B in {1, 7, 64}; outputs NaN-poisoned beforehand, inputs
     unchanged, two calls bitwise equal;
  2. GraphedVocoderStep against the eager step bit for bit over six steps with a new (ids, offsets) table each step and FusedAdam between
     steps in both arms: the loss, the whole gradient bucket, every buffer (batch-norm running statistics, num_batches_tracked, `step`) and
     the parameters after the last step; RAW and MOL, fp32 and bf16 mode.  The eager step is bitwise reproducible (no float atomics), so
     any difference is a defect;
  3. a captured step called under another precision mode raises;
  4. a one-rank torch.distributed (NCCL) run through bucket.allreduce() gives the non-distributed result."""
import numpy as np
import pytest
import torch

from multilingual_text_to_speech_b200 import _lib
from multilingual_text_to_speech_b200.distributed import GradBucket
from multilingual_text_to_speech_b200.graph import GraphedVocoderStep
from multilingual_text_to_speech_b200.modules.wavernn import VocoderCorpus, WaveRNN, mel_window, vocoder_batch, wavernn_loss
from multilingual_text_to_speech_b200.optim import FlatParams, FusedAdam

pytestmark = pytest.mark.gpu

HOP, PAD = 275, 2
DIMS = dict(rnn_dims=512, fc_dims=512, pad=PAD, upsample_factors=(5, 5, 11), feat_dims=80, compute_dims=128, res_out_dims=128,
            res_blocks=10, hop_length=HOP, sample_rate=22050)


@pytest.fixture(autouse=True)
def fp32_mode():
    _lib.set_precision('fp32')
    yield
    _lib.set_precision('fp32')


def make_corpus_data(n, label_max, seq_len, seed=0):
    """Ragged utterances; utterance 0 is just long enough for one window (mel and labels both end where the window does)."""
    rng = np.random.default_rng(seed)
    win = mel_window(seq_len, HOP, PAD)
    frames = [win] + [int(f) for f in rng.integers(win + 8, win + 60, n - 1)]
    mels = [rng.standard_normal((80, f)) for f in frames]          # float64: rounded to fp32 by both paths
    labels = [rng.integers(0, label_max, (PAD * HOP + seq_len + 1) if i == 0 else f * HOP + int(rng.integers(0, HOP)))
              for i, f in enumerate(frames)]
    labels[1][::7] = 0
    labels[1][1::11] = label_max - 1
    return mels, labels


def max_offset(frames, samples, seq_len):
    win = mel_window(seq_len, HOP, PAD)
    return min(frames - win, (samples - seq_len - 1) // HOP - PAD)


@pytest.mark.parametrize('mode,bits', [('RAW', 9), ('RAW', 16), ('MOL', 9)])
@pytest.mark.parametrize('B', [1, 7, 64])
def test_corpus_batch_equals_vocoder_batch(mode, bits, B):
    seq_len = 1375
    mels, labels = make_corpus_data(23, 2 ** (16 if mode == 'MOL' else bits), seq_len, seed=B)
    corpus = VocoderCorpus(mels, labels, mode, bits, seq_len, PAD, HOP, 'cuda')
    before = (corpus.mels.clone(), corpus.labels.clone())
    rng = np.random.default_rng(B + 1)
    ids = [int(u) for u in rng.integers(0, len(mels), B)]
    ids[0] = 0                                                   # the utterance just long enough
    hi = [max_offset(corpus.frames[u], corpus.samples[u], seq_len) for u in ids]
    offsets = [int(rng.integers(0, h + 1)) for h in hi]
    offsets[0] = 0
    if B > 1:
        offsets[-1] = hi[-1]                                    # the largest allowed offset
    x0, y0, m0 = vocoder_batch([mels[u] for u in ids], [labels[u] for u in ids], offsets, mode, bits, seq_len, PAD, HOP)
    poisoned = (torch.full(tuple(x0.shape), float('nan'), device='cuda'),
                torch.full(tuple(y0.shape), float('nan'), device='cuda') if mode == 'MOL' else
                torch.full(tuple(y0.shape), -7, dtype=torch.int64, device='cuda'),
                torch.full(tuple(m0.shape), float('nan'), device='cuda'))
    table = torch.from_numpy(corpus.table(ids, offsets)).cuda()
    x, y, m = corpus.cut(table, poisoned)
    x2, y2, m2 = corpus.batch(ids, offsets)
    torch.cuda.synchronize()
    for got, again, ref in ((x, x2, x0), (y, y2, y0), (m, m2, m0)):
        assert got.dtype == ref.dtype and tuple(got.shape) == tuple(ref.shape)
        assert torch.equal(got.cpu(), ref), (mode, bits, B)
        assert torch.equal(again, got)
    assert torch.equal(corpus.mels, before[0]) and torch.equal(corpus.labels, before[1])


def make_model(mode, seed=0):
    torch.manual_seed(seed)
    m = WaveRNN(**DIMS, bits=9, mode=mode)
    with torch.no_grad():
        for name, p in m.named_parameters():
            if 'batch_norm' in name:
                p.copy_(1 + 0.1 * torch.randn_like(p) if name.endswith('weight') else 0.1 * torch.randn_like(p))
    return m.cuda().train()


def make_arm(mode):
    model = make_model(mode)
    flat, bucket = FlatParams(model), GradBucket(model)
    return model, bucket, FusedAdam(flat, bucket, lr=1e-4, max_grad_norm=4.0)


def tables(corpus, steps, B, seed=5):
    rng = np.random.default_rng(seed)
    out = []
    for _ in range(steps):
        ids = [int(u) for u in rng.integers(1, len(corpus), B)]
        out.append((ids, corpus.draw_offsets(ids, rng)))
    return out


@pytest.mark.parametrize('precision', ['fp32', 'bf16'])
@pytest.mark.parametrize('mode', ['RAW', 'MOL'])
def test_graphed_step_equals_eager_step(mode, precision):
    _lib.set_precision(precision)
    B, seq_len, steps = 8, 1375, 6
    mels, labels = make_corpus_data(17, 512 if mode == 'RAW' else 65536, seq_len, seed=3)
    corpus = VocoderCorpus(mels, labels, mode, 9, seq_len, PAD, HOP, 'cuda')
    eager_model, eager_bucket, eager_opt = make_arm(mode)
    graph_model, graph_bucket, graph_opt = make_arm(mode)
    step = GraphedVocoderStep(graph_model, graph_bucket, corpus, B)
    for k, v in graph_model.named_buffers():                       # constructing the step leaves the buffers as they were
        assert torch.equal(v, dict(eager_model.named_buffers())[k]), k
    for i, (ids, offsets) in enumerate(tables(corpus, steps, B)):
        eager_bucket.zero()
        x, y, m = corpus.batch(ids, offsets)
        loss_e = wavernn_loss(eager_model(x, m), y, mode)
        loss_e.backward()
        eager_opt.step()
        loss_g = step(ids, offsets).clone()
        grad_g = graph_bucket.flat.clone()
        graph_opt.step()
        torch.cuda.synchronize()
        assert torch.equal(loss_g, loss_e.detach()), (i, float(loss_g), float(loss_e))
        assert torch.equal(grad_g, eager_bucket.flat), i
        for (k, a), (_, b) in zip(graph_model.named_buffers(), eager_model.named_buffers()):
            assert torch.equal(a, b), (i, k)
    step.close()
    assert int(graph_model.step) == steps
    for (k, a), (_, b) in zip(graph_model.named_parameters(), eager_model.named_parameters()):
        assert torch.equal(a, b), k


def test_graphed_step_refuses_another_precision_mode():
    mels, labels = make_corpus_data(5, 512, 275, seed=4)
    corpus = VocoderCorpus(mels, labels, 'RAW', 9, 275, PAD, HOP, 'cuda')
    model, bucket, _ = make_arm('RAW')
    step = GraphedVocoderStep(model, bucket, corpus, 2, warmup=1)
    step([1, 2], [0, 0])
    _lib.set_precision('bf16')
    with pytest.raises(ValueError, match='fp32 mode'):
        step([1, 2], [0, 0])
    _lib.set_precision('fp32')
    step.close()


def test_one_rank_distributed_equals_plain(tmp_path):
    import torch.distributed as dist
    mels, labels = make_corpus_data(9, 512, 1375, seed=6)
    corpus = VocoderCorpus(mels, labels, 'RAW', 9, 1375, PAD, HOP, 'cuda')
    plan = tables(corpus, 3, 4, seed=7)
    results = []
    for distributed in (False, True):
        if distributed:
            dist.init_process_group('nccl', init_method=f'file://{tmp_path}/pg', rank=0, world_size=1, device_id=torch.device('cuda', 0))
        try:
            model, bucket, opt = make_arm('RAW')
            step = GraphedVocoderStep(model, bucket, corpus, 4, warmup=1)
            for ids, offsets in plan:
                step(ids, offsets)
                bucket.allreduce()
                opt.step()
            step.close()
            torch.cuda.synchronize()
            results.append((bucket.flat.clone(), [p.detach().clone() for p in model.parameters()]))
        finally:
            if distributed:
                dist.destroy_process_group()
    assert torch.equal(results[0][0], results[1][0])
    assert all(torch.equal(a, b) for a, b in zip(results[0][1], results[1][1]))
