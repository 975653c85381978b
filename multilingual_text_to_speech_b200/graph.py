"""A whole training step (forward + TacotronLoss + backward into the flat gradient bucket) as ONE CUDA graph.

The step of the bf16 mode is ~1200 kernel launches issued from Python; between them the GPU idles for milliseconds per step depending on the
host.  Every library call only enqueues work on the current stream (no allocation, no synchronisation, host
arguments read at enqueue time), so the step can be captured once and replayed: the launch overhead disappears and the step time becomes
the sum of its kernels.  Static shapes are the contract (one graph per batch shape -- bucketed batches, utils/samplers.py, keep the number
of shapes small); dropout masks stay fresh because the graph increments a device-side epoch that the mask generator mixes into its keys
(b200tts_set_mask_epoch).

    step = GraphedTrainStep(model, criterion, bucket, example_batch)     # warm-up + capture (drop every reference to an autograd graph
                                                                         # built before: its AccumulateGrad nodes are bound to ITS stream)
    loss = step(batch)            # copies the batch into the static input buffers, replays, returns the (static) loss tensor
                                  # (batches of the captured shape and layout: a grouped encoder's batch in the reference layout,
                                  # utterance b of language b % G, which the constructor checks on the example batch)
    bucket.allreduce(); optimizer.step()
"""
import ctypes

import torch

from . import _lib
from .modules.encoder import ConvolutionalEncoder, GeneratedConvolutionalEncoder, encoder_layout, language_ids, reference_layout


_CAPTURE_STREAMS = {}


def capture_stream(device):
    """THE side stream (one per device, shared by every GraphedTrainStep) that warm-ups and captures run on.  autograd binds a parameter's
    AccumulateGrad node to the stream the parameter was first used on and keeps it for the life of the parameter; capturing on any other
    stream makes that node a cross-stream consumer, which CUDA rejects (cudaErrorStreamCaptureIsolation) as soon as one backward sends it
    no gradient -- and the library accumulates most gradients in place (functional._grad_targets).  So: one stream for all captures, and
    eager steps that precede the first capture should run under `torch.cuda.stream(capture_stream(device))` as well."""
    dev = torch.device(device)
    key = dev.index if dev.index is not None else torch.cuda.current_device()
    if key not in _CAPTURE_STREAMS:
        _CAPTURE_STREAMS[key] = torch.cuda.Stream(device=dev)
    return _CAPTURE_STREAMS[key]


def _require_reference_layout(model, batch):
    """A grouped encoder routes a batch by reading its language labels, a device-to-host copy that a capture cannot contain.  The layout
    is decided here, from the example batch, before capture: the captured step runs the reference layout (utterance b under language
    b % G) without reading labels, and any other example batch is refused."""
    langs = batch.get('languages')
    for m in model.modules():
        if isinstance(m, (ConvolutionalEncoder, GeneratedConvolutionalEncoder)) and encoder_layout(langs, batch['text'].shape[0], m._groups):
            raise ValueError('GraphedTrainStep captures grouped-encoder batches in the reference layout only (B divisible by the '
                             f'{m._groups} languages and utterance b of language b % {m._groups}); the example batch has languages '
                             f'{language_ids(langs)}.  Run such batches eagerly: the encoder routes them by their labels')


class GraphedTrainStep:
    FIELDS = ('text', 'text_length', 'target', 'target_length', 'stop_target', 'speakers', 'languages')

    def __init__(self, model, criterion, bucket, example_batch, teacher_forcing=1.0, warmup=3):
        if float(teacher_forcing) < 1.0:
            # the per-step teacher-forcing coins are drawn on the host and decide which kernels a decode launches: one captured graph
            # would replay one frozen coin pattern at every step.  Run such steps eagerly (the backward supports them).
            raise ValueError(f'GraphedTrainStep needs teacher_forcing = 1.0 (got {teacher_forcing}): a CUDA graph would replay one fixed '
                             'pattern of free-running steps; run steps with teacher forcing below 1.0 eagerly')
        _require_reference_layout(model, example_batch)
        self.model, self.criterion, self.bucket, self.tf = model, criterion, bucket, float(teacher_forcing)
        dev = next(model.parameters()).device
        self.static = {k: (example_batch[k].to(dev).clone() if example_batch.get(k) is not None else None) for k in self.FIELDS}
        self.epoch = torch.zeros(1, dtype=torch.int64, device=dev)
        _lib.check(_lib.load().b200tts_set_mask_epoch(ctypes.c_void_p(self.epoch.data_ptr())), 'b200tts_set_mask_epoch')
        self.loss, self.parts = None, None
        side = capture_stream(dev)
        side.wait_stream(torch.cuda.current_stream(dev))
        with torch.cuda.stream(side), reference_layout():   # warm-up on a side stream (workspaces, lazy attribute settings, pack caches)
            for _ in range(warmup):
                self._body()
        torch.cuda.current_stream(dev).wait_stream(side)
        torch.cuda.synchronize(dev)
        # capture on the SAME side stream the warm-up ran on: autograd's AccumulateGrad nodes are bound to the stream their parameter was first
        # used on, and the engine joins every such "leaf stream" at the end of backward -- a leaf stream that is not the capture stream would
        # be a dependency on uncaptured work as soon as a step sends it no gradient (the library accumulates most gradients in place)
        self.graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(self.graph, stream=side), reference_layout():
            self._body()
        torch.cuda.synchronize(dev)

    def _body(self):
        b = self.static
        self.epoch.add_(1)
        self.bucket.zero()
        post, pre, stop, align, spk, enc = self.model(b['text'], b['text_length'], b['target'], b['target_length'], b['speakers'], b['languages'],
                                                      self.tf)
        self.loss, self.parts = self.criterion(b['text_length'], b['target_length'], pre, b['target'], post, b['target'], stop, b['stop_target'],
                                               align, b['speakers'], spk, enc, None)
        self.loss.backward()

    def __call__(self, batch):
        for k in self.FIELDS:
            dst = self.static[k]
            if dst is not None:
                dst.copy_(batch[k], non_blocking=True)
        self.graph.replay()
        return self.loss

    def close(self):
        _lib.check(_lib.load().b200tts_set_mask_epoch(None), 'b200tts_set_mask_epoch')
