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
    bucket.allreduce(); optimizer.step()

A grouped encoder (ConvolutionalEncoder / GeneratedConvolutionalEncoder) routes each utterance to its own language's channel block
(modules/encoder.py GroupLayout).  An example batch in the reference layout (utterance b of language b % G) is captured as that reshape,
and its replays read no labels.  With `max_per_language` the step is captured in the routed layout at that fixed capacity of rows
per language; each call then builds the batch's GroupLayout on the host and copies its counts and rows into static device buffers
before the replay, so one graph serves every language pattern within the capacity (StaticRouting).  An example batch outside the
reference layout needs that capacity: without `max_per_language` it is refused.
"""
import ctypes

import torch

from . import _lib
from . import functional as F
from .modules.encoder import ConvolutionalEncoder, GeneratedConvolutionalEncoder, GroupLayout, encoder_layout, given_layout, language_ids


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


class StaticRouting:
    """The routing of a graph captured in the routed layout [capacity, G*F, L]: counts int32 [G] and rows int64 [B] (GroupLayout.counts
    and rows()) in one static int32 buffer on the device, refilled from each batch's labels before its replay.

    `layout(x_langs)` reads the labels and checks them without touching the buffer: CPU labels are read in place with no device
    synchronisation; CUDA labels cost one device-to-host copy of B ints, which waits for the work queued before it on the stream (the
    same read an eager routed step makes).  `load(layout)` fills the buffer with one host-to-device copy from pinned memory."""

    def __init__(self, groups, batch, capacity, device):
        pad = groups + groups % 2             # rows start 8-byte aligned
        self.groups, self.batch, self.capacity = groups, batch, capacity
        self.buffer = torch.zeros(pad + 2 * batch, dtype=torch.int32, device=device)
        self.counts, self.rows = self.buffer[:groups], self.buffer[pad:].view(torch.int64)

    def layout(self, x_langs):
        ids = language_ids(x_langs)
        if len(ids) != self.batch:
            raise ValueError(f'language labels for {len(ids)} utterances given for a graph captured at a batch of {self.batch}')
        return GroupLayout(ids, self.groups, self.capacity)

    def load(self, layout):
        pad = self.buffer.numel() - 2 * self.batch
        host = torch.cat((torch.tensor(layout.counts + [0] * (pad - self.groups), dtype=torch.int32),
                          torch.tensor(layout.rows(), dtype=torch.int64).view(torch.int32)))
        if self.buffer.is_cuda:
            host = host.pin_memory()
        self.buffer.copy_(host, non_blocking=True)

    def given(self):
        """The (counts, rows, capacity) routing of modules.encoder.given_layout."""
        return self.counts, self.rows, self.capacity


def _static_routing(model, batch, max_per_language, device):
    """None when the step is captured as the reference reshape (no grouped encoder, no labels, or no `max_per_language` and an example
    batch that the encoders run unrouted), else the StaticRouting at capacity `max_per_language`.  The capacity fixes the encoder's
    work and the batches a graph accepts, so it is never guessed from one example batch: a routed example without it is refused."""
    groups = [m._groups for m in model.modules() if isinstance(m, (ConvolutionalEncoder, GeneratedConvolutionalEncoder)) and m._groups > 1]
    langs = batch.get('languages')
    if not groups or langs is None:
        return None
    G, B = groups[0], batch['text'].shape[0]
    if max_per_language is None:
        if encoder_layout(langs, B, G) is None:
            return None
        n_max = GroupLayout(language_ids(langs), G).n_max
        raise ValueError('GraphedTrainStep captures grouped-encoder batches outside the reference layout (B divisible by the '
                         f'{G} languages and utterance b of language b % {G}) only at a fixed capacity of utterances per language: '
                         f'pass max_per_language, the most utterances of one language any batch of this shape will have (the example '
                         f'batch has {n_max}).  The encoder then runs {G} x max_per_language rows per step')
    if int(max_per_language) < 1:
        raise ValueError(f'max_per_language must be at least 1 (got {max_per_language})')
    return StaticRouting(G, B, int(max_per_language), device)


class GraphedTrainStep:
    FIELDS = ('text', 'text_length', 'target', 'target_length', 'stop_target', 'speakers', 'languages')

    def __init__(self, model, criterion, bucket, example_batch, teacher_forcing=1.0, warmup=3, max_per_language=None):
        """max_per_language: the capacity, in utterances per language, of the routed layout a grouped encoder is captured in (see the
        module docstring); a batch with more utterances of one language raises ValueError, the example batch included.  Balanced
        samplers (PerfectBatchSampler, BucketedPerfectBatchSampler, shard) give ceil(B / G); imbalanced ones (RandomImbalancedSampler)
        need a bound.  None: the example batch must be in the reference layout, and is captured as the reference's reshape.  Ignored
        without a grouped encoder."""
        if float(teacher_forcing) < 1.0:
            # the per-step teacher-forcing coins are drawn on the host and decide which kernels a decode launches: one captured graph
            # would replay one frozen coin pattern at every step.  Run such steps eagerly (the backward supports them).
            raise ValueError(f'GraphedTrainStep needs teacher_forcing = 1.0 (got {teacher_forcing}): a CUDA graph would replay one fixed '
                             'pattern of free-running steps; run steps with teacher forcing below 1.0 eagerly')
        dev = next(model.parameters()).device
        self.routing = _static_routing(model, example_batch, max_per_language, dev)
        if self.routing is not None:
            self.routing.load(self.routing.layout(example_batch['languages']))
        given = None if self.routing is None else self.routing.given()
        self.model, self.criterion, self.bucket, self.tf = model, criterion, bucket, float(teacher_forcing)
        self.static = {k: (example_batch[k].to(dev).clone() if example_batch.get(k) is not None else None) for k in self.FIELDS}
        self.epoch = torch.zeros(1, dtype=torch.int64, device=dev)
        _lib.check(_lib.load().b200tts_set_mask_epoch(ctypes.c_void_p(self.epoch.data_ptr())), 'b200tts_set_mask_epoch')
        self.loss, self.parts = None, None
        side = capture_stream(dev)
        side.wait_stream(torch.cuda.current_stream(dev))
        with torch.cuda.stream(side), given_layout(given):   # warm-up on a side stream (workspaces, lazy attribute settings, pack caches)
            for _ in range(warmup):
                self._body()
        torch.cuda.current_stream(dev).wait_stream(side)
        torch.cuda.synchronize(dev)
        # capture on the SAME side stream the warm-up ran on: autograd's AccumulateGrad nodes are bound to the stream their parameter was first
        # used on, and the engine joins every such "leaf stream" at the end of backward -- a leaf stream that is not the capture stream would
        # be a dependency on uncaptured work as soon as a step sends it no gradient (the library accumulates most gradients in place)
        self.graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(self.graph, stream=side), given_layout(given):
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
        """Copies the batch into the static buffers and replays.  A routed graph first reads the batch's labels (StaticRouting.layout:
        a batch over the capacity raises ValueError before any static buffer is written) and copies its counts and rows in."""
        if self.routing is not None:
            self.routing.load(self.routing.layout(batch['languages']))
        for k in self.FIELDS:
            dst = self.static[k]
            if dst is not None:
                dst.copy_(batch[k], non_blocking=True)
        self.graph.replay()
        return self.loss

    def close(self):
        _lib.check(_lib.load().b200tts_set_mask_epoch(None), 'b200tts_set_mask_epoch')


class DeferredAbortCheck:
    """The GRU loops' abort flag of a captured vocoder step, read after the replay instead of inside it (a read inside would synchronise).

    After each replay `after_replay(n)` enqueues an asynchronous copy of the flag into a host slot and records an event.  `poll()` (at the
    next call) reads, oldest first, every copied flag whose event has completed, without waiting; `wait()` (check() and close()) waits for
    all of them.  A set flag raises B200TTSError naming its replay.  At most `depth` flags are outstanding: the replay after that waits for
    the oldest copy, which keeps the host at most `depth` replays ahead of the device.

    copy_flag(slot) enqueues the copy into `slot` (int32 [1]); new_event() returns an object with record(), query() and synchronize()
    (torch.cuda.Event on the device; a stand-in in the host tests)."""

    def __init__(self, copy_flag, new_event, depth=4, pin=True):
        from collections import deque
        self._copy, self._new_event, self.depth = copy_flag, new_event, int(depth)
        self._free = [torch.zeros(1, dtype=torch.int32, pin_memory=pin) for _ in range(self.depth)]
        self._pending = deque()

    def after_replay(self, replay):
        while len(self._pending) >= self.depth:
            self._pending[0][2].synchronize()
            self._read_oldest()
        slot = self._free.pop()
        self._copy(slot)
        ev = self._new_event()
        ev.record()
        self._pending.append((replay, slot, ev))

    def poll(self):
        while self._pending and self._pending[0][2].query():
            self._read_oldest()

    def wait(self):
        while self._pending:
            self._pending[0][2].synchronize()
            self._read_oldest()

    def _read_oldest(self):
        replay, slot, _ = self._pending.popleft()
        flag = int(slot[0])
        slot.zero_()
        self._free.append(slot)
        if flag:
            raise _lib.B200TTSError(f'GraphedVocoderStep: a GRU loop of replay {replay} timed out at a grid barrier')


class GraphedVocoderStep:
    """One WaveRNN training step as ONE CUDA graph: the windows cut from a device-resident corpus (modules.wavernn.VocoderCorpus),
    WaveRNN.forward, wavernn_loss and the backward into the flat gradient bucket.  The optimizer step stays outside the graph
    (FusedAdam takes the learning rate and the step count by value), as does the all-reduce of a data-parallel run:

        step = GraphedVocoderStep(model, bucket, corpus, batch_size)     # warm-up + capture on capture_stream(device)
        loss = step(ids, offsets)     # host-validated table -> static device table (one pinned copy), replay; loss: a device tensor
        bucket.allreduce(); optimizer.step()

    A call does not synchronise.  The GRU loops' abort flag (a grid-barrier timeout) is zeroed inside the graph, copied to pinned host memory
    after each replay and read by a later call, check() or close() (DeferredAbortCheck), which raise B200TTSError naming the replay.
    The batch-norm running statistics, num_batches_tracked and the model's `step` buffer are updated inside the graph, as an eager step
    updates them; the warm-up's updates are rolled back, so constructing the step leaves the model's buffers as they were.  The precision
    mode is fixed at capture: a call under another mode raises ValueError.  As with GraphedTrainStep, eager steps that precede the capture
    on the same model should run on capture_stream(device)."""

    def __init__(self, model, bucket, corpus, batch_size, warmup=3, abort_depth=4):
        from .modules.wavernn import MAX_TRAIN_BATCH
        B = int(batch_size)
        if not 1 <= B <= MAX_TRAIN_BATCH:
            raise ValueError(f'batch_size {batch_size}: need 1 to {MAX_TRAIN_BATCH} windows per step')
        n_classes = 2 ** corpus.bits if corpus.mode == 'RAW' else model.n_classes
        if (corpus.mode, corpus.hop, corpus.pad, corpus.feat, n_classes) != (model.mode, model.hop_length, model.pad, model.feat_dims,
                                                                           model.n_classes):
            raise ValueError(f'corpus (mode {corpus.mode}, hop {corpus.hop}, pad {corpus.pad}, {corpus.feat} mel channels, bits '
                             f'{corpus.bits}) does not match the model (mode {model.mode}, hop {model.hop_length}, pad {model.pad}, '
                             f'{model.feat_dims} mel channels, {model.n_classes} classes)')
        first = next((u for u in range(len(corpus)) if corpus.labels_ok[u] and corpus.win <= corpus.frames[u]
                      and corpus.pad * corpus.hop + corpus.seq_len + 1 <= corpus.samples[u]), None)
        if first is None:
            raise ValueError('the corpus has no utterance long enough for one window')
        dev = corpus.device
        self.model, self.bucket, self.corpus, self.batch_size = model, bucket, corpus, B
        self.precision = _lib.get_precision()
        self.table = torch.from_numpy(corpus.table([first] * B, [0] * B)).to(dev)
        self.loss = None
        self.replays = 0
        saved = {k: v.clone() for k, v in model.named_buffers()}
        side = capture_stream(dev)
        side.wait_stream(torch.cuda.current_stream(dev))
        with torch.cuda.stream(side):
            for _ in range(warmup):
                self._body()
        torch.cuda.current_stream(dev).wait_stream(side)
        torch.cuda.synchronize(dev)
        with torch.no_grad():
            for k, v in model.named_buffers():
                v.copy_(saved[k])
        torch.cuda.synchronize(dev)
        model._graph_guard = None
        self.graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(self.graph, stream=side):
            self._body()
        torch.cuda.synchronize(dev)
        self.guard, model._graph_guard = model._graph_guard, None
        if self.guard is None:
            raise _lib.B200TTSError('GraphedVocoderStep: the captured forward left no GRU loop guard')
        self.abort = DeferredAbortCheck(lambda slot: F.gru_seq_abort_flag_copy(self.guard, slot), torch.cuda.Event, abort_depth)

    def _body(self):
        from .modules.wavernn import wavernn_loss
        self.bucket.zero()
        x, y, m = self.corpus.cut(self.table)
        self.loss = wavernn_loss(self.model(x, m), y, self.model.mode)
        self.loss.backward()

    def __call__(self, ids, offsets):
        """Validates the (ids, offsets) table on the host (VocoderCorpus.table), reads the flags of earlier replays that have completed,
        copies the table in and replays.  Returns the loss, a device tensor the next replay overwrites."""
        table = self.corpus.table(ids, offsets)
        if len(table) != self.batch_size:
            raise ValueError(f'{len(table)} windows for a step captured at a batch of {self.batch_size}')
        mode = _lib.get_precision()
        if mode != self.precision:
            raise ValueError(f'GraphedVocoderStep was captured in {self.precision} mode; the precision mode is now {mode}')
        self.abort.poll()
        self.table.copy_(torch.from_numpy(table).pin_memory(), non_blocking=True)
        self.graph.replay()
        self.replays += 1
        self.abort.after_replay(self.replays)
        return self.loss

    def check(self):
        """Waits for every replay's abort flag and raises B200TTSError if one is set."""
        self.abort.wait()

    def close(self):
        self.check()
