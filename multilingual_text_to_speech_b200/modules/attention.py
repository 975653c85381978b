"""Attention modules (surface of reference modules/attention.py:6-124).

LocationSensitiveAttention (the default, hp.attention_type "location_sensitive") and ForwardAttention ("forward") are provided.
Inside training both run fused in the decoder op; the module-level `reset` / `forward` API is kept and calls the library's
single-step ops.  ForwardAttentionWithTransition ("forward_transition_agent") is not: the reference cannot run it (its `reset`
takes three arguments, the decoder passes four), so there is no behaviour to match.
"""
import torch
from torch.nn import Linear, Parameter, Conv1d

from .. import functional as F


class AttentionBase(torch.nn.Module):
    def __init__(self, representation_dim, query_dim, memory_dim):
        super().__init__()
        self._bias = Parameter(torch.zeros(1, representation_dim))
        self._energy = Linear(representation_dim, 1, bias=False)
        self._query = Linear(query_dim, representation_dim, bias=False)
        self._memory = Linear(memory_dim, representation_dim, bias=False)
        self._memory_dim = memory_dim

    def reset(self, encoded_input, batch_size, max_len, device):
        """Prepare the memory projection and zero the cumulative weights / context (attention.py:23-28)."""
        self._memory_transform = F.linear(encoded_input, self._memory.weight)
        self._prev_weights = torch.zeros(batch_size, max_len, device=device)
        self._prev_context = torch.zeros(batch_size, self._memory_dim, device=device)
        return self._prev_context


class LocationSensitiveAttention(AttentionBase):
    """attention.py:48-86 (softmax normalisation; the `smoothing` branch is never enabled by the model)."""

    def __init__(self, kernel_size, channels, smoothing, representation_dim, query_dim, memory_dim):
        super().__init__(representation_dim, query_dim, memory_dim)
        assert not smoothing, 'sigmoid smoothing is not used by any configuration'
        self._location = Linear(channels, representation_dim, bias=False)
        self._loc_features = Conv1d(1, channels, kernel_size, padding=(kernel_size - 1) // 2, bias=False)
        self._smoothing = smoothing

    def forward(self, query, memory, mask, prev_decoder_output):
        """(context, weights) for one decoder step (attention.py:39-45); the module state (`_prev_weights`, `_prev_context`) advances as
        in the reference and carries autograd history: gradients flow to the query, the memory, the memory projection and every
        attention parameter through the library's single-step backward.  (Training inside `Decoder` uses the fused op instead.)"""
        lengths = mask.sum(dim=1).to(torch.int32)
        ctx, w, cum = F.AttentionStepFunction.apply(query, memory, self._memory_transform, self._prev_weights, lengths, self._query.weight,
                                                    self._location.weight, self._loc_features.weight, self._bias, self._energy.weight)
        self._prev_weights = cum
        self._prev_context = ctx
        return ctx, w


class ForwardAttention(AttentionBase):
    """Forward attention without the transition agent (attention.py:89-124, https://arxiv.org/abs/1807.06736).

    Per step: s = softmax(v . tanh(W_q h + memT + b)) over every position (padding included, as in the reference);
    a = (alpha + alpha shifted right by one) * s; a = 0 beyond the text length; w = clamp(a, 1e-6) normalised to sum 1.
    w is the alignment and the next alpha; the context is w . memory over every position.  So unlike the location-sensitive
    attention, the alignments are not exactly zero beyond the text length (they are about 1e-6 / sum there)."""

    def reset(self, encoded_input, batch_size, max_len, device):
        """AttentionBase.reset, then alpha[:, 0] = 1 (attention.py:103-106)."""
        super().reset(encoded_input, batch_size, max_len, device)
        self._prev_weights[:, 0] = 1
        return self._prev_context

    def forward(self, query, memory, mask, prev_decoder_output):
        """(context, weights) for one decoder step; `prev_decoder_output` is unused, as in the reference.  The new alpha (= weights)
        replaces `_prev_weights` with autograd history through the library's single-step backward."""
        lengths = mask.sum(dim=1).to(torch.int32)
        ctx, w = F.ForwardAttentionStepFunction.apply(query, memory, self._memory_transform, self._prev_weights, lengths,
                                                      self._query.weight, self._bias, self._energy.weight)
        self._prev_weights = w
        self._prev_context = ctx
        return ctx, w
