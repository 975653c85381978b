"""Helpers with the reference's names (reference utils/__init__.py:7-37)."""
from collections import OrderedDict

import torch

from ..params.params import Params as hp


def lengths_to_mask(lengths, max_length=None):
    """Boolean mask [B, max_length] with True at positions < length (the kernels take the lengths themselves; the mask only
    exists for callers of the module surface)."""
    width = int(lengths.max()) if max_length is None else int(max_length)
    positions = torch.arange(width, device=lengths.device)
    return positions.unsqueeze(0).lt(lengths.unsqueeze(1))


def to_gpu(x):
    """Contiguous copy on the current CUDA device (asynchronous for pinned sources); None and CPU-only hosts pass through."""
    if x is None or not torch.cuda.is_available():
        return x if x is None else x.contiguous()
    return x.contiguous().cuda(non_blocking=True)


def remove_dataparallel_prefix(state_dict):
    return OrderedDict((k[7:] if k.startswith('module.') else k, v) for k, v in state_dict.items())


def build_model(checkpoint, force_cpu=False):
    """Load hyper-parameters and weights from a reference-format checkpoint and build the model."""
    from ..modules.tacotron2 import Tacotron
    if force_cpu or not torch.cuda.is_available():
        raise RuntimeError('this Tacotron has no CPU path; a CUDA device (H100) is required')
    state = torch.load(checkpoint, map_location='cuda')
    hp.load_state_dict(state['parameters'])
    model = Tacotron()
    model.load_state_dict(remove_dataparallel_prefix(state['model']))
    return model.to('cuda')
