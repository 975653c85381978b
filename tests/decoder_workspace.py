"""Named views of the decoder's forward and backward workspaces.

The fused decoder keeps every step's state in its workspaces (fp32 states, activated gates, queries, cumulative weights, the bf16
operand rows the persistent loops fed to wgmma, the prenet's rows, and in the backward the per-step gate gradients and their bf16
histories).  The offsets come from the library itself (b200tts_debug_decoder_views), so these views follow any change of the layouts.

With R frames per step a decode of T frames runs S = ceil(T / R) steps: every per-step view has S rows (S + 1 for the states, whose
row 0 is the initial state), and the step rows of the [frame ; stop] projection, fs and dfs, are R (N + 1) wide: R frames of N, then
the R stop logits.

Set functional.PROFILE['keep_ws'] = True before a decoder call; functional then keeps that call's workspaces in PROFILE['last_ws'],
PROFILE['last_bws'] and PROFILE['last_shape'].
"""
import ctypes

import torch

FWD = ('ai', 'ca', 'hg', 'cg', 'ga', 'gg', 'q', 'cum', 'memT', 'fs', 'p1', 'aib', 'hgb', 'xtm', 'p0')
BWD = ('dfs', 'dhgd', 'dctxs', 'dgg', 'dhas', 'dga', 'dq', 'dctxt', 'dmemT', 'dggb', 'dgab', 'dp1', 'dp0')
# the library's order: the first 13 forward views, the first 11 backward views, the two row strides, then the views appended later
ORDER = FWD[:13] + BWD[:11] + ('Kp_att', 'Kp_gen') + ('xtm', 'p0', 'dp1', 'dp0')
NVIEWS = len(ORDER)


def offsets(shape):
    """{name: byte offset} of every view, plus 'Kp_att' / 'Kp_gen' (row strides of aib / hgb, in elements)."""
    from multilingual_text_to_speech_b200 import _lib
    out = (ctypes.c_size_t * NVIEWS)()
    n = _lib.load().b200tts_debug_decoder_views(ctypes.byref(shape), out, NVIEWS)
    assert n == NVIEWS, ('decoder shape rejected', n)
    return dict(zip(ORDER, [int(v) for v in out]))


def frames_per_step(shape):
    return max(int(shape.R), 1)       # R = 0 means 1


def steps(shape):
    return -(-int(shape.T) // frames_per_step(shape))


def view_shapes(shape, Kp_att, Kp_gen):
    """{name: (dtype, dims)} of every view, for the decode of shape.T frames at shape.R frames per step."""
    s = shape
    B, D, M, L, A, N, P = s.B, s.D, s.M, s.L, s.A, s.N, s.P
    S, W = steps(s), frames_per_step(s) * (s.N + 1)
    f32, b16 = torch.float32, torch.bfloat16
    return {
        'ai': (f32, (S + 1, B, M + D)), 'ca': (f32, (S + 1, B, D)), 'hg': (f32, (S + 1, B, D)), 'cg': (f32, (S + 1, B, D)),
        'ga': (f32, (S, B, 4 * D)), 'gg': (f32, (S, B, 4 * D)), 'q': (f32, (S, B, A)), 'cum': (f32, (S + 1, B, L)),
        'memT': (f32, (B, L, A)), 'fs': (f32, (S, B, W)), 'p1': (f32, (S, B, P)),
        'aib': (b16, (S + 1, B, Kp_att)), 'hgb': (b16, (S + 1, B, Kp_gen)), 'xtm': (f32, (S, B, N)), 'p0': (f32, (S, B, P)),
        'dfs': (f32, (S, B, W)), 'dhgd': (f32, (S, B, D)), 'dctxs': (f32, (S, B, M)), 'dgg': (f32, (S, B, 4 * D)),
        'dhas': (f32, (S, B, D)), 'dga': (f32, (S, B, 4 * D)), 'dq': (f32, (S, B, A)), 'dctxt': (f32, (S, B, M)),
        'dmemT': (f32, (B, L, A)), 'dggb': (b16, (S, B, 4 * D)), 'dgab': (b16, (S, B, 4 * D)),
        'dp1': (f32, (S, B, P)), 'dp0': (f32, (S, B, P)),
    }


def _view(buf, off, dtype, dims):
    n = 1
    for d in dims:
        n *= d
    esize = torch.finfo(dtype).bits // 8
    assert off % esize == 0 and off + n * esize <= buf.numel(), (off, n, esize, buf.numel())
    return buf[off:off + n * esize].view(dtype).view(*dims)


def views(shape, ws, bws=None):
    """Named views into the uint8 workspaces `ws` (forward) and `bws` (backward, optional)."""
    off = offsets(shape)
    shapes = view_shapes(shape, off['Kp_att'], off['Kp_gen'])
    out = {'Kp_att': off['Kp_att'], 'Kp_gen': off['Kp_gen']}
    for name in FWD:
        out[name] = _view(ws, off[name], *shapes[name])
    if bws is not None:
        for name in BWD:
            out[name] = _view(bws, off[name], *shapes[name])
    return out


def last_views():
    """Views of the workspaces of the last decoder call made with functional.PROFILE['keep_ws'] set."""
    from multilingual_text_to_speech_b200 import functional as F
    return views(F.PROFILE['last_shape'], F.PROFILE['last_ws'], F.PROFILE.get('last_bws'))
