"""CPU oracle of the decoder with r frames per step (hp.outputs_per_step) -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.

The reference has no reduction factor, so nothing here can be pinned to it directly.  This restatement reuses the pieces of
oracle/tacotron_oracle.py (prenet, regularised cells, attention, linear layers) and follows O.decoder_forward step for step; at r = 1
it computes exactly what O.decoder_forward computes.  The tied-weights identity (`tie`) links r > 1 back to that reference-pinned path:
an r = 1 parameter set with its frame / stop projections repeated r times, fed a target in which every frame is repeated r times,
decodes every r = 1 frame r times with the same alignment.

Tape layout at r frames per step (S = ceil(T / r) steps): teacher [S]; prenet0 / prenet1 [B, >= S, P] (row i = step i's teacher-forced
input); att_h, att_c, gen_h, gen_c, step_prenet0 / 1 [S, B, .].  Attention functions are looked up on O at call time, so
forward_attention_oracle.forward_attention() switches this decoder too.
"""
import types

import numpy as np
import torch

import decoder_cases as DC
import forward_attention_oracle as FA
from oracle import tacotron_oracle as O


def steps(frames, r):
    return -(-int(frames) // int(r))


def decoder_forward(sd, hp, encoded, mask, target, speaker, language, tape, training=True, prefix='_decoder', max_frames=None):
    """Decoder._decode at r = getattr(hp, 'outputs_per_step', 1).  -> (spec [B, T, N], stop [B, T], align [B, S, L]).  Step i is fed
    frame i*r - 1 (zeros at step 0): the ground truth when teacher-forced, else the last frame step i-1 predicted.  Inference (target
    None, B == 1) feeds the step's r stop logits to the reference's exit rule in frame order and cuts at a frame."""
    r = int(getattr(hp, 'outputs_per_step', 1))
    tape = tape or {}
    dt = encoded.dtype
    B = encoded.shape[0]
    N, D = hp.num_mels, hp.decoder_dimension
    kind = hp.decoder_regularization
    rates = (hp.zoneout_hidden, hp.zoneout_cell) if kind == 'zoneout' else (hp.dropout_hidden, 0.0)
    memory = O.decoder_memory(sd, hp, encoded, speaker, language, prefix)
    att = f'{prefix}._attention'
    memT, cum, ctx = O.attention_reset(sd, att, memory)
    h_att = torch.zeros(B, D, dtype=dt); c_att = torch.zeros(B, D, dtype=dt)
    h_gen = torch.zeros(B, D, dtype=dt); c_gen = torch.zeros(B, D, dtype=dt)
    frame = torch.zeros(B, N, dtype=dt)
    inference = target is None
    if not inference:
        T = target.shape[2]
        S = steps(T, r)
        fed = target[:, :, r - 1::r][:, :, :S - 1].transpose(1, 2)                   # frames r-1, 2r-1, ... fed to steps 1 .. S-1
        tgt = torch.cat((torch.zeros(B, 1, N, dtype=dt), fed), dim=1)                # [B, S, N]
        keep = [None if tape.get(k) is None else tape[k][:, :S] for k in ('prenet0', 'prenet1')]
        tgt = O.prenet(sd, f'{prefix}._prenet', tgt, hp.dropout, *keep)
        teacher = tape['teacher']
    else:
        T = hp.max_output_length if max_frames is None else max_frames
        S = steps(T, r)
    w_att = O._cell_weights(sd, f'{prefix}._attention_lstm')
    w_gen = O._cell_weights(sd, f'{prefix}._generator_lstm')
    Wf, bf = sd[f'{prefix}._frame_prediction.weight'], sd[f'{prefix}._frame_prediction.bias']
    Ws, bs = sd[f'{prefix}._stop_prediction.weight'], sd[f'{prefix}._stop_prediction.bias']
    assert Wf.shape[0] == r * N and Ws.shape[0] == r, (tuple(Wf.shape), tuple(Ws.shape), r)

    def tm(name, i):
        t = tape.get(name)
        return None if t is None else t[i]

    specs, stops, aligns = [], [], []
    stop_frames, done = -1, False
    for i in range(S):
        if inference or not bool(teacher[i]):
            prev = O.prenet(sd, f'{prefix}._prenet', frame, hp.dropout, tm('step_prenet0', i), tm('step_prenet1', i))
        else:
            prev = tgt[:, i]
        h_att, c_att = O.regularised_cell(kind, training, torch.cat((prev, ctx), dim=1), h_att, c_att, w_att, rates,
                                          tm('att_h', i), tm('att_c', i))
        ctx, w, cum = O.attention_step(sd, att, h_att, memory, memT, cum, mask)
        h_gen, c_gen = O.regularised_cell(kind, training, torch.cat((h_att, ctx), dim=1), h_gen, c_gen, w_gen, rates,
                                          tm('gen_h', i), tm('gen_c', i))
        proto = torch.cat((h_gen, ctx), dim=1)
        frames = O._linear(proto, Wf, bf)               # [B, r*N]: row block j = frame j of the step
        stop = O._linear(proto, Ws, bs)                 # [B, r]
        frame = frames[:, (r - 1) * N:]
        aligns.append(w)
        for j in range(r):
            specs.append(frames[:, j * N:(j + 1) * N]); stops.append(stop[:, j])
            if inference and bool(O._sigmoid(stop[0, j]) >= 0.5):
                if stop_frames == -1:
                    stop_frames = hp.stop_frames
                    continue
                stop_frames -= 1
                if stop_frames == 0:
                    done = True
                    break
        if done:
            break
    n = min(len(specs), T)
    return torch.stack(specs[:n], dim=1), torch.stack(stops[:n], dim=1), torch.stack(aligns, dim=1)


def guided_attention_loss(align, input_lengths, target_lengths, g, r):
    """The guided-attention term on the step grid: align [B, S, L], each utterance's step count ceil(target_length / r) in place of its
    frame count (O.guided_attention_loss with those lengths; r = 1 is the reference's term)."""
    return O.guided_attention_loss(align, input_lengths, (target_lengths + r - 1) // r, g)


PROJECTION_KEYS = ('_decoder._frame_prediction.weight', '_decoder._frame_prediction.bias',
                   '_decoder._stop_prediction.weight', '_decoder._stop_prediction.bias')


def tie(sd, r):
    """The r-frames-per-step parameter set whose r row blocks are all the r = 1 projection (frame_w, frame_b, stop_w, stop_b)."""
    out = dict(sd)
    for k in PROJECTION_KEYS:
        out[k] = sd[k].repeat(r, *([1] * (sd[k].dim() - 1))).clone()
    return out


def repeat_frames(x, r, dim):
    """Every frame along `dim` repeated r times (frame t -> frames t*r .. t*r + r - 1)."""
    return torch.repeat_interleave(x, r, dim=dim)


def block_sum(g, r):
    """Sum of the r row blocks of a projection gradient [r*X, ...] -> [X, ...]."""
    return g.reshape(r, g.shape[0] // r, *g.shape[1:]).sum(0)


def untie(c, r, T, seed=0):
    """Case `c` built for S = ceil(T / r) steps (its tape has S rows) turned into an r-frames-per-step case of T frames: random
    projections of r*N / r rows and a random target of T frames."""
    g = torch.Generator().manual_seed(1000 + seed)
    N, DM = c.sd['_decoder._frame_prediction.weight'].shape
    S = c.target.shape[2]
    assert S == steps(T, r), (S, T, r)
    sd = dict(c.sd)
    s_in = 1.0 / np.sqrt(DM)
    sd['_decoder._frame_prediction.weight'] = torch.randn(r * N, DM, generator=g) * s_in
    sd['_decoder._frame_prediction.bias'] = torch.randn(r * N, generator=g) * 0.1
    sd['_decoder._stop_prediction.weight'] = torch.randn(r, DM, generator=g) * s_in
    sd['_decoder._stop_prediction.bias'] = torch.randn(r, generator=g) * 0.1
    c.sd = sd
    c.target = torch.randn(c.target.shape[0], N, T, generator=g)
    c.r = r
    c.name += f' r{r} T{T}'
    return c


def run(c, r, dtype=torch.float64, with_grad=True):
    """decoder_forward on case `c` (decoder_cases.Case) at r frames per step -> (sd, memory, spec, stop, align); sd / memory are leaves
    with gradients when with_grad."""
    sd = {k: (v.to(dtype).clone().requires_grad_(with_grad) if v.is_floating_point() else v) for k, v in c.sd.items()
          if not (k.startswith('_decoder._prenet.') or k.startswith('_decoder._attention.'))}
    DC._decoder_sd_alias(sd)
    memory = c.memory.to(dtype).clone().requires_grad_(with_grad)
    tape = {k: (v if k == 'teacher' else v.to(dtype)) for k, v in c.tape.items()}
    hp = types.SimpleNamespace(**vars(c.hp))
    hp.multi_speaker = hp.multi_language = False        # memory already carries the embeddings
    hp.outputs_per_step = r
    mask = O.lengths_to_mask(c.lengths, c.memory.shape[1])
    with FA.for_hp(hp):
        spec, stop, align = decoder_forward(sd, hp, memory, mask, c.target.to(dtype), None, None, tape, training=c.training)
    return sd, memory, spec, stop, align
