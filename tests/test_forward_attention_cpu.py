"""Forward attention (hp.attention_type = "forward", reference modules/attention.py:89-124) on the host: the CPU oracle against the
golden vectors of the unmodified reference (tests/golden/make_golden_forward_attention.py), the module surface, the path query and
the no-GPU failure of the new ops."""
import ctypes
import os

import numpy as np
import pytest
import torch

import __graft_entry__ as entry
import forward_attention_oracle as FA
import model_cases
import module_cases as C
from helpers import GOLDEN_DIR, Golden, assert_close
from oracle import tacotron_oracle as O
from multilingual_text_to_speech_b200 import _lib

TRAIN_CASES = ['fwd_lj_dropout', 'fwd_lj_zoneout_tf05', 'fwd_lj_eval_free', 'fwd_generated_ragged']


def _run(g, dtype, with_grad):
    sd = g.cast_sd(dtype, requires_grad=with_grad)
    i = g.inputs
    with FA.for_hp(g.hp):
        out = O.tacotron_forward(sd, g.hp, i['text'], i['text_length'], i['target'].to(dtype), i['target_length'],
                                 i.get('speakers'), i.get('languages'), g.tape_cast(dtype), training=g.train)
    return sd, out


@pytest.mark.parametrize('name', TRAIN_CASES)
def test_oracle_forward_matches_reference(name):
    g = Golden(name)
    assert g.hp.attention_type == 'forward'
    with torch.no_grad():
        _, (post, pre, stop, align, _, enc) = _run(g, torch.float64, False)
    for key, got in (('enc', enc), ('align', align), ('pre', pre), ('stop', stop), ('post', post)):
        assert_close(got, g.out[key], 1e-4, 1e-5, f'{name}: {key}')
    assert torch.equal(align.argmax(2), g.out['align'].argmax(2))
    assert torch.equal(stop > 0, g.out['stop'] > 0)
    # unlike location-sensitive attention, positions beyond the text length keep the clamp floor
    lens = g.inputs['text_length']
    short = int(torch.argmin(lens))
    if int(lens[short]) < g.L:
        assert bool((g.out['align'][short, :, int(lens[short]):] > 0).all())


@pytest.mark.parametrize('name', [n for n in TRAIN_CASES if n != 'fwd_lj_eval_free'])
def test_oracle_loss_and_gradients_match_reference(name):
    g = Golden(name)
    sd, (post, pre, stop, align, spk, enc) = _run(g, torch.float64, True)
    i = g.inputs
    tgt = i['target'].double()
    loss, parts = O.tacotron_loss(g.hp, g.meta['guided_g'], i['text_length'], i['target_length'], pre, tgt, post, tgt,
                                  stop, i['stop_target'], align, i.get('speakers'), spk)
    assert 'guided_att' in parts
    for k, v in parts.items():
        assert abs(float(v.detach()) - g.losses[k]) < 1e-4 * max(1.0, abs(g.losses[k])), (k, float(v.detach()), g.losses[k])
    loss.backward()
    for k, ref in g.grad.items():
        if k.startswith('_decoder._prenet.') or k.startswith('_decoder._attention.'):
            continue
        got = sd[k].grad
        got = torch.zeros_like(ref) if got is None else got.clone()
        if k == '_embedding.weight':
            got[0] = 0          # Embedding(padding_idx=0): row 0 receives no gradient
        scale = float(ref.abs().max()) + 1e-12
        assert_close(got, ref, 2e-3, 2e-4 * scale + 1e-9, 'grad ' + k)


class _OracleForwardAttention(torch.nn.Module):
    """The oracle step behind the module API of ForwardAttention (same parameter names), computed in fp64."""

    def __init__(self, A, D, M):
        super().__init__()
        self._bias = torch.nn.Parameter(torch.zeros(1, A))
        self._energy = torch.nn.Linear(A, 1, bias=False)
        self._query = torch.nn.Linear(D, A, bias=False)
        self._memory = torch.nn.Linear(M, A, bias=False)

    def _sd(self):
        return {'a.' + k: v.double() for k, v in self.named_parameters()}

    def reset(self, memory, B, L, device):
        self._memT, self._alpha, _ = FA.attention_reset(self._sd(), 'a', memory.double())

    def forward(self, query, memory, mask, prev):
        ctx, w, self._alpha = FA.attention_step(self._sd(), 'a', query.double(), memory.double(), self._memT, self._alpha, mask)
        return ctx.float(), w.float()


def test_oracle_module_steps_match_reference():
    """ForwardAttention.reset + three forward steps with gradients of every input and parameter (tests/module_cases.py)."""
    stored = np.load(os.path.join(GOLDEN_DIR, 'fwd_attention_module.npz'))
    d = C.ATT_DIMS
    res = C.attention_case(_OracleForwardAttention(d['A'], d['D'], d['M']), 'cpu')
    assert {f'forward_attention.{k}' for k in res} == {k for k in stored.files if not k.endswith('.absmax')}
    for key, t in res.items():
        got, ref, absmax = C.unpack_like(stored, 'forward_attention', key, t)
        assert_close(got, ref, 1e-4, 1e-5 * absmax + 1e-7, key)


@pytest.mark.parametrize('name', ['fwd_lj_dropout', 'fwd_generated_ragged'])
def test_state_dict_keys_match_reference(name):
    """A model built with attention_type = "forward" has the reference's state_dict keys, in order, and loads its checkpoint strictly."""
    g = Golden(name)
    model = model_cases.build_model(g)
    own = model.state_dict()
    assert list(own.keys()) == list(g.sd.keys())
    att = [k for k in own if k.startswith('_attention.')]
    assert att == ['_attention._bias', '_attention._energy.weight', '_attention._query.weight', '_attention._memory.weight']
    assert model._decoder._param_list()[14:16] == [None, None]


@pytest.fixture(scope='module')
def lib():
    entry.build()
    return _lib.load()


def _shape(att_kind, B=60, L=180, M=288, D=1024, training=1, C=32, K=31):
    return _lib.DecoderShape(B, L, 900, M, D, 256, 128, C, K, 80, 1, training, 0.1, 0.1, 0.5, att_kind)


def test_decoder_path_forward_attention_is_the_per_step_chains(lib):
    """The persistent loops are built around the location term: forward attention runs the per-step chains in both passes."""
    assert lib.b200tts_decoder_path(ctypes.byref(_shape(_lib.ATT_LOCATION))) == 0b111111
    for training in (0, 1):
        for C, K in ((32, 31), (0, 0), (7, 4)):          # C and K are ignored
            s = _shape(_lib.ATT_FORWARD, training=training, C=C, K=K)
            assert lib.b200tts_decoder_path(ctypes.byref(s)) == 0
            assert lib.b200tts_decoder_workspace_bytes(ctypes.byref(s)) > 0
            assert lib.b200tts_decoder_bwd_workspace_bytes(ctypes.byref(s)) > 0
    assert lib.b200tts_decoder_workspace_bytes(ctypes.byref(_shape(2))) == 0
    assert b'attention kind' in lib.b200tts_last_error()


def test_transition_agent_is_refused_with_the_reason():
    from multilingual_text_to_speech_b200.params.params import Params as hp
    from multilingual_text_to_speech_b200.modules.tacotron2 import Tacotron
    hp.reset()
    hp.load_state_dict({'attention_type': 'forward_transition_agent'})
    try:
        with pytest.raises(NotImplementedError, match='takes 3 arguments but the decoder passes 4'):
            Tacotron()
    finally:
        hp.reset()


@pytest.mark.skipif(torch.cuda.is_available(), reason='checks the no-GPU failure mode')
def test_forward_attention_ops_fail_loudly_without_gpu(lib):
    from multilingual_text_to_speech_b200 import functional as F
    B, L, M, D, A = 2, 5, 8, 6, 4
    st = lib.b200tts_forward_attention_step(B, L, M, D, A, *([None] * 12))
    assert st == -2 and b'no CPU fallback' in lib.b200tts_last_error()
    st = lib.b200tts_forward_attention_step_backward(B, L, M, A, *([None] * 16))
    assert st == -2 and b'no CPU fallback' in lib.b200tts_last_error()
    with pytest.raises(_lib.B200TTSError):
        F.ForwardAttentionStepFunction.apply(torch.zeros(B, D), torch.zeros(B, L, M), torch.zeros(B, L, A), torch.zeros(B, L),
                                             torch.full((B,), L), torch.zeros(A, D), torch.zeros(1, A), torch.zeros(1, A))
