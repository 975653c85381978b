"""WaveRNN training from a device-resident corpus, without a GPU: the corpus's packing, every ValueError of VocoderCorpus.batch and
GraphedVocoderStep (raised before any device call: the corpus here lives on the CPU, where any device op would raise B200TTSError instead),
corpus.draw_offsets against draw_offsets, the deferred abort-flag bookkeeping on a host stand-in flag, the new entry points' refusals that
need no device, the window kernel's registers, and the example trainer's --help."""
import ctypes
import os
import re
import subprocess
import sys

import numpy as np
import pytest
import torch

from multilingual_text_to_speech_b200 import _lib, build
from multilingual_text_to_speech_b200.graph import DeferredAbortCheck, GraphedVocoderStep
from multilingual_text_to_speech_b200.modules.wavernn import VocoderCorpus, WaveRNN, draw_offsets, mel_window
from test_wavernn_cpu import REAL, _nvcc

HOP, PAD, SEQ = 275, 2, 1375


def small_corpus(mode='RAW', frames=(30, 45, 60), extra=(0, 100, 274), **kw):
    rng = np.random.default_rng(0)
    mels = [rng.standard_normal((80, f)) for f in frames]
    labels = [rng.integers(0, 512, f * HOP + e) for f, e in zip(frames, extra)]
    return VocoderCorpus(mels, labels, mode, 9, SEQ, PAD, HOP, 'cpu', **kw), mels, labels


def test_packing_offsets_and_lengths():
    c, mels, labels = small_corpus()
    assert len(c) == 3 and c.feat == 80 and c.win == mel_window(SEQ, HOP, PAD) == 9
    assert c.frames == [30, 45, 60] and c.samples == [30 * HOP, 45 * HOP + 100, 60 * HOP + 274]
    assert c.frame_start.tolist() == [0, 30, 75] and c.sample_start.tolist() == [0, 30 * HOP, 75 * HOP + 100]
    assert tuple(c.mels.shape) == (80, 135) and c.mels.dtype == torch.float32
    assert c.labels.dtype == torch.int16 and c.labels.numel() == sum(c.samples)
    np.testing.assert_array_equal(c.mels[:, 30:75].numpy(), mels[1].astype(np.float32))
    np.testing.assert_array_equal(c.labels[c.sample_start[2]:].numpy().view(np.uint16), labels[2])
    assert c.nbytes == 2 * sum(c.samples) + 4 * 80 * 135
    # 16-bit labels above 32767 keep their bits
    big = VocoderCorpus([np.zeros((80, 20))], [np.array([0, 40000, 65535] * 2000)], 'MOL', 9, SEQ, PAD, HOP, 'cpu')
    assert big.labels.numpy().view(np.uint16)[:3].tolist() == [0, 40000, 65535]


def test_draw_offsets_equals_draw_offsets():
    c, _, _ = small_corpus()
    ids = [2, 0, 1, 1, 2]
    a = c.draw_offsets(ids, np.random.default_rng(11))
    b = draw_offsets([c.frames[u] for u in ids], SEQ, HOP, PAD, np.random.default_rng(11))
    assert a == b
    with pytest.raises(ValueError, match='outside'):
        c.draw_offsets([3], np.random.default_rng(0))


def test_batch_value_errors_before_any_device_call():
    c, _, _ = small_corpus()
    launches = _lib.launch_count()
    with pytest.raises(ValueError, match=r'utterance id 3 of item 1 outside \[0, 3\)'):
        c.batch([0, 3], [0, 0])
    with pytest.raises(ValueError, match=r'utterance id -1'):
        c.batch([-1], [0])
    # the mel window leaves the mel: vocoder_batch's wording
    with pytest.raises(ValueError, match=r'offset 22 of item 0 leaves its window outside the mel \(30 frames\) or the labels \(8250\)'):
        c.batch([0], [22])
    # the mel fits (21 + 9 = 30 frames) but the labels do not: (21 + 2) 275 + 1376 > 7000
    rng = np.random.default_rng(0)
    cut = VocoderCorpus([rng.standard_normal((80, 30))], [np.zeros(7000, np.int64)], 'RAW', 9, SEQ, PAD, HOP, 'cpu')
    with pytest.raises(ValueError, match=r'offset 21 of item 0 leaves its window outside the mel \(30 frames\) or the labels \(7000\)'):
        cut.batch([0], [21])
    with pytest.raises(ValueError, match='offset -1'):
        c.batch([1], [-1])
    with pytest.raises(ValueError, match='need 1 to 64'):
        c.batch([0] * 65, [0] * 65)
    with pytest.raises(ValueError, match='at least one'):
        c.batch([], [])
    with pytest.raises(ValueError, match='as many'):
        c.batch([0, 1], [0])
    bad2 = VocoderCorpus([rng.standard_normal((80, 30)), rng.standard_normal((80, 30))],
                         [np.full(30 * HOP, 3), np.full(30 * HOP, 70000)], 'RAW', 9, SEQ, PAD, HOP, 'cpu')
    with pytest.raises(ValueError, match=r'labels of utterance 1 \(item 0\) lie outside \[0, 65536\)'):
        bad2.batch([1], [0])
    neg = VocoderCorpus([rng.standard_normal((80, 30))], [np.full(30 * HOP, -1)], 'RAW', 9, SEQ, PAD, HOP, 'cpu')
    with pytest.raises(ValueError, match='lie outside'):
        neg.batch([0], [0])
    assert _lib.launch_count() == launches
    # a valid table goes on to the device: on a CPU corpus that is the library's refusal, not a ValueError
    with pytest.raises(_lib.B200TTSError, match='CUDA'):
        c.batch([0, 1], [0, 5])


def test_corpus_construction_errors():
    rng = np.random.default_rng(0)
    m, lab = [rng.standard_normal((80, 30))], [np.zeros(30 * HOP, np.int64)]
    with pytest.raises(ValueError, match='mode'):
        VocoderCorpus(m, lab, 'MU', 9, SEQ, PAD, HOP, 'cpu')
    with pytest.raises(ValueError, match='multiple of the hop'):
        VocoderCorpus(m, lab, 'RAW', 9, 1000, PAD, HOP, 'cpu')
    with pytest.raises(ValueError, match='16 hops'):
        VocoderCorpus(m, lab, 'RAW', 9, 17 * HOP, PAD, HOP, 'cpu')
    with pytest.raises(ValueError, match='bits'):
        VocoderCorpus(m, lab, 'RAW', 17, SEQ, PAD, HOP, 'cpu')
    with pytest.raises(ValueError, match='as many'):
        VocoderCorpus(m, lab + lab, 'RAW', 9, SEQ, PAD, HOP, 'cpu')
    with pytest.raises(ValueError, match='mel 1'):
        VocoderCorpus(m + [rng.standard_normal((40, 30))], lab + lab, 'RAW', 9, SEQ, PAD, HOP, 'cpu')
    with pytest.raises(ValueError, match='integer'):
        VocoderCorpus(m, [np.zeros(30 * HOP)], 'RAW', 9, SEQ, PAD, HOP, 'cpu')


def test_graphed_step_value_errors_before_any_device_call():
    c, _, _ = small_corpus()
    model = WaveRNN(**REAL)
    launches = _lib.launch_count()
    with pytest.raises(ValueError, match='batch_size 65'):
        GraphedVocoderStep(model, None, c, 65)
    with pytest.raises(ValueError, match='batch_size 0'):
        GraphedVocoderStep(model, None, c, 0)
    with pytest.raises(ValueError, match='does not match the model'):
        GraphedVocoderStep(WaveRNN(**dict(REAL, mode='MOL')), None, c, 4)
    c16, _, _ = small_corpus()
    c16.bits = 10
    with pytest.raises(ValueError, match='does not match the model'):
        GraphedVocoderStep(model, None, c16, 4)
    short, _, _ = small_corpus(frames=(8,), extra=(0,))
    with pytest.raises(ValueError, match='no utterance long enough'):
        GraphedVocoderStep(model, None, short, 4)
    # a captured step's own call-time checks, on a step object that was never captured
    step = GraphedVocoderStep.__new__(GraphedVocoderStep)
    step.corpus, step.batch_size, step.precision = c, 2, 'bf16'
    assert _lib.get_precision() == 'fp32'
    with pytest.raises(ValueError, match='captured in bf16 mode'):
        step([0, 1], [0, 0])
    with pytest.raises(ValueError, match='3 windows for a step captured at a batch of 2'):
        step([0, 1, 2], [0, 0, 0])
    with pytest.raises(ValueError, match='leaves its window'):
        step([0, 1], [40, 0])
    assert _lib.launch_count() == launches


class StandInEvent:
    """An event whose completion the test controls."""
    done = True

    def record(self):
        self.recorded = True

    def query(self):
        return StandInEvent.done

    def synchronize(self):
        pass


def test_deferred_abort_raises_on_the_next_call_not_before():
    flag = [0]
    copies = []

    def copy(slot):
        copies.append(1)
        slot.fill_(flag[0])

    StandInEvent.done = True
    chk = DeferredAbortCheck(copy, StandInEvent, depth=4, pin=False)
    for n in (1, 2):
        chk.poll()
        chk.after_replay(n)
    flag[0] = 1               # replay 3's loops time out
    chk.poll()
    chk.after_replay(3)       # the call that replays 3 does not raise
    flag[0] = 0
    with pytest.raises(_lib.B200TTSError, match='replay 3'):
        chk.poll()            # the next call does
    chk.after_replay(4)
    chk.wait()
    assert len(copies) == 4


def test_deferred_abort_waits_for_incomplete_copies_and_close_reports_the_last_replay():
    flag = [0]
    StandInEvent.done = False
    chk = DeferredAbortCheck(lambda slot: slot.fill_(flag[0]), StandInEvent, depth=2, pin=False)
    chk.after_replay(1)
    flag[0] = 1
    chk.after_replay(2)
    chk.poll()                # copies not completed: nothing read, nothing raised
    assert len(chk._pending) == 2
    flag[0] = 0
    chk.after_replay(3)       # at the depth: waits for replay 1's copy (flag clear), keeps 2 and 3 outstanding
    assert [p[0] for p in chk._pending] == [2, 3]
    with pytest.raises(_lib.B200TTSError, match='replay 2'):
        chk.wait()
    StandInEvent.done = True
    chk.wait()
    flag[0] = 1
    chk.after_replay(4)
    with pytest.raises(_lib.B200TTSError, match='replay 4'):
        chk.wait()            # close() after the last replay
    StandInEvent.done = True


def test_abi_refusals_without_a_device():
    lib = _lib.load()
    one = ctypes.c_void_p(256)
    args = dict(mode=0, bits=9, B=4, feat=80, seq_len=1375, pad=2, hop=275)

    def call(**kw):
        a = dict(args, **kw)
        ptrs = kw.pop('ptrs', [one] * 8)
        return lib.b200tts_wavernn_cut_windows(a['mode'], a['bits'], a['B'], a['feat'], a['seq_len'], a['pad'], a['hop'], ptrs[0], 100,
                                               *ptrs[1:], None)

    for bad, msg in [(dict(mode=2), b'mode'), (dict(bits=0), b'bits'), (dict(bits=17), b'bits'), (dict(B=0), b'batch'),
                     (dict(B=65), b'batch'), (dict(seq_len=1000), b'multiple of the hop'), (dict(seq_len=17 * 275), b'16 hops'),
                     (dict(seq_len=0), b'multiple'), (dict(pad=-1), b'pad'), (dict(feat=0), b'mel channels')]:
        assert call(**bad) == -1, bad
        assert msg in lib.b200tts_last_error(), (bad, lib.b200tts_last_error())
    assert call(ptrs=[one] * 7 + [None]) == -1 and b'null' in lib.b200tts_last_error()
    shape = _lib.GRUSeqShape(4, 10, 512)
    assert lib.b200tts_gru_seq_abort_flag_copy(ctypes.byref(shape), one, 16, one, None) == -1
    assert b'workspace' in lib.b200tts_last_error()
    assert lib.b200tts_gru_seq_abort_flag_copy(ctypes.byref(shape), one, 1 << 20, None, None) == -1
    assert b'null' in lib.b200tts_last_error()


# measured (CUDA 12.9, sm_90a): 30 registers, no stack
REG_BOUND = 48


def test_window_kernel_registers_and_spills(tmp_path):
    nvcc = _nvcc()
    if nvcc is None:
        pytest.skip('nvcc not available')
    cmd = [nvcc] + build.NVCC_FLAGS + ['-I', os.path.join(build.ROOT, 'include'), '-Xptxas', '-v', '-cubin',
                                       os.path.join(build.CSRC, 'wavernn_windows.cu'), '-o', str(tmp_path / 'wavernn_windows.cubin')]
    res = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    assert res.returncode == 0, res.stdout
    found = re.findall(r'Function properties for (\S+)\n\s*(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads\n'
                       r'[^\n]*Used (\d+) registers', res.stdout)
    assert len(found) == 1 and 'wavernn_cut_windows_kernel' in found[0][0], found
    _, stack, st, ld, regs = found[0]
    assert int(stack) == 0 and int(st) == 0 and int(ld) == 0
    assert int(regs) <= REG_BOUND, regs


def test_example_trainer_help():
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    res = subprocess.run([sys.executable, os.path.join(root, 'examples', 'train_wavernn_synthetic.py'), '--help'], stdout=subprocess.PIPE,
                         stderr=subprocess.STDOUT, text=True, timeout=120)
    assert res.returncode == 0, res.stdout
    for flag in ('--steps', '--batch', '--eager', '--mode', '--precision'):
        assert flag in res.stdout
