"""The stream contract every vocoder stream pool keeps (StreamPool, FoldedStreamPool, GriffinLimStreamPool), from one table: the errors of
open / feed / end / close for an unknown stream, a full pool, a bad seed, a rejected tape, a stream that ends too short and a stream fed
after its end, each leaving the pool usable."""
import numpy as np
import pytest
import torch

from multilingual_text_to_speech_b200 import _lib
from multilingual_text_to_speech_b200.modules.griffinlim import GriffinLimVocoder
from test_gpu_wavernn import make_model

pytestmark = pytest.mark.gpu


@pytest.fixture(scope='module', autouse=True)
def _built():
    import __graft_entry__ as entry
    from multilingual_text_to_speech_b200.params.params import Params as hp
    entry.build()
    assert torch.cuda.is_available()
    hp.reset()
    yield
    _lib.set_precision('fp32')


# pool of two streams, a tape it rejects and the message, the frames a stream needs before end()
POOLS = {
    'unfolded': (lambda: make_model('RAW', seed=80).stream_pool(2), np.zeros((2, 500, 1), np.float32), r'expected \[1, steps, 1\]', 21),
    'folded': (lambda: make_model('RAW', seed=81).stream_pool(2, target=1000, overlap=50), np.zeros((1, 1000, 1), np.float32),
               r'expected \[folds, 1100, 1\]', 21),
    'griffinlim': (lambda: GriffinLimVocoder().stream_pool(2), np.zeros((1, 500, 1), np.float32), 'draws nothing', 2),
}


@pytest.mark.parametrize('kind', sorted(POOLS))
def test_contract_errors(kind):
    make, bad_tape, tape_msg, min_frames = POOLS[kind]
    pool = make()
    frames = lambda n: torch.zeros(pool.v.feat_dims, n, device='cuda')     # noqa: E731
    for op in (lambda: pool.feed(99, frames(1)), lambda: pool.end(99), lambda: pool.close(99)):
        with pytest.raises(ValueError, match='unknown or finished stream 99'):
            op()
    for seed in (-1, 1 << 64, 1.5, True):
        with pytest.raises(ValueError, match=r'a seed is an int in \[0, 2\^64\)'):
            pool.open(seed=seed)
    with pytest.raises(ValueError, match=tape_msg):
        pool.open(uniforms=bad_tape)
    assert pool.streams == {}
    a, b = pool.open(seed=5), pool.open()
    with pytest.raises(ValueError, match='the stream pool is full: 2 streams are open'):
        pool.open()
    pool.feed(a, frames(min_frames - 1))
    with pytest.raises(ValueError, match=f'ended after {min_frames - 1} frames.*at least {min_frames}'):
        pool.end(a)
    pool.feed(a, frames(1))
    pool.end(a)
    for op in (lambda: pool.feed(a, frames(1)), lambda: pool.end(a)):
        with pytest.raises(ValueError, match=f'stream {a} has ended'):
            op()
    pool.close(b)
    c = pool.open()
    assert sorted(pool.streams) == [a, c] == [0, 2] and pool.rows == 2
    pool.close(a)
    pool.close(c)
    with pytest.raises(ValueError, match='unknown or finished stream 0'):
        pool.close(a)
    assert pool.streams == {}
