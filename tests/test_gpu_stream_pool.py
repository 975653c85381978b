"""Concurrent streaming synthesis on the GPU, at the reference's vocoder dimensions:
  * b200tts_wavernn_run_rows: rows with mixed budgets (0 included) and parities each equal a solo b200tts_wavernn_run_stream bit for bit,
    a row idle for some calls continues as if uninterrupted, and a reset row reused by a new stream equals a fresh prepare;
  * the packed upsampling layer equals the single layers, and the pool's windowed features (b200tts_wavernn_window_rows) equal
    b200tts_wavernn_fold's over the whole mel bit for bit;
  * WaveRNN.stream_pool: every stream equals generate(mel, target=F hop, overlap=0) bit for bit under irregular chunkings, staggered opens,
    a freed and reused row and fewer active rows than the capacity; 64 streams at once against one generate_batch;
  * Tacotron.inference_streams against inference_batch and inference_stream; speech_streams against speech_stream;
  * argument errors."""
import numpy as np
import pytest
import torch

from multilingual_text_to_speech_b200 import _lib
from multilingual_text_to_speech_b200 import functional as F
from test_gpu_batch_inference import CASES, _case, _stacked_tape
from test_gpu_streaming import _chunks, _mel, _taped
from test_gpu_wavernn import make_model

pytestmark = pytest.mark.gpu


@pytest.fixture(scope='module', autouse=True)
def _built():
    import __graft_entry__ as entry
    entry.build()
    assert torch.cuda.is_available()
    yield
    _lib.set_precision('fp32')


def _tape(m, frames, seed):
    return torch.rand(m.tape_shape(frames, frames * m.hop_length, 0), generator=torch.Generator().manual_seed(seed))


def _reference(m, mel, tape):
    return m.generate(mel, target=mel.shape[1] * m.hop_length, overlap=0, uniforms=tape)


# ---- the ragged loop ----
def _random_cond(m, T, seed):
    g = torch.Generator(device='cuda').manual_seed(seed)
    R, Fc = m.rnn_dims, m.fc_dims
    r = lambda *s: 0.5 * torch.randn(*s, device='cuda', generator=g)     # noqa: E731
    return [r(T, R), r(T, 3 * R), r(T, 3 * R), r(T, Fc), r(T, Fc)], torch.rand(T, m.uniforms_per_step(), device='cuda', generator=g)


def _solo(m, w, params, cond, uni):
    T = uni.shape[0]
    shape = _lib.WaveRNNShape(1, m.rnn_dims, m.fc_dims, m.n_classes, _lib.WAVERNN_MODES[m.mode], T)
    ws = F.wavernn_workspace(shape, torch.device('cuda'))
    F.wavernn_prepare(shape, params, ws)
    out = torch.zeros(1, T, device='cuda')
    F.wavernn_run_stream(shape, params, [c.unsqueeze(1).contiguous() for c in cond], 0, T, uni.unsqueeze(0).contiguous(), out, ws)
    assert not F.wavernn_aborted(shape, ws)
    return out[0]


@pytest.mark.parametrize('mode', ['RAW', 'MOL'])
def test_run_rows_equal_solo_streams(mode):
    _lib.set_precision('fp32')
    m = make_model(mode, seed=41)
    with torch.no_grad():
        w = m.loop_weights(torch.device('cuda'))
        params = F.wavernn_params(w)
        # per row: the budget of each call; row 2 idles for three calls, row 3 never runs, row 5 ends and is reset for a new stream after
        # call 1; 9 rows: two N tiles, the second with one row
        budgets = {0: [5, 0, 7, 3, 1], 1: [4, 4, 4, 4, 4], 2: [3, 0, 0, 0, 9], 4: [0, 6, 1, 0, 2], 5: [6, 1], 8: [2, 3, 0, 5, 1]}
        reused = [0, 0, 4, 2, 5]                       # the new stream on row 5 from call 2 on
        streams = {r: _random_cond(m, sum(b), 100 + r) for r, b in budgets.items()}
        streams['new'] = _random_cond(m, sum(reused), 200)
        cap, nmax = 10, 9
        shape = _lib.WaveRNNShape(cap, m.rnn_dims, m.fc_dims, m.n_classes, _lib.WAVERNN_MODES[mode], nmax)
        ws = F.wavernn_workspace(shape, torch.device('cuda'))
        F.wavernn_prepare(shape, params, ws)
        got = {k: [] for k in streams}
        done = {k: 0 for k in streams}
        U = m.uniforms_per_step()
        for call in range(5):
            if call == 2:
                F.wavernn_reset_rows(shape, ws, [5])
            plan = {r: (r, b[call]) for r, b in budgets.items() if r != 5}
            plan[5] = ('new', reused[call]) if call >= 2 else (5, budgets[5][call])
            active = 9                                   # below the capacity of 10
            n = max(b for _, b in plan.values())
            cond = [torch.zeros(n, active, c.shape[1], device='cuda') for c in streams[0][0]]
            uni = torch.zeros(active, n, U, device='cuda')
            row_t, row_n = torch.zeros(active, dtype=torch.int64), torch.zeros(active, dtype=torch.int32)
            for r, (k, b) in plan.items():
                t = done[k]
                for c, src in zip(cond, streams[k][0]):
                    c[:b, r] = src[t:t + b]
                uni[r, :b] = streams[k][1][t:t + b]
                row_t[r], row_n[r] = t, b
            out = torch.full((active, n), 7.0, device='cuda')
            F.wavernn_run_rows(shape, params, cond, row_t.cuda(), row_n.cuda(), n, uni, out, ws)
            assert bool((out[3] == 7.0).all())           # an idle row writes nothing
            for r, (k, b) in plan.items():
                got[k].append(out[r, :b].clone())
                assert bool((out[r, b:] == 7.0).all())
                done[k] += b
        assert not F.wavernn_aborted(shape, ws)
        for k, (cond, uni) in streams.items():
            ref = _solo(m, w, params, cond, uni)
            assert torch.equal(torch.cat(got[k]), ref), k


# ---- features ----
def test_packed_upsampling_equals_single_layers():
    m = make_model('RAW', seed=43)
    fir = m.upsample.up_layers[1].weight.detach().reshape(-1).float().cuda()
    xs = [torch.randn(80, n, device='cuda') for n in (7, 1, 64, 130)]
    got = F.wavernn_upsample_segments(torch.cat([x.reshape(-1) for x in xs]), [x.shape[1] for x in xs], fir, 5)
    ref = torch.cat([F.wavernn_upsample_layer(x, fir, 5).reshape(-1) for x in xs])
    assert torch.equal(got, ref)


def _fold_features(m, mel):
    """The whole mel's loop features [F hop, feat_dims + res_out_dims]: b200tts_wavernn_fold over the stage outputs of generate(mel,
    target=F hop, overlap=0)."""
    F_, hop = mel.shape[1], m.hop_length
    trace = {}
    m._generate([mel], [F_], None, F_ * hop, 0, None, torch.device('cuda'), trace)
    fshape = _lib.WaveRNNFoldShape(1, 1, 80, 128, hop, 2, 11, F_ * hop, 0, F_)
    d = lambda a: torch.from_numpy(np.asarray(a)).cuda()     # noqa: E731
    fir = m.upsample.up_layers[-1].weight.detach().reshape(-1).float().contiguous().cuda()
    return F.wavernn_fold(fshape, trace['mel_up'], d(trace['mel_off']), d(np.array([F_], np.int32)), d(np.zeros(1, np.int32)),
                          d(np.zeros(1, np.int32)), fir, trace['aux'], 0, F_ * hop)[:, 0]


def test_loop_window_rows_equal_the_fold():
    _lib.set_precision('fp32')
    m = make_model('RAW', seed=44)
    hop = m.hop_length
    mels = [_mel(900, 45), _mel(40, 46), _mel(300, 47), _mel(25, 48)]
    # (mel, known frames, final, first position, positions), one pool row each: stream starts, middles and final frames of four mels, then
    # six windows of the 40-frame mel; 1 to 39 hops of positions, below and above a 64-column tile of the mel path
    cases = [(0, 900, False, 0, 300), (1, 40, True, 17 * hop, 22 * hop - 5), (2, 300, False, 100 * hop + 7, 40), (3, 25, True, 23 * hop, hop)]
    cases += [(1, known, final, s0, s1 - s0) for s0, s1, known, final in
              [(0, 275, 3, False), (0, 37 * hop, 40, False), (3 * hop, 11 * hop, 13, False), (17 * hop, 39 * hop, 40, True),
               (0, 39 * hop, 40, True), (38 * hop + 5, 39 * hop, 40, True)]]
    with torch.no_grad():
        whole = [_fold_features(m, mel) for mel in mels]
        pool = m.stream_pool(len(cases) + 2)
        sids = [pool.open() for _ in cases]
        for sid, (k, known, final, _, _) in zip(sids, cases):
            pool.feed(sid, mels[k][:, :known])
            pool.streams[sid].ended = final
        plan = {sid: (t, n) for sid, (*_, t, n) in zip(sids, cases)}
        _lib.set_precision('fp32')
        feat = pool.loop.features(pool._loop_rows(plan), len(cases), max(n for _, n in plan.values()))
        for b, (k, known, final, t, n) in enumerate(cases):
            assert torch.equal(feat[:n, b], whole[k][t:t + n]), b
            assert bool((feat[n:, b] == 0).all()), b


# ---- the pool ----
def _drive(pool, script, steps):
    """Runs a pool over `steps` rounds; script(round) -> actions [(op, key, arg)] before that round's run.  -> {key: [chunks]}"""
    sid_of, out = {}, {}
    for k in range(steps):
        for op, key, arg in script(k):
            if op == 'open':
                sid_of[key] = pool.open(arg)
                out[key] = []
            elif op == 'feed':
                pool.feed(sid_of[key], arg)
            else:
                pool.end(sid_of[key])
        for sid, chunk in pool.run().items():
            out[next(k_ for k_, s in sid_of.items() if s == sid)].append(chunk)
    return out


@pytest.mark.parametrize('mode', ['RAW', 'MOL'])
def test_pool_streams_equal_generate(mode):
    _lib.set_precision('fp32')
    m = make_model(mode, seed=50)
    frames = {'a': 21, 'b': 900, 'c': 150, 'd': 333, 'e': 60}
    mels = {k: _mel(f, 51 + i) for i, (k, f) in enumerate(frames.items())}
    tapes = {k: _tape(m, f, 61 + i) for i, (k, f) in enumerate(frames.items())}
    sizes = {'a': [5, 0, 1, 13, 2], 'b': [1] * 20 + [13, 130, 64, 300, 7], 'c': [150], 'd': [40, 3, 90, 0, 200], 'e': [1] * 60}
    parts = {k: _chunks(mels[k], sizes[k]) for k in frames}
    # staggered opens; 'e' opens on the row 'a' frees; capacity 8 with at most 4 rows open
    opens = {'a': 0, 'b': 1, 'c': 3, 'd': 6}

    def script(r):
        acts = []
        for k, r0 in opens.items():
            if r == r0:
                acts.append(('open', k, tapes[k]))
        if r == 40:
            acts.append(('open', 'e', tapes['e']))
        for k in frames:
            r0 = opens.get(k, 40)
            i = r - r0
            if 0 <= i < len(parts[k]):
                acts.append(('feed', k, parts[k][i]))
            if i == len(parts[k]):
                acts.append(('end', k, None))
        return acts
    pool = m.stream_pool(8)
    got = _drive(pool, script, 120)
    assert not pool.streams, list(pool.streams)
    for k in frames:
        ref = _reference(m, mels[k], tapes[k])
        out = torch.cat(got[k])
        assert out.shape == ref.shape, (k, out.shape, ref.shape)
        assert torch.equal(out, ref), (k, int((out != ref).sum()))
    assert len(got['b']) > 3


def test_pool_with_deemphasis_within_bound():
    from test_gpu_wavernn import _deemphasis_bound
    _lib.set_precision('fp32')
    m = make_model('RAW', seed=52)
    a, mels = 0.97, [_mel(60, 53), _mel(33, 54)]
    tapes = [_tape(m, 60, 55), _tape(m, 33, 56)]
    pool = m.stream_pool(2, preemphasis=a)
    sids = [pool.open(t) for t in tapes]
    for sid, mel in zip(sids, mels):
        pool.feed(sid, mel[:, :30])
    out = {sid: [] for sid in sids}
    for r in range(12):
        if r == 2:
            for sid, mel in zip(sids, mels):
                pool.feed(sid, mel[:, 30:])
                pool.end(sid)
        for sid, c in pool.run().items():
            out[sid].append(c)
    for sid, mel, tape in zip(sids, mels, tapes):
        ref = m.generate(mel, target=mel.shape[1] * 275, overlap=0, uniforms=tape, preemphasis=a)
        got = torch.cat(out[sid])
        assert got.shape == ref.shape
        assert float((got - ref).abs().max() / ref.abs().max()) <= _deemphasis_bound(a)


@pytest.mark.parametrize('mode', ['RAW', 'MOL'])
def test_64_concurrent_streams(mode):
    _lib.set_precision('fp32')
    m = make_model(mode, seed=57)
    hop, U = m.hop_length, m.uniforms_per_step()
    rng = np.random.default_rng(58)
    frames = [int(f) for f in rng.integers(100, 221, 64)]
    mels = [_mel(f, 1000 + i) for i, f in enumerate(frames)]
    Tmax = max(frames) * hop
    g = torch.Generator().manual_seed(59)
    long_tapes = [torch.rand(1, Tmax, U, generator=g) for _ in frames]
    # one fold per mel: generate_batch at target >= the longest mel's samples is generate(mel, target=F hop, overlap=0) of each
    assert torch.equal(m.generate(mels[0], target=Tmax, overlap=0, uniforms=long_tapes[0]),
                       _reference(m, mels[0], long_tapes[0][:, :frames[0] * hop]))
    refs = m.generate_batch(mels, target=Tmax, overlap=0, uniforms=long_tapes)
    pool = m.stream_pool(64)
    sids = [pool.open(t) for t in long_tapes]
    out = {sid: [] for sid in sids}
    for k in range(0, max(frames), 32):
        for sid, mel in zip(sids, mels):
            if k < mel.shape[1]:
                pool.feed(sid, mel[:, k:k + 32])
                if k + 32 >= mel.shape[1]:
                    pool.end(sid)
        for sid, c in pool.run().items():
            out[sid].append(c)
    while pool.streams:
        for sid, c in pool.run().items():
            out[sid].append(c)
    for i, sid in enumerate(sids):
        assert torch.equal(torch.cat(out[sid]), refs[i]), i


# ---- decoder and end to end ----
@pytest.mark.parametrize('precision', ['fp32', 'bf16'])
@pytest.mark.parametrize('chunk', [7, 128])
@pytest.mark.parametrize('name', CASES)
def test_inference_streams(name, chunk, precision):
    from helpers import assert_close
    from multilingual_text_to_speech_b200.rng import MaskSource
    model, utts, meta = _case(name)
    _lib.set_precision(precision)
    tape = {'step_prenet0': _stacked_tape([u[3] for u in utts]), 'step_prenet1': _stacked_tape([u[4] for u in utts])}
    speakers = None if utts[0][1] is None else [u[1] for u in utts]
    languages = None if utts[0][2] is None else [u[2] for u in utts]
    texts = [u[0] for u in utts]
    try:
        batch = _taped(tape, lambda: model.inference_batch(texts, speakers, languages))
        items = _taped(tape, lambda: list(model.inference_streams(texts, speakers, languages, chunk_frames=chunk)))
        for j in range(len(utts)):
            got = torch.cat([it[j] for it in items if j in it], 1)
            assert got.shape == batch[j].shape, (j, got.shape, batch[j].shape)
            assert_close(got, batch[j], 1e-3, 1e-4, f'{name}: text {j}')
            if precision == 'fp32':
                col = {k: v[:, j:j + 1] for k, v in tape.items()}
                solo = _taped(col, lambda: list(model.inference_stream(texts[j], None if speakers is None else speakers[j],
                                                                       None if languages is None else languages[j], chunk_frames=chunk)))
                parts = [it[j] for it in items if j in it]
                assert len(parts) == len(solo)
                for a, b in zip(parts, solo):
                    assert torch.equal(a, b), j
    finally:
        MaskSource.use_tape(None)
        _lib.set_precision('fp32')


def test_speech_streams_equal_speech_stream():
    """Seeded weights whose stop token never fires: three texts decode 40 frames each (the vocoder needs at least 21)."""
    from multilingual_text_to_speech_b200.params.params import Params as hp
    from multilingual_text_to_speech_b200.modules.tacotron2 import Tacotron
    from multilingual_text_to_speech_b200.modules.streaming import speech_stream, speech_streams
    hp.reset()
    hp.max_output_length = 40
    torch.manual_seed(70)
    model = Tacotron().cuda().eval()
    try:
        with torch.no_grad():
            model._decoder._stop_prediction.bias.fill_(-1e4)
        _lib.set_precision('fp32')
        voc = make_model('RAW', seed=60)
        widen = lambda m: torch.cat([m] * (80 // m.shape[0] + 1))[:80]      # noqa: E731 -- frame-local
        g = torch.Generator().manual_seed(71)
        texts = [torch.randint(3, 20, (n,), generator=g).cuda() for n in (17, 9, 30)]
        P = model._decoder._prenet._layers[0].weight.shape[0]
        tape = {k: (torch.rand(40, len(texts), P, generator=g) >= 0.5).to(torch.uint8) for k in ('step_prenet0', 'step_prenet1')}
        uni = [torch.rand(1, 40 * 275, 1, generator=g) for _ in texts]
        out = {i: [] for i in range(len(texts))}
        for i, c in _taped(tape, lambda: list(speech_streams(model, voc, texts, None, None, widen, 16, uni))):
            out[i].append(c)
        for i, text in enumerate(texts):
            col = {k: v[:, i:i + 1] for k, v in tape.items()}
            ref = _taped(col, lambda: torch.cat(list(speech_stream(model, voc, text, None, None, widen, 16, uni[i]))))
            assert ref.shape == (39 * 275,)
            assert torch.equal(torch.cat(out[i]), ref), i
    finally:
        hp.reset()


# ---- errors ----
def test_pool_errors():
    _lib.set_precision('fp32')
    m = make_model('RAW', seed=62)
    pool = m.stream_pool(2)
    a, b = pool.open(), pool.open(_tape(m, 30, 63)[:, :2000])
    with pytest.raises(ValueError, match='pool is full'):
        pool.open()
    with pytest.raises(ValueError, match='unknown or finished stream'):
        pool.feed(99, _mel(3, 64))
    with pytest.raises(ValueError, match='non-finite'):
        pool.feed(a, torch.full((80, 2), float('nan'), device='cuda'))
    pool.feed(a, _mel(20, 65))
    with pytest.raises(ValueError, match='at least 21'):
        pool.end(a)
    pool.feed(a, _mel(1, 66))
    pool.end(a)
    with pytest.raises(ValueError, match='has ended'):
        pool.feed(a, _mel(1, 67))
    pool.feed(b, _mel(30, 68))
    with pytest.raises(ValueError, match='uniform tape holds 2000 steps'):
        pool.run()
    with pytest.raises(ValueError, match='1 to 64 streams'):
        m.stream_pool(65)


def test_inference_streams_rejects_more_than_64_texts():
    model, utts, _ = _case('inf_batch_lj')
    with pytest.raises(ValueError, match='at most 64 texts'):
        next(model.inference_streams([utts[0][0]] * 65))
