"""Grouped encoders on batches that are not in the reference layout: each utterance encoded under its own language's weights and
batch-norm statistics (modules/encoder.py GroupLayout, b200tts_convblock_*_counts), against the fp64 per-language oracle of
tests/routed_encoder_oracle.py, at small and at the real dimensions, and against the reference's golden vectors after a permutation."""
import pytest
import torch

import model_cases
import routed_encoder_oracle as RO
from helpers import Golden, assert_close

pytestmark = pytest.mark.gpu


@pytest.fixture(scope='module', autouse=True)
def _built():
    import __graft_entry__ as entry
    entry.build()
    assert torch.cuda.is_available()


def _precision(mode):
    from multilingual_text_to_speech_b200 import _lib
    _lib.set_precision(mode)


def _encoder(kind, F_in, E, G, seed):
    from multilingual_text_to_speech_b200.modules.encoder import ConvolutionalEncoder, GeneratedConvolutionalEncoder
    torch.manual_seed(seed)
    if kind == 'generated':
        enc = GeneratedConvolutionalEncoder(F_in, E, 0.05, 8, 4, groups=G)
    else:
        enc = ConvolutionalEncoder(F_in, E, 0.05, groups=G)
    with torch.no_grad():                  # non-trivial running statistics for the eval cases
        for name, buf in enc.named_buffers():
            if 'running_mean' in name:
                buf.copy_(0.1 * torch.randn_like(buf))
            elif 'running_var' in name:
                buf.copy_(0.5 + torch.rand_like(buf))
    return enc.cuda()


def _run_model_encoder(enc, x, ids, tape, dout):
    from multilingual_text_to_speech_b200.rng import MaskSource
    for p in enc.parameters():
        p.grad = None
    xg = x.cuda().requires_grad_(True)
    MaskSource.use_tape(tape)
    try:
        out = enc(xg, None, torch.tensor(ids).unsqueeze(1).expand(-1, x.shape[1]))
    finally:
        MaskSource.use_tape(None)
    grads = None
    if dout is not None:
        out.backward(dout.cuda())
        grads = {k: p.grad.detach().clone() if p.grad is not None else torch.zeros_like(p) for k, p in enc.named_parameters()}
    torch.cuda.synchronize()
    return out.detach(), grads


def _compare(enc, out, grads, bufs_before, ref, ref_grads, ref_bufs, ids, mode, what):
    """fp32: outputs within rtol 1e-3 / atol 1e-4, each gradient within 2e-3 of its largest element.  bf16 (the wgmma convolutions
    round activations and weights to bf16 in each of the 14 blocks): mean |out - oracle| within 2 % of mean |oracle|, and each
    gradient normwise within 0.3 (|g - r|_2 <= 0.3 |r|_2), the coarse bound DESIGN section 11 uses for bf16 gradients, and each
    running-statistics buffer within 2 % of its largest element."""
    if mode == 'fp32':
        assert_close(out, ref, 1e-3, 1e-4, f'{what}: out')
    else:
        rel = float((out.double().cpu() - ref.cpu()).abs().mean() / ref.abs().mean())
        print(f'{what}: bf16 relative mean |out - oracle| {rel:.3e}')
        assert rel < 2e-2, f'{what}: bf16 relative mean |out - oracle| {rel:.3e}'
    worst = 0.0
    for k, g in (grads or {}).items():
        r = ref_grads[k].cpu()
        scale = float(r.abs().max())
        if scale == 0.0:
            assert bool((g == 0).all()), f'{what}: grad {k} should be exactly 0'
            continue
        if mode == 'fp32':
            err = float((g.double().cpu() - r).abs().max()) / scale
            bound = 2e-3
        else:
            err = float((g.double().cpu() - r).norm() / r.norm())
            bound = 0.3
        worst = max(worst, err)
        assert err <= bound, f'{what}: grad {k} relative error {err:.3e}'
    G = enc._groups
    absent = [g for g in range(G) if g not in set(int(i) for i in ids)]
    for name, buf in enc.named_buffers():
        if 'running' not in name:
            continue
        C = buf.shape[0] // G
        if mode == 'fp32':
            assert_close(buf, ref_bufs[name], 1e-3, 1e-5, f'{what}: {name}')
        else:           # the batch statistics of bf16 products: within 2 % of the buffer's largest value
            err = float((buf.double().cpu() - ref_bufs[name].cpu()).abs().max())
            assert err <= 2e-2 * float(ref_bufs[name].abs().max()), f'{what}: {name} differs by {err:.3e}'

        for g in absent:
            assert torch.equal(buf[g * C:(g + 1) * C].cpu(), bufs_before[name][g * C:(g + 1) * C]), f'{what}: {name} of absent {g} moved'
    if grads is not None and absent and hasattr(enc, '_embedding'):
        for g in absent:
            assert bool((grads['_embedding.weight'][g] == 0).all()), f'{what}: absent language {g} has an embedding gradient'
    if grads is not None and absent and not hasattr(enc, '_embedding'):
        for k, gr in grads.items():
            C = gr.shape[0] // G
            for g in absent:
                assert bool((gr[g * C:(g + 1) * C] == 0).all()), f'{what}: absent language {g} has a gradient in {k}'
    return worst


IDS = [2, 0, 0, 3, 2, 2, 0]          # B = 7, G = 4: language 1 absent, language 3 a single utterance


@pytest.mark.parametrize('training', [True, False], ids=['train', 'eval'])
@pytest.mark.parametrize('mode', ['fp32', 'bf16'])
@pytest.mark.parametrize('kind', ['generated', 'convolutional'])
def test_routed_encoder_against_per_language_oracle(kind, mode, training):
    G, F_in, E, L = 4, 32, 24, 20
    enc = _encoder(kind, F_in, E, G, seed=1).train(training)
    g = torch.Generator().manual_seed(2)
    x = torch.randn(len(IDS), L, F_in, generator=g)
    dout = torch.randn(len(IDS), L, E, generator=g)
    tape = RO.routed_tape(enc, IDS, L, 0.05, g) if training else None
    before = {k: v.detach().cpu().clone() for k, v in enc.named_buffers()}
    ref, ref_grads, ref_bufs = RO.encode(enc, x, IDS, tape, training, dout, device='cuda')
    _precision(mode)
    try:
        out, grads = _run_model_encoder(enc, x, IDS, tape, dout)
    finally:
        _precision('fp32')
    worst = _compare(enc, out, grads, before, ref, ref_grads, ref_bufs, IDS, mode, f'{kind} {mode}')
    print(kind, mode, 'train' if training else 'eval', f'worst relative gradient error {worst:.3e}', '(normwise)' if mode == 'bf16' else '')


@pytest.mark.parametrize('kind', ['generated', 'convolutional'])
def test_order_preserving_permutation_permutes_outputs_bitwise(kind):
    """Moving utterances around while keeping each language's relative order keeps the routed layout, so the outputs permute bit for bit."""
    G, F_in, E, L = 4, 32, 24, 20
    enc = _encoder(kind, F_in, E, G, seed=3).train()
    g = torch.Generator().manual_seed(4)
    x = torch.randn(len(IDS), L, F_in, generator=g)
    tape = RO.routed_tape(enc, IDS, L, 0.05, g)
    perm = [3, 1, 0, 4, 2, 6, 5]          # languages 3, 0, 2, 2, 0, 0, 2: each language's utterances in their original order
    ids_p = [IDS[i] for i in perm]
    for lang in range(G):
        assert [i for i in perm if IDS[i] == lang] == [i for i in range(len(IDS)) if IDS[i] == lang]
    state = {k: v.clone() for k, v in enc.state_dict().items()}
    a, _ = _run_model_encoder(enc, x, IDS, tape, None)
    enc.load_state_dict(state)
    b, _ = _run_model_encoder(enc, x[perm], ids_p, tape, None)
    assert torch.equal(a[perm], b)


def _permute_tape(tape, perm, B):
    out = {}
    for k, v in tape.items():
        if k.startswith('enc') or v.dim() == 1:
            out[k] = v                       # the encoder masks are in the grouped layout, which a language-sorted batch keeps
        elif v.shape[0] == B:
            out[k] = v[perm]
        else:
            out[k] = v[:, perm]
    return out


def test_golden_generated_training_language_sorted():
    """tests/golden/generated_training.npz (B = 6, G = 3, languages b % 3) sorted by language takes the routed path; un-permuted, its
    encoder output is bit-identical to the unpermuted run and the rest meets the golden tolerances of model_cases.run_golden."""
    from multilingual_text_to_speech_b200.modules.tacotron2 import TacotronLoss
    from multilingual_text_to_speech_b200.modules.encoder import encoder_layout
    from multilingual_text_to_speech_b200.rng import MaskSource
    from multilingual_text_to_speech_b200.params.params import Params as hp
    g = Golden('generated_training')
    dev = torch.device('cuda:0')
    B = g.inputs['text'].shape[0]
    langs = g.inputs['languages']
    perm = sorted(range(B), key=lambda b: (int(langs[b]), b))
    inv = [perm.index(b) for b in range(B)]
    assert encoder_layout(langs[perm], B, 3) is not None and encoder_layout(langs, B, 3) is None

    def run(order):
        model = model_cases.build_model(g, dev)
        i = {k: v[order].to(dev) for k, v in g.inputs.items()}
        MaskSource.use_tape(_permute_tape(g.tape, order, B))
        try:
            outs = model(i['text'], i['text_length'], i['target'], i['target_length'], i.get('speakers'), i.get('languages'), g.tf)
        finally:
            MaskSource.use_tape(None)
        crit = TacotronLoss(hp.guided_attention_steps, g.meta['guided_g'], hp.guided_attention_gain)
        post, pre, stop, align, spk, enc = outs
        loss, parts = crit(i['text_length'], i['target_length'], pre, i['target'], post, i['target'], stop, i['stop_target'], align,
                           i.get('speakers'), spk, enc, None)
        loss.backward()
        torch.cuda.synchronize()
        return model, outs, parts

    _, plain, _ = run(list(range(B)))
    model, routed, parts = run(perm)
    post, pre, stop, align, spk, enc = (None if t is None else t.detach()[inv] for t in routed)
    assert torch.equal(enc, plain[5].detach()), 'encoder output differs from the unpermuted run'
    for key, got in (('enc', enc), ('align', align), ('pre', pre), ('stop', stop), ('post', post), ('spk_pred', spk)):
        if got is not None:
            assert_close(got, g.out[key], 1e-3, 1e-4, f'sorted: {key}')
    for k, v in parts.items():
        assert abs(float(v) - g.losses[k]) < 2e-4 * max(1.0, abs(g.losses[k])), (k, float(v), g.losses[k])
    for k, prm in model.named_parameters():
        ref = g.grad[k]
        got = prm.grad if prm.grad is not None else torch.zeros_like(prm)
        scale = float(ref.abs().max()) + 1e-12
        assert_close(got, ref, 3e-3, 3e-4 * scale + 1e-9, f'sorted: grad {k}')
    sd_after = model.state_dict()
    for k, ref in g.sd_after.items():
        if 'num_batches' not in k:
            assert_close(sd_after[k], ref, 1e-3, 1e-5, f'sorted: {k}')


def _full_batch(hp, ids, L, T, seed):
    g = torch.Generator().manual_seed(seed)
    B = len(ids)
    return dict(text=torch.randint(1, hp.symbols_count() + 3, (B, L), generator=g), text_length=torch.full((B,), L),
                target=torch.randn(B, hp.num_mels, T, generator=g), target_length=torch.full((B,), T),
                stop_target=torch.zeros(B, T), languages=torch.tensor(ids))


def _imbalanced_60(G):
    ids = []
    for lang, n in enumerate([9, 1, 0, 8, 7, 6, 8, 7, 6, 8][:G]):     # language 1 a singleton, language 2 absent
        ids += [lang] * n
    g = torch.Generator().manual_seed(9)
    return [ids[i] for i in torch.randperm(len(ids), generator=g).tolist()]


@pytest.mark.parametrize('mode', ['fp32', 'bf16'])
@pytest.mark.parametrize('batch', ['B64', 'B60_imbalanced'])
def test_generated_training_real_dimensions(batch, mode):
    """generated_training (zoneout, G = 10) training step at L = 180, T = 900: the encoder output, every encoder gradient (for the
    gradient the rest of the model sends back) and the running statistics against the per-language fp64 oracle; then FusedAdam steps
    leave an absent language's parameters bit for bit unchanged."""
    from multilingual_text_to_speech_b200 import configs
    from multilingual_text_to_speech_b200.modules.tacotron2 import Tacotron, TacotronLoss
    from multilingual_text_to_speech_b200.rng import MaskSource
    from multilingual_text_to_speech_b200.optim import FlatParams, FusedAdam
    from multilingual_text_to_speech_b200.distributed import GradBucket
    hp = configs.apply('generated_training', decoder_regularization='zoneout')
    G, L, T = hp.language_number, 180, 900
    ids = [b % G for b in range(64)] if batch == 'B64' else _imbalanced_60(G)
    torch.manual_seed(0)
    model = Tacotron().cuda().train()
    enc_mod = model._encoder
    b = {k: v.cuda() for k, v in _full_batch(hp, ids, L, T, 5).items()}
    g = torch.Generator().manual_seed(6)
    tape = RO.routed_tape(enc_mod, ids, L, 0.05, g)
    before = {k: v.detach().cpu().clone() for k, v in enc_mod.named_buffers()}
    crit = TacotronLoss(hp.guided_attention_steps, hp.guided_attention_toleration, hp.guided_attention_gain)
    captured = {}

    def hook(mod, inp, out):
        captured['x'] = inp[0].detach().clone()
        out.register_hook(lambda gr: captured.__setitem__('dout', gr.detach().clone()))
    h = enc_mod.register_forward_hook(hook)
    _precision(mode)
    MaskSource.use_tape({k: v.cuda() for k, v in tape.items()})
    try:
        post, pre, stop, align, spk, enc = model(b['text'], b['text_length'], b['target'], b['target_length'], None, b['languages'], 1.0)
        MaskSource.use_tape(None)
        loss, _ = crit(b['text_length'], b['target_length'], pre, b['target'], post, b['target'], stop, b['stop_target'], align, None,
                       spk, enc, None)
        loss.backward()
        torch.cuda.synchronize()
    finally:
        MaskSource.use_tape(None)
        _precision('fp32')
        h.remove()
    assert bool(torch.isfinite(loss)), float(loss)
    grads = {k: p.grad.detach().clone() if p.grad is not None else torch.zeros_like(p) for k, p in enc_mod.named_parameters()}
    # the oracle runs from this step's starting statistics
    after = {k: v.detach().clone() for k, v in enc_mod.named_buffers()}
    with torch.no_grad():
        for k, v in enc_mod.named_buffers():
            v.copy_(before[k])
    ref, ref_grads, ref_bufs = RO.encode(enc_mod, captured['x'], ids, tape, True, captured['dout'], device='cuda')
    with torch.no_grad():
        for k, v in enc_mod.named_buffers():
            v.copy_(after[k])
    worst = _compare(enc_mod, enc.detach(), grads, before, ref, ref_grads, ref_bufs, ids, mode, f'{batch} {mode}')
    print(batch, mode, f'loss {float(loss):.5f}, worst relative encoder gradient error {worst:.3e}')
    if batch != 'B60_imbalanced' or mode != 'fp32':
        return
    absent = [lang for lang in range(G) if lang not in ids]
    assert absent
    emb0 = enc_mod._embedding.weight.detach().clone()
    flat, bucket = FlatParams(model), GradBucket(model, 1)
    opt = FusedAdam(flat, bucket, lr=1e-3, weight_decay=0.0, max_grad_norm=1.0)
    for _ in range(3):
        bucket.zero()
        post, pre, stop, align, spk, enc = model(b['text'], b['text_length'], b['target'], b['target_length'], None, b['languages'], 1.0)
        loss, _ = crit(b['text_length'], b['target_length'], pre, b['target'], post, b['target'], stop, b['stop_target'], align, None,
                       spk, enc, None)
        loss.backward()
        opt.step()
    torch.cuda.synchronize()
    emb = enc_mod._embedding.weight.detach()
    for lang in absent:
        assert torch.equal(emb[lang], emb0[lang]), f'absent language {lang}: embedding changed'
    present = [lang for lang in range(G) if lang in ids]
    assert not torch.equal(emb[present], emb0[present])


def test_cuda_labels_written_in_place_are_read_again():
    """CUDA labels are read at every forward: an in-place change of the same labels tensor re-routes the batch, and each result equals
    the one from CPU labels."""
    G, F_in, E, L = 4, 32, 24, 20
    enc = _encoder('generated', F_in, E, G, seed=5).eval()
    x = torch.randn(len(IDS), L, F_in, generator=torch.Generator().manual_seed(6)).cuda()
    lab = torch.tensor(IDS, device='cuda')
    other = [0, 1, 2, 3, 0, 1, 2]
    with torch.no_grad():
        a = enc(x, None, lab.unsqueeze(1).expand(-1, L))
        a_cpu = enc(x, None, torch.tensor(IDS).unsqueeze(1).expand(-1, L))
        lab.copy_(torch.tensor(other))
        b = enc(x, None, lab.unsqueeze(1).expand(-1, L))
        b_cpu = enc(x, None, torch.tensor(other).unsqueeze(1).expand(-1, L))
    assert torch.equal(a, a_cpu) and torch.equal(b, b_cpu) and not torch.equal(a, b)


@pytest.mark.parametrize('kind', ['generated', 'convolutional'])
def test_inference_mode_with_cuda_labels(kind):
    """An eval forward under torch.inference_mode with CUDA labels (inference tensors), in the reference layout and routed, gives
    bitwise what the same forward gives under no_grad."""
    G, F_in, E, L = 4, 32, 24, 20
    enc = _encoder(kind, F_in, E, G, seed=7).eval()
    x = torch.randn(8, L, F_in, generator=torch.Generator().manual_seed(8)).cuda()
    for ids in ([b % G for b in range(8)], IDS + [1]):
        with torch.no_grad():
            ref = enc(x, None, torch.tensor(ids, device='cuda').unsqueeze(1).expand(-1, L))
        with torch.inference_mode():
            lab = torch.tensor(ids, device='cuda')
            assert lab.is_inference()
            got = enc(x, None, lab.unsqueeze(1).expand(-1, L))
        assert torch.equal(got, ref), ids


@pytest.mark.parametrize('batch', ['B64', 'B60_imbalanced'])
def test_whole_model_against_oracle_with_per_language_encoder(batch):
    """The whole generated_training model (real widths, G = 10, zoneout) on a routed batch against the fp64 oracle of
    oracle/tacotron_oracle.py whose encoder is the per-language one: encoder output, spectrograms, stop logits and alignments in fp32
    mode within the bounds of tests/test_gpu_model.py, and the mel gate of its bf16 test in bf16 mode.  At L = 48, T = 24: the fp64
    decoder oracle over 900 steps is not run here (test_generated_training_real_dimensions checks the encoder at L = 180, T = 900)."""
    import types
    from multilingual_text_to_speech_b200 import configs
    from multilingual_text_to_speech_b200.modules.tacotron2 import Tacotron
    from multilingual_text_to_speech_b200.rng import MaskSource
    from oracle import tacotron_oracle as O
    hp = configs.apply('generated_training', decoder_regularization='zoneout')
    G, L, T = hp.language_number, 48, 24
    ids = [b % G for b in range(64)] if batch == 'B64' else _imbalanced_60(G)
    B = len(ids)
    torch.manual_seed(0)
    model = Tacotron().train()
    g = torch.Generator().manual_seed(5)
    text = torch.randint(1, hp.symbols_count() + 3, (B, L), generator=g)
    lens = torch.randint(L // 2, L + 1, (B,), generator=g)
    lens[0] = L
    for i in range(B):
        text[i, lens[i]:] = 0
    mel = torch.randn(B, hp.num_mels, T, generator=g)
    tlens = torch.full((B,), T)
    lang = torch.tensor(ids)
    D, P = hp.decoder_dimension, hp.prenet_dimension
    keep = lambda shape, p: (torch.rand(*shape, generator=g) >= p).float()   # noqa: E731
    tape = {'teacher': torch.ones(T, dtype=torch.bool), 'prenet0': keep((B, T + 1, P), 0.5), 'prenet1': keep((B, T + 1, P), 0.5),
            'att_h': keep((T, B, D), 0.1), 'att_c': keep((T, B, D), 0.1), 'gen_h': keep((T, B, D), 0.1), 'gen_c': keep((T, B, D), 0.1)}
    tape.update(RO.routed_tape(model._encoder, ids, L, 0.05, g))
    sd = {k: v.detach().double() for k, v in model.state_dict().items()}
    for k in list(sd):
        if k.startswith('_decoder._prenet.') or k.startswith('_decoder._attention.'):
            sd[k] = sd[k[len('_decoder.'):]]
    ns = types.SimpleNamespace(**hp.state_dict())
    enc_cpu = model._encoder

    def per_language_encoder(sd_, hp_, embedded, tape_, training, stats=None):
        return RO.encode(enc_cpu, embedded, ids, tape_, training, device='cpu')[0]
    reference_encoder = O.generated_encoder
    O.generated_encoder = per_language_encoder
    try:
        with torch.no_grad():
            post_o, pre_o, stop_o, align_o, _, enc_o = O.tacotron_forward(sd, ns, text, lens, mel.double(), tlens, None, lang, tape,
                                                                          training=True)
    finally:
        O.generated_encoder = reference_encoder
    dev = torch.device('cuda:0')
    model = model.to(dev)
    state = {k: v.clone() for k, v in model.state_dict().items()}
    results = {}
    for mode in ('fp32', 'bf16'):
        model.load_state_dict(state)
        _precision(mode)
        MaskSource.use_tape(tape)
        try:
            with torch.no_grad():
                post, pre, stop, align, _, enc = model(text.to(dev), lens.to(dev), mel.to(dev), tlens.to(dev), None, lang.to(dev), 1.0)
        finally:
            MaskSource.use_tape(None)
            _precision('fp32')
        results[mode] = {'pre_l1': float((pre.cpu().double() - pre_o).abs().mean()), 'post_l1': float((post.cpu().double() - post_o).abs().mean()),
                         'argmax': float((align.cpu().argmax(2) == align_o.argmax(2)).float().mean())}
        if mode == 'fp32':
            assert_close(enc, enc_o, 1e-3, 1e-4, 'enc')
            assert_close(pre, pre_o, 1e-3, 1e-4, 'pre')
            assert_close(align, align_o, 1e-3, 1e-4, 'align')
            assert_close(stop, stop_o, 1e-3, 1e-4, 'stop')
            assert torch.equal(align.cpu().argmax(2), align_o.argmax(2))
    print(batch, 'whole model vs fp64 oracle with the per-language encoder:', results)
    assert results['bf16']['pre_l1'] < 1e-3 and results['bf16']['post_l1'] < 5e-2, results
