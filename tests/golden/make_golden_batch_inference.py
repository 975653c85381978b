"""Golden vectors for batched synthesis (build container only; imports the unmodified reference):

    PYTHONDONTWRITEBYTECODE=1 python tests/golden/make_golden_batch_inference.py

Each case is one small model and several utterances.  The reference's own `Tacotron.inference` (modules/tacotron2.py:387-408) runs
once per utterance, batch 1, eval mode, with its always-on prenet dropout masks recorded in call order (2 per decoder step), as in
make_golden_inference.py.  A batched run must give every utterance exactly this output.  Cases:
  inf_batch_lj             vanilla encoder, location-sensitive attention, dropout cell; text lengths 2..30, different stop frames,
                           one utterance that runs to max_output_length
  inf_batch_generated      generated encoder, multi-speaker, multi-language with a decoder language embedding, zoneout: one-hot
                           languages, a code-switched and an accent-blended utterance
  inf_batch_convolutional  the separate_* configurations' convolutional encoder
  inf_batch_forward        forward attention
Every case holds a text of length 2 and one of length 30.  Stop frames: the trajectory of an utterance does not depend on the stop
projection, so pass 1 (stop disabled) records every candidate's stop logits; the bias and the chosen utterances then give at least one
utterance that runs to max_output_length (in inf_batch_lj: distinct cuts, exactly one of them none at all).
"""
import io
import os
import sys
import json
import zipfile
import numpy as np

REF = '/root/reference'
HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
from make_golden import SMALL      # noqa: E402

NARROW = dict(embedding_dimension=16, encoder_dimension=16, prenet_dimension=16, decoder_dimension=32, postnet_dimension=16,
              attention_dimension=16, max_output_length=40)
GEN = dict(multi_language=True, languages=['a', 'b', 'c'], generator_dim=4, generator_bottleneck_dim=2, embedding_dimension=8,
           encoder_dimension=8)
CASES = {
    # name: (hp overrides, number of utterances, speakers)
    'inf_batch_lj': (dict(), 5, 0),
    'inf_batch_generated': (dict(GEN, encoder_type='generated', language_embedding_dimension=4, decoder_regularization='zoneout',
                                 multi_speaker=True), 5, 3),
    'inf_batch_convolutional': (dict(GEN, encoder_type='convolutional', language_embedding_dimension=0, multi_speaker=True), 4, 2),
    'inf_batch_forward': (dict(attention_type='forward'), 4, 0),
}


def _languages(name, lengths, G, rng):
    """Per-character language weights [1, L, G] of every utterance: one-hots in several languages, then (generated case) one
    code-switched and one accent-blended utterance."""
    out = []
    for i, L in enumerate(lengths):
        w = np.zeros((1, L, G), dtype=np.float32)
        if name == 'inf_batch_generated' and i == 3:          # code-switching: a | c | b
            w[0, :L // 3, 0] = 1.0; w[0, L // 3:2 * L // 3, 2] = 1.0; w[0, 2 * L // 3:, 1] = 1.0
        elif name == 'inf_batch_generated' and i == 4:        # accent: b*0.75 + a*0.25 on a stretch, b elsewhere
            w[0, :, 1] = 1.0; w[0, 1:L - 1, 1] = 0.75; w[0, 1:L - 1, 0] = 0.25
        else:
            w[0, :, i % G] = 1.0
        out.append(w)
    return out


def _cut(logits, stop_frames):
    """The reference's exit (tacotron2.py:201-207) on a stop-logit trajectory: frames kept, or None if it never exits."""
    remaining = -1
    for i, fired in enumerate(logits >= 0):
        if not fired:
            continue
        if remaining == -1:
            remaining = stop_frames
            continue
        remaining -= 1
        if remaining == 0:
            return i + 1
    return None


def _save(path, arrays):
    """npz with fixed zip timestamps, so that a rerun reproduces the file byte for byte."""
    buf = io.BytesIO()
    with zipfile.ZipFile(buf, 'w', compression=zipfile.ZIP_DEFLATED) as zf:
        for k in sorted(arrays):
            info = zipfile.ZipInfo(k + '.npy', date_time=(1980, 1, 1, 0, 0, 0))
            info.compress_type = zipfile.ZIP_DEFLATED
            b = io.BytesIO()
            np.save(b, arrays[k], allow_pickle=False)
            zf.writestr(info, b.getvalue())
    with open(path, 'wb') as f:
        f.write(buf.getvalue())


def main():
    sys.path.insert(0, REF)
    import torch
    import torch.nn.functional as F
    import utils  # noqa: F401
    from params.params import Params as hp
    from modules.tacotron2 import Tacotron

    defaults = dict(hp.state_dict())
    real_dropout = F.dropout
    record = []

    def taped_dropout(input, p=0.5, training=True, inplace=False):
        if not training or p == 0.0:
            return input
        keep = (torch.rand(tuple(input.shape)) >= p).to(input.dtype)
        record.append(keep.detach().clone())
        return input * keep * (1.0 / (1.0 - p))

    for name, (over, n, speakers) in CASES.items():
        hp.load_state_dict(defaults)
        hp.load_state_dict(SMALL)
        hp.load_state_dict(NARROW)
        hp.load_state_dict(over)
        hp.language_number = len(hp.languages) if hp.multi_language else 0
        hp.speaker_number = speakers
        G = max(hp.language_number, 1)
        torch.manual_seed(sum(map(ord, name)))
        model = Tacotron()
        with torch.no_grad():
            model._attention._energy.weight.mul_(6.0)
            model._attention._memory.weight.mul_(3.0)
            model._attention._query.weight.mul_(3.0)
            for prm in model._decoder._attention_lstm.parameters():
                prm.mul_(2.0)
            model._decoder._stop_prediction.weight.mul_(4.0)
        model.eval()
        rng = np.random.default_rng(sum(map(ord, name)))
        # candidates: three times as many as needed, lengths spread over 2..30; the first two are the extremes 2 and 30
        lengths = [2, 30] + [int(x) for x in rng.integers(2, 31, size=3 * n - 2)]
        texts = [torch.from_numpy(rng.integers(1, hp.symbols_count() + 3, size=L).astype(np.int64)) for L in lengths]
        langs = _languages(name, lengths, G, rng) if hp.multi_language else [None] * len(lengths)
        spk = [torch.LongTensor([i % speakers]) for i in range(len(lengths))] if speakers else [None] * len(lengths)

        def run(i, bias):
            with torch.no_grad():
                model._decoder._stop_prediction.bias.fill_(bias)
            record.clear()
            torch.manual_seed(99 + i)
            F.dropout = taped_dropout
            try:
                with torch.no_grad():
                    lang = None if langs[i] is None else torch.from_numpy(langs[i])
                    return model.inference(texts[i].clone(), speaker=spk[i], language=lang)
            finally:
                F.dropout = real_dropout

        trajectories = []
        for i in range(len(texts)):
            captured = []
            hook = model._decoder._stop_prediction.register_forward_hook(lambda m, inp, o: captured.append(float(o)))
            run(i, -1000.0)
            hook.remove()
            trajectories.append(np.array(captured) + 1000.0)
        allv = np.concatenate(trajectories)
        if np.mean([t[:10].mean() for t in trajectories]) > np.mean([t[10:].mean() for t in trajectories]):
            with torch.no_grad():
                model._decoder._stop_prediction.weight.neg_()
            trajectories = [-t for t in trajectories]
            allv = -allv
        # required candidates: the shortest and longest texts and (generated case) the code-switched and accent-blended ones; then a
        # threshold under which at least one chosen utterance never exits.  inf_batch_lj, which the retirement test decodes, also needs
        # every utterance to stop at its own frame, exactly one of them never; the other cases keep their required utterances whatever
        # their cuts
        required = [0, 1] + ([3, 4] if name == 'inf_batch_generated' else [])
        distinct = name == 'inf_batch_lj'
        chosen, thr = None, None
        for q in np.linspace(0.3, 0.98, 69):
            t = float(np.quantile(allv, q))
            cuts = [_cut(tr - t, hp.stop_frames) for tr in trajectories]
            frames = [hp.max_output_length if c is None else c for c in cuts]
            pick = list(required)
            if distinct and (len({frames[i] for i in pick}) < len(pick) or sum(cuts[i] is None for i in pick) > 1):
                continue
            for i in range(len(cuts)):
                if len(pick) == n:
                    break
                taken = {frames[j] for j in pick} if distinct else set()
                has_never = any(cuts[j] is None for j in pick)
                if i in pick or frames[i] in taken or (cuts[i] is None and has_never) or (cuts[i] is not None and cuts[i] < 3):
                    continue
                if len(pick) == n - 1 and not has_never and cuts[i] is not None:
                    continue                      # the last place goes to an utterance that runs to max_output_length
                pick.append(i)
            if len(pick) == n and any(cuts[j] is None for j in pick):
                chosen, thr = sorted(pick), t
                break
        assert chosen is not None, f'{name}: no stop threshold gives distinct cuts'
        sd0 = {k: v.detach().clone() for k, v in model.state_dict().items()}
        res = {}
        Ts = []
        P = hp.prenet_dimension
        for j, i in enumerate(chosen):
            out = run(i, -thr)
            T = out.shape[1]
            assert len(record) == 2 * T, (len(record), T)
            Ts.append(T)
            res[f'tape{j}.step_prenet0'] = torch.stack([record[2 * k] for k in range(T)]).reshape(T, P).numpy().astype(np.uint8)
            res[f'tape{j}.step_prenet1'] = torch.stack([record[2 * k + 1] for k in range(T)]).reshape(T, P).numpy().astype(np.uint8)
            res[f'out{j}'] = out.detach().numpy()
            res[f'text{j}'] = texts[i].numpy()
            if langs[i] is not None:
                res[f'language{j}'] = langs[i]
            if spk[i] is not None:
                res[f'speaker{j}'] = spk[i].numpy()
        sd0['_decoder._stop_prediction.bias'] = model._decoder._stop_prediction.bias.detach().clone()
        assert hp.max_output_length in Ts and (len(set(Ts)) == len(Ts) or not distinct), Ts
        res['meta'] = np.frombuffer(json.dumps(dict(
            hp={k: v for k, v in hp.state_dict().items() if isinstance(v, (int, float, str, bool, list))}, n=len(chosen), T=Ts)).encode(),
            dtype=np.uint8)
        for k, v in sd0.items():
            res['sd.' + k] = v.numpy()
        path = os.path.join(HERE, name + '.npz')
        _save(path, res)
        print(f'{name}: texts {[len(texts[i]) for i in chosen]}, T={Ts} of max {hp.max_output_length}, '
              f'{os.path.getsize(path) / 1024:.0f} KiB')


if __name__ == '__main__':
    main()
