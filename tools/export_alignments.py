"""Export forced alignments of a dataset: per utterance, the symbol durations in frames and the alignment scores of a trained Tacotron
(Tacotron.align), as .npy files named by utterance id.

The ground-truth-aligned counterpart of the reference's gta.py, with its batching: grouped-encoder models that train on perfect batches
(hp.multi_language, hp.balanced_sampling and hp.perfect_sampling) get PerfectBatchSampler batches in dataset order, every other model
consecutive batches of --batch_size.  Items are the dataset's 5-tuples (speaker, language, symbol ids, mel [num_mels, frames], linear),
collated unsorted so that row b of a batch is its b-th index.  Per utterance `<id>.durations.npy` holds int32 [L_b] frames per symbol
(summing to the mel's frames) and `<id>.scores.npy` float64 [5]: focus rate, coverage, largest argmax jump, moves back (0 / 1) and the
path's log probability.  Prenet dropout stays on, as in gta.py; MaskSource.manual_seed(--seed) makes the masks repeatable.

With waveforms (the dataset's `waveforms` list, one 1-D array per item, whose 1 + len // hop frames cover the mel's), each utterance also
gets `<id>.pitch.npy`, float64 [L_b]: the mean pYIN f0 in Hz over the voiced frames of each symbol (utils.audio.pitch_batch,
functional.symbol_average; 0 for a symbol without voiced frames), and `<id>.energy.npy`, float64 [L_b]: the mean frame energy over each
symbol's frames (utils.audio.energy_batch).

    python tools/export_alignments.py --checkpoint ckpt.pt --dataset items.pt --output alignments
`items.pt`: torch.save({'ids': [...], 'items': [5-tuples]}), optionally with 'waveforms': [1-D float arrays].
"""
import argparse
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

SCORE_FIELDS = ('focus_rate', 'coverage', 'max_jump', 'moves_back', 'path_logp')


class ItemDataset(torch.utils.data.Dataset):
    """A list of the dataset's 5-tuples, with the `items[i]['language']` view PerfectBatchSampler reads."""

    def __init__(self, items):
        self._items = list(items)
        self.items = [{'language': int(it[1])} for it in self._items]

    def __len__(self):
        return len(self._items)

    def __getitem__(self, i):
        return self._items[i]


def batches(dataset, batch_size):
    """Index lists in gta.py's order."""
    from multilingual_text_to_speech_b200.params.params import Params as hp
    from multilingual_text_to_speech_b200.utils.samplers import PerfectBatchSampler
    if hp.multi_language and hp.balanced_sampling and hp.perfect_sampling:
        return list(PerfectBatchSampler(dataset, hp.languages, batch_size, shuffle=False))
    return [list(range(i, min(i + batch_size, len(dataset)))) for i in range(0, len(dataset), batch_size)]


def symbol_prosody(durations, mel_lengths, waves):
    """(per-symbol mean voiced f0, per-symbol mean energy), each float64 [B, L], of B waveforms under durations [B, L] (CPU)."""
    from multilingual_text_to_speech_b200.functional import symbol_average
    from multilingual_text_to_speech_b200.utils import audio
    pitches, energies = audio.pitch_batch(waves), audio.energy_batch(waves)
    T = max(len(e) for e in energies)
    f0 = torch.zeros(len(waves), T, dtype=torch.float64)
    energy = torch.zeros(len(waves), T, dtype=torch.float64)
    voiced = torch.zeros(len(waves), T, dtype=torch.bool)
    for b, ((f, _), e) in enumerate(zip(pitches, energies)):
        if len(e) < int(mel_lengths[b]):
            raise ValueError(f'waveform {b} has {len(e)} frames for a mel of {int(mel_lengths[b])}')
        f0[b, :len(f)] = torch.from_numpy(np.nan_to_num(f.astype(np.float64)))
        voiced[b, :len(f)] = torch.from_numpy(~np.isnan(f))
        energy[b, :len(e)] = torch.from_numpy(e.astype(np.float64))
    return symbol_average(f0, durations, voiced).numpy(), symbol_average(energy, durations).numpy()


def export(model, dataset, ids, out_dir, batch_size=32, waveforms=None):
    """Align every item of `dataset` (ItemDataset or any dataset of the 5-tuples with `items`) and write its files under out_dir; with
    `waveforms` (one 1-D array per item) the per-symbol pitch and energy as well."""
    from multilingual_text_to_speech_b200.params.params import Params as hp
    from multilingual_text_to_speech_b200.utils import to_gpu
    from multilingual_text_to_speech_b200.utils.data import TextToSpeechCollate
    os.makedirs(out_dir, exist_ok=True)
    collate = TextToSpeechCollate(False, hp.num_mels, hp.stop_frames, hp.multi_speaker, hp.multi_language)
    for idx in batches(dataset, batch_size):
        text, text_len, mel, _, mel_len, _, speakers, languages = map(to_gpu, collate([dataset[i] for i in idx]))
        res = model.align(text, text_len, mel, mel_len, speakers, languages)
        durations = res.durations.cpu().numpy()
        scores = torch.stack([getattr(res, f).double() for f in SCORE_FIELDS], 1).cpu().numpy()
        if waveforms is not None:
            pitch, energy = symbol_prosody(res.durations.cpu(), mel_len.cpu(), [np.asarray(waveforms[i], dtype=np.float32) for i in idx])
        for row, i in enumerate(idx):
            np.save(os.path.join(out_dir, f'{ids[i]}.durations.npy'), durations[row, :int(text_len[row])], allow_pickle=False)
            np.save(os.path.join(out_dir, f'{ids[i]}.scores.npy'), scores[row], allow_pickle=False)
            if waveforms is not None:
                np.save(os.path.join(out_dir, f'{ids[i]}.pitch.npy'), pitch[row, :int(text_len[row])], allow_pickle=False)
                np.save(os.path.join(out_dir, f'{ids[i]}.energy.npy'), energy[row, :int(text_len[row])], allow_pickle=False)


def main():
    parser = argparse.ArgumentParser(description=__doc__.split('\n\n')[0])
    parser.add_argument('--checkpoint', required=True, help='reference-format model checkpoint')
    parser.add_argument('--dataset', required=True, help="torch.save'd {'ids': [...], 'items': [5-tuples]}")
    parser.add_argument('--output', required=True, help='output directory')
    parser.add_argument('--batch_size', type=int, default=32)
    parser.add_argument('--seed', type=int, default=1234, help='MaskSource seed of the prenet dropout masks')
    args = parser.parse_args()
    from multilingual_text_to_speech_b200.rng import MaskSource
    from multilingual_text_to_speech_b200.utils import build_model
    model = build_model(args.checkpoint)
    data = torch.load(args.dataset)
    MaskSource.manual_seed(args.seed)
    export(model, ItemDataset(data['items']), data['ids'], args.output, args.batch_size, data.get('waveforms'))


if __name__ == '__main__':
    main()
