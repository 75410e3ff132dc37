"""The paired (amateur / professional) singing binarizer of the SVB task (reference data_gen/singing/binarize_para.py,
``PopBuTFyENBinarizer`` / ``PopBuTFyENSpkEMBinarizer``, config ``para_bin.yaml``), batched on the GPU.

Pairing, splits, the speaker map, the ``max_mel_tech_gap`` skip (logged to ``bad_case.txt``), the "Empty f0" skip and the files
written follow the reference.  The reference processes one pair per CPU worker; here the pairs of a split are grouped by seconds of
audio (``batch_seconds``, VocoderBinarizer's grouping) and each group costs three device calls: ``wav2spec_batch`` over both takes of
every pair, ``get_pitch_batch`` over the takes that passed the gap check, and ``align_pitch`` (EHSADTW, the reference's choice) over
the pairs that kept a voiced f0.  The takes reach the device through ``utils.audio.load_takes`` (one copy, off-rate files resampled
there); ``wav2spec_batch`` and ``get_pitch_batch`` copy their results back.  Items are written in metadata order.

Each item holds exactly what ``MultiSpkEmbDataset`` reads: ``item_name``, ``mel`` / ``prof_mel`` [T, 80], ``f0`` / ``prof_f0`` (Hz),
``pitch`` / ``prof_pitch`` (coarse ids), ``a2p_f0_alignment`` [T_prof] and ``multi_spk_emb`` [1 + spk_emb_num, 256].  Per split:
``{prefix}.data`` / ``.idx``, ``{prefix}_lengths.npy`` (the longer take of each pair) and ``{prefix}_f0s_mean_std.npy`` over the
nonzero f0 of both takes.

``multi_spk_emb`` is the item's own embedding from ``spk_emb_data_dir`` followed by ``spk_emb_num`` embeddings of pieces of the same
song (the last one repeated when there are fewer).  The reference shuffles the pieces with Python's unseeded global generator in
worker processes, so its datasets do not reproduce; here the shuffle is seeded from the item name, so the same input gives the same
dataset.

The task also reads ``phone_set.json`` from ``binary_data_dir``; the reference binarizer does not write it, and neither does this
one: it checks for the file before any work and names it when it is missing."""
import os
import random
import re
import traceback
import zlib

import numpy as np

from neuralsvb_b200.data_gen.singing.binarize import BinarizationError, SingingBinarizer, split_train_test_set
from neuralsvb_b200.data_gen.tts.base_binarizer import VocoderBinarizer
from neuralsvb_b200.data_gen.tts.data_gen_utils import get_pitch_batch, pitch_frames
from neuralsvb_b200.modules.voice_conversion.dtw.core import align_pitch
from neuralsvb_b200.utils.hparams import hparams
from neuralsvb_b200.utils.indexed_datasets import IndexedDatasetBuilder
from neuralsvb_b200.vocoders.base_vocoder import get_vocoder_cls

ALIGN_METHOD = 'EHSADTW'


class PopBuTFyENBinarizer(SingingBinarizer):
    def load_meta_data(self):
        """Keep the ``#singing#`` amateur items whose ``Professional`` counterpart exists."""
        super().load_meta_data()
        self.amateur2profwavfn = {}
        new_item_names = []
        n_utt_ds = {k: 0 for k in hparams['datasets']}
        unpaired_num = 0
        for item_name in self.item_names:
            if '#singing#' not in item_name or 'Professional' in item_name:
                continue
            for dataset in hparams['datasets']:
                if len(re.findall(rf'{dataset}', item_name)) > 0:
                    prof_item = item_name.replace('Amateur', 'Professional')
                    if self.item2wavfn.get(prof_item) is not None and os.path.exists(self.item2wavfn[prof_item]):
                        self.amateur2profwavfn[item_name] = self.item2wavfn[prof_item]
                        new_item_names.append(item_name)
                        n_utt_ds[dataset] += 1
                    else:
                        unpaired_num += 1
                    break
        print('n_utt_ds: ', n_utt_ds, 'Unpaired data: ', unpaired_num)
        self.item_names = new_item_names
        self._train_item_names, self._test_item_names = split_train_test_set(self.item_names)

    def meta_data(self, prefix):
        for item_name, wav_fn, spk_id in super().meta_data(prefix):
            yield item_name, wav_fn, spk_id, self.amateur2profwavfn[item_name]

    def process(self):
        fn = os.path.join(hparams['binary_data_dir'], 'phone_set.json')
        if not os.path.exists(fn):
            raise FileNotFoundError(f'{fn} is missing: the SVB task reads phone_set.json from binary_data_dir, and the paired '
                                    'binarizer does not write it (nor does the reference); put the phone set there first')
        super().process()

    def extra_fields(self, res):
        """Fields a subclass adds to a finished item; raise to skip the item."""

    def process_data(self, prefix):
        data_dir = hparams['binary_data_dir']
        voc = get_vocoder_cls(hparams)
        builder = IndexedDatasetBuilder(f'{data_dir}/{prefix}')
        mel_lengths, f0s, total_sec = [], [], 0.0
        metas = list(self.meta_data(prefix))
        grouper = VocoderBinarizer([], binary_data_dir=data_dir, batch_seconds=hparams.get('binarize_batch_seconds', 600.0))
        for batch in grouper._batches(metas, wavs_of=lambda m: (m[1], m[3])):
            for res in self.process_batch(voc, batch):
                builder.add_item(res)
                mel_lengths.append(max(len(res['mel']), len(res['prof_mel'])))
                total_sec += len(res['mel']) * hparams['hop_size'] / hparams['audio_sample_rate']
                f0s += [res['f0'], res['prof_f0']]
        builder.finalize()
        np.save(f'{data_dir}/{prefix}_lengths.npy', mel_lengths)
        if f0s:
            f = np.concatenate(f0s, 0)
            f = f[f != 0]
            np.save(f'{data_dir}/{prefix}_f0s_mean_std.npy', [np.mean(f).item(), np.std(f).item()])
        print(f"| {prefix} total duration: {total_sec:.3f}s")

    def process_batch(self, voc, batch):
        """The finished items of one group of pairs, in metadata order (three device calls)."""
        B = len(batch)
        specs = voc.wav2spec_batch([m[1] for m in batch] + [m[3] for m in batch])
        gap = hparams.get('max_mel_tech_gap')
        kept = []
        for m, (wav, mel), (prof_wav, prof_mel) in zip(batch, specs[:B], specs[B:]):
            item_name, wav_fn = m[0], m[1]
            if gap is not None and abs(mel.shape[0] - prof_mel.shape[0]) > gap:
                with open(hparams['binary_data_dir'] + '/bad_case.txt', 'a+') as wf:
                    wf.write('Gap is too large: ' + item_name + str(mel.shape) + str(prof_mel.shape) + '\n')
                continue
            if min(pitch_frames(len(wav), hparams), pitch_frames(len(prof_wav), hparams)) < 1:
                print(f"| Skip item (shorter than one pitch window). item_name: {item_name}, wav_fn: {wav_fn}")
                continue
            kept.append((m, wav, mel, prof_wav, prof_mel))
        if not kept:
            return []
        pitches = get_pitch_batch([k[1] for k in kept] + [k[3] for k in kept], [k[2] for k in kept] + [k[4] for k in kept], hparams)
        voiced = []
        for i, (m, wav, mel, prof_wav, prof_mel) in enumerate(kept):
            (f0, pitch), (prof_f0, prof_pitch) = pitches[i], pitches[len(kept) + i]
            if sum(f0) == 0 or sum(prof_f0) == 0:
                print(f"| Skip item (Empty f0). item_name: {m[0]}, wav_fn: {m[1]}")
                continue
            voiced.append({'item_name': m[0], 'mel': mel, 'prof_mel': prof_mel, 'f0': f0, 'pitch': pitch, 'prof_f0': prof_f0,
                           'prof_pitch': prof_pitch, '_wav_fn': m[1]})
        if not voiced:
            return []
        aligns = align_pitch([r['f0'] for r in voiced], [r['prof_f0'] for r in voiced], ALIGN_METHOD)
        out = []
        for res, a in zip(voiced, aligns):
            res['a2p_f0_alignment'] = a
            wav_fn = res.pop('_wav_fn')
            try:
                self.extra_fields(res)
            except BinarizationError as e:
                print(f"| Skip item ({e}). item_name: {res['item_name']}, wav_fn: {wav_fn}")
                continue
            except Exception:
                traceback.print_exc()
                print(f"| Skip item. item_name: {res['item_name']}, wav_fn: {wav_fn}")
                continue
            out.append(res)
        return out


def song_pieces(item_name, item_names):
    """The items of the same song as ``item_name`` (the reference's rule: its name up to the last '_' is a substring)."""
    song_name = item_name[:-re.search(r'_', item_name[::-1]).span()[0]]
    return [song for song in item_names if song_name in song]


def select_spk_emb_items(item_name, item_names, spk_emb_num):
    """The ``spk_emb_num`` pieces whose embeddings follow the item's own: the song's pieces shuffled by a generator seeded from the
    item name (the reference's generator is unseeded), the last one repeated when there are too few."""
    pieces = song_pieces(item_name, item_names)
    random.Random(zlib.crc32(item_name.encode('utf-8'))).shuffle(pieces)
    sel = pieces[:spk_emb_num]
    return [sel[i] if i < len(sel) else sel[-1] for i in range(spk_emb_num)]


class PopBuTFyENSpkEMBinarizer(PopBuTFyENBinarizer):
    def extra_fields(self, res):
        names = [res['item_name']] + select_spk_emb_items(res['item_name'], self.item_names, hparams['spk_emb_num'])
        res['multi_spk_emb'] = np.stack([np.load(os.path.join(hparams['spk_emb_data_dir'], n + '.npy'), allow_pickle=True)
                                         for n in names], axis=0)
