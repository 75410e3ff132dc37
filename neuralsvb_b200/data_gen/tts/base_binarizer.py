"""GPU-batched binarizer for the vocoder path (SURVEY 8(f) N2).

The reference packs a dataset by calling ``get_vocoder_cls(hparams).wav2spec(wav_fn)`` once per file from a pool of
single-threaded CPU workers (data_gen/tts/base_binarizer.py:128-178, data_gen/singing/binarize_para.py:116-217,
``OMP_NUM_THREADS=1`` at data_gen/tts/bin/binarize.py:3).  Here the files of a split are grouped into ragged batches
and every batch is ONE device call (``HifiGAN.wav2spec_batch``: ``audio.load_takes`` -> ``svb_wav2spec_batch``); the items written are
the reference's: ``item_name, wav_fn, spk_id, mel [T, 80] (log10), wav float16 [T*hop], sec, len`` (+ ``f0`` when a
pitch function is supplied: ``data_gen.tts.data_gen_utils.get_pitch`` is this package's GPU tracker, and the reference's
parselmouth extractor can be passed instead),
in the reference's IndexedDataset format plus ``{prefix}_lengths.npy``.  Text / alignment / speaker-embedding fields
belong to the acoustic model's data preparation and are not produced."""
import os

import numpy as np

from neuralsvb_b200.utils import audio
from neuralsvb_b200.utils.hparams import hparams
from neuralsvb_b200.utils.indexed_datasets import IndexedDatasetBuilder
from neuralsvb_b200.vocoders.base_vocoder import get_vocoder_cls


class VocoderBinarizer:
    def __init__(self, items, binary_data_dir=None, pitch_fn=None, batch_seconds=600.0):
        """items: {prefix: [(item_name, wav_fn_or_array, spk_id), ...]} for prefix in train / valid / test.
        pitch_fn(wav, mel) -> f0 [T] in Hz (0 = unvoiced) or None.  batch_seconds: audio per device call."""
        self.items, self.pitch_fn, self.batch_seconds = items, pitch_fn, float(batch_seconds)
        self.binary_data_dir = binary_data_dir or hparams['binary_data_dir']

    def process(self):
        os.makedirs(self.binary_data_dir, exist_ok=True)
        return {prefix: self.process_data(prefix) for prefix in ('valid', 'test', 'train') if prefix in self.items}

    def _batches(self, metas, wavs_of=lambda m: (m[1],)):
        """Group consecutive items up to ``batch_seconds`` of audio (arrays are at audio_sample_rate; a file's duration is read
        from its WAV header, at the file's own rate).  ``wavs_of(meta)``: the waveforms an item holds (its one take here; both takes
        of a pair in the paired binarizer).  Every clip's output is the same in any batch, so grouping changes no item."""
        sr = hparams['audio_sample_rate']
        cur, sec = [], 0.0
        for m in metas:
            s = sum(audio.wav_seconds(w) if isinstance(w, str) else len(w) / sr for w in wavs_of(m))
            if cur and sec + s > self.batch_seconds:
                yield cur
                cur, sec = [], 0.0
            cur.append(m)
            sec += s
        if cur:
            yield cur

    def process_data(self, prefix):
        voc = get_vocoder_cls(hparams)
        builder = IndexedDatasetBuilder(f'{self.binary_data_dir}/{prefix}')
        lengths, total_sec, f0s = [], 0.0, []
        for batch in self._batches(self.items[prefix]):
            specs = voc.wav2spec_batch([m[1] for m in batch])               # ONE device call per batch
            for (item_name, wav_fn, spk_id), (wav, mel) in zip(batch, specs):
                item = self.make_item(item_name, wav_fn, spk_id, wav, mel)
                builder.add_item(item)
                lengths.append(item['len'])
                total_sec += item['sec']
                if item.get('f0') is not None:
                    f0s.append(item['f0'])
        builder.finalize()
        np.save(f'{self.binary_data_dir}/{prefix}_lengths.npy', lengths)
        if f0s:
            f = np.concatenate(f0s, 0)
            f = f[f != 0]
            if len(f):
                np.save(f'{self.binary_data_dir}/{prefix}_f0s_mean_std.npy', [np.mean(f).item(), np.std(f).item()])
        print(f'| {prefix} total duration: {total_sec:.3f}s')
        return {'items': len(lengths), 'sec': total_sec}

    def make_item(self, item_name, wav_fn, spk_id, wav, mel):
        """data_gen/tts/base_binarizer.py:168-178: wav stored as float16, len = mel frames, sec = samples / sr."""
        res = {'item_name': item_name, 'wav_fn': wav_fn if isinstance(wav_fn, str) else None, 'spk_id': spk_id}
        f0 = None if self.pitch_fn is None else np.asarray(self.pitch_fn(wav, mel), np.float32)
        wav16 = wav.astype(np.float16)
        res.update({'mel': np.ascontiguousarray(mel), 'wav': wav16, 'sec': len(wav16) / hparams['audio_sample_rate'],
                    'len': mel.shape[0]})
        if f0 is not None:
            assert len(f0) == len(mel), (len(f0), len(mel))
            res['f0'] = f0
        return res
