"""The singing binarizer's item bookkeeping (reference data_gen/singing/binarize.py over data_gen/tts/base_binarizer.py): scan
``{processed_data_dir}/data/*/*.wav`` and ``*.flac``, keep the items of ``hparams['datasets']``, split them by ``test_prefixes`` and write
``spk_map.json``.  ``process_data`` is the subclass's (binarize_para.py).

The reference reads PopBuTFy's mp3 files through librosa; here the input is WAV or FLAC at any rate and channel count (folded to mono and
resampled to ``audio_sample_rate`` on the GPU as ``librosa.core.load`` does), so mp3 files are decoded to WAV once beforehand (for
example ``ffmpeg -i x.mp3 x.wav``)."""
import glob
import json
import logging
import os
import random
import re
from copy import deepcopy

from neuralsvb_b200.utils.hparams import hparams


class BinarizationError(Exception):
    pass


def split_train_test_set(item_names):
    """(train, test) item names: an item is a test item when any of ``hparams['test_prefixes']`` occurs in its name."""
    item_names = deepcopy(item_names)
    test_item_names = [x for x in item_names if any([ts in x for ts in hparams['test_prefixes']])]
    train_item_names = [x for x in item_names if x not in set(test_item_names)]
    logging.info("train {}".format(len(train_item_names)))
    logging.info("test {}".format(len(test_item_names)))
    return train_item_names, test_item_names


class SingingBinarizer:
    def __init__(self, processed_data_dir=None):
        if processed_data_dir is None:
            processed_data_dir = hparams['processed_data_dir']
        self.processed_data_dirs = processed_data_dir.split(",")
        self.binarization_args = hparams.get('binarization_args', {}) or {}
        self.item2wavfn = {}
        self.item2spk = {}

    def load_meta_data(self):
        """item2wavfn / item2spk over every processed directory (item name = file basename, speaker = the name up to and including
        its first '#'), sorted names, then only the items of hparams['datasets'], then the train / test split."""
        for ds_id, processed_data_dir in enumerate(self.processed_data_dirs):
            wav_fns = sorted(glob.glob(f'{processed_data_dir}/data/*/*.wav'))
            flac_fns = sorted(glob.glob(f'{processed_data_dir}/data/*/*.flac'))
            if not wav_fns and not flac_fns and glob.glob(f'{processed_data_dir}/data/*/*.mp3'):
                raise ValueError(f'{processed_data_dir}/data holds mp3 files only: the binarizer reads WAV (any rate; it resamples '
                                 f'to {hparams["audio_sample_rate"]} Hz itself); decode them once, e.g. ffmpeg -i x.mp3 x.wav '
                                 '(FLAC is also accepted)')
            if flac_fns:
                seen = {os.path.splitext(os.path.basename(w))[0]: w for w in wav_fns}
                for fn in flac_fns:
                    name = os.path.splitext(os.path.basename(fn))[0]
                    if name in seen:
                        raise ValueError(f'item {name!r} is both {seen[name]} and {fn}: keep one of the two')
                    seen[name] = fn
                wav_fns = sorted(wav_fns + flac_fns)
            for wav_fn in wav_fns:
                item_name = os.path.splitext(os.path.basename(wav_fn))[0]
                if len(self.processed_data_dirs) > 1:
                    item_name = f'ds{ds_id}_{item_name}'
                self.item2wavfn[item_name] = wav_fn
                spk = os.path.splitext(os.path.basename(wav_fn))[0].split('#')[0] + '#'
                self.item2spk[item_name] = f'ds{ds_id}_{spk}' if len(self.processed_data_dirs) > 1 else spk
        self.item_names = sorted(self.item2wavfn)
        print('Total items: ', len(self.item_names))
        if self.binarization_args.get('shuffle', False):
            random.seed(1234)
            random.shuffle(self.item_names)
        self.item_names = [x for x in self.item_names if any(re.findall(rf'{ds}', x) for ds in hparams['datasets'])]
        self._train_item_names, self._test_item_names = split_train_test_set(self.item_names)

    @property
    def train_item_names(self):
        return self._train_item_names

    @property
    def valid_item_names(self):
        return self._test_item_names

    @property
    def test_item_names(self):
        return self._test_item_names

    def build_spk_map(self):
        spk_map = sorted({self.item2spk[x] for x in self.item_names})
        spk_map = {x: i for i, x in enumerate(spk_map)}
        print("| #Spk: ", len(spk_map))
        assert len(spk_map) == 0 or len(spk_map) <= hparams['num_spk'], len(spk_map)
        return spk_map

    def item_name2spk_id(self, item_name):
        return self.spk_map[self.item2spk[item_name]]

    def meta_data(self, prefix):
        item_names = {'valid': self.valid_item_names, 'test': self.test_item_names}.get(prefix, self.train_item_names)
        for item_name in item_names:
            yield item_name, self.item2wavfn[item_name], self.item_name2spk_id(item_name)

    def process(self):
        self.load_meta_data()
        os.makedirs(hparams['binary_data_dir'], exist_ok=True)
        self.spk_map = self.build_spk_map()
        print("| spk_map: ", self.spk_map)
        with open(f"{hparams['binary_data_dir']}/spk_map.json", 'w') as f:
            json.dump(self.spk_map, f)
        self.process_data('valid')
        self.process_data('test')
        self.process_data('train')

    def process_data(self, prefix):
        raise NotImplementedError
