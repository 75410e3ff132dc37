"""The paired-singing dataset of the SVB task (reference: ``MultiSpkEmbDataset``, tasks/singing/svb_vae_task.py:20-45, over
``FastSingingDataset`` / ``FastSpeechDataset`` / ``BaseTTSDataset``, neural_svb_task.py:10-62 and tasks/tts/dataset_utils.py).

On disk, as data_gen/singing/binarize_para.py writes it under ``binary_data_dir``: ``{prefix}.data`` / ``.idx`` (IndexedDataset),
``{prefix}_lengths.npy`` (max of the amateur and professional frame counts), ``train_f0s_mean_std.npy`` and ``phone_set.json``.
Each item holds ``mel`` / ``prof_mel`` [T, 80], ``f0`` / ``prof_f0`` (Hz), ``pitch`` / ``prof_pitch`` (coarse ids),
``a2p_f0_alignment`` [T_prof] (amateur frame of each professional frame), ``multi_spk_emb`` [5, 256] and ``item_name``.

A batch holds only what ``SVBVAEMleTask`` reads: ``mels`` / ``prof_mels`` [B, T, 80], ``pitch`` / ``prof_pitch`` (int64),
``f0`` / ``uv`` / ``prof_f0`` / ``prof_uv`` (float32, normalised and interpolated), ``a2p_f0_alignment`` [B, T_prof],
``multi_spk_emb`` [B, 5, 256], ``item_name`` and ``nsamples``; every field is zero-padded.  The text, ``mel2ph`` and energy fields
of the reference's FastSpeechDataset are not built."""
import os

import numpy as np
import torch

from neuralsvb_b200.utils import batch_by_size, collate_1d, collate_2d
from neuralsvb_b200.utils.indexed_datasets import IndexedDataset
from neuralsvb_b200.utils.pitch_utils import f0_to_coarse, norm_interp_f0

BATCH_KEYS = ('mels', 'prof_mels', 'pitch', 'prof_pitch', 'f0', 'uv', 'prof_f0', 'prof_uv', 'a2p_f0_alignment', 'multi_spk_emb')


def cropped_frames(n_frames, hp):
    """Frames a take of ``n_frames`` keeps: at most ``max_frames``, then a multiple of ``frames_multiple``."""
    return min(n_frames, hp['max_frames']) // hp['frames_multiple'] * hp['frames_multiple']


def take_conditioning(n_frames, f0, pitch, hp, f0_clip):
    """(T, pitch, f0, uv) of one take of ``n_frames`` mel frames, from its binarized f0 (Hz) and pitch ids: T = cropped_frames,
    ``normalize_pitch`` (``f0_clip``: 500 for the amateur take, 900 for the professional one), then norm_interp_f0 on the first T
    frames.  The dataset's items and the beautifier's takes both go through it."""
    T = cropped_frames(n_frames, hp)
    if hp.get('normalize_pitch', False):
        # f0 / uv below come from the moved contour, as in the reference
        f0 = normalized_take_f0(f0, hp, f0_clip)
        pitch = torch.LongTensor(f0_to_coarse(f0)[:T])
    else:
        pitch = torch.LongTensor(pitch)[:T]
    f0, uv = norm_interp_f0(f0[:T], hp)
    return T, pitch, f0, uv


def normalized_take_f0(f0, hp, f0_clip):
    """``normalize_pitch``'s contour (a copy): the take's voiced frames moved to the dataset's f0 statistics, clipped to
    [60, f0_clip]."""
    f0 = np.array(f0, copy=True)
    v = f0 > 0
    if v.any() and f0[v].std() > 0:
        f0[v] = ((f0[v] - f0[v].mean()) / f0[v].std() * hp['f0_std'] + hp['f0_mean']).clip(min=60, max=f0_clip)
    return f0


def clip_alignment(a2p_f0_alignment, prof_T, amateur_T):
    """The a2p alignment of the cropped takes: its first ``prof_T`` frames, never past the cropped amateur take."""
    return torch.LongTensor(a2p_f0_alignment)[:prof_T].clip(max=amateur_T - 1)


class MultiSpkEmbDataset(torch.utils.data.Dataset):
    def __init__(self, prefix, hparams, shuffle=False, data_dir=None):
        """Reads ``{prefix}_lengths.npy`` and the f0 statistics; sets ``hparams['f0_mean']`` / ``['f0_std']`` from
        ``train_f0s_mean_std.npy`` (None when the file is absent), as the reference dataset does."""
        super().__init__()
        self.hparams, self.prefix, self.shuffle = hparams, prefix, shuffle
        self.data_dir = hparams['binary_data_dir'] if data_dir is None else data_dir
        self.indexed_ds = None
        sizes = np.load(f'{self.data_dir}/{prefix}_lengths.npy')
        self.avail_idxs = list(range(len(sizes)))
        if (prefix == 'test' or hparams['infer']) and hparams['num_test_samples'] > 0:
            self.avail_idxs = list(hparams['test_ids']) + [x for x in range(hparams['num_test_samples']) if x < len(sizes)]
        if hparams['min_frames'] > 0:
            self.avail_idxs = [x for x in self.avail_idxs if sizes[x] >= hparams['min_frames']]
        self.sizes = [sizes[i] for i in self.avail_idxs]
        stats = f'{self.data_dir}/train_f0s_mean_std.npy'
        if os.path.exists(stats):
            hparams['f0_mean'], hparams['f0_std'] = (float(x) for x in np.load(stats))
        else:
            hparams['f0_mean'] = hparams['f0_std'] = None

    def __len__(self):
        return len(self.sizes)

    def num_tokens(self, index):
        return min(self.sizes[index], self.hparams['max_frames'])

    def ordered_indices(self):
        """A permutation from numpy's global generator (sorted by length, stable, with ``sort_by_len``) or 0..n-1."""
        if not self.shuffle:
            return np.arange(len(self))
        indices = np.random.permutation(len(self))
        if self.hparams['sort_by_len']:
            indices = indices[np.argsort(np.array(self.sizes)[indices], kind='mergesort')]
        return indices

    def _get_item(self, index):
        if self.indexed_ds is None:
            self.indexed_ds = IndexedDataset(f'{self.data_dir}/{self.prefix}')
        return self.indexed_ds[self.avail_idxs[index]]

    def _take(self, item, prefix, f0_clip):
        """(mel, pitch, f0, uv) of one take (``prefix`` '' = amateur, 'prof_' = professional): cropped to ``max_frames``, then to a
        multiple of ``frames_multiple``."""
        mel = item[f'{prefix}mel']
        T, pitch, f0, uv = take_conditioning(len(mel), item[f'{prefix}f0'], item[f'{prefix}pitch'], self.hparams, f0_clip)
        return torch.Tensor(mel)[:T], pitch, f0, uv

    def __getitem__(self, index):
        item = self._get_item(index)
        assert max(len(item['mel']), len(item['prof_mel'])) == self.sizes[index], (len(item['mel']), self.sizes[index])
        mel, pitch, f0, uv = self._take(item, '', 500)
        prof_mel, prof_pitch, prof_f0, prof_uv = self._take(item, 'prof_', 900)
        align = clip_alignment(item['a2p_f0_alignment'], prof_pitch.shape[0], pitch.shape[0])
        assert align.shape == prof_pitch.shape, ('a2p F0 alignment with unmatched shape: ', align.shape, prof_pitch.shape)
        return {'item_name': item['item_name'], 'mel': mel, 'pitch': pitch, 'f0': f0, 'uv': uv, 'prof_mel': prof_mel,
                'prof_pitch': prof_pitch, 'prof_f0': prof_f0, 'prof_uv': prof_uv, 'a2p_f0_alignment': align,
                'multi_spk_emb': torch.FloatTensor(item['multi_spk_emb'])}

    def collater(self, samples):
        c1 = lambda k, pad=0: collate_1d([s[k] for s in samples], pad)
        return {
            'item_name': [s['item_name'] for s in samples], 'nsamples': len(samples),
            'mels': collate_2d([s['mel'] for s in samples], 0.0), 'pitch': c1('pitch'), 'f0': c1('f0', 0.0), 'uv': c1('uv'),
            'prof_mels': collate_2d([s['prof_mel'] for s in samples], 0.0), 'prof_pitch': c1('prof_pitch'),
            'prof_f0': c1('prof_f0', 0.0), 'prof_uv': c1('prof_uv'), 'a2p_f0_alignment': c1('a2p_f0_alignment'),
            'multi_spk_emb': collate_2d([s['multi_spk_emb'] for s in samples]),
        }


def build_batches(dataset, shuffle, max_tokens=None, max_sentences=None, rank=0, world=1, endless=False, by_size=True):
    """Index batches as the reference's ``build_dataloader`` makes them (tasks/tts/tts.py:57-101), one device per rank:
    the token and sentence limits scale with the world size and batches are cut to multiples of it; numpy's global generator
    orders and shuffles them; ``endless`` repeats 1000 reshuffled epochs.  Rank r takes ``batch[r::world]`` of every batch whose
    length divides by the world size; the other batches are dropped on every rank."""
    if max_tokens is not None:
        max_tokens *= world
    if max_sentences is not None:
        max_sentences *= world
    indices = dataset.ordered_indices()
    if by_size:
        sampler = batch_by_size(indices, dataset.num_tokens, max_tokens=max_tokens, max_sentences=max_sentences,
                                required_batch_size_multiple=world)
    else:
        sampler = [indices[i:i + max_sentences] for i in range(0, len(indices), max_sentences)]

    def shuffled():
        b = list(sampler)
        np.random.shuffle(b)
        return b
    if shuffle:
        batches = shuffled()
        if endless:
            batches = [b for _ in range(1000) for b in shuffled()]
    else:
        batches = [b for _ in range(1000) for b in sampler] if endless else sampler
    if world > 1:
        batches = [x[rank::world] for x in batches if len(x) % world == 0]
    return batches


def build_dataloader(dataset, batches):
    """Batches collated in the calling process (no worker processes to outlive the run)."""
    return torch.utils.data.DataLoader(dataset, collate_fn=dataset.collater, batch_sampler=batches, num_workers=0)
