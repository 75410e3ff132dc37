"""Write tests/golden/svb_dataset.npz from the reference's own paired-singing dataset (``MultiSpkEmbDataset``,
tasks/singing/svb_vae_task.py:20-45) and batch builder (``BaseTask.build_dataloader``, tasks/tts/tts.py:57-101) over a small
``write_svb_binary`` dataset.

    NEURALSVB_REFERENCE=<reference checkout> python oracle/gen_golden_svb_dataset.py

Shims on top of oracle/ref_harness: matplotlib and the g2p / text modules the task modules import are stubbed (nothing here
draws or tokenises); ``torch.cuda.device_count`` is pinned to the world size being recorded, because the reference sizes its
batches by the local device count; ``torch.distributed`` reports the recorded rank and world size.  The fixture stores the
dataset's items (the writer is deterministic, so the test rebuilds the same files), every collated batch tensor for the
first batches, and the index batches for world 1 and for both ranks of world 2."""
import os
import sys
import tempfile
import types

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from oracle import ref_harness as R  # noqa: E402

SEED, N_ITEMS = 1234, 12
HP = {'max_frames': 5000, 'frames_multiple': 4, 'min_frames': 0, 'sort_by_len': True, 'use_pitch_embed': True, 'pitch_norm': 'standard',
      'use_uv': True, 'normalize_pitch': False, 'use_spk_embed': False, 'use_spk_id': False, 'infer': False, 'num_test_samples': 0,
      'test_ids': [], 'max_input_tokens': 1550, 'pitch_type': 'frame', 'ds_workers': 0}
MAX_TOKENS, MAX_SENTENCES = 600, 4
KEYS = ('mels', 'prof_mels', 'pitch', 'prof_pitch', 'f0', 'uv', 'prof_f0', 'prof_uv', 'a2p_f0_alignment', 'multi_spk_emb')


def _stub_modules():
    class _Any(types.ModuleType):
        def __getattr__(self, name):
            if name.startswith('__'):
                raise AttributeError(name)
            return lambda *a, **k: None
    for name in ('matplotlib', 'matplotlib.pyplot', 'g2p_en', 'pypinyin', 'pypinyin.contrib', 'pypinyin.contrib.tone_convert',
                 'jieba', 'tensorboardX', 'torch.utils.tensorboard', 'tqdm'):
        sys.modules.setdefault(name, _Any(name))
    sys.modules['matplotlib'].use = lambda *a, **k: None


def main():
    from neuralsvb_b200.utils.synthetic import write_svb_binary
    R.install()
    _stub_modules()
    import utils.hparams as RH
    from tasks.singing.svb_vae_task import MultiSpkEmbDataset
    from tasks.tts.tts import TtsTask
    out = {}
    with tempfile.TemporaryDirectory() as d:
        write_svb_binary(d, N_ITEMS, SEED, n_valid=1, n_test=1)
        RH.hparams.clear()
        RH.hparams.update(HP, binary_data_dir=d)
        np.random.seed(SEED)
        ds = MultiSpkEmbDataset('train', shuffle=True)
        out['f0_mean_std'] = np.array([RH.hparams['f0_mean'], RH.hparams['f0_std']])
        for world in (1, 2):
            for rank in range(world):
                np.random.seed(SEED)
                task = TtsTask.__new__(TtsTask)
                task.trainer = types.SimpleNamespace(use_ddp=world > 1)
                torch.cuda.device_count = lambda: world
                torch.distributed.get_world_size = lambda: world
                torch.distributed.get_rank = lambda r=rank: r
                loader = TtsTask.build_dataloader(task, ds, True, MAX_TOKENS, MAX_SENTENCES)
                batches = list(loader.batch_sampler)
                out[f'batches_w{world}_r{rank}'] = np.array([len(b) for b in batches])
                out[f'indices_w{world}_r{rank}'] = np.concatenate([np.asarray(b, np.int64) for b in batches])
                if world == 1:
                    for i, batch in enumerate(loader):
                        if i == 4:
                            break
                        for k in KEYS:
                            out[f'b{i}_{k}'] = batch[k].numpy()
                        out[f'b{i}_item_name'] = np.array(batch['item_name'])
    path = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), 'tests', 'golden', 'svb_dataset.npz')
    np.savez_compressed(path, **out)
    print(f'wrote {path}: {len(out)} arrays')


if __name__ == '__main__':
    main()
