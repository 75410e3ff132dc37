"""Helpers the hot path's callers use (reference: utils/__init__.py)."""
import sys
import time

import torch


class Timer:
    """Cumulative wall-clock per name with a device sync on both sides; prints when enabled
    (reference: utils/__init__.py:243-264; wraps the generator call in spec2wav,
    vocoders/hifigan.py:59, gated by hparams['profile_infer'])."""
    timer_map = {}

    def __init__(self, name, enable=False):
        Timer.timer_map.setdefault(name, 0)
        self.name, self.enable = name, enable

    def __enter__(self):
        if self.enable:
            if torch.cuda.is_available():
                torch.cuda.synchronize()
            self.t = time.time()

    def __exit__(self, exc_type, exc_val, exc_tb):
        if self.enable:
            if torch.cuda.is_available():
                torch.cuda.synchronize()
            Timer.timer_map[self.name] += time.time() - self.t
            print(f'[Timer] {self.name}: {Timer.timer_map[self.name]}')


class AvgrageMeter(object):
    """(reference spelling kept: utils/__init__.py:102-115)"""

    def __init__(self):
        self.reset()

    def reset(self):
        self.avg, self.sum, self.cnt = 0, 0, 0

    def update(self, val, n=1):
        self.sum += val * n
        self.cnt += n
        self.avg = self.sum / self.cnt


def move_to_cuda(batch, gpu_id=0):
    """Recursively move tensors in lists / tuples / dicts (reference: utils/__init__.py:80-99)."""
    if callable(getattr(batch, 'cuda', None)):
        return batch.cuda(gpu_id, non_blocking=True)
    if callable(getattr(batch, 'to', None)):
        return batch.to(torch.device('cuda', gpu_id), non_blocking=True)
    if isinstance(batch, list):
        return [move_to_cuda(x, gpu_id) for x in batch]
    if isinstance(batch, tuple):
        return tuple(move_to_cuda(x, gpu_id) for x in batch)
    if isinstance(batch, dict):
        return {k: move_to_cuda(v, gpu_id) for k, v in batch.items()}
    return batch


def move_to_cpu(tensors):
    if isinstance(tensors, dict):
        return {k: move_to_cpu(v) for k, v in tensors.items()}
    if isinstance(tensors, (list, tuple)):
        return type(tensors)(move_to_cpu(v) for v in tensors)
    if isinstance(tensors, torch.Tensor):
        return tensors.cpu()
    return tensors


def collate_1d(values, pad_idx=0):
    """1-D tensors -> [B, max_len], right-padded with ``pad_idx`` (reference: utils/__init__.py:118-133)."""
    res = values[0].new(len(values), max(v.size(0) for v in values)).fill_(pad_idx)
    for i, v in enumerate(values):
        res[i, :len(v)] = v
    return res


def collate_2d(values, pad_idx=0):
    """[T_i, C] tensors -> [B, max T_i, C], right-padded with ``pad_idx`` (reference: utils/__init__.py:136-150)."""
    res = values[0].new(len(values), max(v.size(0) for v in values), values[0].shape[1]).fill_(pad_idx)
    for i, v in enumerate(values):
        res[i, :len(v)] = v
    return res


def batch_by_size(indices, num_tokens_fn, max_tokens=None, max_sentences=None, required_batch_size_multiple=1):
    """Consecutive runs of ``indices`` whose padded size (len x longest) stays within ``max_tokens`` and whose length stays within
    ``max_sentences``; a full batch is cut to a multiple of ``required_batch_size_multiple`` and the rest carried over
    (reference: utils/__init__.py:153-217)."""
    max_tokens = sys.maxsize if max_tokens is None else max_tokens
    max_sentences = sys.maxsize if max_sentences is None else max_sentences
    bsz_mult = required_batch_size_multiple
    sample_len, sample_lens, batch, batches = 0, [], [], []
    for idx in indices:
        num_tokens = num_tokens_fn(idx)
        sample_lens.append(num_tokens)
        sample_len = max(sample_len, num_tokens)
        assert sample_len <= max_tokens, f'sentence at index {idx} of size {sample_len} exceeds max_tokens limit of {max_tokens}!'
        num_tokens = (len(batch) + 1) * sample_len
        if len(batch) > 0 and (len(batch) == max_sentences or num_tokens > max_tokens):
            mod_len = max(bsz_mult * (len(batch) // bsz_mult), len(batch) % bsz_mult)
            batches.append(batch[:mod_len])
            batch = batch[mod_len:]
            sample_lens = sample_lens[mod_len:]
            sample_len = max(sample_lens) if len(sample_lens) > 0 else 0
        batch.append(idx)
    if len(batch) > 0:
        batches.append(batch)
    return batches


def tensors_to_scalars(tensors):
    """(reference: utils/__init__.py:24-43)"""
    if isinstance(tensors, torch.Tensor):
        return tensors.item()
    if isinstance(tensors, dict):
        return {k: tensors_to_scalars(v) for k, v in tensors.items()}
    if isinstance(tensors, list):
        return [tensors_to_scalars(v) for v in tensors]
    return tensors
