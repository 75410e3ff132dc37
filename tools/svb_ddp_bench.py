"""Data-parallel scaling of the SVB training step (BASELINE config 4): SVBVAEMleTask's full step through Trainer.run_training_batch
(the three optimizers, one FlatGradReducer each, gradient clipping, AdamW, the schedules) on 1, 2, 4 and 8 GPUs, as many as are
visible.  Per rank a synthetic B 16 x T 1024 batch (the tools/svb_train_bench.py shape) already on the device, so the loader is
not timed.

  phase2   G step with {a2a,p2p}_a + D step (mel_gan, disc_start_steps 0)
  phase3   the mapping step with a2p_a

Per GPU count it prints one JSON line: ms per step of each phase (rank 0, CUDA events), the all-reduce time each optimizer left
exposed on the compute stream (the wait inside FlatGradReducer.reduce, mean per step), the scaling efficiency against 1 GPU
(ms at 1 GPU / ms at N GPUs: per-rank work is fixed), and the GPU name and power limit read in the same run.

    python tools/svb_ddp_bench.py --steps 20 --warmup 5
"""
import argparse
import json
import os
import sys
import tempfile

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

CONFIG = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), 'egs', 'svb_vae_train_synthetic.yaml')


def _batch(B, T, rank):
    from neuralsvb_b200.utils import synthetic as S
    b = S.make_svb_batch(B, T, T, 1234 + rank)
    rs = np.random.RandomState(99 + rank)
    return {'mels': b['amateur_mel'], 'prof_mels': b['prof_mel'], 'pitch': b['amateur_pitch'], 'prof_pitch': b['prof_pitch'],
            'a2p_f0_alignment': b['a2p_alignment'], 'nsamples': B, 'item_name': [f'x{i}' for i in range(B)],
            'multi_spk_emb': torch.from_numpy(rs.randn(B, 5, 256).astype(np.float32) * 0.5)}


def _worker(rank, world, data_dir, args, port, out):
    import torch.distributed as dist
    from neuralsvb_b200.tasks.singing.svb_vae_task import SVBVAEMleTask
    from neuralsvb_b200.utils import move_to_cuda
    from neuralsvb_b200.utils.ddp_utils import FlatGradReducer, broadcast_module
    from neuralsvb_b200.utils.hparams import set_hparams
    from neuralsvb_b200.utils.trainer import Trainer
    set_hparams(CONFIG, '', f'binary_data_dir={data_dir},pretrain_asr_ckpt={data_dir}/asr,phase_2_steps=1000000', print_hparams=False)
    torch.cuda.set_device(rank)
    if world > 1:
        os.environ.update(MASTER_ADDR='127.0.0.1', MASTER_PORT=str(port))
        dist.init_process_group('nccl', rank=rank, world_size=world)
    np.random.seed(1234)
    tr = Trainer(work_dir=os.path.join(data_dir, f'work{rank}'), seed=1234)
    tr.proc_rank, tr.world_size, tr.root_gpu, tr.use_ddp = rank, world, rank, world > 1
    task = SVBVAEMleTask()
    task.trainer, tr.task = tr, task
    task.build_model()
    task.cuda(rank)
    if world > 1:
        broadcast_module(task)
    tr.optimizers = task.configure_optimizers()
    tr.reducers = [FlatGradReducer([p for g in o.param_groups for p in g['params']]) if world > 1 else None for o in tr.optimizers]
    pending = []
    for i, r in enumerate(tr.reducers):
        if r is None:
            continue

        def timed(r=r, i=i, f=r.reduce):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            f()
            e1.record()
            pending.append((i, e0, e1))
        r.reduce = timed
    batch = move_to_cuda(_batch(args.batch, args.frames, rank), rank)
    res = {}
    for phase, step0 in (('phase2', 1), ('phase3', 1000001)):
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
        for i in range(args.warmup + args.steps):
            if i == args.warmup:
                torch.cuda.synchronize()
                pending.clear()
                ev[0].record()
            tr.global_step = task.global_step = step0 + i
            tr.run_training_batch(i, batch)
        ev[1].record()
        torch.cuda.synchronize()
        exposed = [0.0] * 3
        for i, e0, e1 in pending:
            exposed[i] += e0.elapsed_time(e1) / args.steps
        res[phase] = {'ms': round(ev[0].elapsed_time(ev[1]) / args.steps, 3),
                      'exposed_allreduce_ms': {n: round(x, 3) for n, x in zip(('gen', 'disc', 'map'), exposed)} if world > 1 else None}
    if rank == 0:
        torch.save(res, out)
    if world > 1:
        dist.destroy_process_group()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=20)
    ap.add_argument('--warmup', type=int, default=5)
    ap.add_argument('--batch', type=int, default=16)
    ap.add_argument('--frames', type=int, default=1024)
    ap.add_argument('--max-gpus', type=int, default=8)
    a = ap.parse_args()
    import torch.multiprocessing as mp
    from neuralsvb_b200.utils.synthetic import write_svb_binary
    from tools.fvae_train_bench import gpu_info
    n = torch.cuda.device_count()
    if n == 0:
        raise RuntimeError('svb_ddp_bench needs CUDA devices')
    name, power = gpu_info()
    counts = [c for c in (1, 2, 4, 8) if c <= min(n, a.max_gpus)]
    base = None
    with tempfile.TemporaryDirectory() as d:
        write_svb_binary(d, 2, 1234, n_valid=1, n_test=1)
        for world in counts:
            out = os.path.join(d, f'res{world}.pt')
            mp.start_processes(_worker, args=(world, d, a, 29500 + os.getpid() % 500, out), nprocs=world, join=True, start_method='spawn')
            res = torch.load(out)
            if world == 1:
                base = res
            eff = {p: round(base[p]['ms'] / res[p]['ms'], 3) for p in res}
            print(json.dumps({'gpus': world, 'gpus_visible': n, 'B_per_rank': a.batch, 'T': a.frames, 'steps': a.steps,
                              **{f'{p}_ms': res[p]['ms'] for p in res}, **{f'{p}_exposed_allreduce_ms': res[p]['exposed_allreduce_ms'] for p in res},
                              'scaling_efficiency': eff, 'gpu': name, 'power_limit': power}), flush=True)


if __name__ == '__main__':
    main()
