"""Time one GlobalFVAE training step of the SVB acoustic model (config 4, per GPU): two forwards through one module (the
a2a and p2p calls of MleSVBVAE) and one backward of the sum of their losses, at B = 16, T = 1024 mel frames and the
vae_global_mle_eng sizes (hidden 192, kernel 5, 8 encoder / 4 decoder layers, gin 256, latent 128, 80 mel bins).

Native path (trainable GlobalFVAE, bf16x3 and fp32) against the same graph in PyTorch eager on the same GPU, built from
the oracle functions (oracle/fs2_vae.py) with the poolings' BatchNorm in training mode, with cuDNN TF32 on and off.
Prints one JSON line per configuration plus the GPU name and power limit read in the same run.

    python tools/fvae_train_bench.py --steps 50 --warmup 5
"""
import argparse
import json
import os
import subprocess
import sys

import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

IO, H, LAT, K, LE, LD, GIN, S = 80, 192, 128, 5, 8, 4, 256, 4


def forward_flops(B, T):
    """Algorithmic multiply-add FLOPs (2 per MAC) of one GlobalFVAE forward, from the shapes."""
    conv = lambda t, cin, cout, k: 2.0 * B * t * cin * cout * k
    Te = T // S
    f = conv(Te, GIN, GIN, 2 * S) + conv(Te, IO, H, 2 * S)                                   # g_pre_net, encoder pre_net
    for L, t in ((LE, Te), (LD, T)):                                                          # the two WN stacks
        f += conv(t, GIN, 2 * H * L, 1) + L * conv(t, H, 2 * H, K) + (L - 1) * conv(t, H, 2 * H, 1) + conv(t, H, H, 1)
    f += conv(Te, H, 2 * LAT, 1) + sum(conv(Te >> i, 2 * LAT, 2 * LAT, 3) for i in (1, 2, 3))  # out_proj, poolings
    f += conv(Te, LAT, H, S) + conv(T, H, IO, 1)                                              # decoder pre_net, out_proj
    return f


def inputs(B, T, dev):
    g = torch.Generator().manual_seed(0)
    x = torch.randn(B, IO, T, generator=g)
    mask = torch.ones(B, 1, T)
    for b in range(B):
        mask[b, :, T - 8 * b:] = 0.0 if b else 1.0
    cond = torch.randn(B, GIN, T, generator=g)
    return [t.to(dev) for t in (x * mask, mask, cond)] + [torch.randn(B, IO, T, generator=g).to(dev)]


def eager_step(p, x, mask, cond, cot):
    from oracle import fs2_vae as OW
    w = OW.fold_weight_norm(p)
    e = {k[8:]: v for k, v in w.items() if k.startswith('encoder.')}
    dec = {k[8:]: v for k, v in w.items() if k.startswith('decoder.')}
    loss = 0
    for _ in range(2):
        g_sqz = F.conv1d(cond, w['g_pre_net.0.weight'], w['g_pre_net.0.bias'], stride=S, padding=S // 2)
        h = F.conv1d(x, e['pre_net.0.weight'], e['pre_net.0.bias'], stride=S, padding=S // 2)
        xm = mask[:, :, ::S][:, :, :h.shape[-1]]
        h = OW.wn_forward({k[3:]: v for k, v in e.items() if k.startswith('wn.')}, H, K, 1, LE, h * xm, xm, g_sqz) * xm
        h = F.conv1d(h, e['out_proj.weight'], e['out_proj.bias'])
        for i in (0, 3):
            h = torch.relu(F.conv1d(h, e[f'poolings.{i}.weight'], e[f'poolings.{i}.bias'], stride=2))
            j = i + 2
            h = F.batch_norm(h, p[f'encoder.poolings.{j}.running_mean'], p[f'encoder.poolings.{j}.running_var'], e[f'poolings.{j}.weight'],
                             e[f'poolings.{j}.bias'], training=True, momentum=0.1, eps=1e-5)
        h = F.conv1d(h, e['poolings.6.weight'], e['poolings.6.bias'], stride=2).mean(-1, keepdim=True)
        m_q, logs_q = torch.split(h, LAT, dim=1)
        z = m_q + torch.randn_like(m_q) * torch.exp(logs_q)
        xr = OW.fvae_decoder_forward(dec, H, K, LD, S, z, mask, cond, True)
        kl = (0.5 * (m_q ** 2 + torch.exp(2 * logs_q)) - logs_q - 0.5)
        loss = loss + (xr * cot).sum() + (kl * xm).sum() / xm.sum() / LAT
    loss.backward()


def native_step(m, x, mask, cond, cot):
    loss = 0
    for _ in range(2):
        xr, kl = m(x, mask, cond, infer=False)[:2]
        loss = loss + (xr * cot).sum() + kl
    loss.backward()


def timeit(fn, steps, warmup, zero):
    for _ in range(warmup):
        zero()
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        zero()
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / steps


def gpu_info():
    name = torch.cuda.get_device_name(0)
    try:
        r = subprocess.run(['nvidia-smi', '--query-gpu=power.limit', '--format=csv,noheader', '-i', '0'], capture_output=True,
                           text=True, timeout=30)
        power = r.stdout.strip() or None
    except (OSError, subprocess.SubprocessError):
        power = None
    return name, power


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=50)
    ap.add_argument('--warmup', type=int, default=5)
    ap.add_argument('--batch', type=int, default=16)
    ap.add_argument('--frames', type=int, default=1024)
    ap.add_argument('--profile', action='store_true', help='also print the CUDA time per kernel of 5 native bf16x3 steps')
    a = ap.parse_args()
    from neuralsvb_b200.modules.fastspeech.fs2_vae import GlobalFVAE
    from neuralsvb_b200.utils import synthetic as SY
    dev = torch.device('cuda', 0)
    torch.cuda.set_device(dev)
    B, T = a.batch, a.frames
    sd = SY.make_global_fvae_state_dict(IO, H, LAT, K, LE, LD, GIN, S, 1234)
    x, mask, cond, cot = inputs(B, T, dev)
    name, power = gpu_info()
    step_flops = 3 * 2 * forward_flops(B, T)            # two forwards, backward = data + weight gradients (2 x forward)
    results = []
    for precision in ('bf16x3', 'fp32'):
        m = GlobalFVAE(IO, H, LAT, K, LE, LD, GIN, [S], precision=precision, trainable=True)
        m.load_state_dict(sd, strict=True)
        m = m.to(dev).train()
        ms = timeit(lambda: native_step(m, x, mask, cond, cot), a.steps, a.warmup, lambda: m.zero_grad(set_to_none=True))
        results.append({'path': f'native {precision}', 'ms_per_step': round(ms, 3), 'tflops': round(step_flops / ms / 1e9, 2)})
        del m
    for tf32 in (True, False):
        torch.backends.cudnn.allow_tf32 = tf32
        torch.backends.cuda.matmul.allow_tf32 = tf32
        p = {k: (v.to(dev).float().requires_grad_(True) if v.is_floating_point() and 'running' not in k else v.to(dev).clone())
             for k, v in sd.items()}

        def zero():
            for v in p.values():
                v.grad = None
        ms = timeit(lambda: eager_step(p, x, mask, cond, cot), a.steps, a.warmup, zero)
        results.append({'path': f'eager cudnn tf32={tf32}', 'ms_per_step': round(ms, 3), 'tflops': round(step_flops / ms / 1e9, 2)})
    torch.backends.cudnn.allow_tf32 = True
    if a.profile:               # after every timing: an active profiler slows the steps that follow it
        from torch.profiler import ProfilerActivity, profile
        m = GlobalFVAE(IO, H, LAT, K, LE, LD, GIN, [S], precision='bf16x3', trainable=True)
        m.load_state_dict(sd, strict=True)
        m = m.to(dev).train()
        native_step(m, x, mask, cond, cot)
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(5):
                m.zero_grad(set_to_none=True)
                native_step(m, x, mask, cond, cot)
            torch.cuda.synchronize()
        print(prof.key_averages().table(sort_by='cuda_time_total', row_limit=25, max_name_column_width=70))
    for r in results:
        print(json.dumps(dict(r, B=B, T=T, steps=a.steps, gpu=name, power_limit=power)))
    print(json.dumps({'gpu': name, 'power_limit': power, 'step_gflop': round(step_flops / 1e9, 1),
                      'speedup_bf16x3_vs_eager_tf32': round(results[2]['ms_per_step'] / results[0]['ms_per_step'], 3)}))


if __name__ == '__main__':
    main()
