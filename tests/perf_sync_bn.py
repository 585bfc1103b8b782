"""Cost of synchronized BatchNorm on the ResNet-50 224x224 batch-256 training step (per GPU), sync_bn off and on.

    python tests/perf_sync_bn.py [--steps 20] [--rounds 3]                        (one GPU: a one-rank NCCL group)
    torchrun --nproc-per-node N tests/perf_sync_bn.py [--steps 20] [--rounds 3]   (N GPUs, B200DataParallel)

The two settings are timed alternately, `rounds` times each, every timing a window of `steps` steps between CUDA events
after warm-up.  Printed with the card name and power limit: the per-step times, their spread, and the BatchNorm
collectives per step counted from the runtime's shapes (one exchange of [2C + 2] fp32 per BatchNorm forward, one of
[2C] per backward and one [4C] for a block's last and downsample BatchNorm together).  With one rank nothing is
exchanged, so the two timings must agree within their run-to-run spread.
"""
import argparse
import os
import subprocess
import sys
import types

import torch
import torch.distributed as dist

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def collectives(rt, world):
    """(forward count, forward bytes, backward count, backward bytes) of the BatchNorm exchanges of one step."""
    from simpleaicv_pytorch_training_examples_b200.engine.convnet import ResidualBlockRT
    units = rt.units()
    fwd = [(2 * u.kp + 2) * 4 for u in units]
    bwd = [2 * u.kp * 4 for u in units]
    for b in rt.blocks:
        if isinstance(b, ResidualBlockRT) and b.down is not None:     # paired with the block's last BatchNorm
            bwd.remove(2 * b.down.kp * 4)
            bwd.remove(2 * b.units[-1].kp * 4)
            bwd.append(4 * b.units[-1].kp * 4)
    if world <= 1:
        return 0, 0, 0, 0
    return len(fwd), sum(fwd), len(bwd), sum(bwd)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=20)
    ap.add_argument('--rounds', type=int, default=3)
    ap.add_argument('--batch', type=int, default=256)
    args = ap.parse_args()
    from simpleaicv_pytorch_training_examples_b200.classification import backbones, losses
    from simpleaicv_pytorch_training_examples_b200.tools.utils import build_training_mode
    if 'RANK' in os.environ:
        local = int(os.environ['LOCAL_RANK'])
        torch.cuda.set_device(local)
        dist.init_process_group('nccl', device_id=torch.device('cuda', local))
    else:
        os.environ.setdefault('MASTER_ADDR', '127.0.0.1')
        os.environ.setdefault('MASTER_PORT', '29517')
        torch.cuda.set_device(0)
        dist.init_process_group('nccl', rank=0, world_size=1, device_id=torch.device('cuda', 0))
    rank, world = dist.get_rank(), dist.get_world_size()
    crit = losses.CELoss()
    g = torch.Generator().manual_seed(rank)
    x = torch.randn(args.batch, 3, 224, 224, generator=g).cuda()
    y = torch.randint(0, 1000, (args.batch,), generator=g).cuda()
    runs = {}
    for sync in (False, True):
        torch.manual_seed(0)
        net = backbones.resnet50(num_classes=1000).cuda().train()
        model, _, _ = build_training_mode(types.SimpleNamespace(sync_bn=sync, use_ema_model=False), net)
        opt = torch.optim.SGD(net.parameters(), lr=1e-3, momentum=0.9)
        runs[sync] = (net, model, opt)

    def step(model, opt):
        crit(model(x), y).backward()
        opt.step()
        opt.zero_grad(set_to_none=False)

    for net, model, opt in runs.values():
        for _ in range(3):
            step(model, opt)
    torch.cuda.synchronize()
    times = {False: [], True: []}
    for _ in range(args.rounds):
        for sync, (net, model, opt) in runs.items():
            t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            t0.record()
            for _ in range(args.steps):
                step(model, opt)
            t1.record()
            torch.cuda.synchronize()
            times[sync].append(t0.elapsed_time(t1) / args.steps)
    if rank == 0:
        smi = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader', '-i',
                              str(torch.cuda.current_device())], capture_output=True, text=True).stdout.strip()
        nf, bf, nb, bb = collectives(runs[True][0]._runtime(), world)
        print(f'card: {smi}; world size {world}; ResNet-50 224x224, batch {args.batch} per GPU, eager step, '
              f'{args.rounds} alternating windows of {args.steps} steps')
        for sync in (False, True):
            t = times[sync]
            print(f'  sync_bn={sync!s:5}: {min(t):.2f} .. {max(t):.2f} ms per step (mean {sum(t) / len(t):.2f})')
        print(f'  BatchNorm collectives per step: {nf} forward ({bf / 1024:.1f} KiB), {nb} backward ({bb / 1024:.1f} KiB)'
              + ('' if world > 1 else '; with one rank none is issued (the counts with N >= 2 ranks: '
                 + '{} forward, {} backward)'.format(*[collectives(runs[True][0]._runtime(), 2)[i] for i in (0, 2)])))
    dist.destroy_process_group()


if __name__ == '__main__':
    main()
