"""Synchronized BatchNorm over NCCL.

  python tests/sync_bn_check.py --world-one
      one rank: build_training_mode with sync_bn=True gives a training step (eager, then under GraphedTrainStep) that
      is bit-identical to sync_bn=False (a group of one rank exchanges nothing).
  torchrun --nproc-per-node 2 --master-addr 127.0.0.1 --master-port 29513 tests/sync_bn_check.py
      >= 2 GPUs: ResNet-18 under B200DataParallel with sync_bn=True.  The wrapper's averaged gradients times the world
      size equal the gradients of one process running the whole batch (recomputed on every rank), the outputs are the
      rank's rows of that process's outputs and the running statistics its running statistics (bf16 parity: rel L2
      <= 2e-2, cosine >= 0.999); distributed.overlap_self_check passes bit for bit; the step captures and replays under
      GraphedTrainStep with identical parameters on every rank.
"""
import os
import socket
import sys
import types

import torch
import torch.distributed as dist

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import sync_bn_models as sm  # noqa: E402


def _bits(t):
    return t.detach().float().contiguous().view(torch.int32)


def _state(model):
    return [_bits(p) for p in model.parameters()] + [_bits(b) for b in model.buffers() if b.is_floating_point()]


def world_one():
    from simpleaicv_pytorch_training_examples_b200.classification import losses
    from simpleaicv_pytorch_training_examples_b200.graph import GraphedTrainStep
    from simpleaicv_pytorch_training_examples_b200.tools.utils import build_training_mode
    s = socket.socket()
    s.bind(('127.0.0.1', 0))
    os.environ.update(MASTER_ADDR='127.0.0.1', MASTER_PORT=str(s.getsockname()[1]))
    s.close()
    torch.cuda.set_device(0)
    dist.init_process_group('nccl', rank=0, world_size=1, device_id=torch.device('cuda', 0))
    try:
        crit = losses.CELoss()
        g = torch.Generator().manual_seed(5)
        x, y = torch.randn(16, 3, 64, 64, generator=g).cuda(), torch.randint(0, 10, (16,), generator=g).cuda()
        for name in ('resnet18cifar', 'van_b0'):
            runs = []
            for sync in (False, True):
                model = sm.build(name)
                model, _, _ = build_training_mode(types.SimpleNamespace(sync_bn=sync, use_ema_model=False), model)
                assert (model._runtime().bn_group is not None) == sync
                opt = torch.optim.SGD(model.parameters(), lr=0.1, momentum=0.9)
                loss = crit(model(x), y)
                loss.backward()
                opt.step()
                opt.zero_grad(set_to_none=False)
                eager = [_bits(loss)] + _state(model)
                step = GraphedTrainStep(model, crit, opt, x, y, warmup=2)
                graphed = [_bits(step(x, y)) for _ in range(2)]
                torch.cuda.synchronize()
                runs.append((eager, graphed + _state(model)))
            (ea, ga), (eb, gb) = runs
            assert all(torch.equal(a, b) for a, b in zip(ea, eb)), f'{name}: eager step differs with sync_bn on one rank'
            assert all(torch.equal(a, b) for a, b in zip(ga, gb)), f'{name}: graphed steps differ with sync_bn on one rank'
            print(f'{name}: world one ok (eager and graphed bit-identical)', flush=True)
    finally:
        dist.destroy_process_group()


def two_ranks():
    from simpleaicv_pytorch_training_examples_b200.distributed import overlap_self_check
    from simpleaicv_pytorch_training_examples_b200.graph import GraphedTrainStep
    from simpleaicv_pytorch_training_examples_b200.tools.utils import build_training_mode
    rank, world, local = int(os.environ['RANK']), int(os.environ['WORLD_SIZE']), int(os.environ['LOCAL_RANK'])
    torch.cuda.set_device(local)
    dist.init_process_group('nccl', device_id=torch.device('cuda', local))
    name = 'resnet18'
    per = sm.BATCH // world
    lo, hi = rank * per, (rank + 1) * per
    ref = sm.step(sm.build(name), name, 0, per * world)          # one process, the whole batch, no exchange
    model = sm.build(name)
    ddp, _, _ = build_training_mode(types.SimpleNamespace(sync_bn=True, use_ema_model=False), model)
    assert model._runtime().bn_group is not None
    got = sm.step(model, name, lo, hi, net=ddp)
    rel, cos = sm.rel_cos(got['outs'][0], ref['outs'][0][lo:hi])
    assert rel <= 2e-2 and cos >= 0.999, f'rank {rank}: outputs rel L2 {rel:.3g} cosine {cos:.6f}'
    rel, cos = sm.rel_cos(torch.cat(got['rv']), torch.cat(ref['rv']))
    assert rel <= 2e-2 and cos >= 0.999, f'rank {rank}: running_var rel L2 {rel:.3g}'
    rel, cos = sm.rel_cos(torch.cat(got['rm']), torch.cat(ref['rm']))
    assert rel <= 2e-2 and cos >= 0.999, f'rank {rank}: running_mean rel L2 {rel:.3g}'
    keys = list(ref['grads'])
    rel, cos = sm.rel_cos(torch.cat([got['grads'][k].flatten() * world for k in keys]),
                          torch.cat([ref['grads'][k].flatten() for k in keys]))
    assert rel <= 2e-2 and cos >= 0.999, f'rank {rank}: averaged gradients x world vs full batch: rel L2 {rel:.3g}'
    x, rs, _ = sm.batch(name)
    xl, rl = x[lo:hi].cuda(), rs[0][lo:hi].cuda()
    ndiff = overlap_self_check(ddp, lambda: (ddp(xl) * rl).sum().backward())
    assert ndiff == 0, f'rank {rank}: overlapped all-reduce with sync_bn differs in {ndiff} elements'
    opt = torch.optim.SGD(model.parameters(), lr=0.01, momentum=0.9)
    crit = lambda out, r: (out * r).sum()   # noqa: E731
    step = GraphedTrainStep(ddp, crit, opt, xl, rl, warmup=2)
    for _ in range(3):
        loss = step(xl, rl)
    torch.cuda.synchronize()
    assert torch.isfinite(loss).all()
    flat = torch.cat([p.detach().flatten() for p in model.parameters()] + [b.flatten() for b in model.buffers()
                                                                             if b.is_floating_point()])
    flat0 = flat.clone()
    dist.broadcast(flat0, src=0)
    assert torch.equal(flat, flat0), f'rank {rank}: replicas diverged under the graphed step'
    print(f'rank {rank}: sync bn ok (outputs, running stats, gradients vs one process; overlap check; graphed)', flush=True)
    dist.destroy_process_group()


if __name__ == '__main__':
    world_one() if '--world-one' in sys.argv else two_ranks()
