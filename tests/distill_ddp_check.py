"""Distillation with a trainable teacher (DML) under distributed.B200DataParallel over NCCL.

  torchrun --nproc-per-node N tests/distill_ddp_check.py

KDModel(freeze_teacher=False) hands the wrapper both runtimes' gradient sinks.  After one training step of the
reference's DML loss (CE on teacher and student + DMLLoss), every rank holds the same gradients, teacher included, equal
to the mean of the per-rank gradients of unwrapped copies (bit for bit at N = 1, where the wrapper only changes where
they are written), and after an SGD step the teacher and student parameters are bit-identical on every rank.
"""
import os
import sys

import torch
import torch.distributed as dist

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def _same_on_every_rank(t, world):
    parts = [torch.empty_like(t) for _ in range(world)]
    dist.all_gather(parts, t.contiguous())
    return all(torch.equal(p, parts[0]) for p in parts)


def main():
    from simpleaicv_pytorch_training_examples_b200.distillation import losses
    from simpleaicv_pytorch_training_examples_b200.distillation.distillmodel import KDModel
    from simpleaicv_pytorch_training_examples_b200.distributed import B200DataParallel
    local_rank = int(os.environ['LOCAL_RANK'])
    torch.cuda.set_device(local_rank)
    dist.init_process_group('nccl', device_id=torch.device('cuda', local_rank))
    rank, world = dist.get_rank(), dist.get_world_size()
    try:
        def build():
            torch.manual_seed(0)
            return KDModel(teacher_type='resnet18', student_type='resnet18', freeze_teacher=False, num_classes=10).cuda().train()

        kd, solo = build(), build()
        ce, dml = losses.CELoss(), losses.DMLLoss(4.0)

        def loss_of(model, x, y):
            tea, stu = model(x)
            return ce(tea, y) + ce(stu, y) + dml(stu, tea)

        g = torch.Generator().manual_seed(1)
        xs = torch.randn(world, 4, 3, 64, 64, generator=g).cuda()
        ys = torch.randint(0, 10, (world, 4), generator=g).cuda()
        # the mean of the per-rank gradients, from an unwrapped copy on every rank
        want = {n: torch.zeros_like(p) for n, p in solo.named_parameters()}
        for r in range(world):
            solo.zero_grad(set_to_none=True)
            loss_of(solo, xs[r], ys[r]).backward()
            for n, p in solo.named_parameters():
                want[n] += p.grad / world
        ddp = B200DataParallel(kd)
        loss_of(ddp, xs[rank], ys[rank]).backward()
        torch.cuda.synchronize()
        for n, p in kd.named_parameters():
            assert p.grad is not None and p.grad.abs().sum() > 0, n
            assert _same_on_every_rank(p.grad, world), f'{n}: gradients differ across ranks'
            if world == 1:
                assert torch.equal(p.grad, want[n]), n
            else:
                torch.testing.assert_close(p.grad, want[n], rtol=1e-4, atol=1e-6, msg=n)
        opt = torch.optim.SGD(kd.parameters(), lr=0.1, momentum=0.9)
        opt.step()
        torch.cuda.synchronize()
        for n, p in kd.named_parameters():
            assert _same_on_every_rank(p.detach(), world), f'{n}: parameters differ across ranks after the step'
        print(f'rank {rank}: distill ddp ok', flush=True)
    finally:
        dist.destroy_process_group()


if __name__ == '__main__':
    main()
