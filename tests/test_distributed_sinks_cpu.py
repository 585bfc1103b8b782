"""world_size-2 gloo test of distributed.B200DataParallel over a model whose parameters two runtimes write, each through
its own GradSink (distillation with a trainable teacher): every gradient of both is averaged, and the step's incomplete
buckets are reduced only once both backward passes have ended."""
import os
import socket

import torch
import torch.distributed as dist
import torch.multiprocessing as mp
import torch.nn as nn


class _TwoRuntimes(nn.Module):
    """teacher / student stand-ins, registered in that order like KDModel's, each depositing through its own sink."""

    def __init__(self):
        super().__init__()
        from simpleaicv_pytorch_training_examples_b200.engine.runtime import GradSink
        self.teacher, self.student = nn.Linear(300, 70), nn.Linear(70, 9)
        self.unused = nn.Parameter(torch.ones(5))
        self.__dict__['_sinks'] = {'teacher': GradSink(), 'student': GradSink()}

    def grad_sink(self):
        return [self._sinks['teacher'], self._sinks['student']]

    def fake_backward(self, name, rank):
        sink, m = self._sinks[name], getattr(self, name)
        for i, p in enumerate([m.bias, m.weight]):
            sink.add(p, torch.full_like(p, (rank + 1) * (i + 1) * (10 if name == 'teacher' else 1)))
        sink.on_backward_end()


def _worker(rank, world, port, q):
    os.environ.update(MASTER_ADDR='127.0.0.1', MASTER_PORT=str(port))
    dist.init_process_group('gloo', rank=rank, world_size=world)
    try:
        from simpleaicv_pytorch_training_examples_b200.distributed import B200DataParallel
        for cap in (25, 0.05):           # one bucket shared by both runtimes; several buckets
            torch.manual_seed(rank)
            net = _TwoRuntimes()
            B200DataParallel(net, bucket_cap_mb=cap)
            for _ in range(2):           # the second step starts from a clean end-of-backward count
                for p in net.parameters():
                    p.grad = None
                net.fake_backward('student', rank)
                # the teacher's backward has not run: its gradients were neither zero-filled nor reduced
                assert net.teacher.weight.grad is None and net.unused.grad is None, cap
                net.fake_backward('teacher', rank)
                # averages over ranks of (rank + 1) * k: 1.5 k
                for p, want in [(net.student.bias, 1.5), (net.student.weight, 3.0), (net.teacher.bias, 15.0),
                                (net.teacher.weight, 30.0)]:
                    assert torch.equal(p.grad, torch.full_like(p, want)), (cap, rank, p.shape)
                assert torch.equal(net.unused.grad, torch.zeros(5))
        q.put((rank, 'ok'))
    except Exception as e:  # pragma: no cover
        q.put((rank, repr(e)))
    finally:
        dist.destroy_process_group()


def test_two_runtimes_gradients_are_averaged_after_both_backward_passes():
    s = socket.socket()
    s.bind(('127.0.0.1', 0))
    port = s.getsockname()[1]
    s.close()
    ctx = mp.get_context('spawn')
    q = ctx.Queue()
    procs = [ctx.Process(target=_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    res = [q.get(timeout=120) for _ in procs]
    for p in procs:
        p.join(timeout=60)
    assert sorted(res) == [(0, 'ok'), (1, 'ok')], res


def test_distillation_models_hand_over_the_sinks_that_write_their_gradients():
    from simpleaicv_pytorch_training_examples_b200.distillation.distillmodel import KDModel
    from simpleaicv_pytorch_training_examples_b200.interactive_segmentation import distill_model
    frozen = KDModel(teacher_type='resnet18', student_type='resnet18', num_classes=10)
    assert frozen.grad_sink() is frozen.student.grad_sink()
    dml = KDModel(teacher_type='resnet18', student_type='resnet18', num_classes=10, freeze_teacher=False)
    assert dml.grad_sink() == [dml.teacher.grad_sink(), dml.student.grad_sink()]
    tea = dict(distill_model.SAM_H_TEACHER, image_size=64, block_nums=1, global_attn_indexes=[0])
    stu = dict(distill_model.SAM_B_STUDENT, image_size=64, block_nums=1, global_attn_indexes=[0])
    enc = distill_model.ImageEncoderDistillModel(teacher_params=tea, student_params=stu, freeze_teacher=False)
    assert enc.grad_sink() == [enc.teacher.grad_sink(), enc.student.grad_sink()]
