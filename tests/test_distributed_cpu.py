"""world_size-2 gloo test of the bucketed gradient all-reduce (host-side logic of
distributed.B200DataParallel) with a stand-in model that deposits gradients through GradSink
exactly like the CUDA runtime does."""
import os
import socket

import torch
import torch.distributed as dist
import torch.multiprocessing as mp
import torch.nn as nn


class _FakeNet(nn.Module):
    def __init__(self):
        super().__init__()
        self.a = nn.Linear(300, 70)
        self.b = nn.Linear(70, 9)
        self.unused = nn.Parameter(torch.ones(5))
        from simpleaicv_pytorch_training_examples_b200.engine.runtime import GradSink
        self.__dict__['_sink'] = GradSink()

    def grad_sink(self):
        return self._sink

    def fake_backward(self, rank, scale=1.0):
        sink = self._sink
        for i, p in enumerate(reversed([self.a.weight, self.a.bias, self.b.weight, self.b.bias])):
            sink.add(p, torch.full_like(p, (rank + 1) * (i + 1) * scale))
        if sink.on_backward_end is not None:
            sink.on_backward_end()


def _worker(rank, world, port, q):
    os.environ.update(MASTER_ADDR='127.0.0.1', MASTER_PORT=str(port))
    dist.init_process_group('gloo', rank=rank, world_size=world)
    try:
        from simpleaicv_pytorch_training_examples_b200.distributed import B200DataParallel
        torch.manual_seed(rank)  # different init per rank: the wrapper must broadcast rank 0's
        net = _FakeNet()
        ddp = B200DataParallel(net, bucket_cap_mb=0.05)  # several buckets
        w0 = net.a.weight.detach().clone()
        gathered = [torch.empty_like(w0) for _ in range(world)]
        dist.all_gather(gathered, w0)
        assert all(torch.equal(g, gathered[0]) for g in gathered), 'parameters not broadcast'
        assert len(ddp.buckets) > 1
        # plain step: average of (rank+1)*(i+1) over ranks = 1.5*(i+1)
        net.fake_backward(rank)
        exp = {id(net.b.bias): 1.5, id(net.b.weight): 3.0, id(net.a.bias): 4.5, id(net.a.weight): 6.0}
        for p in [net.a.weight, net.a.bias, net.b.weight, net.b.bias]:
            assert torch.allclose(p.grad, torch.full_like(p, exp[id(p)])), (rank, p.shape)
        assert net.unused.grad is not None and torch.all(net.unused.grad == 0)
        # accumulation: no_sync step then a synced step -> average of the summed gradients
        for p in net.parameters():
            p.grad = None
        with ddp.no_sync():
            net.fake_backward(rank)
        assert torch.allclose(net.b.bias.grad, torch.full_like(net.b.bias, float(rank + 1)))
        net.fake_backward(rank, scale=2.0)
        assert torch.allclose(net.b.bias.grad, torch.full_like(net.b.bias, 1.5 * 3.0))
        # reduce_now(): explicit reduction of gradients produced under no_sync()
        for p in net.parameters():
            p.grad = None
        with ddp.no_sync():
            net.fake_backward(rank)
        ddp.reduce_now()
        assert torch.allclose(net.b.bias.grad, torch.full_like(net.b.bias, 1.5))
        assert torch.allclose(net.a.weight.grad, torch.full_like(net.a.weight, 6.0))
        q.put((rank, 'ok'))
    except Exception as e:  # pragma: no cover
        q.put((rank, repr(e)))
    finally:
        dist.destroy_process_group()


def test_bucketed_allreduce_gloo_world2_gradients_written_through_sink_add():
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
