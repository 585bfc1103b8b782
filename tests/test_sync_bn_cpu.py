"""Host side of sync_bn: build_training_mode over a world-2 gloo group creates a process group of its own for the
BatchNorm exchanges and hands it to every runtime module before the model is wrapped for data parallelism."""
import os
import socket
import types

import torch
import torch.distributed as dist
import torch.multiprocessing as mp
import torch.nn as nn


def _stub_module():
    from simpleaicv_pytorch_training_examples_b200.engine.runtime import Runtime, RuntimeModule

    class _Stub(RuntimeModule):
        """A RuntimeModule with one BatchNorm whose runtime needs no GPU; it records the BatchNorm group it had when the
        data-parallel wrapper first asked for its gradient sink."""

        def __init__(self):
            super().__init__()
            self.conv = nn.Conv2d(3, 8, 1, bias=False)
            self.bn = nn.BatchNorm2d(8)
            self.group_at_wrap = 'not asked'

        def _build_runtime(self):
            return Runtime([])

        def grad_sink(self):
            if self.group_at_wrap == 'not asked':
                self.group_at_wrap = self._runtime().bn_group
            return super().grad_sink()

    return _Stub()


def _worker(rank, world, port, q):
    os.environ.update(MASTER_ADDR='127.0.0.1', MASTER_PORT=str(port))
    dist.init_process_group('gloo', rank=rank, world_size=world)
    try:
        from simpleaicv_pytorch_training_examples_b200.distributed import B200DataParallel
        from simpleaicv_pytorch_training_examples_b200.tools.utils import build_training_mode
        cfg = types.SimpleNamespace(sync_bn=True, use_ema_model=False)
        net = _stub_module()
        keys = list(net.state_dict())
        model, ema, scaler = build_training_mode(cfg, net)
        assert isinstance(model, B200DataParallel) and model.module is net and ema is None and scaler is None
        group = net._runtime().bn_group
        assert group is not None, 'no BatchNorm group attached'
        assert group is not dist.group.WORLD and group != dist.distributed_c10d._get_default_group(), \
            'the BatchNorm exchanges must not share the default group with the gradient all-reduce'
        assert dist.get_world_size(group) == world
        assert net.group_at_wrap is group, 'the group was not attached before the model was wrapped'
        assert list(net.state_dict()) == keys and isinstance(net.bn, nn.BatchNorm2d), 'the shell changed'
        # the group survives a lazily (re)built runtime, and lives outside state_dict
        net.__dict__.pop('_rt')
        assert net._runtime().bn_group is group
        # the group is usable for the exchange: a sum over both ranks
        t = torch.full((3,), float(rank + 1))
        dist.all_reduce(t, group=group)
        assert torch.equal(t, torch.full((3,), 3.0))
        # sync_bn off: nothing attached
        plain = _stub_module()
        build_training_mode(types.SimpleNamespace(sync_bn=False, use_ema_model=False), plain)
        assert plain._runtime().bn_group is None
        q.put((rank, 'ok'))
    except Exception as e:  # pragma: no cover
        q.put((rank, repr(e)))
    finally:
        dist.destroy_process_group()


def test_build_training_mode_sync_bn_gloo_world2():
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
