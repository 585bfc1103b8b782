"""Bit-reproducibility of the H100 runtime (the reference runs with cudnn.deterministic=True,
tools/utils.py:95-107): two consecutive forward+backward passes on the same batch and weights give
bit-identical logits and parameter gradients (no float atomics anywhere in the kernels), and a second
forward run between a training forward and its backward does not disturb that backward (the tape of
saved activations / BN coefficients belongs to the forward that made it)."""
import pytest
import torch

pytestmark = pytest.mark.gpu


def _models():
    from simpleaicv_pytorch_training_examples_b200.classification import backbones
    return [('resnet18cifar', lambda: backbones.resnet18cifar(num_classes=100), (32, 3, 32, 32), 100),
            ('resnet50', lambda: backbones.resnet50(num_classes=1000), (16, 3, 96, 96), 1000),
            ('darknet19', lambda: backbones.darknet19(num_classes=10), (8, 3, 64, 64), 10),
            ('vit_base_patch16', lambda: backbones.vit_base_patch16(image_size=64, num_classes=10), (8, 3, 64, 64), 10)]


def _grads(model):
    return [p.grad.detach().clone() for p in model.parameters()]


@pytest.mark.parametrize('idx', range(4))
def test_two_consecutive_steps_are_bit_identical(idx):
    from simpleaicv_pytorch_training_examples_b200.classification import losses
    name, make, shape, nc = _models()[idx]
    torch.manual_seed(0)
    model = make().cuda().train()
    g = torch.Generator().manual_seed(5)
    x = torch.randn(*shape, generator=g).cuda()
    y = torch.randint(0, nc, (shape[0],), generator=g).cuda()
    crit = losses.CELoss()
    runs = []
    for _ in range(3):
        model.zero_grad(set_to_none=True)
        logits = model(x)
        crit(logits, y).backward()
        torch.cuda.synchronize()
        runs.append((logits.detach().clone(), _grads(model)))
    for lg, gr in runs[1:]:
        assert torch.equal(lg, runs[0][0]), f'{name}: logits differ between identical runs'
        bad = [i for i, (a, b) in enumerate(zip(gr, runs[0][1])) if not torch.equal(a, b)]
        assert not bad, f'{name}: {len(bad)} gradient tensors differ between identical runs (first: {bad[:5]})'


@pytest.mark.parametrize('idx', [0, 3])
def test_interleaved_forward_does_not_disturb_pending_backward(idx):
    from simpleaicv_pytorch_training_examples_b200.classification import losses
    name, make, shape, nc = _models()[idx]
    torch.manual_seed(0)
    model = make().cuda().train()
    g = torch.Generator().manual_seed(6)
    x = torch.randn(*shape, generator=g).cuda()
    x2 = torch.randn(*shape, generator=g).cuda()
    y = torch.randint(0, nc, (shape[0],), generator=g).cuda()
    crit = losses.CELoss()
    crit(model(x), y).backward()
    ref = _grads(model)
    model.zero_grad(set_to_none=True)
    loss = crit(model(x), y)
    with torch.no_grad():
        model(x2)                       # e.g. an EMA / teacher / logging pass on another batch
    model.eval()
    with torch.no_grad():
        model(x2)
    model.train()
    loss.backward()
    torch.cuda.synchronize()
    bad = [i for i, (a, b) in enumerate(zip(_grads(model), ref)) if not torch.equal(a, b)]
    assert not bad, f'{name}: a forward between forward and backward changed {len(bad)} gradients'
