"""Models, seeded batches and one training step shared by the synchronized-BatchNorm tests (tests/test_sync_bn_gpu.py and
tests/sync_bn_check.py).

The loss is sum-reduced, sum over outputs of (output * R) with a fixed R, so a rank's parameter gradients are the
gradients of its rows' share of the loss, and their sum over ranks is exactly (in math) the full-batch gradient."""
import torch
import torch.nn as nn

BATCH = 8


def build(name):
    from simpleaicv_pytorch_training_examples_b200.classification import backbones
    from simpleaicv_pytorch_training_examples_b200.detection import models
    torch.manual_seed(0)
    if name == 'resnet18cifar':
        m = backbones.resnet18cifar(num_classes=10)
    elif name == 'resnet18':
        m = backbones.resnet18(num_classes=10)
    elif name == 'darknettiny':
        m = backbones.darknettiny(num_classes=10)
    elif name == 'van_b0':
        m = backbones.van_b0(num_classes=10)
    elif name == 'van_b0_ckpt':
        m = backbones.van_b0(num_classes=10, use_gradient_checkpoint=True)
    elif name == 'convformer_s18':
        m = backbones.convformer_s18(num_classes=10, drop_path_prob=0.)
    elif name == 'resnet18_detr':
        m = models.resnet18_detr()
        m.transformer.dropout_prob = 0.0       # the comparison needs the same rows to see the same computation
    else:
        raise KeyError(name)
    return m.cuda().train()


def image_shape(name):
    return {'resnet18cifar': (32, 32), 'resnet18': (64, 64), 'resnet18_detr': (128, 160)}.get(name, (64, 64))


def batch(name):
    """The seeded full batch (CPU) and the fixed loss weights R, one per output, batch on dim `bdim`."""
    g = torch.Generator().manual_seed(1234)
    h, w = image_shape(name)
    x = torch.randn(BATCH, 3, h, w, generator=g)
    if name == 'resnet18_detr':
        rs = [torch.randn(6, BATCH, 100, 81, generator=g), torch.randn(6, BATCH, 100, 4, generator=g)]
        return x, rs, 1
    return x, [torch.randn(BATCH, 10, generator=g)], 0


def forward(model, name, x):
    if name == 'resnet18_detr':
        masks = torch.zeros(x.shape[0], x.shape[2], x.shape[3], dtype=torch.bool, device=x.device)
        return list(model(x, masks))
    return [model(x)]


def bn_layers(model):
    return [m for m in model.modules() if isinstance(m, nn.BatchNorm2d)]


def step(model, name, lo, hi, net=None, roll=0, scale=1.0):
    """One forward + backward of rows lo:hi of the batch through `net` (default: the model itself, else its
    data-parallel wrapper); returns outputs, running statistics and gradients (CPU).  roll: the rows run rotated by
    that many images (the same math in another fp32 summation order); the outputs are returned in batch order.
    scale: the images are multiplied by it (1 + 2^-22: a perturbation of the size of an fp32 rounding)."""
    x, rs, bdim = batch(name)
    x = x * scale
    perm = (torch.arange(hi - lo) + roll) % (hi - lo)
    outs = forward(model if net is None else net, name, x[lo:hi][perm].cuda())
    rs = [r.narrow(bdim, lo, hi - lo).index_select(bdim, perm) for r in rs]
    loss = sum((o.float() * r.cuda()).sum() for o, r in zip(outs, rs))
    loss.backward()
    torch.cuda.synchronize()
    inv = torch.argsort(perm).cuda()
    outs = [o.index_select(bdim, inv) for o in outs]
    bns = bn_layers(model)
    return {'outs': [o.detach().float().cpu() for o in outs], 'bdim': bdim,
            'rm': [b.running_mean.detach().cpu().clone() for b in bns],
            'rv': [b.running_var.detach().cpu().clone() for b in bns],
            'nbt': [int(b.num_batches_tracked) for b in bns],
            'grads': {n: p.grad.detach().cpu().clone() for n, p in model.named_parameters() if p.grad is not None}}


def rel_cos(a, b):
    a, b = a.double().flatten(), b.double().flatten()
    return ((a - b).norm() / b.norm()).item(), (torch.dot(a, b) / (a.norm() * b.norm())).item()
