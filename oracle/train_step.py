"""Oracle: one training step of tools/scripts.py:141-270 (train_classification) on CPU fp32.

forward -> CELoss (SimpleAICV/classification/losses.py:14-28) -> backward -> SGD with momentum
where 1-D parameters get zero weight decay (tools/utils.py:292-600 with
global_weight_decay=False, the setting of every shipped ResNet config).  The NaN guards,
barrier and scalar all-reduces of the reference loop do not change the arithmetic of a healthy
step and are omitted.  TEST INFRASTRUCTURE — see oracle/__init__.py.
"""
import torch
import torch.nn.functional as F

from . import convnets


def ce_loss(logits, labels):
    """CELoss: mean cross entropy in fp32; labels int64 [B] or soft/one-hot [B, C]
    (OneHotLabelCELoss, losses.py:78-91)."""
    logits = logits.float()
    if labels.dtype in (torch.int64, torch.int32):
        return F.cross_entropy(logits, labels, reduction='mean')
    return torch.sum(-labels * F.log_softmax(logits, dim=-1), dim=-1).mean()


def loss_and_grads(sd, x, labels, arch, emulate_bf16=False, trace=None):
    """Returns (logits, loss, {param name: grad}); BN running stats in sd are updated.
    emulate_bf16: evaluate with the kernels' bf16 storage points (convnets.forward)."""
    names = convnets.param_names(sd)
    for n in names:
        sd[n].requires_grad_(True)
        sd[n].grad = None
    logits = convnets.forward(sd, x, arch, training=True, emulate_bf16=emulate_bf16, trace=trace)
    loss = ce_loss(logits, labels)
    loss.backward()
    grads = {n: sd[n].grad.detach().clone() for n in names}
    for n in names:
        sd[n].requires_grad_(False)
        sd[n].grad = None
    return logits.detach(), loss.detach(), grads


def sgd_step(sd, grads, momentum_buf, lr, momentum=0.9, weight_decay=1e-4):
    """torch.optim.SGD semantics: g += wd*p (wd = 0 for 1-D params); buf = m*buf + g (buf = g on
    the first step); p -= lr*buf."""
    for n, g in grads.items():
        p = sd[n]
        wd = 0.0 if p.ndim == 1 else weight_decay
        g = g + wd * p if wd != 0 else g
        if n not in momentum_buf:
            momentum_buf[n] = g.clone()
        else:
            momentum_buf[n].mul_(momentum).add_(g)
        p.sub_(lr * momentum_buf[n])


def multistep_lr(base_lr, epoch, milestones, gamma=0.1, warm_up_epochs=0):
    """tools/utils.py:239-246 (Scheduler, MultiStepLR with linear warm-up), epoch fractional."""
    if epoch < warm_up_epochs:
        return epoch / warm_up_epochs * base_lr
    return gamma ** len([m for m in milestones if m <= epoch]) * base_lr


def train_steps(arch, num_classes, seed, batches, lr=0.1, momentum=0.9, weight_decay=1e-4):
    """Runs len(batches) steps from the seeded init; returns (state dict, [loss per step])."""
    sd = convnets.init_state(arch, num_classes, seed)
    buf, losses = {}, []
    for x, y in batches:
        _, loss, grads = loss_and_grads(sd, x, y, arch)
        sgd_step(sd, grads, buf, lr, momentum, weight_decay)
        losses.append(float(loss))
    return sd, losses
