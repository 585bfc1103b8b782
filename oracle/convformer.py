"""Oracle: ConvFormer forward as functional fp32 torch-CPU code over a state dict.

Follows SimpleAICV/classification/backbones/convformer.py:16-44 (Downsampling: [pre BN] -> conv with bias -> [post BN];
stem 7x7/4 pad 2 with post BN, :190-197; stages 2-4 pre BN -> 3x3/2 pad 1, :198-206), :47-79 (SepConv: Linear C->2C ->
ReLU -> depthwise 7x7 pad 3 -> Linear 2C->C, no biases), :82-103 (Mlp: Linear C->4C -> ReLU -> Linear 4C->C, no biases),
:106-139 (DropPathBlock: per-sample fp32 scale), :142-166 (MetaFormerBlock: two pre-norm residual branches), :228-256
(average pool -> Linear head).  TEST INFRASTRUCTURE — see oracle/__init__.py.

Drop path: ``drop_scales`` maps 'stages.{i}.{j}' to the two fp32 [N] scales (token mixer, MLP) of that block, e.g. masks a
reference run drew (tests/golden/make_convformer_golden.py) or the H100 runtime's draws; blocks with drop_path_prob > 0 in
training need them.
"""
import hashlib
import math

import numpy as np
import torch
import torch.nn.functional as F

from .convnets import BN_EPS, BN_MOMENTUM, _keep, _RoundBoth, _RoundGrad, _RoundValue

ARCHS = {
    # name: (embedding planes, block nums)        convformer.py:267-296
    'convformer_s18': ([64, 128, 320, 512], [3, 3, 9, 3]),
    'convformer_s36': ([64, 128, 320, 512], [3, 12, 18, 3]),
    'convformer_m36': ([96, 192, 384, 576], [3, 12, 18, 3]),
    'convformer_b36': ([128, 256, 512, 768], [3, 12, 18, 3]),
}


def _bn_default(sd, name, c):
    sd[f'{name}.weight'], sd[f'{name}.bias'] = torch.ones(c), torch.zeros(c)
    sd[f'{name}.running_mean'], sd[f'{name}.running_var'] = torch.zeros(c), torch.ones(c)
    sd[f'{name}.num_batches_tracked'] = torch.tensor(0, dtype=torch.long)


def init_state(arch, num_classes, seed):
    """Seeded initial state identical to constructing the reference after torch.manual_seed(seed): the default Conv2d /
    Linear initialisers (kaiming_uniform(a=sqrt(5)) weight, uniform(+-1/sqrt(fan_in)) bias) are drawn in construction
    order, then convformer.py:231-238 applies trunc_normal_(std=.02) to every Conv2d / Linear weight (depthwise
    included) in modules() order and zeroes the biases.  Keys are in the reference's state_dict order."""
    planes, nums = ARCHS[arch]
    torch.manual_seed(seed)
    sd, weights = {}, []

    def layer(name, shape, fan_in, bias):
        w = torch.empty(*shape)
        torch.nn.init.kaiming_uniform_(w, a=math.sqrt(5))
        sd[f'{name}.weight'] = w
        if bias:
            bound = 1 / math.sqrt(fan_in)
            sd[f'{name}.bias'] = torch.empty(shape[0]).uniform_(-bound, bound)
        weights.append(name)

    cur = 3
    for i, c in enumerate(planes):
        d = f'downsample_layers.{i}'
        k = 7 if i == 0 else 3
        layer(f'{d}.conv', (c, cur, k, k), cur * k * k, True)
        _bn_default(sd, f'{d}.post_norm' if i == 0 else f'{d}.pre_norm', c if i == 0 else cur)
        cur = c
    for i, (c, n) in enumerate(zip(planes, nums)):
        for j in range(n):
            b = f'stages.{i}.{j}'
            _bn_default(sd, f'{b}.norm1', c)
            layer(f'{b}.token_mixer.pwconv1', (2 * c, c), c, False)
            layer(f'{b}.token_mixer.dwconv', (2 * c, 1, 7, 7), 49, False)
            layer(f'{b}.token_mixer.pwconv2', (c, 2 * c), 2 * c, False)
            _bn_default(sd, f'{b}.norm2', c)
            layer(f'{b}.mlp.fc1', (4 * c, c), c, False)
            layer(f'{b}.mlp.fc2', (c, 4 * c), 4 * c, False)
    layer('head', (num_classes, planes[3]), planes[3], True)
    for name in weights:
        torch.nn.init.trunc_normal_(sd[f'{name}.weight'], std=.02)
        if f'{name}.bias' in sd:
            sd[f'{name}.bias'].zero_()
    return sd


def tensor_hash(t):
    """sha256 of a tensor's bytes (fixture digests of the seeded initial weights)."""
    return hashlib.sha256(t.detach().contiguous().cpu().numpy().tobytes()).hexdigest()


def param_names(sd):
    return [k for k in sd if not (k.endswith('running_mean') or k.endswith('running_var') or k.endswith('num_batches_tracked'))]


def drop_path_rates(arch, drop_path_prob):
    """Per-block drop-path probabilities, 'stages.{i}.{j}' -> p (convformer.py:210-212)."""
    _, nums = ARCHS[arch]
    rates = [x for x in np.linspace(0, drop_path_prob, sum(nums))]
    out, k = {}, 0
    for i, n in enumerate(nums):
        for j in range(n):
            out[f'stages.{i}.{j}'] = rates[k]
            k += 1
    return out


def _bn(sd, name, x, training):
    y = F.batch_norm(x, sd[f'{name}.running_mean'], sd[f'{name}.running_var'], sd[f'{name}.weight'], sd[f'{name}.bias'],
                     training, BN_MOMENTUM, BN_EPS)
    if training:
        sd[f'{name}.num_batches_tracked'] += 1
    return y


def forward(sd, x, arch, training=True, emulate_bf16=False, trace=None, drop_path_prob=0., drop_scales=None):
    """Logits for the NCHW fp32 batch x.  emulate_bf16 inserts round-to-bf16 where the reference under autocast(bf16)
    stores bf16: the inputs and outputs of every conv / Linear / depthwise conv (GEMM weights as bf16 operand copies;
    depthwise weights stay fp32 as in the H100 kernels), BatchNorm outputs, and the residual stream while it is bf16 -
    from each downsampling output up to the first block that applies a drop path (an fp32 mask makes the sum fp32).
    trace receives stem_out, stage{i}_in, stage{i}_out (NCHW) with their gradients."""
    planes, nums = ARCHS[arch]
    rates = drop_path_rates(arch, drop_path_prob)
    emu = emulate_bf16
    rb = (lambda t: _RoundBoth.apply(t)) if emu else (lambda t: t)
    rw = (lambda t: _RoundValue.apply(t)) if emu else (lambda t: t)

    def linear(t, name):                        # NCHW -> Linear over channels (the reference's permutes) -> NCHW
        return F.linear(t.permute(0, 2, 3, 1), rw(sd[f'{name}.weight'])).permute(0, 3, 1, 2)

    if emu:
        x = x.bfloat16().float()
    for i, (c, n) in enumerate(zip(planes, nums)):
        d = f'downsample_layers.{i}'
        if i == 0:
            x = rb(F.conv2d(x, rw(sd[f'{d}.conv.weight']), sd[f'{d}.conv.bias'], 4, 2))
            x = _keep(trace, 'stem_out', rb(_bn(sd, f'{d}.post_norm', x, training)))
        else:
            a = rb(_bn(sd, f'{d}.pre_norm', x, training))
            x = rb(F.conv2d(a, rw(sd[f'{d}.conv.weight']), sd[f'{d}.conv.bias'], 2, 1))
        x = _keep(trace, f'stage{i}_in', x)
        stream_bf16 = True
        for j in range(n):
            b = f'stages.{i}.{j}'
            drop = training and rates[b] > 0.
            if drop:
                if drop_scales is None or b not in drop_scales:
                    raise ValueError(f'{b} applies a drop path: pass its scales in drop_scales')
                s1, s2 = (s.view(-1, 1, 1, 1) for s in drop_scales[b])
            h = rb(F.relu(linear(rb(_bn(sd, f'{b}.norm1', x, training)), f'{b}.token_mixer.pwconv1')))
            h = rb(F.conv2d(h, sd[f'{b}.token_mixer.dwconv.weight'], None, 1, 3, 1, 2 * c))
            h = rb(linear(h, f'{b}.token_mixer.pwconv2'))
            if drop:
                x, stream_bf16 = x + s1 * h, False
            else:
                x = rb(x + h) if stream_bf16 else x + h
            h = rb(F.relu(linear(rb(_bn(sd, f'{b}.norm2', x, training)), f'{b}.mlp.fc1')))
            h = rb(linear(h, f'{b}.mlp.fc2'))
            x = x + s2 * h if drop else (rb(x + h) if stream_bf16 else x + h)
        x = _keep(trace, f'stage{i}_out', x)
    z = rb(F.adaptive_avg_pool2d(x, (1, 1)).flatten(1))
    z = F.linear(z, rw(sd['head.weight']))
    if emu:
        z = _RoundGrad.apply(z)
    return _keep(trace, 'logits', z + sd['head.bias'])


def loss_and_grads(sd, x, labels, arch, emulate_bf16=False, trace=None, drop_path_prob=0., drop_scales=None):
    from .train_step import ce_loss
    names = param_names(sd)
    for n in names:
        sd[n].requires_grad_(True)
        sd[n].grad = None
    logits = forward(sd, x, arch, True, emulate_bf16, trace, drop_path_prob, drop_scales)
    loss = ce_loss(logits, labels)
    loss.backward()
    grads = {n: sd[n].grad.detach().clone() for n in names}
    for n in names:
        sd[n].requires_grad_(False)
        sd[n].grad = None
    return logits.detach(), loss.detach(), grads
