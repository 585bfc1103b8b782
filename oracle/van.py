"""Oracle: VAN forward as functional fp32 torch-CPU code over a state dict.

Follows SimpleAICV/classification/backbones/van.py:20-35 (DWConv 3x3 depthwise), :38-56 (Mlp: 1x1 -> depthwise
3x3 -> ReLU -> 1x1), :59-93 (LKA: depthwise 5x5, depthwise 7x7 dilation 3, 1x1, gate u * attn), :96-115
(Attention: 1x1, ReLU, LKA, 1x1, + shortcut), :154-186 (Block: BN -> Attention / Mlp, layer scale, residual),
:189-208 (OverlapPatchEmbed: strided conv with bias + BN), :289-310 (VAN.forward: 4 stages, BN, avgpool, head).
Dropout / DropPath are identity at the probabilities used for parity (0).  TEST INFRASTRUCTURE — see
oracle/__init__.py.
"""
import math

import torch
import torch.nn.functional as F

from .convnets import BN_EPS, BN_MOMENTUM, _keep, _RoundBoth, _RoundGrad, _RoundValue

ARCHS = {
    # name: (embedding planes, mlp ratios, block nums)
    'van_b0': ([32, 64, 160, 256], [8, 8, 4, 4], [3, 3, 5, 2]),
    'van_b1': ([64, 128, 320, 512], [8, 8, 4, 4], [2, 2, 4, 2]),
    'van_b2': ([64, 128, 320, 512], [8, 8, 4, 4], [3, 3, 12, 3]),
    'van_b3': ([64, 128, 320, 512], [8, 8, 4, 4], [3, 5, 27, 3]),
    'van_b4': ([64, 128, 320, 512], [8, 8, 4, 4], [3, 6, 40, 3]),
    'van_b5': ([96, 192, 480, 768], [8, 8, 4, 4], [3, 3, 24, 3]),
    'van_b6': ([96, 192, 384, 768], [8, 8, 4, 4], [6, 6, 90, 6]),
}


def _conv_default(sd, name, cout, cin_per_group, k):
    """nn.Conv2d.reset_parameters: kaiming_uniform(a=sqrt(5)) weight, uniform(+-1/sqrt(fan_in)) bias."""
    w = torch.empty(cout, cin_per_group, k, k)
    torch.nn.init.kaiming_uniform_(w, a=math.sqrt(5))
    bound = 1 / math.sqrt(cin_per_group * k * k)
    sd[f'{name}.weight'] = w
    sd[f'{name}.bias'] = torch.empty(cout).uniform_(-bound, bound)


def _bn_default(sd, name, c):
    sd[f'{name}.weight'], sd[f'{name}.bias'] = torch.ones(c), torch.zeros(c)
    sd[f'{name}.running_mean'], sd[f'{name}.running_var'] = torch.zeros(c), torch.ones(c)
    sd[f'{name}.num_batches_tracked'] = torch.tensor(0, dtype=torch.long)


def init_state(arch, num_classes, seed):
    """Seeded initial state identical to constructing the reference VAN after torch.manual_seed(seed): default
    Conv2d / Linear inits are drawn in construction order (they consume the generator), then van.py:265-279
    re-draws every conv with normal(0, sqrt(2 / fan_out)) (zero bias) and the head with trunc_normal(.02) in
    modules() order.  Keys are in the reference's state_dict order (a module's own parameters first)."""
    planes, ratios, nums = ARCHS[arch]
    torch.manual_seed(seed)
    sd, convs = {}, []

    def conv(name, cout, cin, k, groups=1):
        _conv_default(sd, name, cout, cin // groups, k)
        convs.append((name, k * k * cout // groups))

    cur = 3
    for i, (c, r, n) in enumerate(zip(planes, ratios, nums)):
        pe = f'patch_embed{i + 1}'
        conv(f'{pe}.proj', c, cur, 7 if i == 0 else 3)
        _bn_default(sd, f'{pe}.norm', c)
        cur = c
        for j in range(n):
            b = f'block{i + 1}.{j}'
            sd[f'{b}.layer_scale_1'] = 1e-5 * torch.ones(1, c, 1, 1)
            sd[f'{b}.layer_scale_2'] = 1e-5 * torch.ones(1, c, 1, 1)
            _bn_default(sd, f'{b}.norm1', c)
            conv(f'{b}.attn.proj_1', c, c, 1)
            conv(f'{b}.attn.spatial_gating_unit.conv0', c, c, 5, groups=c)
            conv(f'{b}.attn.spatial_gating_unit.conv_spatial', c, c, 7, groups=c)
            conv(f'{b}.attn.spatial_gating_unit.conv1', c, c, 1)
            conv(f'{b}.attn.proj_2', c, c, 1)
            _bn_default(sd, f'{b}.norm2', c)
            hid = int(c * r)
            conv(f'{b}.mlp.fc1', hid, c, 1)
            conv(f'{b}.mlp.dwconv.dwconv', hid, hid, 3, groups=hid)
            conv(f'{b}.mlp.fc2', c, hid, 1)
        _bn_default(sd, f'norm{i + 1}', c)
    hw = torch.empty(num_classes, planes[3])
    torch.nn.init.kaiming_uniform_(hw, a=math.sqrt(5))
    bound = 1 / math.sqrt(planes[3])
    sd['head.weight'], sd['head.bias'] = hw, torch.empty(num_classes).uniform_(-bound, bound)
    for name, fan_out in convs:
        sd[f'{name}.weight'].normal_(0, math.sqrt(2.0 / fan_out))
        sd[f'{name}.bias'].zero_()
    torch.nn.init.trunc_normal_(sd['head.weight'], std=.02)
    sd['head.bias'].zero_()
    return sd


def param_names(sd):
    return [k for k in sd if not (k.endswith('running_mean') or k.endswith('running_var') or k.endswith('num_batches_tracked'))]


def _bn(sd, name, x, training):
    y = F.batch_norm(x, sd[f'{name}.running_mean'], sd[f'{name}.running_var'], sd[f'{name}.weight'], sd[f'{name}.bias'],
                     training, BN_MOMENTUM, BN_EPS)
    if training:
        sd[f'{name}.num_batches_tracked'] += 1
    return y


def forward(sd, x, arch, training=True, emulate_bf16=False, trace=None):
    """Logits for the NCHW fp32 batch x.  emulate_bf16 inserts round-to-bf16 at the kernels' storage points
    (every GEMM / depthwise operand and output, BN outputs; the residual stream and all statistics stay fp32)."""
    planes, ratios, nums = ARCHS[arch]
    emu = emulate_bf16
    rb = (lambda t: _RoundBoth.apply(t)) if emu else (lambda t: t)
    rw = (lambda t: _RoundValue.apply(t)) if emu else (lambda t: t)
    if emu:
        x = x.bfloat16().float()
    for i, (c, r, n) in enumerate(zip(planes, ratios, nums)):
        pe = f'patch_embed{i + 1}'
        k, s = (7, 4) if i == 0 else (3, 2)
        y = rb(F.conv2d(x, rw(sd[f'{pe}.proj.weight']), sd[f'{pe}.proj.bias'], s, k // 2))
        x = rb(_bn(sd, f'{pe}.norm', y, training))
        for j in range(n):
            b = f'block{i + 1}.{j}'
            lka = f'{b}.attn.spatial_gating_unit'
            a = rb(_bn(sd, f'{b}.norm1', x, training))
            p1 = rb(F.relu(F.conv2d(a, rw(sd[f'{b}.attn.proj_1.weight']), sd[f'{b}.attn.proj_1.bias'])))
            c0 = rb(F.conv2d(p1, sd[f'{lka}.conv0.weight'], sd[f'{lka}.conv0.bias'], 1, 2, 1, c))
            cs = rb(F.conv2d(c0, sd[f'{lka}.conv_spatial.weight'], sd[f'{lka}.conv_spatial.bias'], 1, 9, 3, c))
            c1 = rb(F.conv2d(cs, rw(sd[f'{lka}.conv1.weight']), sd[f'{lka}.conv1.bias']))
            g = rb(p1 * c1)
            p2 = rb(F.conv2d(g, rw(sd[f'{b}.attn.proj_2.weight']), sd[f'{b}.attn.proj_2.bias']))
            x = x + sd[f'{b}.layer_scale_1'] * (p2 + a)
            m = rb(_bn(sd, f'{b}.norm2', x, training))
            hid = int(c * r)
            f1 = rb(F.conv2d(m, rw(sd[f'{b}.mlp.fc1.weight']), sd[f'{b}.mlp.fc1.bias']))
            d = rb(F.relu(F.conv2d(f1, sd[f'{b}.mlp.dwconv.dwconv.weight'], sd[f'{b}.mlp.dwconv.dwconv.bias'], 1, 1, 1, hid)))
            f2 = rb(F.conv2d(d, rw(sd[f'{b}.mlp.fc2.weight']), sd[f'{b}.mlp.fc2.bias']))
            x = x + sd[f'{b}.layer_scale_2'] * f2
        x = _keep(trace, f'stage{i}_out', rb(_bn(sd, f'norm{i + 1}', x, training)))
    z = rb(F.adaptive_avg_pool2d(x, (1, 1)).flatten(1))
    z = F.linear(z, rw(sd['head.weight']))
    if emu:
        z = _RoundGrad.apply(z)
    return _keep(trace, 'logits', z + sd['head.bias'])


def loss_and_grads(sd, x, labels, arch, emulate_bf16=False, trace=None):
    from .train_step import ce_loss
    names = param_names(sd)
    for n in names:
        sd[n].requires_grad_(True)
        sd[n].grad = None
    logits = forward(sd, x, arch, True, emulate_bf16, trace)
    loss = ce_loss(logits, labels)
    loss.backward()
    grads = {n: sd[n].grad.detach().clone() for n in names}
    for n in names:
        sd[n].requires_grad_(False)
        sd[n].grad = None
    return logits.detach(), loss.detach(), grads
