"""Oracle: ResNet / ResNetCifar forward as functional fp32 torch-CPU code over a state dict.

Follows SimpleAICV/classification/backbones/resnet.py:19-48 (conv -> BN -> ReLU),
:51-97 (BasicBlock), :100-155 (Bottleneck), :226-245 (ResNet.forward: 7x7/2 stem, 3x3/2 max
pool, 4 stages, global average pool, fc) and resnetforcifar.py:38-45,98-108 (3x3/1 stem, no
max pool).  TEST INFRASTRUCTURE — see oracle/__init__.py.
"""
import math

import torch
import torch.nn.functional as F

ARCHS = {
    # name: (block, layer_nums, cifar_stem)
    'resnet18': ('basic', [2, 2, 2, 2], False),
    'resnet34': ('basic', [3, 4, 6, 3], False),
    'resnet50': ('bottleneck', [3, 4, 6, 3], False),
    'resnet101': ('bottleneck', [3, 4, 23, 3], False),
    'resnet152': ('bottleneck', [3, 8, 36, 3], False),
    'resnet18cifar': ('basic', [2, 2, 2, 2], True),
    'resnet34cifar': ('basic', [3, 4, 6, 3], True),
    'resnet50cifar': ('bottleneck', [3, 4, 6, 3], True),
    'resnet101cifar': ('bottleneck', [3, 4, 23, 3], True),
    'resnet152cifar': ('bottleneck', [3, 8, 36, 3], True),
}
BN_EPS, BN_MOMENTUM = 1e-5, 0.1


def _cba_specs(arch, inplanes=64):
    """Yields (prefix, cin, cout, k, stride) for every ConvBnActBlock in construction order."""
    block, nums, cifar = ARCHS[arch]
    exp = 1 if block == 'basic' else 4
    specs = [('conv1', 3, inplanes, 3 if cifar else 7, 1 if cifar else 2)]
    cin = inplanes
    for li, (planes, lstride) in enumerate(zip([inplanes, inplanes * 2, inplanes * 4, inplanes * 8], (1, 2, 2, 2))):
        for bi in range(nums[li]):
            stride = lstride if bi == 0 else 1
            p = f'layer{li + 1}.{bi}'
            if block == 'basic':
                specs += [(f'{p}.conv1', cin, planes, 3, stride), (f'{p}.conv2', planes, planes, 3, 1)]
            else:
                specs += [(f'{p}.conv1', cin, planes, 1, 1), (f'{p}.conv2', planes, planes, 3, stride),
                          (f'{p}.conv3', planes, planes * 4, 1, 1)]
            if stride != 1 or cin != planes * exp:
                specs.append((f'{p}.downsample_conv', cin, planes * exp, 1, stride))
            cin = planes * exp
    return specs, cin


def init_state(arch, num_classes, seed):
    """Seeded initial state dict identical to constructing the reference model after
    torch.manual_seed(seed): nn.Conv2d / nn.Linear default inits are drawn in construction order
    (they consume the generator), then resnet.py:206-213 re-draws every conv with
    kaiming_normal_(fan_out) and sets BN to (1, 0)."""
    torch.manual_seed(seed)
    specs, feat = _cba_specs(arch)
    sd = {}
    for prefix, cin, cout, k, _ in specs:
        w = torch.empty(cout, cin, k, k)
        torch.nn.init.kaiming_uniform_(w, a=math.sqrt(5))  # nn.Conv2d.reset_parameters
        sd[f'{prefix}.layer.0.weight'] = w
        sd[f'{prefix}.layer.1.weight'] = torch.ones(cout)
        sd[f'{prefix}.layer.1.bias'] = torch.zeros(cout)
        sd[f'{prefix}.layer.1.running_mean'] = torch.zeros(cout)
        sd[f'{prefix}.layer.1.running_var'] = torch.ones(cout)
        sd[f'{prefix}.layer.1.num_batches_tracked'] = torch.tensor(0, dtype=torch.long)
    fw = torch.empty(num_classes, feat)
    torch.nn.init.kaiming_uniform_(fw, a=math.sqrt(5))  # nn.Linear.reset_parameters
    bound = 1 / math.sqrt(feat)
    fb = torch.empty(num_classes).uniform_(-bound, bound)
    sd['fc.weight'], sd['fc.bias'] = fw, fb
    for prefix, *_ in specs:
        torch.nn.init.kaiming_normal_(sd[f'{prefix}.layer.0.weight'], mode='fan_out', nonlinearity='relu')
    return sd


def param_names(sd):
    return [k for k in sd if not (k.endswith('running_mean') or k.endswith('running_var') or k.endswith('num_batches_tracked'))]


# ---- optional emulation of the kernels' storage precision -----------------------------------
# The kernels keep activations and activation gradients in bf16 and feed bf16 operands to the
# tensor cores (fp32 accumulation; BN statistics, parameters and parameter gradients in fp32).
# With emulate_bf16=True the SAME reference algorithm is evaluated with a round-to-bf16 at exactly
# those storage points (forward and backward), so the GPU result can be compared tightly; without
# it this is the plain fp32 reference.  (Random-init ResNets amplify bf16 rounding so much that the
# reference's own autocast(bf16) run differs from its fp32 run by ~0.3 relative L2 in early-layer
# gradients — see DESIGN.md "Parity".)
class _RoundBoth(torch.autograd.Function):
    """bf16 storage of an activation: value rounded forward, its gradient rounded backward."""

    @staticmethod
    def forward(ctx, x):
        return x.bfloat16().float()

    @staticmethod
    def backward(ctx, g):
        return g.bfloat16().float()


class _RoundValue(torch.autograd.Function):
    """bf16 operand copy of an fp32 parameter: rounded forward, fp32 gradient passes through."""

    @staticmethod
    def forward(ctx, x):
        return x.bfloat16().float()

    @staticmethod
    def backward(ctx, g):
        return g


class _RoundGrad(torch.autograd.Function):
    """gradient stored in bf16 where the forward value is fp32 (dlogits -> fc GEMMs)."""

    @staticmethod
    def forward(ctx, x):
        return x.view_as(x)

    @staticmethod
    def backward(ctx, g):
        return g.bfloat16().float()


def _act_store(x, emu):
    return _RoundBoth.apply(x) if emu else x


def _w_operand(w, emu):
    return _RoundValue.apply(w) if emu else w


def _conv_bn(sd, prefix, x, k, stride, training, emu):
    """conv (bf16-stored output when emulating) -> training/eval BatchNorm in fp32 (not yet stored)."""
    y = F.conv2d(x, _w_operand(sd[f'{prefix}.layer.0.weight'], emu), None, stride, k // 2)
    y = _act_store(y, emu)
    bn = f'{prefix}.layer.1'
    y = F.batch_norm(y, sd[f'{bn}.running_mean'], sd[f'{bn}.running_var'], sd[f'{bn}.weight'], sd[f'{bn}.bias'],
                     training, BN_MOMENTUM, BN_EPS)
    if training:
        sd[f'{bn}.num_batches_tracked'] += 1
    return y


def _keep(trace, key, t):
    """Records an intermediate tensor (and asks autograd to keep its gradient) for the
    stage-by-stage parity tests."""
    if trace is not None:
        if t.requires_grad:
            t.retain_grad()
        trace[key] = t
    return t


def features(sd, x, arch, training=True, emulate_bf16=False, trace=None, prefix=''):
    """The convolutional body (stem, max pool, 4 stages) of `arch`: returns the last stage's output (C5 for the
    ImageNet nets).  `prefix` is prepended to every state-dict key (DETR keeps the body under 'backbone.',
    SimpleAICV/detection/models/backbones/detr_resnet.py:256-340 — same blocks as resnet.py)."""
    emu = emulate_bf16
    block, nums, cifar = ARCHS[arch]
    specs, _ = _cba_specs(arch)
    spec = {p: (k, s) for p, _, _, k, s in specs}
    P = prefix
    if emu:
        x = x.bfloat16().float()
    x = _keep(trace, 'stem_out', _act_store(F.relu(_conv_bn(sd, P + 'conv1', x, *spec['conv1'], training, emu)), emu))
    if not cifar:
        x = _keep(trace, 'pool_out', F.max_pool2d(x, kernel_size=3, stride=2, padding=1))
    bidx = 0
    for li in range(4):
        for bi in range(nums[li]):
            p = f'layer{li + 1}.{bi}'
            inp = x
            names = ['conv1', 'conv2'] + (['conv3'] if block == 'bottleneck' else [])
            for nm in names[:-1]:
                k, s = spec[f'{p}.{nm}']
                x = _act_store(F.relu(_conv_bn(sd, f'{P}{p}.{nm}', x, k, s, training, emu)), emu)
            k, s = spec[f'{p}.{names[-1]}']
            x = _conv_bn(sd, f'{P}{p}.{names[-1]}', x, k, s, training, emu)       # no activation before the add
            if f'{p}.downsample_conv' in spec:
                k, s = spec[f'{p}.downsample_conv']
                inp = _conv_bn(sd, f'{P}{p}.downsample_conv', inp, k, s, training, emu)
            x = _keep(trace, f'block{bidx}_out', _act_store(F.relu(x + inp), emu))
            bidx += 1
    return x


def forward(sd, x, arch, training=True, emulate_bf16=False, trace=None):
    """Logits of `arch` for the NCHW fp32 batch x; running statistics in `sd` are updated in
    place when training (like nn.BatchNorm2d).  `trace` (a dict) receives the stage boundary
    tensors: 'stem_out', 'pool_out', 'block{i}_out', 'logits'."""
    emu = emulate_bf16
    x = features(sd, x, arch, training, emu, trace)
    x = _act_store(F.adaptive_avg_pool2d(x, (1, 1)).flatten(1), emu)
    z = F.linear(x, _w_operand(sd['fc.weight'], emu))
    if emu:
        z = _RoundGrad.apply(z)
    return _keep(trace, 'logits', z + sd['fc.bias'])
