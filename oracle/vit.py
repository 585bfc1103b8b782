"""Oracle: ViT forward as functional fp32 torch-CPU code over a state dict.

Follows SimpleAICV/classification/backbones/vit.py:18-47 (PatchEmbeddingBlock: 16x16/16 conv,
flatten, transpose), :50-80 (MultiHeadAttention: packed qkv linear, (q k^T)*scale, softmax,
@v, proj), :83-99 (FeedForward: fc1, exact GELU, fc2), :138-163 (pre-LN residual block),
:239-262 (ViT.forward: cls token, positional embedding, blocks, global-pool / cls head).
Dropout / DropPath are identity at the probabilities used for parity (0).  TEST INFRASTRUCTURE —
see oracle/__init__.py.
"""
import math

import torch
import torch.nn.functional as F

from .convnets import _RoundBoth, _RoundGrad, _RoundValue, _keep

ARCHS = {
    # name: (patch, dim, depth, heads, mlp ratio)
    'vit_base_patch16': (16, 768, 12, 12, 4),
    'vit_large_patch16': (16, 1024, 24, 16, 4),
    'vit_huge_patch14': (14, 1280, 32, 16, 4),
}
LN_EPS = 1e-6


def _linear_default(out_f, in_f):
    w = torch.empty(out_f, in_f)
    torch.nn.init.kaiming_uniform_(w, a=math.sqrt(5))
    bound = 1 / math.sqrt(in_f)
    return w, torch.empty(out_f).uniform_(-bound, bound)


def init_state(arch, num_classes, seed, image_size=224, depth=None):
    """Seeded initial state identical to the reference constructor after torch.manual_seed(seed)
    (vit.py:191-237): default Conv2d/Linear inits are drawn in construction order, then every
    Linear is re-drawn trunc_normal(.02)/zero bias, pos_embed trunc_normal(.02), cls_token
    normal(1e-6), fc trunc_normal(2e-5)/zeros.  `depth` overrides the number of blocks (tests)."""
    patch, dim, nblocks, heads, ratio = ARCHS[arch]
    nblocks = depth or nblocks
    torch.manual_seed(seed)
    sd = {}
    w = torch.empty(dim, 3, patch, patch)
    torch.nn.init.kaiming_uniform_(w, a=math.sqrt(5))
    bound = 1 / math.sqrt(3 * patch * patch)
    sd['patch_embed.proj.weight'] = w
    sd['patch_embed.proj.bias'] = torch.empty(dim).uniform_(-bound, bound)
    npatch = (image_size // patch) ** 2
    cls = torch.zeros(1, 1, dim)
    pos = torch.ones(1, npatch + 1, dim)
    linears = []
    blocks = {}
    for i in range(nblocks):
        p = f'blocks.{i}'
        blocks[f'{p}.norm1.weight'], blocks[f'{p}.norm1.bias'] = torch.ones(dim), torch.zeros(dim)
        for name, (o, n) in (('attn.qkv', (dim * 3, dim)), ('attn.proj', (dim, dim))):
            blocks[f'{p}.{name}.weight'], blocks[f'{p}.{name}.bias'] = _linear_default(o, n)
            linears.append(f'{p}.{name}')
        blocks[f'{p}.norm2.weight'], blocks[f'{p}.norm2.bias'] = torch.ones(dim), torch.zeros(dim)
        for name, (o, n) in (('mlp.fc1', (dim * ratio, dim)), ('mlp.fc2', (dim, dim * ratio))):
            blocks[f'{p}.{name}.weight'], blocks[f'{p}.{name}.bias'] = _linear_default(o, n)
            linears.append(f'{p}.{name}')
    norm_w, norm_b = torch.ones(dim), torch.zeros(dim)
    fc_w, fc_b = _linear_default(num_classes, dim)
    sd['cls_token'], sd['pos_embed'] = cls, pos
    # register in the reference's state_dict order: cls_token, pos_embed, patch_embed, blocks, norm, fc
    sd = {'cls_token': cls, 'pos_embed': pos, 'patch_embed.proj.weight': sd['patch_embed.proj.weight'],
          'patch_embed.proj.bias': sd['patch_embed.proj.bias'], **blocks,
          'norm.weight': norm_w, 'norm.bias': norm_b, 'fc.weight': fc_w, 'fc.bias': fc_b}
    for name in linears + ['fc']:
        torch.nn.init.trunc_normal_(sd[f'{name}.weight'], std=.02)
        sd[f'{name}.bias'].zero_()
    torch.nn.init.trunc_normal_(sd['pos_embed'], std=.02)
    torch.nn.init.normal_(sd['cls_token'], std=1e-6)
    torch.nn.init.trunc_normal_(sd['fc.weight'], std=2e-5)
    sd['fc.bias'].zero_()
    return sd


def param_names(sd):
    return list(sd.keys())


def forward(sd, x, arch, global_pool=False, emulate_bf16=False, trace=None, depth=None):
    """Logits for the NCHW fp32 batch x.  emulate_bf16 inserts round-to-bf16 at the kernels'
    storage points (LayerNorm outputs, qkv, attention probabilities/outputs, MLP hidden, GEMM
    operand copies of weights and of output gradients); the residual stream stays fp32."""
    emu = emulate_bf16
    patch, dim, nblocks, heads, ratio = ARCHS[arch]
    nblocks = depth or nblocks
    rb = (lambda t: _RoundBoth.apply(t)) if emu else (lambda t: t)      # bf16-stored activation
    rw = (lambda t: _RoundValue.apply(t)) if emu else (lambda t: t)     # bf16 operand copy
    rg = (lambda t: _RoundGrad.apply(t)) if emu else (lambda t: t)      # bf16 gradient operand
    if emu:
        x = x.bfloat16().float()
    t = F.conv2d(x, rw(sd['patch_embed.proj.weight']), None, stride=patch)
    t = rg(t) + sd['patch_embed.proj.bias'].view(1, -1, 1, 1)
    t = t.flatten(2).transpose(1, 2)
    b, n, c = t.shape
    x = torch.cat((sd['cls_token'].expand(b, -1, -1), t), dim=1) + sd['pos_embed']
    x = _keep(trace, 'tokens', x)
    hd = dim // heads
    scale = hd ** -0.5
    for i in range(nblocks):
        p = f'blocks.{i}'
        y = rb(F.layer_norm(x, (dim,), sd[f'{p}.norm1.weight'], sd[f'{p}.norm1.bias'], LN_EPS))
        qkv = rb(F.linear(y, rw(sd[f'{p}.attn.qkv.weight']), sd[f'{p}.attn.qkv.bias']))
        qkv = qkv.view(b, n + 1, 3, heads, hd).permute(2, 0, 3, 1, 4)
        q, k, v = torch.unbind(qkv, dim=0)
        attn = ((q @ k.transpose(-2, -1)) * scale).softmax(dim=-1)
        o = rb((rw(attn) @ v).transpose(1, 2).reshape(b, n + 1, dim))
        x = x + (rg(F.linear(o, rw(sd[f'{p}.attn.proj.weight']))) + sd[f'{p}.attn.proj.bias'])
        y = rb(F.layer_norm(x, (dim,), sd[f'{p}.norm2.weight'], sd[f'{p}.norm2.bias'], LN_EPS))
        u = rb(F.linear(y, rw(sd[f'{p}.mlp.fc1.weight']), sd[f'{p}.mlp.fc1.bias']))
        h = rb(F.gelu(u))
        x = x + (rg(F.linear(h, rw(sd[f'{p}.mlp.fc2.weight']))) + sd[f'{p}.mlp.fc2.bias'])
        x = _keep(trace, f'block{i}_out', x)
    if global_pool:
        z = x[:, 1:, :].mean(dim=1)
        z = F.layer_norm(z, (dim,), sd['norm.weight'], sd['norm.bias'], LN_EPS)
    else:
        z = F.layer_norm(x, (dim,), sd['norm.weight'], sd['norm.bias'], LN_EPS)[:, 0]
    z = rb(z)
    return _keep(trace, 'logits', rg(F.linear(z, rw(sd['fc.weight']))) + sd['fc.bias'])


def loss_and_grads(sd, x, labels, arch, global_pool=False, emulate_bf16=False, trace=None, depth=None):
    from .train_step import ce_loss
    names = param_names(sd)
    for n in names:
        sd[n].requires_grad_(True)
        sd[n].grad = None
    logits = forward(sd, x, arch, global_pool, emulate_bf16, trace, depth)
    loss = ce_loss(logits, labels)
    loss.backward()
    grads = {n: sd[n].grad.detach().clone() for n in names}
    for n in names:
        sd[n].requires_grad_(False)
        sd[n].grad = None
    return logits.detach(), loss.detach(), grads
