"""Oracle: DINOv3 ViT backbone (+ the SAM neck of the DINOv3 image encoder) forward as functional fp32 torch-CPU code over
a state dict.

Follows SimpleAICV/detection/models/backbones/dinov3vit.py:35-71 (PatchEmbed: 16x16/16 conv with bias, no norm),
:144-268 (RopePositionEmbedding, "separate" coordinates, the rescale factor passed in instead of drawn), :271-282 / :347-367
(rope_apply on q and k), :285-300 (qkv bias * bias_mask), :303-345 (SelfAttention), :370-469 (SelfAttentionBlock with
LayerScale, drop path 0), :93-141 (Mlp with exact GELU / SwiGLUFFN), :550-572 (final LayerNorm, NCHW output) and
dinov3_image_encoder.py:19-75 (neck: 1x1 conv, LayerNorm2d, 3x3 conv, LayerNorm2d).  emulate_bf16 rounds values and
gradients where the runtime's kernels store bf16.  TEST INFRASTRUCTURE — see oracle/__init__.py.
"""
import math

import torch
import torch.nn.functional as F

from .convnets import _keep, _RoundBoth, _RoundGrad, _RoundValue
from .vit import _linear_default

LN_EPS = 1e-6
BUFFERS = ('rope_embed.periods', 'bias_mask')
# constructor name -> (embedding_planes, block_nums, head_nums, ffn_ratio, ffn_layer); rescale_coords = 2 for all
ARCHS = {
    'dinov3_vit_small_patch16_backbone': (384, 12, 6, 4, 'mlp'),
    'dinov3_vit_small_plus_patch16_backbone': (384, 12, 6, 6, 'swiglu'),
    'dinov3_vit_base_patch16_backbone': (768, 12, 12, 4, 'mlp'),
    'dinov3_vit_large_patch16_backbone': (1024, 24, 16, 4, 'mlp'),
    'dinov3_vit_large_plus_patch16_backbone': (1024, 24, 16, 6, 'swiglu'),
    'dinov3_vit_huge_plus_patch16_backbone': (1280, 32, 20, 6, 'swiglu'),
}


def swiglu_hidden(c, ffn_ratio):
    d = int(int(c * ffn_ratio) * 2 / 3)
    return d + (-d % 8)


def init_state(seed, embedding_planes, block_nums, head_nums, ffn_ratio, ffn_layer, out_planes=None, patch_size=16, prefix=''):
    """Seeded state identical to constructing the reference backbone (and, with out_planes, the encoder's neck after it)
    right after torch.manual_seed(seed): default Conv2d / Linear inits drawn in construction order, the PatchEmbed
    uniform re-draw, then every Linear re-drawn trunc_normal(0.02) with zero bias; LayerScale 1e-5, LayerNorm (1, 0)."""
    torch.manual_seed(seed)
    c = embedding_planes
    hd = c // head_nums
    hid = swiglu_hidden(c, ffn_ratio) if ffn_layer == 'swiglu' else int(c * ffn_ratio)
    sd = {}
    w = torch.empty(c, 3, patch_size, patch_size)
    torch.nn.init.kaiming_uniform_(w, a=math.sqrt(5))
    torch.empty(c).uniform_(-1 / math.sqrt(3 * patch_size * patch_size), 1 / math.sqrt(3 * patch_size * patch_size))
    k = 1 / (3 * patch_size ** 2)
    sd['patch_embed.proj.weight'] = torch.nn.init.uniform_(w, -math.sqrt(k), math.sqrt(k))
    sd['patch_embed.proj.bias'] = torch.empty(c).uniform_(-math.sqrt(k), math.sqrt(k))
    sd['rope_embed.periods'] = 100.0 ** (2 * torch.arange(hd // 4) / (hd // 2))
    mask = torch.ones(3 * c)
    mask[c:2 * c] = 0
    linears = []
    for i in range(block_nums):
        p = f'blocks.{i}'
        sd[f'{p}.norm1.weight'], sd[f'{p}.norm1.bias'] = torch.ones(c), torch.zeros(c)
        shapes = [('attn.qkv', 3 * c, c), ('attn.proj', c, c)]
        shapes += ([('mlp.w1', hid, c), ('mlp.w2', hid, c), ('mlp.w3', c, hid)] if ffn_layer == 'swiglu'
                   else [('mlp.fc1', hid, c), ('mlp.fc2', c, hid)])
        for j, (n, o, ii) in enumerate(shapes):
            sd[f'{p}.{n}.weight'], sd[f'{p}.{n}.bias'] = _linear_default(o, ii)
            linears.append(f'{p}.{n}')
            if n == 'attn.qkv':
                sd[f'{p}.attn.qkv.bias_mask'] = mask.clone()
            if n == 'attn.proj':
                sd[f'{p}.ls1.gamma'] = torch.full((c,), 1e-5)
                sd[f'{p}.norm2.weight'], sd[f'{p}.norm2.bias'] = torch.ones(c), torch.zeros(c)
        sd[f'{p}.ls2.gamma'] = torch.full((c,), 1e-5)
    sd['norm.weight'], sd['norm.bias'] = torch.ones(c), torch.zeros(c)
    for n in linears:
        torch.nn.init.trunc_normal_(sd[f'{n}.weight'], std=0.02)
        sd[f'{n}.bias'].zero_()
    sd = {prefix + k: v for k, v in sd.items()}
    if out_planes is not None:
        w0 = torch.empty(out_planes, c, 1, 1)
        torch.nn.init.kaiming_uniform_(w0, a=math.sqrt(5))
        sd['neck.0.weight'] = w0
        sd['neck.1.weight'], sd['neck.1.bias'] = torch.ones(out_planes), torch.zeros(out_planes)
        w2 = torch.empty(out_planes, out_planes, 3, 3)
        torch.nn.init.kaiming_uniform_(w2, a=math.sqrt(5))
        sd['neck.2.weight'] = w2
        sd['neck.3.weight'], sd['neck.3.bias'] = torch.ones(out_planes), torch.zeros(out_planes)
    return sd


def draw_rescale(rescale_coords=2):
    """The rescale factor a training forward draws from torch's CPU generator (dinov3vit.py:247-253)."""
    m = math.log(rescale_coords)
    return torch.empty(1).uniform_(-m, m).exp()


def rope_table(periods, H, W, rescale=None):
    """(sin, cos) [H*W, hd], "separate" normalisation; `rescale`: the factor of a training forward (None in eval)."""
    coords = torch.stack(torch.meshgrid(torch.arange(0.5, H) / H, torch.arange(0.5, W) / W, indexing='ij'), dim=-1).flatten(0, 1)
    coords = 2.0 * coords - 1.0
    if rescale is not None:
        coords = coords * rescale
    angles = (2 * math.pi * coords[:, :, None] / periods[None, None, :]).flatten(1, 2).tile(2)
    return torch.sin(angles), torch.cos(angles)


def rope_apply(x, sin, cos):
    x1, x2 = x.chunk(2, dim=-1)
    return x * cos + torch.cat([-x2, x1], dim=-1) * sin


def forward(sd, x, head_nums, rescale=None, emulate_bf16=False, trace=None, patch_size=16, prefix=''):
    """x: NCHW fp32 image batch -> fp32 NCHW (neck output when sd has neck.* keys, else the final LayerNorm's)."""
    emu = emulate_bf16
    rb = (lambda t: _RoundBoth.apply(t)) if emu else (lambda t: t)
    rw = (lambda t: _RoundValue.apply(t)) if emu else (lambda t: t)
    rg = (lambda t: _RoundGrad.apply(t)) if emu else (lambda t: t)
    P = prefix
    if emu:
        x = x.bfloat16().float()
    t = F.conv2d(x, rw(sd[P + 'patch_embed.proj.weight']), None, stride=patch_size)
    t = rg(t) + sd[P + 'patch_embed.proj.bias'].view(1, -1, 1, 1)
    b, c, h, w = t.shape
    x = t.flatten(2).transpose(1, 2)                                        # [B, L, C]
    x = _keep(trace, 'tokens', x)
    hd = c // head_nums
    sin, cos = rope_table(sd[P + 'rope_embed.periods'], h, w, rescale)
    nblocks = len([k for k in sd if k.startswith(P + 'blocks.') and k.endswith('.norm1.weight')])
    for i in range(nblocks):
        p = f'{P}blocks.{i}'
        y = rb(F.layer_norm(x, (c,), sd[f'{p}.norm1.weight'], sd[f'{p}.norm1.bias'], LN_EPS))
        qkv = rb(F.linear(y, rw(sd[f'{p}.attn.qkv.weight']), sd[f'{p}.attn.qkv.bias'] * sd[f'{p}.attn.qkv.bias_mask']))
        q, k, v = qkv.reshape(b, h * w, 3, head_nums, hd).permute(2, 0, 3, 1, 4).unbind(0)
        q, k = rb(rope_apply(q, sin, cos)), rb(rope_apply(k, sin, cos))
        attn = ((q @ k.transpose(-2, -1)) * hd ** -0.5).softmax(dim=-1)
        o = rb((rw(attn) @ v).transpose(1, 2).reshape(b, h * w, c))
        pa = rb(F.linear(o, rw(sd[f'{p}.attn.proj.weight']), sd[f'{p}.attn.proj.bias']))
        x = x + sd[f'{p}.ls1.gamma'] * pa
        y = rb(F.layer_norm(x, (c,), sd[f'{p}.norm2.weight'], sd[f'{p}.norm2.bias'], LN_EPS))
        if f'{p}.mlp.w3.weight' in sd:
            a = rb(F.linear(y, rw(sd[f'{p}.mlp.w1.weight']), sd[f'{p}.mlp.w1.bias']))
            g = rb(F.linear(y, rw(sd[f'{p}.mlp.w2.weight']), sd[f'{p}.mlp.w2.bias']))
            f = rb(F.linear(rb(rb(F.silu(a)) * g), rw(sd[f'{p}.mlp.w3.weight']), sd[f'{p}.mlp.w3.bias']))
        else:
            u = rb(F.linear(y, rw(sd[f'{p}.mlp.fc1.weight']), sd[f'{p}.mlp.fc1.bias']))
            f = rb(F.linear(rb(F.gelu(u)), rw(sd[f'{p}.mlp.fc2.weight']), sd[f'{p}.mlp.fc2.bias']))
        x = x + sd[f'{p}.ls2.gamma'] * f
        x = _keep(trace, f'block{i}_out', x)
    y = rb(F.layer_norm(x, (c,), sd[P + 'norm.weight'], sd[P + 'norm.bias'], LN_EPS)).view(b, h, w, c)
    if 'neck.0.weight' not in sd:
        return _keep(trace, 'out', y.permute(0, 3, 1, 2))
    y = _keep(trace, 'neck_in', y)
    oc = sd['neck.0.weight'].shape[0]
    y1 = rg(F.linear(y, rw(sd['neck.0.weight'].view(oc, c))))
    l1 = rb(F.layer_norm(y1, (oc,), sd['neck.1.weight'], sd['neck.1.bias'], LN_EPS))
    y2 = rb(F.conv2d(l1.permute(0, 3, 1, 2), rw(sd['neck.2.weight']), None, 1, 1))
    l2 = rb(F.layer_norm(y2.permute(0, 2, 3, 1), (oc,), sd['neck.3.weight'], sd['neck.3.bias'], LN_EPS))
    return _keep(trace, 'out', l2.permute(0, 3, 1, 2))


def loss_and_grads(sd, x, target, head_nums, rescale=None, emulate_bf16=False, trace=None, prefix=''):
    """The distillation loss mean((out - target)^2) (distill_losses.py MSELoss).  Returns (out, loss, grads of every
    parameter; the buffers rope_embed.periods and *.bias_mask get none)."""
    names = [n for n in sd if not n.endswith(BUFFERS)]
    for n in names:
        sd[n].requires_grad_(True)
        sd[n].grad = None
    out = forward(sd, x, head_nums, rescale, emulate_bf16, trace, prefix=prefix)
    loss = F.mse_loss(out.float(), target)
    loss.backward()
    grads = {n: sd[n].grad.detach().clone() for n in names}
    for n in names:
        sd[n].requires_grad_(False)
        sd[n].grad = None
    return out.detach(), loss.detach(), grads
