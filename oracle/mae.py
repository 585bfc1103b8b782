"""Oracle: MAE pre-training model as functional fp32 torch-CPU code over a state dict.

Follows SimpleAICV/masked_image_modeling/models/vit_mae.py: :160-201 (encoder forward: patch embedding + position
encoding, random masking by argsort of noise, gather of the kept tokens, cls token, pre-LN blocks, LayerNorm), :203-225
(random_masking), :339-368 (decoder forward: mask tokens, un-shuffle by restore_ids, position encoding, blocks, LayerNorm,
fc, cls row dropped), :415-428 (model forward) and losses.py:11-31 (MSELoss over removed patches).  The blocks are the ViT
blocks of oracle/vit.py's forward (SimpleAICV/classification/backbones/vit.py:138-163).  The masking noise is an INPUT
(the reference draws it with torch.rand on the model's device), so that CPU oracle and GPU runtime mask the same patches.
TEST INFRASTRUCTURE - see oracle/__init__.py.
"""
import math

import numpy as np
import torch
import torch.nn.functional as F

from .convnets import _RoundBoth, _RoundGrad, _RoundValue
from .vit import LN_EPS, _linear_default

# name: (patch, encoder dim / depth / heads, decoder dim / depth / heads, mlp ratio)
ARCHS = {
    'vit_base_patch16_224_mae_pretrain_model': (16, 768, 12, 12, 512, 8, 16, 4),
    'vit_large_patch16_224_mae_pretrain_model': (16, 1024, 24, 16, 512, 8, 16, 4),
    'vit_huge_patch14_224_mae_pretrain_model': (14, 1280, 32, 16, 512, 8, 16, 4),
}


def sincos_2d(planes, patch_nums):
    """vit_mae.py:100-158 (w coordinate first, zero row for the cls token)."""
    def one_d(p, grid):
        omega = np.arange(p // 2, dtype=np.float32)
        omega /= p / 2.
        omega = 1. / 10000 ** omega
        out = np.einsum('m,d->md', grid.reshape(-1), omega)
        return np.concatenate([np.sin(out), np.cos(out)], axis=1)
    gh = np.arange(patch_nums, dtype=np.float32)
    gw = np.arange(patch_nums, dtype=np.float32)
    grid = np.stack(np.meshgrid(gw, gh), axis=0).reshape([2, 1, patch_nums, patch_nums])
    enc = np.concatenate([one_d(planes // 2, grid[0]), one_d(planes // 2, grid[1])], axis=1)
    enc = np.concatenate([np.zeros([1, planes]), enc], axis=0)
    return torch.from_numpy(enc).float().unsqueeze(0)


def _blocks_default(prefix, dim, depth, ratio, sd, linears):
    for i in range(depth):
        p = f'{prefix}.blocks.{i}'
        sd[f'{p}.norm1.weight'], sd[f'{p}.norm1.bias'] = torch.ones(dim), torch.zeros(dim)
        for name, (o, n) in (('attn.qkv', (dim * 3, dim)), ('attn.proj', (dim, dim))):
            sd[f'{p}.{name}.weight'], sd[f'{p}.{name}.bias'] = _linear_default(o, n)
            linears.append(f'{p}.{name}')
        sd[f'{p}.norm2.weight'], sd[f'{p}.norm2.bias'] = torch.ones(dim), torch.zeros(dim)
        for name, (o, n) in (('mlp.fc1', (dim * ratio, dim)), ('mlp.fc2', (dim, dim * ratio))):
            sd[f'{p}.{name}.weight'], sd[f'{p}.{name}.bias'] = _linear_default(o, n)
            linears.append(f'{p}.{name}')


def _xavier(sd, names):
    for n in names:
        torch.nn.init.xavier_uniform_(sd[f'{n}.weight'])
        sd[f'{n}.bias'].zero_()


def init_state(arch, seed, image_size=224, enc_depth=None, dec_depth=None):
    """Seeded state identical to the reference constructor after torch.manual_seed(seed) (vit_mae.py:25-98, :227-283,
    :370-414): default Conv2d / Linear draws in construction order, then per sub-model the xavier / normal(.02) re-draws."""
    patch, dim, depth, heads, ddim, ddepth, dheads, ratio = ARCHS[arch]
    depth, ddepth = enc_depth or depth, dec_depth or ddepth
    torch.manual_seed(seed)
    pn = image_size // patch
    sd = {}
    # ---- encoder
    sd['encoder.cls_token'] = torch.zeros(1, 1, dim)
    sd['encoder.pos_embed'] = torch.zeros(1, pn * pn + 1, dim)
    w = torch.empty(dim, 3, patch, patch)
    torch.nn.init.kaiming_uniform_(w, a=math.sqrt(5))
    bound = 1 / math.sqrt(3 * patch * patch)
    sd['encoder.patch_embed.proj.weight'] = w
    sd['encoder.patch_embed.proj.bias'] = torch.empty(dim).uniform_(-bound, bound)
    lin_e = []
    _blocks_default('encoder', dim, depth, ratio, sd, lin_e)
    sd['encoder.norm.weight'], sd['encoder.norm.bias'] = torch.ones(dim), torch.zeros(dim)
    sd['encoder.pos_embed'].copy_(sincos_2d(dim, pn))
    torch.nn.init.xavier_uniform_(sd['encoder.patch_embed.proj.weight'].view(dim, -1))
    torch.nn.init.normal_(sd['encoder.cls_token'], std=.02)
    _xavier(sd, lin_e)
    # ---- decoder
    sd['decoder.mask_token'] = torch.zeros(1, 1, ddim)
    sd['decoder.pos_embed'] = torch.zeros(1, pn * pn + 1, ddim)
    lin_d = []
    _blocks_default('decoder', ddim, ddepth, ratio, sd, lin_d)
    sd['decoder.norm.weight'], sd['decoder.norm.bias'] = torch.ones(ddim), torch.zeros(ddim)
    sd['decoder.fc.weight'], sd['decoder.fc.bias'] = _linear_default(patch * patch * 3, ddim)
    sd['decoder.pos_embed'].copy_(sincos_2d(ddim, pn))
    torch.nn.init.normal_(sd['decoder.mask_token'], std=.02)
    _xavier(sd, lin_d + ['decoder.fc'])
    # ---- bridge
    sd['encoder_to_decoder.weight'], sd['encoder_to_decoder.bias'] = _linear_default(ddim, dim)
    _xavier(sd, ['encoder_to_decoder'])
    return sd


FROZEN = ('encoder.pos_embed', 'decoder.pos_embed')


def _blocks(sd, prefix, x, dim, depth, heads, rb, rw, rg):
    b, l, _ = x.shape
    hd = dim // heads
    scale = hd ** -0.5
    for i in range(depth):
        p = f'{prefix}.blocks.{i}'
        y = rb(F.layer_norm(x, (dim,), sd[f'{p}.norm1.weight'], sd[f'{p}.norm1.bias'], LN_EPS))
        qkv = rb(F.linear(y, rw(sd[f'{p}.attn.qkv.weight']), sd[f'{p}.attn.qkv.bias']))
        q, k, v = torch.unbind(qkv.view(b, l, 3, heads, hd).permute(2, 0, 3, 1, 4), dim=0)
        attn = ((q @ k.transpose(-2, -1)) * scale).softmax(dim=-1)
        o = rb((rw(attn) @ v).transpose(1, 2).reshape(b, l, dim))
        x = x + (rg(F.linear(o, rw(sd[f'{p}.attn.proj.weight']))) + sd[f'{p}.attn.proj.bias'])
        y = rb(F.layer_norm(x, (dim,), sd[f'{p}.norm2.weight'], sd[f'{p}.norm2.bias'], LN_EPS))
        u = rb(F.linear(y, rw(sd[f'{p}.mlp.fc1.weight']), sd[f'{p}.mlp.fc1.bias']))
        h = rb(F.gelu(u))
        x = x + (rg(F.linear(h, rw(sd[f'{p}.mlp.fc2.weight']))) + sd[f'{p}.mlp.fc2.bias'])
    return x


def forward(sd, x, noise, arch, mask_ratio=0.75, emulate_bf16=False, enc_depth=None, dec_depth=None):
    """Returns (pred [B, L, p*p*3], mask [B, L]).  emulate_bf16 rounds to bf16 at the kernels' storage points (as
    oracle/vit.py); the residual streams stay fp32."""
    patch, dim, depth, heads, ddim, ddepth, dheads, ratio = ARCHS[arch]
    depth, ddepth = enc_depth or depth, dec_depth or ddepth
    emu = emulate_bf16
    rb = (lambda t: _RoundBoth.apply(t)) if emu else (lambda t: t)
    rw = (lambda t: _RoundValue.apply(t)) if emu else (lambda t: t)
    rg = (lambda t: _RoundGrad.apply(t)) if emu else (lambda t: t)
    if emu:
        x = x.bfloat16().float()
    t = F.conv2d(x, rw(sd['encoder.patch_embed.proj.weight']), None, stride=patch)
    t = rg(t) + sd['encoder.patch_embed.proj.bias'].view(1, -1, 1, 1)
    t = t.flatten(2).transpose(1, 2)
    t = t + sd['encoder.pos_embed'][:, 1:, :]
    b, n, c = t.shape
    keep_len = int(n * (1 - mask_ratio))
    shuffle_ids = torch.argsort(noise, dim=1)
    restore_ids = torch.argsort(shuffle_ids, dim=1)
    keep_ids = shuffle_ids[:, :keep_len]
    mask = torch.ones(b, n)
    mask[:, :keep_len] = 0
    mask = torch.gather(mask, dim=1, index=restore_ids)
    t = torch.gather(t, dim=1, index=keep_ids.unsqueeze(-1).repeat(1, 1, c))
    cls = (sd['encoder.cls_token'] + sd['encoder.pos_embed'][:, :1, :]).expand(b, -1, -1)
    h = torch.cat((cls, t), dim=1)
    h = _blocks(sd, 'encoder', h, dim, depth, heads, rb, rw, rg)
    h = rb(F.layer_norm(h, (dim,), sd['encoder.norm.weight'], sd['encoder.norm.bias'], LN_EPS))
    y = rg(F.linear(h, rw(sd['encoder_to_decoder.weight']))) + sd['encoder_to_decoder.bias']
    mask_tokens = sd['decoder.mask_token'].repeat(b, n + 1 - y.shape[1], 1)
    y_ = torch.cat([y[:, 1:, :], mask_tokens], dim=1)
    y_ = torch.gather(y_, dim=1, index=restore_ids.unsqueeze(-1).repeat(1, 1, ddim))
    h = torch.cat([y[:, :1, :], y_], dim=1) + sd['decoder.pos_embed']
    h = _blocks(sd, 'decoder', h, ddim, ddepth, dheads, rb, rw, rg)
    h = rb(F.layer_norm(h, (ddim,), sd['decoder.norm.weight'], sd['decoder.norm.bias'], LN_EPS))
    pred = rg(F.linear(h, rw(sd['decoder.fc.weight']))) + sd['decoder.fc.bias']
    return pred[:, 1:, :], mask


def images_to_patch(images, patch):
    """vit_mae.py:437-449."""
    pn = images.shape[2] // patch
    x = images.reshape(images.shape[0], 3, pn, patch, pn, patch)
    x = torch.einsum('nchpwq->nhwpqc', x)
    return x.reshape(x.shape[0], pn * pn, patch * patch * 3)


def mse_loss(pred, label, mask):
    """losses.py:17-31."""
    loss = ((pred.float() - label.float()) ** 2).mean(dim=-1)
    return (loss * mask.float()).sum() / (mask.float().sum() + 1e-4)


def loss_and_grads(sd, x, noise, arch, mask_ratio=0.75, emulate_bf16=False, enc_depth=None, dec_depth=None):
    names = [n for n in sd if n not in FROZEN]
    for n in names:
        sd[n].requires_grad_(True)
        sd[n].grad = None
    pred, mask = forward(sd, x, noise, arch, mask_ratio, emulate_bf16, enc_depth, dec_depth)
    loss = mse_loss(pred, images_to_patch(x, ARCHS[arch][0]), mask)
    loss.backward()
    grads = {n: sd[n].grad.detach().clone() for n in names}
    for n in names:
        sd[n].requires_grad_(False)
        sd[n].grad = None
    return pred.detach(), mask, loss.detach(), grads
