"""Oracle: DETR forward as functional fp32 torch-CPU code over a state dict.

Follows SimpleAICV/detection/models/detr.py:44-90 (TransformerEncoderLayer: post-LN, q = k = src + pos, v = src),
:93-180 (TransformerDecoderLayer: self-attention on tgt + query_pos, cross-attention to memory + pos, FFN), :183-270
(DETRTransformer: 6 + 6 layers, decoder_norm on every decoder output), :273-364 (DETR: C5 of the backbone, mask resize,
sine position embedding, 1x1 proj_conv, transformer, heads), backbones/detr_resnet.py:28-64 (PositionEmbeddingBlock),
:256-340 (DetrResNetBackbone: the classification ResNet body) and head.py:184-213 (DETRClsRegHead).

One behaviour of the reference is kept deliberately: DETR.forward hands ``masks.float()`` to the transformer, so
nn.MultiheadAttention receives a FLOAT key_padding_mask, which torch ADDS to the attention logits (+1.0 on padded keys)
instead of excluding those keys (detr.py:333-346; torch.nn.functional._canonical_mask).  `key_bias` below is that
additive term.  Dropout (p = 0.1 in the reference constructor) is the identity here: parity runs set p = 0 on both
sides.  TEST INFRASTRUCTURE — see oracle/__init__.py.
"""
import math

import torch
import torch.nn.functional as F

from . import convnets
from .convnets import _keep, _RoundBoth, _RoundGrad, _RoundValue

LN_EPS = 1e-5
BACKBONES = {'resnet18_detr': 'resnet18', 'resnet34_detr': 'resnet34', 'resnet50_detr': 'resnet50',
             'resnet101_detr': 'resnet101', 'resnet152_detr': 'resnet152'}
HIDDEN, HEADS, FF_RATIO, ENC_LAYERS, DEC_LAYERS = 256, 8, 4, 6, 6


def _linear_default(sd, name, out_f, in_f):
    """nn.Linear.reset_parameters: kaiming_uniform(a=sqrt(5)) weight, uniform(+-1/sqrt(fan_in)) bias."""
    w = torch.empty(out_f, in_f)
    torch.nn.init.kaiming_uniform_(w, a=math.sqrt(5))
    bound = 1 / math.sqrt(in_f)
    sd[f'{name}.weight'] = w
    sd[f'{name}.bias'] = torch.empty(out_f).uniform_(-bound, bound)


def _mha_default(sd, name, c):
    """nn.MultiheadAttention.__init__: out_proj is built (default Linear init) before _reset_parameters draws the
    packed in_proj_weight with xavier_uniform and zeroes in_proj_bias / out_proj.bias."""
    op = {}
    _linear_default(op, 'out_proj', c, c)
    w = torch.empty(3 * c, c)
    torch.nn.init.xavier_uniform_(w)
    sd[f'{name}.in_proj_weight'] = w
    sd[f'{name}.in_proj_bias'] = torch.zeros(3 * c)
    sd[f'{name}.out_proj.weight'] = op['out_proj.weight']
    sd[f'{name}.out_proj.bias'] = torch.zeros(c)


def _ln_default(sd, name, c):
    sd[f'{name}.weight'], sd[f'{name}.bias'] = torch.ones(c), torch.zeros(c)


def init_state(arch, seed, num_classes=80, query_nums=100, enc_layers=ENC_LAYERS, dec_layers=DEC_LAYERS):
    """Seeded initial state identical to constructing the reference DETR after torch.manual_seed(seed); keys in the
    reference's state_dict order.  (enc_layers / dec_layers other than 6 exist for the reduced test fixtures; the
    reference constructor always builds 6 + 6.)"""
    torch.manual_seed(seed)
    res = BACKBONES[arch]
    specs, feat = convnets._cba_specs(res)
    sd = {}
    for prefix, cin, cout, k, _ in specs:                       # backbone convs: default init in construction order
        w = torch.empty(cout, cin, k, k)
        torch.nn.init.kaiming_uniform_(w, a=math.sqrt(5))
        p = f'backbone.{prefix}.layer'
        sd[f'{p}.0.weight'] = w
        sd[f'{p}.1.weight'], sd[f'{p}.1.bias'] = torch.ones(cout), torch.zeros(cout)
        sd[f'{p}.1.running_mean'], sd[f'{p}.1.running_var'] = torch.zeros(cout), torch.ones(cout)
        sd[f'{p}.1.num_batches_tracked'] = torch.tensor(0, dtype=torch.long)
    for prefix, *_ in specs:                                    # detr_resnet.py:311-318
        torch.nn.init.kaiming_normal_(sd[f'backbone.{prefix}.layer.0.weight'], mode='fan_out', nonlinearity='relu')
    c = HIDDEN
    pw = torch.empty(c, feat, 1, 1)                              # proj_conv: nn.Conv2d default init
    torch.nn.init.kaiming_uniform_(pw, a=math.sqrt(5))
    sd['proj_conv.weight'] = pw
    sd['proj_conv.bias'] = torch.empty(c).uniform_(-1 / math.sqrt(feat), 1 / math.sqrt(feat))
    for i in range(enc_layers):
        p = f'transformer.encoder_blocks.{i}'
        _mha_default(sd, f'{p}.attention', c)
        _linear_default(sd, f'{p}.linear1', c * FF_RATIO, c)
        _linear_default(sd, f'{p}.linear2', c, c * FF_RATIO)
        _ln_default(sd, f'{p}.norm1', c)
        _ln_default(sd, f'{p}.norm2', c)
    for i in range(dec_layers):
        p = f'transformer.decoder_blocks.{i}'
        _mha_default(sd, f'{p}.attention', c)
        _mha_default(sd, f'{p}.multihead_attention', c)
        _linear_default(sd, f'{p}.linear1', c * FF_RATIO, c)
        _linear_default(sd, f'{p}.linear2', c, c * FF_RATIO)
        for n in ('norm1', 'norm2', 'norm3'):
            _ln_default(sd, f'{p}.{n}', c)
    _ln_default(sd, 'transformer.decoder_norm', c)
    for k in [k for k in sd if k.startswith('transformer.')]:    # detr.py:228-230: xavier over parameters() with dim > 1
        if sd[k].dim() > 1:
            torch.nn.init.xavier_uniform_(sd[k])
    sd['query_embed.weight'] = torch.empty(query_nums, c).normal_()
    _linear_default(sd, 'head.cls_head', num_classes + 1, c)
    _linear_default(sd, 'head.reg_head.0', c, c)
    _linear_default(sd, 'head.reg_head.2', c, c)
    _linear_default(sd, 'head.reg_head.4', 4, c)
    for k in ('head.cls_head.weight', 'head.reg_head.0.weight', 'head.reg_head.2.weight', 'head.reg_head.4.weight'):
        torch.nn.init.xavier_uniform_(sd[k])                     # head.py:201-203
    return sd


def param_names(sd):
    return [k for k in sd if not (k.endswith('running_mean') or k.endswith('running_var') or k.endswith('num_batches_tracked'))]


def resize_masks(masks, h, w):
    """detr.py:318-320: nearest-neighbour resize of the bool padding masks [B, H, W] to the feature size."""
    return F.interpolate(masks.float().unsqueeze(1), size=[h, w]).to(torch.bool).squeeze(1)


def position_embedding(masks, planes=HIDDEN // 2, temperature=10000, eps=1e-6):
    """detr_resnet.py:28-64: sine embedding of the cumulative counts of unpadded rows / columns; [B, 2*planes, h, w]."""
    not_masks = ~masks
    y_embed = torch.cumsum(not_masks, 1, dtype=torch.float32)
    x_embed = torch.cumsum(not_masks, 2, dtype=torch.float32)
    scale = 2 * math.pi
    y_embed = y_embed / (y_embed[:, -1:, :] + eps) * scale
    x_embed = x_embed / (x_embed[:, :, -1:] + eps) * scale
    dim_t = torch.arange(planes, dtype=torch.float32)
    dim_t = temperature ** (2 * (dim_t // 2) / planes)
    pos_x = x_embed[:, :, :, None] / dim_t
    pos_y = y_embed[:, :, :, None] / dim_t
    pos_x = torch.stack((pos_x[:, :, :, 0::2].sin(), pos_x[:, :, :, 1::2].cos()), dim=4).flatten(3)
    pos_y = torch.stack((pos_y[:, :, :, 0::2].sin(), pos_y[:, :, :, 1::2].cos()), dim=4).flatten(3)
    return torch.cat((pos_y, pos_x), dim=3).permute(0, 3, 1, 2)


def _mha(sd, name, q_in, k_in, v_in, key_bias, fns):
    """nn.MultiheadAttention forward on batch-major tokens: q_in [B, Lq, C], k_in / v_in [B, Lk, C]; key_bias
    [B, Lk] (added to the logits of every head and query) or None.  Returns the out_proj GEMM result WITHOUT its bias
    (the caller adds it on the fp32 stream)."""
    rb, rw, rg, rv = fns
    c = q_in.shape[-1]
    hd = c // HEADS
    w, b = sd[f'{name}.in_proj_weight'], sd[f'{name}.in_proj_bias']
    q = rb(F.linear(q_in, rw(w[:c]), b[:c]))
    k = rb(F.linear(k_in, rw(w[c:2 * c]), b[c:2 * c]))
    v = rb(F.linear(v_in, rw(w[2 * c:]), b[2 * c:]))
    B, Lq, Lk = q.shape[0], q.shape[1], k.shape[1]
    if key_bias is not None:
        q = rb(q * hd ** -0.5)                                # biased path: the scaled copy of q is a stored score operand
    q = q.view(B, Lq, HEADS, hd).transpose(1, 2)
    k = k.view(B, Lk, HEADS, hd).transpose(1, 2)
    v = v.view(B, Lk, HEADS, hd).transpose(1, 2)
    s = q @ k.transpose(-2, -1)
    if key_bias is not None:
        s = s + key_bias.view(B, 1, 1, Lk)
    else:
        s = s * hd ** -0.5                                    # unbiased path: the kernel scales the fp32 scores
    a = s.softmax(dim=-1)
    o = rb((rv(a) @ v).transpose(1, 2).reshape(B, Lq, c))
    return rg(F.linear(o, rw(sd[f'{name}.out_proj.weight']))) + sd[f'{name}.out_proj.bias']


def forward(sd, x, masks, arch, training=True, emulate_bf16=False, trace=None, enc_layers=ENC_LAYERS, dec_layers=DEC_LAYERS):
    """(cls_outputs [dec_layers, B, Q, classes + 1], reg_outputs [dec_layers, B, Q, 4]) for the NCHW fp32 batch x and the
    bool padding masks [B, H, W].  emulate_bf16 inserts round-to-bf16 at the kernels' storage points: GEMM operand
    copies (weights, bf16 copies of the fp32 token stream, attention probabilities), GEMM outputs that are stored in
    bf16 (q, k, v, attention outputs, FFN hidden) and the gradients that travel in bf16; the token stream, LayerNorm
    and softmax stay fp32."""
    emu = emulate_bf16
    rb = (lambda t: _RoundBoth.apply(t)) if emu else (lambda t: t)      # bf16-stored activation (value and gradient)
    rw = (lambda t: _RoundValue.apply(t)) if emu else (lambda t: t)     # bf16 operand copy, fp32 gradient passes
    rg = (lambda t: _RoundGrad.apply(t)) if emu else (lambda t: t)      # fp32 value whose gradient is consumed in bf16
    fns = (rb, rw, rg, rw)
    c5 = convnets.features(sd, x, BACKBONES[arch], training, emu, None, prefix='backbone.')
    c5 = _keep(trace, 'c5', c5)
    B, _, h, w = c5.shape
    fm = resize_masks(masks, h, w)
    pos = position_embedding(fm).flatten(2).transpose(1, 2)             # [B, L, C]
    key_bias = fm.flatten(1).float()                                    # +1.0 on padded keys (see the module docstring)
    src = F.conv2d(c5, rw(sd['proj_conv.weight']))
    src = rg(src) + sd['proj_conv.bias'].view(1, -1, 1, 1)
    src = _keep(trace, 'src', src.flatten(2).transpose(1, 2))           # [B, L, C] fp32 stream
    C = src.shape[-1]

    def ln(t, name):
        return F.layer_norm(t, (C,), sd[f'{name}.weight'], sd[f'{name}.bias'], LN_EPS)

    def ffn(t, p):
        hid = rb(F.relu(F.linear(rw(t), rw(sd[f'{p}.linear1.weight']), sd[f'{p}.linear1.bias'])))
        return rg(F.linear(hid, rw(sd[f'{p}.linear2.weight']))) + sd[f'{p}.linear2.bias']

    mem = src
    for i in range(enc_layers):
        p = f'transformer.encoder_blocks.{i}'
        qk_in = rw(mem + pos)
        mem = ln(mem + _mha(sd, f'{p}.attention', qk_in, qk_in, rw(mem), key_bias, fns), f'{p}.norm1')
        mem = ln(mem + ffn(mem, p), f'{p}.norm2')
        mem = _keep(trace, f'enc{i}_out', mem)
    qpos = sd['query_embed.weight'].unsqueeze(0).expand(B, -1, -1)
    tgt = torch.zeros_like(qpos)
    mem_k, mem_v = rw(mem + pos), rw(mem)
    inter = []
    for i in range(dec_layers):
        p = f'transformer.decoder_blocks.{i}'
        qk_in = rw(tgt + qpos)
        tgt = ln(tgt + _mha(sd, f'{p}.attention', qk_in, qk_in, rw(tgt), None, fns), f'{p}.norm1')
        tgt = ln(tgt + _mha(sd, f'{p}.multihead_attention', rw(tgt + qpos), mem_k, mem_v, key_bias, fns), f'{p}.norm2')
        tgt = ln(tgt + ffn(tgt, p), f'{p}.norm3')
        tgt = _keep(trace, f'dec{i}_out', tgt)
        inter.append(ln(tgt, 'transformer.decoder_norm'))
    hs = rw(torch.stack(inter))                                          # [dec_layers, B, Q, C]
    cls = rg(F.linear(hs, rw(sd['head.cls_head.weight']))) + sd['head.cls_head.bias']
    r = rb(F.relu(F.linear(hs, rw(sd['head.reg_head.0.weight']), sd['head.reg_head.0.bias'])))
    r = rb(F.relu(F.linear(r, rw(sd['head.reg_head.2.weight']), sd['head.reg_head.2.bias'])))
    r = rg(F.linear(r, rw(sd['head.reg_head.4.weight']))) + sd['head.reg_head.4.bias']
    return _keep(trace, 'cls', cls), _keep(trace, 'reg', r.float().sigmoid())


def surrogate_loss(cls, reg, seed=0):
    """Deterministic smooth scalar of both outputs used by the parity tests (the real criterion, DETRLoss, runs a
    Hungarian matcher on top of these tensors; its gradient enters the model through cls / reg exactly like this one)."""
    g = torch.Generator().manual_seed(seed)
    wc = torch.randn(cls.shape, generator=g).to(cls.device)
    wr = torch.randn(reg.shape, generator=g).to(reg.device)
    return (cls.float() * wc).mean() + (reg.float() * wr).mean() + 0.1 * cls.float().square().mean()


def loss_and_grads(sd, x, masks, arch, emulate_bf16=False, trace=None, enc_layers=ENC_LAYERS, dec_layers=DEC_LAYERS):
    names = param_names(sd)
    for n in names:
        sd[n].requires_grad_(True)
        sd[n].grad = None
    cls, reg = forward(sd, x, masks, arch, True, emulate_bf16, trace, enc_layers, dec_layers)
    loss = surrogate_loss(cls, reg)
    loss.backward()
    grads = {n: (sd[n].grad.detach().clone() if sd[n].grad is not None else torch.zeros_like(sd[n])) for n in names}
    for n in names:
        sd[n].requires_grad_(False)
        sd[n].grad = None
    return cls.detach(), reg.detach(), loss.detach(), grads
