"""Forward/backward runtime of the DINOv3 ViT backbones (SimpleAICV/detection/models/backbones/dinov3vit.py) and of the
DINOv3 SAM image encoder (interactive_segmentation/models/dinov3_segment_anything/dinov3_image_encoder.py: backbone +
the SAM neck) on libsaicv_b200.so.

Tokens are an fp32 residual stream [B*H*W, C] (the patch embedding GEMM writes fp32 tokens; there are no cls, register or
position tokens).  Per SelfAttentionBlock (dinov3vit.py:370-469, drop path 0):
    y   = LN1(x)                                            bf16
    qkv = Linear(y) with bias * bias_mask                   wgmma GEMM                  (:285-300 LinearKMaskedBias)
    q,k <- rope(q, k) in place                              csrc/capi_dinov3.cu         (:271-282, :347-367)
    att = softmax(q k^T / sqrt(hd)) v                       wgmma attention on packed qkv
    x   = x + ls1 * proj(att)                               GEMM (bias, bf16 out) + layer-scale residual kernel
    x   = x + ls2 * fc2(gelu(fc1(LN2(x))))                  (or w3(silu(w1 y) * w2 y), the SwiGLU kernel)
The backward mirrors it: dgamma from the layer-scale residual kernel, the transposed rotation applied to dq / dk in place
(the rotation is linear and attention's backward reads the rotated q / k, so the un-rotated values are never kept).
Then the final LayerNorm and, for the encoder, the SAM neck (engine.sam.Neck) on its bf16 output.

The RoPE table [H*W, hd] is computed once per forward by the reference's torch expression (RopePositionEmbedding.forward,
:196-268) from the ``periods`` buffer; in training with ``rescale_coords`` its log-uniform factor is drawn from torch's
CPU generator exactly like the reference, so a seeded run sees the same coordinates.  The table stays on the tape, so a
checkpointed block's recomputation reuses it.
"""
import math

import numpy as np
import torch

from .. import ops
from .operands import Linear, PatchEmbed, rows_wgrad
from .runtime import Runtime
from .sam import Neck
from .vit import layernorm_bwd


def rope_sincos(rope, H, W, training):
    """(sin, cos) fp32 [H*W, hd] of the RopePositionEmbedding module `rope` (dinov3vit.py:196-268), on its device."""
    if rope.shift_coords is not None or rope.jitter_coords is not None:
        raise NotImplementedError('DINOv3 RoPE shift_coords / jitter_coords are not implemented by the H100 runtime (None in '
                                  'every constructor)')
    device = rope.periods.device
    if rope.normalize_coords == 'max':
        coords_h, coords_w = torch.arange(0.5, H) / max(H, W), torch.arange(0.5, W) / max(H, W)
    elif rope.normalize_coords == 'min':
        coords_h, coords_w = torch.arange(0.5, H) / min(H, W), torch.arange(0.5, W) / min(H, W)
    else:
        coords_h, coords_w = torch.arange(0.5, H) / H, torch.arange(0.5, W) / W
    coords = torch.stack(torch.meshgrid(coords_h.to(device), coords_w.to(device), indexing='ij'), dim=-1).flatten(0, 1)
    coords = 2.0 * coords - 1.0
    if training and rope.rescale_coords is not None:
        if device.type == 'cuda' and torch.cuda.is_current_stream_capturing():
            raise RuntimeError('a CUDA graph cannot capture a DINOv3 training forward with rescale_coords: the CPU draw of '
                               'the rescale factor would be frozen into the graph')
        rescale_max = np.log(rope.rescale_coords)
        coords *= torch.empty(1).uniform_(-rescale_max, rescale_max).exp().to(device)
    angles = (2 * math.pi * coords[:, :, None] / rope.periods[None, None, :]).flatten(1, 2).tile(2)
    return torch.sin(angles).contiguous(), torch.cos(angles).contiguous()


class _MaskedQKV(Linear):
    """LinearKMaskedBias (dinov3vit.py:285-300): the GEMM adds bias * bias_mask, and the bias gradient is masked too.
    bias_mask is a persistent buffer (it may come from a checkpoint), read at every prep()."""

    def prep(self):
        super().prep()
        b = self.mod.bias
        self.b_pad[:b.shape[0]].mul_(self.mod.bias_mask.to(b.dtype))

    def bwd(self, dy, x, sink):
        m = self.mod
        rows_wgrad(dy, x, m.weight, sink)
        full = torch.empty(dy.shape[1], device=dy.device)
        ops.colsum(dy, full)
        sink.add(m.bias, full[:m.bias.shape[0]] * m.bias_mask.to(full.dtype))
        return ops.linear_dgrad(dy, self.op.w)


class _Block:

    def __init__(self, blk):
        self.blk = blk
        qkv = blk.attn.qkv
        self.qkv = _MaskedQKV(qkv) if qkv.bias is not None else Linear(qkv)
        self.proj = Linear(blk.attn.proj)
        mlp = blk.mlp
        self.swiglu = hasattr(mlp, 'w3')
        self.ffn = [Linear(mlp.w1), Linear(mlp.w2), Linear(mlp.w3)] if self.swiglu else [Linear(mlp.fc1), Linear(mlp.fc2)]
        self.heads = blk.attn.head_nums
        self.scale = blk.attn.scale

    def linears(self):
        return [self.qkv, self.proj] + self.ffn

    def forward(self, x, t, b, l, rope):
        """x: fp32 [B*L, C] -> fp32 [B*L, C]"""
        blk, c = self.blk, x.shape[1]
        d = c // self.heads
        t['x_in'] = x
        t['ln1'], t['st1'] = ops.layernorm_fwd(x, blk.norm1.weight.detach(), blk.norm1.bias.detach(), blk.norm1.eps)
        qkv = t['qkv'] = self.qkv.fwd(t['ln1'])
        ops.rope_qk(qkv, rope[0], rope[1], b, l, self.heads, d)
        t['att'] = torch.empty(b * l, c, device=x.device, dtype=torch.bfloat16)
        (out,) = ops.head_views(t['att'], b, l, self.heads, d)
        _, t['lse'] = ops.attn_fwd(*ops.head_views(qkv, b, l, self.heads, d), self.scale, out=out)
        t['pa'] = self.proj.fwd(t['att'])
        x = t['x_mid'] = ops.ls_residual_fwd(x, t['pa'], None, blk.ls1.gamma.detach())
        ln2, t['st2'] = ops.layernorm_fwd(x, blk.norm2.weight.detach(), blk.norm2.bias.detach(), blk.norm2.eps)
        t['ln2'] = ln2
        if self.swiglu:
            w1, w2, w3 = self.ffn
            t['a'], t['g'] = w1.fwd(ln2), w2.fwd(ln2)
            t['h'] = ops.swiglu_fwd(t['a'], t['g'])
            t['f'] = w3.fwd(t['h'])
        else:
            fc1, fc2 = self.ffn
            t['u'] = fc1.fwd(ln2)
            t['h'] = ops.gelu_fwd(t['u'])
            t['f'] = fc2.fwd(t['h'])
        return ops.ls_residual_fwd(x, t['f'], None, blk.ls2.gamma.detach())

    def backward(self, dx, t, b, l, rope, sink, want_bf16=False):
        """dx fp32: gradient w.r.t. the block output.  Returns (dx_in fp32, its bf16 copy or None unless want_bf16)."""
        blk = self.blk
        d = dx.shape[1] // self.heads
        # ---- MLP branch
        ls2 = blk.ls2.gamma
        with sink.grad(ls2) as (acc, buf):
            df = ops.ls_residual_bwd(dx, t['f'], None, ls2.detach(), buf, accumulate=acc)
        if self.swiglu:
            w1, w2, w3 = self.ffn
            dh = w3.bwd(df, t['h'], sink)
            da, dg = ops.swiglu_bwd(dh, t['a'], t['g'])
            dln2 = w2.bwd(dg, t['ln2'], sink, add=w1.bwd(da, t['ln2'], sink))
        else:
            fc1, fc2 = self.ffn
            du = fc2.bwd(df, t['h'], sink, gelu_pre=t['u'])
            dln2 = fc1.bwd(du, t['ln2'], sink)
        dx, _ = layernorm_bwd(blk.norm2, dln2, t['x_mid'], t['st2'], sink, dres=dx, want_bf16=False)
        # ---- attention branch
        ls1 = blk.ls1.gamma
        with sink.grad(ls1) as (acc, buf):
            dpa = ops.ls_residual_bwd(dx, t['pa'], None, ls1.detach(), buf, accumulate=acc)
        datt = self.proj.bwd(dpa, t['att'], sink)
        dqkv = torch.empty_like(t['qkv'])
        q, k, v, out, dout, dq, dk, dv = (view for buf in (t['qkv'], t['att'], datt, dqkv)
                                          for view in ops.head_views(buf, b, l, self.heads, d))
        ops.attn_bwd(q, k, v, out, t['lse'], dout, self.scale, dq, dk, dv)
        ops.rope_qk(dqkv, rope[0], rope[1], b, l, self.heads, d, backward=True)
        dln1 = self.qkv.bwd(dqkv, t['ln1'], sink)
        return layernorm_bwd(blk.norm1, dln1, t['x_in'], t['st1'], sink, dres=dx, want_bf16=want_bf16)


class DINOv3RT(Runtime):
    """Whole-model runtime of a DinoVisionTransformer `backbone` (dinov3vit.py:550-572), followed by the SAM `neck`
    (dinov3_image_encoder.py:67-75) when one is given.  Output: fp32 NCHW (the final LayerNorm's bf16 output widened when
    there is no neck)."""

    def __init__(self, backbone, neck=None, neck_checkpoint=False):
        self.backbone = backbone
        self.blocks = [_Block(b) for b in backbone.blocks]
        self.patch = PatchEmbed(backbone.patch_embed.proj)
        self.neck = Neck(neck) if neck is not None else None
        self.neck_checkpoint = neck_checkpoint
        super().__init__([lin for b in self.blocks for lin in b.linears()] + [self.patch])

    def operands(self):
        return super().operands() + (self.neck.operands() if self.neck is not None else [])

    def prep(self):
        super().prep()
        if self.neck is not None:
            self.neck.prep()

    # ---- stages (also driven separately by the teacher-forced parity tests)
    def embed_forward(self, x, training, tape):
        """x: fp32 NCHW image -> fp32 tokens [B*H*W, C]; draws the RoPE table (and, in training, its rescale factor)."""
        ps = self.patch.p
        tok, tape['cols'] = self.patch.fwd(x)
        B, H, W = x.shape[0], x.shape[2] // ps, x.shape[3] // ps
        tape['B'], tape['H'], tape['W'] = B, H, W
        tape['rope'] = rope_sincos(self.backbone.rope_embed, H, W, training)
        return tok

    def head_forward(self, x, tape):
        """x fp32 [B*H*W, C] -> final LayerNorm (-> neck) -> fp32 NCHW."""
        norm = self.backbone.norm
        B, H, W = tape['B'], tape['H'], tape['W']
        tape['x_last'] = x
        y, tape['stn'] = ops.layernorm_fwd(x, norm.weight.detach(), norm.bias.detach(), norm.eps)
        if self.neck is None:
            return y.view(B, H, W, -1).permute(0, 3, 1, 2).float()
        if self.neck_checkpoint:    # dinov3_image_encoder.py:70-71: keep the neck input, recompute in backward
            tape['neck_in'] = y
            return self.neck.forward(y, B, H, W, {})
        tape['neck'] = {}
        return self.neck.forward(y, B, H, W, tape['neck'])

    def head_backward(self, dout, tape):
        """dout fp32 NCHW -> gradient w.r.t. the last block's output (fp32 [B*H*W, C])."""
        sink = self.sink
        B, H, W = tape['B'], tape['H'], tape['W']
        if self.neck is None:
            dy = dout.permute(0, 2, 3, 1).reshape(B * H * W, -1).to(torch.bfloat16).contiguous()
        else:
            if 'neck_in' in tape:
                tape['neck'] = {}
                self.neck.forward(tape.pop('neck_in'), B, H, W, tape['neck'])
            dy = self.neck.backward(dout, tape.pop('neck'), sink, out_f32=False)
        dx, _ = layernorm_bwd(self.backbone.norm, dy, tape['x_last'], tape['stn'], sink, want_bf16=False)
        return dx

    def forward(self, x, training, keep_tape):
        assert x.is_cuda and x.dtype == torch.float32 and x.dim() == 4
        self.prep()
        tape = {'blocks': [dict() for _ in self.blocks]}
        h = self.embed_forward(x.contiguous(), training, tape)
        B, L, rope = tape['B'], tape['H'] * tape['W'], tape['rope']
        ckpt = keep_tape and getattr(self.backbone, 'use_gradient_checkpoint', False)
        for blk, t in zip(self.blocks, tape['blocks']):
            if ckpt:   # dinov3vit.py:561-562: keep the block input, recompute in backward
                t['ckpt_in'] = h
                h = blk.forward(h, {}, B, L, rope)
            else:   # without a tape each block's intermediates are freed as soon as the next block starts
                h = blk.forward(h, t if keep_tape else {}, B, L, rope)
        out = self.head_forward(h, tape)
        return out, (tape if keep_tape else None)

    def backward(self, dout, tape):
        assert tape is not None, 'backward called without a training forward'
        B, L, rope = tape['B'], tape['H'] * tape['W'], tape['rope']
        dx = self.head_backward(dout.contiguous().float(), tape)
        dxb = None
        for i in range(len(self.blocks) - 1, -1, -1):
            t = tape['blocks'][i]
            if 'ckpt_in' in t:
                self.blocks[i].forward(t.pop('ckpt_in'), t, B, L, rope)
            dx, dxb = self.blocks[i].backward(dx, t, B, L, rope, self.sink, want_bf16=(i == 0))
            t.clear()
        self.patch.bwd(dxb, tape['cols'], self.sink)
