"""Forward/backward runtime of the SAM ViT image encoder
(SimpleAICV/interactive_segmentation/models/segment_anything/image_encoder.py) on libsaicv_b200.so.

Tokens are an fp32 residual stream [B*H*W, C] (patch embedding bf16 + fp32 pos_embed promotes to fp32, like the
reference under autocast).  Per Block (image_encoder.py:201-239):
    y   = LN1(x)                                   bf16
    [window partition with zero padding]           csrc/capi_sam.cu            (:32-55)
    qkv = Linear(y)                                wgmma GEMM
    att = softmax(q k^T scale + rel_h + rel_w) v   wgmma attention; the decomposed rel-pos bias (:82-144) rides in
                                                   extra score columns built by ops.relpos_build (one GEMM + gather)
    [window unpartition]                                                       (:58-79)
    x   = x + proj(att);  x = x + lin2(gelu(lin1(LN2(x))))                     GEMM epilogues fuse bias/residual/dGELU
Neck (:299-311): 1x1 conv -> LayerNorm2d -> 3x3 conv -> LayerNorm2d (LayerNorm over channels = the row LayerNorm
kernel on NHWC rows); the 3x3 conv is the TMA-im2col implicit GEMM.
"""
import torch

from .. import ops
from .convnet import GradSink
from .vit import _Linear


def _ln_bwd(norm, dy, x, stats, dres, sink, want_bf16=True):
    gbuf, gacc = sink.begin(norm.weight)
    bbuf, bacc = sink.begin(norm.bias)
    dxb = torch.empty(x.shape, device=x.device, dtype=torch.bfloat16) if want_bf16 else None
    dx = ops.layernorm_bwd(dy, x, norm.weight.detach(), stats, gbuf, bbuf, dres=dres, dx_bf16=dxb, accumulate=gacc)
    sink.done(norm.weight, gbuf)
    sink.done(norm.bias, bbuf)
    return dx, dxb


class _Block:

    def __init__(self, blk):
        self.blk = blk
        self.ws = blk.window_size
        self.qkv, self.proj = _Linear(blk.attn.qkv), _Linear(blk.attn.proj)
        self.lin1, self.lin2 = _Linear(blk.mlp.lin1), _Linear(blk.mlp.lin2)
        self.heads = blk.attn.head_nums
        self.scale = blk.attn.scale

    def linears(self):
        return [self.qkv, self.proj, self.lin1, self.lin2]

    def forward(self, x, t, B, H, W):
        """x: fp32 [B*H*W, C] -> fp32 [B*H*W, C]"""
        blk, C = self.blk, x.shape[1]
        hd = C // self.heads
        t['x_in'] = x
        ln1, t['st1'] = ops.layernorm_fwd(x, blk.norm1.weight.detach(), blk.norm1.bias.detach(), blk.norm1.eps)
        if self.ws > 0:
            xw, (nwy, nwx) = ops.window_partition(ln1.view(B, H, W, C), self.ws)
            Bw, Sh, Sw = B * nwy * nwx, self.ws, self.ws
            xw = xw.view(-1, C)
        else:
            xw, Bw, Sh, Sw = ln1, B, H, W
        L = Sh * Sw
        t['xw'], t['geom'] = xw, (Bw, Sh, Sw)
        qkv = t['qkv'] = self.qkv.fwd(xw)                                           # [Bw*L, 3C] = [Bw][L][3][heads][hd]
        rph, rpw = blk.attn.rel_pos_h.detach(), blk.attn.rel_pos_w.detach()
        assert rph.shape[0] == 2 * Sh - 1 and rpw.shape[0] == 2 * Sw - 1, 'rel-pos interpolation is not implemented'
        t['rp_aux'] = {}
        qe, ke = ops.relpos_build(qkv, rph, rpw, Bw, self.heads, hd, Sh, Sw, self.scale, aux=t['rp_aux'])
        v = qkv.view(Bw, L, 3, self.heads, hd)[:, :, 2].permute(0, 2, 1, 3)         # strided view, no copy
        att = torch.empty(Bw * L, C, device=x.device, dtype=torch.bfloat16)
        out_view = att.view(Bw, L, self.heads, hd).permute(0, 2, 1, 3)
        _, lse = ops.attn_fwd(qe, ke, v, 1.0, out=out_view)
        t['qe'], t['ke'], t['att'], t['lse'] = qe, ke, att, lse
        if self.ws > 0:
            att_full = ops.window_unpartition(att.view(Bw, L, C), B, H, W, self.ws).view(-1, C)
        else:
            att_full = att
        t['att_full'] = att_full
        x = self.proj.fwd(att_full, resid=x, out_f32=True)
        t['x_mid'] = x
        t['ln2'], t['st2'] = ops.layernorm_fwd(x, blk.norm2.weight.detach(), blk.norm2.bias.detach(), blk.norm2.eps)
        t['u'] = self.lin1.fwd(t['ln2'])
        t['h'] = ops.gelu_fwd(t['u'])
        return self.lin2.fwd(t['h'], resid=x, out_f32=True)

    def backward(self, dx, dxb, t, B, H, W, sink):
        """dx fp32 / dxb bf16: gradient w.r.t. the block output.  Returns (dx_in fp32, its bf16 copy)."""
        blk, C = self.blk, dx.shape[1]
        hd = C // self.heads
        Bw, Sh, Sw = t['geom']
        L = Sh * Sw
        # ---- MLP branch
        du = self.lin2.bwd(dxb, t['h'], sink, gelu_pre=t['u'])
        dln2 = self.lin1.bwd(du, t['ln2'], sink)
        dx, dxb = _ln_bwd(blk.norm2, dln2, t['x_mid'], t['st2'], dx, sink)
        # ---- attention branch
        datt_full = self.proj.bwd(dxb, t['att_full'], sink)
        if self.ws > 0:
            datt, _ = ops.window_partition(datt_full.view(B, H, W, C), self.ws)   # padding tokens get zero gradient
            datt = datt.view(-1, C)
        else:
            datt = datt_full
        qkv = t['qkv']
        q5 = qkv.view(Bw, L, 3, self.heads, hd)
        dqkv = torch.empty_like(qkv)
        d5 = dqkv.view(Bw, L, 3, self.heads, hd)
        dqe = torch.empty_like(t['qe'])
        ops.attn_bwd(t['qe'], t['ke'], q5[:, :, 2].permute(0, 2, 1, 3), t['att'].view(Bw, L, self.heads, hd).permute(0, 2, 1, 3),
                     t['lse'], datt.view(Bw, L, self.heads, hd).permute(0, 2, 1, 3), 1.0, dqe,
                     d5[:, :, 1].permute(0, 2, 1, 3), d5[:, :, 2].permute(0, 2, 1, 3), dk_cols=hd)
        rph, rpw = blk.attn.rel_pos_h, blk.attn.rel_pos_w
        hbuf, hacc = sink.begin(rph)
        wbuf, wacc = sink.begin(rpw)
        assert hacc == wacc
        ops.relpos_bwd(dqe, qkv, rph.detach(), rpw.detach(), dqkv, hbuf, wbuf, Bw, self.heads, hd, Sh, Sw, self.scale, accumulate=hacc,
                       aux=t.get('rp_aux'))
        sink.done(rph, hbuf)
        sink.done(rpw, wbuf)
        dxw = self.qkv.bwd(dqkv, t['xw'], sink)
        if self.ws > 0:
            dln1 = ops.window_unpartition(dxw.view(Bw, L, C), B, H, W, self.ws).view(-1, C)
        else:
            dln1 = dxw
        return _ln_bwd(blk.norm1, dln1, t['x_in'], t['st1'], dx, sink)


class SamEncoderRT:
    """Whole-encoder runtime (image_encoder.py:313-331)."""

    def __init__(self, model):
        self.model = model
        self.blocks = [_Block(b) for b in model.blocks]
        self.sink = GradSink()
        self.pw_bf16 = self.n0_bf16 = self.n2_bf16 = None
        self.versions = {}

    def prep(self):
        m = self.model
        for b in self.blocks:
            for lin in b.linears():
                lin.prep()
        w = m.patch_embed.proj.weight
        if self._changed('pw', w):
            k = w.shape[1] * w.shape[2] * w.shape[3]
            self.kpad = ops.stem_kpad(w.shape[1], w.shape[2], w.shape[3])
            if self.pw_bf16 is None:
                self.pw_bf16 = torch.empty(w.shape[0], self.kpad, device=w.device, dtype=torch.bfloat16)
            ops.prep_conv_weight(w.detach(), self.pw_bf16, self.kpad, order=ops.ORDER_CRS)
        w0 = m.neck[0].weight
        if self._changed('n0', w0):
            self.n0_bf16 = ops.cast_bf16(w0.detach().view(w0.shape[0], w0.shape[1]), self.n0_bf16)
        w2 = m.neck[2].weight
        if self._changed('n2', w2):
            if self.n2_bf16 is None:
                self.n2_bf16 = torch.empty(w2.shape[0], 9 * w2.shape[1], device=w2.device, dtype=torch.bfloat16)
            ops.prep_conv_weight(w2.detach(), self.n2_bf16, 9 * w2.shape[1], order=ops.ORDER_RSC)

    def _changed(self, key, w):
        ver = (w.data_ptr(), w._version)
        if self.versions.get(key) != ver:
            self.versions[key] = ver
            return True
        return False

    # ---- stages (also driven separately by the teacher-forced parity tests)
    def embed_forward(self, x, tape):
        m = self.model
        B = x.shape[0]
        ps = m.patch_embed.proj.kernel_size[0]
        cols = ops.stem_im2col(x, ps, ps, ps, 0, self.kpad)
        tape['cols'] = cols
        tok = ops.linear_fwd(cols, self.pw_bf16, bias=m.patch_embed.proj.bias.detach(), out_f32=True)
        H, W = x.shape[2] // ps, x.shape[3] // ps
        tape['B'], tape['H'], tape['W'] = B, H, W
        ops.add_pos_embed(tok, m.pos_embed.detach())
        return tok

    def embed_backward(self, dx, dxb, tape):
        m, sink = self.model, self.sink
        pbuf, pacc = sink.begin(m.pos_embed)
        ops.colsum(dx.view(tape['B'], -1), pbuf.view(-1), accumulate=pacc)        # sum over the batch
        sink.done(m.pos_embed, pbuf)
        w, bias = m.patch_embed.proj.weight, m.patch_embed.proj.bias
        wbuf, wacc = sink.begin(w)
        part = ops.linear_wgrad(dxb, tape['cols'])
        ops.finish_conv_wgrad(part, wbuf, self.kpad, accumulate=wacc, order=ops.ORDER_CRS)
        sink.done(w, wbuf)
        bbuf, bacc = sink.begin(bias)
        ops.colsum(dxb, bbuf, accumulate=bacc)
        sink.done(bias, bbuf)

    def neck_forward(self, x, tape):
        """x fp32 [B*H*W, C] -> fp32 NCHW [B, out_planes, H, W]"""
        m = self.model
        B, H, W = tape['B'], tape['H'], tape['W']
        n1, n3 = m.neck[1], m.neck[3]
        xb = tape['xb'] = ops.cast_bf16(x)
        y1 = tape['y1'] = ops.linear_fwd(xb, self.n0_bf16, out_f32=True)                     # 1x1 conv, no bias
        oc = y1.shape[1]
        l1, tape['s1'] = ops.layernorm_fwd(y1, n1.weight.detach(), n1.bias.detach(), n1.eps)
        tape['l1'] = l1
        cs = tape['cs'] = ops.make_conv_shape(B, H, W, oc, oc, 3, 3, 1, 1)
        y2b = ops.conv_fprop(l1.view(B, H, W, oc), self.n2_bf16, cs)
        y2 = tape['y2'] = y2b.view(-1, oc).float()
        l2, tape['s2'] = ops.layernorm_fwd(y2, n3.weight.detach(), n3.bias.detach(), n3.eps)
        return l2.view(B, H, W, oc).permute(0, 3, 1, 2).float()

    def neck_backward(self, dout, tape):
        """dout fp32 NCHW -> (dx fp32 [B*H*W, C], its bf16 copy)"""
        m, sink = self.model, self.sink
        B, H, W = tape['B'], tape['H'], tape['W']
        n1, n3 = m.neck[1], m.neck[3]
        oc = dout.shape[1]
        dl2 = dout.permute(0, 2, 3, 1).reshape(-1, oc).to(torch.bfloat16).contiguous()
        _, dy2b = _ln_bwd(n3, dl2, tape['y2'], tape['s2'], None, sink)
        w2 = m.neck[2].weight
        wbuf, wacc = sink.begin(w2)
        part = ops.conv_wgrad(dy2b.view(B, H, W, oc), tape['l1'].view(B, H, W, oc), tape['cs'])
        ops.finish_conv_wgrad(part, wbuf, 9 * oc, accumulate=wacc)
        sink.done(w2, wbuf)
        dl1 = ops.conv_dgrad(dy2b.view(B, H, W, oc), self.n2_bf16, tape['cs']).view(-1, oc)
        _, dy1b = _ln_bwd(n1, dl1, tape['y1'], tape['s1'], None, sink)
        w0 = m.neck[0].weight
        wbuf, wacc = sink.begin(w0)
        ops.reduce_partials(ops.linear_wgrad(dy1b, tape['xb']), wbuf, accumulate=wacc)
        sink.done(w0, wbuf)
        dx = ops.linear_dgrad(dy1b, self.n0_bf16, out_f32=True)
        return dx, ops.cast_bf16(dx)

    def forward(self, x, training, keep_tape):
        assert x.is_cuda and x.dtype == torch.float32 and x.dim() == 4
        self.prep()
        tape = {'blocks': [dict() for _ in self.blocks]}
        h = self.embed_forward(x.contiguous(), tape)
        ckpt = keep_tape and getattr(self.model, 'use_gradient_checkpoint', False)
        for blk, t in zip(self.blocks, tape['blocks']):
            if ckpt:
                t['ckpt_in'] = h
                h = blk.forward(h, {}, tape['B'], tape['H'], tape['W'])
            else:
                h = blk.forward(h, t, tape['B'], tape['H'], tape['W'])
        out = self.neck_forward(h, tape)
        return out, (tape if keep_tape else None)

    def backward(self, dout, tape):
        assert tape is not None, 'backward called without a training forward'
        dx, dxb = self.neck_backward(dout.contiguous().float(), tape)
        B, H, W = tape['B'], tape['H'], tape['W']
        for i in range(len(self.blocks) - 1, -1, -1):
            t = tape['blocks'][i]
            if 'ckpt_in' in t:   # use_gradient_checkpoint (image_encoder.py:318-329): replay the block forward
                self.blocks[i].forward(t.pop('ckpt_in'), t, B, H, W)
            dx, dxb = self.blocks[i].backward(dx, dxb, t, B, H, W, self.sink)
            t.clear()
        self.embed_backward(dx, dxb, tape)
        if self.sink.on_backward_end is not None:
            self.sink.on_backward_end()
