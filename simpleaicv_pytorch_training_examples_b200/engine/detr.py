"""Forward/backward runtime of DETR on libsaicv_b200.so.

Reference: SimpleAICV/detection/models/detr.py:44-90 (encoder layer), :93-180 (decoder layer), :183-270
(DETRTransformer), :273-364 (DETR), backbones/detr_resnet.py:256-340 (backbone), head.py:184-213 (heads).

Data flow (tokens batch-major, M = B*L image tokens, Mq = B*Q query tokens, C = 256):
  * the ResNet body runs on engine.convnet's conv/BN units and hands over C5 as NHWC bf16;
  * proj_conv is one GEMM with the bias fused and an fp32 output: the token stream `src` [M, C];
  * every layer is post-LN: z = stream + branch is produced by the branch's last GEMM (fp32 residual fused in the
    epilogue), then ONE saicv_postln_fwd pass writes the new fp32 stream and the bf16 operand copies the next GEMMs need
    (y and y + positional embedding);
  * attention runs on the wgmma attention kernels with head size 32.  The reference passes a FLOAT key_padding_mask
    (detr.py:333-346), which nn.MultiheadAttention adds to the logits; that bias rides in one extra column of the score
    operands (q operand: constant 1, k operand: the bias), so the kernel is the same one SAM's rel-pos bias uses;
  * gradients of a stream tensor that feeds several GEMMs are summed by chaining the fp32 `resid` operand of the
    data-gradient GEMMs, never by a separate add pass; LayerNorm / bias / weight gradients go through the GradSink.
Dropout (residual, feed-forward and attention-probability dropout, p = dropout_prob) uses the counter-hash masks of
csrc/dropout_hash.cuh: the backward recomputes the forward's masks from the per-site seeds kept on the tape.
"""
import torch

from .. import ops
from .convnet import GradSink, ResNetRT, blocks_backward
from .operands import Linear, Operand


class _NoHead:
    """The DETR backbone has no classifier: DetrRT drives the body's stem and blocks itself."""


def _pad_cols_bf16(t, n):
    """fp32 [M, k] -> bf16 [M, n] zero-padded (operand layout of the class-padded head GEMMs)."""
    out = torch.zeros(t.shape[0], n, device=t.device, dtype=torch.bfloat16)
    out[:, :t.shape[1]] = t
    return out


class _MHA:
    """One nn.MultiheadAttention: packed in_proj (q | k | v rows of in_proj_weight) + out_proj."""

    def __init__(self, mod):
        self.mod = mod
        self.C, self.H = mod.embed_dim, mod.num_heads
        self.hd = self.C // self.H
        self.out = Linear(mod.out_proj)
        self.op = Operand(mod.in_proj_weight)

    def prep(self):
        self.op.refresh()

    def _proj(self, x, r0, r1):
        return ops.linear_fwd(x, self.op.w[r0:r1], bias=self.mod.in_proj_bias.detach()[r0:r1])

    def forward(self, q_in, k_in, v_in, t, B, Lq, Lk, key_bias, p, seed, sb=None):
        """q_in [B*Lq, C], k_in / v_in [B*Lk, C] bf16 operand copies (q_in is k_in for self-attention).
        Returns the attention output [B*Lq, C] bf16 (before out_proj)."""
        C, H, hd = self.C, self.H, self.hd
        t['q_in'], t['k_in'], t['v_in'] = q_in, k_in, v_in
        if q_in is k_in:
            qk = self._proj(q_in, 0, 2 * C)
            qsrc, q0, ksrc, k0 = qk, 0, qk, C
        else:
            qsrc, q0, ksrc, k0 = self._proj(q_in, 0, C), 0, self._proj(k_in, C, 2 * C), 0
        v = self._proj(v_in, 2 * C, 3 * C)
        scale = hd ** -0.5
        if key_bias is not None:
            dp = hd + 16
            qe = ops.heads_pack(qsrc, q0, B, Lq, H, hd, dp, scale=scale, extra_const=1.0)
            ke = ops.heads_pack(ksrc, k0, B, Lk, H, hd, dp, extra=key_bias)
            kscale = 1.0
        else:
            qe = qsrc.view(B, Lq, -1)[:, :, q0:q0 + C].unflatten(2, (H, hd)).permute(0, 2, 1, 3)
            ke = ksrc.view(B, Lk, -1)[:, :, k0:k0 + C].unflatten(2, (H, hd)).permute(0, 2, 1, 3)
            kscale = scale
        vv = v.view(B, Lk, H, hd).permute(0, 2, 1, 3)
        att = torch.empty(B * Lq, C, device=v.device, dtype=torch.bfloat16)
        ov = att.view(B, Lq, H, hd).permute(0, 2, 1, 3)
        _, lse = ops.attn_fwd(qe, ke, vv, kscale, out=ov, dropout_p=p, dropout_seed=seed, dropout_seed_base=sb)
        t.update(qe=qe, ke=ke, vv=vv, ov=ov, lse=lse, kscale=kscale, biased=key_bias is not None, p=p, seed=seed, sb=sb,
                 dims=(B, Lq, Lk))
        t['att'] = att
        return att

    def backward(self, datt, t, sink):
        """datt [B*Lq, C] bf16.  Accumulates the in_proj parameter gradients and returns the bf16 gradients of the
        projected (dq, dk, dv) as (tensor [rows, n], ...) ready for the data-gradient GEMMs: self-attention returns
        (dqk [B*L, 2C], None, dv), cross-attention (dq, dk, dv)."""
        C, H, hd = self.C, self.H, self.hd
        B, Lq, Lk = t['dims']
        dev = datt.device
        dov = datt.view(B, Lq, H, hd).permute(0, 2, 1, 3)
        dv = torch.empty(B * Lk, C, device=dev, dtype=torch.bfloat16)
        dvv = dv.view(B, Lk, H, hd).permute(0, 2, 1, 3)
        same = t['q_in'] is t['k_in']
        if same:
            dqk = torch.empty(B * Lq, 2 * C, device=dev, dtype=torch.bfloat16)
            dq_dst, dq0, dk_dst, dk0 = dqk, 0, dqk, C
        else:
            dq_dst, dq0 = torch.empty(B * Lq, C, device=dev, dtype=torch.bfloat16), 0
            dk_dst, dk0 = torch.empty(B * Lk, C, device=dev, dtype=torch.bfloat16), 0
        if t['biased']:
            dqe, dke = torch.empty_like(t['qe']), torch.empty_like(t['ke'])
            ops.attn_bwd(t['qe'], t['ke'], t['vv'], t['ov'], t['lse'], dov, t['kscale'], dqe, dke, dvv, dk_cols=hd,
                         dropout_p=t['p'], dropout_seed=t['seed'], dropout_seed_base=t['sb'])
            ops.heads_unpack(dqe, dq_dst, dq0, hd, scale=hd ** -0.5)
            ops.heads_unpack(dke, dk_dst, dk0, hd)
        else:
            dqv = dq_dst.view(B, Lq, -1)[:, :, dq0:dq0 + C].unflatten(2, (H, hd)).permute(0, 2, 1, 3)
            dkv = dk_dst.view(B, Lk, -1)[:, :, dk0:dk0 + C].unflatten(2, (H, hd)).permute(0, 2, 1, 3)
            ops.attn_bwd(t['qe'], t['ke'], t['vv'], t['ov'], t['lse'], dov, t['kscale'], dqv, dkv, dvv,
                         dropout_p=t['p'], dropout_seed=t['seed'], dropout_seed_base=t['sb'])
        w, b = self.mod.in_proj_weight, self.mod.in_proj_bias
        wbuf, wacc = sink.begin(w)
        bbuf, bacc = sink.begin(b)
        pieces = [(dq_dst, t['q_in'], 0, 2 * C)] if same else [(dq_dst, t['q_in'], 0, C), (dk_dst, t['k_in'], C, 2 * C)]
        pieces.append((dv, t['v_in'], 2 * C, 3 * C))
        for dy, x, r0, r1 in pieces:
            ops.reduce_partials(ops.linear_wgrad(dy, x), wbuf[r0:r1], accumulate=wacc)
            ops.colsum(dy, bbuf[r0:r1], accumulate=bacc)
        sink.done(w, wbuf)
        sink.done(b, bbuf)
        return (dq_dst, None, dv) if same else (dq_dst, dk_dst, dv)

    def dgrad(self, dy, r0, r1, resid=None):
        """fp32 data gradient of the projection rows r0:r1 (+ resid)."""
        return ops.linear_dgrad(dy, self.op.w[r0:r1], resid=resid, out_f32=True)


def _branch_out(lin, a, resid, p, seed, sb):
    """z = resid + dropout(lin(a)): the residual rides in the GEMM epilogue when there is no dropout."""
    if p == 0.:
        return lin.fwd(a, resid=resid, out_f32=True)
    return ops.dropout(lin.fwd(a), p, seed, resid=resid, seed_base=sb)


def _branch_grad(dz, dzb, p, seed, sb):
    """bf16 gradient of the branch output from the gradient of z = resid + dropout(branch)."""
    return dzb if p == 0. else ops.dropout(dz, p, seed, out_f32=False, seed_base=sb)


class _FFN:
    def __init__(self, layer):
        self.l1, self.l2 = Linear(layer.linear1), Linear(layer.linear2)

    def forward(self, yb, y, t, p, seeds, sb):
        """z = y + dropout(linear2(dropout(relu(linear1(yb)))))"""
        h = self.l1.fwd_flags(yb, ops.EPI_RELU)
        if p > 0.:
            ops.dropout(h, p, seeds[0], out=h, seed_base=sb)
        t['ffn_in'], t['h'] = yb, h
        return _branch_out(self.l2, h, y, p, seeds[1], sb)

    def backward(self, dz, dzb, t, sink, p, seeds, sb):
        """Returns the fp32 gradient of y: dz (residual path) + the feed-forward path."""
        g = _branch_grad(dz, dzb, p, seeds[1], sb)
        dh = self.l2.bwd(g, t['h'], sink, relu_out=t['h'])          # zero where relu(.) = 0 or the unit was dropped
        if p > 0.:
            ops.dropout(dh, p, seeds[0], out=dh, seed_base=sb)     # survivors' 1 / (1 - p)
        self.l1.bwd(dh, t['ffn_in'], sink, need_dx=False)
        return ops.linear_dgrad(dh, self.l1.op.w, resid=dz, out_f32=True)


def _norm_fwd(norm, z, pos=None, want_y=True, want_yb=True, want_ypb=False):
    return ops.postln_fwd(z, norm.weight.detach(), norm.bias.detach(), norm.eps, pos=pos, want_y=want_y, want_yb=want_yb,
                          want_ypb=want_ypb)


def _norm_bwd(norm, dy, z, stats, sink, dres=None, want_dz=True, want_dzb=True):
    gbuf, gacc = sink.begin(norm.weight)
    bbuf, bacc = sink.begin(norm.bias)
    dz, dzb = ops.postln_bwd(dy, z, norm.weight.detach(), stats, gbuf, bbuf, dres=dres, want_dz=want_dz, want_dzb=want_dzb,
                             accumulate=gacc)
    sink.done(norm.weight, gbuf)
    sink.done(norm.bias, bbuf)
    return dz, dzb


class _EncLayer:
    def __init__(self, layer):
        self.layer = layer
        self.attn = _MHA(layer.attention)
        self.ffn = _FFN(layer)

    def units(self):
        return [self.attn, self.attn.out, self.ffn.l1, self.ffn.l2]

    def forward(self, x, xb, xpb, t, cx, want_pos_copy):
        """x fp32 stream, xb = bf16(x), xpb = bf16(x + pos).  Returns the same triple for the next layer."""
        p, s, sb = cx['p'], cx['seed'](), cx['sb']
        t['seeds'] = s
        att = self.attn.forward(xpb, xpb, xb, t.setdefault('mha', {}), cx['B'], cx['L'], cx['L'], cx['key_bias'], p, s[0], sb)
        t['z1'] = z1 = _branch_out(self.attn.out, att, x, p, s[1], sb)
        y1, y1b, _, t['st1'] = _norm_fwd(self.layer.norm1, z1)
        t['z2'] = z2 = self.ffn.forward(y1b, y1, t, p, s[2:4], sb)
        y2, y2b, y2pb, t['st2'] = _norm_fwd(self.layer.norm2, z2, pos=cx['pos'], want_ypb=want_pos_copy)
        return y2, y2b, y2pb

    def backward(self, dy2, t, sink, cx):
        """dy2 fp32: gradient of the layer output.  Returns the fp32 gradient of the layer input."""
        p, s, C, sb = cx['p'], t['seeds'], self.attn.C, cx['sb']
        dz2, dz2b = _norm_bwd(self.layer.norm2, dy2, t['z2'], t['st2'], sink, want_dzb=(p == 0.))
        dy1 = self.ffn.backward(dz2, dz2b, t, sink, p, s[2:4], sb)
        dz1, dz1b = _norm_bwd(self.layer.norm1, dy1, t['z1'], t['st1'], sink, want_dzb=(p == 0.))
        datt = self.attn.out.bwd(_branch_grad(dz1, dz1b, p, s[1], sb), t['mha']['att'], sink)
        dqk, _, dv = self.attn.backward(datt, t['mha'], sink)
        dx = self.attn.dgrad(dv, 2 * C, 3 * C, resid=dz1)
        return self.attn.dgrad(dqk, 0, 2 * C, resid=dx)


class _DecLayer:
    def __init__(self, layer):
        self.layer = layer
        self.sa = _MHA(layer.attention)
        self.ca = _MHA(layer.multihead_attention)
        self.ffn = _FFN(layer)

    def units(self):
        return [self.sa, self.sa.out, self.ca, self.ca.out, self.ffn.l1, self.ffn.l2]

    def forward(self, x, xb, xqb, memb, mempb, t, cx):
        """x fp32 [B*Q, C] (tgt), xb = bf16(x), xqb = bf16(x + query_pos); memb / mempb: bf16 copies of the encoder
        memory and memory + pos.  Returns (y3, y3b, y3qb)."""
        p, s, sb = cx['p'], cx['seed'](), cx['sb']
        t['seeds'] = s
        B, Q, L = cx['B'], cx['Q'], cx['L']
        att = self.sa.forward(xqb, xqb, xb, t.setdefault('sa', {}), B, Q, Q, None, p, s[0], sb)
        t['z1'] = z1 = _branch_out(self.sa.out, att, x, p, s[1], sb)
        y1, _, y1qb, t['st1'] = _norm_fwd(self.layer.norm1, z1, pos=cx['qpos'], want_yb=False, want_ypb=True)
        att = self.ca.forward(y1qb, mempb, memb, t.setdefault('ca', {}), B, Q, L, cx['key_bias'], p, s[2], sb)
        t['z2'] = z2 = _branch_out(self.ca.out, att, y1, p, s[3], sb)
        y2, y2b, _, t['st2'] = _norm_fwd(self.layer.norm2, z2)
        t['z3'] = z3 = self.ffn.forward(y2b, y2, t, p, s[4:6], sb)
        y3, y3b, y3qb, t['st3'] = _norm_fwd(self.layer.norm3, z3, pos=cx['qpos'], want_ypb=True)
        return y3, y3b, y3qb

    def backward(self, dy3, t, sink, cx, dmem, dqpos, need_dx):
        """dy3 fp32: gradient of the layer output.  dmem / dqpos: running fp32 sums of the gradients of the encoder
        memory [B*L, C] and of the broadcast query positions [B*Q, C] (None before the first contribution).  Returns
        (dx fp32 | None, dmem, dqpos)."""
        p, s, C, sb = cx['p'], t['seeds'], self.sa.C, cx['sb']
        dz3, dz3b = _norm_bwd(self.layer.norm3, dy3, t['z3'], t['st3'], sink, want_dzb=(p == 0.))
        dy2 = self.ffn.backward(dz3, dz3b, t, sink, p, s[4:6], sb)
        dz2, dz2b = _norm_bwd(self.layer.norm2, dy2, t['z2'], t['st2'], sink, want_dzb=(p == 0.))
        datt = self.ca.out.bwd(_branch_grad(dz2, dz2b, p, s[3], sb), t['ca']['att'], sink)
        dq, dk, dv = self.ca.backward(datt, t['ca'], sink)
        dmem = self.ca.dgrad(dk, C, 2 * C, resid=dmem)               # keys see memory + pos, values memory
        dmem = self.ca.dgrad(dv, 2 * C, 3 * C, resid=dmem)
        gq = self.ca.dgrad(dq, 0, C, resid=dqpos)                    # the query operand was y1 + query_pos:
        dqpos_new = gq                                               #   its gradient joins the query-pos sum ...
        dy1 = self.ca.dgrad(dq, 0, C, resid=dz2)                     #   ... and, with the residual path, y1
        dz1, dz1b = _norm_bwd(self.layer.norm1, dy1, t['z1'], t['st1'], sink, want_dzb=(p == 0.))
        datt = self.sa.out.bwd(_branch_grad(dz1, dz1b, p, s[1], sb), t['sa']['att'], sink)
        dqk, _, dv = self.sa.backward(datt, t['sa'], sink)
        dqpos_new = self.sa.dgrad(dqk, 0, 2 * C, resid=dqpos_new)    # q = k = x + query_pos
        dx = None
        if need_dx:
            dx = self.sa.dgrad(dv, 2 * C, 3 * C, resid=dz1)
            dx = self.sa.dgrad(dqk, 0, 2 * C, resid=dx)
        return dx, dmem, dqpos_new


class _Heads:
    """DETRClsRegHead (head.py:184-213): class logits and the 3-layer box MLP on all decoder outputs at once."""

    def __init__(self, head):
        self.cls = Linear(head.cls_head)
        self.r0, self.r2, self.r4 = Linear(head.reg_head[0]), Linear(head.reg_head[2]), Linear(head.reg_head[4])
        self.ncls = head.cls_head.weight.shape[0]

    def units(self):
        return [self.cls, self.r0, self.r2, self.r4]

    def forward(self, hsb, t):
        t['hsb'] = hsb
        cls = self.cls.fwd(hsb, out_f32=True)[:, :self.ncls]
        t['r1'] = r1 = self.r0.fwd_flags(hsb, ops.EPI_RELU)
        t['r2'] = r2 = self.r2.fwd_flags(r1, ops.EPI_RELU)
        return cls, self.r4.fwd(r2, out_f32=True)[:, :4]

    def backward(self, dcls, dreg, t, sink):
        """fp32 gradients of the class logits [rows, ncls] and box logits [rows, 4] -> fp32 gradient of hs."""
        dcb = _pad_cols_bf16(dcls, self.cls.op.w.shape[0])
        drb = _pad_cols_bf16(dreg, self.r4.op.w.shape[0])
        dr2 = self.r4.bwd(drb, t['r2'], sink, relu_out=t['r2'])
        dr1 = self.r2.bwd(dr2, t['r1'], sink, relu_out=t['r1'])
        self.r0.bwd(dr1, t['hsb'], sink, need_dx=False)
        self.cls.bwd(dcb, t['hsb'], sink, need_dx=False)
        dhs = ops.linear_dgrad(dr1, self.r0.op.w, out_f32=True)
        return ops.linear_dgrad(dcb, self.cls.op.w, resid=dhs, out_f32=True)


class DetrRT:
    """Whole-model runtime; `forward` returns (cls [D, B, Q, classes + 1], box logits [D, B, Q, 4], tape)."""

    def __init__(self, model):
        self.model = model
        self.sink = GradSink()
        self.body = ResNetRT(model.backbone, has_maxpool=True, head=_NoHead(),
                             checkpoint=getattr(model.backbone, 'use_gradient_checkpoint', False))
        self.body.sink = self.sink
        self.proj = Linear(model.proj_conv)
        tr = model.transformer
        self.enc = [_EncLayer(l) for l in tr.encoder_blocks]
        self.dec = [_DecLayer(l) for l in tr.decoder_blocks]
        self.heads = _Heads(model.head)
        self._seed_base = 0
        self._units = self.body.units() + [self.proj] + [u for l in self.enc + self.dec for u in l.units()] + self.heads.units()

    def operands(self):
        return [u.op for u in self._units]

    def prep(self):
        for u in self._units:
            u.prep()

    def _context(self, B, L, pos, key_bias, training):
        tr = self.model.transformer
        p = float(tr.dropout_prob) if training else 0.
        # One random 62-bit word per forward, drawn ON THE DEVICE (torch's CUDA generator: reproducible under
        # torch.manual_seed and graph-safe - a captured step draws a new word on every replay); the kernels add the
        # per-site constants below to it (saicv_dropout's seed_base).
        sb = torch.empty(1, dtype=torch.int64, device=pos.device).random_(0, 1 << 62) if p > 0. else None
        counter = [0]

        def seeds():
            counter[0] += 8
            return [counter[0] + i for i in range(8)]

        return {'B': B, 'L': L, 'Q': self.model.query_embed.weight.shape[0], 'pos': pos, 'key_bias': key_bias, 'p': p,
                'seed': seeds, 'sb': sb, 'qpos': self.model.query_embed.weight.detach()}

    # ---- stages (tests drive them separately with the oracle's tensors)
    def backbone_forward(self, x, tape, training, keep_tape):
        body = self.body
        tape['body'] = bt = {'stem': {}, 'blocks': [dict() for _ in body.blocks]}
        a = body.stem_forward(x, bt, training)
        ckpt = body.checkpoint and keep_tape
        for b, t in zip(body.blocks, bt['blocks']):
            if ckpt:
                t['ckpt_in'] = a
                a = b.forward(a, {}, training)
            else:
                a = b.forward(a, t, training)
        return a

    def backbone_backward(self, da, tape):
        body, bt = self.body, tape['body']
        da = blocks_backward(body.blocks, bt['blocks'], da, self.sink)
        body.stem_backward(da, bt)

    def transformer_forward(self, src, cx, tape):
        """src fp32 [B*L, C] -> (cls, box logits); fills tape['enc'], tape['dec'], tape['heads']."""
        xb, xpb = ops.add_pos_cast(src, cx['pos'])
        x = src
        tape['enc'] = [dict() for _ in self.enc]
        for i, (l, t) in enumerate(zip(self.enc, tape['enc'])):
            x, xb, xpb = l.forward(x, xb, xpb, t, cx, want_pos_copy=True)
        memb, mempb = xb, xpb
        B, Q, C = cx['B'], cx['Q'], x.shape[1]
        tgt = torch.zeros(B * Q, C, device=x.device, dtype=torch.float32)
        tb, tqb = ops.add_pos_cast(tgt, cx['qpos'])
        tape['dec'] = [dict() for _ in self.dec]
        norm = self.model.transformer.decoder_norm
        D = len(self.dec)
        hsb = torch.empty(D, B * Q, C, device=x.device, dtype=torch.bfloat16)
        tape['inter'] = []
        for i, (l, t) in enumerate(zip(self.dec, tape['dec'])):
            tgt, tb, tqb = l.forward(tgt, tb, tqb, memb, mempb, t, cx)
            _, _, _, stats = ops.postln_fwd(tgt, norm.weight.detach(), norm.bias.detach(), norm.eps, want_y=False, yb_out=hsb[i])
            tape['inter'].append((tgt, stats))
        tape['heads'] = {}
        cls, reg = self.heads.forward(hsb.view(D * B * Q, C), tape['heads'])
        ncls = cls.shape[1]
        return cls.reshape(D, B, Q, ncls), reg.reshape(D, B, Q, 4)

    def transformer_backward(self, dcls, dreg, cx, tape):
        """Returns the fp32 gradient of src [B*L, C]."""
        sink = self.sink
        B, Q = cx['B'], cx['Q']
        D = len(self.dec)
        dhs = self.heads.backward(dcls.reshape(D * B * Q, -1).float(), dreg.reshape(D * B * Q, -1).float(), tape['heads'], sink)
        C = dhs.shape[1]
        dhs = dhs.view(D, B * Q, C)
        norm = self.model.transformer.decoder_norm
        gbuf, gacc = sink.begin(norm.weight)
        bbuf, bacc = sink.begin(norm.bias)
        dy, dmem, dqpos = None, None, None
        for i in reversed(range(D)):
            z, stats = tape['inter'][i]
            # gradient through decoder_norm of this layer's output, plus what the next layer sent back
            dy, _ = ops.postln_bwd(dhs[i], z, norm.weight.detach(), stats, gbuf, bbuf, dres=dy, want_dzb=False,
                                   accumulate=gacc or i != D - 1)
            dy, dmem, dqpos = self.dec[i].backward(dy, tape['dec'][i], sink, cx, dmem, dqpos, need_dx=i > 0)
            tape['dec'][i].clear()
        sink.done(norm.weight, gbuf)
        sink.done(norm.bias, bbuf)
        qe = self.model.query_embed.weight
        qbuf, qacc = sink.begin(qe)
        ops.colsum(dqpos.view(B, -1), qbuf.view(-1), accumulate=qacc)      # sum over the batch of the broadcast rows
        sink.done(qe, qbuf)
        dx = dmem
        for l, t in zip(reversed(self.enc), reversed(tape['enc'])):
            dx = l.backward(dx, t, sink, cx)
            t.clear()
        return dx

    def forward(self, x, pos, key_bias, training, keep_tape):
        """x fp32 [B, 3, H, W]; pos fp32 [B*L, C] (sine embedding, batch-major tokens); key_bias fp32 [B*L]."""
        assert x.is_cuda and x.dtype == torch.float32 and x.dim() == 4
        self.prep()
        tape = {}
        c5 = self.backbone_forward(x.contiguous(), tape, training, keep_tape)
        B, h, w, cf = c5.shape
        L = h * w
        assert pos.shape == (B * L, self.proj.mod.weight.shape[0]) and key_bias.numel() == B * L
        tape['c5'] = c5m = c5.view(B * L, cf)
        src = self.proj.fwd(c5m, out_f32=True)
        cx = tape['cx'] = self._context(B, L, pos.contiguous(), key_bias.contiguous().view(-1), training)
        cls, reg = self.transformer_forward(src, cx, tape)
        tape['c5_shape'] = (B, h, w, cf)
        return cls, reg, (tape if keep_tape else None)

    def backward(self, dcls, dreg, tape):
        assert tape is not None, 'backward called without a training forward'
        sink = self.sink
        dsrc = self.transformer_backward(dcls, dreg, tape['cx'], tape)
        dsb = torch.empty(dsrc.shape, device=dsrc.device, dtype=torch.bfloat16)
        ops.cast_bf16(dsrc, dsb)
        dc5 = self.proj.bwd(dsb, tape['c5'], sink)
        self.backbone_backward(dc5.view(tape['c5_shape']), tape)
        if sink.on_backward_end is not None:
            sink.on_backward_end()


class _DetrFunction(torch.autograd.Function):
    """Couples the runtime to autograd (see engine.convnet._NetFunction): the criterion differentiates the two
    outputs, this node receives their gradients and runs the whole backward pass on our kernels."""

    @staticmethod
    def forward(ctx, x, anchor, rt, pos, key_bias):
        ctx.rt = rt
        cls, reg, ctx.tape = rt.forward(x, pos, key_bias, True, True)
        ctx.shapes = (cls.shape, reg.shape)
        return cls, reg

    @staticmethod
    def backward(ctx, dcls, dreg):
        tape, ctx.tape = ctx.tape, None
        assert tape is not None, 'the graph of this forward pass was already differentiated'
        if dcls is None:
            dcls = torch.zeros(ctx.shapes[0], device=dreg.device)
        if dreg is None:
            dreg = torch.zeros(ctx.shapes[1], device=dcls.device)
        ctx.rt.backward(dcls.contiguous(), dreg.contiguous(), tape)
        return None, None, None, None, None


def run_detr(rt, x, pos, key_bias, training):
    if training and torch.is_grad_enabled():
        anchor = torch.zeros((), device=x.device, requires_grad=True)
        return _DetrFunction.apply(x, anchor, rt, pos, key_bias)
    with torch.no_grad():
        cls, reg, _ = rt.forward(x, pos, key_bias, training, False)
        return cls, reg
