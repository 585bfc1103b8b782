"""Forward/backward runtime of the ViT classifiers on libsaicv_b200.so.

Per block (SimpleAICV/classification/backbones/vit.py:159-161, pre-LN):
    x = x + drop_path(proj(attention(qkv(LN1(x)))))        x: fp32 residual stream [B*L, C]
    x = x + drop_path(fc2(gelu(fc1(LN2(x)))))
Every Linear is one launch of the wgmma GEMM engine (csrc/gemm_sm90.cuh): forward with the
bias (+ fp32 residual) fused in the epilogue, data gradient with W consumed MN-major, weight
gradient with both operands MN-major and split-K.  LayerNorm, GELU, token assembly / pooling and
the fused attention are in csrc/capi_vit.cu.  dtype flow = the reference under autocast
(SURVEY.md Appendix C): fp32 residual stream / LN statistics / softmax, bf16 GEMM operands.

DropPath (vit.py:102-135): the per-sample Bernoulli(keep)/keep scale is drawn with torch on the
device (one [B] tensor per branch) and applied to the branch output and to its gradient.
"""
import torch

from .. import ops
from .convnet import GradSink


class _Linear:
    """bf16 operand copy + forward / backward of one nn.Linear."""

    def __init__(self, mod):
        self.mod = mod
        self.w_bf16 = None
        self.version = None

    def prep(self):
        w = self.mod.weight
        ver = (w.data_ptr(), w._version)
        if self.w_bf16 is None or ver != self.version:
            if self.w_bf16 is None or self.w_bf16.device != w.device:
                npad = (w.shape[0] + 7) // 8 * 8
                self.w_bf16 = torch.zeros(npad, w.shape[1], device=w.device, dtype=torch.bfloat16)
                self.b_pad = torch.zeros(npad, device=w.device)
            ops.cast_bf16(w.detach(), self.w_bf16[:w.shape[0]])
            self.version = ver
        self.b_pad[:w.shape[0]].copy_(self.mod.bias.detach())

    def fwd(self, x, resid=None, out_f32=False, row_scale=None, rows_per_scale=0):
        return ops.linear_fwd(x, self.w_bf16, bias=self.b_pad, resid=resid, out_f32=out_f32,
                              row_scale=row_scale, rows_per_scale=rows_per_scale)

    def fwd_flags(self, x, flags):
        """Forward with an activation fused in the epilogue (ops.EPI_RELU / ops.EPI_GELU)."""
        return ops.linear_fwd(x, self.w_bf16, bias=self.b_pad, flags=flags)

    def bwd(self, dy, x, sink, need_dx=True, gelu_pre=None, relu_out=None, add=None):
        """dy bf16 [M, N], x bf16 [M, K]: writes dW, db through the sink, returns dx bf16
        (multiplied by gelu'(gelu_pre) when the input of this layer was gelu(gelu_pre), masked by
        relu_out > 0 when it was a ReLU output, plus `add` when a second gradient joins there)."""
        w, b = self.mod.weight, self.mod.bias
        n = w.shape[0]
        wbuf, wacc = sink.begin(w)
        part = ops.linear_wgrad(dy, x)
        if part.shape[1] == n:
            ops.reduce_partials(part, wbuf, accumulate=wacc)
        else:  # padded class dimension
            tmp = torch.empty(part.shape[1], part.shape[2], device=dy.device)
            ops.reduce_partials(part, tmp)
            wbuf.copy_(tmp[:n] + (wbuf if wacc else 0))
        sink.done(w, wbuf)
        bbuf, bacc = sink.begin(b)
        if dy.shape[1] == n:
            ops.colsum(dy, bbuf, accumulate=bacc)
        else:
            full = torch.empty(dy.shape[1], device=dy.device)
            ops.colsum(dy, full)
            bbuf.copy_(full[:n] + (bbuf if bacc else 0))
        sink.done(b, bbuf)
        return ops.linear_dgrad(dy, self.w_bf16, gelu_pre=gelu_pre, relu_out=relu_out, add=add) if need_dx else None


class _Block:

    def __init__(self, blk):
        self.blk = blk
        self.qkv, self.proj = _Linear(blk.attn.qkv), _Linear(blk.attn.proj)
        self.fc1, self.fc2 = _Linear(blk.mlp.fc1), _Linear(blk.mlp.fc2)
        self.heads = blk.attn.head_nums
        self.scale = blk.attn.scale
        self.drop_path = getattr(blk.drop_path, 'drop_path_prob', 0.)

    def linears(self):
        return [self.qkv, self.proj, self.fc1, self.fc2]

    def _path_scale(self, b, l, training, dev):
        if not training or self.drop_path == 0.:
            return None
        keep = 1. - self.drop_path
        s = torch.empty(b, device=dev).bernoulli_(keep)
        if keep > 0.:
            s.div_(keep)
        return s

    def forward(self, x, t, b, l, training, p=0., seeds=None, scales=None, sb=None):
        """x: fp32 [B*L, C] -> fp32 [B*L, C].  p: dropout probability of this pass (vit.py:59,73-78,90-97: attention
        probabilities, after proj, after GELU, after fc2) with the counter-hash seeds `seeds`; scales: drop-path
        scales to reuse (the recomputation of a checkpointed block must see the forward's draws)."""
        blk, c = self.blk, x.shape[1]
        d = c // self.heads
        t['x_in'], t['p'], t['seeds'], t['sb'] = x, p, seeds, sb
        t['ln1'], t['st1'] = ops.layernorm_fwd(x, blk.norm1.weight.detach(), blk.norm1.bias.detach(), blk.norm1.eps)
        t['qkv'] = self.qkv.fwd(t['ln1'])
        if p > 0.:
            q, k, v = (t['qkv'].view(b, l, 3, self.heads, d)[:, :, i].permute(0, 2, 1, 3) for i in range(3))
            t['att'] = torch.empty(b * l, c, device=x.device, dtype=torch.bfloat16)
            _, t['lse'] = ops.attn_fwd(q, k, v, self.scale, out=t['att'].view(b, l, self.heads, d).permute(0, 2, 1, 3),
                                       dropout_p=p, dropout_seed=seeds[0], dropout_seed_base=sb)
        else:
            t['att'], t['lse'] = ops.attention_fwd(t['qkv'], b, l, self.heads, d, self.scale)
        s1 = t['s1'] = scales[0] if scales is not None else self._path_scale(b, l, training, x.device)
        if p > 0.:
            x = ops.dropout(self.proj.fwd(t['att']), p, seeds[1], resid=x, row_scale=s1, elems_per_scale=l * c, seed_base=sb)
        else:
            x = self.proj.fwd(t['att'], resid=x, out_f32=True, row_scale=s1, rows_per_scale=l)
        t['x_mid'] = x
        t['ln2'], t['st2'] = ops.layernorm_fwd(x, blk.norm2.weight.detach(), blk.norm2.bias.detach(), blk.norm2.eps)
        t['u'] = self.fc1.fwd(t['ln2'])
        t['h'] = ops.gelu_fwd(t['u'])
        if p > 0.:
            ops.dropout(t['h'], p, seeds[2], out=t['h'], seed_base=sb)
        s2 = t['s2'] = scales[1] if scales is not None else self._path_scale(b, l, training, x.device)
        if p > 0.:
            return ops.dropout(self.fc2.fwd(t['h']), p, seeds[3], resid=x, row_scale=s2, elems_per_scale=l * c, seed_base=sb)
        return self.fc2.fwd(t['h'], resid=x, out_f32=True, row_scale=s2, rows_per_scale=l)

    def _ln_bwd(self, norm, dy, x, stats, dres, sink, scale, l):
        """`scale`: drop-path scale of the branch that will consume the bf16 copy of dx."""
        gbuf, gacc = sink.begin(norm.weight)
        bbuf, bacc = sink.begin(norm.bias)
        dxb = torch.empty(x.shape, device=x.device, dtype=torch.bfloat16)
        dx = ops.layernorm_bwd(dy, x, norm.weight.detach(), stats, gbuf, bbuf, dres=dres, dx_bf16=dxb, accumulate=gacc,
                               bf16_row_scale=scale, rows_per_scale=l)
        sink.done(norm.weight, gbuf)
        sink.done(norm.bias, bbuf)
        return dx, dxb

    def backward(self, dx, dxb, t, b, l, sink, next_scale=None):
        """dx fp32: gradient w.r.t. the block output; dxb: its bf16 copy already multiplied by this
        block's MLP drop-path scale (t['s2']).  Returns (dx_in fp32, bf16 copy multiplied by
        `next_scale`, the MLP drop-path scale of the block that consumes it)."""
        blk = self.blk
        d = dx.shape[1] // self.heads
        p, seeds, sb = t['p'], t['seeds'], t['sb']
        # ---- MLP branch: fc2 data gradient comes out already multiplied by gelu'(u)
        g = ops.dropout(dxb, p, seeds[3], seed_base=sb) if p > 0. else dxb
        du = self.fc2.bwd(g, t['h'], sink, gelu_pre=t['u'])
        if p > 0.:
            ops.dropout(du, p, seeds[2], out=du, seed_base=sb)
        dln2 = self.fc1.bwd(du, t['ln2'], sink)
        dx, dxb = self._ln_bwd(blk.norm2, dln2, t['x_mid'], t['st2'], dx, sink, t['s1'], l)
        # ---- attention branch
        g = ops.dropout(dxb, p, seeds[1], seed_base=sb) if p > 0. else dxb
        datt = self.proj.bwd(g, t['att'], sink)
        if p > 0.:
            c = dx.shape[1]
            qv, kv, vv = (t['qkv'].view(b, l, 3, self.heads, d)[:, :, i].permute(0, 2, 1, 3) for i in range(3))
            dqkv = torch.empty_like(t['qkv'])
            dq, dk, dv = (dqkv.view(b, l, 3, self.heads, d)[:, :, i].permute(0, 2, 1, 3) for i in range(3))
            ops.attn_bwd(qv, kv, vv, t['att'].view(b, l, self.heads, d).permute(0, 2, 1, 3), t['lse'],
                         datt.view(b, l, self.heads, d).permute(0, 2, 1, 3), self.scale, dq, dk, dv, dropout_p=p, dropout_seed=seeds[0], dropout_seed_base=sb)
        else:
            dqkv = ops.attention_bwd(t['qkv'], t['att'], datt, t['lse'], b, l, self.heads, d, self.scale)
        dln1 = self.qkv.bwd(dqkv, t['ln1'], sink)
        return self._ln_bwd(blk.norm1, dln1, t['x_in'], t['st1'], dx, sink, next_scale, l)


class ViTRT:
    """Whole-network runtime (vit.py:239-262)."""

    def __init__(self, model):
        self.model = model
        self.blocks = [_Block(b) for b in model.blocks]
        self.fc = _Linear(model.fc)
        self.sink = GradSink()
        self.pw_bf16 = None
        self.pw_version = None

    def prep(self):
        for b in self.blocks:
            for lin in b.linears():
                lin.prep()
        self.fc.prep()
        w = self.model.patch_embed.proj.weight
        ver = (w.data_ptr(), w._version)
        if self.pw_bf16 is None or ver != self.pw_version:
            k = w.shape[1] * w.shape[2] * w.shape[3]
            self.kpad = ops.stem_kpad(w.shape[1], w.shape[2], w.shape[3])
            if self.pw_bf16 is None:
                self.pw_bf16 = torch.empty(w.shape[0], self.kpad, device=w.device, dtype=torch.bfloat16)
            ops.prep_conv_weight(w.detach(), self.pw_bf16, self.kpad, order=ops.ORDER_CRS)
            self.pw_version = ver

    # ---- stages (driven separately by the teacher-forced parity tests)
    def embed_forward(self, x, tape):
        m = self.model
        b = x.shape[0]
        p = m.patch_size
        cols = ops.stem_im2col(x, p, p, p, 0, self.kpad)
        tape['cols'] = cols
        patch = ops.linear_fwd(cols, self.pw_bf16, bias=m.patch_embed.proj.bias.detach(), out_f32=True)
        np_ = cols.shape[0] // b
        c = m.embedding_planes
        tokens = ops.vit_assemble_tokens(patch, m.cls_token.detach().view(-1), m.pos_embed.detach().view(-1, c), b, np_, c)
        tape['b'], tape['l'] = b, np_ + 1
        return tokens.view(b * (np_ + 1), c)

    def head_forward(self, x, tape):
        m = self.model
        b, l, c = tape['b'], tape['l'], m.embedding_planes
        pooled = ops.token_pool_fwd(x.view(b, l, c), m.global_pool)
        tape['pooled'] = pooled
        tape['lnf'], tape['stf'] = ops.layernorm_fwd(pooled, m.norm.weight.detach(), m.norm.bias.detach(), m.norm.eps)
        logits = self.fc.fwd(tape['lnf'], out_f32=True)
        ncls = m.fc.weight.shape[0]
        return logits if logits.shape[1] == ncls else logits[:, :ncls].contiguous()

    def forward(self, x, training, keep_tape):
        assert x.is_cuda and x.dtype == torch.float32 and x.dim() == 4
        self.prep()
        m = self.model
        tape = {'blocks': [dict() for _ in self.blocks]}
        p = float(getattr(m, 'dropout_prob', 0.)) if training else 0.
        # one random 62-bit word per forward drawn on the device (torch's CUDA generator: reproducible under
        # torch.manual_seed, and graph-safe: a captured step draws a new word every replay); per-site constants are added
        sb = torch.empty(1, dtype=torch.int64, device=x.device).random_(0, 1 << 62) if p > 0. else None
        tape['p'], tape['sb'] = p, sb
        h = self.embed_forward(x.contiguous(), tape)
        if p > 0.:   # vit.py:244 embedding_dropout
            ops.dropout(h, p, 0, out=h, seed_base=sb)
        ckpt = keep_tape and getattr(m, 'use_gradient_checkpoint', False)
        for i, (blk, t) in enumerate(zip(self.blocks, tape['blocks'])):
            seeds = [8 * (i + 1) + j for j in range(4)]
            if ckpt:   # vit.py:247-249: keep the block input (and this pass's random draws), recompute in backward
                scratch = {}
                out = blk.forward(h, scratch, tape['b'], tape['l'], training, p, seeds, sb=sb)
                t.update(ckpt_in=h, ckpt_scales=(scratch['s1'], scratch['s2']), s2=scratch['s2'], p=p, seeds=seeds, sb=sb)
                h = out
            else:
                h = blk.forward(h, t, tape['b'], tape['l'], training, p, seeds, sb=sb)
        logits = self.head_forward(h, tape)
        return logits, (tape if keep_tape else None)

    def head_backward(self, dlogits, tape, next_scale=None):
        m, sink = self.model, self.sink
        b, l, c = tape['b'], tape['l'], m.embedding_planes
        ncls = m.fc.weight.shape[0]
        npad = self.fc.w_bf16.shape[0]
        dl = torch.zeros(b, npad, device=dlogits.device, dtype=torch.bfloat16)
        dl[:, :ncls] = dlogits.to(torch.bfloat16)
        # fc bias gradient from the fp32 dlogits
        bbuf, bacc = sink.begin(m.fc.bias)
        ops.colsum(dlogits.contiguous().float(), bbuf, accumulate=bacc)
        dlnf = self._fc_bwd_nobias(dl, tape['lnf'])
        sink.done(m.fc.bias, bbuf)
        gbuf, gacc = sink.begin(m.norm.weight)
        nbuf, nacc = sink.begin(m.norm.bias)
        dpooled = ops.layernorm_bwd(dlnf, tape['pooled'], m.norm.weight.detach(), tape['stf'], gbuf, nbuf, accumulate=gacc)
        sink.done(m.norm.weight, gbuf)
        sink.done(m.norm.bias, nbuf)
        dxb = torch.empty(b * l, c, device=dl.device, dtype=torch.bfloat16)
        dx = ops.token_pool_bwd(dpooled, l, m.global_pool, dx_bf16=dxb.view(b, l, c), bf16_row_scale=next_scale)
        return dx.view(b * l, c), dxb

    def _fc_bwd_nobias(self, dl, x):
        m, sink = self.model, self.sink
        w = m.fc.weight
        n = w.shape[0]
        wbuf, wacc = sink.begin(w)
        part = ops.linear_wgrad(dl, x)
        if part.shape[1] == n:
            ops.reduce_partials(part, wbuf, accumulate=wacc)
        else:
            tmp = torch.empty(part.shape[1], part.shape[2], device=dl.device)
            ops.reduce_partials(part, tmp)
            wbuf.copy_(tmp[:n] + (wbuf if wacc else 0))
        sink.done(w, wbuf)
        return ops.linear_dgrad(dl, self.fc.w_bf16)

    def embed_backward(self, dx, tape):
        m, sink = self.model, self.sink
        b, l, c = tape['b'], tape['l'], m.embedding_planes
        pbuf, pacc = sink.begin(m.pos_embed)
        cbuf, cacc = sink.begin(m.cls_token)
        assert pacc == cacc
        dpatch = torch.empty(b * (l - 1), c, device=dx.device, dtype=torch.bfloat16)
        ops.vit_assemble_tokens_bwd(dx.view(b, l, c), pbuf, cbuf, dpatch, accumulate=pacc)
        sink.done(m.pos_embed, pbuf)
        sink.done(m.cls_token, cbuf)
        w, bias = m.patch_embed.proj.weight, m.patch_embed.proj.bias
        wbuf, wacc = sink.begin(w)
        part = ops.linear_wgrad(dpatch, tape['cols'])
        ops.finish_conv_wgrad(part, wbuf, self.kpad, accumulate=wacc, order=ops.ORDER_CRS)
        sink.done(w, wbuf)
        bbuf, bacc = sink.begin(bias)
        ops.colsum(dpatch, bbuf, accumulate=bacc)
        sink.done(bias, bbuf)

    def backward(self, dlogits, tape):
        sink = self.sink
        assert tape is not None, 'backward called without a training forward'
        tapes = tape['blocks']
        dx, dxb = self.head_backward(dlogits, tape, next_scale=tapes[-1]['s2'] if tapes else None)
        for i in range(len(self.blocks) - 1, -1, -1):
            nxt = tapes[i - 1]['s2'] if i > 0 else None
            t = tapes[i]
            if 'ckpt_in' in t:
                self.blocks[i].forward(t.pop('ckpt_in'), t, tape['b'], tape['l'], True, t['p'], t['seeds'], scales=t.pop('ckpt_scales'), sb=t['sb'])
            dx, dxb = self.blocks[i].backward(dx, dxb, t, tape['b'], tape['l'], sink, next_scale=nxt)
            t.clear()
        if tape['p'] > 0.:
            ops.dropout(dx, tape['p'], 0, out=dx, seed_base=tape['sb'])
        self.embed_backward(dx, tape)
        if sink.on_backward_end is not None:
            sink.on_backward_end()
