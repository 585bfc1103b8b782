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
from .operands import Linear, PatchEmbed, rows_wgrad


def layernorm_bwd(norm, dy, x, stats, sink, dres=None, want_bf16=True, scale=None, rows_per_scale=0):
    """Backward of a row LayerNorm (nn.LayerNorm `norm`): dgamma / dbeta through the sink; returns (dx fp32 (+ dres), its
    bf16 copy multiplied by the row scale `scale` (one per rows_per_scale rows), or None unless want_bf16)."""
    gbuf, gacc = sink.begin(norm.weight)
    bbuf, bacc = sink.begin(norm.bias)
    dxb = torch.empty(x.shape, device=x.device, dtype=torch.bfloat16) if want_bf16 else None
    dx = ops.layernorm_bwd(dy, x, norm.weight.detach(), stats, gbuf, bbuf, dres=dres, dx_bf16=dxb, accumulate=gacc,
                           bf16_row_scale=scale, rows_per_scale=rows_per_scale)
    sink.done(norm.weight, gbuf)
    sink.done(norm.bias, bbuf)
    return dx, dxb


class _Block:

    def __init__(self, blk):
        self.blk = blk
        self.qkv, self.proj = Linear(blk.attn.qkv), Linear(blk.attn.proj)
        self.fc1, self.fc2 = Linear(blk.mlp.fc1), Linear(blk.mlp.fc2)
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
        # the bf16 copies of dx carry the drop-path scale of the branch that consumes them
        dx, dxb = layernorm_bwd(blk.norm2, dln2, t['x_mid'], t['st2'], sink, dres=dx, scale=t['s1'], rows_per_scale=l)
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
        return layernorm_bwd(blk.norm1, dln1, t['x_in'], t['st1'], sink, dres=dx, scale=next_scale, rows_per_scale=l)


class ViTRT:
    """Whole-network runtime (vit.py:239-262)."""

    def __init__(self, model):
        self.model = model
        self.blocks = [_Block(b) for b in model.blocks]
        self.fc = Linear(model.fc)
        self.patch = PatchEmbed(model.patch_embed.proj)
        self._units = [lin for b in self.blocks for lin in b.linears()] + [self.fc, self.patch]
        self.sink = GradSink()

    def operands(self):
        return [u.op for u in self._units]

    def prep(self):
        for u in self._units:
            u.prep()

    # ---- stages (driven separately by the teacher-forced parity tests)
    def embed_forward(self, x, tape):
        m = self.model
        b = x.shape[0]
        patch, tape['cols'] = self.patch.fwd(x)
        np_ = patch.shape[0] // b
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
        npad = self.fc.op.w.shape[0]
        dl = torch.zeros(b, npad, device=dlogits.device, dtype=torch.bfloat16)
        dl[:, :ncls] = dlogits.to(torch.bfloat16)
        # fc bias gradient from the fp32 dlogits
        bbuf, bacc = sink.begin(m.fc.bias)
        ops.colsum(dlogits.contiguous().float(), bbuf, accumulate=bacc)
        rows_wgrad(dl, tape['lnf'], m.fc.weight, sink)
        dlnf = ops.linear_dgrad(dl, self.fc.op.w)
        sink.done(m.fc.bias, bbuf)
        dpooled, _ = layernorm_bwd(m.norm, dlnf, tape['pooled'], tape['stf'], sink, want_bf16=False)
        dxb = torch.empty(b * l, c, device=dl.device, dtype=torch.bfloat16)
        dx = ops.token_pool_bwd(dpooled, l, m.global_pool, dx_bf16=dxb.view(b, l, c), bf16_row_scale=next_scale)
        return dx.view(b * l, c), dxb

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
        self.patch.bwd(dpatch, tape['cols'], sink)

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
