"""Forward/backward runtime of the MAE pre-training model (SURVEY.md 8 f4;
SimpleAICV/masked_image_modeling/models/vit_mae.py) on libsaicv_b200.so.

    patches  = patch_embed(images) + pos[1:]                                  (stem im2col + wgmma GEMM)
    keep     = argsort(noise)[:, :L (1 - mask_ratio)]                         (index work: torch.argsort on the device)
    x        = [cls + pos[0] ; patches[keep] + pos[1 + keep]]                 (saicv_token_gather_fwd)
    x        = encoder blocks (engine.vit._Block, L = 1 + kept tokens), LayerNorm, encoder_to_decoder Linear
    y        = [x[0] ; un-shuffle([x[1:] ; mask tokens])] + decoder pos       (saicv_token_gather_fwd)
    pred     = fc(LayerNorm(decoder blocks(y)))[:, 1:]                        -> loss tail in torch (MSELoss on removed patches)

Every Linear / attention / LayerNorm / GELU is the ViT runtime's kernel path (engine/vit.py); the two token shuffles and
their gradients are one kernel each (csrc/capi_tokens.cu).  dtype flow as in the reference under autocast: fp32 residual
stream, bf16 GEMM operands.  The mask indices are computed with torch.rand / torch.argsort exactly as the reference does
(vit_mae.py:203-225), so a seeded run draws the same masks.
"""
import torch

from .. import ops
from .convnet import GradSink
from .operands import Linear, PatchEmbed
from .vit import _Block, layernorm_bwd


class MAERT:

    def __init__(self, model):
        self.model = model
        enc, dec = model.encoder, model.decoder
        self.enc_blocks = [_Block(b) for b in enc.blocks]
        self.dec_blocks = [_Block(b) for b in dec.blocks]
        self.e2d = Linear(model.encoder_to_decoder)
        self.fc = Linear(dec.fc)
        self.patch = PatchEmbed(enc.patch_embed.proj)
        self._units = [lin for b in self.enc_blocks + self.dec_blocks for lin in b.linears()] + [self.e2d, self.fc, self.patch]
        self.sink = GradSink()

    def operands(self):
        return [u.op for u in self._units]

    def prep(self):
        for u in self._units:
            u.prep()

    # ---- masking indices (vit_mae.py:203-225), int32 index tables for the gather kernels
    def masking(self, b, n, dev, noise=None):
        enc = self.model.encoder
        keep_len = int(n * (1 - enc.mask_ratio))
        if noise is None:
            noise = torch.rand(b, n, device=dev)
        shuffle_ids = torch.argsort(noise, dim=1)
        restore_ids = torch.argsort(shuffle_ids, dim=1)
        keep_ids = shuffle_ids[:, :keep_len]
        mask = torch.ones(b, n, device=dev)
        mask[:, :keep_len] = 0
        mask = torch.gather(mask, dim=1, index=restore_ids)
        neg = torch.full((b, 1), -1, device=dev, dtype=torch.int64)
        zero = torch.zeros(b, 1, device=dev, dtype=torch.int64)
        enc_idx = torch.cat([neg, keep_ids], dim=1).to(torch.int32).contiguous()            # -1: cls token
        enc_pos = torch.cat([zero, keep_ids + 1], dim=1).to(torch.int32).contiguous()
        dec_src = torch.where(restore_ids < keep_len, restore_ids + 1, torch.full_like(restore_ids, -1))   # -1: mask token
        dec_idx = torch.cat([zero, dec_src], dim=1).to(torch.int32).contiguous()
        return keep_len, mask, enc_idx, enc_pos, dec_idx

    def forward(self, x, training, keep_tape, noise=None):
        assert x.is_cuda and x.dtype == torch.float32 and x.dim() == 4
        self.prep()
        enc, dec = self.model.encoder, self.model.decoder
        b, c, cd = x.shape[0], enc.embedding_planes, dec.embedding_planes
        tape = {'enc': [dict() for _ in self.enc_blocks], 'dec': [dict() for _ in self.dec_blocks]}
        patch, tape['cols'] = self.patch.fwd(x.contiguous())                                                 # [B*N, C] fp32
        n = patch.shape[0] // b
        keep_len, mask, enc_idx, enc_pos, dec_idx = self.masking(b, n, x.device, noise)
        le = keep_len + 1
        h = ops.token_gather_fwd(patch.view(b, n, c), enc_idx, enc.cls_token.detach().view(-1),
                                 pos=enc.pos_embed.detach().view(-1, c), pos_idx=enc_pos).view(b * le, c)
        ckpt = keep_tape and enc.use_gradient_checkpoint
        for blk, t in zip(self.enc_blocks, tape['enc']):
            h = self._block_fwd(blk, h, t, b, le, training, ckpt)
        tape['enc_out'] = h
        tape['lne'], tape['ste'] = ops.layernorm_fwd(h, enc.norm.weight.detach(), enc.norm.bias.detach(), enc.norm.eps)
        y = self.e2d.fwd(tape['lne'], out_f32=True)                                                            # [B*le, Cd] fp32
        ld = n + 1
        h = ops.token_gather_fwd(y.view(b, le, cd), dec_idx, dec.mask_token.detach().view(-1),
                                 pos=dec.pos_embed.detach().view(-1, cd)).view(b * ld, cd)
        for blk, t in zip(self.dec_blocks, tape['dec']):
            h = self._block_fwd(blk, h, t, b, ld, training, ckpt)
        tape['dec_out'] = h
        tape['lnd'], tape['std'] = ops.layernorm_fwd(h, dec.norm.weight.detach(), dec.norm.bias.detach(), dec.norm.eps)
        pred = self.fc.fwd(tape['lnd'], out_f32=True).view(b, ld, -1)
        tape.update(b=b, n=n, le=le, ld=ld, enc_idx=enc_idx, dec_idx=dec_idx)
        return pred[:, 1:, :], mask, (tape if keep_tape else None)

    @staticmethod
    def _block_fwd(blk, h, t, b, l, training, ckpt):
        if not ckpt:
            return blk.forward(h, t, b, l, training)
        scratch = {}
        out = blk.forward(h, scratch, b, l, training)       # vit_mae.py:189-192: keep the block input, recompute in backward
        t.update(ckpt_in=h, ckpt_scales=(scratch['s1'], scratch['s2']), s2=scratch['s2'])
        return out

    def _blocks_bwd(self, blocks, tapes, dx, dxb, b, l):
        for i in range(len(blocks) - 1, -1, -1):
            t = tapes[i]
            if 'ckpt_in' in t:
                blocks[i].forward(t.pop('ckpt_in'), t, b, l, True, scales=t.pop('ckpt_scales'))
            dx, dxb = blocks[i].backward(dx, dxb, t, b, l, self.sink)
            t.clear()
        return dx, dxb

    def backward(self, dpred, tape):
        """dpred: gradient of the [B, L, p*p*3] prediction (the cls row of the decoder output gets none)."""
        assert tape is not None, 'backward called without a training forward'
        m, enc, dec, sink = self.model, self.model.encoder, self.model.decoder, self.sink
        b, n, le, ld = tape['b'], tape['n'], tape['le'], tape['ld']
        c, cd = enc.embedding_planes, dec.embedding_planes
        pdim = dpred.shape[2]
        dfull = torch.zeros(b, ld, pdim, device=dpred.device, dtype=torch.bfloat16)
        dfull[:, 1:, :] = dpred
        dlnd = self.fc.bwd(dfull.view(b * ld, pdim), tape['lnd'], sink)
        dx, dxb = layernorm_bwd(dec.norm, dlnd, tape['dec_out'], tape['std'], sink)
        dx, dxb = self._blocks_bwd(self.dec_blocks, tape['dec'], dx, dxb, b, ld)
        # un-shuffle backward: every row of the encoder_to_decoder output is referenced exactly once; mask-token rows sum up
        dy, dmask = ops.token_gather_bwd(dx.view(b, ld, cd), tape['dec_idx'], le, zero=False)
        mbuf, macc = sink.begin(dec.mask_token)
        mbuf.view(-1).copy_(dmask + (mbuf.view(-1) if macc else 0))
        sink.done(dec.mask_token, mbuf)
        dlne = self.e2d.bwd(dy.view(b * le, cd), tape['lne'], sink)
        dx, dxb = layernorm_bwd(enc.norm, dlne, tape['enc_out'], tape['ste'], sink)
        dx, dxb = self._blocks_bwd(self.enc_blocks, tape['enc'], dx, dxb, b, le)
        # gather backward: masked patches get no gradient; the cls rows sum into the cls token (pos_embed is frozen)
        dpatch, dcls = ops.token_gather_bwd(dx.view(b, le, c), tape['enc_idx'], n, zero=True)
        cbuf, cacc = sink.begin(enc.cls_token)
        cbuf.view(-1).copy_(dcls + (cbuf.view(-1) if cacc else 0))
        sink.done(enc.cls_token, cbuf)
        self.patch.bwd(dpatch.view(b * n, c), tape['cols'], sink)
        if sink.on_backward_end is not None:
            sink.on_backward_end()


class _MAEFunction(torch.autograd.Function):
    """The loss tail (torch) differentiates the prediction; this node runs the whole backward on the runtime's kernels
    and deposits the parameter gradients through the GradSink.  The tape lives on ctx (one per forward)."""

    @staticmethod
    def forward(ctx, x, anchor, rt, noise):
        ctx.rt = rt
        pred, mask, ctx.tape = rt.forward(x, True, True, noise)
        ctx.mark_non_differentiable(mask)
        return pred, mask

    @staticmethod
    def backward(ctx, dpred, dmask):
        tape, ctx.tape = ctx.tape, None
        assert tape is not None, 'the graph of this forward pass was already differentiated'
        ctx.rt.backward(dpred.contiguous(), tape)
        return None, None, None, None


def run_mae(rt, x, training, noise=None):
    if training and torch.is_grad_enabled():
        anchor = torch.zeros((), device=x.device, requires_grad=True)
        return _MAEFunction.apply(x, anchor, rt, noise)
    with torch.no_grad():
        pred, mask, _ = rt.forward(x, training, False, noise)
        return pred, mask
