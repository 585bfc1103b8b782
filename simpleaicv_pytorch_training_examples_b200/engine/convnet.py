"""Forward/backward runtime of the ConvBnAct residual networks (ResNet, ResNetCifar).

The nn.Module shells in ``classification/backbones`` keep the reference's parameters, names and
constructors; this runtime executes their math on the H100 kernels of libsaicv_b200.so:

  conv     wgmma implicit GEMM (TMA im2col -> smem -> wgmma -> registers)      csrc/gemm_sm90.cuh
  BN       batch statistics / finalize / apply(+residual)(+ReLU), backward csrc/capi_elementwise.cu
  pooling  max 3x3/2, global average                                       csrc/capi_elementwise.cu

Activations are NHWC bf16; BatchNorm statistics, running stats, parameters and parameter
gradients are fp32 (the reference under autocast: SURVEY.md Appendix C).  Parameter gradients
are written straight into ``param.grad`` (or into the buffers a data-parallel wrapper handed
out through ``grad_buffer_of``), not returned through autograd.

Reference semantics followed: SimpleAICV/classification/backbones/resnet.py:19-48 (ConvBnActBlock),
:51-97 (BasicBlock), :100-155 (Bottleneck), :226-245 (ResNet.forward), resnetforcifar.py:98-108.
"""
import contextlib

import torch

from .. import ops
from .operands import CONV, STEM, Linear, Operand, rows_wgrad
from . import syncbn
from .runtime import Runtime

ACT_NONE, ACT_RELU, ACT_LEAKY, ACT_SILU = 0, 1, 2, 3


def _round_up(v, m):
    return (v + m - 1) // m * m


# BatchNorm's `num_batches_tracked += 1` of every layer of one network forward, applied by ONE torch._foreach_add_ at the end
# of ConvNetRT.forward (53 four-microsecond launches per ResNet-50 step otherwise); None outside a whole-network forward.
_NBT_BATCH = None


def _flush_nbt():
    global _NBT_BATCH
    pending, _NBT_BATCH = _NBT_BATCH, None
    if pending:
        torch._foreach_add_(pending, 1)


class ConvBN:
    """Runtime state of one ConvBnActBlock: conv (no bias) -> BatchNorm2d -> activation.

    Channel counts that are not multiples of 64 (DarkNet's 32-channel layers) run on channel-padded
    activations: filters k..kp-1 and input channels c..cp-1 of the bf16 operand copy are zero, so the
    padded channels stay exactly zero through conv, BatchNorm (shift 0) and the activation, and carry
    zero gradients; parameters, statistics and gradients exposed to torch keep their real sizes."""

    def __init__(self, block, act, res_after_act=False):
        self.conv = block.layer[0]
        self.bn = block.layer[1]
        self.act = act
        self.res_after_act = res_after_act
        k, c, r, s = self.conv.weight.shape
        self.k, self.c, self.r, self.s = k, c, r, s
        self.stride = self.conv.stride[0]
        self.pad = self.conv.padding[0]
        assert self.conv.groups == 1 and self.conv.bias is None and r == s
        assert self.conv.stride[0] == self.conv.stride[1] and self.conv.padding[0] == self.conv.padding[1]
        self.is_stem = (c % 8) != 0            # 3-channel image input: explicit im2col from NCHW fp32
        self.kp = _round_up(k, 64)
        self.cp = c if self.is_stem else _round_up(c, 64)
        self.padded = self.kp != k
        self.op = Operand(self.conv.weight, STEM if self.is_stem else CONV, kp=self.kp, cp=self.cp)
        self.kpad = self.op.kpad
        self.sums = None

    # ---- parameters
    @property
    def w_bf16(self):
        """The bf16 operand copy of the conv weight ([kp][kpad]; None before the first prep())."""
        return self.op.w

    def prep(self):
        bn = self.bn
        dev = self.op.refresh().device
        if self.sums is None or self.sums.device != dev:
            self.sums = torch.zeros(2, self.kp, device=dev)   # backward scratch (consumed within one bn_bwd)
            if self.padded:
                self.gamma_p = torch.ones(self.kp, device=dev)
                self.beta_p = torch.zeros(self.kp, device=dev)
                self.rm_p = torch.zeros(self.kp, device=dev)
                self.rv_p = torch.ones(self.kp, device=dev)
                self.dg_p = torch.empty(self.kp, device=dev)
                self.db_p = torch.empty(self.kp, device=dev)
        if self.padded:
            self.gamma_p[:self.k].copy_(bn.weight.detach())
            self.beta_p[:self.k].copy_(bn.bias.detach())

    def _gamma(self):
        return self.gamma_p if self.padded else self.bn.weight.detach()

    def _beta(self):
        return self.beta_p if self.padded else self.bn.bias.detach()

    # ---- forward
    def out_hw(self, h, w):
        return (ops.conv_out_size(h, self.pad, self.r, self.stride),
                ops.conv_out_size(w, self.pad, self.s, self.stride))

    def conv_fwd(self, a_in, tape, want_stats=False):
        """a_in: NHWC bf16 activation (cp channels), or the NCHW fp32 image batch for the stem.
        want_stats: the GEMM epilogue also accumulates the BatchNorm statistics of its output."""
        if self.is_stem:
            n, _, h, w = a_in.shape
        else:
            n, h, w, cin = a_in.shape
            assert cin == self.cp, f'expected {self.cp} (padded) input channels, got {cin}'
        P, Q = self.out_hw(h, w)
        rows = n * P * Q
        stats = ops.partial_ws(a_in.device, 2 * self.kp) if want_stats else None
        tape['stats'] = (stats, ops.gemm_stats_rows(rows, self.kp)) if want_stats else None
        if self.is_stem:
            cols = ops.stem_im2col(a_in, self.r, self.s, self.stride, self.pad, self.kpad)
            y = ops.linear_fwd(cols, self.op.w, stats=stats).view(n, P, Q, self.kp)
            tape['cols'] = cols
        else:
            cs = ops.make_conv_shape(n, h, w, self.cp, self.kp, self.r, self.s, self.stride, self.pad)
            y = ops.conv_fprop(a_in, self.op.w, cs, stats=stats)
            tape['a_in'] = a_in
            tape['cs'] = cs
        tape['in_hw'] = (h, w)
        tape['y'] = y
        return y

    def bn_prepare(self, y, training, tape):
        """Computes this forward's BN coefficients into the tape: tape['ss'] = (scale, shift) and
        tape['saved'] = (mean, rstd), from batch statistics (training) or running stats (eval).  They
        live in the tape (not on the unit) so that a second forward of the same module before the
        backward of the first (eval pass, micro-batches, EMA/teacher pass) cannot clobber them."""
        bn = self.bn
        rows = y.numel() // self.kp
        track = bn.track_running_stats
        ss = tape['ss'] = torch.empty(2, self.kp, device=y.device)
        saved = tape['saved'] = torch.empty(2, self.kp, device=y.device)
        if training or not track:
            momentum = bn.momentum if bn.momentum is not None else 0.1
            fused = tape.get('stats') if tape is not None else None
            if fused is not None:
                partials, prow = fused
            else:
                partials, prow = ops.bn_stats(y), 0
            if self.padded and track:
                self.rm_p[:self.k].copy_(bn.running_mean)
                self.rv_p[:self.k].copy_(bn.running_var)
            rm = (self.rm_p if self.padded else bn.running_mean) if track else None
            rv = (self.rv_p if self.padded else bn.running_var) if track else None
            # synchronized BatchNorm: the exchanged statistics (global row count) stay in the tape for the backward
            tape['sync'] = syncbn.finalize(partials, prow, rows, self._gamma(), self._beta(), rm, rv, ss, saved, bn.eps,
                                           momentum)
            if self.padded and track:
                bn.running_mean.copy_(self.rm_p[:self.k])
                bn.running_var.copy_(self.rv_p[:self.k])
            if track and bn.num_batches_tracked is not None:
                if _NBT_BATCH is not None:
                    _NBT_BATCH.append(bn.num_batches_tracked)     # one foreach add at the end of the network forward
                else:
                    bn.num_batches_tracked.add_(1)
        else:
            scale = bn.weight.detach() * torch.rsqrt(bn.running_var + bn.eps)
            ss.zero_()
            ss[0, :self.k].copy_(scale)
            ss[1, :self.k].copy_(bn.bias.detach() - bn.running_mean * scale)

    def forward(self, a_in, tape, training, res=None, res_ss=None, want_mask=False):
        """conv -> BN -> (+res) -> act (or act then +res when res_after_act).  res_ss: BN scale/shift
        applied to `res` on the fly (downsample branch).  want_mask: also keep the ReLU mask of the
        output, packed to one bit per element, as tape['bits']."""
        y = self.conv_fwd(a_in, tape, want_stats=training)
        self.bn_prepare(y, training, tape)
        out = torch.empty_like(y)
        act = self.act | (8 if (self.res_after_act and res is not None) else 0)
        bits = tape['bits'] = ops.mask_bits_like(y) if want_mask else None
        ops.bn_apply(y, tape['ss'], out, act, res=res, res_scale_shift=res_ss, mask_bits=bits)
        tape['out'] = out
        return out

    # ---- backward
    @contextlib.contextmanager
    def _bn_grad(self, sink):
        """(gamma, dgamma, dbeta, accumulate) for a BatchNorm backward kernel.  A channel-padded unit's kernel writes kp
        channels of scratch, whose first k go through the sink on exit."""
        if self.padded:
            yield self.gamma_p, self.dg_p, self.db_p, False
            sink.add(self.bn.weight, self.dg_p[:self.k])
            sink.add(self.bn.bias, self.db_p[:self.k])
        else:
            with sink.grad(self.bn.weight, self.bn.bias) as (acc, dg, db):
                yield self.bn.weight.detach(), dg, db, acc

    def bn_bwd(self, dout, tape, sink, bits=None, want_dres=False, act=None):
        """dout: gradient w.r.t. the activated output.  Returns (dy, dres).

        The ReLU mask comes from `bits` (the packed mask of a block output, whose residual was added
        before the activation) or, for plain conv->BN->act units, is recomputed inside the kernels from
        sign(y*scale+shift), which saves reading the activated tensor twice."""
        act = self.act if act is None else act
        y = tape['y']
        ss = tape['ss'] if (act != ACT_NONE and bits is None) else None
        saved = tape['saved']
        ops.bn_bwd_reduce(dout, None, y, saved, self.sums, act, scale_shift=ss, bits=bits)
        sums, sync = syncbn.backward_sums(self.sums, tape.get('sync'), self.kp)
        dy = torch.empty_like(y)
        dres = torch.empty_like(y) if want_dres else None
        with self._bn_grad(sink) as (gamma, dg, db, acc):
            ops.bn_bwd_apply(dout, None, y, saved, gamma, sums, dy, dres, dg, db, act, accumulate=acc,
                             scale_shift=ss, bits=bits, **sync)
        return dy, dres

    def bn_bwd_pair(self, other, g, tape, other_tape, sink, bits):
        """bn_bwd of this unit and of `other` (same rows and channels, no activation of their own) over one gradient:
        g = dout masked by `bits`, or g = dout when bits is None (it arrived masked).  One reduce and one apply read g
        once for both.  Returns (dy, dy_other)."""
        y, yo = tape['y'], other_tape['y']
        sums = torch.empty(4, self.kp, device=y.device)
        ops.bn_bwd_reduce2(g, bits, y, yo, tape['saved'], other_tape['saved'], sums)
        # synchronized: both BatchNorms' sums go in one exchange; they share the row count
        sums, sync = syncbn.backward_sums(sums, tape.get('sync'), self.kp)
        dy, dyo = torch.empty_like(y), torch.empty_like(yo)
        # nested this way round so that this unit's gradients are reported before other's (the inner block exits first)
        with other._bn_grad(sink) as (gb, dgb, dbb, accb), self._bn_grad(sink) as (ga, dga, dba, acca):
            ops.bn_bwd_apply2(g, bits, y, yo, tape['saved'], other_tape['saved'], ga, gb, sums, dy, dyo, dga, dba, dgb, dbb,
                              accumulate_a=acca, accumulate_b=accb, **sync)
        return dy, dyo

    def conv_bwd(self, dy, tape, sink, need_dx=True, add=None, mask_bits=None):
        """dy: gradient w.r.t. the raw conv output [n,P,Q,kp].  Returns the data gradient
        (NHWC bf16, `add` fused in when given, then multiplied by the ReLU mask `mask_bits` when
        given) or None.  A 1x1 stride-2 conv returns ('strided', dd) with the compact gradient
        dd[n,P,Q,cp] that belongs at the even pixels."""
        n, P, Q, _ = dy.shape
        if self.is_stem:
            with sink.grad(self.conv.weight) as (acc, buf):
                part = ops.linear_wgrad(dy.view(-1, self.kp), tape['cols'], transposed=ops.wgrad_transposed(self.kp, self.kpad))
                ops.finish_conv_wgrad(part, buf, self.kpad, accumulate=acc, order=ops.ORDER_CRS, kp=self.kp)
            assert not need_dx, 'the stem has no data gradient'
            return None
        cs = tape['cs']
        with sink.grad(self.conv.weight) as (acc, buf):
            ops.finish_conv_wgrad(ops.conv_wgrad(dy, tape['a_in'], cs), buf, self.kpad, accumulate=acc, kp=self.kp, cp=self.cp)
        if not need_dx:
            return None
        if self.stride == 2 and self.r == 1:
            assert add is None and mask_bits is None
            return 'strided', ops.linear_dgrad(dy.view(-1, self.kp), self.op.w).view(n, P, Q, self.cp)
        return ops.conv_dgrad(dy, self.op.w, cs, add=add, mask_bits=mask_bits)


class ResidualBlockRT:
    """BasicBlock (resnet.py:51-97) or Bottleneck (:100-155): conv chain + identity/downsample."""

    def __init__(self, block):
        names = ['conv1', 'conv2'] + (['conv3'] if hasattr(block, 'conv3') else [])
        self.units = []
        for nm in names:
            # the last unit has no activation of its own: its ReLU is applied after the shortcut add
            self.units.append(ConvBN(getattr(block, nm), ACT_RELU))
        self.down = ConvBN(block.downsample_conv, ACT_NONE) if block.downsample else None

    def all_units(self):
        return self.units + ([self.down] if self.down is not None else [])

    def forward(self, a_in, tape, training):
        tapes = tape.setdefault('u', [dict() for _ in self.units])
        x = a_in
        for u, t in zip(self.units[:-1], tapes[:-1]):
            x = u.forward(x, t, training)
        last, tl = self.units[-1], tapes[-1]
        # the ReLU mask of the block output, one bit per element: the backward applies it instead of reading `out`
        if self.down is not None:
            td = tape.setdefault('d', dict())
            yd = self.down.conv_fwd(a_in, td, want_stats=training)
            self.down.bn_prepare(yd, training, td)
            out = last.forward(x, tl, training, res=yd, res_ss=td['ss'], want_mask=training)
        else:
            out = last.forward(x, tl, training, res=a_in, want_mask=training)
        return out

    @staticmethod
    def out_mask(tape):
        """The packed ReLU mask of the block output kept by forward(), or None (tape of a checkpointed block that has
        not been re-run)."""
        tapes = tape.get('u')
        return tapes[-1].get('bits') if tapes else None

    def backward(self, dout, tape, sink):
        """dout: gradient w.r.t. the block output.  Returns the gradient w.r.t. the block input."""
        return self.backward_chain(dout, tape, sink)[0]

    def backward_chain(self, dout, tape, sink, dout_masked=False, in_mask=None):
        """backward() inside a chain of blocks.  dout_masked: dout is already multiplied by the ReLU mask of this block's
        output (the next block applied it in its data-gradient epilogue).  in_mask: the packed ReLU mask of this block's
        input (the previous block's output), applied to the input gradient in the epilogue of the data-gradient GEMM that
        adds the shortcut gradient, when there is one.  Returns (dx, dx_masked): dx_masked tells whether in_mask was
        applied to dx."""
        tapes = tape['u']
        last, tl = self.units[-1], tapes[-1]
        # g = dout * relu'(out) flows to both the last BN and the shortcut; with dout_masked, dout is g
        bits = None if dout_masked else tl['bits']
        strided = None
        if self.down is None:
            dy, g = last.bn_bwd(dout, tl, sink, bits=bits, want_dres=not dout_masked,
                                act=ACT_NONE if dout_masked else None)
            shortcut = dout if dout_masked else g
        else:
            td = tape['d']
            dy, dyd = last.bn_bwd_pair(self.down, dout, tl, td, sink, bits)
            shortcut = self.down.conv_bwd(dyd, td, sink)
            if isinstance(shortcut, tuple):
                strided, shortcut = shortcut[1], None
        # The shortcut gradient joins the main path inside the data-gradient GEMM of the block's FIRST conv: its tile is
        # the aux operand of that launch's epilogue (TMA-loaded into the staging slice, gemm_sm90.cuh aux_tma), which
        # replaces a separate read-read-write pass over the block input (add_bf16: 13 launches, 1.06 ms per ResNet-50 step).
        first_unit = self.units[0]
        fuse = shortcut is not None and not (first_unit.stride == 2 and first_unit.r == 1)   # that case returns a compact gradient
        # the previous block's ReLU mask rides on the same epilogue: its BatchNorms then read neither its output nor a
        # masked copy of dx (bit-identical: the mask multiplies by 0 / 1 exactly as their kernels would)
        mask = in_mask if fuse else None
        n_main = len(self.units) - 1
        dx = last.conv_bwd(dy, tl, sink, add=shortcut if (fuse and n_main == 0) else None,
                           mask_bits=mask if n_main == 0 else None)
        for i, (u, t) in enumerate(zip(reversed(self.units[:-1]), reversed(tapes[:-1]))):
            dy, _ = u.bn_bwd(dx, t, sink)
            dx = u.conv_bwd(dy, t, sink, add=shortcut if (fuse and i == n_main - 1) else None,
                            mask_bits=mask if i == n_main - 1 else None)
        if shortcut is not None and not fuse:
            ops.add_bf16(dx, shortcut)
        if strided is not None:
            ops.add_strided2(dx, strided)
        return dx, mask is not None


def blocks_backward(blocks, tapes, da, sink):
    """Backward through a chain of stages (last to first); `da` is the gradient w.r.t. the last stage's output.
    Re-runs checkpointed stages first (tape['ckpt_in']) and drops each tape once used.  Between two residual blocks the
    gradient travels masked by the ReLU of the earlier block's output when the later block could apply that mask in its
    data-gradient epilogue; a checkpointed block's mask does not exist yet at that point, so it is masked by itself."""
    masked = False
    for i in reversed(range(len(blocks))):
        b, t = blocks[i], tapes[i]
        if 'ckpt_in' in t:
            b.forward(t.pop('ckpt_in'), t, True)
        if isinstance(b, ResidualBlockRT):
            prev = blocks[i - 1] if i > 0 else None
            in_mask = prev.out_mask(tapes[i - 1]) if isinstance(prev, ResidualBlockRT) else None
            da, masked = b.backward_chain(da, t, sink, dout_masked=masked, in_mask=in_mask)
        else:
            assert not masked
            da = b.backward(da, t, sink)
        t.clear()
    return da


class PlainUnitRT:
    """A single conv -> BN -> act unit used as a stage (DarkNet's strided 3x3 convs)."""

    def __init__(self, block, act):
        self.unit = ConvBN(block, act)

    def all_units(self):
        return [self.unit]

    def forward(self, a_in, tape, training):
        return self.unit.forward(a_in, tape, training)

    def backward(self, dout, tape, sink):
        dy, _ = self.unit.bn_bwd(dout, tape, sink)
        return self.unit.conv_bwd(dy, tape, sink)


class DarkBlockRT:
    """Darknet53Block (darknet.py:116-144): x + act(bn(conv3x3(act(bn(conv1x1(x)))))) — the shortcut is
    added AFTER the activation, so the block gradient flows unmasked into the shortcut."""

    def __init__(self, block, act):
        self.u1 = ConvBN(block.conv[0], act)
        self.u2 = ConvBN(block.conv[1], act, res_after_act=True)

    def all_units(self):
        return [self.u1, self.u2]

    def forward(self, a_in, tape, training):
        t1, t2 = tape.setdefault('u', [dict(), dict()])
        return self.u2.forward(self.u1.forward(a_in, t1, training), t2, training, res=a_in)

    def backward(self, dout, tape, sink):
        t1, t2 = tape['u']
        dy, _ = self.u2.bn_bwd(dout, t2, sink)          # mask of u2's own activation, recomputed from y
        dx = self.u2.conv_bwd(dy, t2, sink)
        dy, _ = self.u1.bn_bwd(dx, t1, sink)
        return self.u1.conv_bwd(dy, t1, sink, add=dout)   # 1x1 stride-1 conv: the shortcut gradient is the epilogue's aux operand


class MaxPoolRT:
    """nn.MaxPool2d stage (DarkNet-19 / tiny 2x2 pools, darknet.py:105,161-213)."""

    def __init__(self, k, stride, pad=0, pad_hi=None, oob_zero=False):
        self.k, self.stride, self.pad, self.pad_hi, self.oob_zero = k, stride, pad, pad_hi, oob_zero

    def all_units(self):
        return []

    def forward(self, a_in, tape, training):
        tape['in_hw'] = (a_in.shape[1], a_in.shape[2])
        out, tape['argmax'] = ops.maxpool_fwd(a_in, self.k, self.stride, self.pad, self.pad_hi, self.oob_zero)
        return out

    def backward(self, dout, tape, sink):
        h, w = tape['in_hw']
        return ops.maxpool_bwd(dout, tape['argmax'], h, w, self.k, self.stride, self.pad, self.pad_hi)


class FcHeadRT:
    """Global average pool -> nn.Linear (resnet.py:203-204,240-243)."""

    def __init__(self, fc):
        self.fc = fc
        self.lin = Linear(fc)
        self.op = self.lin.op

    def prep(self):
        self.lin.prep()

    def forward(self, a, tape):
        tape['feat_hw'] = (a.shape[1], a.shape[2])
        pooled = ops.avgpool_fwd(a)
        feat = self.fc.weight.shape[1]
        if pooled.shape[1] != feat:   # channel-padded feature map (e.g. 16/32-channel stacks)
            pooled = pooled[:, :feat].contiguous()
        return self.fc_forward(pooled, tape)

    def fc_forward(self, pooled, tape):
        """pooled bf16 [B, feat] -> fp32 logits [B, num_classes]."""
        tape['pooled'] = pooled
        ncls = self.fc.weight.shape[0]
        logits = self.lin.fwd(pooled, out_f32=True)
        if logits.shape[1] != ncls:
            logits = logits[:, :ncls].contiguous()
        return logits

    def backward(self, dlogits, tape, sink, cpad):
        """dlogits fp32 [B, num_classes] -> gradient w.r.t. the last feature map (NHWC bf16, cpad channels)."""
        dpooled = self.fc_backward(dlogits, tape, sink)
        feat = self.fc.weight.shape[1]
        if cpad != feat:
            full = torch.zeros(dpooled.shape[0], cpad, device=dpooled.device, dtype=torch.bfloat16)
            full[:, :feat] = dpooled
            dpooled = full
        h, w = tape['feat_hw']
        return ops.avgpool_bwd(dpooled, h, w)

    def fc_backward(self, dlogits, tape, sink):
        """dlogits fp32 [B, num_classes]: writes the Linear's gradients, returns dpooled bf16 [B, feat]."""
        ncls = self.fc.weight.shape[0]
        npad = self.op.w.shape[0]
        dlogits = dlogits.contiguous().float()
        with sink.grad(self.fc.bias) as (acc, buf):
            ops.colsum(dlogits, buf, accumulate=acc)
        dl =torch.zeros(dlogits.shape[0], npad, device=dlogits.device, dtype=torch.bfloat16)
        if npad == ncls:
            ops.cast_bf16(dlogits, dl)
        else:
            dl[:, :ncls] = dlogits.to(torch.bfloat16)
        rows_wgrad(dl, tape['pooled'], self.fc.weight, sink)
        return ops.linear_dgrad(dl, self.op.w)


class ConvHeadRT:
    """Darknet19's classifier (darknet.py:289-297,316-318): 1x1 conv WITH bias, no BN, no activation,
    then global average pool.  The conv is one GEMM over [N*H*W, C]; classes are padded to a multiple of 8."""

    def __init__(self, conv):
        self.conv = conv
        assert conv.kernel_size == (1, 1) and conv.bias is not None
        self.lin = Linear(conv)
        self.op = self.lin.op

    def prep(self):
        self.lin.prep()

    def forward(self, a, tape):
        n, h, w, c = a.shape
        tape['a_in'] = a
        y = self.lin.fwd(a.view(n * h * w, c))      # bf16 [N*H*W, npad]
        pooled = ops.avgpool_fwd(y.view(n, h, w, -1))
        return pooled[:, :self.conv.weight.shape[0]].float()

    def backward(self, dlogits, tape, sink, cpad):
        a = tape['a_in']
        n, h, w, c = a.shape
        ncls = self.conv.weight.shape[0]
        npad = self.op.w.shape[0]
        dl = torch.zeros(n, npad, device=a.device, dtype=torch.bfloat16)
        dl[:, :ncls] = dlogits.to(torch.bfloat16)
        dy = ops.avgpool_bwd(dl, h, w).view(n * h * w, npad)
        rows_wgrad(dy, a.view(n * h * w, c), self.conv.weight, sink)
        full = torch.empty(npad, device=a.device)
        ops.colsum(dy, full)
        sink.add(self.conv.bias, full[:ncls])
        return ops.linear_dgrad(dy, self.op.w).view(n, h, w, c)


class ResNetRT(Runtime):
    """Whole-network runtime for the conv -> BN -> act classifiers: ResNet (resnet.py:158-245),
    ResNetCifar (resnetforcifar.py:27-108), DarknetTiny / Darknet19 / Darknet53 (darknet.py:147-432):
    stem [+ maxpool] + a sequence of stages + head (global average pool + fc, or Darknet19's 1x1-conv
    classifier + pool).

    checkpoint=True (use_gradient_checkpoint, resnet.py:230-234): the tape keeps only each stage's input;
    the backward pass re-runs the stage forward before differentiating it, trading one extra forward for
    the activation memory of all stages.  Like torch.utils.checkpoint in the reference, the replay runs in
    training mode, so BatchNorm running statistics of the checkpointed stages receive a second momentum
    update per step (tests/test_reference_semantics_cpu.py pins that behaviour of the reference)."""

    def __init__(self, model, has_maxpool, stem=None, blocks=None, head=None, checkpoint=False):
        self.model = model
        self.has_maxpool = has_maxpool
        if stem is None:
            stem = ConvBN(model.conv1, ACT_RELU)
            blocks = []
            for layer in (model.layer1, model.layer2, model.layer3, model.layer4):
                for blk in layer:
                    blocks.append(ResidualBlockRT(blk))
        self.stem = stem
        self.blocks = blocks
        self.head = head if head is not None else FcHeadRT(model.fc)
        self.checkpoint = checkpoint
        super().__init__(self.units() + [self.head])

    def units(self):
        us = [self.stem]
        for b in self.blocks:
            us += b.all_units()
        return us

    # The network is run as three stages (stem / residual blocks / head) so that tests can drive
    # each stage with the oracle's tensors (tests/test_resnet_gpu.py, teacher-forced parity).
    def stem_forward(self, x, tape, training):
        a = self.stem.forward(x, tape['stem'], training)
        if self.has_maxpool:
            tape['pool_in_hw'] = (a.shape[1], a.shape[2])
            a, tape['argmax'] = ops.maxpool3x3s2_fwd(a)
        return a

    def blocks_forward(self, a, tapes, training, checkpoint):
        """Runs the blocks on the stem output `a`, one tape each; with checkpoint a tape keeps only its block's input."""
        for b, t in zip(self.blocks, tapes):
            if checkpoint:
                t['ckpt_in'] = a
                a = b.forward(a, {}, training)
            else:
                a = b.forward(a, t, training)
        return a

    def head_forward(self, a, tape):
        tape['feat_c'] = a.shape[3]
        return self.head.forward(a, tape)

    def forward(self, x, training, keep_tape):
        """Returns (logits, tape); the tape (None unless keep_tape) is what backward() consumes."""
        assert x.is_cuda and x.dtype == torch.float32 and x.dim() == 4
        global _NBT_BATCH
        x = x.contiguous()
        self.prep()
        tape = {'stem': {}, 'blocks': [dict() for _ in self.blocks]}
        _NBT_BATCH = [] if training else None
        try:
            a = self.stem_forward(x, tape, training)
            a = self.blocks_forward(a, tape['blocks'], training, self.checkpoint and keep_tape)
            logits = self.head_forward(a, tape)
        finally:
            _flush_nbt()
        return logits, (tape if keep_tape else None)

    def head_backward(self, dlogits, tape):
        return self.head.backward(dlogits, tape, self.sink, tape['feat_c'])

    def stem_backward(self, da, tape):
        if self.has_maxpool:
            ph, pw = tape['pool_in_hw']
            da = ops.maxpool3x3s2_bwd(da, tape['argmax'], ph, pw)
        dy, _ = self.stem.bn_bwd(da, tape['stem'], self.sink)
        self.stem.conv_bwd(dy, tape['stem'], self.sink, need_dx=False)

    def backward(self, dlogits, tape):
        assert tape is not None, 'backward called without a training forward'
        da = self.head_backward(dlogits, tape)
        da = blocks_backward(self.blocks, tape['blocks'], da, self.sink)
        self.stem_backward(da, tape)
