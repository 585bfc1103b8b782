"""The bf16 GEMM operand copies the runtimes keep of their fp32 weights, and the units built directly on them.

An ``Operand`` owns the copy of one ``nn.Parameter`` in the layout its GEMM reads:

  rows  Linear / 1x1-conv weight [N][K], rows zero-padded to a multiple of 8                   saicv_cast_bf16
  conv  tap-major [kp][R*S*cp], column tap*cp + c; filters K..kp-1 and channels C..cp-1 zero  saicv_prep_conv_weight (RSC)
  stem  [kp][kpad], column (c*R + r)*S8 + s, the layout of the explicit stem im2col          saicv_prep_conv_weight (CRS)

``refresh()`` re-creates the copy when the parameter's storage or version changed.  The fused optimizers (optim.py) write
the ``rows`` and ``conv`` copies inside their update and leave those parameters' version alone, so the next ``refresh()``
skips them; ``stem`` copies are not fusable and are re-created by ``refresh()`` after every update.  Each runtime lists its
operands once, in ``operands()``, and its ``prep()`` refreshes exactly those.
"""
import torch

from .. import ops

ROWS, CONV, STEM = 'rows', 'conv', 'stem'


class Operand:

    def __init__(self, param, layout=ROWS, kp=0, cp=0):
        self.param, self.layout = param, layout
        self.fusable = layout != STEM
        self.conv = None       # (c, r*s, cp, kpad) of a conv copy for the optimizer; None for rows
        if layout == ROWS:
            n = param.shape[0]
            self.shape = ((n + 7) // 8 * 8, param.numel() // n)
        else:
            k, c, r, s = param.shape
            self.kp, self.cp = kp or k, cp or c
            self.kpad = r * s * self.cp if layout == CONV else ops.stem_kpad(c, r, s)
            self.shape = (self.kp, self.kpad)
            if layout == CONV:
                self.conv = (c, r * s, self.cp, self.kpad)
        self.w = None          # the bf16 copy, allocated by the first refresh() on the parameter's device
        self._key = None

    def refresh(self):
        """Brings the copy up to date with the parameter and returns it."""
        p = self.param
        key = (p.data_ptr(), p._version)
        if key != self._key:
            if self.w is None or self.w.device != p.device:
                alloc = torch.zeros if self.layout == ROWS else torch.empty
                self.w = alloc(self.shape, device=p.device, dtype=torch.bfloat16)
            if self.layout == ROWS:
                ops.cast_bf16(p.detach(), self.w[:p.shape[0]])
            elif self.layout == CONV:
                ops.prep_conv_weight(p.detach(), self.w, self.kpad, order=ops.ORDER_RSC, kp=self.kp, cp=self.cp)
            else:
                ops.prep_conv_weight(p.detach(), self.w, self.kpad, order=ops.ORDER_CRS, kp=self.kp)
            self._key = key
        return self.w


def rows_wgrad(dy, x, weight, sink):
    """Weight gradient of a GEMM with a ``rows`` operand: dy bf16 [M, N8] (N8 = the padded rows), x bf16 [M, K].  Writes
    the [N, K] gradient of `weight` through the sink."""
    n = weight.shape[0]
    wbuf, wacc = sink.begin(weight)
    part = ops.linear_wgrad(dy, x)
    if part.shape[1] == n:
        ops.reduce_partials(part, wbuf, accumulate=wacc)
    else:
        tmp = torch.empty(part.shape[1], part.shape[2], device=dy.device)
        ops.reduce_partials(part, tmp)
        g = tmp[:n].view_as(wbuf)
        wbuf.copy_(g + wbuf if wacc else g)
    sink.done(weight, wbuf)


class Linear:
    """bf16 operand copy + forward / backward of one nn.Linear (or 1x1 conv), with or without bias."""

    def __init__(self, mod):
        self.mod = mod
        self.op = Operand(mod.weight)
        self.b_pad = None

    def prep(self):
        w, b = self.op.refresh(), self.mod.bias
        if b is None:
            return
        if self.b_pad is None or self.b_pad.device != w.device:
            self.b_pad = torch.zeros(w.shape[0], device=w.device)
        self.b_pad[:b.shape[0]].copy_(b.detach())

    def fwd(self, x, resid=None, out_f32=False, row_scale=None, rows_per_scale=0):
        return ops.linear_fwd(x, self.op.w, bias=self.b_pad, resid=resid, out_f32=out_f32,
                              row_scale=row_scale, rows_per_scale=rows_per_scale)

    def fwd_flags(self, x, flags):
        """Forward with an activation fused in the epilogue (ops.EPI_RELU / ops.EPI_GELU)."""
        return ops.linear_fwd(x, self.op.w, bias=self.b_pad, flags=flags)

    def bwd(self, dy, x, sink, need_dx=True, gelu_pre=None, relu_out=None, add=None):
        """dy bf16 [M, N], x bf16 [M, K]: writes dW, db through the sink, returns dx bf16
        (multiplied by gelu'(gelu_pre) when the input of this layer was gelu(gelu_pre), masked by
        relu_out > 0 when it was a ReLU output, plus `add` when a second gradient joins there)."""
        b = self.mod.bias
        rows_wgrad(dy, x, self.mod.weight, sink)
        if b is not None:
            n = b.shape[0]
            bbuf, bacc = sink.begin(b)
            if dy.shape[1] == n:
                ops.colsum(dy, bbuf, accumulate=bacc)
            else:
                full = torch.empty(dy.shape[1], device=dy.device)
                ops.colsum(dy, full)
                bbuf.copy_(full[:n] + (bbuf if bacc else 0))
            sink.done(b, bbuf)
        return ops.linear_dgrad(dy, self.op.w, gelu_pre=gelu_pre, relu_out=relu_out, add=add) if need_dx else None


class PatchEmbed:
    """Non-overlapping patch embedding of an NCHW fp32 image (Conv2d with bias, kernel = stride = patch size, no
    padding): stem im2col + one GEMM with the bias fused, fp32 tokens out."""

    def __init__(self, conv):
        self.conv = conv
        self.p = conv.kernel_size[0]
        self.op = Operand(conv.weight, STEM)

    def prep(self):
        self.op.refresh()

    def fwd(self, x):
        """Returns (patch tokens fp32 [B*P*Q, C], the im2col matrix bwd() needs)."""
        cols = ops.stem_im2col(x, self.p, self.p, self.p, 0, self.op.kpad)
        return ops.linear_fwd(cols, self.op.w, bias=self.conv.bias.detach(), out_f32=True), cols

    def bwd(self, dy, cols, sink):
        """dy bf16 [B*P*Q, C]: writes the weight and bias gradients through the sink."""
        w, b = self.conv.weight, self.conv.bias
        wbuf, wacc = sink.begin(w)
        part = ops.linear_wgrad(dy, cols)
        ops.finish_conv_wgrad(part, wbuf, self.op.kpad, accumulate=wacc, order=ops.ORDER_CRS)
        sink.done(w, wbuf)
        bbuf, bacc = sink.begin(b)
        ops.colsum(dy, bbuf, accumulate=bacc)
        sink.done(b, bbuf)
