"""Forward/backward runtime of the VAN classifiers (SimpleAICV/classification/backbones/van.py) on
libsaicv_b200.so.

Per Block (van.py:154-186), residual stream x fp32 [rows, C] (rows = N*H*W, NHWC):
    a  = BN1(x)                         bf16     csrc/capi_van.cu  (BatchNorm over the fp32 stream)
    p1 = relu(proj_1(a))                         wgmma GEMM, bias + ReLU in the epilogue   (van.py:101,106-108)
    c1 = conv1(dw7x7d3(dw5x5(p1)))               depthwise kernels + GEMM                    (van.py:63-90)
    y  = proj_2(p1 * c1) + a                     gate multiply, GEMM                         (van.py:91,109-110)
    x  = x + drop_path(ls1 * y)                  layer-scale residual kernel                 (van.py:183)
    m  = BN2(x);  x = x + drop_path(ls2 * fc2(relu(dw3x3(fc1(m)))))                          (van.py:38-56,184)
Stages: OverlapPatchEmbed (7x7/4 or 3x3/2 conv with bias + BN, van.py:189-208) -> blocks -> BN (norm_i);
head: global average pool + Linear.  dtype flow = the reference under autocast: bf16 GEMM / depthwise
operands and outputs, fp32 statistics, parameters and residual stream (the fp32 layer-scale parameter
promotes the stream to fp32 after the first block of every stage).
"""
import torch

from .. import ops
from .convnet import FcHeadRT, GradSink
from .operands import CONV, STEM, Linear, Operand


def _bn_forward(bn, x, training, out_f32, tape):
    """x: [..., C] bf16 or fp32 -> BN(x) in bf16 / fp32; keeps what the backward needs in `tape`."""
    c = x.shape[-1]
    rows = x.numel() // c
    ss = torch.empty(2, c, device=x.device)
    if training or not bn.track_running_stats:
        saved = torch.empty(2, c, device=x.device)
        partial, prow = ops.bn_stats_generic(x)
        track = bn.track_running_stats
        momentum = bn.momentum if bn.momentum is not None else 0.1
        ops.bn_finalize(partial, bn.weight.detach(), bn.bias.detach(), bn.running_mean if track else None,
                        bn.running_var if track else None, ss, saved, rows, bn.eps, momentum, partial_rows=prow)
        if track and bn.num_batches_tracked is not None:
            bn.num_batches_tracked.add_(1)
        tape['saved'] = saved
    else:
        scale = bn.weight.detach() * torch.rsqrt(bn.running_var + bn.eps)
        ss[0].copy_(scale)
        ss[1].copy_(bn.bias.detach() - bn.running_mean * scale)
    tape['x'] = x
    return ops.bn_apply_generic(x, ss, out_f32)


def _bn_backward(bn, g, tape, sink, dres=None, dx_f32=True):
    gbuf, gacc = sink.begin(bn.weight)
    bbuf, bacc = sink.begin(bn.bias)
    assert gacc == bacc
    dx = ops.bn_bwd_generic(tape['x'], g, tape['saved'], bn.weight.detach(), gbuf, bbuf, dres=dres, dx_f32=dx_f32, accumulate=gacc)
    sink.done(bn.weight, gbuf)
    sink.done(bn.bias, bbuf)
    return dx


class _DW:
    """One depthwise conv (weight [C, 1, k, k], bias [C]) on NHWC bf16."""

    def __init__(self, conv):
        self.conv = conv
        self.k = conv.kernel_size[0]
        self.dil = conv.dilation[0]
        assert conv.groups == conv.in_channels == conv.out_channels and conv.stride == (1, 1)
        assert conv.padding[0] == self.dil * (self.k - 1) // 2

    def fwd(self, x, relu=False):
        return ops.dwconv_fwd(x, self.conv.weight.detach(), self.conv.bias.detach(), self.k, self.dil, relu=relu)

    def bwd(self, dy, x, sink):
        """dy: gradient w.r.t. the conv output (pre-ReLU), x: the conv input.  Returns dx."""
        w, b = self.conv.weight, self.conv.bias
        wbuf, wacc = sink.begin(w)
        ops.dwconv_wgrad(dy, x, wbuf, self.k, self.dil, accumulate=wacc)
        sink.done(w, wbuf)
        bbuf, bacc = sink.begin(b)
        ops.colsum(dy.view(-1, dy.shape[-1]), bbuf, accumulate=bacc)
        sink.done(b, bbuf)
        return ops.dwconv_fwd(dy, w.detach(), None, self.k, self.dil, flip=True)


class _Block:

    def __init__(self, blk):
        self.blk = blk
        at, lka, mlp = blk.attn, blk.attn.spatial_gating_unit, blk.mlp
        self.proj1, self.proj2, self.conv1 = Linear(at.proj_1), Linear(at.proj_2), Linear(lka.conv1)
        self.conv0, self.conv_sp = _DW(lka.conv0), _DW(lka.conv_spatial)
        self.fc1, self.fc2, self.dw = Linear(mlp.fc1), Linear(mlp.fc2), _DW(mlp.dwconv.dwconv)
        self.drop_path = getattr(blk.drop_path, 'drop_path_prob', 0.)
        if getattr(mlp.drop, 'p', 0.) > 0.:
            raise NotImplementedError('VAN dropout_prob > 0 is not implemented by the H100 runtime (0 in every shipped config)')

    def linears(self):
        return [self.proj1, self.proj2, self.conv1, self.fc1, self.fc2]

    def _path_scale(self, n, training, dev):
        if not training or self.drop_path == 0.:
            return None
        keep = 1. - self.drop_path
        s = torch.empty(n, device=dev).bernoulli_(keep)
        if keep > 0.:
            s.div_(keep)
        return s

    def forward(self, x, t, shape, training):
        """x: stream [rows, C] (bf16 for the first block of a stage, fp32 afterwards) -> fp32 [rows, C]."""
        n, h, w, c = shape
        blk = self.blk
        t['bn1'], t['bn2'] = {}, {}
        a = t['a'] = _bn_forward(blk.norm1, x, training, False, t['bn1'])
        p1 = t['p1'] = self.proj1.fwd_flags(a, ops.EPI_RELU)
        c0 = t['c0'] = self.conv0.fwd(p1.view(n, h, w, c))
        cs = t['cs'] = self.conv_sp.fwd(c0)
        c1 = t['c1'] = self.conv1.fwd(cs.view(-1, c))
        g = t['g'] = ops.mul_bf16(p1, c1)
        p2 = t['p2'] = self.proj2.fwd(g)
        s1 = t['s1'] = self._path_scale(n, training, x.device)
        ls1 = blk.layer_scale_1.detach().view(-1)
        x1 = t['x1'] = ops.ls_residual_fwd(x, p2, a, ls1, s1, h * w)
        m = t['m'] = _bn_forward(blk.norm2, x1, training, False, t['bn2'])
        f1 = t['f1'] = self.fc1.fwd(m)
        hid = f1.shape[1]
        d = t['d'] = self.dw.fwd(f1.view(n, h, w, hid), relu=True)
        f2 = t['f2'] = self.fc2.fwd(d.view(-1, hid))
        s2 = t['s2'] = self._path_scale(n, training, x.device)
        return ops.ls_residual_fwd(x1, f2, None, blk.layer_scale_2.detach().view(-1), s2, h * w)

    def backward(self, dx2, t, shape, sink, dx_f32=True):
        """dx2 fp32: gradient w.r.t. the block output.  Returns the gradient w.r.t. the block input
        (fp32, or bf16 when the input stream was the bf16 patch-embedding output)."""
        n, h, w, c = shape
        blk = self.blk
        hw = h * w
        # ---- MLP branch
        lbuf, lacc = sink.begin(blk.layer_scale_2)
        df2 = ops.ls_residual_bwd(dx2, t['f2'], None, blk.layer_scale_2.detach().view(-1), lbuf.view(-1), accumulate=lacc,
                                  row_scale=t['s2'], rows_per_scale=hw)
        sink.done(blk.layer_scale_2, lbuf)
        hid = t['f1'].shape[1]
        dpre = self.fc2.bwd(df2, t['d'].view(-1, hid), sink, relu_out=t['d'].view(-1, hid))     # masked by relu'(d)
        df1 = self.dw.bwd(dpre.view(n, h, w, hid), t['f1'].view(n, h, w, hid), sink)
        dm = self.fc1.bwd(df1.view(-1, hid), t['m'], sink)
        dx1 = _bn_backward(blk.norm2, dm, t['bn2'], sink, dres=dx2)
        # ---- attention branch
        lbuf, lacc = sink.begin(blk.layer_scale_1)
        dy = ops.ls_residual_bwd(dx1, t['p2'], t['a'], blk.layer_scale_1.detach().view(-1), lbuf.view(-1), accumulate=lacc,
                                 row_scale=t['s1'], rows_per_scale=hw)
        sink.done(blk.layer_scale_1, lbuf)
        dg = self.proj2.bwd(dy, t['g'], sink)
        dc1 = ops.mul_bf16(dg, t['p1'])
        dcs = self.conv1.bwd(dc1, t['cs'].view(-1, c), sink)
        dc0 = self.conv_sp.bwd(dcs.view(n, h, w, c), t['c0'], sink)
        dlk = self.conv0.bwd(dc0, t['p1'].view(n, h, w, c), sink)
        dp1 = ops.gate_bwd(dg, t['c1'], dlk.view(-1, c), t['p1'])
        da = self.proj1.bwd(dp1, t['a'], sink, add=dy)                     # + the shortcut's gradient (y = p2 + a)
        return _bn_backward(blk.norm1, da, t['bn1'], sink, dres=dx1, dx_f32=dx_f32)


class StridedConv:
    """Square strided conv with bias as explicit im2col + one GEMM: from the NCHW fp32 image (stem im2col, STEM operand)
    when the input has fewer than 8 channels, else from NHWC bf16 (im2col_nhwc, CONV operand; col2im in the backward)."""

    def __init__(self, conv):
        self.conv = conv
        self.k, self.stride, self.pad = conv.kernel_size[0], conv.stride[0], conv.padding[0]
        self.from_image = conv.in_channels % 8 != 0
        self.op = Operand(conv.weight, STEM if self.from_image else CONV)
        self.kpad = self.op.kpad

    def prep(self):
        self.op.refresh()

    def forward(self, x, t):
        """x: NCHW fp32 image or NHWC bf16 -> (bf16 [rows, C], (n, P, Q, C))."""
        if self.from_image:
            n, _, h, w = x.shape
            cols = ops.stem_im2col(x, self.k, self.k, self.stride, self.pad, self.kpad)
            P, Q = ops.conv_out_size(h, self.pad, self.k, self.stride), ops.conv_out_size(w, self.pad, self.k, self.stride)
        else:
            n, h, w, _ = x.shape
            cols, P, Q = ops.im2col_nhwc(x, self.k, self.stride, self.pad)
        t['cols'], t['in_shape'] = cols, tuple(x.shape)
        y = ops.linear_fwd(cols, self.op.w, bias=self.conv.bias.detach())
        return y, (n, P, Q, self.conv.out_channels)

    def backward(self, dy, t, sink):
        """dy: bf16 gradient [rows, C] w.r.t. the conv output.  Returns the NHWC bf16 input gradient (None for an image)."""
        w, b = self.conv.weight, self.conv.bias
        wbuf, wacc = sink.begin(w)
        part = ops.linear_wgrad(dy, t['cols'])
        ops.finish_conv_wgrad(part, wbuf, self.kpad, accumulate=wacc, order=ops.ORDER_CRS if self.from_image else ops.ORDER_RSC)
        sink.done(w, wbuf)
        bbuf, bacc = sink.begin(b)
        ops.colsum(dy, bbuf, accumulate=bacc)
        sink.done(b, bbuf)
        if self.from_image:
            return None
        n, h, ww, c = t['in_shape']
        dcols = ops.linear_dgrad(dy, self.op.w)
        return ops.col2im_nhwc(dcols, n, h, ww, c, self.k, self.stride, self.pad)


class _PatchEmbed:
    """OverlapPatchEmbed (van.py:189-208): conv (with bias) -> BatchNorm; output = the stage's bf16 stream input."""

    def __init__(self, pe):
        self.conv, self.bn = StridedConv(pe.proj), pe.norm
        self.op = self.conv.op

    def prep(self):
        self.conv.prep()

    def forward(self, x, t, training):
        """x: NCHW fp32 image (stage 1) or NHWC bf16 -> (bf16 stream [rows, C], (n, P, Q, C))."""
        t['bn'] = {}
        y, shape = self.conv.forward(x, t)
        return _bn_forward(self.bn, y, training, False, t['bn']), shape

    def backward(self, dout, t, sink):
        """dout: gradient w.r.t. the BN output (bf16 or fp32 [rows, C]).  Returns the NHWC bf16 input gradient
        (None for the image stage)."""
        return self.conv.backward(_bn_backward(self.bn, dout, t['bn'], sink, dx_f32=False), t, sink)


class VANRT:
    """Whole-network runtime (van.py:289-310)."""

    def __init__(self, model):
        self.model = model
        self.stages = []
        for i in range(len(model.block_nums)):
            pe = _PatchEmbed(getattr(model, f'patch_embed{i + 1}'))
            blocks = [_Block(b) for b in getattr(model, f'block{i + 1}')]
            self.stages.append((pe, blocks, getattr(model, f'norm{i + 1}')))
        self.head = FcHeadRT(model.head)
        self.sink = GradSink()
        self._units = [u for pe, blocks, _ in self.stages for u in [pe] + [lin for b in blocks for lin in b.linears()]] + [self.head]

    def operands(self):
        return [u.op for u in self._units]

    def prep(self):
        for u in self._units:
            u.prep()

    # stage-level entry points (also driven by the teacher-forced parity tests)
    def stage_forward(self, i, x, t, training):
        pe, blocks, norm = self.stages[i]
        t['pe'], t['blocks'], t['norm'] = {}, [dict() for _ in blocks], {}
        s, shape = pe.forward(x, t['pe'], training)
        t['shape'] = shape
        for b, bt in zip(blocks, t['blocks']):
            s = b.forward(s, bt, shape, training)
        out = _bn_forward(norm, s, training, False, t['norm'])
        return out.view(*shape)

    def stage_backward(self, i, dout, t):
        pe, blocks, norm = self.stages[i]
        shape = t['shape']
        d = _bn_backward(norm, dout.reshape(-1, shape[3]), t['norm'], self.sink, dx_f32=True)
        for j in range(len(blocks) - 1, -1, -1):
            d = blocks[j].backward(d, t['blocks'][j], shape, self.sink, dx_f32=(j > 0))
        return pe.backward(d, t['pe'], self.sink)

    def forward(self, x, training, keep_tape):
        assert x.is_cuda and x.dtype == torch.float32 and x.dim() == 4
        self.prep()
        tape = {'stages': [dict() for _ in self.stages], 'head': {}}
        a = x.contiguous()
        for i, t in enumerate(tape['stages']):
            a = self.stage_forward(i, a, t, training)
        tape['head']['feat_c'] = a.shape[3]
        logits = self.head.forward(a, tape['head'])
        return logits, (tape if keep_tape else None)

    def backward(self, dlogits, tape):
        assert tape is not None, 'backward called without a training forward'
        d = self.head.backward(dlogits, tape['head'], self.sink, tape['head']['feat_c'])
        for i in range(len(self.stages) - 1, -1, -1):
            d = self.stage_backward(i, d, tape['stages'][i])
        if self.sink.on_backward_end is not None:
            self.sink.on_backward_end()
