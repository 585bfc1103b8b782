"""Forward/backward runtime of the ConvFormer classifiers (SimpleAICV/classification/backbones/convformer.py) on
libsaicv_b200.so.

Per MetaFormerBlock (convformer.py:142-166), stream x [rows, C] NHWC (rows = N*H*W):
    n1 = BN1(x)                                   bf16  generic BatchNorm over the bf16 / fp32 stream   (:146,162-163)
    r1 = relu(pwconv1(n1))                              GEMM, ReLU in the epilogue                       (:53-54,65-66)
    dd = dw7x7(r1)                                      depthwise kernel, no bias                         (:55-60,70)
    x  = x + drop_path(pwconv2(dd))                     GEMM, residual + drop-path row scale in the epilogue (:62,75,162-163)
    r2 = relu(fc1(BN2(x)));  x = x + drop_path(fc2(r2))                                                    (:82-103,164)
Backward of dw7x7(relu(h)): one depthwise data-gradient kernel that also applies the ReLU mask (r1 > 0).
Downsampling (:16-44, :186-208): stem = 7x7/4 conv with bias (stem im2col + GEMM) -> BN; stages 2-4 = BN of the stream ->
3x3/2 conv with bias (im2col + GEMM).  Head (:228-229,251-254): global average pool of the stream (fp32 sum, one bf16
write) -> Linear.

dtype flow = the reference under autocast(bf16): conv / Linear / depthwise outputs are bf16, BatchNorm returns its input's
dtype, and DropPathBlock multiplies by an fp32 [B,1,1,1] mask (:131-137), so ``x + drop_path(branch)`` is fp32.  In
training the stream is therefore bf16 from each downsampling output up to the first block of the stage with
drop_path_prob > 0 and fp32 from there on; in eval mode, or with drop_path_prob = 0, it stays bf16 and every residual
sum is rounded to bf16 (GEMM branch, then add_bf16).  At the switch the block input is cast to fp32 once (exact: the
BatchNorm statistics and outputs are those of the bf16 input).  Stream GRADIENTS are kept fp32 everywhere; the GEMMs read
them as bf16(drop-path scale * gradient).

use_gradient_checkpoint (:240-249): the tape keeps only each downsampling layer's and each stage's input and the
drop-path scales drawn in the forward; the backward replays a layer's forward with those scales (the effect of torch's
preserve_rng_state) before differentiating it.  Like torch.utils.checkpoint in the reference, the replay runs in training
mode, so every BatchNorm receives a second running-statistics momentum update (and num_batches_tracked += 1) per step.
"""
import torch

from .. import ops
from .convnet import FcHeadRT, GradSink
from .operands import Linear
from .van import StridedConv, _bn_backward, _bn_forward


def _bf16_scaled(d, scale, rows_per_scale):
    """bf16(scale[row // rows_per_scale] * d) for d fp32 [rows, C]: the gradient a branch GEMM reads (the dropout kernel
    at p = 0 keeps every element and applies only the row scale)."""
    if scale is None:
        return ops.cast_bf16(d)
    return ops.dropout(d, 0.0, 0, row_scale=scale, elems_per_scale=rows_per_scale * d.shape[-1], out_f32=False)


def _to_f32(x):
    """Exact bf16 -> fp32 copy (dropout kernel at p = 0 without a row scale)."""
    return x if x.dtype == torch.float32 else ops.dropout(x, 0.0, 0, out_f32=True)


class _Block:
    """MetaFormerBlock with SepConv token mixer and Mlp (convformer.py:47-103,142-166)."""

    def __init__(self, blk):
        self.blk = blk
        tm, mlp = blk.token_mixer, blk.mlp
        self.pw1, self.pw2, self.fc1, self.fc2 = Linear(tm.pwconv1), Linear(tm.pwconv2), Linear(mlp.fc1), Linear(mlp.fc2)
        self.dw = tm.dwconv
        assert self.dw.kernel_size == (7, 7) and self.dw.padding == (3, 3) and self.dw.dilation == (1, 1) and self.dw.bias is None
        self.drop_path = getattr(blk.drop_path, 'drop_path_prob', 0.)
        assert mlp.drop1.p == 0. and mlp.drop2.p == 0., 'dropout_prob > 0 is rejected by the model constructor'

    def linears(self):
        return [self.pw1, self.pw2, self.fc1, self.fc2]

    def draw_scales(self, n, training, dev):
        """The two per-sample drop-path scales (token mixer, then MLP), drawn on the device in the reference's order
        (convformer.py:131-135: bernoulli_(keep) / keep), or (None, None) when drop path is off."""
        if not training or self.drop_path == 0.:
            return None, None
        keep = 1. - self.drop_path
        out = []
        for _ in range(2):
            s = torch.empty(n, device=dev).bernoulli_(keep)
            if keep > 0.:
                s.div_(keep)
            out.append(s)
        return tuple(out)

    def _residual(self, lin, x, h, scale, hw):
        """x + scale * lin(h): fp32 in the GEMM epilogue on an fp32 stream, else bf16(x + bf16(lin(h)))."""
        if x.dtype == torch.float32:
            return lin.fwd(h, resid=x, out_f32=True, row_scale=scale, rows_per_scale=hw if scale is not None else 0)
        assert scale is None
        return ops.add_bf16(lin.fwd(h), x)

    def forward(self, x, t, shape, training, scales=None):
        """x: stream [rows, C] (bf16 or fp32) -> stream [rows, C] (fp32 once a drop path has been applied)."""
        n, h, w, c = shape
        hw = h * w
        s1, s2 = scales if scales is not None else self.draw_scales(n, training, x.device)
        t['s1'], t['s2'] = s1, s2
        if s1 is not None:
            x = _to_f32(x)
        t['bn1'], t['bn2'] = {}, {}
        n1 = t['n1'] = _bn_forward(self.blk.norm1, x, training, False, t['bn1'])
        r1 = t['r1'] = self.pw1.fwd_flags(n1, ops.EPI_RELU)
        dd = t['dd'] = ops.dwconv_fwd(r1.view(n, h, w, 2 * c), self.dw.weight.detach(), None, 7, 1).view(-1, 2 * c)
        x1 = self._residual(self.pw2, x, dd, s1, hw)
        n2 = t['n2'] = _bn_forward(self.blk.norm2, x1, training, False, t['bn2'])
        r2 = t['r2'] = self.fc1.fwd_flags(n2, ops.EPI_RELU)
        return self._residual(self.fc2, x1, r2, s2, hw)

    def backward(self, dx2, t, shape, sink):
        """dx2 fp32 [rows, C]: gradient w.r.t. the block output.  Returns the fp32 gradient w.r.t. the block input."""
        n, h, w, c = shape
        hw = h * w
        dr2 = self.fc2.bwd(_bf16_scaled(dx2, t['s2'], hw), t['r2'], sink, relu_out=t['r2'])
        dn2 = self.fc1.bwd(dr2, t['n2'], sink)
        dx1 = _bn_backward(self.blk.norm2, dn2, t['bn2'], sink, dres=dx2)
        ddd = self.pw2.bwd(_bf16_scaled(dx1, t['s1'], hw), t['dd'], sink).view(n, h, w, 2 * c)
        r1 = t['r1'].view(n, h, w, 2 * c)
        wbuf, wacc = sink.begin(self.dw.weight)
        ops.dwconv_wgrad(ddd, r1, wbuf, 7, 1, accumulate=wacc)
        sink.done(self.dw.weight, wbuf)
        dh = ops.dwconv_dgrad_masked(ddd, self.dw.weight.detach(), r1, 7)        # * relu'(pwconv1 output)
        dn1 = self.pw1.bwd(dh.view(-1, 2 * c), t['n1'], sink)
        return _bn_backward(self.blk.norm1, dn1, t['bn1'], sink, dres=dx1)


class _Downsampling:
    """Downsampling (convformer.py:16-44): [pre BN of the stream] -> strided conv with bias -> [post BN]; the output is
    the next stage's bf16 stream."""

    def __init__(self, ds):
        self.pre = ds.pre_norm if isinstance(ds.pre_norm, torch.nn.BatchNorm2d) else None
        self.post = ds.post_norm if isinstance(ds.post_norm, torch.nn.BatchNorm2d) else None
        self.conv = StridedConv(ds.conv)
        self.op = self.conv.op

    def prep(self):
        self.conv.prep()

    def forward(self, x, shape, t, training):
        """x: NCHW fp32 image (stem, shape None) or stream [rows, C] with its (n, h, w, c) -> (bf16 [rows', C'], shape')."""
        if self.pre is not None:
            t['pre'] = {}
            x = _bn_forward(self.pre, x, training, False, t['pre']).view(*shape)
        y, shape = self.conv.forward(x, t)
        if self.post is not None:
            t['post'] = {}
            y = _bn_forward(self.post, y, training, False, t['post'])
        return y, shape

    def backward(self, dy, t, sink):
        """dy fp32 [rows', C']: returns the fp32 stream gradient [rows, C] (None for the stem)."""
        if self.post is not None:
            g = _bn_backward(self.post, dy, t['post'], sink, dx_f32=False)
        else:
            g = ops.cast_bf16(dy)
        dx = self.conv.backward(g, t, sink)
        if self.pre is None:
            return None
        return _bn_backward(self.pre, dx.view(-1, dx.shape[-1]), t['pre'], sink, dx_f32=True)


class _Head(FcHeadRT):
    """AdaptiveAvgPool2d of the bf16 / fp32 stream -> Linear with bias (convformer.py:228-229,251-254)."""

    def forward(self, s, shape, tape):
        tape['shape'] = shape
        return self.fc_forward(ops.avgpool_stream_fwd(s.view(*shape)), tape)

    def backward(self, dlogits, tape, sink):
        """Returns the fp32 gradient w.r.t. the stream [rows, C]."""
        n, h, w, c = tape['shape']
        return ops.avgpool_stream_bwd(self.fc_backward(dlogits, tape, sink), h, w).view(-1, c)


class ConvFormerRT:
    """Whole-network runtime (convformer.py:169-256)."""

    def __init__(self, model):
        self.model = model
        self.downs = [_Downsampling(d) for d in model.downsample_layers]
        self.stages = [[_Block(b) for b in stage] for stage in model.stages]
        self.head = _Head(model.head)
        self.sink = GradSink()
        self._units = [u for d, blocks in zip(self.downs, self.stages) for u in [d] + [lin for b in blocks for lin in b.linears()]]
        self._units.append(self.head)

    def operands(self):
        return [u.op for u in self._units]

    def prep(self):
        for u in self._units:
            u.prep()

    # layer-level entry points (also driven by the teacher-forced parity tests); stream tensors are [rows, C]
    def stem_forward(self, x, t, training):
        return self.downs[0].forward(x, None, t, training)

    def stem_backward(self, d, t):
        self.downs[0].backward(d, t, self.sink)

    def down_forward(self, i, s, shape, t, training):
        return self.downs[i].forward(s, shape, t, training)

    def down_backward(self, i, d, t):
        return self.downs[i].backward(d, t, self.sink)

    def stage_forward(self, i, s, shape, t, training, scales=None):
        """scales: per-block (s1, s2) drop-path scales to use instead of drawing new ones (checkpoint replay, tests)."""
        t['shape'], t['blocks'] = shape, [dict() for _ in self.stages[i]]
        for j, (b, bt) in enumerate(zip(self.stages[i], t['blocks'])):
            s = b.forward(s, bt, shape, training, None if scales is None else scales[j])
        return s

    def stage_backward(self, i, d, t):
        for j in range(len(self.stages[i]) - 1, -1, -1):
            d = self.stages[i][j].backward(d, t['blocks'][j], t['shape'], self.sink)
        return d

    @staticmethod
    def stage_scales(t):
        return [(bt['s1'], bt['s2']) for bt in t['blocks']]

    def forward(self, x, training, keep_tape):
        assert x.is_cuda and x.dtype == torch.float32 and x.dim() == 4
        self.prep()
        ckpt = self.model.use_gradient_checkpoint and keep_tape
        tape = {'downs': [], 'stages': [], 'head': {}}
        s, shape = x.contiguous(), None
        for i in range(len(self.stages)):
            t = {}
            if ckpt:
                tape['downs'].append({'in': s, 'in_shape': shape})
            s, shape = self.down_forward(i, s, shape, t, training)
            if not ckpt:
                tape['downs'].append(t)
            t = {}
            s_in = s
            s = self.stage_forward(i, s, shape, t, training)
            tape['stages'].append({'in': s_in, 'shape': shape, 'scales': self.stage_scales(t)} if ckpt else t)
        logits = self.head.forward(s, shape, tape['head'])
        return logits, (tape if keep_tape else None)

    def backward(self, dlogits, tape):
        assert tape is not None, 'backward called without a training forward'
        d = self.head.backward(dlogits, tape['head'], self.sink)
        for i in range(len(self.stages) - 1, -1, -1):
            t = tape['stages'][i]
            if 'in' in t:                                   # checkpointed: replay with the forward's drop-path scales
                ck, t = t, {}
                self.stage_forward(i, ck['in'], ck['shape'], t, True, scales=ck['scales'])
            d = self.stage_backward(i, d, t)
            tape['stages'][i] = None
            t = tape['downs'][i]
            if 'in' in t:
                ck, t = t, {}
                self.down_forward(i, ck['in'], ck['in_shape'], t, True)
            d = self.down_backward(i, d, t)
            tape['downs'][i] = None
        if self.sink.on_backward_end is not None:
            self.sink.on_backward_end()
