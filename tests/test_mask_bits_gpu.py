"""The 1-bit ReLU mask of residual-block outputs, bit for bit against the paths it replaces.

bn_apply packs (out > 0); the data-gradient GEMM applies it after the shortcut add; the BatchNorm backward kernels read
it instead of the block output, alone or for the bn3 + downsample pair in one pass.  Every one of these keeps the
arithmetic and the summation order, so the comparisons are exact (bf16 compared as raw bits, signed zeros included).
Shapes are ResNet-50's channel counts with row counts that are not multiples of 128."""
import pytest
import torch

pytestmark = pytest.mark.gpu


def _ops():
    from simpleaicv_pytorch_training_examples_b200 import ops
    return ops


def _bf(*shape, seed=0, scale=1.0, shift=0.0):
    g = torch.Generator(device='cuda').manual_seed(seed)
    return (torch.randn(*shape, device='cuda', generator=g) * scale + shift).to(torch.bfloat16)


def _same(a, b, what):
    if a.dtype == torch.bfloat16:
        a, b = a.view(torch.int16), b.view(torch.int16)
    elif a.dtype == torch.float32:
        a, b = a.view(torch.int32), b.view(torch.int32)
    bad = (a != b).sum().item()
    assert bad == 0, f'{what}: {bad} of {a.numel()} elements differ'


def _unpack(bits, c):
    b = bits.view(torch.uint8).long()   # little-endian: byte k of a word holds channels 8k .. 8k+7 of it
    shifts = torch.arange(8, device=b.device)
    return ((b.unsqueeze(-1) >> shifts) & 1).reshape(b.shape[0], c).bool()


def _bn_coefs(ops, y, seed):
    c = y.shape[-1]
    g = torch.Generator(device='cuda').manual_seed(seed)
    gamma = torch.rand(c, device='cuda', generator=g) + 0.5
    beta = torch.randn(c, device='cuda', generator=g)
    ss, saved = torch.empty(2, c, device='cuda'), torch.empty(2, c, device='cuda')
    ops.bn_finalize(ops.bn_stats(y), gamma, beta, None, None, ss, saved, y.shape[0], 1e-5, 0.1)
    return gamma, ss, saved


def _block_output(ops, rows, c):
    """bn3(y3) + bn_d(yd) -> ReLU, as in a downsample block; returns the pieces and the packed mask."""
    y3 = _bf(rows, c, seed=1, scale=2.0, shift=0.3)
    yd = _bf(rows, c, seed=2, scale=1.5, shift=-0.2)
    gamma3, ss3, saved3 = _bn_coefs(ops, y3, 3)
    gammad, ssd, savedd = _bn_coefs(ops, yd, 4)
    out = torch.empty_like(y3)
    bits = ops.mask_bits_like(y3)
    ops.bn_apply(y3, ss3, out, 1, res=yd, res_scale_shift=ssd, mask_bits=bits)
    return y3, yd, (gamma3, ss3, saved3), (gammad, ssd, savedd), out, bits


@pytest.mark.parametrize('rows,c', [(3000, 256), (1000, 512), (392, 1024), (98, 2048)])
def test_bn_apply_mask_bits_are_out_positive(rows, c):
    ops = _ops()
    y3, yd, (_, ss3, _), (_, ssd, _), out, bits = _block_output(ops, rows, c)
    assert bits.shape == (rows, c // 32)
    assert torch.equal(_unpack(bits, c), out.float() > 0)
    ref = torch.empty_like(out)
    ops.bn_apply(y3, ss3, ref, 1, res=yd, res_scale_shift=ssd)
    _same(out, ref, 'bn_apply output with / without the mask')
    # identity block: residual without BatchNorm
    out2, bits2 = torch.empty_like(y3), ops.mask_bits_like(y3)
    ops.bn_apply(y3, ss3, out2, 1, res=yd, mask_bits=bits2)
    assert torch.equal(_unpack(bits2, c), out2.float() > 0)


@pytest.mark.parametrize('n,h,w,c,k,r,pad', [(3, 56, 56, 256, 64, 1, 0), (2, 28, 28, 512, 128, 1, 0),
                                              (2, 14, 14, 1024, 256, 1, 0), (2, 7, 7, 2048, 512, 1, 0),
                                              (2, 14, 14, 256, 256, 3, 1)])
def test_conv_dgrad_mask_bits_equals_masking_the_sum(n, h, w, c, k, r, pad):
    ops = _ops()
    dy = _bf(n, h, w, k, seed=5)
    wt = _bf(k, r * r * c, seed=6, scale=0.05)
    add = _bf(n, h, w, c, seed=7)
    rows = n * h * w
    ya = _bf(rows, c, seed=8, shift=0.1)
    _, ss, _ = _bn_coefs(ops, ya, 9)
    act_out, bits = torch.empty_like(ya), ops.mask_bits_like(ya)
    ops.bn_apply(ya, ss, act_out, 1, res=_bf(rows, c, seed=10), mask_bits=bits)
    cs = ops.make_conv_shape(n, h, w, c, k, r, r, 1, pad)
    got = ops.conv_dgrad(dy, wt, cs, add=add, mask_bits=bits)
    ref = ops.conv_dgrad(dy, wt, cs, add=add)
    ref = (ref.float() * (act_out.view(n, h, w, c).float() > 0).float()).to(torch.bfloat16)   # what bn_bwd's act_grad did
    _same(got, ref, 'conv_dgrad(add, mask_bits)')


def _partials(ops, width, fn):
    """Runs fn and returns the partial rows it wrote into the shared workspace (pre-filled with NaN)."""
    ws = ops.partial_ws(torch.device('cuda', torch.cuda.current_device()), width)
    ws.fill_(float('nan'))
    fn()
    p = ws.view(-1, width)
    return p[~torch.isnan(p[:, 0])].clone()


@pytest.mark.parametrize('rows,c', [(3000, 256), (1000, 512), (392, 1024), (98, 2048)])
def test_bits_and_two_bn_backward_equal_out_mode(rows, c):
    ops = _ops()
    y3, yd, (gamma3, ss3, saved3), (gammad, ssd, savedd), out, bits = _block_output(ops, rows, c)
    dout = _bf(rows, c, seed=11)
    e = lambda: torch.empty(c, device='cuda')

    def single(g, y, saved, gamma, mask_out, mask_bits, act, want_dres):
        sums = torch.zeros(2, c, device='cuda')
        part = _partials(ops, 2 * c, lambda: ops.bn_bwd_reduce(g, mask_out, y, saved, sums, act, bits=mask_bits))
        dy, dres, dg, db = torch.empty_like(y), (torch.empty_like(y) if want_dres else None), e(), e()
        ops.bn_bwd_apply(g, mask_out, y, saved, gamma, sums, dy, dres, dg, db, act, bits=mask_bits)
        return part, sums, dy, dres, dg, db

    ref3 = single(dout, y3, saved3, gamma3, out, None, 1, True)
    refd = single(dout, yd, savedd, gammad, out, None, 1, False)
    names = ('partials', 'sums', 'dy', 'dres', 'dgamma', 'dbeta')
    for nm, a, b in zip(names, single(dout, y3, saved3, gamma3, None, bits, 1, True), ref3):
        _same(a, b, f'bits mode {nm}')
    # the gradient arriving already masked (dres of the out-mode call): no mask in the BatchNorm kernels
    g = ref3[3]
    for nm, a, b in zip(names, single(g, y3, saved3, gamma3, None, None, 0, False), ref3):
        if b is not None and nm != 'dres':
            _same(a, b, f'masked input {nm}')

    for mask_bits, gin in ((bits, dout), (None, g)):
        sums = torch.empty(4, c, device='cuda')
        part = _partials(ops, 4 * c, lambda: ops.bn_bwd_reduce2(gin, mask_bits, y3, yd, saved3, savedd, sums))
        what = 'two-BN ' + ('bits' if mask_bits is not None else 'masked input')
        _same(part[:, :2 * c], ref3[0], f'{what} partials A')
        _same(part[:, 2 * c:], refd[0], f'{what} partials B')
        _same(sums[:2], ref3[1], f'{what} sums A')
        _same(sums[2:], refd[1], f'{what} sums B')
        dya, dyb, dga, dba, dgb, dbb = torch.empty_like(y3), torch.empty_like(yd), e(), e(), e(), e()
        ops.bn_bwd_apply2(gin, mask_bits, y3, yd, saved3, savedd, gamma3, gammad, sums, dya, dyb, dga, dba, dgb, dbb)
        for nm, a, b in (('dy A', dya, ref3[2]), ('dgamma A', dga, ref3[4]), ('dbeta A', dba, ref3[5]),
                         ('dy B', dyb, refd[2]), ('dgamma B', dgb, refd[4]), ('dbeta B', dbb, refd[5])):
            _same(a, b, f'{what} {nm}')


def test_resnet50_block_chain_matches_per_block_backward():
    """ResNet-50's 16 blocks at batch 2, 72 px (rows 648 / 162 / 50 / 18): the chained backward, where each block hands
    the previous one its gradient already masked, with and without gradient checkpointing, equals running every block's
    backward on its own (each masks its own gradient from its bits), bit for bit: input gradient and every parameter
    gradient."""
    from simpleaicv_pytorch_training_examples_b200.classification import backbones
    from simpleaicv_pytorch_training_examples_b200.engine.convnet import blocks_backward
    torch.manual_seed(0)
    model = backbones.resnet50(num_classes=10).cuda().train()
    rt = model._runtime()
    rt.prep()
    x = torch.randn(2, 3, 72, 72, generator=torch.Generator().manual_seed(1)).cuda()
    a0 = rt.stem_forward(x, {'stem': {}}, True)
    params = [p for b in rt.blocks for u in b.all_units() for p in (u.conv.weight, u.bn.weight, u.bn.bias)]

    def run(mode):
        model.zero_grad(set_to_none=True)
        tapes = [dict() for _ in rt.blocks]
        a = a0
        for b, t in zip(rt.blocks, tapes):
            if mode == 'ckpt':
                t['ckpt_in'] = a
                a = b.forward(a, {}, True)
            else:
                a = b.forward(a, t, True)
        da = _bf(*a.shape, seed=12, scale=1e-2)
        if mode == 'per_block':
            for b, t in zip(reversed(rt.blocks), reversed(tapes)):
                da = b.backward(da, t, rt.sink)
        else:
            da = blocks_backward(rt.blocks, tapes, da, rt.sink)
        torch.cuda.synchronize()
        return da.clone(), [p.grad.clone() for p in params]

    ref_dx, ref_g = run('per_block')
    for mode in ('chain', 'ckpt'):
        dx, gr = run(mode)
        _same(dx, ref_dx, f'{mode}: input gradient')
        for i, (a, b) in enumerate(zip(gr, ref_g)):
            _same(a, b, f'{mode}: parameter gradient {i}')
