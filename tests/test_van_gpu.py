"""VAN on the H100 runtime vs the CPU oracle (oracle/van.py, pinned to the reference by tests/golden/van_*.pt and
tests/test_oracle_vs_reference.py): kernel-level parity of the depthwise / gating / layer-scale / generic-BN
kernels against plain torch fp32, stage-by-stage parity driven with the oracle's boundary tensors, and an end to
end step.  Layer scales are raised from the 1e-5 initial value to 0.5 in the model-level tests so that the
attention / MLP branches actually contribute to the compared outputs."""
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu


def _rel(a, b):
    return ((a.float().cpu() - b.float().cpu()).norm() / b.float().cpu().norm().clamp_min(1e-12)).item()


def _nhwc(t, dtype=torch.bfloat16):
    return t.detach().permute(0, 2, 3, 1).contiguous().to(dtype).cuda()


@pytest.mark.parametrize('k,dil,c,hw', [(3, 1, 256, 14), (5, 1, 64, 28), (7, 3, 64, 28), (7, 3, 160, 9), (3, 1, 32, 5)])
def test_depthwise_conv_fwd_dgrad_wgrad(k, dil, c, hw):
    from simpleaicv_pytorch_training_examples_b200 import ops
    g = torch.Generator().manual_seed(k * 100 + c)
    x = torch.randn(3, c, hw, hw, generator=g).bfloat16().float()
    w = (torch.randn(c, 1, k, k, generator=g) * 0.2)
    b = torch.randn(c, generator=g) * 0.1
    dy = torch.randn(3, c, hw, hw, generator=g).bfloat16().float()
    xr, wr, br = x.clone().requires_grad_(True), w.clone().requires_grad_(True), b.clone().requires_grad_(True)
    ref = F.conv2d(xr, wr, br, 1, dil * (k - 1) // 2, dil, c)
    ref.backward(dy)
    y = ops.dwconv_fwd(_nhwc(x), w.cuda(), b.cuda(), k, dil)
    assert (y.float().cpu() - ref.detach().permute(0, 2, 3, 1)).abs().max().item() <= 2e-2 * max(1.0, ref.abs().max().item())
    yr = ops.dwconv_fwd(_nhwc(x), w.cuda(), b.cuda(), k, dil, relu=True)
    assert _rel(yr, F.relu(ref.detach()).permute(0, 2, 3, 1)) <= 5e-3
    dx = ops.dwconv_fwd(_nhwc(dy), w.cuda(), None, k, dil, flip=True)
    assert _rel(dx, xr.grad.permute(0, 2, 3, 1)) <= 5e-3
    dw = torch.empty(c, 1, k, k, device='cuda')
    ops.dwconv_wgrad(_nhwc(dy), _nhwc(x), dw, k, dil)
    assert _rel(dw, wr.grad) <= 1e-4
    dw2 = dw.clone()
    ops.dwconv_wgrad(_nhwc(dy), _nhwc(x), dw2, k, dil, accumulate=True)
    assert _rel(dw2, 2 * wr.grad) <= 1e-4


def test_gate_layer_scale_and_generic_bn_kernels():
    from simpleaicv_pytorch_training_examples_b200 import ops
    g = torch.Generator().manual_seed(3)
    rows, c, hw = 6 * 49, 96, 49
    bf = lambda *s: torch.randn(*s, generator=g).bfloat16()
    a, b2, c3, d4 = bf(rows, c), bf(rows, c), bf(rows, c), bf(rows, c)
    assert _rel(ops.mul_bf16(a.cuda(), b2.cuda()), a.float() * b2.float()) <= 4e-3
    want = (a.float() * b2.float() + c3.float()) * (d4.float() > 0)
    assert _rel(ops.gate_bwd(a.cuda(), b2.cuda(), c3.cuda(), d4.cuda()), want) <= 4e-3
    # layer-scale residual, forward and backward, with a drop-path row scale
    x = torch.randn(rows, c, generator=g)
    ls = torch.rand(c, generator=g)
    rs = torch.tensor([0., 1.25, 1.25, 0., 1.25, 1.25])
    out = ops.ls_residual_fwd(x.cuda(), a.cuda(), b2.cuda(), ls.cuda(), rs.cuda(), hw)
    wantf = x + rs.repeat_interleave(hw)[:, None] * ls * (a.float() + b2.float())
    assert _rel(out, wantf) <= 1e-6
    outb = ops.ls_residual_fwd(x.bfloat16().cuda(), a.cuda(), None, ls.cuda())
    assert _rel(outb, x.bfloat16().float() + ls * a.float()) <= 1e-6
    dxn = torch.randn(rows, c, generator=g)
    dls = torch.empty(c, device='cuda')
    dy = ops.ls_residual_bwd(dxn.cuda(), a.cuda(), b2.cuda(), ls.cuda(), dls, row_scale=rs.cuda(), rows_per_scale=hw)
    assert _rel(dy, rs.repeat_interleave(hw)[:, None] * ls * dxn) <= 4e-3
    assert _rel(dls, (rs.repeat_interleave(hw)[:, None] * dxn * (a.float() + b2.float())).sum(0)) <= 1e-5
    # BatchNorm over fp32 / bf16 inputs
    for x_f32, g_f32, dx_f32 in [(True, False, True), (False, True, False), (True, True, True)]:
        xin = torch.randn(rows, c, generator=g) * 2 + 1
        xin = xin if x_f32 else xin.bfloat16()
        gam, bet = torch.rand(c, generator=g) + 0.5, torch.randn(c, generator=g)
        gout = torch.randn(rows, c, generator=g)
        gout = gout if g_f32 else gout.bfloat16()
        dres = torch.randn(rows, c, generator=g)
        xr = xin.float().clone().requires_grad_(True)
        gr, br_ = gam.clone().requires_grad_(True), bet.clone().requires_grad_(True)
        rm, rv = torch.zeros(c), torch.ones(c)
        ref = F.batch_norm(xr, rm, rv, gr, br_, True, 0.1, 1e-5)
        ref.backward(gout.float())
        partial, prow = ops.bn_stats_generic(xin.cuda())
        ss, saved = torch.empty(2, c, device='cuda'), torch.empty(2, c, device='cuda')
        rmc, rvc = torch.zeros(c, device='cuda'), torch.ones(c, device='cuda')
        ops.bn_finalize(partial, gam.cuda(), bet.cuda(), rmc, rvc, ss, saved, rows, 1e-5, 0.1, partial_rows=prow)
        y = ops.bn_apply_generic(xin.cuda(), ss, out_f32=False)
        assert (y.float().cpu() - ref.detach()).abs().max().item() <= 3e-2
        torch.testing.assert_close(rmc.cpu(), rm, rtol=1e-4, atol=1e-5)
        torch.testing.assert_close(rvc.cpu(), rv, rtol=1e-4, atol=1e-5)
        dg, db = torch.empty(c, device='cuda'), torch.empty(c, device='cuda')
        dx = ops.bn_bwd_generic(xin.cuda(), gout.cuda(), saved, gam.cuda(), dg, db, dres=dres.cuda(), dx_f32=dx_f32)
        assert _rel(dx, xr.grad + dres) <= (1e-4 if dx_f32 else 5e-3)
        assert _rel(dg, gr.grad) <= 1e-4 and _rel(db, br_.grad) <= 1e-4


def test_im2col_col2im_nhwc():
    from simpleaicv_pytorch_training_examples_b200 import ops
    g = torch.Generator().manual_seed(8)
    x = torch.randn(2, 32, 9, 9, generator=g).bfloat16().float()
    cols, P, Q = ops.im2col_nhwc(_nhwc(x), 3, 2, 1)
    ref = F.unfold(x, 3, padding=1, stride=2)                       # [n, c*9, P*Q], column order c*9 + tap
    ref = ref.view(2, 32, 9, P * Q).permute(0, 3, 2, 1).reshape(2 * P * Q, 9 * 32)   # -> [rows][tap*C + c]
    assert torch.equal(cols.float().cpu(), ref)
    dcols = torch.randn(2 * P * Q, 9 * 32, generator=g).bfloat16()
    dx = ops.col2im_nhwc(dcols.cuda(), 2, 9, 9, 32, 3, 2, 1)
    want = F.fold(dcols.float().view(2, P * Q, 9, 32).permute(0, 3, 2, 1).reshape(2, 32 * 9, P * Q), (9, 9), 3, padding=1, stride=2)
    assert _rel(dx, want.permute(0, 2, 3, 1)) <= 4e-3


def _setup(arch, shape, nc=10, seed=0, ls=0.5):
    from oracle import van
    from simpleaicv_pytorch_training_examples_b200.classification import backbones
    g = torch.Generator().manual_seed(41)
    x = torch.randn(*shape, generator=g)
    y = torch.randint(0, nc, (shape[0],), generator=g)
    sd = van.init_state(arch, nc, seed)
    torch.manual_seed(seed)
    model = backbones.__dict__[arch](num_classes=nc).cuda().train()
    for k in sd:
        if 'layer_scale' in k:
            sd[k].fill_(ls)
    with torch.no_grad():
        for n, p in model.named_parameters():
            if 'layer_scale' in n:
                p.fill_(ls)
    return van, sd, model, x, y


@pytest.mark.parametrize('arch', ['van_b0', 'van_b1'])
def test_van_step_matches_oracle(arch):
    from simpleaicv_pytorch_training_examples_b200.classification import losses
    van, sd, model, x, y = _setup(arch, (8, 3, 128, 128))
    sd32 = {k: v.clone() for k, v in sd.items()}
    l32, ls32, g32 = van.loss_and_grads(sd32, x, y, arch)
    le, lse, ge = van.loss_and_grads(sd, x, y, arch, emulate_bf16=True)
    logits = model(x.cuda())
    loss = losses.CELoss()(logits, y.cuda())
    loss.backward()
    torch.cuda.synchronize()
    noise = _rel(le, l32)
    assert _rel(logits.detach(), le) <= 2.5 * noise + 1e-2, (_rel(logits.detach(), le), noise)
    assert abs(float(loss.detach()) - float(lse)) <= 1e-2 * abs(float(lse)) + 2.5 * abs(float(lse) - float(ls32))
    grads = {n: p.grad.detach().float().cpu() for n, p in model.named_parameters()}
    assert set(grads) == set(g32)
    cat = lambda d: torch.cat([d[n].flatten() for n in g32])
    mine_all, emu_all = _rel(cat(grads), cat(g32)), _rel(cat(ge), cat(g32))
    assert mine_all <= 2.0 * emu_all + 5e-2, (mine_all, emu_all)
    k0 = 'patch_embed1.norm.running_mean'
    torch.testing.assert_close(model.state_dict()[k0].cpu(), sd[k0], rtol=1e-2, atol=1e-3)
    print(f'{arch}: logits rel L2 {_rel(logits.detach(), le):.4g} (storage noise {noise:.4g}); whole-gradient rel L2 to fp32 {mine_all:.4g} '
          f'(storage noise {emu_all:.4g})')


@pytest.mark.parametrize('arch', ['van_b0', 'van_b1'])
def test_van_stagewise_parity_with_oracle_tensors(arch):
    van, sd, model, x, y = _setup(arch, (8, 3, 128, 128))
    trace = {}
    _, _, ge = van.loss_and_grads(sd, x, y, arch, emulate_bf16=True, trace=trace)
    rt = model._runtime()
    rt.prep()
    failures, report = [], []
    params = dict(model.named_parameters())
    for i in range(4):
        inp = x.cuda() if i == 0 else _nhwc(trace[f'stage{i - 1}_out'])
        t = {}
        out = rt.stage_forward(i, inp, t, True)
        ref = trace[f'stage{i}_out']
        err = (out.float().cpu() - ref.detach().permute(0, 2, 3, 1)).abs()
        bad = (err > 2e-2 + 2e-2 * ref.detach().permute(0, 2, 3, 1).abs()).float().mean().item()
        report.append((err.max().item(), f'stage{i} output'))
        if bad > 1e-3:
            failures.append(f'stage{i} output: {bad:.2e} of the values off, max err {err.max().item():.4g}')
        din = rt.stage_backward(i, _nhwc(ref.grad), t)
        if i > 0:
            r = _rel(din, trace[f'stage{i - 1}_out'].grad.permute(0, 2, 3, 1))
            report.append((r, f'stage{i} input gradient'))
            if r > 8e-2:
                failures.append(f'stage{i} input gradient rel L2 {r:.4g}')
        prefixes = (f'patch_embed{i + 1}.', f'block{i + 1}.', f'norm{i + 1}.')
        names = [n for n in params if n.startswith(prefixes)]
        gmax = max(ge[n].abs().max().item() for n in names)
        for n in names:
            p = params[n]
            r = _rel(p.grad, ge[n])
            report.append((r, n))
            # A whole stage (up to 5 blocks x 2 branches, ~12 bf16 storage points each) is teacher-forced at once, so
            # independent rounding noise accumulates to a few percent: 8e-2 (the kernel-level tests above are tight).
            # Per-channel constants added to a stream that only BatchNorms consume (conv biases in front of a BN,
            # BN shifts, proj_2 / fc2 biases) have an analytically ZERO gradient, and other 1-D tensors have small ones:
            # a tensor may instead be within 3 % of the stage's largest gradient entry in absolute terms.
            if r > 8e-2 and (p.grad.float().cpu() - ge[n]).abs().max().item() > 3e-2 * gmax:
                failures.append(f'{n}: rel L2 {r:.4g}, abs {(p.grad.float().cpu() - ge[n]).abs().max().item():.3g} (stage max |g| {gmax:.3g})')
    torch.cuda.synchronize()
    print(f'{arch} stagewise: worst {sorted(report)[-3:]}')
    assert not failures, f'{len(failures)} stage checks failed: ' + '; '.join(failures[:12])
