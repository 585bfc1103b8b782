"""DarknetTiny / Darknet19 / Darknet53 on the H100 runtime vs the CPU oracle (oracle/darknet.py): end to end and stage by
stage with the oracle's boundary tensors (same method and tolerances as tests/test_resnet_gpu.py).
The 32-channel layers run channel-padded to 64 inside the runtime; only real channels are compared
and the padded ones must be exactly zero."""
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu


def _rel_l2(a, b):
    return ((a.float().cpu() - b.float().cpu()).norm() / b.float().norm().clamp_min(1e-12)).item()


def _nhwc_padded(t, dtype=torch.bfloat16):
    """NCHW fp32 oracle tensor -> NHWC, channels zero-padded to a multiple of 64, on the GPU."""
    t = t.detach().permute(0, 2, 3, 1).contiguous()
    c = t.shape[-1]
    cp = (c + 63) // 64 * 64
    if cp != c:
        t = F.pad(t, (0, cp - c))
    return t.to(dtype).cuda().contiguous()


ARCHS = ['darknettiny', 'darknet19', 'darknet53']


def _setup(arch, shape, nc=100, seed=0, act_type='leakyrelu'):
    from oracle import darknet
    from simpleaicv_pytorch_training_examples_b200.classification import backbones
    g = torch.Generator().manual_seed(41)
    x = torch.randn(*shape, generator=g)
    y = torch.randint(0, nc, (shape[0],), generator=g)
    sd = darknet.init_state(nc, seed, arch=arch)
    torch.manual_seed(seed)
    model = backbones.__dict__[arch](num_classes=nc, act_type=act_type).cuda().train()
    return darknet, sd, model, x, y


@pytest.mark.parametrize('arch,act_type', [(a, 'leakyrelu') for a in ARCHS] + [('darknettiny', 'silu'), ('darknet19', 'relu')])
def test_darknet_step_matches_oracle(arch, act_type):
    from simpleaicv_pytorch_training_examples_b200.classification import losses
    darknet, sd, model, x, y = _setup(arch, (8, 3, 128, 128), act_type=act_type)
    sd32 = {k: v.clone() for k, v in sd.items()}
    l32, ls32, g32 = darknet.loss_and_grads(sd32, x, y, arch=arch, act_type=act_type)
    le, lse, ge = darknet.loss_and_grads(sd, x, y, emulate_bf16=True, arch=arch, act_type=act_type)
    logits = model(x.cuda())
    loss = losses.CELoss()(logits, y.cuda())
    loss.backward()
    torch.cuda.synchronize()
    noise = _rel_l2(le, l32)
    assert _rel_l2(logits.detach(), le) <= 2.5 * noise + 1e-2, (_rel_l2(logits.detach(), le), noise)
    assert abs(float(loss.detach()) - float(lse)) <= 1e-2 * abs(float(lse)) + 2.5 * abs(float(lse) - float(ls32))
    grads = {n: p.grad.detach().float().cpu() for n, p in model.named_parameters()}
    cat = lambda d: torch.cat([d[n].flatten() for n in g32])
    mine_all, emu_all = _rel_l2(cat(grads), cat(g32)), _rel_l2(cat(ge), cat(g32))
    assert mine_all <= 2.0 * emu_all + 5e-2, (mine_all, emu_all)
    k0 = next(k for k in sd if k.endswith('running_mean'))
    torch.testing.assert_close(model.state_dict()[k0].cpu(), sd[k0], rtol=1e-2, atol=1e-3)
    print(f'{arch}/{act_type}: logits rel L2 {_rel_l2(logits.detach(), le):.4g}; whole-gradient rel L2 to fp32 {mine_all:.4g} (storage noise {emu_all:.4g})')


@pytest.mark.parametrize('arch', ARCHS)
def test_darknet_stagewise_parity_with_oracle_tensors(arch):
    darknet, sd, model, x, y = _setup(arch, (8, 3, 128, 128))
    trace = {}
    _, _, ge = darknet.loss_and_grads(sd, x, y, emulate_bf16=True, trace=trace, arch=arch)
    names = {id(p): n for n, p in model.named_parameters()}
    rt = model._runtime()
    rt.prep()
    failures, report = [], []

    def values_close(got, ref_nchw, what, loose):
        ref = ref_nchw.detach().permute(0, 2, 3, 1).float()
        c = ref.shape[-1]
        got = got.float().cpu()
        assert (got[..., c:] == 0).all(), f'{what}: padded channels are not zero'
        err = (got[..., :c] - ref).abs()
        bad = (err > 2e-2 + 2e-2 * ref.abs()).float().mean().item()
        report.append((err.max().item(), what))
        if bad > 1e-3 * loose:
            failures.append(f'{what}: {bad:.2e} of the values off, max err {err.max().item():.4g}')

    def grad_close(got, ref, what, tol):
        rl = _rel_l2(got, ref)
        report.append((rl, what))
        if not rl <= tol:
            failures.append(f'{what}: rel L2 {rl:.4g} > {tol:.3g}')

    tape = {'stem': {}}
    a = rt.stem_forward(x.cuda(), tape, True)
    values_close(a, trace['stem_out'], 'stem output', 1.0)
    rt.stem_backward(_nhwc_padded(trace['stem_out'].grad), tape)
    for p in (rt.stem.conv.weight, rt.stem.bn.weight, rt.stem.bn.bias):
        grad_close(p.grad, ge[names[id(p)]], f'stem {names[id(p)]}', 3e-2 if p.ndim == 4 else 6e-2)
    prev = 'stem_out'
    for i, blk in enumerate(rt.blocks):
        ref_out = trace[f'block{i}_out']
        n, _, h, w = ref_out.shape
        loose = 1.0 if n * h * w >= 2048 else 4.0
        t = {}
        out = blk.forward(_nhwc_padded(trace[prev]), t, True)
        values_close(out, ref_out, f'stage{i} output', loose)
        dx = blk.backward(_nhwc_padded(ref_out.grad), t, rt.sink)
        cin = trace[prev].shape[1]
        grad_close(dx[..., :cin], trace[prev].grad.permute(0, 2, 3, 1), f'stage{i} input gradient', 2e-2 * loose)
        for u in blk.all_units():
            for p in (u.conv.weight, u.bn.weight, u.bn.bias):
                grad_close(p.grad, ge[names[id(p)]], f'stage{i} {names[id(p)]}', (3e-2 if p.ndim == 4 else 6e-2) * loose)
        prev = f'block{i}_out'
    tape = {}
    logits = rt.head_forward(_nhwc_padded(trace[prev]), tape)
    grad_close(logits, trace['logits'].detach(), 'logits', 2e-2)
    da = rt.head_backward(trace['logits'].grad.cuda(), tape)
    grad_close(da, trace[prev].grad.permute(0, 2, 3, 1), 'head input gradient', 2e-2)
    hw = 'layer7.layer.0.weight' if arch == 'darknet19' else 'fc.weight'
    grad_close(dict(model.named_parameters())[hw].grad, ge[hw], hw, 2e-2)
    hb = hw.replace('weight', 'bias')
    grad_close(dict(model.named_parameters())[hb].grad, ge[hb], hb, 2e-2)
    torch.cuda.synchronize()
    print(f'{arch} stagewise: worst {max(report)}')
    assert not failures, f'{len(failures)} stage checks failed: ' + '; '.join(failures[:12])
