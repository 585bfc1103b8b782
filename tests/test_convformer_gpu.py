"""ConvFormer on the H100 runtime vs the CPU oracle (oracle/convformer.py, pinned to the reference by
tests/golden/convformer_*.ptf and tests/test_convformer_cpu.py): the two new kernels (ReLU-masked depthwise data gradient,
average pool of an fp32 / bf16 stream) against plain torch fp32, stem / downsampling / stage parity driven with the
oracle's boundary tensors, an end-to-end step, checkpointing, determinism, the fused optimizer and the graphed step."""
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu


def _rel(a, b):
    return ((a.float().cpu() - b.float().cpu()).norm() / b.float().cpu().norm().clamp_min(1e-12)).item()


def _nhwc(t, dtype=torch.bfloat16):
    return t.detach().permute(0, 2, 3, 1).contiguous().to(dtype).cuda()


def _rows(t, dtype):
    return _nhwc(t, dtype).view(-1, t.shape[1])


@pytest.mark.parametrize('c,h,w', [(128, 14, 14), (192, 9, 7), (640, 5, 11), (1536, 3, 5)])
def test_masked_depthwise_dgrad(c, h, w):
    from simpleaicv_pytorch_training_examples_b200 import ops
    g = torch.Generator().manual_seed(c + h)
    pre = torch.randn(2, c, h, w, generator=g).bfloat16().float()
    wt = torch.randn(c, 1, 7, 7, generator=g) * 0.1
    dy = torch.randn(2, c, h, w, generator=g).bfloat16().float()
    r = F.relu(pre)
    pr = pre.clone().requires_grad_(True)
    F.conv2d(F.relu(pr), wt, None, 1, 3, 1, c).backward(dy)
    dx = ops.dwconv_dgrad_masked(_nhwc(dy), wt.cuda(), _nhwc(r), 7)
    assert _rel(dx, pr.grad.permute(0, 2, 3, 1)) <= 5e-3
    # bit for bit: the unmasked flipped-tap kernel, then the mask
    plain = ops.dwconv_fwd(_nhwc(dy), wt.cuda(), None, 7, 1, flip=True)
    assert torch.equal(dx, torch.where(_nhwc(r) > 0, plain, torch.zeros_like(plain)))


@pytest.mark.parametrize('c,h,w', [(128, 7, 7), (192, 5, 9), (640, 3, 3), (1536, 2, 5)])
@pytest.mark.parametrize('dtype', [torch.float32, torch.bfloat16])
def test_stream_avgpool_fwd_bwd(c, h, w, dtype):
    from simpleaicv_pytorch_training_examples_b200 import ops
    g = torch.Generator().manual_seed(c * w)
    x = (torch.randn(3, h, w, c, generator=g) * 2 + 0.5).to(dtype)
    y = ops.avgpool_stream_fwd(x.cuda())
    want = x.float().sum(dim=(1, 2)) * (1.0 / (h * w))
    assert y.dtype == torch.bfloat16
    assert (y.float().cpu() - want).abs().max().item() <= 2 ** -8 * want.abs().max().item() + 1e-6
    dp = torch.randn(3, c, generator=g).bfloat16()
    dx = ops.avgpool_stream_bwd(dp.cuda(), h, w)
    assert dx.dtype == torch.float32
    torch.testing.assert_close(dx.cpu(), (dp.float() * (1.0 / (h * w)))[:, None, None, :].expand(3, h, w, c), rtol=0, atol=0)
    dxb = ops.avgpool_stream_bwd(dp.cuda(), h, w, dx_f32=False)
    assert torch.equal(dxb, dx.bfloat16())


def _setup(arch, shape, dp=0., nc=10, seed=0, ckpt=False):
    from oracle import convformer
    from simpleaicv_pytorch_training_examples_b200.classification import backbones
    g = torch.Generator().manual_seed(41)
    x = torch.randn(*shape, generator=g)
    y = torch.randint(0, nc, (shape[0],), generator=g)
    sd = convformer.init_state(arch, nc, seed)
    torch.manual_seed(seed)
    model = backbones.__dict__[arch](num_classes=nc, drop_path_prob=dp, use_gradient_checkpoint=ckpt).cuda().train()
    return convformer, sd, model, x, y


def _runtime_step(model, x, y):
    """One training forward / backward through the runtime, returning (logits, loss, drop scales by block)."""
    from simpleaicv_pytorch_training_examples_b200.classification import losses
    rt = model._runtime()
    logits, tape = rt.forward(x.cuda(), True, True)
    scales = {}
    for i, t in enumerate(tape['stages']):
        sc = t['scales'] if 'scales' in t else rt.stage_scales(t)
        for j, (s1, s2) in enumerate(sc):
            if s1 is not None:
                scales[f'stages.{i}.{j}'] = (s1.cpu(), s2.cpu())
    lg = logits.detach().requires_grad_(True)
    loss = losses.CELoss()(lg, y.cuda())
    loss.backward()
    rt.backward(lg.grad, tape)
    torch.cuda.synchronize()
    return logits.detach(), loss.detach(), scales


@pytest.mark.parametrize('arch,dp,batch', [('convformer_s18', 0., 8), ('convformer_s18', 0.3, 8), ('convformer_m36', 0., 4)])
def test_convformer_step_matches_oracle(arch, dp, batch):
    cf, sd, model, x, y = _setup(arch, (batch, 3, 128, 128), dp)
    logits, loss, scales = _runtime_step(model, x, y)
    if dp > 0:
        assert set(scales) == {k for k, p in cf.drop_path_rates(arch, dp).items() if p > 0}
    sd32, sde = {k: v.clone() for k, v in sd.items()}, {k: v.clone() for k, v in sd.items()}
    l32, ls32, g32 = cf.loss_and_grads(sd32, x, y, arch, drop_path_prob=dp, drop_scales=scales)
    le, lse, ge = cf.loss_and_grads(sde, x, y, arch, emulate_bf16=True, drop_path_prob=dp, drop_scales=scales)
    noise = _rel(le, l32)
    assert _rel(logits, le) <= 2.5 * noise + 1e-2, (_rel(logits, le), noise)
    assert abs(float(loss) - float(lse)) <= 1e-2 * abs(float(lse)) + 2.5 * abs(float(lse) - float(ls32))
    grads = {n: p.grad.detach().float().cpu() for n, p in model.named_parameters()}
    assert set(grads) == set(g32)
    cat = lambda d: torch.cat([d[n].flatten() for n in g32])
    mine_all, emu_all = _rel(cat(grads), cat(g32)), _rel(cat(ge), cat(g32))
    assert mine_all <= 2.0 * emu_all + 5e-2, (mine_all, emu_all)
    state = model.state_dict()
    for k in ('downsample_layers.0.post_norm.running_mean', 'downsample_layers.0.post_norm.running_var',
              'stages.3.2.norm2.running_mean', 'stages.3.2.norm2.running_var'):
        torch.testing.assert_close(state[k].cpu(), sde[k], rtol=2e-2, atol=2e-3, msg=k)
    assert int(state['stages.1.0.norm1.num_batches_tracked']) == 1
    # eval mode: running statistics, bf16 stream throughout
    model.eval()
    with torch.no_grad():
        ev = model(x.cuda())
        ev_ref32 = cf.forward(sd32, x, arch, training=False)
        ev_ref = cf.forward(sde, x, arch, training=False, emulate_bf16=True)
    assert _rel(ev, ev_ref) <= 2.5 * _rel(ev_ref, ev_ref32) + 1e-2, (_rel(ev, ev_ref), _rel(ev_ref, ev_ref32))
    print(f'{arch} dp {dp}: logits rel L2 {_rel(logits, le):.4g} (storage noise {noise:.4g}); whole-gradient rel L2 to fp32 '
          f'{mine_all:.4g} (storage noise {emu_all:.4g}); eval logits {_rel(ev, ev_ref):.4g}')


@pytest.mark.parametrize('dp', [0., 0.3])
def test_convformer_stagewise_parity_with_oracle_tensors(dp):
    arch = 'convformer_s18'
    cf, sd, model, x, y = _setup(arch, (8, 3, 128, 128), dp)
    rt = model._runtime()
    rt.prep()
    # the runtime's own drop-path draws, injected into the oracle and into the teacher-forced stages below
    draws = []
    for i, stage in enumerate(rt.stages):
        draws.append([b.draw_scales(8, True, 'cuda') for b in stage])
    scales = {f'stages.{i}.{j}': (s1.cpu(), s2.cpu()) for i, st in enumerate(draws) for j, (s1, s2) in enumerate(st) if s1 is not None}
    trace = {}
    _, _, ge = cf.loss_and_grads(sd, x, y, arch, emulate_bf16=True, trace=trace, drop_path_prob=dp, drop_scales=scales)
    params = dict(model.named_parameters())
    failures, report = [], []
    stream = torch.float32 if dp > 0 else torch.bfloat16        # dtype of a stage's output stream in training

    def check_out(out, ref, what):
        ref = ref.detach().permute(0, 2, 3, 1).reshape(out.shape)
        err = (out.float().cpu() - ref).abs()
        bad = (err > 2e-2 + 2e-2 * ref.abs()).float().mean().item()
        report.append((err.max().item(), what))
        if bad > 1e-3:
            failures.append(f'{what}: {bad:.2e} of the values off, max err {err.max().item():.4g}')

    def check_grad(din, ref, what):
        r = _rel(din, ref.permute(0, 2, 3, 1).reshape(din.shape))
        report.append((r, what))
        if r > 8e-2:
            failures.append(f'{what} rel L2 {r:.4g}')

    def check_params(prefix):
        names = [n for n in params if n.startswith(prefix)]
        gmax = max(ge[n].abs().max().item() for n in names)
        for n in names:
            g = params[n].grad.float().cpu()
            r = _rel(g, ge[n])
            report.append((r, n))
            # same criterion as test_van_gpu.py: BN shifts / conv biases in front of a BN have an analytically zero gradient
            if r > 8e-2 and (g - ge[n]).abs().max().item() > 3e-2 * gmax:
                failures.append(f'{n}: rel L2 {r:.4g}, abs {(g - ge[n]).abs().max().item():.3g} (max |g| {gmax:.3g})')

    t = {}
    s, shape = rt.stem_forward(x.cuda(), t, True)
    check_out(s, trace['stem_out'], 'stem output')
    rt.stem_backward(_rows(trace['stem_out'].grad, torch.float32), t)
    check_params('downsample_layers.0.')
    for i in range(4):
        if i > 0:
            prev = trace[f'stage{i - 1}_out']
            t = {}
            s, shape = rt.down_forward(i, _rows(prev, stream), tuple(prev.permute(0, 2, 3, 1).shape), t, True)
            check_out(s, trace[f'stage{i}_in'], f'downsampling {i} output')
            din = rt.down_backward(i, _rows(trace[f'stage{i}_in'].grad, torch.float32), t)
            check_grad(din, prev.grad, f'downsampling {i} input gradient')
            check_params(f'downsample_layers.{i}.')
        t = {}
        inp = trace[f'stage{i}_in']
        out = rt.stage_forward(i, _rows(inp, torch.bfloat16), tuple(inp.permute(0, 2, 3, 1).shape), t, True, scales=draws[i])
        assert out.dtype == stream
        check_out(out, trace[f'stage{i}_out'], f'stage{i} output')
        din = rt.stage_backward(i, _rows(trace[f'stage{i}_out'].grad, torch.float32), t)
        check_grad(din, inp.grad, f'stage{i} input gradient')
        check_params(f'stages.{i}.')
    torch.cuda.synchronize()
    print(f'{arch} dp {dp} stagewise: worst {sorted(report)[-3:]}')
    assert not failures, f'{len(failures)} checks failed: ' + '; '.join(failures[:12])


def _grads_of_step(arch, dp, ckpt, x, y, seed=5):
    from simpleaicv_pytorch_training_examples_b200.classification import backbones, losses
    torch.manual_seed(0)
    model = backbones.__dict__[arch](num_classes=10, drop_path_prob=dp, use_gradient_checkpoint=ckpt).cuda().train()
    out = []
    for _ in range(2):
        torch.manual_seed(seed)                     # the same drop-path draws in every run
        model.zero_grad(set_to_none=True)
        losses.CELoss()(model(x), y).backward()
        out.append({n: p.grad.detach().clone() for n, p in model.named_parameters()})
    torch.cuda.synchronize()
    return out, model


def test_checkpointing_and_determinism():
    g = torch.Generator().manual_seed(3)
    x, y = torch.randn(8, 3, 96, 96, generator=g).cuda(), torch.randint(0, 10, (8,), generator=g).cuda()
    (a1, a2), plain = _grads_of_step('convformer_s18', 0.3, False, x, y)
    (b1, _), ckpt = _grads_of_step('convformer_s18', 0.3, True, x, y)
    for n in a1:
        assert torch.equal(a1[n], a2[n]), f'{n}: two consecutive steps differ'
        assert torch.equal(a1[n], b1[n]), f'{n}: use_gradient_checkpoint changed the gradient'
    # the checkpoint replay updates every BatchNorm's running statistics a second time (as torch checkpointing does)
    k = 'stages.2.4.norm1.num_batches_tracked'
    assert int(plain.state_dict()[k]) == 2 and int(ckpt.state_dict()[k]) == 4


def _adamw_cfg():
    class Cfg:   # the shipped convformer_s18 config's optimizer (00.classification_training/imagenet/convformer_s18)
        optimizer = ('AdamW', {'lr': 2e-3, 'global_weight_decay': False, 'weight_decay': 5e-2, 'no_weight_decay_layer_name_list': []})
    return Cfg


def test_fused_adamw_refreshes_every_operand_copy():
    from simpleaicv_pytorch_training_examples_b200 import optim
    from simpleaicv_pytorch_training_examples_b200.classification import backbones, losses
    from simpleaicv_pytorch_training_examples_b200.engine.operands import Operand
    from simpleaicv_pytorch_training_examples_b200.tools import utils as tutils
    torch.manual_seed(0)
    model = backbones.convformer_s18(num_classes=10, drop_path_prob=0.2).cuda().train()
    opt, _ = tutils.build_optimizer(_adamw_cfg(), model)
    fusable = [op for op in model._runtime().operands() if op.fusable]
    assert isinstance(opt, optim.FusedAdamW) and len(opt._shadows) == len(fusable)
    g = torch.Generator(device='cuda').manual_seed(1)
    x, y = torch.randn(8, 3, 64, 64, device='cuda', generator=g), torch.randint(0, 10, (8,), device='cuda', generator=g)
    for _ in range(2):
        losses.CELoss()(model(x), y).backward()
        opt.clip_grad_norm(1.0)
        opt.step()
        opt.zero_grad()
    for op in fusable:
        fresh = Operand(op.param, op.layout, kp=op.kp, cp=op.cp) if op.conv else Operand(op.param)
        assert torch.equal(fresh.refresh(), op.w)


def test_graphed_step_equals_eager_step():
    from simpleaicv_pytorch_training_examples_b200.classification import backbones, losses
    from simpleaicv_pytorch_training_examples_b200.graph import GraphedTrainStep
    from simpleaicv_pytorch_training_examples_b200.tools import utils as tutils
    g = torch.Generator(device='cuda').manual_seed(2)
    x = torch.randn(8, 3, 64, 64, device='cuda', generator=g)
    lab = torch.randint(0, 10, (8,), device='cuda', generator=g)
    y = 0.5 * F.one_hot(lab, 10).float() + 0.5 * F.one_hot(lab.roll(1), 10).float()
    crit = losses.OneHotLabelCELoss()
    models = []
    for _ in range(2):
        torch.manual_seed(0)
        m = backbones.convformer_s18(num_classes=10).cuda().train()
        models.append((m, tutils.build_optimizer(_adamw_cfg(), m)[0]))
    (me, oe), (mg, og) = models
    graphed = GraphedTrainStep(mg, crit, og, x, y, warmup=2)         # two eager warm-up steps, then the capture
    for _ in range(2):
        loss = crit(me(x), y)
        loss.backward()
        oe.step()
        oe.zero_grad()
    for _ in range(2):
        lg = graphed(x, y).clone()
        loss = crit(me(x), y)
        loss.backward()
        oe.step()
        oe.zero_grad()
        assert torch.equal(lg, loss.detach())
    torch.cuda.synchronize()
    for (n, p), q in zip(me.named_parameters(), mg.parameters()):
        assert torch.equal(p, q), n
    for k, v in me.state_dict().items():
        assert torch.equal(v, mg.state_dict()[k]), k
