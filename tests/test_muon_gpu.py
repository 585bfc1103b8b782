"""Muon on the H100: the batched Newton-Schulz GEMMs (csrc/capi_gemm.cu saicv_ns_gemm) against a float64 iteration, with
torch's bf16 matmuls running the same iteration as the yardstick; optim.FusedMuon against the reference's three steps
(tests/golden/muon_3steps.pto); and FusedMuon through tools.utils.build_optimizer on ResNet-18 and a small ViT
(operand copies, clip, Nesterov, determinism, CUDA-graph replay, checkpoint resume, training progress)."""
import copy
import os
import sys

import pytest
import torch

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, 'golden'))
COEF = (3.4445, -4.7750, 2.0315)


def _ns_torch(x, steps, dtype):
    """The reference's iteration (normalised x, m <= n) with torch matmuls in `dtype`."""
    a, b, c = COEF
    x = x.to(dtype)
    for _ in range(steps):
        m = x @ x.mT
        bm = b * m + c * m @ m
        x = a * x + bm @ x
    return x


def _ns_ours(gs, steps=5):
    """gs: [batch, r, c] fp32 -> the batched kernels' result [batch, r, c] (transposed in and out when r > c)."""
    from simpleaicv_pytorch_training_examples_b200 import optim
    tall = gs.shape[1] > gs.shape[2]
    x = gs.mT if tall else gs
    batch, m, n = x.shape
    mp, np_ = (m + 7) // 8 * 8, (n + 7) // 8 * 8
    xs = torch.zeros(batch, mp, np_, dtype=torch.bfloat16, device='cuda')
    xs[:, :m, :n] = (x / (x.norm(dim=(1, 2), keepdim=True) + 1e-7)).to(torch.bfloat16)
    ws = [torch.empty_like(xs), torch.empty_like(xs), torch.empty(batch, mp, mp, dtype=torch.bfloat16, device='cuda'),
          torch.empty(batch, mp, mp, dtype=torch.bfloat16, device='cuda')]
    optim.newton_schulz(xs, steps, *ws)
    assert not xs[:, m:].any() and not xs[:, :, n:].any(), 'zero padding did not stay zero'
    out = xs[:, :m, :n].float()
    return out.mT if tall else out


@pytest.mark.parametrize('r,c,batch', [(256, 256, 1), (128, 512, 4), (768, 192, 3), (147, 1000, 2), (1000, 2304, 1),
                                       (768, 2304, 24), (64, 147, 7)])
def test_batched_newton_schulz_against_float64(r, c, batch):
    g = torch.Generator(device='cuda').manual_seed(r * 7 + c + batch)
    gs = torch.randn(batch, r, c, device='cuda', generator=g)
    ours = _ns_ours(gs)
    x = gs.mT if r > c else gs
    xn = x.double() / (x.double().norm(dim=(1, 2), keepdim=True) + 1e-7)
    want = _ns_torch(xn, 5, torch.float64)
    torch_bf16 = _ns_torch(xn.to(torch.bfloat16), 5, torch.bfloat16).double()
    if r > c:
        want, torch_bf16 = want.mT, torch_bf16.mT
    err = ((ours.double() - want).norm() / want.norm()).item()
    err_torch = ((torch_bf16 - want).norm() / want.norm()).item()
    assert err <= 1.5 * err_torch, f'batched NS rel L2 {err:.4g} vs torch bf16 {err_torch:.4g}'
    # a matrix alone and inside the batch: the same tiles, the same bits
    k = batch // 2
    assert torch.equal(_ns_ours(gs[k:k + 1].contiguous())[0], ours[k])


def _fixture():
    return torch.load(os.path.join(HERE, 'golden', 'muon_3steps.pto'), weights_only=False)


class _Cfg:
    def __init__(self, optimizer):
        self.optimizer = optimizer


def _fixture_run():
    import make_muon_golden
    from simpleaicv_pytorch_training_examples_b200 import optim
    from simpleaicv_pytorch_training_examples_b200.tools import utils
    fx = _fixture()
    model = make_muon_golden.ParamSet().cuda()
    with torch.no_grad():
        for n, p in model.named_parameters():
            p.copy_(fx['params0'][n])
    opt, info = utils.build_optimizer(_Cfg(fx['optimizer']), model)
    assert isinstance(opt, optim.FusedMuon) and info == fx['descr']
    out = []
    for gs in fx['grads']:
        for n, p in model.named_parameters():
            p.grad = None if gs[n] is None else gs[n].cuda()
        opt.step()
        out.append({n: p.detach().cpu().clone() for n, p in model.named_parameters()})
    return fx, model, opt, out


def test_fused_muon_matches_the_reference_fixture():
    from oracle import muon as omuon
    fx, model, opt, out = _fixture_run()
    o = fx['optimizer'][1]
    g0 = fx['param_groups'][0]
    use = {n: n in fx['descr'][0]['name'] for n in fx['order']}
    params = {n: fx['params0'][n].double().clone() for n in fx['order']}
    state = {}
    for k, gs in enumerate(fx['grads']):
        omuon.step(params, gs, state, use, o['lr'], o['weight_decay'], g0['momentum'], g0['nesterov'], g0['ns_steps'],
                   g0['adamw_betas'], g0['adamw_eps'])
        for n in fx['order']:
            want = fx['params'][k][n].double()
            d = (out[k][n].double() - want).abs().max().item()
            if use[n]:
                # the reference's own bf16 error (against the float64 iteration) sets the scale
                ref_err = (params[n] - want).abs().max().item()
                assert d <= 2.5 * ref_err, f'step {k} {n}: {d:.3g} vs reference bf16 error {ref_err:.3g}'
            else:
                assert d <= 1e-6, f'step {k} {n}: {d:.3g}'
    sd = opt.state_dict()
    order = fx['order']
    for i, st in sd['state'].items():
        want = fx['state'][order[i]]
        assert set(st) == set(want), order[i]
        for key, v in want.items():
            if torch.is_tensor(v):
                assert st[key].shape == v.shape
                assert torch.allclose(st[key].cpu(), v, rtol=1e-5, atol=1e-6), (order[i], key)
            else:
                assert st[key] == v, (order[i], key)
    # the reference's checkpoint loads into FusedMuon and continues
    opt.load_state_dict({'state': {order.index(n): v for n, v in fx['state'].items()}, 'param_groups': fx['param_groups']})
    assert opt.state_dict()['state'][order.index('norm_bias')]['step'] == 2


def _model_step(family, seed=0):
    import test_operands_cpu
    from simpleaicv_pytorch_training_examples_b200.classification import losses
    torch.manual_seed(seed)
    model = test_operands_cpu._families()[family]().cuda().train()
    g = torch.Generator(device='cuda').manual_seed(1)
    side = 32 if family == 'resnet18cifar' else 64
    x = torch.randn(8, 3, side, side, device='cuda', generator=g)
    y = torch.randint(0, 10, (8,), device='cuda', generator=g)
    crit = losses.CELoss()
    return model, lambda: crit(model(x), y)


def _train(family, opt_cfg, steps, clip):
    from simpleaicv_pytorch_training_examples_b200.tools import utils
    model, loss_fn = _model_step(family)
    opt, _ = utils.build_optimizer(_Cfg(('Muon', opt_cfg)), model)
    losses = []
    for _ in range(steps):
        loss = loss_fn()
        loss.backward()
        losses.append(float(loss.detach()))
        if clip:
            opt.clip_grad_norm(1.0)
        opt.step()
        opt.zero_grad()
    torch.cuda.synchronize()
    return model, opt, losses


@pytest.mark.parametrize('family', ['resnet18cifar', 'vit_base_patch16'])
@pytest.mark.parametrize('clip,nesterov', [(False, True), (True, False)])
def test_build_optimizer_trains_deterministically(family, clip, nesterov):
    from simpleaicv_pytorch_training_examples_b200.engine.operands import Operand
    cfg = {'lr': 0.02 if family == 'resnet18cifar' else 2e-3, 'weight_decay': 0.01, 'nesterov': nesterov}
    m1, opt1, l1 = _train(family, cfg, 6, clip)
    m2, _, l2 = _train(family, cfg, 6, clip)
    assert l1 == l2
    for (n, p), q in zip(m1.named_parameters(), m2.parameters()):
        assert torch.equal(p, q), f'two runs differ at {n}'
    assert l1[-1] < l1[0], f'loss did not decrease: {l1}'
    fusable = [op for op in m1._runtime().operands() if op.fusable]
    assert len(opt1._shadows) == len(fusable) > 0
    for op in fusable:
        fresh = Operand(op.param, op.layout, kp=op.kp, cp=op.cp) if op.conv else Operand(op.param)
        assert torch.equal(fresh.refresh(), op.w)


def _fixture_opt(seed=0):
    import make_muon_golden
    from simpleaicv_pytorch_training_examples_b200.tools import utils
    model = make_muon_golden.ParamSet(seed).cuda()
    opt, _ = utils.build_optimizer(_Cfg(('Muon', {'lr': 0.02, 'weight_decay': 0.05})), model)
    return model, opt


def _grads(model, step):
    g = torch.Generator(device='cuda').manual_seed(50 + step)
    return [torch.randn(p.shape, device='cuda', generator=g) for p in model.parameters()]


def test_captured_step_equals_eager():
    ma, oa = _fixture_opt()
    mb, ob = _fixture_opt()
    static = [torch.zeros_like(p) for p in mb.parameters()]
    for p, s in zip(mb.parameters(), static):
        p.grad = s
    lrs = [0.02 * 0.9 ** i for i in range(10)]

    def feed(step):
        for p, s, g in zip(ma.parameters(), static, _grads(ma, step)):
            p.grad = g.clone()
            s.copy_(g)
        for o in (oa, ob):
            o.param_groups[0]['lr'] = lrs[step]
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):      # eager warm-up steps allocate the Newton-Schulz buffers
        for step in range(2):
            feed(step)
            oa.step()
            ob.step()
    torch.cuda.current_stream().wait_stream(side)
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        ob.step()
    for step in range(2, 10):
        feed(step)
        oa.step()
        ob.sync_hyper()
        graph.replay()
        ob.after_replay()
    torch.cuda.synchronize()
    for p, q in zip(ma.parameters(), mb.parameters()):
        assert torch.equal(p, q)


def test_state_dict_resumes_bit_identically():
    ma, oa = _fixture_opt()
    for step in range(3):
        for p, g in zip(ma.parameters(), _grads(ma, step)):
            p.grad = g
        oa.step()
    mb = copy.deepcopy(ma)
    from simpleaicv_pytorch_training_examples_b200.tools import utils
    ob, _ = utils.build_optimizer(_Cfg(('Muon', {'lr': 0.02, 'weight_decay': 0.05})), mb)
    ob.load_state_dict(copy.deepcopy(oa.state_dict()))
    for step in range(3, 6):
        for m, o in ((ma, oa), (mb, ob)):
            for p, g in zip(m.parameters(), _grads(m, step)):
                p.grad = g
            o.step()
    torch.cuda.synchronize()
    for p, q in zip(ma.parameters(), mb.parameters()):
        assert torch.equal(p, q)


def _three_steps_on_this_device(out):
    m, o = _fixture_opt()
    for step in range(3):
        for p, g in zip(m.parameters(), _grads(m, step)):
            p.grad = g
        o.step()
    torch.save([p.detach().cpu() for p in m.parameters()], out)


def test_devices_stay_bit_identical(tmp_path):
    """Data-parallel ranks apply the same all-reduced gradients, one process per GPU: their parameters must stay equal."""
    import subprocess
    if torch.cuda.device_count() < 2:
        pytest.skip('needs two GPUs')
    code = f'import sys; sys.path[:0] = [{HERE!r}, {os.path.dirname(HERE)!r}]; import test_muon_gpu as t; ' \
           't._three_steps_on_this_device(sys.argv[1])'
    outs = []
    for dev in (0, 1):
        out = str(tmp_path / f'rank{dev}.pt')
        subprocess.run([sys.executable, '-c', code, out], check=True, env=dict(os.environ, CUDA_VISIBLE_DEVICES=str(dev)))
        outs.append(torch.load(out))
    for a, b in zip(*outs):
        assert torch.equal(a, b)
