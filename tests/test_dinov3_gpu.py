"""DINOv3 on the H100 runtime: the RoPE and SwiGLU kernels against the torch expressions of the reference, block-by-block
parity driven with the oracle's boundary tensors, end-to-end encoder forward / backward against oracle/dinov3.py (pinned to
the reference by tests/golden/dinov3_*.ptf), checkpointing, the CPU rescale draw, and two distillation training steps."""
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu


def _rel(a, b):
    return ((a.float().cpu() - b.float().cpu()).norm() / b.float().cpu().norm().clamp_min(1e-12)).item()


def _rope_ref(x, sin, cos):
    """dinov3vit.py:271-282 / :347-367 under autocast: bf16 q or k -> fp32 -> x*cos + rotate_half(x)*sin -> bf16."""
    x1, x2 = x.float().chunk(2, dim=-1)
    return (x.float() * cos + torch.cat([-x2, x1], dim=-1) * sin).to(torch.bfloat16)


@pytest.mark.parametrize('b,L,heads,hd', [(1, 1, 1, 64), (1, 37, 6, 64), (3, 49, 12, 64), (2, 16, 20, 64), (2, 9, 3, 8),
                                          (1, 25, 2, 24)])
def test_rope_kernel_is_bit_identical_to_reference_expression(b, L, heads, hd):
    from oracle import dinov3 as od
    from simpleaicv_pytorch_training_examples_b200 import ops
    g = torch.Generator().manual_seed(L * heads + hd)
    qkv = (torch.randn(b * L, 3 * heads * hd, generator=g) * 3).bfloat16().cuda()
    periods = 100.0 ** (2 * torch.arange(hd // 4) / (hd // 2))
    sin, cos = od.rope_table(periods, L, 1, torch.tensor([1.37]))
    sin, cos = sin.cuda().contiguous(), cos.cuda().contiguous()
    q5 = qkv.view(b, L, 3, heads, hd)
    want_q, want_k = _rope_ref(q5[:, :, 0], sin[:, None], cos[:, None]), _rope_ref(q5[:, :, 1], sin[:, None], cos[:, None])
    v = q5[:, :, 2].clone()
    out = ops.rope_qk(qkv.clone(), sin, cos, b, L, heads, hd).view(b, L, 3, heads, hd)
    assert torch.equal(out[:, :, 0], want_q) and torch.equal(out[:, :, 1], want_k) and torch.equal(out[:, :, 2], v)
    # backward: autograd through the reference expression (the fp32 cast's backward rounds to bf16 once)
    dq = (torch.randn(b * L, 3 * heads * hd, generator=g)).bfloat16().cuda()
    d5 = dq.view(b, L, 3, heads, hd)
    want = []
    for s in (0, 1):
        xf = q5[:, :, s].float().requires_grad_(True)
        x1, x2 = xf.chunk(2, dim=-1)
        (xf * cos[:, None] + torch.cat([-x2, x1], dim=-1) * sin[:, None]).backward(d5[:, :, s].float())
        want.append(xf.grad.to(torch.bfloat16))
    got = ops.rope_qk(dq.clone(), sin, cos, b, L, heads, hd, backward=True).view(b, L, 3, heads, hd)
    assert torch.equal(got[:, :, 0], want[0]) and torch.equal(got[:, :, 1], want[1]) and torch.equal(got[:, :, 2], d5[:, :, 2])


def test_rope_rejects_bad_head_size():
    from simpleaicv_pytorch_training_examples_b200 import ops
    qkv = torch.zeros(4, 3 * 12, device='cuda', dtype=torch.bfloat16)
    t = torch.zeros(4, 12, device='cuda')
    with pytest.raises(RuntimeError, match='multiple of 8'):
        ops.rope_qk(qkv, t, t, 1, 4, 1, 12)


@pytest.mark.parametrize('n', [8, 4096, 3 * 1536 * 7])
def test_swiglu_matches_torch_autocast(n):
    from simpleaicv_pytorch_training_examples_b200 import ops
    g = torch.Generator().manual_seed(n)
    a = (torch.randn(n, generator=g) * 4).bfloat16().cuda()
    b = torch.randn(n, generator=g).bfloat16().cuda()
    dh = torch.randn(n, generator=g).bfloat16().cuda()
    ar, br = a.clone().requires_grad_(True), b.clone().requires_grad_(True)
    with torch.autocast('cuda', dtype=torch.bfloat16):
        h = F.silu(ar) * br
    h.backward(dh)
    got = ops.swiglu_fwd(a, b)
    da, db = ops.swiglu_bwd(dh, a, b)
    assert h.dtype == torch.bfloat16
    assert torch.equal(got, h.detach())
    assert torch.equal(db, br.grad)
    # da: torch's silu backward may contract into an FMA; allow one bf16 rounding step
    torch.testing.assert_close(da, ar.grad, rtol=2 ** -7, atol=1e-30)
    print(f'swiglu n={n}: da bit-identical on {(da == ar.grad).float().mean().item():.4f} of the elements')


def _randomize(model, seed):
    """Layer scales, biases and norm affines away from their init values so that every block and term matters."""
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        for n, p in model.named_parameters():
            if n.endswith('gamma'):
                p.copy_(0.3 + 0.7 * torch.rand(p.shape, generator=g))
            elif n.endswith('bias'):
                p.copy_(0.1 * torch.randn(p.shape, generator=g))
            elif 'norm' in n or n.startswith('neck.1') or n.startswith('neck.3'):
                p.copy_(1 + 0.1 * torch.randn(p.shape, generator=g))


def _setup(arch, size=64, batch=2, ckpt=False, seed=8):
    from simpleaicv_pytorch_training_examples_b200.interactive_segmentation.models.dinov3_segment_anything import DINOV3ViTImageEncoder
    torch.manual_seed(seed)
    model = DINOV3ViTImageEncoder(arch, image_size=size, use_gradient_checkpoint=ckpt)
    _randomize(model, seed)
    model = model.cuda().train()
    sd = {n: v.detach().cpu().clone() for n, v in model.state_dict().items()}
    g = torch.Generator().manual_seed(77)
    x = torch.randn(batch, 3, size, size, generator=g)
    target = torch.randn(batch, 256, size // 16, size // 16, generator=g)
    return model, sd, x, target


@pytest.mark.parametrize('arch,size', [('dinov3_vit_small_patch16_backbone', 64), ('dinov3_vit_small_plus_patch16_backbone', 48),
                                       ('dinov3_vit_base_patch16_backbone', 80)])
def test_encoder_step_matches_oracle(arch, size):
    from oracle import dinov3 as od
    model, sd, x, target = _setup(arch, size)
    heads = od.ARCHS[arch][2]
    torch.manual_seed(31)
    fac = od.draw_rescale(2)
    o32, l32, g32 = od.loss_and_grads({k: v.clone() for k, v in sd.items()}, x, target, heads, fac, prefix='backbone.')
    oe, le, ge = od.loss_and_grads(sd, x, target, heads, fac, emulate_bf16=True, prefix='backbone.')
    torch.manual_seed(31)
    out = model(x.cuda())
    loss = F.mse_loss(out, target.cuda())
    loss.backward()
    torch.cuda.synchronize()
    noise = _rel(oe, o32)
    assert out.shape == o32.shape and out.dtype == torch.float32
    assert _rel(out.detach(), oe) <= 2.5 * noise + 1e-2, (_rel(out.detach(), oe), noise)
    assert abs(loss.item() - le.item()) <= 2e-2 * le.item()
    grads = {n: p.grad.detach().float().cpu() for n, p in model.named_parameters()}
    assert set(grads) == set(g32)
    cat = lambda d: torch.cat([d[n].flatten() for n in g32])
    mine_all, emu_all = _rel(cat(grads), cat(g32)), _rel(cat(ge), cat(g32))
    assert mine_all <= 2.0 * emu_all + 5e-2, (mine_all, emu_all)
    worst = max((_rel(grads[n], ge[n]), n) for n in g32)
    print(f'dinov3 {arch} {size}px: out rel L2 {_rel(out.detach(), oe):.4g} (storage noise {noise:.4g}); whole-gradient rel L2 '
          f'{mine_all:.4g} (storage noise {emu_all:.4g}); worst tensor vs emulated oracle {worst}')
    assert worst[0] <= 8e-2, worst
    k_bias = [grads[f'backbone.blocks.{i}.attn.qkv.bias'][384 if 'small' in arch else 768:][:8] for i in range(2)]
    assert all(t.abs().max().item() == 0 for t in k_bias), 'the k slice of the qkv bias must get no gradient'


def test_blockwise_parity_with_oracle_tensors():
    from oracle import dinov3 as od
    arch = 'dinov3_vit_small_plus_patch16_backbone'
    model, sd, x, target = _setup(arch, 64)
    heads = od.ARCHS[arch][2]
    trace = {}
    torch.manual_seed(4)
    fac = od.draw_rescale(2)
    _, _, ge = od.loss_and_grads(sd, x, target, heads, fac, emulate_bf16=True, trace=trace, prefix='backbone.')
    rt = model._runtime()
    rt.prep()
    params = dict(model.named_parameters())
    failures, report = [], []

    def check(got, want, what, tol):
        r = _rel(got, want)
        report.append((r, what))
        if not r <= tol:
            failures.append(f'{what}: rel L2 {r:.4g} > {tol}')

    tape = {}
    torch.manual_seed(4)
    tok = rt.embed_forward(x.cuda(), True, tape)
    B, L, rope = tape['B'], tape['H'] * tape['W'], tape['rope']
    C = tok.shape[1]
    check(tok.view(B, L, C), trace['tokens'].detach(), 'tokens', 1e-2)
    prev = 'tokens'
    for i, blk in enumerate(rt.blocks):
        t = {}
        out = blk.forward(trace[prev].detach().reshape(-1, C).cuda().contiguous(), t, B, L, rope)
        ref_out = trace[f'block{i}_out']
        check(out.view(B, L, C), ref_out.detach(), f'block{i} output', 1e-2)
        dx, _ = blk.backward(ref_out.grad.reshape(-1, C).cuda().contiguous(), t, B, L, rope, rt.sink)
        check(dx.view(B, L, C), trace[prev].grad, f'block{i} input gradient', 2e-2)
        for n, p in params.items():
            if n.startswith(f'backbone.blocks.{i}.'):
                check(p.grad, ge[n], n, 3e-2 if p.ndim > 1 else 6e-2)
        prev = f'block{i}_out'
    tape2 = dict(tape)
    out = rt.head_forward(trace[prev].detach().reshape(-1, C).cuda().contiguous(), tape2)
    check(out, trace['out'].detach(), 'norm + neck output', 1e-2)
    dx = rt.head_backward(trace['out'].grad.cuda().contiguous(), tape2)
    check(dx.view(B, L, C), trace[prev].grad, 'norm + neck input gradient', 2e-2)
    for n in ('backbone.norm.weight', 'backbone.norm.bias', 'neck.0.weight', 'neck.1.weight', 'neck.2.weight', 'neck.3.bias'):
        check(params[n].grad, ge[n], n, 3e-2)
    torch.cuda.synchronize()
    print(f'dinov3 blockwise: worst {sorted(report)[-3:]}')
    assert not failures, f'{len(failures)} checks failed: ' + '; '.join(failures[:12])


def test_checkpointing_gives_bit_identical_gradients_and_eval_draws_nothing():
    arch = 'dinov3_vit_small_plus_patch16_backbone'
    m1, _, x, target = _setup(arch, 48, ckpt=False)
    m2, _, _, _ = _setup(arch, 48, ckpt=True)
    assert m2.backbone.use_gradient_checkpoint
    outs = []
    for m in (m1, m2):
        torch.manual_seed(9)
        o = m(x.cuda())
        F.mse_loss(o, target.cuda()).backward()
        outs.append(o.detach())
    assert torch.equal(outs[0], outs[1])
    for (n, p), (_, q) in zip(m1.named_parameters(), m2.named_parameters()):
        assert torch.equal(p.grad, q.grad), n
    m1.eval()
    state = torch.get_rng_state()
    with torch.no_grad():
        e1 = m1(x.cuda())
        e2 = m1(x.cuda())
    assert torch.equal(torch.get_rng_state(), state) and torch.equal(e1, e2)
    # training forwards draw one factor each: different coordinates, different outputs
    m1.train()
    torch.manual_seed(1)
    with torch.no_grad():
        t1 = m1(x.cuda())
    assert not torch.equal(torch.get_rng_state(), state) and not torch.equal(t1, e1)


def test_backbone_alone_returns_fp32_nchw():
    from oracle import dinov3 as od
    from simpleaicv_pytorch_training_examples_b200.detection.models.backbones import dinov3vit
    torch.manual_seed(3)
    m = dinov3vit.DinoVisionTransformer(embedding_planes=768, block_nums=2, head_nums=12, pos_embed_rope_rescale_coords=2)
    _randomize(m, 3)
    sd = {n: v.detach().clone() for n, v in m.state_dict().items()}
    m = m.cuda().train()
    x = torch.randn(2, 3, 48, 48, generator=torch.Generator().manual_seed(5))
    target = torch.randn(2, 768, 3, 3, generator=torch.Generator().manual_seed(6))
    torch.manual_seed(2)
    fac = od.draw_rescale(2)
    oe, _, ge = od.loss_and_grads(sd, x, target, 12, fac, emulate_bf16=True)
    torch.manual_seed(2)
    out = m(x.cuda())
    F.mse_loss(out, target.cuda()).backward()
    assert out.dtype == torch.float32 and out.shape == (2, 768, 3, 3)
    assert _rel(out.detach(), oe) <= 2e-2
    assert max(_rel(p.grad, ge[n]) for n, p in m.named_parameters()) <= 8e-2


def test_distillation_trains_through_train_distill_sam_encoder(monkeypatch):
    import logging
    from simpleaicv_pytorch_training_examples_b200 import optim
    from simpleaicv_pytorch_training_examples_b200.interactive_segmentation import distill_model
    from simpleaicv_pytorch_training_examples_b200.interactive_segmentation.distill_losses import MSELoss
    from simpleaicv_pytorch_training_examples_b200.tools import interactive_segmentation_scripts as iss
    from simpleaicv_pytorch_training_examples_b200.tools import utils as tutils
    monkeypatch.setattr(tutils, 'CudaPrefetcher', lambda loader, **kw: loader)
    tea = dict(distill_model.SAM_H_TEACHER, image_size=224, block_nums=2, global_attn_indexes=[1])
    stu = dict(distill_model.DINOV3_B_STUDENT, image_size=224)
    torch.manual_seed(0)
    model = distill_model.DINOV3ImageEncoderDistillModel(teacher_params=tea, student_params=stu).cuda()
    params = [p for p in model.parameters() if p.requires_grad]
    opt = optim.FusedAdamW([{'params': params, 'weight_decay': 0.}], lr=1e-3)
    tea0 = {n: p.detach().clone() for n, p in model.teacher.named_parameters()}
    stu0 = {n: p.detach().clone() for n, p in model.student.named_parameters()}
    g = torch.Generator().manual_seed(1)
    batches = [{'image': torch.randn(2, 3, 224, 224, generator=g).cuda()} for _ in range(2)]

    class Loader(list):
        dataset = list(range(4))

    class Sched:
        current_lr = 1e-3

        def step(self, optimizer, epoch):
            pass

    class Cfg:
        accumulation_steps, batch_size, print_interval, local_rank, freeze_teacher = 1, 2, 1, 0, True

    avg = iss.train_distill_sam_encoder(Loader(batches), model, MSELoss(), opt, Sched(), 1, logging.getLogger('t'), Cfg)
    torch.cuda.synchronize()
    assert avg > 0 and not model.teacher.training and model.student.training
    for n, p in model.teacher.named_parameters():
        assert p.grad is None and torch.equal(p, tea0[n]), n
    changed = sum(not torch.equal(p, stu0[n]) for n, p in model.student.named_parameters())
    assert changed == len(stu0), f'{len(stu0) - changed} student tensors did not change'
