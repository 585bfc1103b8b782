"""DETR on the H100 runtime vs the CPU oracle (oracle/detr.py, pinned to the reference by
tests/golden/resnet18_detr_*.pt and live in tests/test_oracle_vs_reference.py).

Kernel level: post-LayerNorm forward / backward, dropout, head packing, attention with the additive key-bias column and
attention-probability dropout (masks re-derived in torch from the same counter hash) against plain torch fp32.
Model level: the transformer driven with the oracle's token stream (teacher forced: outputs, every transformer / head
parameter gradient and the stream gradient against the bf16-storage oracle), and the whole model end to end."""
import importlib.util
import os

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
_spec = importlib.util.spec_from_file_location('make_golden', os.path.join(HERE, 'golden', 'make_golden.py'))
make_golden = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(make_golden)


def _rel(a, b):
    return ((a.float().cpu() - b.float().cpu()).norm() / b.float().cpu().norm().clamp_min(1e-12)).item()


# ------------------------------------------------------------------------------------------------ counter hash in torch
def hash_keep(seed, a, b, p):
    """csrc/dropout_hash.cuh in int64 arithmetic masked to 32 bits: keep mask for index tensors a, b (int64)."""
    M = 0xFFFFFFFF
    lo, hi = seed & M, (seed >> 32) & M
    x = ((a + lo) & M) * 0x9E3779B1 & M
    x = x ^ (((b + hi) & M) * 0x85EBCA77 & M)
    x = x ^ (x >> 16)
    x = x * 0x7FEB352D & M
    x = x ^ (x >> 15)
    x = x * 0x846CA68B & M
    x = x ^ (x >> 16)
    t = min(int(p * 4294967296.0), 0xFFFFFFFF)
    return x >= t


def test_dropout_kernel_matches_hash_and_backward_is_same_mask():
    from simpleaicv_pytorch_training_examples_b200 import ops
    n, p, seed = 1 << 16, 0.1, 0x1234567890ABCDEF & ((1 << 62) - 1)
    x = torch.randn(n).bfloat16()
    idx = torch.arange(n, dtype=torch.int64)
    keep = hash_keep(seed, idx, torch.zeros_like(idx), p)
    want = torch.where(keep, x.float() / (1 - p), torch.zeros(()))
    got = ops.dropout(x.cuda(), p, seed)
    assert got.dtype == torch.bfloat16 and _rel(got, want.bfloat16()) < 1e-6
    assert abs(keep.float().mean().item() - 0.9) < 0.01
    r = torch.randn(n)
    got2 = ops.dropout(x.cuda(), p, seed, resid=r.cuda())
    assert got2.dtype == torch.float32
    torch.testing.assert_close(got2.cpu(), want + r, rtol=1e-6, atol=1e-6)
    base = torch.tensor([123456789012345], dtype=torch.int64, device='cuda')   # device-resident part of the seed
    assert torch.equal(ops.dropout(x.cuda(), p, seed - 123456789012345, seed_base=base), got)
    g = torch.randn(n)
    gb = ops.dropout(g.cuda(), p, seed, out_f32=False)          # backward of the residual-branch dropout
    assert _rel(gb, torch.where(keep, g / (1 - p), torch.zeros(())).bfloat16()) < 1e-4     # x * (1 / (1 - p)) vs x / (1 - p): 1 ulp before the bf16 rounding


@pytest.mark.parametrize('rows,c,pos_rows', [(400, 256, 100), (1000, 256, 1000), (77, 128, 7)])
def test_postln_forward_backward(rows, c, pos_rows):
    from simpleaicv_pytorch_training_examples_b200 import ops
    g = torch.Generator().manual_seed(rows)
    z = torch.randn(rows, c, generator=g) * 2 + 0.5
    gamma, beta = torch.randn(c, generator=g), torch.randn(c, generator=g)
    pos = torch.randn(pos_rows, c, generator=g)
    y, yb, ypb, stats = ops.postln_fwd(z.cuda(), gamma.cuda(), beta.cuda(), 1e-5, pos=pos.cuda(), want_ypb=True)
    zr = z.clone().requires_grad_(True)
    gr, br = gamma.clone().requires_grad_(True), beta.clone().requires_grad_(True)
    want = F.layer_norm(zr, (c,), gr, br, 1e-5)
    torch.testing.assert_close(y.cpu(), want.detach(), rtol=1e-5, atol=1e-5)
    assert torch.equal(yb.cpu(), y.cpu().bfloat16())
    wantp = (y.cpu() + pos.repeat(rows // pos_rows, 1)).bfloat16()
    assert _rel(ypb, wantp) < 1e-3
    dy = torch.randn(rows, c, generator=g)
    dres = torch.randn(rows, c, generator=g)
    want.backward(dy)
    dg, db = torch.empty(c, device='cuda'), torch.empty(c, device='cuda')
    dz, dzb = ops.postln_bwd(dy.cuda(), z.cuda(), gamma.cuda(), stats, dg, db, dres=dres.cuda())
    torch.testing.assert_close(dz.cpu(), zr.grad + dres, rtol=1e-4, atol=1e-4)
    assert torch.equal(dzb.cpu(), dz.cpu().bfloat16())
    torch.testing.assert_close(dg.cpu(), gr.grad, rtol=1e-4, atol=1e-3)
    torch.testing.assert_close(db.cpu(), br.grad, rtol=1e-4, atol=1e-3)
    dg2, db2 = dg.clone(), db.clone()
    ops.postln_bwd(dy.cuda(), z.cuda(), gamma.cuda(), stats, dg2, db2, accumulate=True, want_dz=False, want_dzb=False)
    torch.testing.assert_close(dg2.cpu(), 2 * dg.cpu(), rtol=1e-5, atol=1e-5)


def test_heads_pack_unpack():
    from simpleaicv_pytorch_training_examples_b200 import ops
    B, L, H, hd, dp = 2, 37, 8, 32, 48
    g = torch.Generator().manual_seed(3)
    src = torch.randn(B * L, 2 * H * hd, generator=g).bfloat16()
    bias = torch.randint(0, 2, (B * L,), generator=g).float()
    qe = ops.heads_pack(src.cuda(), 0, B, L, H, hd, dp, scale=hd ** -0.5, extra_const=1.0).cpu()
    ke = ops.heads_pack(src.cuda(), H * hd, B, L, H, hd, dp, extra=bias.cuda()).cpu()
    q = src[:, :H * hd].view(B, L, H, hd).permute(0, 2, 1, 3).float()
    k = src[:, H * hd:].view(B, L, H, hd).permute(0, 2, 1, 3).float()
    assert torch.equal(qe[..., :hd], (q * hd ** -0.5).bfloat16()) and torch.equal(ke[..., :hd], k.bfloat16())
    assert (qe[..., hd] == 1).all() and torch.equal(ke[..., hd].float(), bias.view(B, 1, L).expand(B, H, L))
    assert qe[..., hd + 1:].abs().max() == 0 and ke[..., hd + 1:].abs().max() == 0
    back = torch.zeros(B * L, 2 * H * hd, dtype=torch.bfloat16, device='cuda')
    ops.heads_unpack(ke.cuda(), back, H * hd, hd)
    assert torch.equal(back.cpu()[:, H * hd:], src[:, H * hd:]) and back.cpu()[:, :H * hd].abs().max() == 0


def _attn_reference(qe, ke, v, scale, keep=None, p=0.0):
    s = (qe.float() @ ke.float().transpose(-2, -1)) * scale
    a = s.softmax(-1)
    if keep is not None:
        a = torch.where(keep, a / (1 - p), torch.zeros(()))
    return a @ v.float()


@pytest.mark.parametrize('B,H,Lq,Lk,dqk,p', [(2, 8, 100, 20, 48, 0.0), (2, 8, 300, 300, 48, 0.0), (1, 8, 100, 100, 32, 0.0),
                                            (2, 8, 100, 150, 48, 0.1), (2, 4, 130, 130, 32, 0.1), (1, 2, 197, 197, 64, 0.2)])
def test_attention_bias_column_and_probability_dropout(B, H, Lq, Lk, dqk, p):
    """(48, 32): DETR's head size 32 + the key-bias column; (32, 32) / (64, 64): plain.  With p > 0 the torch reference
    uses the same counter-hash mask, so forward and all three gradients must agree to bf16 accuracy."""
    from simpleaicv_pytorch_training_examples_b200 import ops
    g = torch.Generator().manual_seed(B * 1000 + Lq + dqk)
    hd = 32 if dqk in (32, 48) else 64
    q = (torch.randn(B, H, Lq, dqk, generator=g) * 0.5).bfloat16()
    k = (torch.randn(B, H, Lk, dqk, generator=g) * 0.5).bfloat16()
    if dqk == 48:
        q[..., hd] = 1.0
        k[..., hd] = torch.randint(0, 2, (B, 1, Lk), generator=g).float().expand(B, H, Lk)
        q[..., hd + 1:] = 0
        k[..., hd + 1:] = 0
    v = torch.randn(B, H, Lk, hd, generator=g).bfloat16()
    scale = 1.0 if dqk == 48 else hd ** -0.5
    seed = 0x0ABCDEF012345 + Lq
    keep = None
    if p > 0:
        rows = (torch.arange(B * H).view(B, H, 1, 1) * Lq + torch.arange(Lq).view(1, 1, Lq, 1)).expand(B, H, Lq, Lk)
        cols = torch.arange(Lk).view(1, 1, 1, Lk).expand(B, H, Lq, Lk)
        keep = hash_keep(seed, rows.to(torch.int64), cols.to(torch.int64), p)
    qr, kr, vr = (t.float().requires_grad_(True) for t in (q, k, v))
    want = _attn_reference(qr, kr, vr, scale, keep, p)
    do = torch.randn(B, H, Lq, hd, generator=g).bfloat16()
    want.backward(do.float())
    qc, kc, vc = q.cuda(), k.cuda(), v.cuda()
    out, lse = ops.attn_fwd(qc, kc, vc, scale, dropout_p=p, dropout_seed=seed)
    assert _rel(out, want.detach()) < 1.5e-2, _rel(out, want.detach())
    if p > 0:   # the same seed split into a launch constant and a device-resident base gives the same masks
        base = torch.tensor([seed - 77], dtype=torch.int64, device='cuda')
        out2, _ = ops.attn_fwd(qc, kc, vc, scale, dropout_p=p, dropout_seed=77, dropout_seed_base=base)
        assert torch.equal(out2, out)
    dq, dk, dv = torch.zeros_like(qc), torch.zeros_like(kc), torch.empty_like(vc)
    doc = do.cuda().permute(0, 2, 1, 3).contiguous().permute(0, 2, 1, 3)      # the layout of `out` ([B, L, H, D] storage)
    ops.attn_bwd(qc, kc, vc, out, lse, doc, scale, dq, dk, dv, dk_cols=hd if dqk == 48 else 0, dropout_p=p, dropout_seed=seed)
    assert _rel(dv, vr.grad) < 2e-2, _rel(dv, vr.grad)
    assert _rel(dq[..., :hd], qr.grad[..., :hd]) < 2e-2, _rel(dq[..., :hd], qr.grad[..., :hd])
    assert _rel(dk[..., :hd], kr.grad[..., :hd]) < 2e-2, _rel(dk[..., :hd], kr.grad[..., :hd])


# ------------------------------------------------------------------------------------------------ model level
def _setup(seed=3, shape=(2, 3, 128, 160)):
    from simpleaicv_pytorch_training_examples_b200.detection import models
    sd = make_golden.oracle_init('detr', 'resnet18_detr', {}, 80, seed)
    torch.manual_seed(seed)
    model = models.resnet18_detr().cuda().train()
    model.transformer.dropout_prob = 0.0
    msd = model.state_dict()
    assert all(torch.equal(msd[k].cpu(), sd[k]) for k in sd)        # same seeded initialisation as the reference
    g = torch.Generator().manual_seed(77)
    x = torch.randn(*shape, generator=g)
    return sd, model, x, make_golden.detr_masks(shape)


def test_detr_transformer_teacher_forced():
    """Transformer + heads driven with the oracle's token stream: outputs, the gradient of the stream and every
    transformer / head parameter gradient against the bf16-storage oracle (5e-2 relative L2; the few tensors whose
    gradient bf16 storage itself perturbs by more than that - the box-head MLP and the query embedding, 11-16 % between
    the fp32 and the bf16-storage oracle - are held to that perturbation)."""
    from oracle import detr as od
    sd, model, x, masks = _setup()
    trace = {}
    sd32 = {n: v.clone() for n, v in sd.items()}
    _, _, _, g32 = od.loss_and_grads(sd32, x, masks, 'resnet18_detr')
    cls_e, reg_e, _, ge = od.loss_and_grads(sd, x, masks, 'resnet18_detr', emulate_bf16=True, trace=trace)
    rt = model._runtime()
    rt.prep()
    src = trace['src'].detach()
    B, L, C = src.shape
    fm = od.resize_masks(masks, *trace['c5'].shape[2:])
    pos = od.position_embedding(fm).flatten(2).transpose(1, 2).reshape(B * L, C).contiguous().cuda()
    key_bias = fm.flatten(1).float().reshape(-1).cuda()
    cx = rt._context(B, L, pos, key_bias, True)
    tape = {}
    cls, reg = rt.transformer_forward(src.reshape(B * L, C).contiguous().cuda(), cx, tape)
    assert _rel(cls, cls_e) < 2e-2, _rel(cls, cls_e)
    assert _rel(reg.sigmoid(), reg_e) < 1e-2, _rel(reg.sigmoid(), reg_e)
    dcls = trace['cls'].grad
    dreg = trace['reg'].grad * reg_e * (1 - reg_e)                  # through the sigmoid, at the oracle's values
    dsrc = rt.transformer_backward(dcls.cuda(), dreg.cuda(), cx, tape)
    torch.cuda.synchronize()
    assert _rel(dsrc.view(B, L, C), trace['src'].grad) < 5e-2, _rel(dsrc.view(B, L, C), trace['src'].grad)
    bad, worst = [], (0.0, '')
    for n, p in model.named_parameters():
        if n.startswith('backbone.') or n.startswith('proj_conv.'):
            continue
        assert p.grad is not None, n
        r = _rel(p.grad, ge[n]) if ge[n].norm() > 0 else float(p.grad.abs().max())
        noise = _rel(ge[n], g32[n]) if g32[n].norm() > 0 else 0.0     # what bf16 storage alone does to this tensor
        worst = max(worst, (r, n))
        if r > max(5e-2, noise):
            bad.append((n, r, noise))
    print(f'detr transformer (teacher forced): cls rel L2 {_rel(cls, cls_e):.4g}, dsrc {_rel(dsrc.view(B, L, C), trace["src"].grad):.4g}, '
          f'worst parameter gradient {worst}')
    assert not bad, bad[:10]


def test_detr_step_matches_oracle_end_to_end():
    from oracle import detr as od
    sd, model, x, masks = _setup()
    sd32 = {n: v.clone() for n, v in sd.items()}
    c32, r32, _, g32 = od.loss_and_grads(sd32, x, masks, 'resnet18_detr')
    ce, re_, _, ge = od.loss_and_grads(sd, x, masks, 'resnet18_detr', emulate_bf16=True)
    cls, reg = model(x.cuda(), masks.cuda())
    od.surrogate_loss(cls, reg).backward()
    torch.cuda.synchronize()
    assert cls.shape == c32.shape and reg.shape == r32.shape and cls.dtype == torch.float32
    noise_c, noise_r = _rel(ce, c32), _rel(re_, r32)
    assert _rel(cls.detach(), c32) <= 2.5 * noise_c + 1e-2, (_rel(cls.detach(), c32), noise_c)
    assert _rel(reg.detach(), r32) <= 2.5 * noise_r + 1e-2, (_rel(reg.detach(), r32), noise_r)
    grads = {n: p.grad.detach().float().cpu() for n, p in model.named_parameters()}
    assert set(grads) == set(g32)
    tr = [n for n in g32 if not n.startswith('backbone.')]
    cat = lambda d, names: torch.cat([d[n].flatten() for n in names])
    mine_t, emu_t = _rel(cat(grads, tr), cat(g32, tr)), _rel(cat(ge, tr), cat(g32, tr))
    mine_all, emu_all = _rel(cat(grads, list(g32)), cat(g32, list(g32))), _rel(cat(ge, list(g32)), cat(g32, list(g32)))
    print(f'detr end to end: cls rel L2 to fp32 {_rel(cls.detach(), c32):.4g} (storage noise {noise_c:.4g}); transformer+head gradient '
          f'{mine_t:.4g} (noise {emu_t:.4g}); whole gradient {mine_all:.4g} (noise {emu_all:.4g})')
    # the random-init BatchNorm body amplifies bf16 storage noise (DESIGN.md "Parity"): bounded by the oracle's own noise
    assert mine_t <= 2.0 * emu_t + 5e-2, (mine_t, emu_t)
    assert mine_all <= 2.0 * emu_all + 5e-2, (mine_all, emu_all)
    # running statistics of the body moved like the reference's
    torch.testing.assert_close(model.state_dict()['backbone.conv1.layer.1.running_mean'].cpu(), sd32['backbone.conv1.layer.1.running_mean'],
                               rtol=2e-2, atol=2e-3)


def test_detr_eval_determinism_and_dropout_training():
    sd, model, x, masks = _setup(shape=(2, 3, 96, 128))
    xc, mc = x.cuda(), masks.cuda()
    model.eval()
    with torch.no_grad():
        a = model(xc, mc)
        b = model(xc, mc)
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])
    # training with the reference's dropout 0.1: runs, is reproducible under the same torch seed, differs across seeds
    model.train()
    model.transformer.dropout_prob = 0.1
    outs = []
    for seed in (5, 5, 6):
        torch.manual_seed(seed)
        for p in model.parameters():
            p.grad = None
        cls, reg = model(xc, mc)
        (cls.float().square().mean() + reg.mean()).backward()
        outs.append((cls.detach().clone(), model.transformer.decoder_norm.weight.grad.clone()))
    assert torch.equal(outs[0][0], outs[1][0]) and torch.equal(outs[0][1], outs[1][1])
    assert not torch.equal(outs[0][0], outs[2][0])
    assert torch.isfinite(outs[2][1]).all()
    with pytest.raises(RuntimeError):
        model(x, masks)                                           # CPU tensors: there is no fallback path


def test_detr_split_graph_step_matches_eager_steps():
    """graph.GraphedSplitStep (forward graph + eager DETRLoss with the host-side Hungarian matcher + backward / optimizer
    graph) reproduces eager training steps bit for bit (dropout 0: same kernels, same order, same inputs)."""
    from simpleaicv_pytorch_training_examples_b200.detection import models
    from simpleaicv_pytorch_training_examples_b200.detection.losses import DETRLoss
    from simpleaicv_pytorch_training_examples_b200.graph import GraphedSplitStep
    shape = (2, 3, 128, 160)
    g = torch.Generator().manual_seed(5)
    xs = [torch.randn(*shape, generator=g).cuda() for _ in range(3)]
    masks = make_golden.detr_masks(shape).cuda()
    ann = torch.cat([torch.rand(2, 4, 2, generator=g) * 0.6 + 0.2, torch.rand(2, 4, 2, generator=g) * 0.3 + 0.05,
                     torch.randint(0, 80, (2, 4, 1), generator=g).float()], dim=2).cuda()
    crit = DETRLoss().cuda()

    def build():
        torch.manual_seed(3)
        m = models.resnet18_detr().cuda().train()
        m.transformer.dropout_prob = 0.0
        return m, torch.optim.AdamW(m.parameters(), lr=1e-4, capturable=True)

    m1, o1 = build()
    eager = []
    for i in range(6):                       # 3 warm-up steps (the graphed step warms up on its example batch) + 3 compared
        out = m1(xs[0] if i < 3 else xs[i - 3], masks)
        loss = sum(crit(out, ann).values())
        loss.backward()
        o1.step()
        o1.zero_grad()
        eager.append(float(loss))
    m2, o2 = build()
    step = GraphedSplitStep(lambda x: m2(x, masks), crit, o2, [xs[0]], ann)
    graphed = [float(step([x], ann)) for x in xs]
    assert graphed == eager[3:], (graphed, eager[3:])
    for (n, p), (_, q) in zip(m1.named_parameters(), m2.named_parameters()):
        assert torch.equal(p, q), n
