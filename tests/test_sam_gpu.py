"""SAM ViT image encoder on the H100 runtime vs the CPU oracle (oracle/sam_encoder.py, pinned to the reference by
tests/golden/sam_enc_*.pt and live in tests/test_oracle_vs_reference.py): kernel-level parity of the window
partition / rel-pos kernels against plain torch, block-by-block parity driven with the oracle's boundary tensors
(windowed blocks with padding and a global block), and an end-to-end forward / backward.  pos_embed and the rel-pos
tables (zero at init) are randomised so that they matter."""
import importlib.util
import os

import pytest
import torch

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
_spec = importlib.util.spec_from_file_location('make_golden', os.path.join(HERE, 'golden', 'make_golden.py'))
make_golden = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(make_golden)


def _rel(a, b):
    return ((a.float().cpu() - b.float().cpu()).norm() / b.float().cpu().norm().clamp_min(1e-12)).item()


@pytest.mark.parametrize('B,H,W,C,ws', [(2, 20, 20, 128, 14), (1, 28, 28, 64, 14), (3, 9, 7, 32, 4)])
def test_window_partition_roundtrip_matches_reference_semantics(B, H, W, C, ws):
    from oracle import sam_encoder as se
    from simpleaicv_pytorch_training_examples_b200 import ops
    x = torch.randn(B, H, W, C).bfloat16()
    win, (nwy, nwx) = ops.window_partition(x.cuda(), ws)
    ref, pad_hw = se.window_partition(x.float(), ws)
    assert torch.equal(win.float().cpu().view(ref.shape), ref)
    back = ops.window_unpartition(win, B, H, W, ws)
    assert torch.equal(back.cpu(), x)
    assert torch.equal(se.window_unpartition(ref, ws, pad_hw, (H, W)), x.float())


@pytest.mark.parametrize('hd,S,heads', [(64, 14, 2), (80, 14, 2), (64, 20, 1), (80, 20, 2), (32, 5, 3)])
def test_relpos_columns_forward_backward(hd, S, heads):
    from oracle import sam_encoder as se
    from simpleaicv_pytorch_training_examples_b200 import ops
    g = torch.Generator().manual_seed(hd + S)
    Bw, L = 3, S * S
    qkv = torch.randn(Bw, L, 3, heads, hd, generator=g).bfloat16()
    rph, rpw = torch.randn(2 * S - 1, hd, generator=g) * 0.3, torch.randn(2 * S - 1, hd, generator=g) * 0.3
    scale = hd ** -0.5
    qe, ke = ops.relpos_build(qkv.cuda(), rph.cuda(), rpw.cuda(), Bw, heads, hd, S, S, scale)
    q = qkv[:, :, 0].permute(0, 2, 1, 3).float()          # [Bw, heads, L, hd]
    k = qkv[:, :, 1].permute(0, 2, 1, 3).float()
    rq = q.reshape(Bw * heads, S, S, hd)
    Rh, Rw = se._rel_table(S, rph.bfloat16().float()), se._rel_table(S, rpw.bfloat16().float())
    rel_h = torch.einsum('bhwc,hkc->bhwk', rq, Rh)
    rel_w = torch.einsum('bhwc,wkc->bhwk', rq, Rw)
    want = ((q * scale) @ k.transpose(-2, -1)).view(-1, S, S, S, S) + rel_h[..., None] + rel_w[:, :, :, None, :]
    got = (qe.float() @ ke.float().transpose(-2, -1)).cpu().view(-1, S, S, S, S)
    assert (got - want).abs().max().item() <= 3e-2 * max(1.0, want.abs().max().item())
    assert qe[..., hd + 2 * S:].abs().max().item() == 0 and ke[..., hd + 2 * S:].abs().max().item() == 0
    # backward: d(qe) -> dq, d rel_pos tables
    dqe = torch.randn(qe.shape, generator=g).bfloat16()
    dqkv = torch.zeros_like(qkv).cuda()
    dh, dw = torch.empty(2 * S - 1, hd, device='cuda'), torch.empty(2 * S - 1, hd, device='cuda')
    ops.relpos_bwd(dqe.cuda(), qkv.cuda(), rph.cuda(), rpw.cuda(), dqkv, dh, dw, Bw, heads, hd, S, S, scale)
    qr = q.clone().requires_grad_(True)
    rphr, rpwr = rph.bfloat16().float().requires_grad_(True), rpw.bfloat16().float().requires_grad_(True)
    rq = qr.reshape(Bw * heads, S, S, hd)
    cols = torch.cat([qr * scale,
                      torch.einsum('bhwc,hkc->bhwk', rq, se._rel_table(S, rphr)).reshape(Bw, heads, L, S),
                      torch.einsum('bhwc,wkc->bhwk', rq, se._rel_table(S, rpwr)).reshape(Bw, heads, L, S)], dim=-1)
    (cols * dqe.float()[..., :hd + 2 * S]).sum().backward()
    assert _rel(dqkv[:, :, 0].permute(0, 2, 1, 3), qr.grad) <= 1e-2
    assert _rel(dh, rphr.grad) <= 1e-3 and _rel(dw, rpwr.grad) <= 1e-3
    dh2 = dh.clone()
    ops.relpos_bwd(dqe.cuda(), qkv.cuda(), rph.cuda(), rpw.cuda(), dqkv, dh2, dw, Bw, heads, hd, S, S, scale, accumulate=True)
    assert _rel(dh2, 2 * rphr.grad) <= 1e-3


CFGS = {'e128': dict(image_size=320, patch_size=16, embedding_planes=128, block_nums=3, head_nums=2, out_planes=256, window_size=14,
                     global_attn_indexes=(1,)),
        'e1280': dict(image_size=320, patch_size=16, embedding_planes=1280, block_nums=2, head_nums=16, out_planes=256, window_size=14,
                      global_attn_indexes=(1,))}


def _setup(cfg, batch, seed=8):
    from simpleaicv_pytorch_training_examples_b200.interactive_segmentation.models.segment_anything.image_encoder import ViTImageEncoder
    k = CFGS[cfg]
    sd = make_golden.oracle_init('sam', 'ViTImageEncoder', k, 0, seed)
    make_golden.sam_randomize(sd, seed)
    torch.manual_seed(seed)
    model = ViTImageEncoder(**k).cuda().train()
    with torch.no_grad():
        for n, p in model.named_parameters():
            p.copy_(sd[n])
    g = torch.Generator().manual_seed(77)
    x = torch.randn(batch, 3, k['image_size'], k['image_size'], generator=g)
    grid = k['image_size'] // k['patch_size']
    proj = torch.randn(batch, k['out_planes'], grid, grid, generator=g)
    return k, sd, model, x, proj


@pytest.mark.parametrize('cfg', ['e128', 'e1280'])
def test_sam_encoder_step_matches_oracle(cfg):
    from oracle import sam_encoder as se
    k, sd, model, x, proj = _setup(cfg, 2)
    args = (k['head_nums'], k['window_size'], k['global_attn_indexes'], k['patch_size'])
    sd32 = {n: v.clone() for n, v in sd.items()}
    o32, l32, g32 = se.loss_and_grads(sd32, x, proj, *args)
    oe, le, ge = se.loss_and_grads(sd, x, proj, *args, emulate_bf16=True)
    out = model(x.cuda())
    loss = (out.float() * proj.cuda()).mean()
    loss.backward()
    torch.cuda.synchronize()
    noise = _rel(oe, o32)
    assert out.shape == o32.shape and out.dtype == torch.float32
    assert _rel(out.detach(), oe) <= 2.5 * noise + 1e-2, (_rel(out.detach(), oe), noise)
    grads = {n: p.grad.detach().float().cpu() for n, p in model.named_parameters()}
    assert set(grads) == set(g32)
    cat = lambda d: torch.cat([d[n].flatten() for n in g32])
    mine_all, emu_all = _rel(cat(grads), cat(g32)), _rel(cat(ge), cat(g32))
    assert mine_all <= 2.0 * emu_all + 5e-2, (mine_all, emu_all)
    worst = max((_rel(grads[n], ge[n]), n) for n in g32)
    print(f'sam encoder {cfg}: out rel L2 {_rel(out.detach(), oe):.4g} (storage noise {noise:.4g}); whole-gradient rel L2 to fp32 '
          f'{mine_all:.4g} (storage noise {emu_all:.4g}); worst tensor vs emulated oracle {worst}')
    assert worst[0] <= 8e-2, worst


def test_sam_encoder_blockwise_parity_with_oracle_tensors():
    from oracle import sam_encoder as se
    k, sd, model, x, proj = _setup('e128', 2)
    trace = {}
    _, _, ge = se.loss_and_grads(sd, x, proj, k['head_nums'], k['window_size'], k['global_attn_indexes'], k['patch_size'],
                                 emulate_bf16=True, trace=trace)
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
    tok = rt.embed_forward(x.cuda(), tape)
    B, H, W = tape['B'], tape['H'], tape['W']
    C = k['embedding_planes']
    check(tok.view(B, H, W, C), trace['tokens'].detach(), 'tokens', 1e-2)
    dtok = trace['tokens'].grad.reshape(-1, C).cuda().contiguous()
    rt.embed_backward(dtok, dtok.to(torch.bfloat16), tape)
    for n in ('pos_embed', 'patch_embed.proj.weight', 'patch_embed.proj.bias'):
        check(params[n].grad, ge[n], n, 2e-2)
    prev = 'tokens'
    for i, blk in enumerate(rt.blocks):
        t = {}
        out = blk.forward(trace[prev].detach().reshape(-1, C).cuda().contiguous(), t, B, H, W)
        ref_out = trace[f'block{i}_out']
        check(out.view(B, H, W, C), ref_out.detach(), f'block{i} output', 1e-2)
        dout = ref_out.grad.reshape(-1, C).cuda().contiguous()
        dx, _ = blk.backward(dout, dout.to(torch.bfloat16), t, B, H, W, rt.sink)
        check(dx.view(B, H, W, C), trace[prev].grad, f'block{i} input gradient', 2e-2)
        for n, p in params.items():
            if n.startswith(f'blocks.{i}.'):
                check(p.grad, ge[n], n, 3e-2 if p.ndim > 1 else 6e-2)
        prev = f'block{i}_out'
    tape2 = dict(tape)
    out = rt.neck_forward(trace[prev].detach().reshape(-1, C).cuda().contiguous(), tape2)
    check(out, trace['out'].detach(), 'neck output', 1e-2)
    dx, _ = rt.neck_backward(trace['out'].grad.cuda(), tape2)
    check(dx.view(B, H, W, C), trace[prev].grad, 'neck input gradient', 2e-2)
    for n in ('neck.0.weight', 'neck.1.weight', 'neck.1.bias', 'neck.2.weight', 'neck.3.weight', 'neck.3.bias'):
        check(params[n].grad, ge[n], n, 3e-2)
    torch.cuda.synchronize()
    print(f'sam blockwise: worst {sorted(report)[-3:]}')
    assert not failures, f'{len(failures)} checks failed: ' + '; '.join(failures[:12])


def test_sam_constructors_and_checkpointing():
    """sam_b-style constructor surface; use_gradient_checkpoint gives bit-identical gradients (deterministic kernels)."""
    from simpleaicv_pytorch_training_examples_b200.interactive_segmentation.models.segment_anything import sam
    torch.manual_seed(0)
    m1 = sam.sam_b(image_size=224, image_encoder_block_nums=2, image_encoder_global_attn_indexes=[1]).cuda().train()
    torch.manual_seed(0)
    m2 = sam.sam_b(image_size=224, image_encoder_block_nums=2, image_encoder_global_attn_indexes=[1], use_gradient_checkpoint=True).cuda().train()
    assert list(m1.state_dict().keys())[0] == 'image_encoder.pos_embed'
    g = torch.Generator().manual_seed(1)
    with torch.no_grad():
        for (n, p), (_, q) in zip(m1.named_parameters(), m2.named_parameters()):
            if 'rel_pos' in n or n.endswith('pos_embed'):
                p.copy_(torch.randn(p.shape, generator=g) * 0.1)
            q.copy_(p)
    x = torch.randn(2, 3, 224, 224, generator=g).cuda()
    o1 = m1.forward_image_encoder(x)
    o1.square().mean().backward()
    o2 = m2.forward_image_encoder(x)
    o2.square().mean().backward()
    assert o1.shape == (2, 256, 14, 14) and torch.equal(o1, o2)
    for (n, p), (_, q) in zip(m1.named_parameters(), m2.named_parameters()):
        assert torch.equal(p.grad, q.grad), n
    with pytest.raises(NotImplementedError):
        m1(x, None, None)
