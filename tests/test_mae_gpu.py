"""MAE pre-training on the H100 runtime (SURVEY.md 8 f4): the token gather / scatter kernels against torch.gather, and the
whole training step (masking, encoder, un-shuffle, decoder, MSELoss on removed patches, backward) against the CPU oracle
(oracle/mae.py, pinned to the reference by tests/test_mae_cpu.py) with the masks pinned through the noise input.
Tolerances as tests/test_vit_gpu.py: outputs vs the bf16-storage oracle, gradients bounded by the bf16 storage noise."""
import pytest
import torch

pytestmark = pytest.mark.gpu
ARCH = 'vit_base_patch16_224_mae_pretrain_model'


def _rel_l2(a, b):
    return ((a.float().cpu() - b.float().cpu()).norm() / b.float().cpu().norm().clamp_min(1e-12)).item()


def test_token_gather_and_scatter_match_torch():
    from simpleaicv_pytorch_training_examples_b200 import ops
    g = torch.Generator(device='cuda').manual_seed(0)
    b, s, c, keep = 5, 37, 96, 9
    src = torch.randn(b, s, c, device='cuda', generator=g)
    fill = torch.randn(c, device='cuda', generator=g)
    pos = torch.randn(s + 1, c, device='cuda', generator=g)
    perm = torch.stack([torch.randperm(s, device='cuda', generator=g) for _ in range(b)])
    keep_ids = perm[:, :keep]
    # encoder form: row 0 = fill + pos[0], rows 1.. = src[keep] + pos[1 + keep]
    idx = torch.cat([torch.full((b, 1), -1, device='cuda'), keep_ids], 1).to(torch.int32).contiguous()
    pidx = torch.cat([torch.zeros(b, 1, device='cuda', dtype=torch.int64), keep_ids + 1], 1).to(torch.int32).contiguous()
    out = ops.token_gather_fwd(src, idx, fill, pos=pos, pos_idx=pidx)
    ref = torch.cat([fill.expand(b, 1, c), torch.gather(src, 1, keep_ids.unsqueeze(-1).repeat(1, 1, c))], 1) + pos[pidx.long()]
    assert torch.equal(out, ref)
    dout = torch.randn(b, keep + 1, c, device='cuda', generator=g)
    for dt in (torch.float32, torch.bfloat16):
        dsrc, dfill = ops.token_gather_bwd(dout, idx, s, dsrc_dtype=dt, zero=True)
        want = torch.zeros(b, s, c, device='cuda')
        want.scatter_(1, keep_ids.unsqueeze(-1).repeat(1, 1, c), dout[:, 1:])
        assert torch.equal(dsrc, want.to(dt))
        torch.testing.assert_close(dfill, dout[:, 0].sum(0), rtol=1e-5, atol=1e-5)
    # decoder form: un-shuffle with mask tokens, position = row
    restore = torch.argsort(perm, dim=1)
    y = torch.randn(b, keep + 1, c, device='cuda', generator=g)
    didx = torch.cat([torch.zeros(b, 1, device='cuda', dtype=torch.int64), torch.where(restore < keep, restore + 1, -1)], 1).to(torch.int32).contiguous()
    out = ops.token_gather_fwd(y, didx, fill, pos=pos)
    y_ = torch.cat([y[:, 1:], fill.expand(b, s - keep, c)], 1)
    ref = torch.cat([y[:, :1], torch.gather(y_, 1, restore.unsqueeze(-1).repeat(1, 1, c))], 1) + pos
    assert torch.equal(out, ref)
    dout = torch.randn(b, s + 1, c, device='cuda', generator=g)
    dy, dmask = ops.token_gather_bwd(dout, didx, keep + 1, dsrc_dtype=torch.float32, zero=False)
    yl = y.clone().requires_grad_(True)
    fl = fill.clone().requires_grad_(True)
    y2 = torch.cat([yl[:, 1:], fl.expand(b, s - keep, c)], 1)
    r2 = torch.cat([yl[:, :1], torch.gather(y2, 1, restore.unsqueeze(-1).repeat(1, 1, c))], 1) + pos
    r2.backward(dout)
    assert torch.equal(dy, yl.grad)
    torch.testing.assert_close(dmask, fl.grad, rtol=1e-5, atol=1e-5)


@pytest.mark.parametrize('image_size,batch,enc,dec,ckpt', [(64, 4, 2, 2, False), (96, 3, 3, 2, True)])
def test_mae_step_matches_oracle(image_size, batch, enc, dec, ckpt):
    from oracle import mae
    from simpleaicv_pytorch_training_examples_b200.masked_image_modeling import losses
    from simpleaicv_pytorch_training_examples_b200.masked_image_modeling.models import vit_mae
    g = torch.Generator().manual_seed(11)
    x = torch.randn(batch, 3, image_size, image_size, generator=g)
    n = (image_size // 16) ** 2
    noise = torch.rand(batch, n, generator=g)
    sd = mae.init_state(ARCH, 2, image_size=image_size, enc_depth=enc, dec_depth=dec)
    sd32 = {k: v.clone() for k, v in sd.items()}
    p32, m32, l32, g32 = mae.loss_and_grads(sd32, x, noise, ARCH, enc_depth=enc, dec_depth=dec)
    pe, me, le, ge = mae.loss_and_grads(sd, x, noise, ARCH, emulate_bf16=True, enc_depth=enc, dec_depth=dec)
    torch.manual_seed(2)
    model = vit_mae.VITMAEPretrainModel(patch_size=16, image_size=image_size, encoder_embedding_planes=768, encoder_block_nums=enc,
                                        encoder_head_nums=12, decoder_embedding_planes=512, decoder_block_nums=dec,
                                        decoder_head_nums=16, use_gradient_checkpoint=ckpt).cuda().train()
    for k, v in model.state_dict().items():
        assert torch.equal(v.cpu(), sd[k]), k
    xd = x.cuda()
    pred, mask = model(xd, noise=noise.cuda())
    assert torch.equal(mask.cpu(), me)                          # index work: bit exact
    loss = losses.MSELoss()(pred, model.images_to_patch(xd), mask)
    loss.backward()
    torch.cuda.synchronize()
    assert _rel_l2(pred.detach(), pe) <= 3e-2, _rel_l2(pred.detach(), pe)
    assert abs(float(loss.detach()) - float(le)) <= 5e-3 * abs(float(le))
    worst = (0., None)
    for name, p in model.named_parameters():
        if not p.requires_grad:
            assert p.grad is None, name
            continue
        assert p.grad is not None, name
        mine, emu = _rel_l2(p.grad, g32[name]), _rel_l2(ge[name], g32[name])
        worst = max(worst, (_rel_l2(p.grad, ge[name]), name))
        assert mine <= 2.0 * emu + 5e-2, f'{name}: rel L2 to fp32 {mine:.4g} vs bf16-storage noise {emu:.4g}'
    print(f'mae {image_size}px b{batch}: pred rel L2 {_rel_l2(pred.detach(), pe):.4g}, worst grad vs bf16-storage oracle {worst}')
    # eval forward: same masks, no tape
    model.eval()
    with torch.no_grad():
        pred2, mask2 = model(xd, noise=noise.cuda())
    assert torch.equal(mask2, mask) and _rel_l2(pred2, pred.detach()) <= 1e-6


def test_mae_trains_with_fused_adamw_and_seeded_masks():
    """Three optimizer steps through tools.utils.build_optimizer (fused AdamW): the loss goes down and a seeded run draws the
    same masks twice (torch.rand on the device, as the reference)."""
    from simpleaicv_pytorch_training_examples_b200 import optim
    from simpleaicv_pytorch_training_examples_b200.masked_image_modeling import losses
    from simpleaicv_pytorch_training_examples_b200.masked_image_modeling.models import vit_mae
    from simpleaicv_pytorch_training_examples_b200.tools import utils as tutils

    class Cfg:
        optimizer = ('AdamW', {'lr': 1e-3, 'global_weight_decay': False, 'weight_decay': 0.05, 'no_weight_decay_layer_name_list': []})
    torch.manual_seed(0)
    model = vit_mae.VITMAEPretrainModel(patch_size=16, image_size=64, encoder_embedding_planes=768, encoder_block_nums=2,
                                        encoder_head_nums=12, decoder_embedding_planes=512, decoder_block_nums=1,
                                        decoder_head_nums=16).cuda().train()
    opt, _ = tutils.build_optimizer(Cfg, model)
    assert isinstance(opt, optim.FusedAdamW)
    x = torch.randn(8, 3, 64, 64, device='cuda')
    crit = losses.MSELoss()
    torch.manual_seed(5)
    _, m1 = model(x)
    torch.manual_seed(5)
    _, m2 = model(x)
    assert torch.equal(m1, m2) and int(m1.sum()) == 8 * 12
    vals = []
    for _ in range(4):
        torch.manual_seed(5)
        pred, mask = model(x)
        loss = crit(pred, model.images_to_patch(x), mask)
        loss.backward()
        opt.step()
        opt.zero_grad()
        vals.append(float(loss))
    assert vals[-1] < vals[0], vals
