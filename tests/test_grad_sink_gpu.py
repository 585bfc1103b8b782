"""Every runtime family writes its parameter gradients through its GradSink (engine/runtime.py): one training backward
reports each trainable parameter to on_ready exactly once and leaves .grad in the sink's own buffer, and a second backward
of the same seeded forward without zero_grad doubles every gradient (an ignored or misapplied accumulate flag leaves the
first gradient, or garbage).

Each family runs one small configuration built the way its model tests build it; torch.manual_seed before each forward
repeats the random draws of the step (drop path, dropout, MAE's mask noise, the DINOv3 RoPE rescale factor), and
BatchNorm normalizes with batch statistics in training, so the second backward computes the first one's gradient again."""
import pytest
import torch

pytestmark = pytest.mark.gpu


def _proj_loss(outs, seed=77):
    """sum(out * fixed random projection) over the differentiable outputs: every output element gets a gradient."""
    g = torch.Generator().manual_seed(seed)
    return sum((o.float() * torch.randn(o.shape, generator=g).cuda()).sum() for o in outs)


def _classifier(name, **kw):
    from simpleaicv_pytorch_training_examples_b200.classification import backbones
    model = backbones.__dict__[name](num_classes=10, **kw).cuda().train()
    x = torch.randn(4, 3, 64, 64, generator=torch.Generator().manual_seed(1)).cuda()
    return model, lambda: _proj_loss([model(x)])


def _sam_encoder():
    from simpleaicv_pytorch_training_examples_b200.interactive_segmentation.models.segment_anything.image_encoder import ViTImageEncoder
    model = ViTImageEncoder(image_size=320, patch_size=16, embedding_planes=128, block_nums=2, head_nums=2, out_planes=256,
                            window_size=14, global_attn_indexes=(1,)).cuda().train()
    x = torch.randn(1, 3, 320, 320, generator=torch.Generator().manual_seed(1)).cuda()
    return model, lambda: _proj_loss([model(x)])


def _dinov3_encoder():
    from simpleaicv_pytorch_training_examples_b200.interactive_segmentation.models.dinov3_segment_anything import DINOV3ViTImageEncoder
    model = DINOV3ViTImageEncoder('dinov3_vit_small_patch16_backbone', image_size=64).cuda().train()
    x = torch.randn(2, 3, 64, 64, generator=torch.Generator().manual_seed(1)).cuda()
    return model, lambda: _proj_loss([model(x)])


def _mae():
    from simpleaicv_pytorch_training_examples_b200.masked_image_modeling.models import vit_mae
    model = vit_mae.VITMAEPretrainModel(patch_size=16, image_size=64, encoder_embedding_planes=768, encoder_block_nums=2,
                                        encoder_head_nums=12, decoder_embedding_planes=512, decoder_block_nums=1,
                                        decoder_head_nums=16).cuda().train()
    x = torch.randn(2, 3, 64, 64, generator=torch.Generator().manual_seed(1)).cuda()
    return model, lambda: _proj_loss([model(x)[0]])                 # the mask is not differentiable


def _detr():
    from simpleaicv_pytorch_training_examples_b200.detection import models
    model = models.resnet18_detr().cuda().train()                   # the reference's dropout 0.1
    x = torch.randn(2, 3, 128, 160, generator=torch.Generator().manual_seed(1)).cuda()
    masks = torch.zeros(2, 128, 160, dtype=torch.bool, device='cuda')
    masks[0, :, 120:] = True
    return model, lambda: _proj_loss(model(x, masks))


FAMILIES = {
    'resnet18': lambda: _classifier('resnet18'),
    'darknettiny': lambda: _classifier('darknettiny'),
    'van_b0': lambda: _classifier('van_b0'),
    'convformer_s18_drop_path': lambda: _classifier('convformer_s18', drop_path_prob=0.2),
    'vit_drop_path_dropout': lambda: _classifier('vit_base_patch16', image_size=64, drop_path_prob=0.1, dropout_prob=0.1),
    'sam_encoder': _sam_encoder,
    'dinov3_small_encoder': _dinov3_encoder,
    'mae': _mae,
    'detr_r18': _detr,
}


def _backward(model, loss_fn, seed):
    """One seeded training forward / backward; returns the names of the parameters on_ready reported, in order."""
    names = {id(p): n for n, p in model.named_parameters()}
    reported = []
    model.grad_sink().on_ready = lambda p: reported.append(names[id(p)])
    torch.manual_seed(seed)
    loss_fn().backward()
    torch.cuda.synchronize()
    return reported


@pytest.mark.parametrize('family', list(FAMILIES))
def test_every_gradient_goes_through_the_sink_once_and_accumulates(family):
    torch.manual_seed(0)
    model, loss_fn = FAMILIES[family]()
    sink = model.grad_sink()
    # every trainable parameter is reported (MAE's frozen sine-cosine position embeddings are not trainable)
    trainable = {n: p for n, p in model.named_parameters() if p.requires_grad}
    for p in model.parameters():
        p.grad = None

    reported = _backward(model, loss_fn, seed=5)
    assert len(reported) == len(set(reported)), sorted({n for n in reported if reported.count(n) > 1})
    assert set(reported) == set(trainable), (sorted(set(trainable) - set(reported)), sorted(set(reported) - set(trainable)))
    for n in reported:
        p, buf = trainable[n], sink.views[id(trainable[n])]
        assert p.grad is not None and p.grad.data_ptr() == buf.data_ptr() and p.grad.shape == p.shape, n
    g1 = {n: p.grad.clone() for n, p in trainable.items()}

    reported = _backward(model, loss_fn, seed=5)                   # no zero_grad: this backward accumulates
    assert len(reported) == len(set(reported)) and set(reported) == set(trainable)
    bad = []
    for n, g in g1.items():
        want = 2 * g
        err = (trainable[n].grad - want).norm().item()
        if not err <= 1e-5 * want.norm().item():
            bad.append((n, err, want.norm().item()))
    assert not bad, bad[:10]
