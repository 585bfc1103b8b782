"""The bf16 weight operands each runtime lists in operands() (engine/operands.py): the fused optimizers refresh exactly
these copies and prep() re-creates the rest, so the list must name every weight a GEMM reads, once.  Runtimes are built
on the CPU; building one allocates no copy."""
import pytest
import torch


def _families():
    from simpleaicv_pytorch_training_examples_b200.classification import backbones
    from simpleaicv_pytorch_training_examples_b200.detection import models
    from simpleaicv_pytorch_training_examples_b200.interactive_segmentation.models.segment_anything.image_encoder import ViTImageEncoder
    from simpleaicv_pytorch_training_examples_b200.masked_image_modeling.models import vit_mae
    return {
        'resnet18cifar': lambda: backbones.resnet18cifar(num_classes=10),
        'darknet19': lambda: backbones.darknet19(num_classes=10),
        'darknettiny': lambda: backbones.darknettiny(num_classes=10),
        'van_b0': lambda: backbones.van_b0(num_classes=10),
        'vit_base_patch16': lambda: backbones.vit_base_patch16(image_size=64, num_classes=10),
        'resnet18_detr': lambda: models.resnet18_detr(),
        'sam_encoder': lambda: ViTImageEncoder(image_size=320, patch_size=16, embedding_planes=128, block_nums=3, head_nums=2,
                                               out_planes=256, window_size=14, global_attn_indexes=(1,)),
        'mae': lambda: vit_mae.VITMAEPretrainModel(patch_size=16, image_size=64, encoder_embedding_planes=768, encoder_block_nums=2,
                                                   encoder_head_nums=12, decoder_embedding_planes=512, decoder_block_nums=1,
                                                   decoder_head_nums=16),
    }


FAMILIES = ['resnet18cifar', 'darknet19', 'darknettiny', 'van_b0', 'vit_base_patch16', 'resnet18_detr', 'sam_encoder', 'mae']


def _gemm_weights(model):
    """Names of the parameters a GEMM consumes: Linear and (non-depthwise) conv weights, attention in_proj weights.
    Position embeddings, cls / mask tokens, rel-pos tables, query embeddings and layer scales are not among them."""
    out = set()
    for name, mod in model.named_modules():
        pre = f'{name}.' if name else ''
        if isinstance(mod, torch.nn.Linear) or (isinstance(mod, torch.nn.Conv2d) and mod.groups == 1):
            out.add(pre + 'weight')
        elif isinstance(mod, torch.nn.MultiheadAttention):
            out.add(pre + 'in_proj_weight')
    return out


@pytest.mark.parametrize('family', FAMILIES)
def test_runtime_lists_every_gemm_weight_once(family):
    from simpleaicv_pytorch_training_examples_b200.engine.operands import STEM
    torch.manual_seed(0)
    model = _families()[family]()
    rt = model._runtime()
    ops = rt.operands()
    names = {id(p): n for n, p in model.named_parameters()}
    listed = [names.get(id(op.param)) for op in ops]
    assert None not in listed, 'an operand names a parameter the model does not have'
    assert len(set(listed)) == len(listed), sorted(n for n in listed if listed.count(n) > 1)
    want = _gemm_weights(model)
    assert want <= set(names.values())
    assert set(listed) == want, (sorted(want - set(listed)), sorted(set(listed) - want))
    assert all(op.param.dim() >= 2 for op in ops)
    assert [op.layout == STEM for op in ops] == [not op.fusable for op in ops], 'exactly the stem copies stay on prep()'
    assert all(op.w is None for op in ops), 'building the runtime allocated an operand copy'
