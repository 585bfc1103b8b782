"""Writes tests/golden/dinov3_*.ptf: what the reference (installed into oracle/_ref by build()) computes on the CPU in fp32
for the DINOv3 image encoder / backbone.  Each fixture records the seeded input and distillation target, the RoPE rescale
factor the reference drew from torch's CPU generator in its training forward, the output, the MSE loss, a digest of every
parameter gradient (norm and fixed samples), and the eval-mode output (no draw).  The suffix is .ptf so that the SAM /
ViT golden loader, which globs *.pt, does not pick these up.

    python tests/golden/make_dinov3_golden.py
"""
import os
import sys

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

# name -> (kind, constructor arguments, image size, batch)
CASES = {
    'dinov3_small_enc64': ('encoder', {'backbone_type': 'dinov3_vit_small_patch16_backbone', 'image_size': 64}, 64, 2),
    'dinov3_smallplus_enc64': ('encoder', {'backbone_type': 'dinov3_vit_small_plus_patch16_backbone', 'image_size': 64}, 64, 2),
    'dinov3_b768_d2_bb48': ('backbone', {'embedding_planes': 768, 'block_nums': 2, 'head_nums': 12, 'pos_embed_rope_rescale_coords': 2},
                            48, 2),
}
SEED, DATA_SEED, DRAW_SEED = 3, 4, 11


def sample_index(numel):
    """Fixed positions of a gradient recorded in the fixture."""
    return torch.unique(torch.linspace(0, numel - 1, min(numel, 16)).round().long())


def build_reference(kind, kwargs):
    from baseline import ref_import
    torch.manual_seed(SEED)
    if kind == 'encoder':
        return ref_import.module('SimpleAICV.interactive_segmentation.models.dinov3_segment_anything.dinov3_image_encoder') \
            .DINOV3ViTImageEncoder(**kwargs)
    return ref_import.module('SimpleAICV.detection.models.backbones.dinov3vit').DinoVisionTransformer(**kwargs)


def make(name):
    kind, kwargs, size, batch = CASES[name]
    torch.set_num_threads(1)
    ref = build_reference(kind, kwargs).train()
    g = torch.Generator().manual_seed(DATA_SEED)
    x = torch.randn(batch, 3, size, size, generator=g)
    with torch.no_grad():
        shape = ref.eval()(x[:1]).shape
    ref.train()
    target = torch.randn(batch, *shape[1:], generator=g)
    torch.manual_seed(DRAW_SEED)
    state = torch.get_rng_state()
    rescale = torch.empty(1).uniform_(-torch.log(torch.tensor(2.)).item(), torch.log(torch.tensor(2.)).item()).exp()
    torch.set_rng_state(state)
    out = ref(x)
    after = torch.get_rng_state()
    loss = torch.nn.functional.mse_loss(out, target)
    loss.backward()
    grads = {n: p.grad.detach() for n, p in ref.named_parameters()}
    with torch.no_grad():
        eval_out = ref.eval()(x)
    sd = ref.state_dict()
    return {'kind': kind, 'kwargs': kwargs, 'seed': SEED, 'draw_seed': DRAW_SEED, 'x': x, 'target': target,
            'rescale': rescale, 'rng_after': after, 'keys': list(sd), 'out': out.detach(), 'loss': loss.detach(),
            'grad_norm': {n: v.norm().item() for n, v in grads.items()},
            'grad_sample': {n: v.flatten()[sample_index(v.numel())].clone() for n, v in grads.items()},
            'eval_out': eval_out}


if __name__ == '__main__':
    for name in CASES:
        torch.save(make(name), os.path.join(HERE, f'{name}.ptf'))
        print('wrote', name)
