"""``sam_b / sam_l / sam_h`` with the reference's signatures (segment_anything/sam.py:180-210).

The image encoder (BASELINE.json config #4, SURVEY.md 8 a5) runs on the H100 runtime and keeps the reference's
``image_encoder.*`` state_dict keys.  The prompt encoder and the mask decoder are SURVEY.md 8(f1) ("next") rows:
they are not built yet, so ``forward`` / ``forward_prompt_encoder_mask_decoder`` raise NotImplementedError instead
of silently falling back to anything; ``forward_image_encoder`` is the hot path of the encoder-distillation and
SAM training loops (tools/interactive_segmentation_scripts.py:372-377)."""
import torch.nn as nn

from .image_encoder import ViTImageEncoder

__all__ = ['sam_b', 'sam_l', 'sam_h']


class SAM(nn.Module):

    def __init__(self, image_size=1024, patch_size=16, inplanes=3, image_encoder_embedding_planes=768, image_encoder_block_nums=12,
                 image_encoder_head_nums=12, image_encoder_mlp_ratio=4, image_encoder_window_size=14,
                 image_encoder_global_attn_indexes=[2, 5, 8, 11], prompt_encoder_embedding_planes=256,
                 use_gradient_checkpoint=False, frozen_image_encoder=False, **unused_decoder_kwargs):
        super().__init__()
        self.image_encoder = ViTImageEncoder(image_size=image_size, patch_size=patch_size, inplanes=inplanes,
                                             embedding_planes=image_encoder_embedding_planes, block_nums=image_encoder_block_nums,
                                             head_nums=image_encoder_head_nums, mlp_ratio=image_encoder_mlp_ratio,
                                             out_planes=prompt_encoder_embedding_planes, window_size=image_encoder_window_size,
                                             global_attn_indexes=image_encoder_global_attn_indexes,
                                             use_gradient_checkpoint=use_gradient_checkpoint)
        if frozen_image_encoder:
            for p in self.image_encoder.parameters():
                p.requires_grad = False

    def grad_sink(self):
        return self.image_encoder.grad_sink()

    def forward_image_encoder(self, batch_images):
        return self.image_encoder(batch_images)

    def forward_prompt_encoder_mask_decoder(self, *args, **kwargs):
        raise NotImplementedError('SAM prompt encoder / mask decoder are not built yet (SURVEY.md 8 f1); only the image encoder '
                                  'runs on the H100 runtime')

    def forward(self, *args, **kwargs):
        raise NotImplementedError('SAM.forward needs the prompt encoder / mask decoder (SURVEY.md 8 f1); use forward_image_encoder')


def _sam(**kwargs):
    return SAM(**kwargs)


def _variant(defaults, image_size, patch_size, kwargs):
    cfg = dict(image_size=image_size, patch_size=patch_size, prompt_encoder_embedding_planes=256, **defaults)
    cfg.update(kwargs)
    return _sam(**cfg)


def sam_b(image_size=1024, patch_size=16, **kwargs):
    return _variant(dict(image_encoder_embedding_planes=768, image_encoder_block_nums=12, image_encoder_head_nums=12,
                         image_encoder_global_attn_indexes=[2, 5, 8, 11]), image_size, patch_size, kwargs)


def sam_l(image_size=1024, patch_size=16, **kwargs):
    return _variant(dict(image_encoder_embedding_planes=1024, image_encoder_block_nums=24, image_encoder_head_nums=16,
                         image_encoder_global_attn_indexes=[5, 11, 17, 23]), image_size, patch_size, kwargs)


def sam_h(image_size=1024, patch_size=16, **kwargs):
    return _variant(dict(image_encoder_embedding_planes=1280, image_encoder_block_nums=32, image_encoder_head_nums=16,
                         image_encoder_global_attn_indexes=[7, 15, 23, 31]), image_size, patch_size, kwargs)
