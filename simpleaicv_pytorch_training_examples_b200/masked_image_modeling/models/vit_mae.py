"""MAE pre-training model (SURVEY.md 8 f4) with the reference's constructor surface and state_dict layout
(SimpleAICV/masked_image_modeling/models/vit_mae.py:25-98 encoder, :227-283 decoder, :370-430 VITMAEPretrainModel,
:473-530 constructors), executed by engine.mae.MAERT on the ViT kernels of this package plus the token gather / scatter
of csrc/capi_tokens.cu.

The nn.Modules are parameter containers built and initialised in the reference's order (same random draws under a seed:
Conv2d / Linear defaults in construction order, sin-cos position encodings, xavier re-draws, normal(.02) tokens);
``forward(images)`` returns ``(pred [B, L, p*p*3], mask [B, L])`` like the reference.  CPU tensors raise.
"""
import numpy as np
import torch
import torch.nn as nn

from ...classification.backbones.vit import PatchEmbeddingBlock, TransformerEncoderLayer

__all__ = ['vit_base_patch16_224_mae_pretrain_model', 'vit_large_patch16_224_mae_pretrain_model',
           'vit_huge_patch14_224_mae_pretrain_model']


def sincos_2d(planes, patch_nums, cls_token=True):
    """vit_mae.py:100-158: fixed 2-D sin-cos position encoding ([1 +] patch_nums^2 rows, w coordinate first)."""
    def one_d(p, grid):
        omega = np.arange(p // 2, dtype=np.float32)
        omega /= p / 2.
        omega = 1. / 10000 ** omega
        out = np.einsum('m,d->md', grid.reshape(-1), omega)
        return np.concatenate([np.sin(out), np.cos(out)], axis=1)
    grid_h = np.arange(patch_nums, dtype=np.float32)
    grid_w = np.arange(patch_nums, dtype=np.float32)
    grid = np.stack(np.meshgrid(grid_w, grid_h), axis=0).reshape([2, 1, patch_nums, patch_nums])
    enc = np.concatenate([one_d(planes // 2, grid[0]), one_d(planes // 2, grid[1])], axis=1)
    if cls_token:
        enc = np.concatenate([np.zeros([1, planes]), enc], axis=0)
    return enc


def _xavier_linears(module):
    for m in module.modules():
        if isinstance(m, nn.Linear):
            nn.init.xavier_uniform_(m.weight)
            if m.bias is not None:
                nn.init.constant_(m.bias, 0)
        elif isinstance(m, nn.LayerNorm):
            nn.init.constant_(m.bias, 0)
            nn.init.constant_(m.weight, 1.0)


class VITMAEPretrainModelEncoder(nn.Module):

    def __init__(self, patch_size, image_size, embedding_planes, block_nums, head_nums, feedforward_ratio, mask_ratio=0.75,
                 dropout_prob=0., use_gradient_checkpoint=False):
        super().__init__()
        self.image_size, self.patch_size, self.embedding_planes = image_size, patch_size, embedding_planes
        self.block_nums, self.head_nums, self.feedforward_ratio = block_nums, head_nums, feedforward_ratio
        self.mask_ratio = mask_ratio
        self.use_gradient_checkpoint = use_gradient_checkpoint
        self.dropout_prob = dropout_prob
        self.patch_embed = PatchEmbeddingBlock(3, embedding_planes, kernel_size=patch_size, stride=patch_size, padding=0)
        self.cls_token = nn.Parameter(torch.zeros(1, 1, embedding_planes))
        self.pos_embed = nn.Parameter(torch.zeros(1, (image_size // patch_size) ** 2 + 1, embedding_planes), requires_grad=False)
        self.blocks = nn.ModuleList([TransformerEncoderLayer(embedding_planes, head_nums, feedforward_ratio=feedforward_ratio,
                                                             dropout_prob=dropout_prob, drop_path_prob=0.) for _ in range(block_nums)])
        self.norm = nn.LayerNorm(embedding_planes, eps=1e-6)
        self.pos_embed.data.copy_(torch.from_numpy(sincos_2d(embedding_planes, image_size // patch_size)).float().unsqueeze(0))
        w = self.patch_embed.proj.weight.data
        nn.init.xavier_uniform_(w.view([w.shape[0], -1]))      # patch_embed initialised like a Linear (vit_mae.py:83-87)
        nn.init.normal_(self.cls_token, std=.02)
        _xavier_linears(self)


class VITMAEPretrainModelDecoder(nn.Module):

    def __init__(self, patch_size, image_size, embedding_planes, block_nums, head_nums, feedforward_ratio, dropout_prob=0.1,
                 use_gradient_checkpoint=False):
        super().__init__()
        self.image_size, self.patch_size, self.embedding_planes = image_size, patch_size, embedding_planes
        self.block_nums, self.head_nums, self.feedforward_ratio = block_nums, head_nums, feedforward_ratio
        self.use_gradient_checkpoint = use_gradient_checkpoint
        self.dropout_prob = dropout_prob
        self.mask_token = nn.Parameter(torch.zeros(1, 1, embedding_planes))
        self.pos_embed = nn.Parameter(torch.zeros(1, (image_size // patch_size) ** 2 + 1, embedding_planes), requires_grad=False)
        self.blocks = nn.ModuleList([TransformerEncoderLayer(embedding_planes, head_nums, feedforward_ratio=feedforward_ratio,
                                                             dropout_prob=dropout_prob, drop_path_prob=0.) for _ in range(block_nums)])
        self.norm = nn.LayerNorm(embedding_planes, eps=1e-6)
        self.fc = nn.Linear(embedding_planes, patch_size * patch_size * 3)
        self.pos_embed.data.copy_(torch.from_numpy(sincos_2d(embedding_planes, image_size // patch_size)).float().unsqueeze(0))
        nn.init.normal_(self.mask_token, std=.02)
        _xavier_linears(self)


class VITMAEPretrainModel(nn.Module):

    def __init__(self, patch_size=16, image_size=224, mask_ratio=0.75, encoder_embedding_planes=768, encoder_block_nums=12,
                 encoder_head_nums=12, encoder_feedforward_ratio=4, encoder_dropout_prob=0., decoder_embedding_planes=384,
                 decoder_block_nums=4, decoder_head_nums=6, decoder_feedforward_ratio=4, decoder_dropout_prob=0.,
                 use_gradient_checkpoint=False):
        super().__init__()
        assert image_size % patch_size == 0
        self.patch_size, self.image_size = patch_size, image_size
        self.encoder = VITMAEPretrainModelEncoder(patch_size, image_size, encoder_embedding_planes, encoder_block_nums,
                                                  encoder_head_nums, encoder_feedforward_ratio, mask_ratio=mask_ratio,
                                                  dropout_prob=encoder_dropout_prob, use_gradient_checkpoint=use_gradient_checkpoint)
        self.decoder = VITMAEPretrainModelDecoder(patch_size, image_size, decoder_embedding_planes, decoder_block_nums,
                                                  decoder_head_nums, decoder_feedforward_ratio, dropout_prob=decoder_dropout_prob,
                                                  use_gradient_checkpoint=use_gradient_checkpoint)
        self.encoder_to_decoder = nn.Linear(encoder_embedding_planes, decoder_embedding_planes)
        _xavier_linears(self.encoder_to_decoder)
        if encoder_dropout_prob > 0. or decoder_dropout_prob > 0.:
            raise NotImplementedError('MAE on the H100 runtime: dropout_prob > 0 is not wired (the shipped MAE configs use 0)')

    def _runtime(self):
        rt = self.__dict__.get('_rt')
        if rt is None:
            from ...engine.mae import MAERT
            rt = MAERT(self)
            self.__dict__['_rt'] = rt
        return rt

    def grad_sink(self):
        return self._runtime().sink

    def forward(self, x, noise=None):
        """x: fp32 [B, 3, H, W] on the GPU.  noise: optional [B, L] uniform draws that decide the masking (the reference
        draws them with torch.rand inside random_masking, vit_mae.py:203-225; tests pass them in to pin the masks)."""
        if not x.is_cuda:
            raise RuntimeError('this model runs on H100 kernels only; move the batch to the GPU (no CPU fallback exists)')
        from ...engine.mae import run_mae
        return run_mae(self._runtime(), x.float(), self.training, noise)

    def images_to_patch(self, images):
        """(N, 3, H, W) -> (N, L, patch_size**2 * 3), vit_mae.py:437-449."""
        pn, p = self.image_size // self.patch_size, self.patch_size
        x = images.reshape(images.shape[0], 3, pn, p, pn, p)
        x = torch.einsum('nchpwq->nhwpqc', x)
        return x.reshape(x.shape[0], pn * pn, p * p * 3)

    def patch_to_images(self, x):
        """(N, L, patch_size**2 * 3) -> (N, 3, H, W), vit_mae.py:451-464."""
        h = int(x.shape[1] ** 0.5)
        p = self.patch_size
        images = x.reshape(x.shape[0], h, h, p, p, 3)
        images = torch.einsum('nhwpqc->nchpwq', images)
        return images.reshape(images.shape[0], 3, h * p, h * p)


def vit_base_patch16_224_mae_pretrain_model(**kwargs):
    return VITMAEPretrainModel(patch_size=16, image_size=224, encoder_embedding_planes=768, encoder_block_nums=12,
                               encoder_head_nums=12, encoder_feedforward_ratio=4, decoder_embedding_planes=512,
                               decoder_block_nums=8, decoder_head_nums=16, decoder_feedforward_ratio=4, **kwargs)


def vit_large_patch16_224_mae_pretrain_model(**kwargs):
    return VITMAEPretrainModel(patch_size=16, image_size=224, encoder_embedding_planes=1024, encoder_block_nums=24,
                               encoder_head_nums=16, encoder_feedforward_ratio=4, decoder_embedding_planes=512,
                               decoder_block_nums=8, decoder_head_nums=16, decoder_feedforward_ratio=4, **kwargs)


def vit_huge_patch14_224_mae_pretrain_model(**kwargs):
    return VITMAEPretrainModel(patch_size=14, image_size=224, encoder_embedding_planes=1280, encoder_block_nums=32,
                               encoder_head_nums=16, encoder_feedforward_ratio=4, decoder_embedding_planes=512,
                               decoder_block_nums=8, decoder_head_nums=16, decoder_feedforward_ratio=4, **kwargs)
