"""GPU parity of the ViT kernels (LayerNorm, GELU, token assembly / pooling, fused attention)
against plain torch fp32 on the same bf16-representable inputs."""
import math

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu


def _ops():
    from simpleaicv_pytorch_training_examples_b200 import ops
    return ops


def _rel(a, b):
    return ((a.float() - b.float()).norm() / b.float().norm().clamp_min(1e-12)).item()


@pytest.mark.parametrize('rows,c', [(197 * 3, 768), (1000, 1024), (64, 1280), (77, 256)])
def test_layernorm_fwd_bwd(rows, c):
    ops = _ops()
    g = torch.Generator(device='cuda').manual_seed(0)
    x = torch.randn(rows, c, device='cuda', generator=g) * 2 + 0.3
    gamma = torch.rand(c, device='cuda', generator=g) + 0.5
    beta = torch.randn(c, device='cuda', generator=g)
    y, stats = ops.layernorm_fwd(x, gamma, beta, 1e-6)
    xr = x.clone().requires_grad_(True)
    gr, br = gamma.clone().requires_grad_(True), beta.clone().requires_grad_(True)
    ref = F.layer_norm(xr, (c,), gr, br, 1e-6)
    assert (y.float() - ref).abs().max().item() <= 2e-2 + 1e-2 * ref.abs().max().item()
    dy = torch.randn(rows, c, device='cuda', generator=g).to(torch.bfloat16)
    dres = torch.randn(rows, c, device='cuda', generator=g)
    ref.backward(dy.float())
    dgamma, dbeta = torch.empty(c, device='cuda'), torch.empty(c, device='cuda')
    dxb = torch.empty(rows, c, device='cuda', dtype=torch.bfloat16)
    dx = ops.layernorm_bwd(dy, x, gamma, stats, dgamma, dbeta, dres=dres, dx_bf16=dxb)
    assert _rel(dx, xr.grad + dres) <= 1e-4
    assert _rel(dxb, xr.grad + dres) <= 5e-3
    assert _rel(dgamma, gr.grad) <= 1e-3 and _rel(dbeta, br.grad) <= 1e-3


def test_gelu_and_tokens_and_pool():
    ops = _ops()
    g = torch.Generator(device='cuda').manual_seed(1)
    u = (torch.randn(512, 3072, device='cuda', generator=g) * 2).to(torch.bfloat16)
    h = ops.gelu_fwd(u)
    assert (h.float() - F.gelu(u.float())).abs().max().item() <= 2e-2
    B, NP, C = 5, 196, 768
    patch = torch.randn(B * NP, C, device='cuda', generator=g)
    cls, pos = torch.randn(C, device='cuda', generator=g), torch.randn(NP + 1, C, device='cuda', generator=g)
    x = ops.vit_assemble_tokens(patch, cls, pos, B, NP, C)
    ref = torch.cat([cls.expand(B, 1, C), patch.view(B, NP, C)], 1) + pos
    assert torch.equal(x, ref)
    dx = torch.randn(B, NP + 1, C, device='cuda', generator=g)
    dpos, dcls = torch.empty(NP + 1, C, device='cuda'), torch.empty(C, device='cuda')
    dpatch = torch.empty(B * NP, C, device='cuda', dtype=torch.bfloat16)
    ops.vit_assemble_tokens_bwd(dx, dpos, dcls, dpatch)
    assert _rel(dpos, dx.sum(0)) <= 1e-5 and _rel(dcls, dx[:, 0].sum(0)) <= 1e-5
    assert torch.equal(dpatch, dx[:, 1:].reshape(B * NP, C).to(torch.bfloat16))
    for mean_pool in (True, False):
        p = ops.token_pool_fwd(x, mean_pool)
        refp = x[:, 1:].mean(1) if mean_pool else x[:, 0]
        assert _rel(p, refp) <= 1e-5
        dp = torch.randn(B, C, device='cuda', generator=g)
        dxb = torch.empty(B, NP + 1, C, device='cuda', dtype=torch.bfloat16)
        dxx = ops.token_pool_bwd(dp, NP + 1, mean_pool, dx_bf16=dxb)
        xr = x.clone().requires_grad_(True)
        (xr[:, 1:].mean(1) if mean_pool else xr[:, 0]).backward(dp)
        assert _rel(dxx, xr.grad) <= 1e-5 and _rel(dxb, xr.grad) <= 5e-3


@pytest.mark.parametrize('B,L,H', [(2, 197, 12), (3, 64, 4), (1, 256, 2), (2, 50, 3), (1, 17, 1)])
def test_attn_on_packed_qkv_views(B, L, H):
    ops = _ops()
    D = 64
    g = torch.Generator(device='cuda').manual_seed(2)
    qkv = torch.randn(B, L, 3, H, D, device='cuda', generator=g).to(torch.bfloat16)
    scale = D ** -0.5
    out = torch.empty(B * L, H * D, device='cuda', dtype=torch.bfloat16)
    heads = ops.head_views(qkv.view(B * L, -1), B, L, H, D)   # the ViT runtime's packed-qkv views
    (o,) = ops.head_views(out, B, L, H, D)
    _, lse = ops.attn_fwd(*heads, scale, out=o)
    qr = qkv.float().requires_grad_(True)
    q, k, v = qr.permute(2, 0, 3, 1, 4).unbind(0)  # [B, H, L, D] as in vit.py:66-69
    attn = ((q @ k.transpose(-2, -1)) * scale).softmax(-1)
    ref = (attn @ v).transpose(1, 2).reshape(B * L, H * D)
    assert (out.float() - ref).abs().max().item() <= 2e-2, (out.float() - ref).abs().max().item()
    ref_lse = torch.logsumexp((q @ k.transpose(-2, -1)) * scale, -1) / math.log(2.0)
    assert (lse - ref_lse).abs().max().item() <= 1e-2
    dout = torch.randn(B * L, H * D, device='cuda', generator=g).to(torch.bfloat16)
    ref.backward(dout.float())
    dqkv = torch.empty_like(qkv)
    (do,) = ops.head_views(dout, B, L, H, D)
    ops.attn_bwd(*heads, o, lse, do, scale, *ops.head_views(dqkv.view(B * L, -1), B, L, H, D))
    for i, name in enumerate('qkv'):
        r = _rel(dqkv[:, :, i], qr.grad[:, :, i])
        assert r <= 2e-2, f'd{name} rel L2 {r}'
