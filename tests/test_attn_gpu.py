"""GPU parity of the wgmma attention family (csrc/attn_sm90.cuh) through the general C-ABI entry
(saicv_attn_fwd / saicv_attn_bwd) against plain fp32 torch attention on the same bf16-representable inputs:
every supported (score width, value width), long sequences (several key blocks / row tiles), cross attention
(Lq != Lk), key-padding masks and strided (packed / head-major) layouts.  Tolerances: outputs 2e-2 abs,
gradients relative L2 2e-2 (bf16 P / dS operands, fp32 accumulation)."""
import math

import pytest
import torch

pytestmark = pytest.mark.gpu


def _ops():
    from simpleaicv_pytorch_training_examples_b200 import ops
    return ops


def _rel(a, b):
    return ((a.float() - b.float()).norm() / b.float().norm().clamp_min(1e-12)).item()


def _ref(q, k, v, scale, mask):
    s = (q @ k.transpose(-2, -1)) * scale
    if mask is not None:
        s = s.masked_fill(mask[:, None, None, :], float('-inf'))
    return s.softmax(-1) @ v, torch.logsumexp(s, -1) / math.log(2.0)


CASES = [
    # B, H, Lq, Lk, dqk, dv, masked
    (2, 3, 197, 197, 64, 64, False),       # ViT-B
    (1, 2, 1000, 1000, 64, 64, False),     # 8 row tiles x 8 key blocks
    (2, 2, 100, 777, 32, 32, True),        # DETR decoder cross attention with key padding
    (1, 8, 600, 600, 32, 32, True),        # DETR encoder self attention with key padding
    (2, 2, 196, 196, 80, 80, False),       # SAM-H window
    (1, 2, 196, 196, 96, 64, False),       # SAM-B window + 28(32) bias columns
    (1, 2, 196, 196, 112, 80, False),      # SAM-H window + bias columns
    (1, 1, 300, 300, 192, 64, False),      # SAM-B global (64 + 128 bias columns)
    (1, 1, 300, 300, 208, 80, False),      # SAM-H global
    (3, 1, 17, 5, 64, 64, False),          # tiny / ragged
]


@pytest.mark.parametrize('B,H,Lq,Lk,dqk,dv,masked', CASES)
def test_attn_fwd_bwd_matches_torch(B, H, Lq, Lk, dqk, dv, masked):
    ops = _ops()
    g = torch.Generator(device='cuda').manual_seed(11)
    q = torch.randn(B, H, Lq, dqk, device='cuda', generator=g).to(torch.bfloat16)
    k = torch.randn(B, H, Lk, dqk, device='cuda', generator=g).to(torch.bfloat16)
    v = torch.randn(B, H, Lk, dv, device='cuda', generator=g).to(torch.bfloat16)
    scale = min(dqk, 80) ** -0.5
    mask = bits = None
    if masked:
        valid = torch.randint(Lk // 2, Lk, (B,), generator=torch.Generator().manual_seed(1))
        mask = (torch.arange(Lk)[None, :] >= valid[:, None]).cuda()
        mask[:, 3] = True   # a hole in the middle as well
        bits = ops.pack_key_mask(mask, Lk)
    out, lse = ops.attn_fwd(q, k, v, scale, mask_bits=bits)
    qf, kf, vf = (t.float().requires_grad_(True) for t in (q, k, v))
    ref, ref_lse = _ref(qf, kf, vf, scale, mask)
    err = (out.float() - ref).abs().max().item()
    assert err <= 2e-2, f'out max err {err}'
    assert (lse - ref_lse).abs().max().item() <= 1e-2
    dout = torch.randn(B, Lq, H, dv, device='cuda', generator=g).to(torch.bfloat16).permute(0, 2, 1, 3)   # layout of out
    ref.backward(dout.float())
    dq, dk, dvv = torch.empty_like(q), torch.empty_like(k), torch.empty_like(v)
    ops.attn_bwd(q, k, v, out, lse, dout, scale, dq, dk, dvv, mask_bits=bits)
    torch.cuda.synchronize()
    for name, got, want in (('dq', dq, qf.grad), ('dk', dk, kf.grad), ('dv', dvv, vf.grad)):
        r = _rel(got, want)
        assert r <= 2e-2, f'{name} rel L2 {r}'
    if masked:   # masked keys receive exactly zero gradient
        assert dk[mask[:, None, :, None].expand_as(dk)].abs().max().item() == 0
        assert dvv[mask[:, None, :, None].expand_as(dvv)].abs().max().item() == 0


def test_attn_partial_dk_columns_and_strided_views():
    """dk_cols < dqk (bias columns of k carry no gradient) and packed [B, L, 3, H, D] views."""
    ops = _ops()
    B, H, L, D = 2, 3, 150, 64
    g = torch.Generator(device='cuda').manual_seed(5)
    qkv = torch.randn(B, L, 3, H, D, device='cuda', generator=g).to(torch.bfloat16)
    q, k, v = (qkv[:, :, i].permute(0, 2, 1, 3) for i in range(3))
    out, lse = ops.attn_fwd(q, k, v, D ** -0.5)
    out2, lse2 = ops.attention_fwd(qkv, B, L, H, D, D ** -0.5)
    assert torch.equal(out.permute(0, 2, 1, 3).reshape(B * L, H * D), out2) and torch.equal(lse, lse2)
    dout = torch.randn(B, L, H, D, device='cuda', generator=g).to(torch.bfloat16).permute(0, 2, 1, 3)
    dqkv = torch.zeros_like(qkv)
    dq, dk, dv = (dqkv[:, :, i].permute(0, 2, 1, 3) for i in range(3))
    ops.attn_bwd(q, k, v, out, lse, dout, D ** -0.5, dq, dk, dv, dk_cols=32)
    full = ops.attention_bwd(qkv, out2, dout.permute(0, 2, 1, 3).reshape(B * L, H * D).contiguous(), lse2, B, L, H, D, D ** -0.5)
    assert torch.equal(dqkv[:, :, 0], full[:, :, 0]) and torch.equal(dqkv[:, :, 2], full[:, :, 2])
    assert torch.equal(dqkv[:, :, 1, :, :32], full[:, :, 1, :, :32]) and dqkv[:, :, 1, :, 32:].abs().max().item() == 0


def test_attn_is_bit_reproducible():
    ops = _ops()
    g = torch.Generator(device='cuda').manual_seed(3)
    qkv = torch.randn(4, 197, 3, 12, 64, device='cuda', generator=g).to(torch.bfloat16)
    dout = torch.randn(4 * 197, 12 * 64, device='cuda', generator=g).to(torch.bfloat16)
    runs = []
    for _ in range(2):
        out, lse = ops.attention_fwd(qkv, 4, 197, 12, 64, 0.125)
        runs.append((out.clone(), lse.clone(), ops.attention_bwd(qkv, out, dout, lse, 4, 197, 12, 64, 0.125).clone()))
    assert all(torch.equal(a, b) for a, b in zip(*runs))
