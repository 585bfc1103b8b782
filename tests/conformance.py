"""The acceptance rule of the float64 conformance suites (tests/test_*_conformance_gpu.py), and what they share.

Every suite computes the exact value v of each output element in float64 from the same bf16 / fp32 values the kernel
read, and derives from the kernel's operations an absolute allowance B' (u = 2^-24 is one fp32 rounding; rnd() carries
an allowance through one).  Allowances are never fitted to measured errors, and never relative: where the exact value
is tiny a relative bound would be meaningless.  Acceptance, for every element (no fraction of misses is allowed):
  * a bf16 output lies in [rne_bf16(v - B'), rne_bf16(v + B')]: it is a correctly rounded bf16 of some value within the
    allowance of the exact result.  Truncation, a second rounding (e.g. an accumulator rounded before a bias add) or a
    dropped term all fail it;
  * an fp32 output lies within B' of v;
  * a non-finite output fails.
check() applies it, prints the largest fraction of B' an element used (for a bf16 output: the distance from v to the
rounding interval of the stored value), and records that share under the check's family.  A suite that imports the
module-scope `report` fixture prints the largest share per family it recorded at its end (run with -s); exact()
records a bit-exact family as 0.

Invariants are compared as raw bits (same()): floats by their bit patterns, so signed zeros and NaN payloads count.
"""
import math

import numpy as np
import pytest
import torch

from simpleaicv_pytorch_training_examples_b200 import _lib, ops

U = 2.0 ** -24          # one fp32 rounding, relative
NAN = float('nan')
M32 = 0xFFFFFFFF
PARTIAL_ROWS = 264      # SAICV_BN_PARTIAL_ROWS
USED = {}               # family -> largest share of its allowance used, for the running suite's report


# ------------------------------------------------------------------ the rounding model
def quantum_bf16(x):
    """The bf16 spacing at float64 values x (8 significant bits; subnormal spacing 2^-133), exactly."""
    _, e = torch.frexp(x)
    e = torch.where(x == 0, -200, e.to(torch.int64) - 8)
    return ((e.clamp_min(-133) + 1023) << 52).view(torch.float64)


def rne_bf16(x):
    """float64 -> nearest bf16 value (ties to even), as float64, in one rounding (x.to(bfloat16) rounds through fp32)."""
    q = quantum_bf16(x)
    return torch.round(x / q) * q


def rnd(v, a):
    """Allowance after one fp32 rounding of a value within a of v."""
    return a + U * (v.abs() + a)


# ------------------------------------------------------------------ the acceptance rule and the invariants
def check(family, what, out, v, allow, s=None):
    """out: kernel output; v: exact float64 value of the same shape; allow: its allowance B' (broadcastable to v).
    s: the absolute product sum of a reduction, to print max |out - v| / S as well.  family: the report row the share of
    B' is recorded under (None: not recorded)."""
    assert out.shape == v.shape, f'{what}: shape {tuple(out.shape)} vs {tuple(v.shape)}'
    allow = torch.as_tensor(allow, dtype=torch.float64, device=v.device).expand(v.shape)
    o = out.double()
    if out.dtype == torch.bfloat16:
        lo, hi = rne_bf16(v - allow), rne_bf16(v + allow)
        bad = (o < lo) | (o > hi)
        dist = ((o - v).abs() - quantum_bf16(o) / 2).clamp_min(0)   # nearest value that rounds to o (to a factor 2 below a power of 2)
    else:
        bad = (o - v).abs() > allow
        dist = (o - v).abs()
    bad |= ~torch.isfinite(o)
    used = (dist / allow.clamp_min(1e-300)).max().item() if o.numel() else 0.0
    if family is not None and math.isfinite(used):
        USED[family] = max(USED.get(family, 0.0), used)
    ratio = '' if s is None else f'max |out - ref| / S = {(dist / s.clamp_min(1e-30)).max().item():.3g}, '
    print(f'{what}: {ratio}allowance used {used:.3g}')
    n_bad = int(bad.sum())
    if n_bad:
        i = int(bad.flatten().nonzero()[0])
        raise AssertionError(
            f'{what}: {n_bad}/{out.numel()} elements outside the allowance; first at flat index {i}: '
            f'out {o.flatten()[i].item():.9g}, exact {v.flatten()[i].item():.9g}, allowance {allow.flatten()[i].item():.3g}')


def same(what, a, b):
    """Raw-bit equality (floats as their bit patterns, so signed zeros and NaN payloads count too)."""
    assert a.shape == b.shape and a.dtype == b.dtype, f'{what}: {tuple(a.shape)} {a.dtype} vs {tuple(b.shape)} {b.dtype}'
    bits = {torch.bfloat16: torch.int16, torch.float32: torch.int32}.get(a.dtype)
    n_bad = int((a != b).sum()) if bits is None else int((a.view(bits) != b.view(bits)).sum())
    assert n_bad == 0, f'{what}: {n_bad}/{a.numel()} elements differ (max |diff| {(a.float() - b.float()).abs().max().item():.3g})'


def exact(family, what, out, want):
    """A bit-exact family: same(), reported with a share of 0."""
    same(what, out, want)
    USED.setdefault(family, 0.0)
    print(f'{what}: bit-exact')


@pytest.fixture(scope='module', autouse=True)
def report():
    USED.clear()
    yield
    if USED:
        print('\nlargest share of the allowance used, by family (0: bit-exact):')
        for k in sorted(USED):
            print(f'  {k:28s} {USED[k]:.3g}')


# ------------------------------------------------------------------ inputs and launches
def gen(seed):
    return torch.Generator(device='cuda').manual_seed(seed)


def randn(*shape, scale=1.0, seed=0):
    return torch.randn(*shape, device='cuda', generator=gen(seed)) * scale


def rand(*shape, seed=0):
    return torch.rand(*shape, device='cuda', generator=gen(seed))


def nan(*shape, dtype=torch.float32):
    return torch.full(shape, NAN, device='cuda', dtype=dtype)


def f32(x):
    """x rounded to fp32, as a Python float."""
    return float(np.float32(x))


def every_bf16(width):
    """Every finite bf16 value, zero-padded to rows of `width`."""
    u = torch.arange(-2 ** 15, 2 ** 15, device='cuda', dtype=torch.int32).to(torch.int16).view(torch.bfloat16)
    u = u[torch.isfinite(u.float())]
    return torch.cat([u, u.new_zeros((-u.numel()) % width)]).view(-1, width).contiguous()


def call(name, *args):
    """Call C entry `name` on the current stream; tensors are passed as pointers, None as a null pointer."""
    _lib.call(name, *[ops._p(a) if isinstance(a, torch.Tensor) else a for a in args], ops._stream())


# ------------------------------------------------------------------ mirrors of the library that several suites use
def acc_allowance(ref, s):
    """The fp32 accumulation allowance of the wgmma GEMM engine (test_gemm_conformance_gpu.py)."""
    return 2.0 ** -16 * s + 2.0 ** -22 * ref.abs()


def next_pow2(v):
    p = 1
    while p < v:
        p <<= 1
    return p


def van_slab(rows, c):
    """capi_van.cu slab: (ty_count, rows_per_block, blocks)."""
    tx = min(next_pow2(c // 8), 256)
    ty = 256 // tx
    b = max(1, min(-(-rows // (ty * 8)), PARTIAL_ROWS))
    rpb = -(-(-(-rows // b)) // ty) * ty
    return ty, rpb, -(-rows // rpb)


def dropout_hash(seed, a, b):
    """csrc/dropout_hash.cuh on int64 tensors a, b (32-bit values): int64 products wrap, the low 32 bits are exact."""
    lo, hi = seed & M32, (seed >> 32) & M32
    x = ((a + lo) & M32) * 0x9E3779B1 & M32
    x = x ^ (((b + hi) & M32) * 0x85EBCA77 & M32)
    x = x ^ (x >> 16)
    x = x * 0x7FEB352D & M32
    x = x ^ (x >> 15)
    x = x * 0x846CA68B & M32
    return x ^ (x >> 16)


def dropout_threshold(p):
    """dropout_threshold((float)p): the entries take p as a C float."""
    t = float(np.float32(p)) * 4294967296.0
    return M32 if t >= 4294967295.0 else int(t)


def dropout_keep(seed, a, b, p):
    return dropout_hash(seed, a, b) >= dropout_threshold(p)


def drop_scale(p):
    """AttnDrop.scale = 1.f / (1.f - p) in fp32."""
    return float(np.float32(1.0) / (np.float32(1.0) - np.float32(p)))
