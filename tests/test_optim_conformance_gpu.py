"""Conformance of the fused optimizer kernels (csrc/capi_optim.cu) and the Newton-Schulz GEMMs (saicv_ns_gemm, the
VAR_NS variant of the GEMM engine) against a float64 reference.

Reference.  Every step is checked against the exact float64 operation applied to that step's stored inputs: p, g and
the state tensors are snapshot before the step, the hyper-parameters are the fp32 values the kernel reads (lr, weight
decay, momentum, betas, eps; the Muon scale `adj` read back from the device table), the gradient scale is the stored
clip coefficient, and the Newton-Schulz result U that the Muon apply reads is read back from its slot.  An allowance
therefore belongs to one launch, and error cannot drift across steps; runs still take several steps, so that the
ring of hyper-parameter tables wraps and the step counters advance.  A value the kernel stores and then uses in the
same thread (the new momentum buffer, moments) is checked, then taken as an exact input of what follows it.

Allowances are derived from the operation, never fitted to measured errors (u = 2^-24, one fp32 rounding):
  * Every fp32 operation is one rounding of u times the sum of the magnitudes of the terms it combines, and each
    operation carries the allowances of its operands (x +- y: a_x + a_y; x y: |x| a_y + |y| a_x + a_x a_y;
    x / y: (a_x + |x / y| a_y) / (|y| - a_y); sqrt(x): sqrt(x) - sqrt(x - a_x)), so a result within a of v is within
    a + u (|terms| + a) after it.  FMA contraction only removes roundings, so the bound holds with or without it;
    sqrtf and / are IEEE (the library is built without fast math).
  * AdamW's bias corrections: 1 - beta1^t and sqrt(1 - beta2^t) in float64 from the fp32 betas (as the kernel
    computes them in double), t the parameter's own step count (torch.optim.AdamW's, run in lockstep); the step size
    lr / (1 - beta1^t) and sqrt(1 - beta2^t) are then rounded once to fp32.  The Muon AdamW rows: t = adam_steps + 1
    read before the step, step size lr sqrt(1 - beta2^t) / (1 - beta1^t) rounded once.
  * Sums of squares: the global norm of the clip adds g^2 (one rounding), a per-thread chain of <= 32 terms, 5 shuffle
    levels and the 8 warp partials in order: d = 1 + 32 + 5 + 8 = 46 roundings of u sum g^2; the fold of the chunk
    partials in double adds (ceil(chunks / 256) + 8) 2^-53 sum g^2; the square root halves the relative allowance
    (as the interval above), and the cast to fp32 is one more rounding.  The coefficient is bit-exact against
    min(1, max_norm / (norm + 1e-6)) in fp32 from the stored norm, NaN when the norm is NaN (as torch.clamp keeps it).
  * Muon prep: u = nesterov ? g' + mu b' : b' (from the stored b'), then bf16(u): |bf16(u) - u| <= a_u + half a bf16
    spacing at |u| + a_u (without Nesterov u = b' is stored, so bf16(u) is exact).  ||bf16(u)||^2 gets the uncertainty
    of bf16(u)^2, 2 |u| a + a^2 per element, plus the same 46-rounding fold and the double fold of the tensor's chunk
    partials; X = bf16(bf16(u) * (1 / (norm + 1e-7))).
  * Newton-Schulz GEMMs: the GEMM-conformance bound B = 2^-16 S + 2^-22 |ref| (S = sum |a b| over the reduction),
    carried through fmaf(beta, aux, alpha acc) as |alpha| B + 2u (|alpha| (|ref| + B) + |beta aux|).
  * The bf16 operand copies must equal rne_bf16 of the stored fp32 p' bit for bit, and every element of a copy the
    layout does not map (extra rows, channel and tap padding) keeps its sentinel.
Largest shares of the allowance, measured on an NVIDIA H100 80GB HBM3 at a 700 W power limit: SGD 99.7 % and the Muon
prep 99.6 % (a correctly rounded final operation may use all of its rounding), the Muon apply 90 %, AdamW 83 %, the
Newton-Schulz GEMMs 36 %, the clip norm 3.4 %; the operand copies are bit-exact.  The file runs in about 25 s.

Cases.  The SGD / AdamW tensors cover the chunk edges (numel 1, 3, 4, 7, 8191, 8192, 8193, 3 * 8192 + 5 and 2304 * 768),
gradient views at float offsets 1, 2 and 3 (the scalar path), a tensor whose last chunk has n % 4 != 0 after float4
chunks, and more than 256 chunks in all, so clip_coef_kernel folds several partials per thread;
test_cases_reach_every_chunk_path_cpu checks that from a mirror of the chunk table and the float4 condition.  Three
groups (momentum 0.9 / 0 / 0.9 Nesterov, different weight decays) run 10 steps with the learning rate rewritten every
step.  AdamW also runs with some gradients None on some steps.  Muon covers the transposed slot, three matrices in one
shape class, padded slots, a 1024 x 4096 matrix of 512 chunks, Nesterov on and off and clip.
"""
import copy
import ctypes
import math

import numpy as np
import pytest
import torch

from conformance import U, acc_allowance, call, check, exact, f32, gen, quantum_bf16, rne_bf16, same
from conformance import report  # noqa: F401  (autouse: this module's allowance report)

gpu = pytest.mark.gpu

CHUNK = 8192            # SAICV_OPT_CHUNK
THREADS = 256           # kOptThreads
SUMSQ_DEPTH = 1 + CHUNK // THREADS + 5 + THREADS // 32   # g^2, the per-thread chain, the shuffles, the warp partials
SENTINEL = 0x5A5A       # bf16 bit pattern of the unmapped elements of an operand copy
BIG = 2304 * 768

# (numel, float offset of the gradient view mod 4, group): chunk edges, both memory paths, > 256 chunks in all
GEOM = [(1, 0, 0), (3, 0, 1), (4, 0, 2), (7, 0, 0), (8191, 0, 1), (8192, 0, 2), (8193, 0, 0), (3 * CHUNK + 5, 0, 1),
        (BIG, 0, 2), (CHUNK, 1, 0), (CHUNK + 1, 2, 1), (3 * CHUNK + 5, 3, 2), (BIG, 1, 0)]
# group rows: (lr at step 0, weight decay, momentum, nesterov) for SGD; AdamW takes lr and weight decay
SGD_GROUPS = [(0.1, 1e-2, 0.9, False), (0.05, 0.0, 0.0, False), (0.2, 5e-2, 0.9, True)]
ADAMW_GROUPS = [(1e-2, 1e-2), (5e-3, 0.0), (2e-2, 5e-2)]
BETAS, EPS = (0.9, 0.99), 1e-8
STEPS = 10              # > SAICV_OPT_RING

# Muon: matrices (three in one shape class, one of them transposed; padded slots; 512 chunks) and AdamW rows
MUON_MATS = [(96, 200), (96, 200), (200, 96), (8, 5, 3, 3), (130, 70), (1024, 4096)]
MUON_ADAMW = [(77,), (CHUNK + 1,), (3, 5)]


# ------------------------------------------------------------------ interval arithmetic of the fp32 kernels
class _V:
    """A float64 value v with a bound a on the distance of the kernel's fp32 result from it; every operation adds one fp32
    rounding of u times the magnitudes of the terms it combines."""

    def __init__(self, v, a=None):
        self.v = v.double() if isinstance(v, torch.Tensor) else torch.tensor(float(v), dtype=torch.float64, device='cuda')
        self.a = torch.zeros_like(self.v) if a is None else a

    @staticmethod
    def _rnd(v, a, mag):
        return _V(v, a + U * (mag + a))

    def __add__(self, o):
        return _V._rnd(self.v + o.v, self.a + o.a, self.v.abs() + o.v.abs())

    def __sub__(self, o):
        return _V._rnd(self.v - o.v, self.a + o.a, self.v.abs() + o.v.abs())

    def __mul__(self, o):
        v = self.v * o.v
        return _V._rnd(v, self.v.abs() * o.a + o.v.abs() * self.a + self.a * o.a, v.abs())

    def __truediv__(self, o):
        v = self.v / o.v
        den = o.v.abs() - o.a
        assert bool((den > 0).all()), 'a divisor within its allowance of 0'
        return _V._rnd(v, (self.a + v.abs() * o.a) / den, v.abs())

    def sqrt(self):
        v = self.v.sqrt()
        return _V._rnd(v, v - (self.v - self.a).clamp_min(0).sqrt(), v)

    def rounded(self):
        """One fp32 rounding of an otherwise exact (double) result."""
        return _V._rnd(self.v, self.a, self.v.abs())


def _c(x):
    """An fp32 constant as the kernel reads it (exact)."""
    return _V(f32(float(x)))


def _dbl(x):
    """A value the kernel computes in double (pow, sqrt, division: within 2^-50 relative) and rounds once to fp32."""
    t = _V(x)
    t.a = 2.0 ** -50 * t.v.abs()
    return t.rounded()


def _fold_allowance(sumsq, chunks):
    """Allowance of the multi-tensor sum of squares (fp32 chunk partials, then the double fold)."""
    return SUMSQ_DEPTH * U * sumsq + (math.ceil(chunks / THREADS) + 8) * 2.0 ** -53 * sumsq


# ------------------------------------------------------------------ chunk geometry mirrors
def _grad_starts(cases):
    """Float offset of each tensor's gradient view in one flat buffer: 16-byte aligned plus the case's offset."""
    starts, pos = [], 0
    for numel, off, _ in cases:
        pos = (pos + 3) // 4 * 4 + off
        starts.append(pos)
        pos += numel
    return starts, pos + 4


def _chunks(cases):
    """Mirror of optim._build's chunk table and of the kernels' float4 condition (p and the state tensors are separate
    allocations, 16-byte aligned; the gradient view is aligned when its offset is): [(tensor, chunk, n, vec)]."""
    out = []
    for i, (numel, off, _) in enumerate(cases):
        for c in range(-(-numel // CHUNK)):
            n = min(CHUNK, numel - c * CHUNK)
            out.append((i, c, n, off == 0 and n % 4 == 0))
    return out


def test_cases_reach_every_chunk_path_cpu():
    """The chunk-geometry cases reach every path of the multi-tensor kernels: every chunk edge size, a full float4
    chunk, the scalar path for each misaligned gradient offset, float4 chunks followed by a ragged last chunk, and more
    than 256 chunks for the clip fold; the Muon case has a matrix of more than 256 chunks."""
    from simpleaicv_pytorch_training_examples_b200 import _lib
    assert _lib.load().saicv_opt_chunk() == CHUNK
    chunks = _chunks(GEOM)
    sizes = {numel for numel, _, _ in GEOM}
    assert {1, 3, 4, 7, 8191, 8192, 8193, 3 * CHUNK + 5, BIG} <= sizes
    assert any(vec and n == CHUNK for _, _, n, vec in chunks)
    for off in (1, 2, 3):
        assert any(GEOM[i][1] == off and not vec for i, _, _, vec in chunks), off
    mixed = [i for i in range(len(GEOM)) if any(t == i and vec for t, _, _, vec in chunks)
             and [n for t, _, n, _ in chunks if t == i][-1] % 4]
    assert mixed, 'no tensor with float4 chunks and a ragged last chunk'
    assert len(chunks) > THREADS
    for gi in range(3):        # every group has a float4 and a scalar chunk (the Nesterov group included)
        vecs = {vec for i, _, _, vec in chunks if GEOM[i][2] == gi}
        assert vecs == {True, False}, gi
    assert SGD_GROUPS[2][3] and any(GEOM[i][2] == 2 and vec for i, _, _, vec in chunks)
    assert max(-(-math.prod(s) // CHUNK) for s in MUON_MATS) > THREADS
    starts, _ = _grad_starts(GEOM)
    assert [s % 4 for s in starts] == [off for _, off, _ in GEOM]


# ------------------------------------------------------------------ SGD / AdamW over the chunk geometry
def _geom_params(seed):
    g = gen(seed)
    return [torch.randn(numel, device='cuda', generator=g).requires_grad_(True) for numel, _, _ in GEOM]


def _geom_grads(ps, step, scale=1.0):
    """Gradient views at the cases' offsets into one flat buffer (the same storage every step)."""
    starts, total = _grad_starts(GEOM)
    flat = torch.randn(total, device='cuda', generator=gen(1000 + step)) * scale
    return flat, [flat[s:s + p.numel()] for s, p in zip(starts, ps)]


def _sgd(ps, **kw):
    from simpleaicv_pytorch_training_examples_b200 import optim
    groups = [{'params': [p for (_, _, gi), p in zip(GEOM, ps) if gi == k], 'lr': lr, 'weight_decay': wd, 'momentum': mom,
               'nesterov': nest} for k, (lr, wd, mom, nest) in enumerate(SGD_GROUPS)]
    return optim.FusedSGD(groups, **kw)


def _adamw(ps, fused=True):
    from simpleaicv_pytorch_training_examples_b200 import optim
    groups = [{'params': [p for (_, _, gi), p in zip(GEOM, ps) if gi == k], 'lr': lr, 'weight_decay': wd}
              for k, (lr, wd) in enumerate(ADAMW_GROUPS)]
    cls = optim.FusedAdamW if fused else torch.optim.AdamW
    return cls(groups, betas=BETAS, eps=EPS)


def _state(opt, p, key):
    st = opt.state[p]
    return st[key].detach().clone() if key in st else torch.zeros_like(p)


def _snap(opt, ps, keys):
    """Stored inputs of the next step: p, g and the state tensors (zeros before the state exists)."""
    return [(p.detach().clone(), None if p.grad is None else p.grad.clone(), [_state(opt, p, k) for k in keys]) for p in ps]


def _sgd_check(what, p0, g0, b0, p1, b1, gs, lr, wd, mom, nest):
    """multi_sgd_kernel: d = g gs + wd p, b' = mu b + d, p' = p - lr (nesterov ? d + mu b' : b')."""
    g = _V(g0) if gs is None else _V(g0) * _c(gs)
    d = g + _c(wd) * _V(p0)
    bn = _c(mom) * _V(b0) + d
    check('sgd', f'{what} momentum buffer', b1, bn.v, bn.a)
    upd = d + _c(mom) * _V(b1) if nest else _V(b1)
    pn = _V(p0) - _c(lr) * upd
    check('sgd', f'{what} parameter', p1, pn.v, pn.a)


def _adamw_check(what, p0, g0, m0, v0, p1, m1, v1, gs, lr, wd, t):
    """multi_adamw_kernel (torch.optim.AdamW): p *= 1 - lr wd; m' = m + (g - m)(1 - b1); v' = b2 v + (1 - b2) g g;
    p' = p - fp32(lr / (1 - b1^t)) m' / (sqrt(v') / fp32(sqrt(1 - b2^t)) + eps)."""
    b1, b2 = f32(BETAS[0]), f32(BETAS[1])
    g = _V(g0) if gs is None else _V(g0) * _c(gs)
    mn = _V(m0) + (g - _V(m0)) * (_c(1) - _c(b1))
    vn = _c(b2) * _V(v0) + (_c(1) - _c(b2)) * g * g
    check('adamw', f'{what} exp_avg', m1, mn.v, mn.a)
    check('adamw', f'{what} exp_avg_sq', v1, vn.v, vn.a)
    step, bc2s = _dbl(f32(lr) / (1.0 - b1 ** t)), _dbl(math.sqrt(1.0 - b2 ** t))
    pd = _V(p0) * (_c(1) - _c(lr) * _c(wd))
    pn = pd - step * (_V(m1) / (_V(v1).sqrt() / bc2s + _c(EPS)))
    check('adamw', f'{what} parameter', p1, pn.v, pn.a)


def _set_lr(opt, step, base):
    for g, row in zip(opt.param_groups, base):
        g['lr'] = row[0] * 0.9 ** step


def _check_table(opt):
    """The device chunk table against the mirror; its rows are the tensors in param-group order."""
    chunks = _chunks([case for gi in range(len(SGD_GROUPS)) for case in GEOM if case[2] == gi])
    tab = opt._tab
    assert tab['ct'].tolist() == [i for i, _, _, _ in chunks] and tab['ci'].tolist() == [c for _, c, _, _ in chunks]


@gpu
@pytest.mark.parametrize('kind', ['sgd', 'adamw'])
def test_multi_tensor_step_conforms(kind):
    """10 steps over the chunk-geometry tensors in three groups, lr rewritten every step (the ring wraps): every element
    of p and the state against the float64 step on that step's stored inputs."""
    ps = _geom_params(1)
    opt = _sgd(ps) if kind == 'sgd' else _adamw(ps)
    base = SGD_GROUPS if kind == 'sgd' else ADAMW_GROUPS
    keys = ['momentum_buffer'] if kind == 'sgd' else ['exp_avg', 'exp_avg_sq']
    for step in range(STEPS):
        _set_lr(opt, step, base)
        _, grads = _geom_grads(ps, step)
        for p, g in zip(ps, grads):
            p.grad = g
        snap = _snap(opt, ps, keys)
        opt.step()
        torch.cuda.synchronize()
        if step == 0:
            _check_table(opt)
            for p, (_, off, _) in zip(ps, GEOM):
                assert p.data_ptr() % 16 == 0 and p.grad.data_ptr() % 16 == 4 * off
                assert all(opt.state[p][k].data_ptr() % 16 == 0 for k in keys)
        for i, (p, (p0, g0, st0)) in enumerate(zip(ps, snap)):
            gi = GEOM[i][2]
            lr = opt.param_groups[gi]['lr']
            what = f'{kind} step {step} tensor {i} (numel {GEOM[i][0]}, offset {GEOM[i][1]})'
            if kind == 'sgd':
                _, wd, mom, nest = SGD_GROUPS[gi]
                _sgd_check(what, p0, g0, st0[0], p.detach(), opt.state[p]['momentum_buffer'], None, lr, wd, mom, nest)
            else:
                _adamw_check(what, p0, g0, st0[0], st0[1], p.detach(), opt.state[p]['exp_avg'], opt.state[p]['exp_avg_sq'],
                             None, lr, ADAMW_GROUPS[gi][1], step + 1)
    assert int(opt._step_dev) == STEPS


@gpu
def test_adamw_with_intermittent_gradients_keeps_per_parameter_steps():
    """Parameters whose .grad is None on some steps (zero_grad(), an unused branch) are skipped, as torch.optim.AdamW
    skips them: each update uses the parameter's own step count, per element against the float64 step with torch's
    count; the skipped parameters and their moments keep every bit; state_dict()'s 'step' equals torch's and a
    state_dict round trip continues bit for bit."""
    ps = _geom_params(2)
    ref_ps = [p.detach().clone().requires_grad_(True) for p in ps]
    opt, ref = _adamw(ps), _adamw(ref_ps, fused=False)
    has = lambda i, step: (i + step) % 3 != 1 or step == 0   # noqa: E731  every tensor misses some steps
    for step in range(STEPS):
        _set_lr(opt, step, ADAMW_GROUPS)
        _set_lr(ref, step, ADAMW_GROUPS)
        _, grads = _geom_grads(ps, step)
        for i, (p, q, g) in enumerate(zip(ps, ref_ps, grads)):
            p.grad = g if has(i, step) else None
            q.grad = g.clone() if has(i, step) else None
        snap = _snap(opt, ps, ['exp_avg', 'exp_avg_sq'])
        opt.step()
        ref.step()
        torch.cuda.synchronize()
        for i, (p, q, (p0, g0, st0)) in enumerate(zip(ps, ref_ps, snap)):
            if g0 is None:
                same(f'adamw step {step} tensor {i} without a gradient', p.detach(), p0)
                for k, s0 in zip(['exp_avg', 'exp_avg_sq'], st0):
                    if k in opt.state[p]:
                        same(f'adamw step {step} tensor {i} {k} without a gradient', opt.state[p][k], s0)
                continue
            t = int(ref.state[q]['step'])
            gi = GEOM[i][2]
            _adamw_check(f'adamw intermittent step {step} tensor {i} (t = {t})', p0, g0, st0[0], st0[1], p.detach(),
                         opt.state[p]['exp_avg'], opt.state[p]['exp_avg_sq'], None, opt.param_groups[gi]['lr'],
                         ADAMW_GROUPS[gi][1], t)
    sd, rsd = opt.state_dict(), ref.state_dict()
    assert sorted(sd['state']) == sorted(rsd['state'])
    for i in rsd['state']:
        assert float(sd['state'][i]['step']) == float(rsd['state'][i]['step']), i
    # the counts round-trip: a second optimizer loaded from the state dict continues bit for bit
    ps2 = [p.detach().clone().requires_grad_(True) for p in ps]
    opt2 = _adamw(ps2)
    opt2.load_state_dict(copy.deepcopy(sd))
    for step in range(STEPS, STEPS + 2):
        for o in (opt, opt2):
            _set_lr(o, step, ADAMW_GROUPS)
        _, grads = _geom_grads(ps, step)
        for i, (p, p2, g) in enumerate(zip(ps, ps2, grads)):
            p.grad = g if has(i, step) else None
            p2.grad = g.clone() if has(i, step) else None
        opt.step()
        opt2.step()
    torch.cuda.synchronize()
    for i, (p, p2) in enumerate(zip(ps, ps2)):
        same(f'adamw tensor {i} after a state_dict round trip', p2.detach(), p.detach())


# ------------------------------------------------------------------ the global-norm clip
def _clip_check(what, opt, grads, max_norm):
    """Stored norm against float64 sqrt(sum g^2) within the fold allowance; the coefficient bit-exact from the stored
    norm.  Returns the stored coefficient (fp32, 0-dim)."""
    clip = opt._clip.clone()
    sumsq = sum(float(g.double().square().sum()) for g in grads)
    chunks = sum(-(-g.numel() // CHUNK) for g in grads)
    sq = _V(torch.tensor(sumsq, dtype=torch.float64, device='cuda'), torch.tensor(_fold_allowance(sumsq, chunks),
                                                                                  dtype=torch.float64, device='cuda'))
    norm = sq.sqrt()
    check('clip', f'{what}: norm ({chunks} chunks)', clip[1:2], norm.v.view(1), norm.a.view(1))
    c = torch.tensor(f32(max_norm), device='cuda') / (clip[1] + torch.tensor(1e-6, device='cuda'))
    want = c if bool(torch.isnan(c)) else torch.clamp(c, max=1.0)
    same(f'{what}: coefficient', clip[0:1], want.view(1))
    if float(clip[1]) + f32(1e-6) <= f32(max_norm):
        assert float(clip[0]) == 1.0
    return clip[0]


@gpu
def test_clip_conforms_and_scales_exactly_one_step():
    """More than 256 chunks (several partials per thread of the fold), a coefficient < 1 used by exactly the next SGD
    step (on both memory paths, every group), then a step without clip using the raw gradients; all-zero gradients and a
    single tensor give coefficient 1."""
    ps = _geom_params(3)
    opt = _sgd(ps)
    for step in range(3):
        _set_lr(opt, step, SGD_GROUPS)
        _, grads = _geom_grads(ps, step)
        for p, g in zip(ps, grads):
            p.grad = g
        clipped = step < 2
        gs = None
        if clipped:
            opt.clip_grad_norm(5.0)
            torch.cuda.synchronize()
            gs = _clip_check(f'clip step {step}', opt, grads, 5.0)
            assert float(gs) < 0.01
        snap = _snap(opt, ps, ['momentum_buffer'])
        opt.step()
        torch.cuda.synchronize()
        for i, (p, (p0, g0, st0)) in enumerate(zip(ps, snap)):
            gi = GEOM[i][2]
            _, wd, mom, nest = SGD_GROUPS[gi]
            _sgd_check(f'sgd {"clipped " if clipped else ""}step {step} tensor {i}', p0, g0, st0[0], p.detach(),
                       opt.state[p]['momentum_buffer'], gs, opt.param_groups[gi]['lr'], wd, mom, nest)
    # all-zero gradients: norm 0, coefficient 1
    zeros = [torch.zeros_like(p) for p in ps]
    for p, z in zip(ps, zeros):
        p.grad = z
    opt.clip_grad_norm(1.0)
    torch.cuda.synchronize()
    assert float(_clip_check('clip of zero gradients', opt, zeros, 1.0)) == 1.0 and float(opt._clip[1]) == 0.0
    # a single tensor (one chunk) whose norm is below max_norm
    from simpleaicv_pytorch_training_examples_b200 import optim
    q = torch.randn(77, device='cuda', generator=gen(4)).requires_grad_(True)
    q.grad = torch.randn(77, device='cuda', generator=gen(5)) * 0.01
    one = optim.FusedSGD([q], lr=0.1, momentum=0.9)
    one.clip_grad_norm(1.0)
    torch.cuda.synchronize()
    assert float(_clip_check('clip of a single tensor', one, [q.grad], 1.0)) == 1.0


@gpu
@pytest.mark.parametrize('bad', ['nan', 'inf'])
def test_clip_with_a_non_finite_gradient_follows_torch(bad):
    """One non-finite gradient element, clip then SGD, against torch.nn.utils.clip_grad_norm_ + torch.optim.SGD on the
    same data.  NaN: the norm and the coefficient are NaN and every element of every parameter becomes NaN, as in torch.
    inf: the norm is inf, the coefficient 0, and only that element becomes NaN; the others take the step with g = 0."""
    from simpleaicv_pytorch_training_examples_b200 import optim
    shapes = [(1000, 64), (8193,), (5, 3, 3, 3)]
    g = gen(6)
    ps = [torch.randn(*s, device='cuda', generator=g).requires_grad_(True) for s in shapes]
    ref_ps = [p.detach().clone().requires_grad_(True) for p in ps]
    grads = [torch.randn(*s, device='cuda', generator=g) for s in shapes]
    grads[1][4321] = float(bad)
    for p, q, gr in zip(ps, ref_ps, grads):
        p.grad, q.grad = gr.clone(), gr.clone()
    opt = optim.FusedSGD(ps, lr=0.1, momentum=0.9, weight_decay=1e-2)
    ref = torch.optim.SGD(ref_ps, lr=0.1, momentum=0.9, weight_decay=1e-2)
    opt.clip_grad_norm(1.0)
    torch.nn.utils.clip_grad_norm_(ref_ps, 1.0)
    snap = _snap(opt, ps, ['momentum_buffer'])
    opt.step()
    ref.step()
    torch.cuda.synchronize()
    clip = opt._clip.clone()
    if bad == 'nan':
        assert bool(torch.isnan(clip).all()), f'stored clip {clip.tolist()}: a NaN norm must give a NaN coefficient'
    else:
        assert float(clip[1]) == math.inf and float(clip[0]) == 0.0, clip.tolist()
    for i, (p, q, (p0, g0, st0)) in enumerate(zip(ps, ref_ps, snap)):
        nan_mine, nan_ref = torch.isnan(p.detach()), torch.isnan(q.detach())
        assert torch.equal(nan_mine, nan_ref), \
            f'tensor {i}: {int(nan_mine.sum())} NaN elements, torch has {int(nan_ref.sum())}'
        if bad == 'inf':
            keep = ~nan_ref
            assert int(nan_ref.sum()) == (1 if i == 1 else 0)
            _sgd_check(f'sgd after an inf clip, tensor {i}', p0[keep], g0[keep], st0[0][keep], p.detach()[keep],
                       opt.state[p]['momentum_buffer'][keep], clip[0], 0.1, 1e-2, 0.9, False)


# ------------------------------------------------------------------ bf16 operand copies
SHADOW_CONV = [(8, 5, 3, 3, 8, 80), (16, 30, 3, 3, 32, 296), (32, 6, 1, 1, 8, 16), (64, 60, 3, 3, 64, 584)]   # k, c, r, s, cp, kpad
SHADOW_LIN = [(100, 64, 12), (300, 77, 5)]   # n, k, extra rows


def _shadow_setup(opt_kind, offset, seed):
    """Parameters with operand copies (Linear [N + extra][K] and conv [K][kpad], tap-major with cp >= c), filled with the
    sentinel; gradients at a float offset (0: float4 path where numel % 4 == 0, 1: scalar path)."""
    from simpleaicv_pytorch_training_examples_b200 import optim
    g = gen(seed)
    params, copies = [], []
    for n, k, extra in SHADOW_LIN:
        params.append(torch.randn(n, k, device='cuda', generator=g).requires_grad_(True))
        copies.append((torch.full((n + extra, k), SENTINEL, dtype=torch.int16, device='cuda').view(torch.bfloat16), None))
    for k, c, r, s, cp, kpad in SHADOW_CONV:
        params.append(torch.randn(k, c, r, s, device='cuda', generator=g).requires_grad_(True))
        copies.append((torch.full((k, kpad), SENTINEL, dtype=torch.int16, device='cuda').view(torch.bfloat16),
                       (c, r * s, cp, kpad)))
    if opt_kind == 'sgd':
        opt = optim.FusedSGD(params, lr=0.1, momentum=0.9, weight_decay=1e-2)
    elif opt_kind == 'adamw':
        opt = optim.FusedAdamW(params, lr=1e-2)
    else:
        opt = optim.FusedMuon(lr=0.02, wd=0.05, muon_params=params[:-1], adamw_params=params[-1:])
    for p, (w, conv) in zip(params, copies):
        opt.register_shadow(p, w, conv=conv)
    total = sum(p.numel() + 4 for p in params)
    flat = torch.randn(total, device='cuda', generator=g)
    pos = offset
    for p in params:
        p.grad = flat[pos:pos + p.numel()].view_as(p)
        pos += (p.numel() + 3) // 4 * 4
    return opt, params, copies


def _mapped(p, w, conv):
    """(mapped elements of the copy w as they would hold rne(p), mask of the mapped positions)."""
    want = torch.full_like(w, 0)
    mask = torch.zeros(w.shape, dtype=torch.bool, device='cuda')
    pb = p.detach().to(torch.bfloat16)          # fp32 -> bf16 rounds to nearest even, once
    if conv is None:
        want[:p.shape[0]] = pb
        mask[:p.shape[0]] = True
    else:
        c, rs, cp, kpad = conv
        k = p.shape[0]
        wv, mv = want[:, :rs * cp].view(k, rs, cp), mask[:, :rs * cp].view(k, rs, cp)
        wv[:, :, :c] = pb.reshape(k, c, rs).permute(0, 2, 1)
        mv[:, :, :c] = True
    return want, mask


@gpu
@pytest.mark.parametrize('offset', [0, 1])
@pytest.mark.parametrize('opt_kind', ['sgd', 'adamw', 'muon'])
def test_operand_copies_are_exact_and_padding_is_untouched(opt_kind, offset):
    """Every mapped element of each copy equals rne_bf16 of the stored fp32 p' bit for bit; every unmapped one (extra
    rows, channel padding cp > c, tap padding kpad > rs cp) keeps its sentinel.  Conv shapes with c rs not a multiple of
    4, so float4 groups cross filters; offset 0 takes the float4 path, offset 1 the scalar one (SGD / AdamW)."""
    opt, params, copies = _shadow_setup(opt_kind, offset, 7 + offset)
    for step in range(2):
        opt.step()
        torch.cuda.synchronize()
        for i, (p, (w, conv)) in enumerate(zip(params, copies)):
            want, mask = _mapped(p, w, conv)
            what = f'{opt_kind} offset {offset} step {step} copy {i} ({tuple(p.shape)})'
            exact('operand copies', f'{what} mapped elements', w[mask], want[mask])
            bits = w.view(torch.int16)[~mask]
            assert bool((bits == SENTINEL).all()), f'{what}: {int((bits != SENTINEL).sum())} unmapped elements written'


# ------------------------------------------------------------------ Newton-Schulz GEMMs
NS_SHAPES = [(8, 8, 1), (8, 72, 3), (120, 72, 24), (120, 1000, 3), (120, 2304, 24), (136, 8, 24), (136, 1000, 1),
             (200, 1000, 24), (200, 2304, 3), (768, 1000, 3), (768, 2304, 1)]   # m, n, batch
# mode 1 reads only [m][m] operands: one case per (m, batch)
NS_CASES = [(mode, m, m if mode == 1 else n, b) for mode in (0, 1, 2) for m, n, b in NS_SHAPES]
NS_CASES = sorted(set(NS_CASES), key=NS_CASES.index)
NS_ALPHA_BETA = {0: (1.0, 0.0), 1: (2.0315, -4.7750), 2: (1.0, 3.4445)}          # the quintic iteration's (c, b), (1, a)


def _ns_operand(batch, rows, cols, seed):
    """bf16 [batch, rows, cols] whose neighbouring matrices differ in magnitude by 2^8 and 2^16: a tile that read or wrote
    rows of the next matrix would leave the bound."""
    scale = torch.tensor([2.0 ** (8 * (j % 3)) for j in range(batch)], device='cuda').view(batch, 1, 1)
    return (torch.randn(batch, rows, cols, device='cuda', generator=gen(seed)) * scale).to(torch.bfloat16)


@gpu
@pytest.mark.parametrize('mode,m,n,batch', NS_CASES)
def test_ns_gemm_conforms(mode, m, n, batch):
    """saicv_ns_gemm, the batched VAR_NS GEMM over 3-D TMA maps: mode 0 X X^T, mode 1 alpha A A + beta A, mode 2
    alpha B X + beta X (aux by TMA), per element against float64 in every matrix of the batch; the output starts as NaN,
    so an element no tile wrote fails."""
    alpha, beta = NS_ALPHA_BETA[mode]
    x = _ns_operand(batch, m, n if mode == 0 else m, 10 + mode)
    y = _ns_operand(batch, m, n, 20) if mode == 2 else None
    out = torch.full((batch, m, n if mode == 2 else m), float('nan'), device='cuda', dtype=torch.bfloat16)
    call('saicv_ns_gemm', mode, x, y, out, batch, m, n, ctypes.c_float(alpha), ctypes.c_float(beta))
    xd = x.double()
    if mode == 0:
        ref, s = xd @ xd.mT, xd.abs() @ xd.abs().mT
    elif mode == 1:
        ref, s = xd @ xd, xd.abs() @ xd.abs()
    else:
        ref, s = xd @ y.double(), xd.abs() @ y.double().abs()
    allow = acc_allowance(ref, s)
    v = ref
    if mode:
        a, b = f32(alpha), f32(beta)
        aux = (x if mode == 1 else y).double()
        v = a * ref + b * aux
        allow = abs(a) * allow + 2 * U * (abs(a) * (ref.abs() + allow) + (b * aux).abs())
    check(None, f'ns_gemm mode {mode} {batch}x{m}x{n}', out, v, allow, s)


# ------------------------------------------------------------------ Muon prep and apply
def _muon_setup(nesterov, seed):
    from simpleaicv_pytorch_training_examples_b200 import optim
    g = gen(seed)
    mats = [(torch.randn(*s, device='cuda', generator=g) * 0.1).requires_grad_(True) for s in MUON_MATS]
    adams = [(torch.randn(*s, device='cuda', generator=g) * 0.1).requires_grad_(True) for s in MUON_ADAMW]
    opt = optim.FusedMuon(lr=0.02, wd=0.05, muon_params=mats, momentum=0.95, nesterov=nesterov, ns_steps=5,
                          adamw_params=adams, adamw_betas=BETAS, adamw_eps=EPS)
    return opt, mats, adams


def _muon_has(kind, i, step):
    """Gradient schedule: one matrix and one AdamW row miss steps."""
    if kind == 'mat':
        return not (i == 4 and step == 1)
    return not (i == 2 and step in (1, 2))


def _slot(opt, ns, p):
    """The parameter's slot of the Newton-Schulz buffer ([round8(min)][ld]), and its [rows][cols] view of the matrix."""
    off, ld = opt._slots[id(p)]
    r, c = p.shape[0], p.numel() // p.shape[0]
    mp = (min(r, c) + 7) // 8 * 8
    slot = ns[off:off + mp * ld].view(mp, ld)
    return slot, (slot[:c, :r].t() if r > c else slot[:r, :c]), min(r, c), max(r, c)


def _muon_table(opt):
    from simpleaicv_pytorch_training_examples_b200 import optim
    rows = np.frombuffer(opt._tab['muon'].cpu().numpy().tobytes(), dtype=optim._MUON_DTYPE)
    return {id(p): rows[i] for i, (_, p) in enumerate(opt._params())}


@gpu
@pytest.mark.parametrize('nesterov,clip', [(True, False), (False, False), (True, True)])
def test_muon_prep_and_apply_conform(nesterov, clip, monkeypatch):
    """FusedMuon over 4 steps with lr rewritten every step and gradients missing on some steps.  Prep: the momentum buffer
    and the slot X = bf16(u / (||bf16(u)||_F + 1e-7)) per element (read before the Newton-Schulz iterations; transposed
    when rows > cols; padding rows and columns zero).  Apply: Muon rows p' = p (1 - lr wd) - lr adj U with U the slot after
    the iterations, AdamW rows by the reference's formula with t = adam_steps + 1; adam_steps advance only for rows with
    a gradient, the ring step once per step."""
    from simpleaicv_pytorch_training_examples_b200 import optim
    opt, mats, adams = _muon_setup(nesterov, 30 + nesterov + 2 * clip)
    real_ns = optim.newton_schulz
    prep = []

    def spy(x, *args):
        if not prep:
            prep.append(opt._ns.clone())
        return real_ns(x, *args)

    monkeypatch.setattr(optim, 'newton_schulz', spy)
    b1, b2 = f32(BETAS[0]), f32(BETAS[1])
    mom = 0.95
    for step in range(4):
        opt.param_groups[0]['lr'] = 0.02 * 0.9 ** step
        lr, wd = opt.param_groups[0]['lr'], opt.param_groups[0]['wd']
        g = gen(100 + step)
        for i, p in enumerate(mats):
            p.grad = torch.randn(p.shape, device='cuda', generator=g) if _muon_has('mat', i, step) else None
        for i, p in enumerate(adams):
            p.grad = torch.randn(p.shape, device='cuda', generator=g) if _muon_has('adam', i, step) else None
        gs = None
        if clip:
            opt.clip_grad_norm(1.0)
            torch.cuda.synchronize()
            gs = _clip_check(f'muon clip step {step}', opt, [p.grad for p in mats + adams if p.grad is not None], 1.0)
            assert float(gs) < 1.0
        snap_m = [(p.detach().clone(), None if p.grad is None else p.grad.clone(),
                   opt.state[p]['momentum_buffer'].clone() if 'momentum_buffer' in opt.state[p]
                   else torch.zeros(p.shape[0], p.numel() // p.shape[0], device='cuda')) for p in mats]
        snap_a = _snap(opt, adams, ['moment1', 'moment2'])
        adam0 = opt._adam_steps.clone() if opt._adam_steps is not None else torch.zeros(len(adams), dtype=torch.int32, device='cuda')
        ring0 = int(opt._step_dev) if opt._hyper_host is not None else 0
        prep.clear()
        opt.step()
        torch.cuda.synchronize()
        table = _muon_table(opt)
        ns_after = opt._ns
        for i, (p, (p0, g0, b0)) in enumerate(zip(mats, snap_m)):
            what = f'muon step {step} matrix {i} {tuple(p.shape)}'
            slot0, x0, lo, hi = _slot(opt, prep[0], p)
            slot1, u1, _, _ = _slot(opt, ns_after, p)
            for name, sl in (('prep', slot0), ('apply', slot1)):
                assert not sl[lo:].any() and not sl[:, hi:].any(), f'{what}: {name} slot padding is not zero'
            if g0 is None:
                same(f'{what} without a gradient', p.detach(), p0)
                continue
            r, c = b0.shape
            gm = _V(g0.reshape(r, c)) if gs is None else _V(g0.reshape(r, c)) * _c(gs)
            b1s = opt.state[p]['momentum_buffer']
            bn = _c(mom) * _V(b0) + gm
            check('muon prep', f'{what} momentum buffer', b1s, bn.v, bn.a)
            if nesterov:
                u = gm + _c(mom) * _V(b1s)
                ub = _V(u.v, u.a + quantum_bf16(u.v.abs() + u.a) / 2)
            else:
                ub = _V(rne_bf16(b1s.double()))
            sumsq = float(ub.v.square().sum())
            unc = float((2 * ub.v.abs() * ub.a + ub.a.square()).sum())
            chunks = -(-p.numel() // CHUNK)
            sq = _V(torch.tensor(sumsq, dtype=torch.float64, device='cuda'),
                    torch.tensor(unc + _fold_allowance(sumsq + unc, chunks), dtype=torch.float64, device='cuda'))
            inv = _c(1) / (sq.sqrt() + _c(1e-7))
            x = ub * inv
            check('muon prep', f'{what} slot X ({"transposed" if p.shape[0] > c else "direct"})', x0, x.v, x.a)
            row = table[id(p)]
            assert int(row['transposed']) == int(p.shape[0] > c)
            pn = _V(p0) * (_c(1) - _c(lr) * _c(wd)) - _c(lr) * _V(float(row['adj'])) * _V(u1.reshape(p.shape))
            check('muon apply', f'{what} parameter', p.detach(), pn.v, pn.a)
        for i, (p, (p0, g0, st0)) in enumerate(zip(adams, snap_a)):
            what = f'muon step {step} AdamW row {i} {tuple(p.shape)}'
            if g0 is None:
                same(f'{what} without a gradient', p.detach(), p0)
                continue
            t = int(adam0[i]) + 1
            gv = _V(g0) if gs is None else _V(g0) * _c(gs)
            m1, v1 = opt.state[p]['moment1'], opt.state[p]['moment2']
            mn = _V(st0[0]) + (gv - _V(st0[0])) * (_c(1) - _c(b1))
            vn = _V(st0[1]) + (gv * gv - _V(st0[1])) * (_c(1) - _c(b2))
            check('muon apply', f'{what} moment1', m1, mn.v, mn.a)
            check('muon apply', f'{what} moment2', v1, vn.v, vn.a)
            a = _dbl(f32(lr) * math.sqrt(1.0 - b2 ** t) / (1.0 - b1 ** t))
            pn = _V(p0) * (_c(1) - _c(lr) * _c(wd)) - a * (_V(m1) / (_c(EPS) + _V(v1).sqrt()))
            check('muon apply', f'{what} parameter', p.detach(), pn.v, pn.a)
        want = adam0 + torch.tensor([int(_muon_has('adam', i, step)) for i in range(len(adams))], dtype=torch.int32,
                                    device='cuda')
        assert torch.equal(opt._adam_steps, want), (step, opt._adam_steps.tolist(), want.tolist())
        assert int(opt._step_dev) == ring0 + 1
