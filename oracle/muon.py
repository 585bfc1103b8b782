"""Float64 restatement of one step of the Muon optimizer as the reference defines it (tools/muon_optimizer.py): SGD
momentum (optionally Nesterov) whose update of every >= 2-D weight is replaced by a quintic Newton-Schulz
orthogonalisation, and an AdamW backup with the reference's own update (moments by lerp, bias corrections folded into the
step size, eps outside the square root, a per-parameter step count).

``emulate_bf16=True`` rounds to bf16 where the reference's iteration stores bf16 tensors (every product, scaled term and
sum), so that it reproduces what the reference computes on the CPU; with False the iteration runs in float64 throughout.
"""
import math

import torch

NS_COEFFS = (3.4445, -4.7750, 2.0315)


def _round(t, emulate_bf16):
    return t.to(torch.bfloat16).to(torch.float64) if emulate_bf16 else t


def zeropower(g, steps, emulate_bf16=False):
    """Newton-Schulz orthogonalisation of the 2-D matrix g (float64 result, g's orientation)."""
    r = lambda t: _round(t, emulate_bf16)   # noqa: E731
    a, b, c = NS_COEFFS
    x = r(g.to(torch.float64))
    tall = x.shape[0] > x.shape[1]
    if tall:
        x = x.T
    nrm = r(r(x.norm()) + 1e-7)
    x = r(x / nrm)
    for _ in range(steps):
        m = r(x @ x.T)
        bm = r(r(b * m) + r(r(c * m) @ m))
        x = r(r(a * x) + r(bm @ x))
    return x.T if tall else x


def step(params, grads, state, use_muon, lr, wd, momentum=0.95, nesterov=True, ns_steps=5, betas=(0.9, 0.999), eps=1e-8,
         emulate_bf16=False):
    """One optimizer step in place.  params: {name: float64 tensor}; grads: {name: tensor or None}; state: {name: dict}
    with the reference's keys (momentum_buffer 2-D; step, moment1, moment2); use_muon: {name: bool}."""
    for name, p in params.items():
        g = grads.get(name)
        if g is None:
            continue
        g = g.to(torch.float64)
        st = state.setdefault(name, {})
        if use_muon[name]:
            g2 = g.reshape(g.shape[0], -1)
            buf = st.get('momentum_buffer')
            buf = g2.clone() if buf is None else momentum * buf.to(torch.float64) + g2
            st['momentum_buffer'] = buf
            u = zeropower(g2 + momentum * buf if nesterov else buf, ns_steps, emulate_bf16)
            adj = lr * 0.2 * math.sqrt(max(p.shape[0], p.shape[1]))
            p.mul_(1 - lr * wd).sub_(adj * u.reshape(p.shape))
        else:
            if 'step' not in st:
                st['step'] = 0
                st['moment1'] = torch.zeros_like(p)
                st['moment2'] = torch.zeros_like(p)
            st['step'] += 1
            t = st['step']
            m1 = st['moment1'].to(torch.float64)
            m2 = st['moment2'].to(torch.float64)
            m1 = m1 + (g - m1) * (1 - betas[0])
            m2 = m2 + (g * g - m2) * (1 - betas[1])
            st['moment1'], st['moment2'] = m1, m2
            scale = (1 - betas[0] ** t) / (1 - betas[1] ** t) ** 0.5
            p.mul_(1 - lr * wd).sub_((lr / scale) * m1 / (eps + m2.sqrt()))
    return params
