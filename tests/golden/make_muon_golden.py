"""Writes tests/golden/muon_3steps.pto (not .pt: tests/test_oracle_golden.py loads every *.pt): three steps of the
reference's Muon optimizer (tools/muon_optimizer.py, built by the reference's tools/utils.py build_optimizer) on the
CPU, over a seeded parameter set with wide, tall and square
matrices, a 4-D conv weight, 1-D parameters, a name on the default exclude list (cls_token), one on a configured exclude
list (extra_head), and two parameters (one Muon, one AdamW) without a gradient in step 2.  The Newton-Schulz function is
called uncompiled (``__wrapped__`` of the reference's torch.compile wrapper).  Stored: the initial parameters, the
gradients, the parameters after every step, the final state_dict by parameter name, the reference's description list and
the optimizer configuration.

    python tests/golden/make_muon_golden.py
"""
import os
import sys

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

OUT = os.path.join(HERE, 'muon_3steps.pto')
SHAPES = {
    'wide': (48, 136), 'tall': (152, 40), 'square': (64, 64), 'conv': (32, 16, 3, 3), 'nograd': (24, 40),
    'extra_head': (40, 24), 'norm_weight': (64,), 'norm_bias': (64,), 'cls_token': (1, 1, 64),
}
NO_GRAD_IN_STEP2 = ('nograd', 'norm_bias')
OPTIMIZER = ('Muon', {'lr': 0.02, 'weight_decay': 0.05, 'exclude_muon_layer_name_list': ['extra_head']})
STEPS = 3


class ParamSet(torch.nn.Module):
    """The fixture's parameters, seeded."""

    def __init__(self, seed=0):
        super().__init__()
        g = torch.Generator().manual_seed(seed)
        for name, shape in SHAPES.items():
            setattr(self, name, torch.nn.Parameter(torch.randn(*shape, generator=g) * 0.1))


def gradients(model, step):
    g = torch.Generator().manual_seed(100 + step)
    out = {}
    for name, p in model.named_parameters():
        t = torch.randn(p.shape, generator=g) * (0.5 + step)
        out[name] = None if step == 1 and name in NO_GRAD_IN_STEP2 else t
    return out


def main():
    from baseline import ref_import
    utils = ref_import.module('tools.utils')
    muon_mod = ref_import.module('tools.muon_optimizer')
    # the reference wraps Newton-Schulz in torch.compile; the fixture runs the plain function on the CPU
    muon_mod.zeropower_via_newtonschulz5 = muon_mod.zeropower_via_newtonschulz5.__wrapped__

    class Config:
        optimizer = OPTIMIZER

    model = ParamSet()
    params0 = {n: p.detach().clone() for n, p in model.named_parameters()}
    optimizer, descr = utils.build_optimizer(Config, model)
    order = [n for d in descr for n in d['name']]   # the optimizer's parameter order: the Muon list, then the AdamW list
    grads, after = [], []
    for step in range(STEPS):
        gs = gradients(model, step)
        for n, p in model.named_parameters():
            p.grad = None if gs[n] is None else gs[n].clone()
        optimizer.step()
        grads.append(gs)
        after.append({n: p.detach().clone() for n, p in model.named_parameters()})
    sd = optimizer.state_dict()
    state = {order[i]: v for i, v in sd['state'].items()}
    torch.save({'params0': params0, 'grads': grads, 'params': after, 'state': state, 'order': order, 'descr': descr,
                'optimizer': OPTIMIZER, 'param_groups': sd['param_groups']}, OUT)
    print('wrote', OUT)


if __name__ == '__main__':
    main()
