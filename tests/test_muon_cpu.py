"""Muon on the host side: build_optimizer's parameter split and description list against the reference (live when its
copy is installed, and always against tests/golden/muon_3steps.pto), the float64 oracle (oracle/muon.py) against the
fixture the reference's Muon wrote, and the clear error on CPU parameters."""
import os
import sys

import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, 'golden'))
FIXTURE = os.path.join(HERE, 'golden', 'muon_3steps.pto')


def _fixture():
    return torch.load(FIXTURE, weights_only=False)


class _Cfg:
    def __init__(self, optimizer):
        self.optimizer = optimizer


def test_split_and_description_match_the_fixture():
    import make_muon_golden
    from simpleaicv_pytorch_training_examples_b200.tools import utils
    fx = _fixture()
    muon, adamw, info = utils.muon_split(fx['optimizer'][1], make_muon_golden.ParamSet())
    assert info == fx['descr']
    assert [n for n, _ in muon + adamw] == fx['order']


def _models():
    import test_operands_cpu
    import make_muon_golden
    fam = test_operands_cpu._families()
    return {'fixture': make_muon_golden.ParamSet, 'vit_base_patch16': fam['vit_base_patch16'],
            'resnet18cifar': fam['resnet18cifar'], 'mae': fam['mae']}


@pytest.mark.parametrize('model_name', ['fixture', 'vit_base_patch16', 'resnet18cifar', 'mae'])
@pytest.mark.parametrize('extra', [None, ['fc', 'blocks.0.']])
def test_split_and_description_match_the_reference(model_name, extra):
    from baseline import ref_import
    if not ref_import.available():
        pytest.skip('reference not installed (oracle/build_ref.py)')
    from simpleaicv_pytorch_training_examples_b200.tools import utils
    opt = {'lr': 1e-3, 'weight_decay': 0.1}
    if extra is not None:
        opt['exclude_muon_layer_name_list'] = extra
    model = _models()[model_name]()
    ref_opt, ref_info = ref_import.module('tools.utils').build_optimizer(_Cfg(('Muon', opt)), model)
    muon, adamw, info = utils.muon_split(opt, model)
    assert info == ref_info
    ref_use = {id(p): ref_opt.state[p]['use_muon'] for g in ref_opt.param_groups for p in g['params']}
    assert all(ref_use[id(p)] for _, p in muon) and not any(ref_use[id(p)] for _, p in adamw)
    assert ref_opt.defaults['momentum'] == 0.95 and ref_opt.defaults['nesterov'] and ref_opt.defaults['ns_steps'] == 5


def _run_oracle(emulate_bf16):
    from oracle import muon as omuon
    fx = _fixture()
    opt = fx['optimizer'][1]
    g0 = fx['param_groups'][0]
    use = {n: n in fx['descr'][0]['name'] for n in fx['order']}
    params = {n: fx['params0'][n].to(torch.float64).clone() for n in fx['order']}
    state, out = {}, []
    for gs in fx['grads']:
        omuon.step(params, gs, state, use, opt['lr'], opt['weight_decay'], g0['momentum'], g0['nesterov'], g0['ns_steps'],
                   g0['adamw_betas'], g0['adamw_eps'], emulate_bf16=emulate_bf16)
        out.append({n: p.clone() for n, p in params.items()})
    return fx, out, state


@pytest.mark.parametrize('emulate_bf16', [True, False])
def test_oracle_reproduces_the_fixture(emulate_bf16):
    fx, out, state = _run_oracle(emulate_bf16)
    lr = fx['optimizer'][1]['lr']
    for k, (want, got) in enumerate(zip(fx['params'], out)):
        for n in fx['order']:
            d = (got[n] - want[n].to(torch.float64)).abs().max().item()
            if n in fx['descr'][0]['name']:
                # update = lr * adj * U with |U| <= ~1: the emulation may differ by one bf16 ulp of U (a different
                # rounding tie), float64 by the reference's bf16 error (~2% of the update over three steps)
                tol = (8e-3 if emulate_bf16 else 5e-2) * lr * 0.2 * max(want[n].shape[:2]) ** 0.5
            else:
                tol = 1e-6
            assert d <= tol, f'step {k} {n}: {d} > {tol}'
    for n, st in fx['state'].items():
        for key, v in st.items():
            if torch.is_tensor(v):
                assert v.shape == state[n][key].shape, (n, key)
                assert torch.allclose(state[n][key], v.to(torch.float64), rtol=1e-5, atol=1e-6), (n, key)
            elif key != 'use_muon':
                assert state[n][key] == v, (n, key)


def test_cpu_parameters_raise():
    import make_muon_golden
    from simpleaicv_pytorch_training_examples_b200.tools import utils
    with pytest.raises(RuntimeError, match='GPU'):
        utils.build_optimizer(_Cfg(('Muon', {'lr': 1e-3, 'weight_decay': 0.1})), make_muon_golden.ParamSet())
