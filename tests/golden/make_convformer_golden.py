"""Generates tests/golden/convformer_*.ptf by running the REFERENCE ConvFormer (oracle/_ref, installed by build()) on the
CPU in fp32.  The fixtures hold the seeded input batch, the state_dict key list and sha256 digests of the seeded initial
weights, the logits, loss, per-parameter gradient digests (L2 norm + a seeded sample of values), two BatchNorm buffers
after the step and the eval-mode logits.  The drop-path case also holds the per-sample scales each DropPathBlock drew
(convformer.py:131-137), so the oracle can replay them.  convformer_init_c10.ptf holds the key list, shapes and init
digests of all four variants.  (.ptf, not .pt: tests/test_oracle_golden.py replays every *.pt through make_golden.py.)

    python tests/golden/make_convformer_golden.py
"""
import os
import sys

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
from baseline import ref_import  # noqa: E402
from oracle import convformer  # noqa: E402

# (tag, arch, kwargs, num_classes, batch shape, seed)
CASES = [
    ('convformer_s18_c10_b2_64px', 'convformer_s18', {}, 10, (2, 3, 64, 64), 0),
    ('convformer_s18_c10_b4_64px_dp03', 'convformer_s18', {'drop_path_prob': 0.3}, 10, (4, 3, 64, 64), 1),
    ('convformer_m36_c10_b1_64px', 'convformer_m36', {}, 10, (1, 3, 64, 64), 2),
]
INIT_TAG, INIT_NC, INIT_SEED = 'convformer_init_c10', 10, 0
SAMPLES = 16


def make_input(shape, nc, seed):
    g = torch.Generator().manual_seed(2000 + seed)
    return torch.randn(*shape, generator=g), torch.randint(0, nc, (shape[0],), generator=g)


def sample_index(n, name):
    """Seeded positions of the gradient values a fixture stores for one tensor of n elements."""
    g = torch.Generator().manual_seed(sum(name.encode()) + n)
    return torch.randint(0, n, (min(n, SAMPLES),), generator=g)


def record_drop_scales(model):
    """Wraps every DropPathBlock so that the scales it draws are recorded: 'stages.{i}.{j}' -> [token mixer, MLP]."""
    rec = {}
    for name, mod in model.named_modules():
        if type(mod).__name__ != 'DropPathBlock':
            continue
        key = name.rsplit('.drop_path', 1)[0]
        rec[key] = []

        def fwd(x, mod=mod, orig=mod.forward, calls=rec[key]):
            before = torch.get_rng_state()
            out = orig(x)
            if mod.training and mod.drop_path_prob > 0.:
                after = torch.get_rng_state()
                torch.set_rng_state(before)        # redraw the same mask (convformer.py:131-135), then continue as before
                s = torch.empty(x.shape[0], 1, 1, 1).bernoulli_(mod.keep_path_prob).div_(mod.keep_path_prob)
                assert torch.equal(torch.get_rng_state(), after) and torch.equal(out, s * x)
                calls.append(s.view(-1).clone())
            return out
        mod.forward = fwd
    return rec


def main():
    backbones = ref_import.backbones()
    CELoss = ref_import.module('SimpleAICV.classification.losses').CELoss
    torch.set_num_threads(1)  # fixed reduction order for the recorded numbers
    init = {}
    for arch in convformer.ARCHS:
        torch.manual_seed(INIT_SEED)
        sd = backbones.__dict__[arch](num_classes=INIT_NC).state_dict()
        osd = convformer.init_state(arch, INIT_NC, INIT_SEED)
        assert list(sd) == list(osd) and all(torch.equal(sd[k], osd[k]) for k in sd), f'{arch}: oracle init != reference init'
        init[arch] = {'keys': list(sd), 'shapes': {k: tuple(v.shape) for k, v in sd.items()},
                      'hash': {k: convformer.tensor_hash(v) for k, v in sd.items()}}
    torch.save({'num_classes': INIT_NC, 'seed': INIT_SEED, 'archs': init, 'torch_version': torch.__version__},
               os.path.join(HERE, INIT_TAG + '.ptf'))
    for tag, arch, kwargs, nc, shape, seed in CASES:
        torch.manual_seed(seed)
        model = backbones.__dict__[arch](num_classes=nc, **kwargs)
        sd0 = model.state_dict()
        osd = convformer.init_state(arch, nc, seed)
        assert list(sd0) == list(osd) and all(torch.equal(sd0[k], osd[k]) for k in sd0), 'oracle init != reference init'
        hashes = {k: convformer.tensor_hash(v) for k, v in sd0.items()}
        scales = record_drop_scales(model)
        x, y = make_input(shape, nc, seed)
        model.train()
        logits = model(x)
        loss = CELoss()(logits, y)
        loss.backward()
        params = dict(model.named_parameters())
        fix = {
            'arch': arch, 'kwargs': kwargs, 'num_classes': nc, 'seed': seed, 'shape': shape, 'x': x, 'y': y,
            'keys': list(sd0), 'init_hash': hashes,
            'logits': logits.detach(), 'loss': loss.detach(),
            'grad_norm': {n: p.grad.norm().item() for n, p in params.items()},
            'grad_sample': {n: p.grad.flatten()[sample_index(p.numel(), n)].clone() for n, p in params.items()},
            'buffers': {k: v.clone() for k, v in model.state_dict().items()
                        if k.startswith(('downsample_layers.0.post_norm.', 'stages.3.2.norm2.'))},
            'drop_scales': {k: v for k, v in scales.items() if v},
            'torch_version': torch.__version__,
        }
        model.eval()
        with torch.no_grad():
            fix['eval_logits'] = model(x).clone()
        path = os.path.join(HERE, tag + '.ptf')
        torch.save(fix, path)
        print(tag, 'loss', float(fix['loss']),'drop-path blocks', len(fix['drop_scales']), os.path.getsize(path), 'bytes')


if __name__ == '__main__':
    main()
