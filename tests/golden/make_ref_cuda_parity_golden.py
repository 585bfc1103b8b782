"""Writes tests/golden/ref_cuda_bs256_<arch>.ptc: what the unmodified reference computes on a GPU at the benchmarked shape
(batch 256, 224x224), under torch.autocast(bf16) - what its tools/scripts.py training loop does - and in fp32, on the
seeded weights and batch of tests/test_reference_cuda_parity_gpu.py.  Needs a CUDA device and the reference importable
through baseline/ref_import.py; run from the repository root:

    python tests/golden/make_ref_cuda_parity_golden.py [OUT_DIR]

Stored (each file well under 1 MB): sha256 of every initial state_dict tensor, loss (bf16 / fp32 runs), the logits of a
seeded sample of rows, the whole-tensor max |logit| and max |bf16 - fp32| logit difference, a seeded sample of every BN
running statistic, and for every parameter gradient: its relative L2 bf16-vs-fp32 noise, its norms, and a seeded sample
of both gradients scaled by the bf16 gradient's norm (fp16).
"""
import hashlib
import importlib.util
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from baseline import ref_import  # noqa: E402

_spec = importlib.util.spec_from_file_location('parity', os.path.join(ROOT, 'tests', 'test_reference_cuda_parity_gpu.py'))
parity = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(parity)


def sha(t):
    return hashlib.sha256(t.detach().cpu().contiguous().numpy().tobytes()).hexdigest()


def run(model, crit, x, y, autocast):
    model.zero_grad(set_to_none=True)
    with torch.autocast('cuda', dtype=torch.bfloat16, enabled=autocast):
        out = model(x)
        loss = crit(out, y)
    loss.backward()
    torch.cuda.synchronize()
    return out.detach().float(), loss.detach().float(), {n: p.grad.detach().float().clone() for n, p in model.named_parameters()
                                                         if p.grad is not None}


def main(out_dir):
    for arch, kw, loss_name, batch in parity.CASES:
        x, y = parity.batch_for(loss_name, batch)
        x, y = x.cuda(), y.cuda()
        torch.manual_seed(0)
        ref = ref_import.backbones().__dict__[arch](num_classes=1000, **kw).cuda().train()
        init_sha = {k: sha(v) for k, v in ref.state_dict().items()}
        sd0 = {k: v.clone() for k, v in ref.state_dict().items()}
        crit = ref_import.module('SimpleAICV.classification.losses').__dict__[loss_name]().cuda()
        lo32, ls32, g32 = run(ref, crit, x, y, autocast=False)
        ref.load_state_dict(sd0)                                   # undo the BN running-stat update
        lo16, ls16, g16 = run(ref, crit, x, y, autocast=True)
        rows = parity.logit_rows(batch)
        stats = {}
        for i, (k, v) in enumerate((k, v) for k, v in ref.state_dict().items() if 'running_' in k):
            idx = parity.sample_index(v.numel(), parity.N_STAT_SAMPLES, i)
            stats[k] = {'values': v.reshape(-1).float().cpu()[idx], 'absmax': v.abs().max().item()}
        grads = {}
        for i, n in enumerate(g16):
            a, b = g16[n].reshape(-1), g32[n].reshape(-1)
            norm16 = a.double().norm().item()
            idx = parity.sample_index(a.numel(), parity.N_GRAD_SAMPLES, i).cuda()
            grads[n] = {'noise': parity._rel(g16[n], g32[n]), 'norm16': norm16, 'norm32': b.double().norm().item(),
                        'g16': (a[idx] / max(norm16, 1e-30)).half().cpu(), 'g32': (b[idx] / max(norm16, 1e-30)).half().cpu()}
        gold = {'arch': arch, 'init_sha': init_sha, 'loss16': ls16.item(), 'loss32': ls32.item(),
                'logit_rows': rows, 'logits16': lo16[rows].cpu(), 'logits32': lo32[rows].cpu(),
                'logit_absmax16': lo16.abs().max().item(), 'logit_noise': (lo16 - lo32).abs().max().item(),
                'bn_stats': stats, 'grads': grads,
                'device': torch.cuda.get_device_name(), 'torch': torch.__version__}
        path = os.path.join(out_dir, f'ref_cuda_bs256_{arch}.ptc')
        torch.save(gold, path)
        print(path, os.path.getsize(path), 'bytes', f'loss16 {ls16.item():.6f} loss32 {ls32.item():.6f}')
        del ref
        torch.cuda.empty_cache()


if __name__ == '__main__':
    main(sys.argv[1] if len(sys.argv) > 1 else os.path.join(ROOT, 'tests', 'golden'))
