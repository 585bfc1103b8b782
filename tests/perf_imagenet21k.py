"""ImageNet-21K semantic-softmax training step on one GPU: ResNet-50 at 224x224, batch 256, 10 450 classes, the configs'
AdamW (lr 2e-3, wd 1e-4) on the fused optimizer, SemanticSoftmaxLoss(smoothing 0.2) on a synthetic 11-level tree
(tests/golden/make_semantic_softmax_golden.py; the real tree's per-level class counts are assumed).  Prints one JSON
line: ms/step eager and replayed from one CUDA graph, the fused loss tail alone (forward and backward kernels, CUDA
events), and the card's name and power limit, read in the same run.

    python tests/perf_imagenet21k.py [--steps 20] [--warmup 3] [--batch 256] [--torch-ref]

--torch-ref adds the unmodified reference (oracle/_ref, installed by build(); skipped when absent) on the same card:
its ResNet-50 under torch.autocast(bf16), its ImageNet21KSemanticTreeLabelDataset conversion (host loop + sync), its
SemanticSoftmaxLoss and torch.optim.AdamW; and the reference's conversion + loss tail alone.
"""
import argparse
import importlib.util
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from perf_convformer import card, timed  # noqa: E402

_spec = importlib.util.spec_from_file_location('mk_semantic', os.path.join(ROOT, 'tests', 'golden', 'make_semantic_softmax_golden.py'))
mk = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(mk)
ADAMW = ('AdamW', {'lr': 2e-3, 'global_weight_decay': False, 'weight_decay': 1e-4, 'no_weight_decay_layer_name_list': []})


class _TreeData:
    """The attributes of the reference dataset the tree is built from (restated by oracle/semantic_softmax.py)."""

    def __init__(self, class_tree_list):
        from oracle import semantic_softmax as osem
        self.class_tree_list = class_tree_list
        self.hierarchy_indices_list, self.normalization_factor_list = osem.tree_levels(class_tree_list)


def batch(B, nc):
    g = torch.Generator().manual_seed(1234)
    return torch.randn(B, 3, 224, 224, generator=g).cuda(), torch.randint(0, nc, (B,), generator=g).cuda()


def measure_runtime(args, data, x, y):
    from simpleaicv_pytorch_training_examples_b200 import _lib, ops
    from simpleaicv_pytorch_training_examples_b200.classification import backbones, losses
    from simpleaicv_pytorch_training_examples_b200.classification.semantic import SemanticTree
    from simpleaicv_pytorch_training_examples_b200.graph import GraphedTrainStep
    from simpleaicv_pytorch_training_examples_b200.tools import utils as tutils

    class Cfg:
        optimizer = ADAMW

    tree = SemanticTree(data)
    nc = tree.num_classes
    torch.manual_seed(0)
    model = backbones.resnet50(num_classes=nc).cuda().train()
    opt = tutils.build_optimizer(Cfg, model)[0]
    sem_loss = losses.SemanticSoftmaxLoss(data.normalization_factor_list, smoothing=0.2).cuda()

    def crit(logits, labels):
        return sem_loss(tree.convert_outputs_to_semantic_outputs(logits), tree.convert_single_labels_to_semantic_labels(labels))

    def step():
        loss = crit(model(x), y)
        loss.backward()
        opt.step()
        opt.zero_grad()
        return loss

    for _ in range(max(3, args.warmup)):
        step()
    l0 = _lib.launch_count()
    eager_ms = timed(step, args.steps)
    launches = (_lib.launch_count() - l0) / args.steps
    graphed = GraphedTrainStep(model, crit, opt, x, y)
    graphed.replay()
    graph_ms = timed(graphed.replay, args.steps)
    rec = {'eager_ms_per_step': eager_ms, 'graphed_ms_per_step': graph_ms, 'images_per_s_graphed': args.batch / graph_ms * 1e3,
           'launches_per_step': launches, 'last_loss': float(graphed.static_loss), 'peak_mem_gb': torch.cuda.max_memory_allocated() / 2 ** 30}
    del graphed, model, opt
    torch.cuda.empty_cache()
    # the loss tail alone, on fp32 logits [B, N]: conversion + fused forward, fused backward
    t = tree.tables('cuda')
    logits = torch.randn(args.batch, nc, device='cuda')
    one = torch.ones((), device='cuda')
    sem = tree.convert_single_labels_to_semantic_labels(y)
    state = {}

    def fwd():
        state['lse'] = ops.semantic_softmax_fwd(logits, tree.convert_single_labels_to_semantic_labels(y), t.level_cols, t.level_off,
                                                t.factors, 0.2)[1]

    def bwd():
        ops.semantic_softmax_bwd(logits, sem, t.col_level, t.level_cols, t.level_off, t.factors, state['lse'], one, 0.2)

    for _ in range(10):
        fwd()
        bwd()
    reps = 200
    rec['loss_tail_fwd_us'] = timed(fwd, reps) * 1e3
    rec['loss_tail_bwd_us'] = timed(bwd, reps) * 1e3
    rec['loss_tail_bytes'] = {'fwd_logits_read': args.batch * nc * 4, 'bwd_logits_read_plus_grad_write': args.batch * nc * 8}
    return rec


def measure_reference(args, tree_dict, x, y):
    from baseline import ref_import
    if not ref_import.available():
        return 'skipped: reference not installed (oracle/_ref)'
    ref_losses = ref_import.module('SimpleAICV.classification.losses')
    ds = mk.reference_dataset(tree_dict)
    nc = len(tree_dict['class_tree_list'])
    torch.manual_seed(0)
    model = ref_import.backbones().resnet50(num_classes=nc).cuda().train()
    crit = ref_losses.SemanticSoftmaxLoss(ds.normalization_factor_list, smoothing=0.2)
    opt = torch.optim.AdamW(model.parameters(), lr=2e-3, weight_decay=1e-4)

    def step():
        with torch.autocast('cuda', dtype=torch.bfloat16):
            outputs = model(x)
            loss = crit(ds.convert_outputs_to_semantic_outputs(outputs), ds.convert_single_labels_to_semantic_labels(y))
        loss.backward()
        opt.step()
        opt.zero_grad()

    for _ in range(max(3, args.warmup)):
        step()
    ms = timed(step, args.steps)
    logits = torch.randn(args.batch, nc, device='cuda', requires_grad=True)

    def tail():
        loss = crit(ds.convert_outputs_to_semantic_outputs(logits), ds.convert_single_labels_to_semantic_labels(y))
        loss.backward()

    for _ in range(3):
        tail()
    tail_ms = timed(tail, 10)
    return {'ms_per_step': ms, 'images_per_s': args.batch / ms * 1e3, 'loss_tail_fwd_bwd_ms': tail_ms,
            'mode': 'eager torch, autocast(bf16), reference label conversion + SemanticSoftmaxLoss, torch.optim.AdamW'}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=20)
    ap.add_argument('--warmup', type=int, default=3)
    ap.add_argument('--batch', type=int, default=256)
    ap.add_argument('--torch-ref', action='store_true')
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('perf_imagenet21k.py needs a CUDA device')
    tree = mk.make_tree(mk.LARGE_DEPTH_COUNTS, seed=0)
    data = _TreeData(tree['class_tree_list'])
    x, y = batch(args.batch, len(tree['class_tree_list']))
    line = {'workload': f'resnet50 224x224 bs{args.batch}, 10450 classes, SemanticSoftmaxLoss(0.2) on a synthetic 11-level tree, AdamW',
            'card': card(), 'timed_steps': args.steps, 'runtime': measure_runtime(args, data, x, y)}
    if args.torch_ref:
        line['torch_reference'] = measure_reference(args, tree, x, y)
    print(json.dumps(line), flush=True)


if __name__ == '__main__':
    main()
