"""Generates tests/golden/semantic_softmax_c316_b24.pts by running the REFERENCE ImageNet-21K semantic-tree code on a seeded
synthetic tree (316 classes, depths 0..6, so 6 levels):

- the unmodified ImageNet21KSemanticTreeLabelDataset constructor (SimpleAICV/classification/datasets/imagenet21kdataset.py:
  106-253) on a temporary root holding the tree as imagenet21k_miil_tree.pth and empty train/ and val/ directories;
- its convert_single_labels_to_semantic_labels / convert_outputs_to_semantic_outputs;
- SemanticSoftmaxLoss (classification/losses.py:94-140) with autograd, for smoothing 0.2 and 0;
- SemanticSoftmaxMeter.compute_per_batch (classification/common.py:712-757).

The 24 labels include shallow classes (no label at the deeper levels) and classes at the maximum depth (in no level); the
logits are quantised to quarters, so levels have tied maxima.  The file is not a .pt: tests/test_oracle_golden.py loads
every *.pt as a network fixture.

    python tests/golden/make_semantic_softmax_golden.py
"""
import os
import sys
import tempfile

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))

FIXTURE = os.path.join(HERE, 'semantic_softmax_c316_b24.pts')
SMALL_DEPTH_COUNTS = (3, 8, 20, 45, 80, 100, 60)           # classes at depth 0..6 (max depth 6: levels 0..5)
# 10 450 classes, depths 0..11 (11 levels, as the reference's docstring says of the real tree); the per-depth counts of
# the real imagenet21k_miil_tree.pth are not known here, these are assumed
LARGE_DEPTH_COUNTS = (4, 20, 90, 260, 600, 1100, 1700, 2100, 1950, 1400, 800, 426)


def make_tree(depth_counts, seed):
    """A semantic tree in the layout of imagenet21k_miil_tree.pth: class indices are a seeded permutation (so a level's
    classes are not contiguous), each class below depth 0 has a random parent one depth up."""
    g = torch.Generator().manual_seed(seed)
    n = sum(depth_counts)
    perm = torch.randperm(n, generator=g).tolist()
    by_depth, k = [], 0
    for c in depth_counts:
        by_depth.append(perm[k:k + c])
        k += c
    parent = {}
    for d in range(1, len(depth_counts)):
        ups = by_depth[d - 1]
        for c in by_depth[d]:
            parent[c] = ups[int(torch.randint(0, len(ups), (1,), generator=g))]
    class_tree_list = []
    for c in range(n):
        chain = [c]
        while chain[-1] in parent:
            chain.append(parent[chain[-1]])
        class_tree_list.append(chain)
    names = [f'n{c:08d}' for c in range(n)]
    return {'class_list': names,
            'child_2_parent': {names[c]: names[p] for c, p in parent.items()},
            'class_tree_list': class_tree_list,
            'class_description': {nm: f'synthetic class {i}' for i, nm in enumerate(names)}}


def reference_dataset(tree):
    """The reference's ImageNet21KSemanticTreeLabelDataset built on a temporary root holding ``tree``."""
    from baseline import ref_import
    ds_mod = ref_import.module('SimpleAICV.classification.datasets.imagenet21kdataset')
    with tempfile.TemporaryDirectory() as root:
        torch.save(tree, os.path.join(root, 'imagenet21k_miil_tree.pth'))
        for s in ('train', 'val'):
            os.makedirs(os.path.join(root, s))
        return ds_mod.ImageNet21KSemanticTreeLabelDataset(root_dir=root, set_name='train')


def make_inputs(tree, batch=24, seed=1):
    """Labels with shallow classes and maximum-depth classes among them; logits quantised to quarters (tied maxima)."""
    g = torch.Generator().manual_seed(seed)
    depth = torch.tensor([len(c) - 1 for c in tree['class_tree_list']])
    max_depth = int(depth.max())
    shallow = torch.nonzero(depth <= 2).reshape(-1)
    deepest = torch.nonzero(depth == max_depth).reshape(-1)
    labels = torch.randint(0, len(depth), (batch,), generator=g)
    labels[:4] = shallow[torch.randint(0, len(shallow), (4,), generator=g)]
    labels[4:8] = deepest[torch.randint(0, len(deepest), (4,), generator=g)]
    logits = torch.round(torch.randn(batch, len(depth), generator=g) * 8.) / 4.
    return labels, logits


def main():
    from baseline import ref_import
    ref_losses = ref_import.module('SimpleAICV.classification.losses')
    ref_common = ref_import.module('SimpleAICV.classification.common')
    tree = make_tree(SMALL_DEPTH_COUNTS, seed=0)
    ds = reference_dataset(tree)
    labels, logits = make_inputs(tree)
    sem = ds.convert_single_labels_to_semantic_labels(labels)
    out = {'tree': tree, 'hierarchy_indices_list': [ix.clone() for ix in ds.hierarchy_indices_list],
           'normalization_factor_list': ds.normalization_factor_list.clone(), 'labels': labels, 'semantic_labels': sem,
           'logits': logits}
    for s in (0.2, 0.):
        x = logits.clone().requires_grad_(True)
        loss = ref_losses.SemanticSoftmaxLoss(ds.normalization_factor_list, smoothing=s)(ds.convert_outputs_to_semantic_outputs(x), sem)
        loss.backward()
        out[f'loss_s{s}'] = loss.detach()
        out[f'grad_s{s}'] = x.grad.clone()
        print(f'smoothing {s}: loss {float(loss.detach()):.6f}')
    result, valid = ref_common.SemanticSoftmaxMeter().compute_per_batch(ds.convert_outputs_to_semantic_outputs(logits), sem)
    out['meter_result'], out['meter_valid'] = torch.as_tensor(result).float(), torch.as_tensor(valid)
    out['torch_version'] = torch.__version__
    print(f'meter: result {float(result)}, valid {int(valid)}')
    torch.save(out, FIXTURE)


if __name__ == '__main__':
    main()
