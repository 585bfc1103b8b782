"""Oracle: ImageNet-21K semantic-softmax training tail in float64 on CPU.  TEST INFRASTRUCTURE — see oracle/__init__.py.

Restates, from the reference:
- the level lists and normalisation factors of ImageNet21KSemanticTreeLabelDataset.__init__
  (SimpleAICV/classification/datasets/imagenet21kdataset.py:117-172): depth(c) = len(class_tree_list[c]) - 1, depth i is
  a level when i < max_depth and more than one class has it; factor i = sum(hist) / sum(hist[i:]), clamped to <= 20;
- convert_single_labels_to_semantic_labels (:227-253): the ancestor at depth d sits in column d, looked up in
  hierarchy_indices_list[d];
- SemanticSoftmaxLoss.forward (classification/losses.py:94-140): per level, label-smoothed cross entropy over the level's
  columns masked by (label >= 0), batch mean, weighted by factor[l] (the level's ordinal, not its depth), summed in order;
- SemanticSoftmaxMeter.compute_per_batch (classification/common.py:712-757): per level, first argmax vs the label on valid
  rows; result = sum_l mean_valid(correct) * n_valid.
"""
import torch
import torch.nn.functional as F


def tree_levels(class_tree_list):
    """(hierarchy_indices_list, normalization_factor_list) as imagenet21kdataset.py:117-172 computes them."""
    depth = torch.tensor([len(chain) - 1 for chain in class_tree_list], dtype=torch.int64)
    max_depth = int(depth.max())
    hist = torch.bincount(depth, minlength=max_depth + 1).double()
    levels = [torch.nonzero(depth == i).reshape(-1) for i in range(max_depth) if int(hist[i]) > 1]
    tail = torch.tensor([float(hist[i:].sum()) for i in range(max_depth + 1)], dtype=torch.float64)
    factors = (hist.sum() / tail).clamp(max=20.)
    return levels, factors


def semantic_labels(labels, hierarchy_indices_list, class_tree_list):
    """int64 [B, L]; raises LookupError where the reference's torch.where lookup finds nothing."""
    levels = len(hierarchy_indices_list)
    out = torch.full((len(labels), levels), -1, dtype=torch.int64)
    for i, lab in enumerate(labels.tolist()):
        chain = class_tree_list[int(lab)]
        for j, cls in enumerate(chain):
            d = len(chain) - j - 1
            if levels <= d:
                continue
            hit = torch.nonzero(hierarchy_indices_list[d] == int(cls)).reshape(-1)
            if hit.numel() != 1:
                raise LookupError(f'class {int(cls)} not in level {d}')
            out[i, d] = hit[0]
    return out


def level_losses(logits, sem_labels, hierarchy_indices_list, smoothing):
    """float64 [L]: loss_l = mean_b(v_b * sum_c -((1-s) delta(c, y) + s / n_l) log_softmax(x_b[level l])_c)."""
    x = logits.double()
    out = []
    for lv, index in enumerate(hierarchy_indices_list):
        xl = x[:, index]
        y = sem_labels[:, lv]
        logp = F.log_softmax(xl, dim=1)
        target = torch.zeros_like(xl).scatter_(1, y.clamp(min=0).unsqueeze(1), 1.)
        target = target * (1 - smoothing) + smoothing / xl.shape[1]
        per_row = -(target * logp).sum(dim=1) * (y >= 0).double()
        out.append(per_row.mean())
    return torch.stack(out)


def loss(logits, sem_labels, hierarchy_indices_list, factors, smoothing):
    """float64 scalar: sum_l loss_l * factors[l], summed in level order."""
    per_level = level_losses(logits, sem_labels, hierarchy_indices_list, smoothing)
    total = torch.zeros((), dtype=torch.float64)
    for lv in range(len(hierarchy_indices_list)):
        total = total + per_level[lv] * float(factors[lv])
    return total


def loss_and_grad(logits, sem_labels, hierarchy_indices_list, factors, smoothing):
    """(float64 loss, float64 d loss / d logits [B, N]) by autograd through loss()."""
    x = logits.detach().double().requires_grad_(True)
    value = loss(x, sem_labels, hierarchy_indices_list, factors, smoothing)
    value.backward()
    return value.detach(), x.grad


def accuracy_counts(logits, sem_labels, hierarchy_indices_list):
    """int64 [L, 2]: per level (correct, valid) with torch.argmax's first-maximum / NaN-largest rule."""
    out = torch.zeros(len(hierarchy_indices_list), 2, dtype=torch.int64)
    for lv, index in enumerate(hierarchy_indices_list):
        pred = logits[:, index].argmax(dim=-1)
        y = sem_labels[:, lv]
        valid = y >= 0
        out[lv, 0] = int((pred[valid] == y[valid]).sum())
        out[lv, 1] = int(valid.sum())
    return out
