"""The ImageNet-21K semantic tree on the device: the reference's ImageNet21KSemanticTreeLabelDataset
(SimpleAICV/classification/datasets/imagenet21kdataset.py:106-253) converts every batch on the host, with ``labels.cpu()``
(a device sync) and a Python loop over labels and levels, and gathers ``outputs[:, index]`` once per level.
``SemanticTree`` reads the dataset's tables once and keeps them on the device, so label conversion is one gather and the
loss / accuracy kernels (csrc/capi_loss.cu) read the whole logit row; a step that uses them stays capturable.

The dataset itself (images, transforms, the tree file) stays the reference's: any object with its
``hierarchy_indices_list``, ``class_tree_list`` and ``normalization_factor_list`` attributes will do.
"""
import types

import torch

__all__ = ['SemanticTree', 'SemanticOutputs']

MAX_LEVELS = 16   # kSemMaxLevels of csrc/capi_loss.cu


class SemanticOutputs:
    """What ``convert_outputs_to_semantic_outputs`` returns: the full logits [B, N] and the tree.  ``len()`` and ``[l]``
    behave like the reference's list of ``outputs[:, index_l]`` (a level's slice is gathered only when asked for);
    SemanticSoftmaxLoss and SemanticSoftmaxMeter read the whole row instead."""

    __slots__ = ('logits', 'tree')

    def __init__(self, logits, tree):
        assert logits.dim() == 2 and logits.shape[1] == tree.num_classes, (tuple(logits.shape), tree.num_classes)
        self.logits, self.tree = logits, tree

    def __len__(self):
        return self.tree.num_levels

    def __getitem__(self, level):
        level = range(self.tree.num_levels)[level]
        return self.logits[:, self.tree.tables(self.logits.device).level_index[level]]

    def __iter__(self):
        return (self[i] for i in range(len(self)))


class SemanticTree:
    """Device tables of one semantic tree, built once from a dataset with the reference's attributes:

    - ``col_level`` int32 [N]: the level of each class column, -1 for classes in no level (those at the tree's max depth);
    - ``level_cols`` int32: the concatenated per-level class lists, ``level_off`` int32 [L + 1] their offsets, so level l
      has ``level_off[l+1] - level_off[l]`` classes;
    - ``factors`` fp32 [L]: the first L normalisation factors;
    - ``label_table`` int64 [N, L]: the semantic-label row of each class, exactly what the reference's
      ``convert_single_labels_to_semantic_labels`` produces for it.

    Raises ValueError for a tree the reference cannot convert: the reference looks the ancestor at depth d up in level d's
    class list, so conversion fails when a depth below the deepest kept one has a single class (it is not a level) or a
    chain disagrees with the levels."""

    _cache = {}

    def __init__(self, dataset):
        index_list = [torch.as_tensor(ix).reshape(-1).long().cpu() for ix in dataset.hierarchy_indices_list]
        class_tree_list = dataset.class_tree_list
        factors = torch.as_tensor(dataset.normalization_factor_list).reshape(-1).float().cpu()
        n, levels = len(class_tree_list), len(index_list)
        if not 1 <= levels <= MAX_LEVELS:
            raise ValueError(f'semantic tree with {levels} levels: 1..{MAX_LEVELS} are supported')
        if factors.numel() < levels:
            raise ValueError(f'{factors.numel()} normalisation factors for {levels} levels')
        col_level = torch.full((n,), -1, dtype=torch.int32)
        positions = []
        for lv, ix in enumerate(index_list):
            if ix.numel() == 0 or int(ix.min()) < 0 or int(ix.max()) >= n:
                raise ValueError(f'level {lv} lists classes outside 0..{n - 1}')
            if (col_level[ix] >= 0).any() or ix.unique().numel() != ix.numel():
                raise ValueError(f'level {lv} repeats a class of another level')
            col_level[ix] = lv
            positions.append({int(c): i for i, c in enumerate(ix.tolist())})
        rows = []
        for c in range(n):
            chain = [int(a) for a in class_tree_list[c]]
            row = [-1] * levels
            for j, anc in enumerate(chain):
                depth = len(chain) - j - 1
                if depth >= levels:            # imagenet21kdataset.py:241-243: deeper than the kept levels
                    continue
                pos = positions[depth].get(anc)
                if pos is None:
                    raise ValueError(f'class {c}: its ancestor {anc} at depth {depth} is not in level {depth}; the reference '
                                     'converts labels only when every depth below the deepest level is a level')
                row[depth] = pos
            rows.append(row)
        self.num_classes, self.num_levels = n, levels
        self.hierarchy_indices_list = index_list
        self.normalization_factor_list = factors
        self._host = types.SimpleNamespace(
            col_level=col_level,
            level_cols=torch.cat(index_list).int(),
            level_off=torch.tensor([0] + [int(ix.numel()) for ix in index_list], dtype=torch.int32).cumsum(0, dtype=torch.int32),
            factors=factors[:levels].contiguous(),
            label_table=torch.tensor(rows, dtype=torch.int64).reshape(n, levels),
            level_index=index_list)
        self._device = {}

    @classmethod
    def of(cls, dataset):
        """The tree of ``dataset``, built on first use and cached for the dataset's lifetime in this process."""
        hit = cls._cache.get(id(dataset))
        if hit is None or hit[0] is not dataset:
            hit = cls._cache[id(dataset)] = (dataset, cls(dataset))
        return hit[1]

    def tables(self, device):
        """The tables on ``device`` (copied there once)."""
        device = torch.device(device)
        if device.type == 'cuda' and device.index is None:
            device = torch.device('cuda', torch.cuda.current_device())
        t = self._device.get(device)
        if t is None:
            h = self._host
            t = self._device[device] = types.SimpleNamespace(
                **{k: v.to(device) for k, v in vars(h).items() if k != 'level_index'},
                level_index=[ix.to(device) for ix in h.level_index])
        return t

    def convert_outputs_to_semantic_outputs(self, outputs):
        """imagenet21kdataset.py:215-225, without the per-level gathers: see SemanticOutputs."""
        return SemanticOutputs(outputs, self)

    def convert_single_labels_to_semantic_labels(self, labels):
        """imagenet21kdataset.py:227-253 as one gather on the labels' device (no host sync): [B] -> int64 [B, L], the
        position of each label's ancestor within every level's class list, -1 where the label has none."""
        return self.tables(labels.device).label_table.index_select(0, labels.reshape(-1).long())
