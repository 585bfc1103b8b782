"""ImageNet-21K semantic-softmax training, host side: the semantic tree's device tables against the live reference dataset
(skipped without oracle/_ref), the float64 oracle against the committed reference fixture, trees the reference cannot
convert, and the 21K epoch body's guard / accumulation / schedule behaviour."""
import importlib.util
import logging
import os

import pytest
import torch

from oracle import semantic_softmax as osem
from simpleaicv_pytorch_training_examples_b200.classification.semantic import SemanticOutputs, SemanticTree

HERE = os.path.dirname(os.path.abspath(__file__))
_spec = importlib.util.spec_from_file_location('mk_semantic', os.path.join(HERE, 'golden', 'make_semantic_softmax_golden.py'))
mk = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(mk)


class _TreeData:
    """The three attributes SemanticTree reads, as the reference dataset computes them (via the oracle)."""

    def __init__(self, tree):
        self.class_tree_list = tree['class_tree_list']
        self.hierarchy_indices_list, self.normalization_factor_list = osem.tree_levels(self.class_tree_list)


def _fixture():
    return torch.load(os.path.join(HERE, 'golden', 'semantic_softmax_c316_b24.pts'), weights_only=False)


@pytest.mark.parametrize('counts,levels', [(mk.LARGE_DEPTH_COUNTS, 11), (mk.SMALL_DEPTH_COUNTS, 6)], ids=['c10450', 'c316'])
def test_tree_tables_match_live_reference(counts, levels):
    from baseline import ref_import
    if not ref_import.available():
        pytest.skip('reference not installed (oracle/build_ref.py)')
    tree = mk.make_tree(counts, seed=0)
    ds = mk.reference_dataset(tree)
    assert len(ds.hierarchy_indices_list) == levels
    mine = SemanticTree(ds)
    oracle_levels, oracle_factors = osem.tree_levels(tree['class_tree_list'])
    for a, b, c in zip(ds.hierarchy_indices_list, mine.hierarchy_indices_list, oracle_levels):
        assert torch.equal(a, b) and torch.equal(a, c)
    assert torch.equal(mine.normalization_factor_list, ds.normalization_factor_list.float())
    torch.testing.assert_close(oracle_factors, ds.normalization_factor_list.double(), rtol=1e-7, atol=0)
    every = torch.arange(len(tree['class_tree_list']))
    ref = ds.convert_single_labels_to_semantic_labels(every)
    got = mine.convert_single_labels_to_semantic_labels(every)
    assert got.dtype == ref.dtype == torch.int64 and torch.equal(got, ref)
    # the tables: every class column in exactly one level, or none at the maximum depth
    t = mine.tables('cpu')
    depth = torch.tensor([len(c) - 1 for c in tree['class_tree_list']])
    assert torch.equal(t.col_level >= 0, depth < len(counts) - 1)
    assert t.level_off.tolist() == [0] + list(torch.tensor(counts[:levels]).cumsum(0).tolist())


def test_oracle_reproduces_reference_fixture():
    fix = _fixture()
    hier, factors = osem.tree_levels(fix['tree']['class_tree_list'])
    assert all(torch.equal(a, b) for a, b in zip(hier, fix['hierarchy_indices_list']))
    torch.testing.assert_close(factors.float(), fix['normalization_factor_list'].float(), rtol=0, atol=0)
    sem = osem.semantic_labels(fix['labels'], hier, fix['tree']['class_tree_list'])
    assert torch.equal(sem, fix['semantic_labels'])
    assert (sem[:4] < 0).any() and (sem[4:8] >= 0).all()           # shallow labels leave deeper levels invalid
    for s in (0.2, 0.):
        loss, grad = osem.loss_and_grad(fix['logits'], sem, hier, fix['normalization_factor_list'].double(), s)
        torch.testing.assert_close(loss.float(), fix[f'loss_s{s}'], rtol=2e-6, atol=0)
        torch.testing.assert_close(grad.float(), fix[f'grad_s{s}'], rtol=1e-5, atol=1e-7)
    counts = osem.accuracy_counts(fix['logits'], sem, hier)
    assert int(counts[:, 1].sum()) == int(fix['meter_valid'])
    assert int(counts[:, 0].sum()) == round(float(fix['meter_result']))
    # the device tables convert the fixture's labels to the reference's semantic labels
    tree = SemanticTree(_TreeData(fix['tree']))
    assert torch.equal(tree.convert_single_labels_to_semantic_labels(fix['labels']), fix['semantic_labels'])


def test_semantic_outputs_keep_the_reference_call_shape():
    fix = _fixture()
    tree = SemanticTree(_TreeData(fix['tree']))
    out = tree.convert_outputs_to_semantic_outputs(fix['logits'])
    assert isinstance(out, SemanticOutputs) and len(out) == len(fix['hierarchy_indices_list'])
    for lv, ix in enumerate(fix['hierarchy_indices_list']):
        assert torch.equal(out[lv], fix['logits'][:, ix])
    assert torch.equal(out[-1], fix['logits'][:, fix['hierarchy_indices_list'][-1]])
    with pytest.raises(IndexError):
        out[len(out)]


def test_loss_and_meter_refuse_plain_lists_and_cpu():
    from simpleaicv_pytorch_training_examples_b200.classification import losses
    from simpleaicv_pytorch_training_examples_b200.classification.common import SemanticSoftmaxMeter
    fix = _fixture()
    tree = SemanticTree(_TreeData(fix['tree']))
    crit = losses.__dict__['SemanticSoftmaxLoss'](fix['normalization_factor_list'], smoothing=0.2)
    slices = [fix['logits'][:, ix] for ix in fix['hierarchy_indices_list']]
    with pytest.raises(TypeError, match='convert_outputs_to_semantic_outputs'):
        crit(slices, fix['semantic_labels'])
    with pytest.raises(TypeError, match='convert_outputs_to_semantic_outputs'):
        SemanticSoftmaxMeter().compute_per_batch(slices, fix['semantic_labels'])
    with pytest.raises(RuntimeError, match='no CPU fallback'):
        crit(tree.convert_outputs_to_semantic_outputs(fix['logits']), fix['semantic_labels'])


def _tree_with_depth_counts(counts):
    tree = mk.make_tree(counts, seed=3)
    return tree, _TreeData(tree)


@pytest.mark.parametrize('counts', [(1, 6, 20, 30), (4, 1, 20, 30, 10)], ids=['single_root', 'single_middle'])
def test_tree_the_reference_cannot_convert_raises(counts):
    tree, data = _tree_with_depth_counts(counts)
    with pytest.raises(ValueError, match='not in level'):
        SemanticTree(data)
    with pytest.raises(LookupError):   # the oracle's restatement of the reference's lookup fails on the same tree
        osem.semantic_labels(torch.arange(len(tree['class_tree_list'])), data.hierarchy_indices_list, tree['class_tree_list'])
    from baseline import ref_import
    if ref_import.available():
        ds = mk.reference_dataset(tree)
        with pytest.raises(RuntimeError):
            ds.convert_single_labels_to_semantic_labels(torch.arange(len(tree['class_tree_list'])))


def test_imagenet21k_epoch_body_guards_accumulation_and_schedule(monkeypatch):
    """train_imagenet21k_classification: the tree of config.train_dataset is built once, NaN batches are skipped without an
    optimizer step, gradients accumulate over `accumulation_steps` micro-batches, the scheduler advances once per
    optimizer step with the reference's epoch fraction, and the returned average is the mean loss.  Host logic only: a
    torch Linear on CPU and a float64 restatement of the criterion stand in for the model and the kernels."""
    from simpleaicv_pytorch_training_examples_b200.tools import scripts, utils as tutils
    monkeypatch.setattr(tutils, 'CudaPrefetcher', lambda loader, **kw: loader)
    tree_data = _TreeData(mk.make_tree(mk.SMALL_DEPTH_COUNTS, seed=0))
    nc = len(tree_data.class_tree_list)
    built = []
    orig_init = SemanticTree.__init__

    def counting_init(self, ds):
        built.append(ds)
        orig_init(self, ds)
    monkeypatch.setattr(SemanticTree, '__init__', counting_init)

    def crit(outputs, labels):
        assert isinstance(outputs, SemanticOutputs) and labels.shape == (outputs.logits.shape[0], len(outputs))
        return osem.loss(outputs.logits, labels, tree_data.hierarchy_indices_list, tree_data.normalization_factor_list, 0.2).float()

    torch.manual_seed(0)
    model, ref = torch.nn.Linear(6, nc), torch.nn.Linear(6, nc)
    ref.load_state_dict(model.state_dict())
    opt, ropt = torch.optim.SGD(model.parameters(), lr=0.1), torch.optim.SGD(ref.parameters(), lr=0.1)
    g = torch.Generator().manual_seed(1)
    batches = [{'image': torch.randn(3, 6, generator=g), 'label': torch.randint(0, nc, (3,), generator=g)} for _ in range(6)]
    batches[2]['image'][0, 0] = float('nan')

    class Loader(list):
        dataset = list(range(18))

    class Cfg:
        accumulation_steps, batch_size, print_interval, local_rank = 2, 3, 1, 0
        train_dataset = tree_data

    class Sched:
        current_lr = 0.1

        def __init__(self):
            self.calls = []

        def step(self, optimizer, epoch):
            self.calls.append(epoch)

    sched = Sched()
    avg = scripts.train_imagenet21k_classification(Loader(batches), model, crit, opt, sched, 3, logging.getLogger('t'), Cfg)
    scripts.train_imagenet21k_classification(Loader(batches[:1]), model, crit, opt, Sched(), 4, logging.getLogger('t'), Cfg)
    assert built == [tree_data]                       # one tree per dataset, reused by the next epoch
    totals, it = [], 1
    for b in batches:
        if not torch.isfinite(b['image']).all():
            ropt.zero_grad()
            continue
        sem = osem.semantic_labels(b['label'], tree_data.hierarchy_indices_list, tree_data.class_tree_list)
        loss = osem.loss(ref(b['image']), sem, tree_data.hierarchy_indices_list, tree_data.normalization_factor_list, 0.2).float() / 2
        loss.backward()
        if it % 2 == 0:
            ropt.step()
            ropt.zero_grad()
            totals.append(float(loss.detach()))
        it += 1
    assert sched.calls == [2 / 6 + 2, 4 / 6 + 2]
    assert abs(avg - 2 * sum(totals) / len(totals)) < 1e-5 * abs(avg)


def test_shared_entry_point_passes_the_epoch_bodies(monkeypatch):
    import inspect
    from simpleaicv_pytorch_training_examples_b200.tools import scripts, train_classification_model, train_imagenet21k_classification_model
    sig = inspect.signature(train_classification_model.main)
    assert sig.parameters['train_fn'].default is scripts.train_classification
    assert sig.parameters['test_fn'].default is scripts.test_classification
    calls = []
    monkeypatch.setattr(train_imagenet21k_classification_model, '_main', lambda tr, te: calls.append((tr, te)))
    train_imagenet21k_classification_model.main()
    assert calls == [(scripts.train_imagenet21k_classification, scripts.test_imagenet21k_classification)]
