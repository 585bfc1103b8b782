"""The drop-in entry points write what the reference's do: the same latest.pth keys and the same best / per-epoch / renamed
checkpoint file names, read from the reference's entry-point sources with ast (skipped when the reference is absent).
The classification entry points keep their checkpoint keys and passing of the epoch bodies."""
import ast
import os

import pytest

from simpleaicv_pytorch_training_examples_b200.tools import (driver, scripts, train_classification_model,
                                                            train_distill_classification_model,
                                                            train_interactive_segmentation_distill_encoder_model,
                                                            train_mae_self_supervised_model)


def _ref_tool(name):
    from baseline import ref_import
    if not ref_import.available():
        pytest.skip('reference not installed (oracle/build_ref.py)')
    return os.path.join(ref_import.root(), 'tools', name)


def _tree(path):
    with open(path) as f:
        return ast.parse(f.read())


def _template(node):
    """A file-name expression as a template: 'best.pth', or an f-string with each field reduced to its format spec."""
    if isinstance(node, ast.Constant) and isinstance(node.value, str):
        return node.value
    if isinstance(node, ast.JoinedStr):
        out = ''
        for v in node.values:
            if isinstance(v, ast.Constant):
                out += v.value
            else:
                spec = ''.join(c.value for c in v.format_spec.values) if v.format_spec is not None else ''
                out += '{' + (':' + spec if spec else '') + '}'
        return out
    return None


def _file_names(path):
    """Every '.pth' name the module spells out, other than latest.pth."""
    nodes = list(ast.walk(_tree(path)))
    parts = {id(v) for n in nodes if isinstance(n, ast.JoinedStr) for v in ast.walk(n) if v is not n}
    names = {_template(n) for n in nodes if id(n) not in parts}
    return {n for n in names if n and n.endswith('.pth') and n != 'latest.pth'}


def _ref_latest_keys(path):
    """Keys of the dict literals the reference saves to latest.pth (the union over its EMA / no-EMA branches)."""
    keys = set()
    for node in ast.walk(_tree(path)):
        if (isinstance(node, ast.Call) and isinstance(node.func, ast.Attribute) and node.func.attr == 'save'
                and len(node.args) == 2 and isinstance(node.args[0], ast.Dict)
                and any(_template(a) == 'latest.pth' for a in ast.walk(node.args[1]))):
            keys |= {k.value for k in node.args[0].keys if isinstance(k, ast.Constant)}
    assert keys, path
    return keys


def _latest_keys(task):
    """The keys run() writes for `task`: the constant keys of its latest.pth dict, the task's state and the EMA model."""
    common = None
    for node in ast.walk(_tree(driver.__file__)):
        if isinstance(node, ast.Dict) and any(isinstance(k, ast.Constant) and k.value == 'epoch' for k in node.keys):
            common = {k.value for k in node.keys if isinstance(k, ast.Constant)}
    return common | set(task.state) | ({'ema_model_state_dict'} if task.keep_ema else set())


@pytest.mark.parametrize('module,task', [
    (train_distill_classification_model, train_distill_classification_model.DistillClassificationTask),
    (train_mae_self_supervised_model, train_mae_self_supervised_model.MAETask),
    (train_interactive_segmentation_distill_encoder_model,
     train_interactive_segmentation_distill_encoder_model.DistillEncoderTask),
])
def test_latest_keys_and_file_names_match_the_reference(module, task):
    ref = _ref_tool(os.path.basename(module.__file__))
    assert _latest_keys(task()) == _ref_latest_keys(ref)
    assert _file_names(module.__file__) == _file_names(ref)


def test_classification_entry_point_keeps_its_keys_and_files():
    task = train_classification_model.ClassificationTask(scripts.train_classification, scripts.test_classification)
    assert _latest_keys(task) == {'epoch', 'time', 'best_acc1', 'test_loss', 'lr', 'model_state_dict', 'optimizer_state_dict',
                                  'scheduler_state_dict', 'ema_model_state_dict'}
    assert _file_names(train_classification_model.__file__) == {'best.pth', '{}-acc{:.3f}.pth'}


def test_tasks_pass_their_epoch_bodies():
    from simpleaicv_pytorch_training_examples_b200.tools import interactive_segmentation_scripts as iss
    kd = train_distill_classification_model.DistillClassificationTask()
    assert (kd.train_fn, kd.test_fn, kd.keep_ema) == (scripts.train_distill_classification,
                                                      scripts.test_distill_classification, False)
    mae = train_mae_self_supervised_model.MAETask()
    assert (mae.train_fn, mae.test_fn, mae.keep_ema) == (scripts.train_mae_self_supervised_learning, None, True)
    enc = train_interactive_segmentation_distill_encoder_model.DistillEncoderTask()
    assert (enc.train_fn, enc.test_fn, enc.keep_ema) == (iss.train_distill_sam_encoder, None, False)


def test_distill_evaluation_runs_teacher_then_student(monkeypatch):
    """test_distill_classification returns test_classification's numbers for the teacher, then for the student, reached
    through a data-parallel wrapper (reference tools/scripts.py:278-288)."""
    import torch.nn as nn
    seen = []

    def fake_test(loader, model, criterion, config):
        seen.append(model)
        return (len(seen) * 10., len(seen) * 20., len(seen) * 0.5)

    monkeypatch.setattr(scripts, 'test_classification', fake_test)

    class KD(nn.Module):
        def __init__(self):
            super().__init__()
            self.teacher, self.student = nn.Linear(2, 2), nn.Linear(2, 2)

    class Wrapper(nn.Module):
        def __init__(self, m):
            super().__init__()
            self.module = m

    kd = KD()
    assert scripts.test_distill_classification(None, Wrapper(kd), None, None) == (10., 20., 0.5, 20., 40., 1.0)
    assert seen == [kd.teacher, kd.student]



def test_entry_points_without_ema_refuse_use_ema_model():
    class Cfg:
        use_ema_model = True

    for task in (train_distill_classification_model.DistillClassificationTask(),
                 train_interactive_segmentation_distill_encoder_model.DistillEncoderTask()):
        with pytest.raises(ValueError, match='use_ema_model = False'):
            task.check(Cfg)
    train_mae_self_supervised_model.MAETask().check(Cfg)
    Cfg.use_ema_model = False
    train_distill_classification_model.DistillClassificationTask().check(Cfg)
