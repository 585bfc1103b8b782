"""DETR heads with the reference's state_dict layout (SimpleAICV/detection/models/head.py:184-213): class logits and a
3-layer box MLP on every decoder output.  Parameter container; executed by engine.detr._Heads."""
import torch.nn as nn


class DETRClsRegHead(nn.Module):

    def __init__(self, hidden_inplanes, num_classes, num_layers=3):
        super().__init__()
        assert num_layers == 3, 'the H100 runtime implements the 3-layer box head DETR builds'
        self.cls_head = nn.Linear(hidden_inplanes, num_classes)
        reg_layers = []
        for _ in range(num_layers - 1):
            reg_layers.append(nn.Linear(hidden_inplanes, hidden_inplanes))
            reg_layers.append(nn.ReLU(inplace=True))
        reg_layers.append(nn.Linear(hidden_inplanes, 4))
        self.reg_head = nn.Sequential(*reg_layers)
        self.sigmoid = nn.Sigmoid()
        for m in self.parameters():
            if m.dim() > 1:
                nn.init.xavier_uniform_(m)

    def forward(self, x):
        raise RuntimeError('DETRClsRegHead is executed by engine.detr.DetrRT; call the DETR model')
