"""Drop-in replacement for the reference `model.refinenet` module (model/refinenet.py): `RefineNet()` with the same
state-dict keys (block.layer{1..4}.{0,1}.*, block.layer5.*), `.to()`, `.eval()`, `.load_state_dict()` and
`refine_model(inp)` for inp fp32 [n,75] on a CUDA device -> fp32 [n,45] (exps/stage3_root2/test_util.py:115-116),
computed by libsmap_b200.so (smapb_refine_mlp).  Inference only.
"""
import torch
import torch.nn as nn

from smap_b200.engine import Engine

_DIMS = (75, 160, 256, 256, 128, 45)


class RefineNet_base(nn.Module):
    def __init__(self, in_dim=75, out_dim=45, flatten_size=1):
        super().__init__()
        if (in_dim, out_dim, flatten_size) != (75, 45, 1):
            raise NotImplementedError("smap_b200 implements the 75 -> 45 RefineNet of the stage3_root2 pipeline")
        for i in range(4):  # parameter holders only: Linear + BatchNorm1d (+ ReLU, which owns no state)
            setattr(self, "layer%d" % (i + 1), nn.Sequential(nn.Linear(_DIMS[i], _DIMS[i + 1]), nn.BatchNorm1d(_DIMS[i + 1]), nn.ReLU()))
        self.layer5 = nn.Linear(_DIMS[4], _DIMS[5])
        self.out_dim = out_dim


class RefineNet(nn.Module):
    def __init__(self):
        super().__init__()
        self.block = RefineNet_base()
        self._engines = {}
        self._synced = {}

    def _weights_version(self):
        return tuple(p._version for p in self.parameters()) + tuple(b._version for b in self.buffers())

    def forward(self, input_x):
        if self.training:
            raise NotImplementedError("smap_b200.RefineNet is inference only: call .eval()")
        if not input_x.is_cuda:
            raise RuntimeError("smap_b200.RefineNet runs on an H100 only: move the model and the input to 'cuda'")
        dev = input_x.device.index
        eng = self._engines.get(dev)
        if eng is None:
            eng = self._engines[dev] = Engine(dev, max_batch=1, in_h=64, in_w=64)
        ver = self._weights_version()
        if self._synced.get(dev) != ver:
            eng.load_refine_state_dict(self.state_dict())
            self._synced[dev] = ver
        with torch.cuda.device(input_x.device):
            return eng.refine_mlp(input_x.float())
