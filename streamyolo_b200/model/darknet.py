"""CSPDarknet container (mirror of /root/reference/exps/model/darknet.py:97-165; the dead
``Darknet``-53 class of :10-94 is not instantiated by any cfg and is not built)."""
import torch
from torch import nn

from . import engine
from .network_blocks import BaseConv, CSPLayer, DWConv, Focus, SPPBottleneck


class CSPDarknet(nn.Module):
    def __init__(self, dep_mul, wid_mul, out_features=("dark3", "dark4", "dark5"), depthwise=False, act="silu"):
        super().__init__()
        assert out_features, "please provide output features of Darknet"
        self.out_features = out_features
        base = int(wid_mul * 64)
        depth = max(round(dep_mul * 3), 1)
        Conv = DWConv if depthwise else BaseConv
        self.stem = Focus(3, base, ksize=3, act=act)
        self.dark2 = nn.Sequential(Conv(base, base * 2, 3, 2, act=act),
                                   CSPLayer(base * 2, base * 2, n=depth, depthwise=depthwise, act=act))
        self.dark3 = nn.Sequential(Conv(base * 2, base * 4, 3, 2, act=act),
                                   CSPLayer(base * 4, base * 4, n=depth * 3, depthwise=depthwise, act=act))
        self.dark4 = nn.Sequential(Conv(base * 4, base * 8, 3, 2, act=act),
                                   CSPLayer(base * 8, base * 8, n=depth * 3, depthwise=depthwise, act=act))
        self.dark5 = nn.Sequential(Conv(base * 8, base * 16, 3, 2, act=act),
                                   SPPBottleneck(base * 16, base * 16, activation=act),
                                   CSPLayer(base * 16, base * 16, n=depth, shortcut=False, depthwise=depthwise, act=act))

    def forward(self, x):
        """Standalone use: NCHW 3-channel float input -> {name: NCHW tensor}."""
        x = x.float().contiguous()
        ctx = engine.Ctx(self.training, x.shape[0], x.shape[0], x.device)
        with torch.no_grad(), engine.forward_scope(x.device):
            outs = engine.darknet(ctx, self, x, 1)
        names = ("stem", "dark2", "dark3", "dark4", "dark5")
        return {k: engine.as_nchw(v) for k, v in zip(names, outs) if k in self.out_features}
