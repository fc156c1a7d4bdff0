"""Parameter containers with the attribute names (= state_dict keys) of the yolox==0.3.0 blocks the
reference imports (/root/reference/exps/model/darknet.py:7, dfp_pafpn.py:10, tal_head.py:16).
They hold ``nn.Conv2d`` / ``nn.BatchNorm2d`` sub-modules so that ``init_yolo``
(/root/reference/cfgs/s_s50_onex_dfp_tal_flip.py:40-44), the optimizer's parameter grouping, EMA,
DDP and checkpoints see exactly the reference's structure; the arithmetic runs in
libstreamyolo_sm100.so through ``engine``.  Calling a block directly takes / returns NCHW tensors.
"""
import torch
from torch import nn

from . import engine
from ..ops import View


def _run_standalone(module, fn, x):
    v = engine.as_view(x)
    ctx = engine.Ctx(module.training, v.n, v.n, x.device)
    with torch.no_grad(), engine.forward_scope(x.device):
        return engine.as_nchw(fn(ctx, v))


# [yolox] get_activation: the module each ``act`` name builds (and so the module type, repr and state dict of ``self.act``)
ACTIVATIONS = {"silu": lambda: nn.SiLU(inplace=True), "relu": lambda: nn.ReLU(inplace=True),
               "lrelu": lambda: nn.LeakyReLU(0.1, inplace=True)}


class BaseConv(nn.Module):
    """Conv2d(bias=False, pad=(k-1)//2) -> BatchNorm2d -> act, act = "silu" (SiLU), "relu" (ReLU) or "lrelu"
    (LeakyReLU(0.1))."""

    def __init__(self, in_channels, out_channels, ksize, stride, groups=1, bias=False, act="silu"):
        super().__init__()
        if bias or groups not in (1, in_channels) or (groups > 1 and in_channels != out_channels):
            raise NotImplementedError("streamyolo_b200: BaseConv is dense (groups=1) or depthwise (groups=in=out), without bias")
        if act not in ACTIVATIONS:
            raise NotImplementedError(f"activation {act!r}: the kernels implement 'silu', 'relu' and 'lrelu'")
        self.conv = nn.Conv2d(in_channels, out_channels, ksize, stride, (ksize - 1) // 2, groups=groups, bias=False)
        self.bn = nn.BatchNorm2d(out_channels)
        self.act = ACTIVATIONS[act]()
        self.ksize, self.stride, self.act_name = ksize, stride, act

    def forward(self, x):
        return _run_standalone(self, lambda c, v: engine.base_conv(c, self, v), x)

    def fuseforward(self, x):
        return self.forward(x)


class DWConv(nn.Module):
    """[yolox] DWConv: depthwise k x k BaseConv (groups = in_channels) then 1x1 pointwise BaseConv.  Forward only (train-mode
    BatchNorm and eval): the depthwise half runs on sy_dwconv2d (coalesced CUDA-core kernel, HBM-bound), the pointwise half
    on the tensor-core kernel.  Both halves apply ``act`` (silu / relu / lrelu, see BaseConv).  The training backward
    (model/backward.py) does not cover depthwise layers -- no shipped cfg sets depthwise=True."""

    def __init__(self, in_channels, out_channels, ksize, stride=1, act="silu"):
        super().__init__()
        self.dconv = BaseConv(in_channels, in_channels, ksize, stride, groups=in_channels, act=act)
        self.pconv = BaseConv(in_channels, out_channels, 1, 1, groups=1, act=act)

    def forward(self, x):
        return _run_standalone(self, lambda c, v: engine.base_conv(c, self, v), x)


class Bottleneck(nn.Module):
    def __init__(self, in_channels, out_channels, shortcut=True, expansion=0.5, depthwise=False, act="silu"):
        super().__init__()
        hidden = int(out_channels * expansion)
        Conv = DWConv if depthwise else BaseConv
        self.conv1 = BaseConv(in_channels, hidden, 1, 1, act=act)
        self.conv2 = Conv(hidden, out_channels, 3, 1, act=act)
        self.use_add = shortcut and in_channels == out_channels

    def forward(self, x):
        def fn(c, v):
            t = engine.base_conv(c, self.conv1, v)
            return engine.base_conv(c, self.conv2, t, res=v if self.use_add else None)
        return _run_standalone(self, fn, x)


class CSPLayer(nn.Module):
    def __init__(self, in_channels, out_channels, n=1, shortcut=True, expansion=0.5, depthwise=False, act="silu"):
        super().__init__()
        hidden = int(out_channels * expansion)
        self.conv1 = BaseConv(in_channels, hidden, 1, 1, act=act)
        self.conv2 = BaseConv(in_channels, hidden, 1, 1, act=act)
        self.conv3 = BaseConv(2 * hidden, out_channels, 1, 1, act=act)
        self.m = nn.Sequential(*[Bottleneck(hidden, hidden, shortcut, 1.0, depthwise, act=act) for _ in range(n)])

    def forward(self, x):
        return _run_standalone(self, lambda c, v: engine.csp_layer(c, self, v), x)


class Focus(nn.Module):
    """[yolox] Focus: space-to-depth, then a 3x3 BaseConv with activation ``act`` (silu / relu / lrelu)."""

    def __init__(self, in_channels, out_channels, ksize=1, stride=1, act="silu"):
        super().__init__()
        if in_channels != 3 or ksize != 3 or stride != 1:
            raise NotImplementedError("Focus is built for the 3-channel, 3x3 stem of CSPDarknet")
        self.conv = BaseConv(in_channels * 4, out_channels, ksize, stride, act=act)

    def forward(self, x):
        x = x.float().contiguous()
        ctx = engine.Ctx(self.training, x.shape[0], x.shape[0], x.device)
        with torch.no_grad(), engine.forward_scope(x.device):
            return engine.as_nchw(engine.focus_stem(ctx, self, x, 1))


class SPPBottleneck(nn.Module):
    """[yolox] SPPBottleneck: conv1, max pools 5 / 9 / 13, conv2; both BaseConvs apply ``activation`` (silu / relu / lrelu),
    which may differ from the rest of the network's ``act``."""

    def __init__(self, in_channels, out_channels, kernel_sizes=(5, 9, 13), activation="silu"):
        super().__init__()
        if tuple(kernel_sizes) != (5, 9, 13):
            raise NotImplementedError("SPP kernel sizes other than (5, 9, 13)")
        hidden = in_channels // 2
        self.conv1 = BaseConv(in_channels, hidden, 1, 1, act=activation)
        self.m = nn.ModuleList([nn.MaxPool2d(k, 1, k // 2) for k in kernel_sizes])   # parameter-free, for parity of repr
        self.conv2 = BaseConv(hidden * 4, out_channels, 1, 1, act=activation)

    def forward(self, x):
        return _run_standalone(self, lambda c, v: engine.spp_bottleneck(c, self, v), x)
