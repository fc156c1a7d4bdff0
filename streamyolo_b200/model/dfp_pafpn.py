"""DFPPAFPN: PAFPN + Dual-Flow Perception (mirror of /root/reference/exps/model/dfp_pafpn.py).

Same constructor, sub-module names and forward(input, buffer, mode) contract; outputs are
NCHW-shaped bf16 tensors (channels-last memory, i.e. zero-copy views of the NHWC buffers the
kernels write).  ``activation_dtype = torch.float16`` (eval only): every activation, the outputs and the on_pipe
buffers are fp16 instead."""
import torch
from torch import nn

from . import engine
from .darknet import CSPDarknet
from .network_blocks import BaseConv, CSPLayer, DWConv


class DFPPAFPN(nn.Module):
    def __init__(self, depth=1.0, width=1.0, in_features=("dark3", "dark4", "dark5"),
                 in_channels=[256, 512, 1024], depthwise=False, act="silu"):
        super().__init__()
        if tuple(in_features) != ("dark3", "dark4", "dark5"):
            raise NotImplementedError("in_features other than (dark3, dark4, dark5)")
        self.backbone = CSPDarknet(depth, width, depthwise=depthwise, act=act)
        self.in_features = in_features
        self.in_channels = in_channels
        c3, c4, c5 = (int(c * width) for c in in_channels)
        Conv = DWConv if depthwise else BaseConv            # dfp_pafpn.py:31
        n = round(3 * depth)
        self.lateral_conv0 = BaseConv(c5, c4, 1, 1, act=act)
        self.C3_p4 = CSPLayer(2 * c4, c4, n, False, depthwise=depthwise, act=act)
        self.reduce_conv1 = BaseConv(c4, c3, 1, 1, act=act)
        self.C3_p3 = CSPLayer(2 * c3, c3, n, False, depthwise=depthwise, act=act)
        self.bu_conv2 = Conv(c3, c3, 3, 2, act=act)
        self.C3_n3 = CSPLayer(2 * c3, c4, n, False, depthwise=depthwise, act=act)
        self.bu_conv1 = Conv(c4, c4, 3, 2, act=act)
        self.C3_n4 = CSPLayer(2 * c4, c5, n, False, depthwise=depthwise, act=act)
        self.jian2 = Conv(c3, c3 // 2, 1, 1, act=act)
        self.jian1 = Conv(c4, c4 // 2, 1, 1, act=act)
        self.jian0 = Conv(c5, c5 // 2, 1, 1, act=act)
        self.activation_dtype = torch.bfloat16      # activation storage: bf16, or fp16 in eval mode (engine.Ctx)

    # ---- reference: off_forward (:109-175)
    def off_forward(self, input):
        x = input.float().contiguous()
        b = x.shape[0]
        ctx = engine.Ctx(self.training, 2 * b, b, x.device, dtype=self.activation_dtype)
        with torch.no_grad(), engine.forward_scope(x.device):
            pans = engine.pafpn_frames(ctx, self, x, 2)
            cur = tuple(p.imgs(0, b) for p in pans)
            sup = tuple(p.imgs(b, b) for p in pans)
            fused = engine.dfp_fuse(ctx, self, cur, sup)
        return tuple(engine.as_nchw(v) for v in fused)

    # ---- reference: online_forward (:177-228)
    def online_forward(self, input, buffer=None, node="star"):
        x = input.float().contiguous()
        b = x.shape[0]
        ctx = engine.Ctx(self.training, b, b, x.device, dtype=self.activation_dtype)
        with torch.no_grad(), engine.forward_scope(x.device):
            cur = engine.pafpn_frames(ctx, self, x, 1)
            if node == "star":
                sup = cur
            elif ctx.f16:
                sup = tuple(engine.as_view(t, torch.float16) for t in buffer)
            else:
                sup = tuple(engine.as_view(t) for t in buffer)
            fused = engine.dfp_fuse(ctx, self, cur, sup)
        return tuple(engine.as_nchw(v) for v in fused), tuple(engine.as_nchw(v) for v in cur)

    def forward(self, input, buffer=None, mode="off_pipe"):
        if mode == "off_pipe":
            if input.size()[1] == 3:
                input = torch.cat([input, input], dim=1)
            elif input.size()[1] != 6:
                raise ValueError("off_pipe expects 3 or 6 input channels")
            return self.off_forward(input)
        elif mode == "on_pipe":
            if buffer is None:
                return self.online_forward(input, node="star")
            assert len(buffer) == 3
            assert input.size()[1] == 3
            return self.online_forward(input, buffer=buffer, node="buffer")
        raise ValueError(mode)
