"""The same-box LIBRARY bar (SURVEY section 2.1: "whatever cuDNN / ATen picks on the GPU ... is the bar on the same box"):
the reference's network (CSPDarknet + PAFPN on both frames with shared weights, DFP fusion, TALHead towers and prediction
convs -- /root/reference/exps/model/{darknet,dfp_pafpn,tal_head}.py) assembled from the in-repo stand-in of the yolox 0.3.0
blocks (oracle/ref_shim: nn.Conv2d + nn.BatchNorm2d + nn.SiLU), run the way the reference trains on GPUs: CUDA, bf16
autocast, channels_last, cudnn.benchmark, train-mode BatchNorm.  Forward and forward+backward (the loss itself is excluded:
< 1 % of the work, and the reference's loss code synchronises with the host per image).  TEST INFRASTRUCTURE: the product
never imports this; it only says what a stock PyTorch user gets on the same GPU.

    python tests/tools/bench_cudnn.py [s|m|l] [pairs] [steps]"""
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "oracle", "ref_shim"))
import torch
import torch.nn as nn
import torch.nn.functional as F
from yolox.models.network_blocks import BaseConv, CSPLayer, Focus, SPPBottleneck      # oracle/ref_shim stand-in

MODELS = {"s": (0.33, 0.50), "m": (0.67, 0.75), "l": (1.0, 1.0)}
GFLOP = {"s": 61.43, "m": 176.81, "l": 384.30}


class Net(nn.Module):
    """dfp_pafpn.py:109-175 (off_pipe) + tal_head.py:152-199 (towers + prediction convs), train-mode semantics."""

    def __init__(self, depth, width, nc=8):
        super().__init__()
        b = int(width * 64)
        d = max(round(depth * 3), 1)
        n = round(3 * depth)
        c3, c4, c5 = int(256 * width), int(512 * width), int(1024 * width)
        self.stem = Focus(3, b, ksize=3)
        self.dark2 = nn.Sequential(BaseConv(b, b * 2, 3, 2), CSPLayer(b * 2, b * 2, n=d))
        self.dark3 = nn.Sequential(BaseConv(b * 2, b * 4, 3, 2), CSPLayer(b * 4, b * 4, n=d * 3))
        self.dark4 = nn.Sequential(BaseConv(b * 4, b * 8, 3, 2), CSPLayer(b * 8, b * 8, n=d * 3))
        self.dark5 = nn.Sequential(BaseConv(b * 8, b * 16, 3, 2), SPPBottleneck(b * 16, b * 16), CSPLayer(b * 16, b * 16, n=d, shortcut=False))
        self.lateral_conv0 = BaseConv(c5, c4, 1, 1)
        self.C3_p4 = CSPLayer(2 * c4, c4, n, False)
        self.reduce_conv1 = BaseConv(c4, c3, 1, 1)
        self.C3_p3 = CSPLayer(2 * c3, c3, n, False)
        self.bu_conv2 = BaseConv(c3, c3, 3, 2)
        self.C3_n3 = CSPLayer(2 * c3, c4, n, False)
        self.bu_conv1 = BaseConv(c4, c4, 3, 2)
        self.C3_n4 = CSPLayer(2 * c4, c5, n, False)
        self.jian = nn.ModuleList([BaseConv(c3, c3 // 2, 1, 1), BaseConv(c4, c4 // 2, 1, 1), BaseConv(c5, c5 // 2, 1, 1)])
        hw = int(256 * width)
        self.stems = nn.ModuleList([BaseConv(c, hw, 1, 1) for c in (c3, c4, c5)])
        self.cls_convs = nn.ModuleList([nn.Sequential(BaseConv(hw, hw, 3, 1), BaseConv(hw, hw, 3, 1)) for _ in range(3)])
        self.reg_convs = nn.ModuleList([nn.Sequential(BaseConv(hw, hw, 3, 1), BaseConv(hw, hw, 3, 1)) for _ in range(3)])
        self.cls_preds = nn.ModuleList([nn.Conv2d(hw, nc, 1) for _ in range(3)])
        self.reg_preds = nn.ModuleList([nn.Conv2d(hw, 4, 1) for _ in range(3)])
        self.obj_preds = nn.ModuleList([nn.Conv2d(hw, 1, 1) for _ in range(3)])

    def pafpn(self, x):
        x = self.dark2(self.stem(x))
        x2 = self.dark3(x)
        x1 = self.dark4(x2)
        x0 = self.dark5(x1)
        fpn0 = self.lateral_conv0(x0)
        f0 = self.C3_p4(torch.cat([F.interpolate(fpn0, size=x1.shape[2:4], mode="nearest"), x1], 1))
        fpn1 = self.reduce_conv1(f0)
        p2 = self.C3_p3(torch.cat([F.interpolate(fpn1, size=x2.shape[2:4], mode="nearest"), x2], 1))
        p1 = self.C3_n3(torch.cat([self.bu_conv2(p2), fpn1], 1))
        p0 = self.C3_n4(torch.cat([self.bu_conv1(p1), fpn0], 1))
        return p2, p1, p0

    def forward(self, x):
        cur, sup = self.pafpn(x[:, :3]), self.pafpn(x[:, 3:])
        outs = []
        for k, (c, s) in enumerate(zip(cur, sup)):
            f = torch.cat([self.jian[k](c), self.jian[k](s)], 1) + c
            t = self.stems[k](f)
            cf, rf = self.cls_convs[k](t), self.reg_convs[k](t)
            outs.append(torch.cat([self.reg_preds[k](rf), self.obj_preds[k](rf), self.cls_preds[k](cf)], 1).flatten(2))
        return torch.cat(outs, 2)


def main():
    tag = sys.argv[1] if len(sys.argv) > 1 else "l"
    B = int(sys.argv[2]) if len(sys.argv) > 2 else 8
    steps = int(sys.argv[3]) if len(sys.argv) > 3 else 10
    torch.backends.cudnn.benchmark = True
    depth, width = MODELS[tag]
    net = Net(depth, width).cuda().to(memory_format=torch.channels_last).train()
    for m in net.modules():
        if isinstance(m, nn.BatchNorm2d):
            m.eps, m.momentum = 1e-3, 0.03
    x = (torch.rand(B, 6, 600, 960, device="cuda") * 255).contiguous(memory_format=torch.channels_last)

    def fwd():
        with torch.autocast("cuda", dtype=torch.bfloat16):
            return net(x)

    def fwd_bwd():
        for p in net.parameters():
            p.grad = None
        fwd().float().square().mean().backward()

    def timed(fn, grad):
        ctx = torch.enable_grad() if grad else torch.no_grad()
        with ctx:
            for _ in range(4):
                fn()
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(steps):
                fn()
            e1.record()
            torch.cuda.synchronize()
        return e0.elapsed_time(e1) / steps

    f_ms = timed(fwd, False)
    fb_ms = timed(fwd_bwd, True)
    print(json.dumps({"what": "stock PyTorch (cuDNN / ATen), bf16 autocast, channels_last, cudnn.benchmark, train-mode BN, eager",
                      "model": tag, "pairs": B, "forward_ms": round(f_ms, 3), "forward_pairs_per_s": round(B / f_ms * 1e3, 1),
                      "forward_tflops": round(B * GFLOP[tag] / f_ms, 1), "fwd_bwd_ms": round(fb_ms, 3),
                      "fwd_bwd_pairs_per_s": round(B / fb_ms * 1e3, 1), "fwd_bwd_tflops": round(3 * B * GFLOP[tag] / fb_ms, 1),
                      "params": sum(p.numel() for p in net.parameters())}))


if __name__ == "__main__":
    main()
