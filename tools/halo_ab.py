"""Time 3x3 stride-1 conv shapes with linear tiles (nine im2col loads per channel block) against halo mode (one halo
load per channel block): CUDA graph of 20 back-to-back launches over rotating buffers.  usage: python tools/halo_ab.py"""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

from streamyolo_b200 import ops
from streamyolo_b200.ops import View

SHAPES = [(16, 128, 128, 75, 120), (8, 256, 256, 75, 120), (16, 64, 64, 150, 240), (16, 256, 256, 38, 60),
          (16, 512, 512, 19, 30), (8, 256, 256, 38, 60), (8, 256, 256, 19, 30)]


def run(n, ci, co, h, w, tile_mode, sets=4):
    xs = [View(torch.randn((n, h, w, ci), device="cuda").to(torch.bfloat16)) for _ in range(sets)]
    ys = [View.empty(n, h, w, co, "cuda") for _ in range(sets)]
    wt = ops.pack_conv_weight(torch.randn((co, ci, 3, 3), device="cuda") * 0.05)
    part = torch.empty((ops.conv_stat_rows(), 4 * co), device="cuda")

    def go(i):
        ops.conv2d(xs[i % sets], wt, ys[i % sets], 3, 1, ops.SY_CONV_RAW, partials=part, split_n=n // 2, tile_mode=tile_mode)
    go(0)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    st = torch.cuda.Stream()
    with torch.cuda.stream(st):
        with torch.cuda.graph(g):
            for i in range(20):
                go(i)
        g.replay()
        torch.cuda.synchronize()
        best = 1e9
        for _ in range(3):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(); g.replay(); e1.record(); torch.cuda.synchronize()
            best = min(best, e0.elapsed_time(e1) * 1e3 / 20)
    return best, ys[0].torch().float()


for shape in SHAPES:
    t_lin, y_lin = run(*shape, tile_mode=1)
    t_halo, y_halo = run(*shape, tile_mode=2)
    n, ci, co, h, w = shape
    fl = 2.0 * n * h * w * co * ci * 9
    print(f"{str(shape):28s} linear {t_lin:6.1f} us {fl / t_lin / 1e6:6.0f} TF/s | halo {t_halo:6.1f} us {fl / t_halo / 1e6:6.0f} TF/s | x{t_lin / t_halo:.2f}", flush=True)
