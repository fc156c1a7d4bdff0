"""Dissect the conv pipeline: time a shape (CUDA graph of 20 back-to-back launches, so host launch cost is
excluded) as it runs and with the TMA loads switched off (debug flag 2: the barriers still cycle, the MMAs read stale
shared memory).  The gap between the two is what operand supply costs the shape.  The plan column is the A mode
(1 linear, 2 halo) and the tile width.
L2 state: no model runs first, and there is no persisting-L2 set-aside (the library never asks for one).  The graphs are
captured on the step's capture stream.
    usage: python tools/conv_dissect.py"""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from streamyolo_b200 import ops
from streamyolo_b200.model import engine
from streamyolo_b200.ops import View

DEV = torch.device("cuda", 0)

def run(n, ci, co, h, w, k, s, flags, mode=ops.SY_CONV_RAW):
    x = View(torch.randn((n, h, w, ci), device="cuda").to(torch.bfloat16))
    wt = ops.pack_conv_weight(torch.randn((co, ci, k, k), device="cuda") * 0.05)
    ho, wo = ops.conv_out_hw(h, w, k, s)
    y = View.empty(n, ho, wo, co, DEV)
    part = torch.empty((ops.conv_stat_rows(), 4 * co), device="cuda") if mode == ops.SY_CONV_RAW else None
    def go():
        ops.conv2d(x, wt, y, k, s, mode, partials=part, split_n=n // 2, debug_flags=flags)
    go(); torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    st = engine.graph_capture_stream(DEV)
    with torch.cuda.stream(st):
        with torch.cuda.graph(g):
            for _ in range(20):
                go()
        g.replay(); torch.cuda.synchronize()
        best = 1e9
        for _ in range(3):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(); g.replay(); e1.record(); torch.cuda.synchronize()
            best = min(best, e0.elapsed_time(e1) * 1e3 / 20)
    return best

SHAPES = [(8, 256, 256, 75, 120, 3, 1), (16, 128, 128, 75, 120, 3, 1), (16, 64, 64, 150, 240, 3, 1), (16, 256, 256, 38, 60, 3, 1),
          (16, 512, 512, 19, 30, 3, 1), (8, 256, 256, 19, 30, 3, 1), (16, 128, 128, 75, 120, 1, 1), (16, 512, 512, 38, 60, 1, 1),
          (16, 64, 128, 300, 480, 3, 2), (16, 1024, 1024, 19, 30, 1, 1)]
if __name__ == "__main__":
    for shape in SHAPES:
        t = [run(*shape, f) for f in (0, 2)]
        n, ci, co, h, w, k, s = shape
        ho, wo = ops.conv_out_hw(h, w, k, s)
        pl = ops.conv2d_plan(n, h, w, ci, co, k, s)
        fl = 2.0 * n * ho * wo * co * ci * k * k
        by = 2.0 * n * (h * w * ci + ho * wo * co)
        print(f"{str(shape):38s} A{pl['mode']} BN{pl['bn']:<4d} full {t[0]:6.1f} us {fl / t[0] / 1e6:7.0f} TF/s {by / t[0] / 1e3:6.0f} GB/s"
              f" | no-TMA {t[1]:6.1f} us | supply {t[0] - t[1]:6.1f} us ({(t[0] - t[1]) / t[0] * 100:3.0f} %)", flush=True)
