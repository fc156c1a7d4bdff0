"""Pipeline timeline of CTA 0 of the wgmma conv kernel (debug instrumentation) + event timing.
usage: python tools/conv_timeline.py n cin cout h w k s [reps]"""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

from streamyolo_b200 import ops
from streamyolo_b200.ops import View

n, ci, co, h, w = map(int, sys.argv[1:6])
kh, kw = (map(int, sys.argv[6].split("x")) if "x" in sys.argv[6] else (int(sys.argv[6]),) * 2)
s = int(sys.argv[7])
k = (kh, kw)
FLAGS = int(sys.argv[8]) if len(sys.argv) > 8 else 0
x = View(torch.randn((n, h, w, ci), device="cuda").to(torch.bfloat16))
wt = ops.pack_conv_weight(torch.randn((co, ci, kh, kw), device="cuda") * 0.05)
ho, wo = (h + 2 * ((kh - 1) // 2) - kh) // s + 1, (w + 2 * ((kw - 1) // 2) - kw) // s + 1
y = View.empty(n, ho, wo, co, "cuda")
part = torch.empty((ops.conv_stat_rows(), 4 * co), device="cuda")
BN = {}
if os.environ.get("SY_TL_BN"):            # include the BatchNorm tail (grid barrier + finalize) in every launch
    BN = dict(bn=[(torch.ones(co, device="cuda"), torch.zeros(co, device="cuda"), torch.zeros(co, device="cuda"),
                   torch.ones(co, device="cuda"), torch.zeros((), dtype=torch.long, device="cuda"), 0)], momentum=0.03, eps=1e-3,
              scale_shift=torch.empty((2, 2, co), device="cuda"), sync=torch.zeros(4, dtype=torch.int32, device="cuda"))
for _ in range(3):
    ops.conv2d(x, wt, y, k, s, ops.SY_CONV_RAW, partials=part, split_n=n // 2, **BN)
torch.cuda.synchronize()
ts = []
for _ in range(5):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    ops.conv2d(x, wt, y, k, s, ops.SY_CONV_RAW, partials=part, split_n=n // 2, **BN)
    e1.record()
    torch.cuda.synchronize()
    ts.append(e0.elapsed_time(e1) * 1e3)
fl = 2.0 * n * ho * wo * co * ci * kh * kw
print(f"shape {sys.argv[1:8]}: {min(ts):.1f} us best, {fl / min(ts) / 1e6:.0f} TFLOP/s, {(x.buf.numel() + y.buf.numel()) * 2 / min(ts) / 1e3:.0f} GB/s")
cap = 8192
tl = torch.zeros(2 * cap, dtype=torch.int64, device="cuda")
ops.conv2d(x, wt, y, k, s, ops.SY_CONV_RAW, partials=part, split_n=n // 2, timeline=tl, debug_flags=FLAGS, **BN)
torch.cuda.synchronize()
t = tl.view(cap, 2).cpu().numpy()
ev = [(int(c), int(e) >> 28, (int(e) >> 24) & 15, (int(e) >> 8) & 0xffff, int(e) & 255) for e, c in t if c != 0]
ev.sort()
t0 = ev[0][0]
names = {(0, 0): "PA slot-free", (3, 0): "PB slot-free", (0, 1): "PA expect-tx", (3, 1): "PB expect-tx", (0, 2): "PA tma-issued", (3, 2): "PB tma-issued", (1, 0): "M acc-free", (1, 1): "M data-landed", (1, 2): "M issued", (1, 3): "M committed", (4, 0): "K entry", (4, 1): "K setup-done", (4, 2): "K tiles-done", (4, 3): "K all-synced", (4, 4): "K tmem-freed", (4, 5): "K partials-written", (4, 6): "K grid-barrier-passed", (4, 7): "K bn-finalized", (4, 8): "K partial-rows-summed", (4, 9): "K lanes-combined", (2, 0): "E tile-start", (2, 1): "E acc-ready",
         (2, 2): "E converted", (2, 3): "E staged", (2, 4): "E slab-done", (5, 0): "S staged-seen", (5, 1): "S rows-loaded",
         (5, 2): "S reduced", (6, 0): "T staged-seen", (6, 1): "T store-read-done"}
tiles = sorted({e[3] for e in ev})
print("events", len(ev), "tiles of CTA0", len(tiles), "span cycles", ev[-1][0] - t0)
import time
for _ in range(3):
    t_0 = time.perf_counter(); ops.conv2d(x, wt, y, k, s, ops.SY_CONV_RAW, partials=part, split_n=n // 2, **BN); torch.cuda.synchronize(); print("wall us", (time.perf_counter() - t_0) * 1e6)
g = torch.cuda.CUDAGraph()
st = torch.cuda.Stream()
with torch.cuda.stream(st):
    with torch.cuda.graph(g):
        for _ in range(20):
            ops.conv2d(x, wt, y, k, s, ops.SY_CONV_RAW, partials=part, split_n=n // 2, **BN)
    g.replay(); torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(); g.replay(); e1.record(); torch.cuda.synchronize()
    print("graph of 20 back-to-back launches: us per launch", e0.elapsed_time(e1) * 1e3 / 20)
if os.environ.get("SY_TL_TAIL"):          # only the kernel-level events and the last epilogue events
    ev = [e for e in ev if e[1] == 4] + [e for e in ev if e[1] in (2, 5, 6)][-12:]
    ev.sort()
for c, role, ph, tile, kb in ev[:int(os.environ.get('SY_TL_EVENTS', 260))]:
    print(f"{c - t0:9d}  tile {tile:5d} kb {kb:3d}  {names.get((role, ph), (role, ph))}")
