"""Per-layer tiling plan of one training-forward step (no GPU needed): dry-runs the engine with the kernels mocked
(tools/op_sequence.py) and asks the library's host-only planner (sy_conv2d_plan) what sy_conv2d_tc does for each conv:
A-operand mode (linear = im2col-mode TMA / halo), tile width, tiles, rounds of the persistent grid (one CTA per SM).

    python tools/conv_plan.py [model] [pairs]"""
import os
import re
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from streamyolo_b200 import ops

plan = ops.conv2d_plan           # keep the real planner before the dry run mocks the compute entry points
import op_sequence  # noqa: E402

model = sys.argv[1] if len(sys.argv) > 1 else "l"
batch = int(sys.argv[2]) if len(sys.argv) > 2 else 8
seq = [s for s in op_sequence.sequence(model, batch) if s["kind"] == "conv"]
MODE = {1: "linear", 2: "halo"}
print(f"StreamYOLO-{model}, {batch} frame pairs: {len(seq)} conv launches per step")
WALK = {0: "N-major", 1: "M-band"}
print(f"{'layer':50s} {'shape':34s} {'mode':7s} {'BN':>4s} {'tiles':>6s} {'rounds':>6s} {'K blk':>6s} {'fill':>5s} "
      f"{'walk':8s} {'grid':>4s}")
tot, walks = {}, {}
for s in seq:
    m = re.match(r"(\d+)x(\d+)x(\d+) (\d+)->(\d+) k(\d+)x(\d+)s(\d+)", s["shape"])
    n, h, w, ci, co, kh, kw, st = map(int, m.groups())
    p = plan(n, h, w, ci, co, (kh, kw), st)
    tiles = p["m_tiles"] * p["n_tiles"]
    fill = tiles / (p["rounds"] * ops.conv_stat_rows())
    tot[MODE[p["mode"]]] = tot.get(MODE[p["mode"]], 0) + 1
    walks[WALK[p["walk"]]] = walks.get(WALK[p["walk"]], 0) + 1
    print(f"{s['name'][-50:]:50s} {s['shape']:34s} {MODE[p['mode']]:7s} {p['bn']:4d} {tiles:6d} {p['rounds']:6d} {p['kblocks']:6d} {fill:5.2f} "
          f"{WALK[p['walk']]:8s} {p['grid']:4d}")
print("launches per mode:", tot)
print("launches per walk:", walks)
