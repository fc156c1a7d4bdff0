"""Per-layer time INSIDE a CUDA graph (what the step really pays), for every distinct BaseConv launch of the benchmark
workload: the train-mode conv (wgmma kernel with statistics + BatchNorm finalize) and its normalise pass, each replayed
R times back to back in one graph (PDL edges like the real step), next to the layer's roofline time
max(FLOPs / tensor peak, algorithmic bytes / HBM peak).  The sum over the step's launches is compared with bench.py.

L2 state: the same as bench.py's step.  The model's forward runs first, there is no persisting-L2 set-aside (the library
never asks for one), and the graphs are captured on engine.graph_capture_stream like the step's.

    python tools/layer_graph_bench.py [model] [pairs] [reps]"""
import collections
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

import bench
from streamyolo_b200 import ops, synth
from streamyolo_b200.model import engine
from streamyolo_b200.ops import View

tag = sys.argv[1] if len(sys.argv) > 1 else "l"
B = int(sys.argv[2]) if len(sys.argv) > 2 else 8
R = int(sys.argv[3]) if len(sys.argv) > 3 else 20
dev = torch.device("cuda", 0)
torch.cuda.set_device(dev)
peaks = bench.load_peaks()
model = bench.build_model(tag, dev)
engine.name_modules(model)
x = synth.synth_frames(B, 600, 960, seed=1234).to(dev)
fut, cur = synth.synth_labels(B, 600, 960, seed=1)
calls = []
orig = engine.conv_bn_act


def spy(ctx, mods, xv, wpk, k, s, y, res=None, act=1, y_goff1=0, res_goff1=0, **kw):
    kh, kw_ = (k, k) if isinstance(k, int) else k
    calls.append(dict(name="|".join(getattr(m, "_sy_name", "?") for m in mods), n=xv.n, h=xv.h, w=xv.w, cin=xv.c,
                      cout=sum(m.conv.out_channels for m in mods), k=(kh, kw_), s=s, res=res is not None, split=ctx.split if ctx.groups == 2 else 0,
                      mods=mods, wpk=wpk, goff=y_goff1 != 0))
    return orig(ctx, mods, xv, wpk, k, s, y, res, act, y_goff1, res_goff1, **kw)


engine.conv_bn_act = spy
with torch.no_grad():
    model(x, (fut.to(dev), cur.to(dev)))
torch.cuda.synchronize()
engine.conv_bn_act = orig


def timed_graph(fn, reps):
    fn()
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    st = engine.graph_capture_stream(dev)
    with torch.cuda.stream(st):
        with torch.cuda.graph(g):
            for _ in range(reps):
                fn()
        g.replay()
        torch.cuda.synchronize()
        best = 1e9
        for _ in range(3):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(st)
            g.replay()
            e1.record(st)
            torch.cuda.synchronize()
            best = min(best, e0.elapsed_time(e1) * 1e3 / reps)
    return best


groups = collections.OrderedDict()
for c in calls:
    key = (c["n"], c["h"], c["w"], c["cin"], c["cout"], c["k"], c["s"], c["res"], c["split"], len(c["mods"]))
    groups.setdefault(key, []).append(c)

print(f"StreamYOLO-{tag}, {B} pairs: {len(calls)} BaseConv launches, {len(groups)} distinct; in-graph us per launch ({R} reps back to back)")
print(f"{'shape':44s} {'x':>3s} {'conv':>8s} {'apply':>8s} {'both':>8s} {'roof':>7s} {'TF/s':>7s} {'GB/s':>6s}  first layer")
tot = dict(conv=0.0, apply=0.0, both=0.0, roof=0.0)
for key, cs in groups.items():
    c = cs[0]
    n, h, w, cin, cout, (kh, kw), s = c["n"], c["h"], c["w"], c["cin"], c["cout"], c["k"], c["s"]
    ho, wo = (h + 2 * ((kh - 1) // 2) - kh) // s + 1, (w + 2 * ((kw - 1) // 2) - kw) // s + 1
    xin = View(torch.randn((n, h, w, cin), device=dev).to(torch.bfloat16))
    raw, y = View.empty(n, ho, wo, cout, dev), View.empty(n, ho, wo, cout, dev)
    resv = View(torch.randn((n, ho, wo, cout), device=dev).to(torch.bfloat16)) if c["res"] else None
    mods, wpk = c["mods"], c["wpk"]
    partials = torch.empty((ops.conv_stat_rows(), 4 * cout), dtype=torch.float32, device=dev)
    ss = torch.empty((2, 2, cout), dtype=torch.float32, device=dev)
    segs, c0 = [], 0
    for m in mods:
        segs.append(engine._bn_seg(m, c0))
        c0 += m.conv.out_channels
    split = c["split"]
    sync = engine._sync(mods[0], dev)

    def conv():
        ops.conv2d(xin, wpk, raw, (kh, kw), s, ops.SY_CONV_RAW, impl="tc", partials=partials, split_n=split, bn=segs, momentum=0.03,
                   eps=1e-3, scale_shift=ss, sync=sync)

    def apply():
        ops.bn_act_apply(raw, ss[0].data_ptr(), ss[1].data_ptr(), split if split else n, 1, resv, y)

    def both():
        conv()
        apply()

    tc, ta, tb = timed_graph(conv, R), timed_graph(apply, R), timed_graph(both, R)
    flops = 2.0 * n * ho * wo * cout * cin * kh * kw
    byts = 2.0 * (n * h * w * cin + n * ho * wo * cout * (2 if c["res"] else 1))
    roof = max(flops / (peaks["sustained"] * 1e12), byts / (peaks["hbm"] * 1e9)) * 1e6
    mult = len(cs)
    for k_, v in (("conv", tc), ("apply", ta), ("both", tb), ("roof", roof)):
        tot[k_] += v * mult
    shape = f"{n}x{h}x{w} {cin}->{cout} k{kh}x{kw}s{s}" + (" +res" if c["res"] else "")
    print(f"{shape:44s} {mult:3d} {tc:8.1f} {ta:8.1f} {tb:8.1f} {roof:7.1f} {flops / tc / 1e6:7.0f} {byts / tb / 1e3:6.0f}  {c['name'][-40:]}", flush=True)
print(f"sum over the step's launches: conv {tot['conv'] / 1e3:.3f} ms, apply {tot['apply'] / 1e3:.3f} ms, conv+apply chained "
      f"{tot['both'] / 1e3:.3f} ms, roofline {tot['roof'] / 1e3:.3f} ms")
