"""Layer-by-layer comparison of the CUDA product with the CPU oracle (storage rounding emulated).
usage: python tools/layer_trace.py [depth width H W B impl train|eval]"""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

from oracle.streamyolo_oracle import OracleCfg, StreamYoloOracle, bf16_round, model_shapes
from streamyolo_b200 import synth
from streamyolo_b200.model import DFPPAFPN, TALHead, YOLOX, engine

a = sys.argv[1:]
depth, width = float(a[0]) if a else 0.33, float(a[1]) if len(a) > 1 else 0.125
H, W, B = (int(a[2]), int(a[3]), int(a[4])) if len(a) > 4 else (120, 160, 2)
engine.CONV_IMPL = a[5] if len(a) > 5 else "tc"
train = (a[6] if len(a) > 6 else "train") == "train"
torch.backends.cudnn.allow_tf32 = False
ch = [256, 512, 1024]
m = YOLOX(DFPPAFPN(depth, width, in_channels=ch), TALHead(8, width, in_channels=ch))
for mod in m.modules():
    if isinstance(mod, torch.nn.BatchNorm2d):
        mod.eps, mod.momentum = 1e-3, 0.03
shapes = {k: tuple(v.shape) for k, v in m.state_dict().items()}
m.load_state_dict(synth.synth_state_dict(shapes))
m.head.use_l1 = True
m.cuda().train(train)
engine.name_modules(m)
x = synth.synth_frames(B, H, W)
engine.TRACE = {}
feats = m.backbone(x.cuda())
torch.cuda.synchronize()
tr = dict(engine.TRACE)
o = StreamYoloOracle(OracleCfg(depth=depth, width=width), synth.synth_state_dict(model_shapes(depth, width)), q=bf16_round)
o.training = train
x6 = o.q(x)
o.trace = {}
cur = o.pafpn(x6[:, 0:3])
tc_ = dict(o.trace)
o.trace = {}
sup = o.pafpn(x6[:, 3:6])
ts_ = dict(o.trace)
print(f"{'layer':55s} {'rel(cur)':>10s} {'rel(sup)':>10s}")
worst = 0
for k, v in tr.items():
    ko = k + ".out"
    if ko not in tc_:
        continue
    n = v.shape[0] // 2
    rc = ((v[:n] - tc_[ko]).norm() / tc_[ko].norm()).item()
    rs = ((v[n:] - ts_[ko]).norm() / ts_[ko].norm()).item()
    flag = " <<<" if max(rc, rs) > 3 * max(worst, 1e-3) else ""
    worst = max(worst, rc, rs)
    print(f"{k:55s} {rc:10.2e} {rs:10.2e}{flag}")
fo = o._fuse(cur, sup)
for name, a_, b_ in zip(("jian2", "jian1", "jian0"), feats, fo):
    print("fused", name, ((a_.float().cpu() - b_).norm() / b_.norm()).item())
