"""Dry-run the engine with the CUDA ops mocked (CPU, no GPU) to list the per-step kernel sequence with
shapes, algorithmic FLOPs and bytes; optionally join it with an ncu launch list (by launch order)
to get per-layer achieved TFLOP/s / GB/s.

    python tools/op_sequence.py [model] [batch] [launches.csv]
"""
import csv
import os
import re
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

from streamyolo_b200 import ops
from streamyolo_b200.model import DFPPAFPN, TALHead, YOLOX, engine

MODELS = {"s": (0.33, 0.50), "m": (0.67, 0.75), "l": (1.0, 1.0), "tiny": (0.33, 0.125)}
SEQ = []


def record(kind, kernel, name, flops, bytes_, shape):
    SEQ.append(dict(kind=kind, kernel=kernel, name=name, flops=flops, bytes=bytes_, shape=shape))


def install_mocks():
    cur = {"name": "?"}
    orig_base = engine.base_conv

    def conv2d(x, wpk, y, k, s, mode, impl="tc", scale=None, shift=None, act=1, res=None, partials=None, **kw):
        kh, kw_ = (k, k) if isinstance(k, int) else k
        k = f"{kh}x{kw_}"
        fl = 2.0 * y.n * y.h * y.w * y.c * x.c * kh * kw_
        by = 2.0 * (x.n * x.h * x.w * x.c + y.n * y.h * y.w * y.c) + (2.0 * y.n * y.h * y.w * y.c if res is not None else 0)
        record("conv", "conv_tc_kernel", cur["name"], fl, by, f"{x.n}x{x.h}x{x.w} {x.c}->{y.c} k{k}s{s}")
        return 132                  # statistic rows = SMs of an H100 SXM

    def bn_finalize(partials, *a, **k):
        record("finalize", "bn_finalize_kernel", cur["name"], 0, partials.numel() * 4.0, f"P={partials.shape[0]} C={partials.shape[2]}")

    def bn_act_apply(x, sc, sh, split, act, res, y, *a):
        by = 2.0 * x.n * x.h * x.w * x.c * (3 if res is not None else 2)
        record("apply", "bn_act_apply_kernel", cur["name"], 0, by, f"{x.n}x{x.h}x{x.w}x{x.c}")

    def simple(kernel):
        def f(*a, **k):
            v = [t for t in a if isinstance(t, ops.View)]
            by = sum(2.0 * t.n * t.h * t.w * t.c for t in v)
            record("glue", kernel, cur["name"], 0, by, "")
        return f

    def focus_pack(x, frames, y):
        record("glue", "focus_pack_kernel", "stem", 0, x.numel() * 4.0 + 2.0 * y.n * y.h * y.w * y.c, "")

    def head_pred(cf, rf, *a, **k):
        record("glue", "head_pred_kernel", "head.pred", 2.0 * cf.n * cf.h * cf.w * cf.c * 13, 4.0 * cf.n * cf.h * cf.w * cf.c, "")

    def tal_loss(*a, **k):
        for kn in ("k_labels", "k_anchor_prep", "k_pair", "k_dynk", "k_resolve_loss", "k_final"):
            record("loss", kn, "loss", 0, 0, "")

    ops.conv2d, ops.bn_finalize, ops.bn_act_apply = conv2d, bn_finalize, bn_act_apply
    ops.pack_conv_weight = ops.pack_stem_weight = ops.pack_dw_weight = lambda *ws: None    # the mocked conv reads no operand
    ops.upsample_nearest, ops.spp_maxpool, ops.copy = simple("upsample_nearest_kernel"), simple("spp_maxpool_kernel"), simple("copy_kernel")
    ops.focus_pack, ops.head_pred_decode, ops.tal_loss = focus_pack, head_pred, tal_loss
    ops.channel_stats = simple("channel_stats_kernel")
    ops.conv_stat_rows = lambda: 132
    ops.tal_loss_workspace_bytes = lambda *a: 1024

    def named_base(ctx, m, x, y=None, res=None):
        cur["name"] = getattr(m, "_sy_name", "?")
        return orig_base(ctx, m, x, y, res)
    engine.base_conv = named_base
    orig_cba = engine.conv_bn_act

    def named_cba(ctx, mods, *a, **k):
        cur["name"] = "|".join(getattr(m, "_sy_name", "?") for m in mods)
        return orig_cba(ctx, mods, *a, **k)
    engine.conv_bn_act = named_cba
    orig_stem = engine.focus_stem

    def named_stem(ctx, m, x, frames):
        cur["name"] = "backbone.backbone.stem.conv"
        return orig_stem(ctx, m, x, frames)
    engine.focus_stem = named_stem


def sequence(model="l", batch=8, train=True):
    install_mocks()
    d, w = MODELS[model]
    m = YOLOX(DFPPAFPN(d, w), TALHead(8, w))
    m.head.use_l1 = True
    m.train(train)
    engine.name_modules(m)
    x = torch.empty((batch, 6, 600, 960))
    lab = (torch.zeros((batch, 120, 5)), torch.zeros((batch, 120, 5)))
    with torch.no_grad():
        m(x, lab) if train else m(x)
    return SEQ


def load_ncu(path):
    lines = [l for l in open(path) if not l.startswith("==")]
    out = []
    for row in csv.DictReader(lines):
        v = float(row["Metric Value"].replace(",", ""))
        u = row["Metric Unit"]
        v = v / 1e3 if u == "ns" else v * 1e3 if u == "ms" else v * 1e6 if u == "s" else v
        out.append((re.sub(r"\(.*", "", row["Kernel Name"]), v))
    return out


if __name__ == "__main__":
    model = sys.argv[1] if len(sys.argv) > 1 else "l"
    batch = int(sys.argv[2]) if len(sys.argv) > 2 else 8
    seq = sequence(model, batch)
    print(len(seq), "kernels per step")
    if len(sys.argv) > 3:
        ncu = [(n, t) for n, t in load_ncu(sys.argv[3]) if "at::" not in n]
        names = [s["kernel"].split("<")[0] for s in seq]
        off = None
        for o in range(len(ncu) - len(seq) + 1):
            if all(names[i] in ncu[o + i][0] for i in range(len(seq))):
                off = o
                break
        if off is None:
            sys.exit("could not align the launch list with the op sequence")
        agg = {}
        print(f"{'us':>8s} {'TFLOP/s':>8s} {'GB/s':>7s}  kernel / layer / shape")
        for i, s in enumerate(seq):
            t = ncu[off + i][1]
            s["us"] = t
            if s["kind"] == "conv":
                kn = re.sub(r".*conv_tc_kernel", "tc", ncu[off + i][0])
                print(f"{t:8.1f} {s['flops'] / t / 1e6:8.1f} {s['bytes'] / t / 1e3:7.0f}  {kn:8s} {s['name'][-48:]:48s} {s['shape']}")
            a = agg.setdefault(s["kind"], [0.0, 0.0, 0.0])
            a[0] += t; a[1] += s["flops"]; a[2] += s["bytes"]
        for k, (t, f, b) in agg.items():
            print(f"{k:10s} {t / 1e3:8.3f} ms  {f / max(t, 1e-9) / 1e6:8.1f} TFLOP/s  {b / max(t, 1e-9) / 1e3:8.0f} GB/s")
    else:
        for s in seq[:40]:
            print(s)
