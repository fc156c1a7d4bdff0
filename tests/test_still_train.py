"""CPU: training the still-image baseline, YOLOX(DFPPAFPN, PIPEHead) on single frames (cfgs/l_s50_still_dfp_flip.py), with
every kernel replaced by its torch emulation (tests/emul_ops.py, with the repeated running-statistics update added by
``install`` below).

The reference duplicates each frame into a pair (dfp_pafpn.py:236-238) and so runs the backbone + PAFPN twice on the same
batch; the product runs it once with each BatchNorm's running update applied twice (model/backward.py ``_record``).  The
oracle here is the reference's arithmetic itself: autograd through the fp32 oracle on ``(cat(x, x), (labels, labels))`` with
gamma = 0 (PIPEHead = TALHead without the trend weights), which tests/test_oracle_golden.py pins to the reference's
``loss.backward()``.  Also the host-side argument checks of the two C entry points this feature adds."""
import ctypes as C
import os
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import emul_ops  # noqa: E402
import test_cpu_backward as T  # noqa: E402
from oracle.make_golden import CASES  # noqa: E402
from oracle.streamyolo_oracle import OracleCfg, StreamYoloOracle, model_shapes  # noqa: E402
from streamyolo_b200 import ops, synth, train  # noqa: E402
from streamyolo_b200.model import DFPPAFPN, PIPEHead, YOLOX, backward  # noqa: E402

LOSSES = ("total_loss", "iou_loss", "l1_loss", "conf_loss", "cls_loss", "num_fg")


def install(monkeypatch):
    """tests/emul_ops.py with fp32 storage, plus SyConvDesc.stat_updates: the emulated conv applies one running-statistics
    update per statistics group; a launch with ``stat_updates=2`` (one group) gets its second update here, from the same
    stored output and in the same arithmetic, and num_batches_tracked += 1 more."""
    emul_ops.install(monkeypatch, exact=True)
    base = ops.conv2d

    def conv2d(x, wpk, y, k, s, mode, *a, stat_updates=1, **kw):
        rows = base(x, wpk, y, k, s, mode, *a, **kw)
        bn = kw.get("bn")
        assert stat_updates in (0, 1, 2)
        if stat_updates == 2:
            assert bn and mode == ops.SY_CONV_RAW and not 0 < kw.get("split_n", 0) < x.n, "stat_updates=2: one group, with bn"
            stored = y.torch().permute(0, 3, 1, 2).float()
            mean, var = stored.mean((0, 2, 3)), stored.var((0, 2, 3), unbiased=False)
            cnt = stored.numel() / stored.shape[1]
            mom = kw.get("momentum", 0.03)
            ends = [seg[5] for seg in bn[1:]] + [stored.shape[1]]
            for (_, _, rm, rv, nbt, c0), c1 in zip(bn, ends):
                if rm is not None:
                    rm.mul_(1 - mom).add_(mom * mean[c0:c1])
                    rv.mul_(1 - mom).add_(mom * var[c0:c1] * (cnt / max(cnt - 1, 1)))
                if nbt is not None:
                    nbt.add_(1)
        return rows

    monkeypatch.setattr(ops, "conv2d", conv2d)


def build_still(c):
    ch = [256, 512, 1024]
    m = YOLOX(DFPPAFPN(c["depth"], c["width"], in_channels=ch), PIPEHead(8, c["width"], in_channels=ch))
    for mod in m.modules():
        if isinstance(mod, torch.nn.BatchNorm2d):
            mod.eps, mod.momentum = 1e-3, 0.03
    m.load_state_dict(synth.synth_state_dict({k: tuple(v.shape) for k, v in m.state_dict().items()}), strict=True)
    m.head.use_l1 = True
    return m.train()


def still_batch(c):
    x = synth.synth_frames(c["B"], c["H"], c["W"])[:, :3].contiguous()
    labels, _ = synth.synth_labels(c["B"], c["H"], c["W"], empty_image=c["empty"])
    return x, labels


def oracle(c):
    cfg = OracleCfg(depth=c["depth"], width=c["width"], gamma=0.0, ignore_thr=0.0, ignore_value=1.0)
    o = StreamYoloOracle(cfg, synth.synth_state_dict(model_shapes(c["depth"], c["width"])), q=None)
    for k, t in o.P.items():
        if t.dtype.is_floating_point and not k.endswith(("running_mean", "running_var")):
            t.requires_grad_(True)
    return o


@pytest.mark.parametrize("name", ["tiny_120x160", "tiny_empty_96x160"])
def test_still_step_equals_duplicated_pair_reference(name, monkeypatch):
    """The reference trainer's sequence on a still model -- ``model(inps [B, 3, H, W], targets [B, M, 5])`` then
    ``loss.backward()`` -- against the oracle on the duplicated pair: the six losses, every parameter gradient and every
    BatchNorm buffer (two running updates per backbone / PAFPN / jian module, num_batches_tracked = 2), on a NaN-poisoned
    gradient arena (the DFP residual lands on one channel half of a region the two jian data gradients then write whole: a
    partly covered region)."""
    c = CASES[name]
    install(monkeypatch)
    monkeypatch.setattr(backward, "POISON", True)
    x, labels = still_batch(c)
    model = build_still(c)
    out = model(x, labels)
    assert out["total_loss"].requires_grad
    out["total_loss"].backward()
    o = oracle(c)
    ref = o.forward(torch.cat([x, x], 1), (labels, labels))
    ref["total_loss"].backward()
    for k in LOSSES:
        got, want = (float(t.detach()) if torch.is_tensor(t) else float(t) for t in (out[k], ref[k]))
        assert abs(got - want) <= 2e-5 * abs(want) + 1e-6, k
    report = []
    for k, p in model.named_parameters():
        assert p.grad is not None and torch.isfinite(p.grad).all(), f"no finite gradient reached {k}"
        g, r = p.grad.float().flatten(), o.P[k].grad.float().flatten()
        report.append((float((g - r).norm() / (r.norm() + 1e-12)), k))
    report.sort(reverse=True)
    assert report[0][0] < 1e-3, "largest deviations:\n" + "\n".join(f"{rel:8.3e} {k}" for rel, k in report[:10])
    sd = model.state_dict()
    n_bn = 0
    for k, v in sd.items():
        if k.endswith(("running_mean", "running_var")):
            assert torch.allclose(v, o.P[k].detach(), rtol=1e-4, atol=1e-6), k
            n_bn += 1
        elif k.endswith("num_batches_tracked"):
            assert int(v) == (1 if k.startswith("head.") else 2), k        # the head runs once per step, as in the reference
    assert n_bn == 2 * sum(isinstance(m, torch.nn.BatchNorm2d) for m in model.modules())


def test_still_recording_forward_runs_the_backbone_once(monkeypatch):
    """One backbone + PAFPN pass over B images: every conv launch of it sees B images and updates its running statistics
    twice; the DFP jian convs still run twice (jian(cur), jian(sup)), the head once per level."""
    c = CASES["tiny_120x160"]
    install(monkeypatch)
    seen = []
    real = ops.conv2d

    def spy(x, wpk, y, *a, **kw):
        if kw.get("bn"):
            seen.append((x.n, kw.get("stat_updates", 1)))
        return real(x, wpk, y, *a, **kw)

    monkeypatch.setattr(ops, "conv2d", spy)
    x, labels = still_batch(c)
    model = build_still(c)
    tape, _ = backward._record(model, x, labels)
    net, head = model.backbone, model.head
    jian = {id(net.jian2), id(net.jian1), id(net.jian0)}
    heads = {id(m) for m in head.modules()}
    plan = train.conv_groups_forward_order(model)
    assert {id(g[0]): tape.uses[id(g[0])] for g in plan} == {id(g[0]): 2 if id(g[0]) in jian else 1 for g in plan}
    convs = [r for r in tape.ops if r["t"] == "conv"]
    assert len(convs) == len(seen) == len(plan) + 3
    for r, (n, upd) in zip(convs, seen):
        m = id(r["mods"][0])
        assert n == c["B"] and r["split"] == 0
        assert upd == (1 if (m in jian or m in heads) else 2)


def test_trainer_still_step_matches_stock_pytorch_step(monkeypatch):
    """Three ``Trainer.step`` calls on 3-channel frames and one label tensor == three steps of torch SGD + Python ModelEMA
    around the same backward: losses, every parameter, the EMA copy and the BatchNorm buffers."""
    install(monkeypatch)
    c = CASES["tiny_120x160"]
    x, labels = still_batch(c)
    ref = build_still(c)
    opt = train.build_optimizer(ref, lr=2e-4)
    ema = train.ModelEMA(ref)
    model = build_still(c)
    tr = train.Trainer(model, lr=2e-4)
    wants = [train.train_step(ref, opt, x, labels, ema) for _ in range(3)]
    for i in range(3):
        got = tr.step(x, labels)
        assert abs(float(got["total_loss"]) - float(wants[i]["total_loss"])) <= 1e-5 * abs(float(wants[i]["total_loss"])), i
    net = model.backbone
    assert tr.sink.uses[id(net.jian0)] == 2 and tr.sink.uses[id(net.backbone.dark3[0])] == 1
    for (k, p), q in zip(model.named_parameters(), ref.parameters()):
        assert torch.allclose(p, q, rtol=1e-5, atol=1e-7), k
    esd, rsd = tr.ema_state_dict(), ema.ema.state_dict()
    for k in rsd:
        if rsd[k].dtype.is_floating_point:
            assert torch.allclose(esd[k], rsd[k], rtol=1e-5, atol=1e-7), k
    sd, rs = model.state_dict(), ref.state_dict()
    for k in ("backbone.backbone.stem.conv.bn.running_mean", "backbone.C3_n4.conv3.bn.running_var",
              "head.stems.0.bn.running_var", "backbone.jian1.bn.running_mean"):
        assert torch.allclose(sd[k], rs[k], rtol=1e-5, atol=1e-7), k
    assert int(sd["backbone.backbone.dark2.0.bn.num_batches_tracked"]) == 6 and int(sd["backbone.jian1.bn.num_batches_tracked"]) == 6


def test_tal_head_refuses_a_single_label_tensor(monkeypatch):
    """A TALHead trains on (future, current) labels; one tensor used to be indexed as that pair (the labels of images 0 and
    1).  Every training entry point now says so."""
    install(monkeypatch)
    c = CASES["tiny_120x160"]
    x = synth.synth_frames(c["B"], c["H"], c["W"])
    fut, _ = synth.synth_labels(c["B"], c["H"], c["W"])
    model = T.build_product(c)
    with pytest.raises(TypeError, match="PIPEHead"):
        model(x, fut)
    with pytest.raises(TypeError, match="PIPEHead"):
        backward.forward_backward(model, x, fut)
    with pytest.raises(TypeError, match="PIPEHead"):
        train.Trainer(model).step(x, fut)
    with pytest.raises(ValueError, match="channels|frames"):
        backward.forward_backward(build_still(c), x[:, :4].contiguous(), fut)


def _aligned(nbytes):
    raw = (C.c_uint8 * (nbytes + 16))()
    return raw, (C.addressof(raw) + 15) // 16 * 16


def test_conv_rejects_stat_updates_misuse():
    """sy_conv2d_tc checks stat_updates before anything reaches the device: only 0, 1, 2; 2 needs the BatchNorm finalize
    and a single statistics group."""
    lib = ops.load_library()
    keep, p = _aligned(1 << 16)
    d = ops.SyConvDesc()
    d.x = ops.SyTensor(p, 2, 4, 4, 16, 16)
    d.y = ops.SyTensor(p, 2, 4, 4, 16, 16)
    d.w, d.kh, d.kw, d.stride, d.mode = p, 1, 1, 1, ops.SY_CONV_RAW
    d.stat_partials, d.n_partials = p, 256
    d.bn[0].gamma = d.bn[0].beta = p
    d.scale_shift = d.sync = p
    d.stat_updates = 3
    assert lib.sy_conv2d_tc(C.byref(d), None) == 1
    assert b"stat_updates 3" in lib.sy_last_error_string()
    d.stat_updates, d.split_n = 2, 1                                          # two statistics groups
    assert lib.sy_conv2d_tc(C.byref(d), None) == 1
    assert b"single statistics group" in lib.sy_last_error_string()
    d.split_n, d.bn[0].gamma = 0, None                                        # no BatchNorm to update
    assert lib.sy_conv2d_tc(C.byref(d), None) == 1
    assert b"BatchNorm finalize" in lib.sy_last_error_string()
    d.bn[0].gamma, d.mode = p, ops.SY_CONV_FUSED
    assert lib.sy_conv2d_tc(C.byref(d), None) == 1
    d.stat_updates = -1
    assert lib.sy_conv2d_tc(C.byref(d), None) == 1


def test_frame_labels_rejects_bad_descriptors():
    """Host-side validation of sy_frame_labels: SY_EINVAL before anything reaches the device."""
    lib = ops.load_library()
    buf = (C.c_uint8 * 64)()
    out = (C.c_float * 64)()
    d = ops.SyFrameLabelsDesc(C.addressof(out), C.addressof(buf), C.addressof(buf), 1, 2, 0, 1, 8, 1.0,
                              C.addressof(out), C.addressof(buf))                              # max_labels 0
    assert lib.sy_frame_labels(C.byref(d), None) == 1
    d.max_labels, d.n = 4, 0                                                                    # no frames
    assert lib.sy_frame_labels(C.byref(d), None) == 1
    d.n, d.r = 1, 0.0                                                                           # no scale
    assert lib.sy_frame_labels(C.byref(d), None) == 1
    d.r, d.mirror = 1.0, None                                                                   # flip without bits
    assert lib.sy_frame_labels(C.byref(d), None) == 1
    assert b"mirror" in lib.sy_last_error_string()
    d.flip, d.labels = 0, None
    assert lib.sy_frame_labels(C.byref(d), None) == 1
    assert b"null" in lib.sy_last_error_string()
