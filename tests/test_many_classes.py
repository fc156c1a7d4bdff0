"""Training with more than 27 classes (COCO's 80 included): ``sy_head_pred_backward_wide`` and everything around it.

The forward takes any class count the head's shared-memory weight tile holds; the training backward of the prediction
convs above 27 classes runs ``sy_head_pred_backward_wide`` (``model/backward.py`` picks it from the head's class count).

CPU:
  * the oracle with 80 classes against fixtures of the unmodified reference (oracle/make_classes_golden.py): the pair
    model's losses, SimOTA assignment, BatchNorm / conv statistics, gradients, and the still model's losses, assignment and
    gradients;
  * the backward walk with every kernel emulated (tests/emul_ops.py, fp32 storage, NaN-poisoned gradient arena) for an
    80-class pair model and still model against autograd through the oracle, and ``Trainer.step`` against the stock
    ``torch.optim.SGD`` + EMA step;
  * which of the two prediction-conv backward kernels the walk picks, and that the new kernels compile without spills.
GPU:
  * the new kernel against float64 at every head level of StreamYOLO-s and -l (600x960, 8 images) for 28, 80 and 195
    classes, with ``accumulate``, repeat launches and the partial-row bar; bit-identical to the old kernel at 8 classes;
  * ``sy_tal_loss`` / ``sy_tal_loss_backward`` at 80 classes and the full anchor count;
  * StreamYOLO-s with 80 classes, pair and still: every conv's backward in situ, graph replay over three sizes equal to
    eager steps, and a resumed run equal to an uninterrupted one."""
import os
import re
import subprocess
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import emul_ops  # noqa: E402
import test_still_train as still_emul  # noqa: E402
from oracle.make_classes_golden import CASE, NAME, NUM_CLASSES  # noqa: E402
from oracle.streamyolo_oracle import OracleCfg, StreamYoloOracle, model_shapes  # noqa: E402
from streamyolo_b200 import ops, synth, train  # noqa: E402
from streamyolo_b200.model import DFPPAFPN, PIPEHead, TALHead, YOLOX, backward  # noqa: E402

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
LOSSES = ("total_loss", "iou_loss", "l1_loss", "conf_loss", "cls_loss", "num_fg")


def stat3(t):
    t = t.detach().double()
    return np.array([t.mean().item(), t.abs().mean().item(), t.pow(2).mean().sqrt().item()])


def build(c, nc=NUM_CLASSES, still=False, device="cpu", momentum=0.03):
    """the product model as the fixtures' reference model is built: TALHead (pair) or PIPEHead (still) with ``nc`` classes"""
    ch = [256, 512, 1024]
    head = (PIPEHead(nc, c["width"], in_channels=ch) if still else
            TALHead(nc, c["width"], in_channels=ch, gamma=c["gamma"], ignore_thr=c["thr"], ignore_value=c["val"]))
    m = YOLOX(DFPPAFPN(c["depth"], c["width"], in_channels=ch), head)
    for mod in m.modules():
        if isinstance(mod, torch.nn.BatchNorm2d):
            mod.eps, mod.momentum = 1e-3, momentum
    m.head.initialize_biases(1e-2)
    m.load_state_dict(synth.synth_state_dict({k: tuple(v.shape) for k, v in m.state_dict().items()}), strict=True)
    m.head.use_l1 = True
    return m.to(device).train()


def oracle(c, still=False, grad=False):
    """fp32 oracle with 80 classes; the still model is the oracle of the duplicated pair with gamma = 0 (no trend weights)"""
    kw = dict(gamma=0.0, ignore_thr=0.0, ignore_value=1.0) if still else dict(gamma=c["gamma"], ignore_thr=c["thr"],
                                                                               ignore_value=c["val"])
    cfg = OracleCfg(depth=c["depth"], width=c["width"], num_classes=NUM_CLASSES, **kw)
    o = StreamYoloOracle(cfg, synth.synth_state_dict(model_shapes(c["depth"], c["width"], NUM_CLASSES)), q=None)
    if grad:
        for k, t in o.P.items():
            if t.dtype.is_floating_point and not k.endswith(("running_mean", "running_var")):
                t.requires_grad_(True)
    return o


def pair_batch(c):
    return (synth.synth_frames(c["B"], c["H"], c["W"]),
            synth.synth_labels(c["B"], c["H"], c["W"], empty_image=c["empty"], num_classes=NUM_CLASSES))


def still_batch(c):
    x, tg = pair_batch(c)
    return x[:, :3].contiguous(), tg[0]


# ================================================================================================ CPU: oracle vs reference
def test_oracle_matches_reference_80_classes():
    c = CASE
    g = np.load(os.path.join(GOLD, NAME + ".npz"))
    x, tg = pair_batch(c)
    o = oracle(c)
    o.trace = {}
    outputs, origin, grid = o.flatten_decode(o.head_levels(o.backbone_off(x)), sigmoid=False)
    assert outputs.shape[2] == 5 + NUM_CLASSES
    res = o.losses(outputs, origin, grid, tg, return_aux=True)
    np.testing.assert_allclose(np.array([float(res[k]) for k in LOSSES]), g["train_loss"], rtol=2e-4, atol=1e-5)
    aux = res["aux"]
    bi, ai = aux["fg"].nonzero(as_tuple=True)
    assert len(ai) > 0
    assert np.array_equal(bi.numpy().astype(np.int32), g["fg_image"])
    assert np.array_equal(ai.numpy().astype(np.int32), g["fg_anchor"])
    assert np.array_equal(aux["matched"][bi, ai].numpy().astype(np.int32), g["fg_gt"])
    np.testing.assert_allclose(aux["pred_iou"][bi, ai].numpy(), g["fg_iou"], rtol=1e-4, atol=1e-6)
    for k, ref in zip(g["bn_keys"].tolist(), g["bn_stats_after_train"]):
        np.testing.assert_allclose(stat3(o.P[k]), ref, rtol=1e-4, atol=1e-6, err_msg=k)
    for k, ref in zip(g["conv_keys"].tolist(), g["conv_stats_train"]):
        if not k.startswith("backbone.jian"):
            np.testing.assert_allclose(stat3(o.trace[k]), ref, rtol=2e-4, atol=1e-6, err_msg=k)
    # the labels reach classes above 27: the wide kernel's range is what the fixtures pin
    assert int(tg[0][..., 0].max()) > 27


def _check_grads(o, g, prefix=""):
    keys = g[prefix + "grad_keys"].tolist()
    assert set(keys) == {k for k, t in o.P.items() if t.grad is not None}
    l2 = dict(zip(keys, g[prefix + "grad_l2"].tolist()))
    worst = max(abs(float(o.P[k].grad.norm()) - l2[k]) / (l2[k] + 1e-6) for k in keys)
    assert worst < 5e-3, f"worst relative gradient-norm error {worst:.2e}"
    n = 0
    for f in g.files:
        if f.startswith(prefix + "g:"):
            ref = torch.from_numpy(g[f])
            got = o.P[f[len(prefix) + 2:]].grad
            assert tuple(got.shape) == tuple(ref.shape), f
            assert torch.allclose(got, ref, rtol=2e-3, atol=2e-5 * float(ref.abs().max()) + 1e-7), f
            n += 1
    assert n >= 18                      # reg / obj / cls weight and bias at three levels


def test_oracle_backward_matches_reference_80_classes():
    c = CASE
    g = np.load(os.path.join(GOLD, "grad_" + NAME + ".npz"))
    o = oracle(c, grad=True)
    x, tg = pair_batch(c)
    loss = o.forward(x, tg)["total_loss"]
    assert abs(float(loss.detach()) - float(g["total_loss"])) <= 2e-4 * abs(float(g["total_loss"]))
    loss.backward()
    _check_grads(o, g)


def test_oracle_still_matches_reference_80_classes():
    """the reference's still model on single frames == the oracle on the duplicated pair with gamma = 0: losses,
    assignment, gradients"""
    c = CASE
    g, gg = np.load(os.path.join(GOLD, NAME + ".npz")), np.load(os.path.join(GOLD, "grad_" + NAME + ".npz"))
    x, labels = still_batch(c)
    o = oracle(c, still=True, grad=True)
    xx = torch.cat([x, x], 1)
    outputs, origin, grid = o.flatten_decode(o.head_levels(o.backbone_off(xx)), sigmoid=False)
    res = o.losses(outputs, origin, grid, (labels, labels), return_aux=True)
    np.testing.assert_allclose(np.array([float(res[k]) for k in LOSSES]), g["still_train_loss"], rtol=2e-4, atol=1e-5)
    aux = res["aux"]
    bi, ai = aux["fg"].nonzero(as_tuple=True)
    assert np.array_equal(bi.numpy().astype(np.int32), g["still_fg_image"])
    assert np.array_equal(ai.numpy().astype(np.int32), g["still_fg_anchor"])
    assert np.array_equal(aux["matched"][bi, ai].numpy().astype(np.int32), g["still_fg_gt"])
    np.testing.assert_allclose(aux["pred_iou"][bi, ai].numpy(), g["still_fg_iou"], rtol=1e-4, atol=1e-6)
    o = oracle(c, still=True, grad=True)
    loss = o.forward(xx, (labels, labels))["total_loss"]
    assert abs(float(loss.detach()) - float(gg["still_total_loss"])) <= 2e-4 * abs(float(gg["still_total_loss"]))
    loss.backward()
    _check_grads(o, gg, "still_")


# ================================================================================================ CPU: emulated kernels
def install(monkeypatch):
    """every kernel emulated in torch with fp32 storage (tests/emul_ops.py plus the still model's repeated running update),
    and the two prediction-conv backward entry points emulated with their class-count ranges: the old one refuses more
    than 27 classes as sy_head_pred_backward does.  Returns the list of (entry point, classes) the walk called."""
    still_emul.install(monkeypatch)
    calls = []

    def narrow(grad_raw, cf, rf, dcf, drf, w_reg, w_obj, w_cls, *a, **kw):
        if not 1 <= w_cls.shape[0] <= 27:
            raise RuntimeError("libstreamyolo_sm100 error 1: head_pred_backward: num_classes out of range")
        calls.append(("narrow", w_cls.shape[0]))
        emul_ops.head_pred_backward(grad_raw, cf, rf, dcf, drf, w_reg, w_obj, w_cls, *a, **kw)

    def wide(grad_raw, cf, rf, dcf, drf, w_reg, w_obj, w_cls, *a, **kw):
        assert 1 <= w_cls.shape[0] <= 251 and (5 + w_cls.shape[0]) * cf.c * 4 <= 200 * 1024
        calls.append(("wide", w_cls.shape[0]))
        emul_ops.head_pred_backward_wide(grad_raw, cf, rf, dcf, drf, w_reg, w_obj, w_cls, *a, **kw)

    monkeypatch.setattr(ops, "head_pred_backward", narrow)
    monkeypatch.setattr(ops, "head_pred_backward_wide", wide)
    monkeypatch.setattr(backward, "POISON", True)
    return calls


@pytest.mark.parametrize("still", [False, True], ids=["pair", "still"])
def test_walk_80_classes_equals_oracle_autograd(still, monkeypatch):
    """forward_backward of an 80-class tiny model, every kernel emulated in fp32, on a NaN-poisoned gradient arena, against
    autograd through the oracle: the six losses to 2e-5 and every parameter gradient to 1e-4 (relative norm)"""
    c = CASE
    calls = install(monkeypatch)
    model = build(c, still=still)
    if still:
        x, labels = still_batch(c)
        out = backward.forward_backward(model, x, labels)
        o = oracle(c, still=True, grad=True)
        ref = o.forward(torch.cat([x, x], 1), (labels, labels))
    else:
        x, tg = pair_batch(c)
        out = backward.forward_backward(model, x, tg)
        o = oracle(c, grad=True)
        ref = o.forward(x, tg)
    ref["total_loss"].backward()
    assert calls == [("wide", NUM_CLASSES)] * 3
    for k in LOSSES:
        got, want = float(out[k]), float(ref[k])
        assert abs(got - want) <= 2e-5 * abs(want) + 1e-6, (k, got, want)
    report = []
    for k, p in model.named_parameters():
        assert p.grad is not None and torch.isfinite(p.grad).all(), f"no finite gradient reached {k}"
        g, r = p.grad.float().flatten(), o.P[k].grad.float().flatten()
        report.append((float((g - r).norm() / (r.norm() + 1e-12)), k))
    report.sort(reverse=True)
    assert report[0][0] < 1e-4, "largest deviations:\n" + "\n".join(f"{rel:8.3e} {k}" for rel, k in report[:10])


@pytest.mark.parametrize("nc,kernel", [(27, "narrow"), (28, "wide")])
def test_walk_picks_the_kernel_from_the_class_count(nc, kernel, monkeypatch):
    c = CASE
    calls = install(monkeypatch)
    x = synth.synth_frames(c["B"], c["H"], c["W"])
    tg = synth.synth_labels(c["B"], c["H"], c["W"], num_classes=nc)
    backward.forward_backward(build(c, nc=nc), x, tg)
    assert calls == [(kernel, nc)] * 3


def test_trainer_step_80_classes_matches_stock_pytorch_step(monkeypatch):
    """three Trainer.step calls (FlatState / FlatSink with 80-class head slices) == three steps of torch SGD + Python
    ModelEMA around the same backward: losses, every parameter, the EMA copy, BatchNorm buffers; and the state dict
    round trip"""
    install(monkeypatch)
    c = CASE
    x, tg = pair_batch(c)
    ref = build(c)
    opt = train.build_optimizer(ref, lr=2e-4)
    ema = train.ModelEMA(ref)
    model = build(c)
    tr = train.Trainer(model, lr=2e-4)
    wants = [train.train_step(ref, opt, x, tg, ema) for _ in range(3)]
    for i in range(3):
        got = tr.step(x, tg)
        assert abs(float(got["total_loss"]) - float(wants[i]["total_loss"])) <= 1e-5 * abs(float(wants[i]["total_loss"])), i
    for (k, p), q in zip(model.named_parameters(), ref.parameters()):
        assert torch.allclose(p, q, rtol=1e-5, atol=1e-7), k
    esd, rsd = tr.ema_state_dict(), ema.ema.state_dict()
    for k in rsd:
        if rsd[k].dtype.is_floating_point:
            assert torch.allclose(esd[k], rsd[k], rtol=1e-5, atol=1e-7), k
    assert tuple(esd["head.cls_preds.0.weight"].shape)[0] == NUM_CLASSES
    sd = tr.state_dict()
    tr2 = train.Trainer(build(c), lr=2e-4)
    tr2.load_state_dict(sd)
    for (k, p), q in zip(tr2.model.named_parameters(), model.parameters()):
        assert torch.equal(p, q), k
    assert torch.equal(tr2.fs.mom, tr.fs.mom) and torch.equal(tr2.fs.ema, tr.fs.ema)


def test_wide_head_backward_kernels_compile_without_spills(tmp_path):
    """head_pred_bwd_data_wide_kernel and head_pred_bwd_weight_wide_kernel: 0 spill bytes, no stack frame, no ptxas warning"""
    import shutil
    from streamyolo_b200 import build as B
    nvcc = B.NVCC if os.path.exists(B.NVCC) else shutil.which("nvcc")
    if nvcc is None:
        pytest.skip("no nvcc")
    r = subprocess.run([nvcc] + B.COMMON + B.SOURCES["bwd_glue.cu"] + ["-c", os.path.join(B.CSRC, "bwd_glue.cu"), "-o",
                       str(tmp_path / "b.o")], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=600)
    assert r.returncode == 0, r.stdout
    assert not [ln for ln in r.stdout.splitlines() if ln.startswith("ptxas") and "warning" in ln.lower()], r.stdout
    found = re.findall(r"Compiling entry function '(\w*head_pred_bwd_\w+_wide_kernel\w*)'[^\n]*\n[^\n]*\n\s*(\d+) bytes stack "
                       r"frame, (\d+) bytes spill stores, (\d+) bytes spill loads", r.stdout)
    assert len(found) == 2, found
    for name, st, sp, ld in found:
        assert (st, sp, ld) == ("0", "0", "0"), f"{name}: {st} bytes stack, {sp} bytes spill stores, {ld} bytes spill loads"


# ================================================================================================ GPU
DEV = "cuda"
SY_EINVAL = 1
HEAD_LEVELS = [(75, 120, 0), (38, 60, 9000), (19, 30, 11280)]          # 600x960: anchor offsets in a_total = 11 850
A_TOTAL = 11850
HW = [(75, 120), (38, 60), (19, 30)]
STRIDES = (8, 16, 32)
# images, channels (l: 256, s: 128), level, classes
WIDE_CASES = [(8, c, h, w, off, nc) for c in (256, 128) for h, w, off in HEAD_LEVELS for nc in (28, 80, 195)]


def _head_operands(b, c, h, w, nc, seed):
    from test_gpu_parity_bwd import _gen, post_silu
    g = _gen(seed)
    cfv, rfv = post_silu(b, h, w, c, seed + 1), post_silu(b, h, w, c, seed + 2)
    ws = [torch.randn((o, c), generator=g, device=DEV) * 0.05 for o in (4, 1, nc)]
    grad_raw = torch.randn((b, A_TOTAL, 5 + nc), generator=g, device=DEV) * 1e-3
    return cfv, rfv, ws, grad_raw


def _launch(fn, grad_raw, cfv, rfv, ws, off, accumulate=False, start=None):
    from streamyolo_b200.ops import View
    b, h, w, c = cfv.n, cfv.h, cfv.w, cfv.c
    nc = ws[2].shape[0]
    dcf, drf = View.empty(b, h, w, c, DEV), View.empty(b, h, w, c, DEV)
    if start is None:
        dws = [torch.full((o, c), float("nan"), device=DEV) for o in (4, 1, nc)]
        dbs = [torch.full((o,), float("nan"), device=DEV) for o in (4, 1, nc)]
    else:
        dws, dbs = [t.clone() for t in start[0]], [t.clone() for t in start[1]]
    fn(grad_raw, cfv, rfv, dcf, drf, *ws, A_TOTAL, off, *dws, *dbs, accumulate=accumulate)
    return dcf, drf, dws, dbs


@pytest.mark.gpu
@pytest.mark.parametrize("case", WIDE_CASES, ids=lambda c: "x".join(map(str, c)))
def test_head_pred_backward_wide_vs_float64(case):
    """data gradients within one bf16 rounding of float64, weight / bias gradients within the fp32 reduction bar; a
    second launch is bit-identical, ``accumulate`` adds onto a non-zero start, and the bar rejects the sums with one
    256-pixel partial row left out"""
    from test_gpu_ops import check_close
    from test_gpu_parity_bwd import _head_ref, assert_rejects_sum, check_sum
    b, c, h, w, off, nc = case
    cfv, rfv, ws, grad_raw = _head_operands(b, c, h, w, nc, 31 + nc)
    dcf, drf, dws, dbs = _launch(ops.head_pred_backward_wide, grad_raw, cfv, rfv, ws, off)
    torch.cuda.synchronize()
    P = b * h * w
    gl = grad_raw[:, off:off + h * w].double().reshape(P, 5 + nc)
    fr, fc = rfv.torch().double().reshape(P, c), cfv.torch().double().reshape(P, c)
    w64 = [t.double() for t in ws]
    d_rf, d_cf, dw_ref = _head_ref(gl, fr, fc, *w64)
    check_close(drf.torch().double().reshape(P, c), d_rf, f"wide{case}: d reg_feat")
    check_close(dcf.torch().double().reshape(P, c), d_cf, f"wide{case}: d cls_feat")
    del d_rf, d_cf
    _, _, s2w = _head_ref(gl.square(), fr.square(), fc.square(), *w64)
    dw = torch.cat(dws, 0)
    check_sum(dw, dw_ref, s2w, P, f"wide{case}: dW")
    db, db_ref, s2b = torch.cat(dbs), gl.sum(0), gl.square().sum(0)
    check_sum(db, db_ref, s2b, P, f"wide{case}: db")
    rows = -(-P // 256)
    r = rows // 2
    q0, q1 = 256 * r, min(P, 256 * r + 256)
    _, _, part = _head_ref(gl[q0:q1], fr[q0:q1], fc[q0:q1], *w64)
    assert_rejects_sum(dw, dw_ref - part, s2w, P, f"wide{case}: dW, row {r} left out")
    assert_rejects_sum(db, db_ref - gl[q0:q1].sum(0), s2b, P, f"wide{case}: db, row {r} left out")
    # a second launch: the same bits
    dcf2, drf2, dws2, dbs2 = _launch(ops.head_pred_backward_wide, grad_raw, cfv, rfv, ws, off)
    assert torch.equal(dcf2.torch(), dcf.torch()) and torch.equal(drf2.torch(), drf.torch())
    assert all(torch.equal(a, b_) for a, b_ in zip(dws2 + dbs2, dws + dbs))
    # accumulate onto a start: start + (the same sums), one fp32 addition per element
    gen = torch.Generator(device=DEV).manual_seed(5)
    start = ([torch.randn(t.shape, generator=gen, device=DEV) for t in dws], [torch.randn(t.shape, generator=gen, device=DEV)
                                                                             for t in dbs])
    _, _, dws3, dbs3 = _launch(ops.head_pred_backward_wide, grad_raw, cfv, rfv, ws, off, accumulate=True, start=start)
    torch.cuda.synchronize()
    for got, s0, once in zip(dws3 + dbs3, start[0] + start[1], dws + dbs):
        assert torch.equal(got, s0 + once)


@pytest.mark.gpu
@pytest.mark.parametrize("c,h,w,off", [(256, 75, 120, 0), (128, 38, 60, 9000)])
def test_head_pred_backward_wide_equals_old_kernel_at_8_classes(c, h, w, off):
    """at 8 classes both entry points run the same sums in the same order: bit-identical results"""
    cfv, rfv, ws, grad_raw = _head_operands(8, c, h, w, 8, 77)
    old = _launch(ops.head_pred_backward, grad_raw, cfv, rfv, ws, off)
    new = _launch(ops.head_pred_backward_wide, grad_raw, cfv, rfv, ws, off)
    torch.cuda.synchronize()
    assert torch.equal(old[0].torch(), new[0].torch()) and torch.equal(old[1].torch(), new[1].torch())
    for a, b_ in zip(old[2] + old[3], new[2] + new[3]):
        assert torch.equal(a, b_)


@pytest.mark.gpu
@pytest.mark.parametrize("c,nc", [(256, 196), (8, 252), (64, 0)])
def test_head_pred_backward_wide_rejects_what_the_forward_rejects(c, nc):
    """above the forward's limits -- (5 + nc) * c * 4 > 200 KiB, more than 251 classes, no class -- the entry point
    refuses before it launches"""
    from streamyolo_b200.ops import View
    from test_gpu_parity_bwd import post_silu
    b, h, w = 1, 8, 10
    cfv, rfv = post_silu(b, h, w, c, 12), post_silu(b, h, w, c, 13)
    ws = [torch.zeros((o, c), device=DEV) for o in (4, 1, nc)]
    grad_raw = torch.zeros((b, h * w, 5 + nc), device=DEV)
    dws = [torch.zeros((o, c), device=DEV) for o in (4, 1, nc)]
    dbs = [torch.zeros((o,), device=DEV) for o in (4, 1, nc)]
    with pytest.raises(RuntimeError, match=f"libstreamyolo_sm100 error {SY_EINVAL}:"):
        ops.head_pred_backward_wide(grad_raw, cfv, rfv, View.empty(b, h, w, c, DEV), View.empty(b, h, w, c, DEV), *ws, h * w,
                                    0, *dws, *dbs)


def _outputs_80(b, fut, seed):
    """plausible decoded head outputs [b, 11850, 85] (fp32): boxes near their anchors, a few anchors per ground truth
    predicting that box (and its class) well, low obj / cls logits elsewhere"""
    g = torch.Generator().manual_seed(seed)
    outs, origin = [], []
    for (h, w), s in zip(HW, STRIDES):
        yv, xv = torch.meshgrid(torch.arange(h), torch.arange(w), indexing="ij")
        raw = torch.randn((b, h * w, 4), generator=g) * 0.4
        xy = (raw[..., :2] + torch.stack([xv, yv], -1).reshape(1, -1, 2)) * s
        wh = torch.exp(raw[..., 2:4] + 1.2) * s
        outs.append(torch.cat([xy, wh, torch.randn((b, h * w, 1 + NUM_CLASSES), generator=g) * 1.5 - 3.0], -1))
        origin.append(raw)
    out, org = torch.cat(outs, 1), torch.cat(origin, 1)
    for bi in range(b):
        for gt in fut[bi]:
            if gt[3] <= 0:
                continue
            d = (out[bi, :, 0] - gt[1]).abs() + (out[bi, :, 1] - gt[2]).abs()
            idx = torch.topk(d, 12, largest=False).indices
            out[bi, idx, 0:4] = gt[1:5] * (1 + 0.05 * torch.randn((12, 4), generator=g))
            out[bi, idx, 4] = 1.0
            out[bi, idx, 5 + int(gt[0])] = 1.5
    return out.contiguous(), org.contiguous()


@pytest.mark.gpu
@pytest.mark.parametrize("n_gt", [0, 1, 12, 120])
def test_tal_loss_80_classes_full_anchor_count(n_gt):
    """sy_tal_loss at 80 classes and A = 11 850: foreground set and matched ids bit-exact against the oracle, the loss
    values close; sy_tal_loss_backward element-wise against float64 autograd (the bar of
    test_gpu_parity_bwd.test_tal_loss_backward_full_anchor_count)"""
    b, gamma, thr, val = 4, 1.5, 0.5, 1.6
    fut, cur = synth.synth_labels(b, 600, 960, n_obj=max(n_gt, 2), seed=40 + n_gt, num_classes=NUM_CLASSES)
    if n_gt < 2:
        fut[:, n_gt:] = 0
        cur[:, n_gt:] = 0
    if n_gt >= 12:
        fut[1] = 0
        cur[1] = 0
    outputs, origin = _outputs_80(b, fut, 50 + n_gt)
    o = StreamYoloOracle(OracleCfg(gamma=gamma, ignore_thr=thr, ignore_value=val, num_classes=NUM_CLASSES), {})
    grid = tuple(t.float() for t in o.grids(HW, STRIDES))
    ref = o.losses(outputs, origin, grid, (fut, cur), return_aux=True)
    L = fut.shape[1]
    ws = torch.empty(ops.tal_loss_workspace_bytes(b, A_TOTAL, L, NUM_CLASSES), dtype=torch.uint8, device=DEV)
    loss = torch.empty(6, device=DEV)
    fg = torch.empty((b, A_TOTAL), dtype=torch.int32, device=DEV)
    mt = torch.empty((b, A_TOTAL), dtype=torch.int32, device=DEV)
    pi = torch.empty((b, A_TOTAL), device=DEV)
    od, ogd, fd, cd = outputs.to(DEV), origin.to(DEV), fut.to(DEV), cur.to(DEV)
    ops.tal_loss(od, ogd, fd, cd, HW, STRIDES, gamma, thr, val, True, ws, loss, fg, mt, pi)
    g_raw = torch.full((b, A_TOTAL, 5 + NUM_CLASSES), float("nan"), device=DEV)
    g_out = torch.full((b, A_TOTAL, 5 + NUM_CLASSES), float("nan"), device=DEV)
    g_org = torch.full((b, A_TOTAL, 4), float("nan"), device=DEV)
    ops.tal_loss_backward(od, ogd, fd, HW, STRIDES, gamma, True, ws, 1.0, grad_outputs=g_out, grad_origin=g_org,
                          grad_raw=g_raw)
    torch.cuda.synchronize()
    aux = ref["aux"]
    assert torch.equal(fg.cpu().bool(), aux["fg"]), "foreground set differs from the oracle's"
    assert torch.equal(mt.cpu().long(), aux["matched"]), "matched GT ids differ from the oracle's"
    assert (n_gt == 0) == (int(aux["fg"].sum()) == 0)
    want = torch.tensor([float(ref[k]) for k in ("total_loss", "iou_loss", "conf_loss", "cls_loss", "l1_loss", "num_fg")])
    assert torch.allclose(loss.cpu(), want, rtol=1e-4, atol=1e-6), (loss, want)
    if n_gt >= 12:                       # classes above 27 are matched
        assert int(fut[aux["fg"].nonzero()[:, 0], aux["matched"][aux["fg"]], 0].max()) > 27
    # float64 autograd of the oracle's loss on the same fp32 outputs
    o64 = StreamYoloOracle(OracleCfg(gamma=gamma, ignore_thr=thr, ignore_value=val, num_classes=NUM_CLASSES), {})
    grid64 = tuple(t.double() for t in o64.grids(HW, STRIDES))
    out64, org64 = outputs.double().requires_grad_(True), origin.double().requires_grad_(True)
    r64 = o64.losses(out64, org64, grid64, (fut, cur), return_aux=True, dtype=torch.float64)
    assert torch.equal(r64["aux"]["fg"], aux["fg"])
    r64["total_loss"].backward()
    gout_ref = out64.grad
    gorg_ref = org64.grad if org64.grad is not None else torch.zeros_like(org64)
    graw_ref = gout_ref.clone()
    graw_ref[..., 0:2] = gout_ref[..., 0:2] * grid64[2][None, :, None] + gorg_ref[..., 0:2]
    graw_ref[..., 2:4] = gout_ref[..., 2:4] * out64.detach()[..., 2:4] + gorg_ref[..., 2:4]
    for got, want, what in ((g_out, gout_ref, "grad_outputs"), (g_org, gorg_ref, "grad_origin"), (g_raw, graw_ref, "grad_raw")):
        got = got.cpu().double()
        assert bool(torch.isfinite(got).all()), what
        nz = (want != 0).sum((0, 1)).clamp(min=1)
        rms = (want.square().sum((0, 1)) / nz).sqrt()
        err, tol = (got - want).abs(), 2.0 ** -12 * (want.abs() + rms)
        assert bool((err <= tol).all()), f"{what}: worst err / tol {float((err / tol.clamp(min=1e-300)).max()):.3g}"


S80 = dict(depth=0.33, width=0.50, gamma=1.0, thr=0.5, val=1.5)          # StreamYOLO-s (cfgs/s_s50_onex_dfp_tal_flip.py)


@pytest.mark.gpu
@pytest.mark.parametrize("still", [False, True], ids=["pair", "still"])
def test_walk_in_situ_s_80_classes(still):
    """one forward_backward of StreamYOLO-s with 80 classes at 600x960, 8 pairs / 8 frames: every recorded conv's backward
    checked in situ against float64 (test_gpu_parity_bwd.run_walk_checked), on a NaN-poisoned gradient arena"""
    from test_gpu_parity_bwd import run_walk_checked
    m = build(S80, still=still, device=DEV)
    x = synth.synth_frames(8, 600, 960, seed=4321).cuda()
    tg = tuple(t.cuda() for t in synth.synth_labels(8, 600, 960, seed=11, num_classes=NUM_CLASSES))
    if still:
        x, tg = x[:, :3].contiguous(), tg[0]
    seen = run_walk_checked(m, x, tg)
    assert len(seen) == 68, len(seen)
    assert all(bool(torch.isfinite(p.grad).all()) for p in m.head.cls_preds.parameters())


@pytest.mark.gpu
@pytest.mark.parametrize("still", [False, True], ids=["pair", "still"])
def test_graph_equals_eager_s_80_classes(still):
    """Trainer.capture_sizes over three of the cfg's sizes, replayed in random order == eager Trainer.step, bit for bit
    (losses, flat state, momentum, EMA, BatchNorm buffers)"""
    from test_multiscale_train import _graph_equals_eager
    _graph_equals_eager(lambda: build(S80, still=still, device=DEV), [(496, 800), (688, 1120), (600, 960)], (600, 960), 2,
                        still, steps=6)


@pytest.mark.gpu
def test_resume_s_80_classes():
    """an interrupted multi-scale graphed run of the 80-class StreamYOLO-s, saved through torch.save and resumed in a fresh
    model + Trainer, ends where the uninterrupted run ends, bit for bit"""
    from test_gpu_trainer_checkpoint import _lr, _roundtrip
    from test_multiscale_train import _Inputs, _assert_same, _snapshot
    dev = torch.device("cuda")
    sizes = [(496, 800), (600, 960), (688, 1120)]
    seq = [sizes[0], sizes[1], sizes[2], sizes[1], sizes[2], sizes[0]]

    def run(tr, inp, steps):
        out = []
        for i in steps:
            inp.load(100 + i)
            out.append(float(tr.replay_size(seq[i], lr=_lr(i))["total_loss"]))
        return out

    inp = _Inputs(2, (600, 960), False, dev, sizes)
    a = train.Trainer(build(S80, device=DEV), lr=1e-4)
    a.capture_sizes(sizes, inp.make_inputs, inp.prologue)
    want = run(a, inp, range(6))
    snap_a = _snapshot(a)
    del a, inp
    inp_b = _Inputs(2, (600, 960), False, dev, sizes)
    b = train.Trainer(build(S80, device=DEV), lr=1e-4)
    b.capture_sizes(sizes, inp_b.make_inputs, inp_b.prologue)
    run(b, inp_b, range(3))
    sd = _roundtrip(b.state_dict())
    del b, inp_b
    inp_c = _Inputs(2, (600, 960), False, dev, sizes)
    c = train.Trainer(build(S80, device=DEV), lr=1e-4)
    c.load_state_dict(sd)
    c.capture_sizes(sizes, inp_c.make_inputs, inp_c.prologue)
    got = run(c, inp_c, range(3, 6))
    torch.cuda.synchronize()
    assert got == want[3:], (got, want)
    _assert_same(_snapshot(c), snap_a, "resumed 80-class run")
