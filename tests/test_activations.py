"""StreamYOLO built with yolox's ReLU and LeakyReLU(0.1) activations (``act="relu"`` / ``"lrelu"``) through every path.

CPU:
  * the modules construct with the yolox activation modules and the reference's state dict layout; other names are refused;
  * the oracle (oracle/act_oracle.py) against fixtures written by the unmodified reference (oracle/make_act_golden.py);
  * the product's host code on the emulated kernels (tests/emul_ops.py with tests/emul_act.py, fp32 storage) against the
    oracle: the train step's losses and every parameter gradient (NaN-poisoned gradient arena), eval and on_pipe, the still
    model, and Trainer.step against the stock torch.optim.SGD + EMA step.
GPU (H100):
  * every kernel that takes an activation code, for codes 2 and 3, against float64 on identical operands, with inputs at
    z = +0, -0 and a few ulp either side of 0 (the derivative convention of autograd there: 0 for ReLU, 0.1 for LeakyReLU);
  * StreamYOLO-s: every BaseConv teacher-forced against the oracle, every recorded conv's backward in situ, CUDA-graph
    replays of the Trainer, the fp16-storage eval forward launch by launch, and the StreamDetector against the eager loop.
"""
import os
import sys
from collections import Counter
from types import SimpleNamespace

import numpy as np
import pytest
import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import emul_act  # noqa: E402
from oracle.act_oracle import ActOracle  # noqa: E402
from oracle.make_act_golden import ACT_CASES  # noqa: E402
from oracle.make_golden import CASES  # noqa: E402
from oracle.streamyolo_oracle import OracleCfg, bf16_round, model_shapes  # noqa: E402
from streamyolo_b200 import ops, synth, train  # noqa: E402
from streamyolo_b200.model import DFPPAFPN, PIPEHead, TALHead, YOLOX, backward, engine  # noqa: E402
from streamyolo_b200.model.network_blocks import BaseConv  # noqa: E402

GOLD = os.path.join(os.path.dirname(__file__), "golden")
ACTS = ["relu", "lrelu"]
CODES = {"relu": ops.SY_ACT_RELU, "lrelu": ops.SY_ACT_LRELU}
LOSSES = ["total_loss", "iou_loss", "l1_loss", "conf_loss", "cls_loss", "num_fg"]
TINY = CASES["tiny_120x160"]
CH = [256, 512, 1024]


def act64(t, code):
    """the activation of an SY_ACT_* code in the dtype of ``t``"""
    if code == ops.SY_ACT_RELU:
        return F.relu(t)
    if code == ops.SY_ACT_LRELU:
        return F.leaky_relu(t, 0.1)
    return F.silu(t) if code else t


def dact64(z, code):
    """d act / dz, autograd's convention at z = 0"""
    if code == ops.SY_ACT_RELU:
        return (z > 0).to(z.dtype)
    if code == ops.SY_ACT_LRELU:
        return torch.where(z > 0, torch.ones_like(z), torch.full_like(z, 0.1))
    s = torch.sigmoid(z)
    return s * (1 + z * (1 - s)) if code else torch.ones_like(z)


def build(c, act, head=TALHead, momentum=0.03, device="cpu"):
    m = YOLOX(DFPPAFPN(c["depth"], c["width"], in_channels=CH, act=act),
              head(8, c["width"], in_channels=CH, act=act, gamma=c.get("gamma", 1.0), ignore_thr=c.get("thr", 0.5),
                   ignore_value=c.get("val", 1.5)) if head is TALHead else head(8, c["width"], in_channels=CH, act=act))
    for mod in m.modules():
        if isinstance(mod, torch.nn.BatchNorm2d):
            mod.eps, mod.momentum = 1e-3, momentum
    if head is TALHead:
        m.head.initialize_biases(1e-2)
    m.load_state_dict(synth.synth_state_dict({k: tuple(v.shape) for k, v in m.state_dict().items()}), strict=True)
    m.head.use_l1 = True
    return m.to(device).train()


def oracle(c, act, q=None, momentum=0.03, gamma=None, grads=False):
    cfg = OracleCfg(depth=c["depth"], width=c["width"], gamma=c.get("gamma", 1.0) if gamma is None else gamma,
                    ignore_thr=c.get("thr", 0.5), ignore_value=c.get("val", 1.5), bn_momentum=momentum)
    o = ActOracle(cfg, synth.synth_state_dict(model_shapes(c["depth"], c["width"])), q=q, act=act)
    if grads:
        for k, t in o.P.items():
            if t.dtype.is_floating_point and not k.endswith(("running_mean", "running_var")):
                t.requires_grad_(True)
    return o


# Bars where the activation's kink at 0 meets fp32 summation order.  A pre-activation within rounding of 0 takes the other
# branch (ReLU: 0 instead of z; derivative 0 <-> 1, LeakyReLU 0.1 <-> 1) and the random-init train-mode BatchNorm net
# carries the difference on: the unmodified reference and the oracle, both fp32 on the CPU, differ by up to 2.2e-2 in a
# parameter's gradient norm (LeakyReLU; 7.8e-3 ReLU, against < 5e-3 with SiLU) and by 4 of 10 400 eval outputs beyond 2e-3.
# Those comparisons use whole-tensor bars; the losses, the assignment and the per-BaseConv statistics keep SiLU's bars.
KINK_REL = 1e-3           # relative L2 error of eval / on_pipe outputs
KINK_GRAD = 5e-2          # relative error of a parameter's gradient norm, oracle vs reference
KINK_PRODUCT_GRAD = 5e-2  # median relative L2 error of the parameter gradients, emulated product vs oracle (each one: cosine
                          # above 0.99 -- a routing mistake is O(1))
KINK_LOSS = 1e-4          # relative loss error, emulated product vs oracle


def rel_l2(a, b):
    a, b = a.double(), b.double()
    return float((a - b).norm() / (b.norm() + 1e-12))


def stat3(t):
    t = t.detach().double()
    return np.array([t.mean().item(), t.abs().mean().item(), t.pow(2).mean().sqrt().item()])


# ================================================================================================ CPU: construction
@pytest.mark.parametrize("act", ACTS)
def test_modules_construct_with_yolox_activations(act):
    want = {"relu": torch.nn.ReLU, "lrelu": torch.nn.LeakyReLU}[act]
    g = np.load(os.path.join(GOLD, "state_shapes.npz"))
    for head in (TALHead, PIPEHead):
        m = YOLOX(DFPPAFPN(0.33, 0.5, in_channels=CH, act=act), head(8, 0.5, in_channels=CH, act=act))
        ref = YOLOX(DFPPAFPN(0.33, 0.5, in_channels=CH), head(8, 0.5, in_channels=CH))
        sd, rsd = m.state_dict(), ref.state_dict()
        assert list(sd) == list(rsd) == g["s_keys"].tolist()
        assert ["x".join(map(str, v.shape)) for v in sd.values()] == g["s_shapes"].tolist()
        convs = [mod for mod in m.modules() if isinstance(mod, BaseConv)]
        assert len(convs) == 77
        for mod in convs:
            assert type(mod.act) is want and mod.act.inplace, mod
            if act == "lrelu":
                assert mod.act.negative_slope == 0.1
            assert engine.act_code(mod) == CODES[act]
        assert [type(x).__name__ for x in m.modules()] == [
            {"SiLU": want.__name__}.get(type(x).__name__, type(x).__name__) for x in ref.modules()]
    with pytest.raises(NotImplementedError):
        BaseConv(16, 16, 3, 1, act="gelu")
    with pytest.raises(NotImplementedError):
        DFPPAFPN(0.33, 0.125, in_channels=CH, act="hardswish")


def test_act_codes_mirror_the_header():
    import re
    hdr = open(os.path.join(os.path.dirname(GOLD), "..", "include", "streamyolo_sm100.h")).read()
    codes = dict((k, int(v)) for k, v in re.findall(r"(SY_ACT_\w+) = (\d+)", hdr))
    assert codes == {n: getattr(ops, n) for n in ("SY_ACT_NONE", "SY_ACT_SILU", "SY_ACT_RELU", "SY_ACT_LRELU")}
    assert ops.ACT_CODES == {"silu": 1, "relu": 2, "lrelu": 3}


def test_kink_conv_kernels_compile_without_spills(tmp_path):
    """conv_tc_kink_kernel (FUSED ReLU / LeakyReLU, bf16 and fp16, BN = 64 / 128, linear / halo): 0 spill bytes and no ptxas
    warning, like the production instantiations of conv_tc_kernel"""
    import re
    import shutil
    import subprocess
    from streamyolo_b200 import build as B
    nvcc = B.NVCC if os.path.exists(B.NVCC) else shutil.which("nvcc")
    if nvcc is None:
        pytest.skip("no nvcc")
    r = subprocess.run([nvcc] + B.COMMON + ["-c", os.path.join(B.CSRC, "conv_tc.cu"), "-o", str(tmp_path / "conv_tc.o")],
                       capture_output=True, text=True, timeout=900)
    out = r.stdout + r.stderr
    assert r.returncode == 0, out
    assert not [ln for ln in out.splitlines() if ln.startswith("ptxas") and "warning" in ln.lower()], out
    found = re.findall(r"Compiling entry function '(\w*conv_tc_kink_kernel\w*)'[^\n]*\n[^\n]*\n\s*\d+ bytes stack frame, "
                       r"(\d+) bytes spill stores, (\d+) bytes spill loads", out)
    assert len(found) == 8, found
    for name, st, ld in found:
        assert (int(st), int(ld)) == (0, 0), f"{name}: {st} bytes spill stores, {ld} bytes spill loads"


# ================================================================================================ CPU: oracle vs reference
@pytest.mark.parametrize("name", list(ACT_CASES))
def test_oracle_matches_reference(name):
    c = ACT_CASES[name]
    g = np.load(os.path.join(GOLD, name + ".npz"))
    x = synth.synth_frames(c["B"], c["H"], c["W"])
    tg = synth.synth_labels(c["B"], c["H"], c["W"], empty_image=c["empty"])
    o = oracle(c, c["act"])
    o.trace = {}
    feats = o.backbone_off(x)
    outputs, origin, grid = o.flatten_decode(o.head_levels(feats), sigmoid=False)
    res = o.losses(outputs, origin, grid, tg, return_aux=True)
    got = np.array([float(res[k]) for k in LOSSES])
    np.testing.assert_allclose(got, g["train_loss"], rtol=2e-4, atol=1e-5)
    aux = res["aux"]
    bi, ai = aux["fg"].nonzero(as_tuple=True)
    assert np.array_equal(bi.numpy().astype(np.int32), g["fg_image"])
    assert np.array_equal(ai.numpy().astype(np.int32), g["fg_anchor"])
    assert np.array_equal(aux["matched"][bi, ai].numpy().astype(np.int32), g["fg_gt"])
    # matched IoUs of the tiny net's few-pixel boxes move with fp32 summation order (2e-3 measured for ReLU); the losses
    # above carry the 2e-4 bar
    np.testing.assert_allclose(aux["pred_iou"][bi, ai].numpy(), g["fg_iou"], rtol=5e-3, atol=1e-4)
    for k, ref in zip(g["bn_keys"].tolist(), g["bn_stats_after_train"]):
        np.testing.assert_allclose(stat3(o.P[k]), ref, rtol=1e-4, atol=1e-6, err_msg=k)
    n = 0
    for k, ref in zip(g["conv_keys"].tolist(), g["conv_stats_train"]):
        if not k.startswith("backbone.jian"):
            np.testing.assert_allclose(stat3(o.trace[k]), ref, rtol=2e-4, atol=1e-6, err_msg=k)
            n += 1
    assert n == 77 - 3
    # eval after a calibration pass (momentum 1), and on_pipe
    o = oracle(c, c["act"], momentum=1.0)
    xc = torch.cat([x[:, 0:3], x[:, 0:3]], 1)
    o.forward(xc, tg)
    o.training = False
    ev = o.forward(xc)
    sub = int(g["eval_sub_step"])
    assert rel_l2(ev[:, ::sub], torch.from_numpy(g["eval_sub"])) < KINK_REL
    o1, buf = o.forward(x[:1, 0:3], mode="on_pipe")
    o2, buf2 = o.forward(x[1:2, 0:3], buffer=buf, mode="on_pipe")
    np.testing.assert_allclose(np.stack([stat3(o1), stat3(o2)] + [stat3(b) for b in buf2]), g["on_pipe_stats"], rtol=2e-3,
                               atol=1e-5)
    assert rel_l2(o2[:, ::sub], torch.from_numpy(g["on_pipe_sub2"])) < KINK_REL


@pytest.mark.parametrize("name", list(ACT_CASES))
def test_oracle_backward_matches_reference(name):
    c = ACT_CASES[name]
    g = np.load(os.path.join(GOLD, "grad_" + name + ".npz"))
    o = oracle(c, c["act"], grads=True)
    x = synth.synth_frames(c["B"], c["H"], c["W"])
    tg = synth.synth_labels(c["B"], c["H"], c["W"], empty_image=c["empty"])
    loss = o.forward(x, tg)["total_loss"]
    assert abs(float(loss) - float(g["total_loss"])) <= 2e-4 * abs(float(g["total_loss"]))
    loss.backward()
    keys = g["grad_keys"].tolist()
    assert set(keys) == {k for k, t in o.P.items() if t.grad is not None}
    worst = max(abs(float(o.P[k].grad.norm()) - l2) / (l2 + 1e-6) for k, l2 in zip(keys, g["grad_l2"].tolist()))
    assert worst < KINK_GRAD, f"worst relative gradient-norm error {worst:.2e}"
    n = 0
    for f in g.files:
        if f.startswith(("g:head.cls_preds", "g:head.reg_preds", "g:head.obj_preds")) and f.endswith(".bias"):
            ref = torch.from_numpy(g[f])
            assert torch.allclose(o.P[f[2:]].grad, ref, rtol=2e-3, atol=2e-5 * float(ref.abs().max()) + 1e-7), f
            n += 1
    assert n == 9


def test_fixtures_differ_between_activations():
    """the three fixtures pin three different networks (a silently ignored ``act`` would give identical losses)"""
    losses = [np.load(os.path.join(GOLD, n + ".npz"))["train_loss"] for n in ["tiny_120x160"] + list(ACT_CASES)]
    assert all(np.abs(a[:5] - b[:5]).max() > 1e-2 for i, a in enumerate(losses) for b in losses[i + 1:])


# ================================================================================================ CPU: emulated product
def _grad_report(model, o):
    report = []
    for k, p in model.named_parameters():
        assert p.grad is not None and torch.isfinite(p.grad).all(), f"no finite gradient reached {k}"
        g, r = p.grad.float().flatten(), o.P[k].grad.float().flatten()
        report.append((float((g - r).norm() / (r.norm() + 1e-12)), float(torch.dot(g, r) / (g.norm() * r.norm() + 1e-20)), k))
    report.sort(reverse=True)
    return report


def _check_grads(report):
    msg = "largest deviations:\n" + "\n".join(f"{r:8.3e} cos {c_:.5f} {k}" for r, c_, k in report[:10])
    assert report[len(report) // 2][0] < KINK_PRODUCT_GRAD and min(c_ for _, c_, _ in report) > 0.99, msg


@pytest.mark.parametrize("act", ACTS)
def test_emulated_train_step_equals_oracle_autograd(act, monkeypatch):
    """the recording forward + backward walk with fp32 storage against autograd through the fp32 oracle: losses within
    2e-5, every parameter gradient within 1e-3, the BatchNorm buffers; the gradient arena starts as NaN"""
    emul_act.install(monkeypatch, exact=True)
    monkeypatch.setattr(backward, "POISON", True)
    c = TINY
    x = synth.synth_frames(c["B"], c["H"], c["W"])
    tg = synth.synth_labels(c["B"], c["H"], c["W"])
    model = build(c, act)
    acts = []
    real = ops.bn_act_apply
    monkeypatch.setattr(ops, "bn_act_apply", lambda *a, **k: (acts.append(a[4]), real(*a, **k))[1])
    loss = backward.forward_backward(model, x, tg)
    assert set(acts) == {CODES[act]}
    o = oracle(c, act, grads=True)
    ref = o.forward(x, tg)
    ref["total_loss"].backward()
    for k in LOSSES:
        got, want = (float(t.detach()) if torch.is_tensor(t) else float(t) for t in (loss[k], ref[k]))
        assert abs(got - want) <= KINK_LOSS * abs(want) + 1e-6, k
    _check_grads(_grad_report(model, o))
    sd = model.state_dict()
    for k in ("backbone.backbone.stem.conv.bn.running_mean", "backbone.C3_n4.conv3.bn.running_var", "backbone.jian1.bn.running_var"):
        assert torch.allclose(sd[k], o.P[k].detach(), rtol=1e-3, atol=1e-5), k


@pytest.mark.parametrize("act", ACTS)
def test_emulated_eval_and_on_pipe_equal_oracle(act, monkeypatch):
    emul_act.install(monkeypatch, exact=True)
    c = TINY
    x = synth.synth_frames(c["B"], c["H"], c["W"])
    tg = synth.synth_labels(c["B"], c["H"], c["W"])
    xc = torch.cat([x[:, 0:3], x[:, 0:3]], 1)
    o = oracle(c, act, momentum=1.0)
    o.forward(xc, tg)
    o.training = False
    m = YOLOX(DFPPAFPN(c["depth"], c["width"], in_channels=CH, act=act), TALHead(8, c["width"], in_channels=CH, act=act))
    for mod in m.modules():
        if isinstance(mod, torch.nn.BatchNorm2d):
            mod.eps = 1e-3
    m.load_state_dict({k: v.detach().clone() for k, v in o.P.items()}, strict=True)
    m.eval()
    with torch.no_grad():
        got, want = m(xc), o.forward(xc)
        assert rel_l2(got, want) < KINK_REL, rel_l2(got, want)
        g1, gb = m(x[:1, 0:3], mode="on_pipe")
        g2, gb2 = m(x[1:2, 0:3], buffer=gb, mode="on_pipe")
        r1, rb = o.forward(x[:1, 0:3], mode="on_pipe")
        r2, rb2 = o.forward(x[1:2, 0:3], buffer=rb, mode="on_pipe")
    for a, b in [(g1, r1), (g2, r2)] + list(zip(gb2, rb2)):
        assert rel_l2(a, b) < KINK_REL, rel_l2(a, b)


@pytest.mark.parametrize("act", ACTS)
def test_emulated_still_step_equals_duplicated_pair_oracle(act, monkeypatch):
    """the still model (PIPEHead on single frames, one backbone pass with two running updates) against the oracle on the
    duplicated pair"""
    from test_still_train import install
    install(monkeypatch)
    emul_act.wrap(monkeypatch)
    monkeypatch.setattr(backward, "POISON", True)
    c = TINY
    x = synth.synth_frames(c["B"], c["H"], c["W"])[:, :3].contiguous()
    labels, _ = synth.synth_labels(c["B"], c["H"], c["W"])
    model = build(c, act, head=PIPEHead)
    out = model(x, labels)
    out["total_loss"].backward()
    o = oracle(c, act, gamma=0.0, grads=True)
    o.cfg.ignore_thr, o.cfg.ignore_value = 0.0, 1.0
    ref = o.forward(torch.cat([x, x], 1), (labels, labels))
    ref["total_loss"].backward()
    for k in LOSSES:
        got, want = (float(t.detach()) if torch.is_tensor(t) else float(t) for t in (out[k], ref[k]))
        assert abs(got - want) <= KINK_LOSS * abs(want) + 1e-6, k
    _check_grads(_grad_report(model, o))


@pytest.mark.parametrize("act", ACTS)
def test_emulated_trainer_step_matches_stock_pytorch_step(act, monkeypatch):
    emul_act.install(monkeypatch, exact=True)
    c = TINY
    x = synth.synth_frames(c["B"], c["H"], c["W"])
    tg = synth.synth_labels(c["B"], c["H"], c["W"])
    ref = build(c, act)
    opt = train.build_optimizer(ref, lr=2e-4)
    ema = train.ModelEMA(ref)
    model = build(c, act)
    tr = train.Trainer(model, lr=2e-4)
    wants = [train.train_step(ref, opt, x, tg, ema) for _ in range(2)]
    for want in wants:
        got = tr.step(x, tg)
        assert abs(float(got["total_loss"]) - float(want["total_loss"])) <= 1e-5 * abs(float(want["total_loss"]))
    for (k, p), q in zip(model.named_parameters(), ref.parameters()):
        assert torch.allclose(p, q, rtol=1e-5, atol=1e-7), k
    esd, rsd = tr.ema_state_dict(), ema.ema.state_dict()
    for k in rsd:
        if rsd[k].dtype.is_floating_point:
            assert torch.allclose(esd[k], rsd[k], rtol=1e-5, atol=1e-7), k


def test_mixed_activations_run_and_match_per_module(monkeypatch):
    """a network whose modules mix activations (SPP's ``activation=`` is its own argument; here also one head tower pair
    with different activations, which then takes two launches): every BaseConv launch carries its own module's code"""
    emul_act.install(monkeypatch, exact=True)
    c = TINY
    m = build(c, "silu")
    m.backbone.backbone.dark5[1].conv1.act_name = "relu"
    m.backbone.backbone.dark5[1].conv2.act_name = "lrelu"
    m.head.reg_convs[0][0].act_name = "relu"
    seen = Counter()
    real = ops.bn_act_apply
    monkeypatch.setattr(ops, "bn_act_apply", lambda *a, **k: (seen.update([a[4]]), real(*a, **k))[1])
    x = synth.synth_frames(c["B"], c["H"], c["W"])
    tg = synth.synth_labels(c["B"], c["H"], c["W"])
    backward.forward_backward(m, x, tg)
    assert seen[ops.SY_ACT_RELU] == 2 and seen[ops.SY_ACT_LRELU] == 1, seen
    for p in m.parameters():
        assert p.grad is not None and torch.isfinite(p.grad).all()


# ================================================================================================ GPU: kernels
DEV = "cuda"
F64 = torch.float64
GPU_CODES = [ops.SY_ACT_RELU, ops.SY_ACT_LRELU]
# values at and around z = 0 (exact in bf16 and fp16): +0, -0, the smallest fp16 subnormal, a few ulp either side of 0
SPECIALS = [0.0, -0.0, 2.0 ** -24, -(2.0 ** -24), 3 * 2.0 ** -24, -3 * 2.0 ** -24, 2.0 ** -14, -(2.0 ** -14), 1e-3, -1e-3]


def _gen(seed):
    return torch.Generator(device=DEV).manual_seed(seed)


def _nchw64(v):
    return v.torch().permute(0, 3, 1, 2).to(F64)


def _act32(t, code):
    """the kernel's fp32 expression on fp32 ``t`` (v > 0 ? v : 0 | v * 0.1f), for bit comparisons"""
    if code == ops.SY_ACT_RELU:
        return torch.where(t > 0, t, torch.zeros_like(t))
    return torch.where(t > 0, t, t * torch.tensor(0.1, dtype=torch.float32, device=t.device))


def _check_specials(got, want, code, what):
    """the special channels: the value of one rounding of the kernel's fp32 expression (a folded scale of 0 gives z = +0 or
    -0 depending on the accumulator's sign, so zeros are compared by value), and ReLU never writes -0"""
    assert torch.equal(got.float(), want.float()), f"{what}: z at and around 0"
    if code == ops.SY_ACT_RELU:
        assert not bool((got.view(torch.int16) == -32768).any()), f"{what}: ReLU wrote -0"


def _special_block(shape, dtype):
    """NHWC tensor whose channels 0..len(SPECIALS)-1 hold the special values at every pixel"""
    t = torch.zeros(shape, dtype=torch.float32, device=DEV)
    for i, v in enumerate(SPECIALS):
        t[..., i] = v
    return t.to(dtype)


@pytest.mark.gpu
def test_gpu_unknown_act_codes_refused():
    from test_gpu_ops import rand_w
    v = ops.View(torch.zeros((1, 8, 8, 64), dtype=torch.bfloat16, device=DEV))
    y = ops.View(torch.zeros((1, 8, 8, 64), dtype=torch.bfloat16, device=DEV))
    one, zero = torch.ones(2 * 64, device=DEV), torch.zeros(2 * 64, device=DEV)
    wpk = ops.pack_conv_weight(rand_w(64, 64, 1, 1))
    dw = ops.pack_dw_weight(torch.randn(64, 1, 3, 3, device=DEV))
    for bad in (4, -1, 99):
        for impl, w in (("tc", wpk), ("simt", wpk), ("dw", dw)):
            with pytest.raises(RuntimeError, match="act"):
                ops.conv2d(v, w, y, 1 if impl != "dw" else 3, 1, ops.SY_CONV_FUSED, impl=impl, scale=one[:64], shift=zero[:64],
                           act=bad)
        with pytest.raises(RuntimeError, match="act"):
            ops.bn_act_apply(v, one, zero, 1, bad, None, y)
        dg, db = torch.zeros(64, device=DEV), torch.zeros(64, device=DEV)
        ss = torch.ones((2, 64), device=DEV)
        with pytest.raises(RuntimeError, match="act"):
            ops.bn_act_backward(v, v, y, ss, ss, ss, ss, 0, bad, dg, db)
    torch.cuda.synchronize()


@pytest.mark.gpu
@pytest.mark.parametrize("res", [False, True], ids=["plain", "res"])
@pytest.mark.parametrize("split", [0, 3], ids=["one_group", "two_groups"])
@pytest.mark.parametrize("code", GPU_CODES, ids=["relu", "lrelu"])
def test_gpu_bn_act_apply(code, split, res):
    from test_gpu_ops import check_close
    n, h, w, c = 6, 19, 30, 96
    g = _gen(1)
    xb = (torch.randn((n, h, w, c), generator=g, device=DEV) * 2).to(torch.bfloat16)
    xb[..., :len(SPECIALS)] = _special_block((n, h, w, c), torch.bfloat16)[..., :len(SPECIALS)]
    x = ops.View(xb)
    scale = torch.rand((2, c), generator=g, device=DEV) + 0.5
    shift = torch.rand((2, c), generator=g, device=DEV) - 0.5
    scale[:, :len(SPECIALS)], shift[:, :len(SPECIALS)] = 1.0, -0.0          # z = x * 1 + (-0) = x exactly, -0 included
    r = ops.View(torch.randn((n, h, w, c), generator=g, device=DEV).to(torch.bfloat16)) if res else None
    y = ops.View.empty(n, h, w, c, DEV)
    ops.bn_act_apply(x, scale, shift, split or n, code, r, y)
    torch.cuda.synchronize()
    gi = torch.zeros(n, dtype=torch.long, device=DEV)
    if split:
        gi[split:] = 1
    sc, sh = scale.to(F64)[gi][:, :, None, None], shift.to(F64)[gi][:, :, None, None]
    z = _nchw64(x) * sc + sh
    ref = act64(z, code) + (_nchw64(r) if res else 0)
    got = _nchw64(y)
    check_close(got[:, len(SPECIALS):], ref[:, len(SPECIALS):], f"bn_act_apply act={code}")
    # the special channels bit for bit: z = x, one bf16 rounding of the fp32 expression (+ residual)
    z32 = x.torch()[..., :len(SPECIALS)].float()
    want = _act32(z32, code)
    if res:
        want = want + r.torch()[..., :len(SPECIALS)].float()
    assert torch.equal(y.torch()[..., :len(SPECIALS)].view(torch.int16), want.to(torch.bfloat16).view(torch.int16))


def _fused_ref(x64, w64, s, sc, sh, code, r64):
    kh, kw = w64.shape[2], w64.shape[3]
    t = F.conv2d(x64, w64, None, s, ((kh - 1) // 2, (kw - 1) // 2)) * sc[None, :, None, None] + sh[None, :, None, None]
    return act64(t, code) + (r64 if r64 is not None else 0)


def _zero_channels(scale, shift, n_special):
    """channels whose folded scale is 0: z = 0 * acc + shift = +-0 or +-tiny exactly"""
    vals = torch.tensor(SPECIALS, dtype=torch.float32, device=DEV)
    scale[:n_special], shift[:n_special] = 0.0, vals[:n_special]


@pytest.mark.gpu
@pytest.mark.parametrize("tiling", [(1, 64), (1, 128), (2, 64), (2, 128)], ids=lambda t: f"mode{t[0]}_bn{t[1]}")
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16], ids=["bf16", "fp16"])
@pytest.mark.parametrize("code", GPU_CODES, ids=["relu", "lrelu"])
def test_gpu_conv_tc_fused(code, dtype, tiling):
    from test_gpu_ops import check_close, rand_w
    tile_mode, tile_bn = tiling
    n, h, w, ci, co, k = 2, 38, 60, 64, 256, 3
    plan = ops.conv2d_plan(n, h, w, ci, co, k, 1, tile_mode=tile_mode, tile_bn=tile_bn)
    assert (plan["mode"], plan["bn"]) == tiling
    g = _gen(2)
    xv = ops.View(torch.randn((n, h, w, ci), generator=g, device=DEV).to(dtype))
    wt = rand_w(co, ci, k, 3)
    wpk = ops.pack_conv_weight(wt, dtype=dtype)
    scale = torch.rand(co, generator=g, device=DEV) + 0.5
    shift = torch.rand(co, generator=g, device=DEV) - 0.5
    _zero_channels(scale, shift, len(SPECIALS))
    rb = torch.randn((n, h, w, co), generator=g, device=DEV).to(dtype)
    for res in (None, ops.View(rb)):
        y = ops.View.empty(n, h, w, co, DEV, dtype) if dtype == torch.float16 else ops.View.empty(n, h, w, co, DEV)
        ops.conv2d(xv, wpk, y, k, 1, ops.SY_CONV_FUSED, scale=scale, shift=shift, act=code, res=res,
                   tile_mode=tile_mode, tile_bn=tile_bn)
        torch.cuda.synchronize()
        r64 = _nchw64(res) if res is not None else None
        ref = _fused_ref(_nchw64(xv), wt.to(dtype).to(F64), 1, scale.to(F64), shift.to(F64), code, r64)
        got = _nchw64(y)
        check_close(got, ref, f"conv_tc FUSED act={code} {dtype} {tiling}", ulp=2.0 ** -7 if dtype == torch.bfloat16 else 2.0 ** -10)
        sp = _act32(torch.tensor(SPECIALS, device=DEV), code)[None, :, None, None]
        want = sp + (r64[:, :len(SPECIALS)].float() if res is not None else 0)
        _check_specials(y.torch()[..., :len(SPECIALS)], want.expand(n, -1, h, w).permute(0, 2, 3, 1).to(dtype), code,
                        f"conv_tc {dtype} {tiling}")


@pytest.mark.gpu
@pytest.mark.parametrize("code", GPU_CODES, ids=["relu", "lrelu"])
def test_gpu_conv_tc_fused_linear_1x1(code):
    """the 1x1 (linear-tile) FUSED path, with a residual read from a slice of another buffer and the output written into a
    channel slice (the DFP jian launches)"""
    from test_gpu_ops import check_close, rand_w
    n, h, w, ci, co = 2, 75, 120, 128, 64
    g = _gen(4)
    xv = ops.View(torch.randn((n, h, w, ci), generator=g, device=DEV).to(torch.bfloat16))
    wt = rand_w(co, ci, 1, 5)
    wpk = ops.pack_conv_weight(wt)
    scale, shift = torch.rand(co, generator=g, device=DEV) + 0.5, torch.rand(co, generator=g, device=DEV) - 0.5
    out = ops.View.empty(n, h, w, 2 * co, DEV)
    ops.conv2d(xv, wpk, out.ch(co, co), 1, 1, ops.SY_CONV_FUSED, scale=scale, shift=shift, act=code, res=xv.ch(co, co))
    torch.cuda.synchronize()
    ref = _fused_ref(_nchw64(xv), wt.to(F64), 1, scale.to(F64), shift.to(F64), code, _nchw64(xv.ch(co, co)))
    check_close(_nchw64(out.ch(co, co)), ref, f"conv_tc 1x1 act={code}")


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16], ids=["bf16", "fp16"])
@pytest.mark.parametrize("k,stride", [(1, 1), (3, 1), (3, 2), (5, 1), (5, 2)])
@pytest.mark.parametrize("code", GPU_CODES, ids=["relu", "lrelu"])
def test_gpu_dwconv_fused(code, k, stride, dtype):
    from test_gpu_ops import check_close
    n, h, w, c = 2, 19, 31, 48
    g = _gen(5)
    xv = ops.View(torch.randn((n, h, w, c), generator=g, device=DEV).to(dtype))
    wt = torch.randn((c, 1, k, k), generator=g, device=DEV) / k
    wpk = ops.pack_dw_weight(wt, dtype=dtype)
    ho, wo = ops.conv_out_hw(h, w, k, stride)
    scale, shift = torch.rand(c, generator=g, device=DEV) + 0.5, torch.rand(c, generator=g, device=DEV) - 0.5
    _zero_channels(scale, shift, len(SPECIALS))
    res = ops.View(torch.randn((n, ho, wo, c), generator=g, device=DEV).to(dtype))
    y = ops.View.empty(n, ho, wo, c, DEV, dtype) if dtype == torch.float16 else ops.View.empty(n, ho, wo, c, DEV)
    ops.conv2d(xv, wpk, y, k, stride, ops.SY_CONV_FUSED, impl="dw", scale=scale, shift=shift, act=code, res=res)
    torch.cuda.synchronize()
    ref = F.conv2d(_nchw64(xv), wt.to(dtype).to(F64), None, stride, (k - 1) // 2, groups=c)
    ref = act64(ref * scale.to(F64)[None, :, None, None] + shift.to(F64)[None, :, None, None], code) + _nchw64(res)
    check_close(_nchw64(y), ref, f"dwconv act={code}", ulp=2.0 ** -7 if dtype == torch.bfloat16 else 2.0 ** -10)
    sp = _act32(torch.tensor(SPECIALS, device=DEV), code)[None, None, None, :]
    want = (sp + res.torch()[..., :len(SPECIALS)].float()).to(dtype)
    _check_specials(y.torch()[..., :len(SPECIALS)], want, code, f"dwconv k={k} s={stride} {dtype}")


@pytest.mark.gpu
@pytest.mark.parametrize("code", GPU_CODES, ids=["relu", "lrelu"])
def test_gpu_conv_simt_fused(code):
    from test_gpu_ops import check_close, rand_w
    n, h, w, ci, co, k, s = 2, 19, 30, 64, 64, 3, 2
    g = _gen(6)
    xv = ops.View(torch.randn((n, h, w, ci), generator=g, device=DEV).to(torch.bfloat16))
    wt = rand_w(co, ci, k, 7)
    wpk = ops.pack_conv_weight(wt)
    scale, shift = torch.rand(co, generator=g, device=DEV) + 0.5, torch.rand(co, generator=g, device=DEV) - 0.5
    _zero_channels(scale, shift, len(SPECIALS))
    ho, wo = ops.conv_out_hw(h, w, k, s)
    y = ops.View.empty(n, ho, wo, co, DEV)
    ops.conv2d(xv, wpk, y, k, s, ops.SY_CONV_FUSED, impl="simt", scale=scale, shift=shift, act=code)
    torch.cuda.synchronize()
    ref = _fused_ref(_nchw64(xv), wt.to(F64), s, scale.to(F64), shift.to(F64), code, None)
    check_close(_nchw64(y), ref, f"conv_simt act={code}")
    sp = _act32(torch.tensor(SPECIALS, device=DEV), code).to(torch.bfloat16)
    _check_specials(y.torch()[..., :len(SPECIALS)], sp.expand(n, ho, wo, -1), code, "conv_simt")


def bn_act_backward_ref(raw, gy, ss, mi, groups, code):
    """tests/test_gpu_parity_bwd.py's float64 reference with the derivative of an SY_ACT_* code"""
    c = raw.shape[1]
    draw = torch.empty_like(raw)
    dg, db, s2g, s2b = (torch.zeros(c, dtype=F64, device=raw.device) for _ in range(4))
    dz_all, t_all = torch.empty_like(raw), torch.empty_like(raw)
    for a, b, g in groups:
        sc, sh, mu, iv = (t.double()[None, :, None, None] for t in (ss[0, g], ss[1, g], mi[0, g], mi[1, g]))
        z = raw[a:b] * sc + sh
        dz = gy[a:b] * dact64(z, code)
        xh = (raw[a:b] - mu) * iv
        t = dz * xh
        draw[a:b] = sc * (dz - dz.mean((0, 2, 3), keepdim=True) - xh * t.mean((0, 2, 3), keepdim=True))
        dg += t.sum((0, 2, 3))
        db += dz.sum((0, 2, 3))
        s2g += t.pow(2).sum((0, 2, 3))
        s2b += dz.pow(2).sum((0, 2, 3))
        dz_all[a:b], t_all[a:b] = dz, t
    return draw, dg, db, s2g, s2b, t_all, dz_all


@pytest.mark.gpu
@pytest.mark.parametrize("case", [(16, 64, 150, 240, 8, False), (16, 192, 38, 60, 8, True), (8, 1024, 19, 30, 0, False)],
                         ids=lambda c: "x".join(map(str, c)))
@pytest.mark.parametrize("code", GPU_CODES, ids=["relu", "lrelu"])
def test_gpu_bn_act_backward(code, case):
    """reduce, finalize and apply of sy_bn_act_backward against float64 (the bars of test_gpu_parity_bwd.py), and the
    reference formula against autograd of F.batch_norm + the activation"""
    from test_gpu_ops import check_close
    from test_gpu_parity_bwd import check_sum, small_grad
    n, c, h, w, split, acc = case
    eps = 1e-3
    g = _gen(7)
    mu = torch.rand(c, generator=g, device=DEV) * 4.0 - 2.0
    sd = torch.rand(c, generator=g, device=DEV) + 0.5
    rawv = ops.View((torch.randn((n, h, w, c), generator=g, device=DEV) * sd + mu).to(torch.bfloat16))
    dyv = small_grad(n, h, w, c, 8)
    raw64, dy64 = _nchw64(rawv), _nchw64(dyv)
    gamma, beta = torch.rand(c, generator=g, device=DEV) + 0.5, torch.rand(c, generator=g, device=DEV) - 0.5
    groups = [(0, split, 0), (split, n, 1)] if split else [(0, n, 0)]
    mean, invstd = torch.zeros((2, c), device=DEV), torch.ones((2, c), device=DEV)
    for a, b, gi in groups:
        mean[gi] = raw64[a:b].mean((0, 2, 3)).float()
        invstd[gi] = (raw64[a:b].var((0, 2, 3), unbiased=False) + eps).rsqrt().float()
    scale = gamma[None] * invstd
    shift = beta[None] - mean * scale
    d0 = torch.randn((2, c), generator=g, device=DEV) if acc else torch.full((2, c), float("nan"), device=DEV)
    dgamma, dbeta = d0[0].clone(), d0[1].clone()
    draw = ops.View.empty(n, h, w, c, DEV)
    ops.bn_act_backward(rawv, dyv, draw, scale, shift, mean, invstd, split, code, dgamma, dbeta, accumulate=acc)
    torch.cuda.synchronize()
    ss, mi = torch.stack([scale, shift]), torch.stack([mean, invstd])
    draw_ref, dg, db, s2g, s2b, _, _ = bn_act_backward_ref(raw64, dy64, ss, mi, groups, code)
    if acc:
        dg, db = dg + d0[0].double(), db + d0[1].double()
    check_close(_nchw64(draw), draw_ref, f"bn backward act={code}: d raw")
    K = n * h * w
    check_sum(dgamma, dg, s2g, K, f"bn backward act={code}: dgamma")
    check_sum(dbeta, db, s2b, K, f"bn backward act={code}: dbeta")
    a, b, _ = groups[0]
    xr = raw64[a:b].clone().requires_grad_(True)
    gr, br = gamma.double().requires_grad_(True), beta.double().requires_grad_(True)
    act64(F.batch_norm(xr, None, None, gr, br, True, 0.0, eps), code).backward(dy64[a:b])
    m64, v64 = raw64[a:b].mean((0, 2, 3)), raw64[a:b].var((0, 2, 3), unbiased=False)
    iv64 = (v64 + eps).rsqrt()
    ss64 = torch.stack([gamma.double() * iv64, beta.double() - m64 * gamma.double() * iv64])[:, None]
    d_ex, dg_ex, db_ex, _, _, _, _ = bn_act_backward_ref(raw64[a:b], dy64[a:b], ss64, torch.stack([m64, iv64])[:, None],
                                                        [(0, b - a, 0)], code)
    assert torch.allclose(d_ex, xr.grad, rtol=1e-9, atol=1e-12 * float(xr.grad.abs().max()))
    assert torch.allclose(db_ex, br.grad, rtol=1e-9, atol=1e-9 * float(br.grad.abs().max()))


@pytest.mark.gpu
@pytest.mark.parametrize("code", GPU_CODES, ids=["relu", "lrelu"])
def test_gpu_bn_act_backward_derivative_at_zero(code):
    """scale 1, shift 0: z = raw exactly.  Channel i holds SPECIALS[i] at every pixel, dy = 1: dbeta = sum act'(z) counts
    the derivative convention (z = +-0: 0 for ReLU, 0.1 for LeakyReLU), and the pass-through draw (mean 0, invstd 1) is 0"""
    n, h, w, c = 4, 19, 30, 16
    raw = ops.View(_special_block((n, h, w, c), torch.bfloat16))
    dy = ops.View(torch.ones((n, h, w, c), dtype=torch.bfloat16, device=DEV))
    one, zero = torch.ones((2, c), device=DEV), torch.zeros((2, c), device=DEV)
    dgamma, dbeta = torch.zeros(c, device=DEV), torch.zeros(c, device=DEV)
    draw = ops.View.empty(n, h, w, c, DEV)
    ops.bn_act_backward(raw, dy, draw, one, zero, zero, one, 0, code, dgamma, dbeta)
    torch.cuda.synchronize()
    z = raw.torch()[0, 0, 0].double()
    slope = 0.0 if code == ops.SY_ACT_RELU else 0.1
    want = torch.where(z > 0, 1.0, slope).double() * (n * h * w)
    assert torch.allclose(dbeta.double(), want, rtol=1e-5, atol=0), (dbeta, want)       # fp32 partial sums of 0.1f
    assert bool((draw.torch().float().abs() <= 1e-6).all())


# ================================================================================================ GPU: StreamYOLO-s
S = dict(depth=0.33, width=0.50, H=192, W=320, B=2, gamma=1.0, thr=0.5, val=1.5, empty=-1)


def _ulp_check(got, ref, what, allowed=0):
    got, ref = got.float().cpu(), ref.float().cpu()
    rms = ref.pow(2).mean().sqrt().item() + 1e-12
    err = (got - ref).abs()
    bad = err > (2.0 ** -6) * ref.abs() + (2.0 ** -6) * rms
    r = ((got - ref).norm() / (ref.norm() + 1e-12)).item()
    assert int(bad.sum()) <= allowed and r < 4e-3, f"{what}: {int(bad.sum())}/{bad.numel()} beyond 2 ulp, rel l2 {r:.2e}"


@pytest.mark.gpu
@pytest.mark.parametrize("impl", ["tc", "simt"])
@pytest.mark.parametrize("mode", ["train", "eval"])
@pytest.mark.parametrize("act", ACTS)
def test_gpu_every_layer_teacher_forced(act, mode, impl, monkeypatch):
    """each BaseConv of StreamYOLO-s fed the oracle's own input / residual reproduces the oracle's stored output within 2 bf16
    ulp and a relative L2 error of 4e-3 (DESIGN.md section 2, item 1); the stem and the DFP fusion as blocks.  Train mode
    admits one element per layer beyond 2 ulp: SPP conv2 normalises with the statistics of 120 pixels per group at this
    size, and one pre-activation within the statistics' fp32 noise of 0 lands on the other side of the kink (measured on an
    H100: 1 of 61 440 elements, relative L2 error 1e-4 to 3e-4)."""
    monkeypatch.setattr(engine, "CONV_IMPL", impl)
    c = S
    x = synth.synth_frames(c["B"], c["H"], c["W"])
    tg = synth.synth_labels(c["B"], c["H"], c["W"])
    train_ = mode == "train"
    o = oracle(c, act, q=bf16_round)
    o.training = train_
    o.trace = {}
    o.forward(x, tg) if train_ else o.forward(x)
    tr = o.trace
    m = build(c, act, device=DEV)
    m.train(train_)
    dev = torch.device(DEV)
    n_checked = 0
    for name, mod in m.named_modules():
        if not isinstance(mod, BaseConv) or name + ".in" not in tr or name.endswith("stem.conv") or ".jian" in name:
            continue
        xin = ops.from_nchw(tr[name + ".in"].to(dev))
        res = ops.from_nchw(tr[name + ".res"].to(dev)) if name + ".res" in tr else None
        with torch.no_grad():
            y = engine.base_conv(engine.Ctx(train_, xin.n, xin.n, dev), mod, xin, res=res)
        torch.cuda.synchronize()
        _ulp_check(y.nchw_float(), tr[name + ".out"], name, allowed=1 if train_ else 0)
        n_checked += 1
    assert n_checked == 77 - 1 - 3
    with torch.no_grad():
        y = engine.focus_stem(engine.Ctx(train_, c["B"], c["B"], dev), m.backbone.backbone.stem, x[:, 3:6].contiguous().cuda(), 1)
    _ulp_check(y.nchw_float(), tr["backbone.backbone.stem.conv.out"], "stem")
    o2 = oracle(c, act, q=bf16_round)
    o2.training = train_
    xq = o2.q(x)
    cur, sup = o2.pafpn(xq[:, 0:3]), o2.pafpn(xq[:, 3:6])
    fused = o2._fuse(cur, sup)
    with torch.no_grad():
        both = [ops.from_nchw(torch.cat([a, b], 0).to(dev)) for a, b in zip(cur, sup)]
        got = engine.dfp_fuse(engine.Ctx(train_, 2 * c["B"], c["B"], dev), m.backbone,
                              tuple(v.imgs(0, c["B"]) for v in both), tuple(v.imgs(c["B"], c["B"]) for v in both))
    for g_, f_, nm in zip(got, fused, ("jian2", "jian1", "jian0")):
        _ulp_check(g_.nchw_float(), f_, "dfp " + nm)


@pytest.mark.gpu
@pytest.mark.parametrize("act", ACTS)
def test_gpu_walk_in_situ_every_conv_backward(act, monkeypatch):
    """tests/test_gpu_parity_bwd.py's in-situ checker of every recorded conv launch of the backward walk, with this
    activation's derivative in its float64 reference"""
    import test_gpu_parity_bwd as P
    monkeypatch.setattr(P, "bn_act_backward_ref", bn_act_backward_ref)
    m = build(S, act, device=DEV)
    x = synth.synth_frames(S["B"], S["H"], S["W"]).cuda()
    tg = tuple(t.cuda() for t in synth.synth_labels(S["B"], S["H"], S["W"]))
    acts = set()
    real = backward.ops.bn_act_backward
    monkeypatch.setattr(ops, "bn_act_backward", lambda *a, **k: (acts.add(a[8]), real(*a, **k))[1])
    seen = P.run_walk_checked(m, x, tg)
    assert len(seen) == 77 - 8 - 3 + 3 - 1, len(seen)
    assert acts == {CODES[act]}


@pytest.mark.gpu
@pytest.mark.parametrize("act", ACTS)
def test_gpu_trainer_graph_replay_equals_eager_steps(act):
    x = synth.synth_frames(S["B"], S["H"], S["W"]).cuda()
    tg = tuple(t.cuda() for t in synth.synth_labels(S["B"], S["H"], S["W"]))
    a = build(S, act, device=DEV)
    ta = train.Trainer(a, lr=2e-4)
    lrs = [2e-4, 1.5e-4, 1e-4]
    want = [float(ta.step(x, tg, lr=lr)["total_loss"]) for lr in lrs]
    b = build(S, act, device=DEV)
    tb = train.Trainer(b, lr=lrs[0])
    tb.capture(x.clone(), tuple(t.clone() for t in tg))
    got = [float(tb.replay(lr=lr)["total_loss"]) for lr in lrs[1:]]
    torch.cuda.synchronize()
    assert np.isfinite(want).all() and got == want[1:], (got, want)
    assert torch.equal(ta.fs.state, tb.fs.state) and torch.equal(ta.fs.ema, tb.fs.ema) and torch.equal(ta.fs.mom, tb.fs.mom)


def _calibrated_s(act, x):
    m = build(dict(S, H=x.shape[2], W=x.shape[3]), act, momentum=1.0, device=DEV)
    engine.name_modules(m)
    fut, cur = synth.synth_labels(x.shape[0], x.shape[2], x.shape[3], seed=11)
    with torch.no_grad():
        m(x, (fut.cuda(), cur.cuda()))
    return m.eval()


@pytest.mark.gpu
@pytest.mark.parametrize("act", ACTS)
def test_gpu_f16_eval_every_launch(act, monkeypatch):
    """the fp16-storage eval forward of StreamYOLO-s at 600x960, every launch against float64 with the bars of
    tests/test_fp16_storage.py (its checker, with this activation in the references)"""
    import test_gpu_parity_fwd as P
    from test_fp16_storage import make_f16_checker
    fn = {"relu": F.relu, "lrelu": lambda t: F.leaky_relu(t, 0.1)}[act]
    monkeypatch.setattr(P, "F", SimpleNamespace(**{**vars(F), "silu": fn}))
    monkeypatch.setattr(P.FwdChecker, "_act", staticmethod(lambda mods: 1))
    x = synth.synth_frames(2, 600, 960, seed=99).cuda()
    m = _calibrated_s(act, x)
    m.activation_dtype = torch.float16
    with torch.no_grad():
        m(x)
        with make_f16_checker(m, nondegenerate=False) as ck:
            out = m(x)
    assert ck.n == Counter(conv=P.conv_launches(m, jian_twice=True), head=3, focus=1), ck.n
    assert bool(torch.isfinite(out).all())


@pytest.mark.gpu
@pytest.mark.parametrize("act", ACTS)
def test_gpu_stream_detector_bit_identical_to_driver_loop(act):
    from streamyolo_b200 import data, stream
    from test_stream import CONF, NMS, driver_inference, same_dets, uint8_frames
    m = _calibrated_s(act, synth.synth_frames(2, 600, 960, seed=99).cuda())
    frame_hw, in_scale, size = (1200, 1920), 0.5, (600, 960)
    det = stream.StreamDetector(m, frame_hw=frame_hw, in_scale=in_scale, streams=1, conf_thre=CONF, nms_thre=NMS)
    frames = uint8_frames(5, *frame_hw, seed=31)
    buffer = None
    for i in range(5):
        if i in (0, 3):
            det.reset()
            buffer = None
        with torch.no_grad():
            xi = data.stream_frame(frames[i].cuda(), size)
            result, buffer = m(xi, buffer=buffer, mode="on_pipe")
            want = driver_inference(result[0].cpu(), m.head.num_classes, in_scale)
        got = det.step(frames[i].numpy())
        assert torch.equal(det.last_raw(), result), f"frame {i}: raw head outputs"
        assert same_dets(got[0], want), f"frame {i}: detections"
