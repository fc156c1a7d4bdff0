"""GPU: the product model (streamyolo_b200.model, CUDA kernels through the C ABI) against the CPU
oracle on identical synthetic weights / frames / labels, and against the reference-generated
golden fixtures.

Tolerances
  * per layer, IDENTICAL inputs (teacher forced from the oracle's trace): every stored element within
    2 bf16 ulp (2^-6 relative) and ||a-b||/||b|| <= 4e-3 -- this is the parity bar proper.
  * end to end, train mode: bf16 storage makes a random-init batch-norm network chaotic -- two runs of
    the SAME oracle code whose inputs differ by 1e-6 relative drift 8-18 % apart in the fused features
    (measured; see DESIGN.md).  The product must be indistinguishable from that rounding noise:
    err(product, oracle_q) <= 1.5 x err(oracle_q, oracle_q on inputs * (1+1e-6)) + 1e-2; losses 5e-2.
  * SimOTA/TAL given IDENTICAL fp32 head outputs: foreground set, matched GT ids bit exact,
    matched IoUs / loss values 1e-4 (north_star: integer indexing bit-exact).
  * golden fixtures (reference in fp32): losses within 5e-2 relative (bf16 activations vs fp32).
"""
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from oracle.make_golden import CASES  # noqa: E402
from oracle.streamyolo_oracle import OracleCfg, StreamYoloOracle, bf16_round, model_shapes  # noqa: E402
from streamyolo_b200 import ops, synth  # noqa: E402
from streamyolo_b200.model import DFPPAFPN, TALHead, YOLOX, engine  # noqa: E402

GOLD = os.path.join(os.path.dirname(__file__), "golden")
ORDER = ["total_loss", "iou_loss", "l1_loss", "conf_loss", "cls_loss", "num_fg"]


def build_product(depth, width, gamma=1.0, thr=0.5, val=1.5, momentum=0.03):
    ch = [256, 512, 1024]
    m = YOLOX(DFPPAFPN(depth, width, in_channels=ch),
              TALHead(8, width, in_channels=ch, gamma=gamma, ignore_thr=thr, ignore_value=val))
    for mod in m.modules():
        if isinstance(mod, torch.nn.BatchNorm2d):
            mod.eps, mod.momentum = 1e-3, momentum
    m.head.initialize_biases(1e-2)
    shapes = {k: tuple(v.shape) for k, v in m.state_dict().items()}
    m.load_state_dict(synth.synth_state_dict(shapes), strict=True)
    m.head.use_l1 = True
    return m.cuda()


def build_oracle(depth, width, gamma=1.0, thr=0.5, val=1.5, momentum=0.03, q=bf16_round):
    cfg = OracleCfg(depth=depth, width=width, gamma=gamma, ignore_thr=thr, ignore_value=val, bn_momentum=momentum)
    return StreamYoloOracle(cfg, synth.synth_state_dict(model_shapes(depth, width)), q=q)


def rel(a, b):
    a, b = a.float().cpu(), b.float().cpu()
    return ((a - b).norm() / (b.norm() + 1e-12)).item()


@pytest.fixture(params=["tc", "simt"])
def impl(request, monkeypatch):
    monkeypatch.setattr(engine, "CONV_IMPL", request.param)
    return request.param


@pytest.mark.parametrize("case", ["tiny_120x160", "tiny_empty_96x160"])
def test_train_forward_vs_oracle(case, impl):
    c = CASES[case]
    x = synth.synth_frames(c["B"], c["H"], c["W"])
    tg = synth.synth_labels(c["B"], c["H"], c["W"], empty_image=c["empty"])
    m = build_product(c["depth"], c["width"], c["gamma"], c["thr"], c["val"])
    m.train()
    feats = m.backbone(x.cuda())
    o = build_oracle(c["depth"], c["width"], c["gamma"], c["thr"], c["val"])
    ofeats = o.backbone_off(x)
    o_pert = build_oracle(c["depth"], c["width"], c["gamma"], c["thr"], c["val"])
    pfeats = o_pert.backbone_off(x * (1 + 1e-6))          # the same code, inputs nudged by 1e-6: rounding-noise floor
    for name, a, b, p in zip(("jian2", "jian1", "jian0"), feats, ofeats, pfeats):
        r, floor = rel(a, b), rel(p, b)
        assert r <= 1.5 * floor + 1e-2, f"fused {name}: rel l2 {r:.4f} vs rounding-noise floor {floor:.4f}"
    # running statistics after the (two-group) step: first layer is noise free, deep ones carry the noise
    sd = m.state_dict()
    k0 = "backbone.backbone.stem.conv.bn.running_mean"
    assert torch.allclose(sd[k0].cpu(), o.P[k0], rtol=2e-3, atol=2e-4), k0
    k1 = "backbone.backbone.stem.conv.bn.running_var"
    assert torch.allclose(sd[k1].cpu(), o.P[k1], rtol=2e-3, atol=2e-4), k1
    for k in ("backbone.C3_n4.conv3.bn.running_var", "backbone.jian1.bn.running_mean"):
        assert rel(sd[k], o.P[k]) < 5e-2, k
    assert int(sd["backbone.backbone.stem.conv.bn.num_batches_tracked"]) == 2
    assert int(sd["backbone.jian0.bn.num_batches_tracked"]) == 2
    # full forward + loss
    m2 = build_product(c["depth"], c["width"], c["gamma"], c["thr"], c["val"])
    m2.train()
    with torch.no_grad():                                    # the plain forward (engine.py); the recording forward has its own tests
        loss = m2(x.cuda(), (tg[0].cuda(), tg[1].cuda()))
    torch.cuda.synchronize()
    assert int(m2.state_dict()["head.stems.0.bn.num_batches_tracked"]) == 1
    o2 = build_oracle(c["depth"], c["width"], c["gamma"], c["thr"], c["val"])
    ref = o2.forward(x, tg)
    pert = build_oracle(c["depth"], c["width"], c["gamma"], c["thr"], c["val"]).forward(x * (1 + 1e-6), tg)
    got = np.array([float(loss[k]) for k in ORDER])
    want = np.array([float(ref[k]) for k in ORDER])
    floor = np.abs(np.array([float(pert[k]) for k in ORDER]) - want)      # the oracle's own rounding-noise floor on the losses
    tol = 2.0 * floor + 5e-2 * np.abs(want) + 5e-3
    assert (np.abs(got - want)[:5] <= tol[:5]).all(), f"losses {got} vs oracle {want} (noise floor {floor})"
    assert abs(got[5] - want[5]) <= 0.15 + 2.0 * floor[5]          # num_fg / num_gt: a few discrete assignments may flip
    gold = np.load(os.path.join(GOLD, case + ".npz"))["train_loss"]
    np.testing.assert_allclose(got[:5], gold[:5], rtol=1.5e-1, atol=1e-2)   # tiny random-init nets: chaotic


def _ulp_check(got, ref, what):
    got, ref = got.float().cpu(), ref.float().cpu()
    rms = ref.pow(2).mean().sqrt().item() + 1e-12
    err = (got - ref).abs()
    bad = err > (2.0 ** -6) * ref.abs() + (2.0 ** -6) * rms
    r = ((got - ref).norm() / (ref.norm() + 1e-12)).item()
    assert not bad.any() and r < 4e-3, f"{what}: {int(bad.sum())}/{bad.numel()} beyond 2 ulp, rel l2 {r:.2e}"


@pytest.mark.parametrize("mode", ["train", "eval"])
def test_every_layer_teacher_forced(mode, impl):
    """Each BaseConv of the product, fed the oracle's own (bf16-exact) input / residual, must
    reproduce the oracle's stored output to rounding: the per-layer parity bar."""
    from streamyolo_b200.model import engine
    from streamyolo_b200.model.network_blocks import BaseConv
    c = CASES["tiny_120x160"]
    x = synth.synth_frames(c["B"], c["H"], c["W"])
    tg = synth.synth_labels(c["B"], c["H"], c["W"])
    train = mode == "train"
    o = build_oracle(c["depth"], c["width"])
    o.training = train
    o.trace = {}
    if train:
        o.forward(x, tg)
    else:
        o.forward(x)
    tr = o.trace
    m = build_product(c["depth"], c["width"])
    m.train(train)
    dev = torch.device("cuda")
    n_checked = 0
    for name, mod in m.named_modules():
        if not isinstance(mod, BaseConv) or name + ".in" not in tr:
            continue
        if name.endswith("stem.conv") or ".jian" in name:
            continue
        xin = ops.from_nchw(tr[name + ".in"].to(dev))
        res = ops.from_nchw(tr[name + ".res"].to(dev)) if name + ".res" in tr else None
        ctx = engine.Ctx(train, xin.n, xin.n, dev)
        with torch.no_grad():
            y = engine.base_conv(ctx, mod, xin, res=res)
        torch.cuda.synchronize()
        _ulp_check(y.nchw_float(), tr[name + ".out"], name)
        n_checked += 1
    assert n_checked == 77 - 1 - 3
    # stem: last oracle call is the support frame (channels 3:6)
    with torch.no_grad():
        ctx = engine.Ctx(train, c["B"], c["B"], dev)
        y = engine.focus_stem(ctx, m.backbone.backbone.stem, x[:, 3:6].contiguous().cuda(), 1)
    _ulp_check(y.nchw_float(), tr["backbone.backbone.stem.conv.out"], "stem")
    # DFP fusion as a block, from the oracle's un-fused PAN outputs of both frames
    o2 = build_oracle(c["depth"], c["width"])
    o2.training = train
    xq = o2.q(x)
    cur, sup = o2.pafpn(xq[:, 0:3]), o2.pafpn(xq[:, 3:6])
    fused = o2._fuse(cur, sup)
    with torch.no_grad():
        ctx = engine.Ctx(train, 2 * c["B"], c["B"], dev)
        both = [ops.from_nchw(torch.cat([a, b], 0).to(dev)) for a, b in zip(cur, sup)]
        got = engine.dfp_fuse(ctx, m.backbone, tuple(v.imgs(0, c["B"]) for v in both),
                              tuple(v.imgs(c["B"], c["B"]) for v in both))
    for g_, f_, nm in zip(got, fused, ("jian2", "jian1", "jian0")):
        _ulp_check(g_.nchw_float(), f_, "dfp " + nm)


def test_loss_kernels_bit_exact_assignment():
    """Feed the oracle's own fp32 head outputs to sy_tal_loss: integer results must be identical."""
    c = CASES["tiny_120x160"]
    x = synth.synth_frames(4, c["H"], c["W"])
    tg = synth.synth_labels(4, c["H"], c["W"], empty_image=2)
    o = build_oracle(c["depth"], c["width"], q=None)
    feats = o.backbone_off(x)
    outputs, origin, grid = o.flatten_decode(o.head_levels(feats), sigmoid=False)
    ref = o.losses(outputs, origin, grid, tg, return_aux=True)
    b, a, no = outputs.shape
    dev = "cuda"
    ws = torch.empty(ops.tal_loss_workspace_bytes(b, a, 120, 8), dtype=torch.uint8, device=dev)
    loss = torch.empty(6, device=dev)
    fg = torch.empty((b, a), dtype=torch.int32, device=dev)
    mt = torch.empty((b, a), dtype=torch.int32, device=dev)
    pi = torch.empty((b, a), device=dev)
    ops.tal_loss(outputs.cuda().contiguous(), origin.cuda().contiguous(), tg[0].cuda(), tg[1].cuda(), o.hw,
                 (8, 16, 32), 1.0, 0.5, 1.5, True, ws, loss, fg, mt, pi)
    torch.cuda.synchronize()
    aux = ref["aux"]
    assert torch.equal(fg.cpu().bool(), aux["fg"]), "foreground anchor set differs"
    assert torch.equal(mt.cpu().long(), aux["matched"]), "matched GT ids differ"
    assert torch.allclose(pi.cpu(), aux["pred_iou"], rtol=1e-5, atol=1e-6)
    got = loss.cpu().numpy()
    want = np.array([float(ref[k]) for k in ORDER])[[0, 1, 3, 4, 2, 5]]   # kernel order: total, iou, obj, cls, l1, num_fg
    np.testing.assert_allclose(got, want, rtol=1e-4, atol=1e-5)


def test_eval_and_on_pipe_vs_oracle(impl):
    c = CASES["tiny_120x160"]
    x = synth.synth_frames(c["B"], c["H"], c["W"])
    tg = synth.synth_labels(c["B"], c["H"], c["W"])
    xc = torch.cat([x[:, 0:3], x[:, 0:3]], 1)
    o = build_oracle(c["depth"], c["width"], momentum=1.0)
    o.forward(xc, tg)                       # calibration pass: running stats := batch stats
    o.training = False
    ref = o.forward(xc)
    m = build_product(c["depth"], c["width"])
    # drop-in property: the oracle's (== reference's) state_dict loads into the product
    m.load_state_dict({k: v.clone() for k, v in o.P.items()}, strict=True)
    m.eval()
    got = m(xc.cuda())
    torch.cuda.synchronize()
    assert list(map(tuple, m.head.hw)) == [tuple(h) for h in o.hw]
    assert got.shape == ref.shape
    r = rel(got[..., :4], ref[..., :4])
    assert r < 3e-2, f"eval boxes rel l2 {r}"      # eval mode: no batch statistics, noise stays at the ulp level
    assert (got[..., 4:].cpu() - ref[..., 4:]).abs().max().item() < 3e-2
    gold = np.load(os.path.join(GOLD, "tiny_120x160.npz"))
    sub = int(gold["eval_sub_step"])
    g = torch.from_numpy(gold["eval_sub"])
    assert rel(got[:, ::sub, :4], g[..., :4]) < 1e-1     # bf16 product vs fp32 reference fixture
    # on_pipe: star call == buffered call on the same frame; buffered call on a new frame vs oracle
    o1, buf = m(x[:1, 0:3].cuda(), mode="on_pipe")
    o1b, _ = m(x[:1, 0:3].cuda(), buffer=buf, mode="on_pipe")
    assert torch.equal(o1, o1b)
    o2, buf2 = m(x[1:2, 0:3].cuda(), buffer=buf, mode="on_pipe")
    r1, rbuf = o.forward(x[:1, 0:3], mode="on_pipe")
    r2, _ = o.forward(x[1:2, 0:3], buffer=rbuf, mode="on_pipe")
    torch.cuda.synchronize()
    assert rel(o1[..., :4], r1[..., :4]) < 3e-2 and rel(o2[..., :4], r2[..., :4]) < 3e-2
    # un-fused PAN buffers (~70 bf16 layers deep, down to a 4x5 map): judged against the rounding-noise floor,
    # i.e. the same oracle code on inputs nudged by 1e-6
    _, pbuf = o.forward(x[:1, 0:3] * (1 + 1e-6), mode="on_pipe")
    for a, b, pb in zip(buf, rbuf, pbuf):
        assert rel(a, b) <= 1.5 * rel(pb, b) + 2e-2


def test_s_model_full_resolution_golden():
    """StreamYOLO-s, 600x960, B=2 (BASELINE.json config 1) against the reference-generated fixture."""
    c = CASES["s_600x960"]
    x = synth.synth_frames(c["B"], c["H"], c["W"])
    tg = synth.synth_labels(c["B"], c["H"], c["W"])
    m = build_product(c["depth"], c["width"])
    m.train()
    m.head.keep_assignment = True
    with torch.no_grad():
        loss = m(x.cuda(), (tg[0].cuda(), tg[1].cuda()))
    torch.cuda.synchronize()
    got = np.array([float(loss[k]) for k in ORDER])
    gold = np.load(os.path.join(GOLD, "s_600x960.npz"))
    np.testing.assert_allclose(got[:5], gold["train_loss"][:5], rtol=8e-2, atol=1e-2)
    assert abs(got[5] - gold["train_loss"][5]) <= 0.15
    assert m.head.hw == [(75, 120), (38, 60), (19, 30)]
    # size-independent property at full size: every foreground anchor is a candidate of its matched GT
    asg = m.head.last_assignment
    fg = asg["fg_out"].bool()
    assert int(fg.sum()) >= 1 and (asg["matched_out"][fg] >= 0).all() and (asg["matched_out"][~fg] == -1).all()
    assert (asg["pred_iou_out"][fg] >= 0).all() and (asg["pred_iou_out"][fg] <= 1).all()


def test_loss_backward_vs_oracle_autograd():
    """sy_tal_loss_backward on the oracle's own fp32 head outputs against torch.autograd through the oracle's loss
    (which tests/test_oracle_golden.py pins to the reference's loss.backward()): d loss / d outputs, d loss / d origin
    and the folded d loss / d raw head outputs, element-wise; then the per-level channel sums of the raw gradient against
    the reference's own head prediction-conv bias gradients (tests/golden/grad_*.npz).  Tolerance 2e-4 relative to the
    largest gradient entry (fp32 kernels, different summation order of the normalisers)."""
    c = CASES["tiny_120x160"]
    x = synth.synth_frames(c["B"], c["H"], c["W"])
    tg = synth.synth_labels(c["B"], c["H"], c["W"], empty_image=c["empty"])
    o = build_oracle(c["depth"], c["width"], c["gamma"], c["thr"], c["val"], q=None)
    with torch.no_grad():
        feats = o.backbone_off(x)
        levels = o.head_levels(feats)
        outputs, origin, grid = o.flatten_decode(levels, sigmoid=False)
    out_l = outputs.clone().requires_grad_(True)
    org_l = origin.clone().requires_grad_(True)
    ref = o.losses(out_l, org_l, grid, tg)
    ref["total_loss"].backward()
    b, a, no = outputs.shape
    dev = "cuda"
    ws = torch.empty(ops.tal_loss_workspace_bytes(b, a, 120, 8), dtype=torch.uint8, device=dev)
    loss = torch.empty(6, device=dev)
    od, gd = outputs.cuda().contiguous(), origin.cuda().contiguous()
    fut = tg[0].cuda()
    ops.tal_loss(od, gd, fut, tg[1].cuda(), o.hw, (8, 16, 32), c["gamma"], c["thr"], c["val"], True, ws, loss)
    g_out, g_org, g_raw = torch.full_like(od, float("nan")), torch.full_like(gd, float("nan")), torch.full_like(od, float("nan"))
    ops.tal_loss_backward(od, gd, fut, o.hw, (8, 16, 32), c["gamma"], True, ws, 1.0, g_out, g_org, g_raw)
    torch.cuda.synchronize()
    assert abs(float(loss[0]) - float(ref["total_loss"])) < 1e-4 * abs(float(ref["total_loss"]))

    def close(got, want, what):
        got, want = got.cpu(), want
        scale = float(want.abs().max())
        err = float((got - want).abs().max())
        assert torch.isfinite(got).all() and err <= 2e-4 * scale + 1e-9, f"{what}: max err {err:.3e} vs scale {scale:.3e}"

    close(g_out, out_l.grad, "d loss / d outputs")
    close(g_org, org_l.grad, "d loss / d origin")
    gx, gy, gs = grid
    want_raw = out_l.grad.clone()
    want_raw[..., 0:2] = out_l.grad[..., 0:2] * gs[None, :, None] + org_l.grad[..., 0:2]
    want_raw[..., 2:4] = out_l.grad[..., 2:4] * outputs[..., 2:4] + org_l.grad[..., 2:4]
    close(g_raw, want_raw, "d loss / d raw head outputs")
    # the reference's own bias gradients = channel sums of the raw gradient per level ([reg4, obj1, cls8] order)
    gold = np.load(os.path.join(GOLD, "grad_tiny_120x160.npz"))
    off = 0
    for k, (h, w) in enumerate(o.hw):
        sums = g_raw[:, off:off + h * w].sum((0, 1)).cpu().double()
        off += h * w
        for name, sl in (("reg", slice(0, 4)), ("obj", slice(4, 5)), ("cls", slice(5, 13))):
            want = torch.from_numpy(gold[f"g:head.{name}_preds.{k}.bias"]).double()
            assert torch.allclose(sums[sl], want, rtol=2e-3, atol=2e-4 * float(want.abs().max()) + 1e-7), \
                f"head.{name}_preds.{k}.bias: {sums[sl].tolist()} vs {want.tolist()}"


def test_forward_backward_vs_oracle_autograd():
    """streamyolo_b200.model.backward.forward_backward on the GPU against autograd through the oracle with bf16 storage
    (which tests/test_oracle_golden.py pins to the reference's loss.backward()).  A random-init train-mode BatchNorm net is
    chaotic under bf16 storage (tests/tools/diag_bwd.py: nudging the inputs by half a bf16
    ulp decorrelates the stride-32 gradients of the ORACLE ITSELF at 120x160, rel ~1.0), so the element-wise bar lives in
    tests/test_gpu_train.py::test_walk_in_situ_every_conv_backward (identical inputs per op); here, on a larger map where
    the noise is moderate, every parameter gradient must be finite, point the right way and have the right size:
    per-parameter deviation within 2 x the oracle's own rounding-noise floor + 0.25 (for 95 % of the parameters), median and
    10th-percentile cosine against the oracle's gradients not worse than the oracle's own under a half-ulp input nudge
    (minus 0.15 / 0.25; capped at 0.85 / 0.6)."""
    from streamyolo_b200.model import backward
    c = dict(CASES["tiny_120x160"], H=256, W=320)
    x = synth.synth_frames(c["B"], c["H"], c["W"])
    tg = synth.synth_labels(c["B"], c["H"], c["W"], empty_image=c["empty"])
    m = build_product(c["depth"], c["width"], c["gamma"], c["thr"], c["val"])
    m.train()
    loss = backward.forward_backward(m, x.cuda(), (tg[0].cuda(), tg[1].cuda()))
    torch.cuda.synchronize()

    def oracle_grads(xin):
        o = build_oracle(c["depth"], c["width"], c["gamma"], c["thr"], c["val"])
        for k, t in o.P.items():
            if t.dtype.is_floating_point and not k.endswith(("running_mean", "running_var")):
                t.requires_grad_(True)
        r = o.forward(xin, tg)
        r["total_loss"].backward()
        return float(r["total_loss"].detach()), {k: t.grad for k, t in o.P.items() if t.grad is not None}

    want_loss, want = oracle_grads(x)
    _, pert = oracle_grads(x * (1 + 2.0 ** -9))            # half a bf16 ulp on every input
    assert abs(float(loss["total_loss"]) - want_loss) < 5e-2 * abs(want_loss)
    bad, cos, cos_floor = [], [], []

    def cosine(a, b):
        a, b = a.float().cpu().flatten(), b.float().flatten()
        return float(torch.dot(a, b) / (a.norm() * b.norm() + 1e-20))

    for k, p in m.named_parameters():
        assert p.grad is not None and torch.isfinite(p.grad).all(), k
        cos.append(cosine(p.grad, want[k]))
        cos_floor.append(cosine(pert[k], want[k]))
        r, floor = rel(p.grad, want[k]), rel(pert[k], want[k])
        if r > 2.0 * floor + 0.25:
            bad.append(f"{k}: rel {r:.3f} vs rounding-noise floor {floor:.3f}")
    cos.sort()
    cos_floor.sort()
    n = len(cos)
    # at most 5 % of the 249 parameters may exceed their own floor criterion (heavy-tailed noise), none may be wild
    assert len(bad) <= n // 20, "\n".join(bad[:20])
    med, p10 = cos[n // 2], cos[n // 10]
    assert med >= min(0.85, cos_floor[n // 2] - 0.15) and p10 >= min(0.6, cos_floor[n // 10] - 0.25), \
        (med, p10, cos_floor[n // 2], cos_floor[n // 10])
