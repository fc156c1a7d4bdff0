"""GPU parity on the BENCHMARKED configuration (StreamYOLO-l / -m, 600x960), the cases VERDICT r01 found missing:

  * every distinct conv launch shape of StreamYOLO-l at 8 pairs (34 shapes incl. 2048->1024, 1024->1024 with 4 N tiles,
    512->512 @19x30, the halo-mode 64->64 @150x240, two-segment BatchNorm pairs up to Cout 1024): conv + statistics +
    in-kernel BatchNorm finalize + normalise pass, against fp32 PyTorch on the same bf16 operands;
  * the fp32 accumulators themselves (validation store, before any bf16 rounding) within 1e-3 relative of F.conv2d --
    north_star's tolerance taken literally (measured ~1e-6);
  * SimOTA / TAL on identical fp32 head outputs at the full anchor count A = 11 850 for G in {0, 1, 12, 120} ground truths,
    with constructed ties (duplicated ground-truth boxes = equal cost columns, duplicated predictions = equal IoUs / costs):
    foreground set and matched ids bit-exact against the oracle;
  * StreamYOLO-l and -m end to end at 600x960, B = 2, train mode, against the bf16-storage oracle (rounding-noise-floor
    criterion of tests/test_gpu_model.py) + the six losses.
"""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

from oracle.streamyolo_oracle import OracleCfg, StreamYoloOracle  # noqa: E402
from streamyolo_b200 import ops, synth  # noqa: E402
from streamyolo_b200.ops import View  # noqa: E402
from test_gpu_model import ORDER, build_oracle, build_product, rel  # noqa: E402
from test_gpu_ops import bf, check_close, rand_w  # noqa: E402

DEV = "cuda"

# (n, cin, cout, h, w, k, stride, conv1|conv2 pair) -- the distinct conv shapes of StreamYOLO-l at 8 pairs
L_SHAPES = [
    (16, 64, 128, 300, 480, 3, 2, False),
    (16, 128, 128, 150, 240, 1, 1, True),
    (16, 64, 64, 150, 240, 1, 1, False),
    (16, 64, 64, 150, 240, 3, 1, False),
    (16, 128, 128, 150, 240, 1, 1, False),
    (16, 128, 256, 150, 240, 3, 2, False),
    (16, 256, 256, 75, 120, 1, 1, True),
    (16, 128, 128, 75, 120, 1, 1, False),
    (16, 128, 128, 75, 120, 3, 1, False),
    (16, 256, 256, 75, 120, 1, 1, False),
    (16, 256, 512, 75, 120, 3, 2, False),
    (16, 512, 512, 38, 60, 1, 1, True),
    (16, 256, 256, 38, 60, 1, 1, False),
    (16, 256, 256, 38, 60, 3, 1, False),
    (16, 512, 512, 38, 60, 1, 1, False),
    (16, 512, 1024, 38, 60, 3, 2, False),
    (16, 1024, 512, 19, 30, 1, 1, False),
    (16, 2048, 1024, 19, 30, 1, 1, False),
    (16, 1024, 1024, 19, 30, 1, 1, True),
    (16, 512, 512, 19, 30, 1, 1, False),
    (16, 512, 512, 19, 30, 3, 1, False),
    (16, 1024, 1024, 19, 30, 1, 1, False),
    (16, 1024, 512, 38, 60, 1, 1, True),
    (16, 512, 256, 38, 60, 1, 1, False),
    (16, 512, 256, 75, 120, 1, 1, True),
    (16, 256, 256, 75, 120, 3, 2, False),
    (16, 512, 512, 38, 60, 3, 2, False),
    (16, 256, 128, 75, 120, 1, 1, False),
    (8, 256, 256, 75, 120, 1, 1, False),
    (8, 256, 256, 75, 120, 3, 1, False),
    (8, 512, 256, 38, 60, 1, 1, False),
    (8, 256, 256, 38, 60, 3, 1, False),
    (8, 1024, 256, 19, 30, 1, 1, False),
    (8, 256, 256, 19, 30, 3, 1, False),
]


def _act(n, c, h, w, seed):
    g = torch.Generator(device=DEV).manual_seed(seed)
    return torch.randn((n, h, w, c), generator=g, device=DEV).to(torch.bfloat16)       # NHWC bf16


@pytest.mark.parametrize("case", L_SHAPES, ids=lambda c: "x".join(map(str, c)))
def test_l_layer_shape_conv_bn_apply(case):
    n, ci, co, h, w, k, s, pair = case
    xb = _act(n, ci, h, w, 1)
    wt = rand_w(co, ci, k, 2)
    g = torch.Generator().manual_seed(3)
    gamma, beta = (torch.rand(co, generator=g) + 0.5).to(DEV), (torch.rand(co, generator=g) - 0.5).to(DEV)
    rm, rv = torch.zeros(co, device=DEV), torch.ones(co, device=DEV)
    nbt = [torch.zeros((), dtype=torch.long, device=DEV) for _ in range(2)]
    half = co // 2
    if pair:                      # two BatchNorm parameter segments (CSPLayer conv1 | conv2 in one launch)
        segs = [(gamma[:half].contiguous(), beta[:half].contiguous(), rm[:half], rv[:half], nbt[0], 0),
                (gamma[half:].contiguous(), beta[half:].contiguous(), rm[half:], rv[half:], nbt[1], half)]
    else:
        segs = [(gamma, beta, rm, rv, nbt[0], 0)]
    split = n // 2                # current / support frames
    ho, wo = ops.conv_out_hw(h, w, k, s)
    xv = View(xb)
    raw, y = View.empty(n, ho, wo, co, DEV), View.empty(n, ho, wo, co, DEV)
    raw.buf.fill_(float("nan"))
    y.buf.fill_(float("nan"))
    res = View(_act(n, co, ho, wo, 4)) if (k == 3 and s == 1 and ci == co) else None      # bottleneck shortcut
    partials = torch.empty((ops.conv_stat_rows(), 4 * co), device=DEV)
    ss = torch.empty((2, 2, co), device=DEV)
    sync = torch.zeros(2, dtype=torch.int32, device=DEV)
    acc = torch.full((n * ho * wo, co), float("nan"), device=DEV)
    ops.conv2d(xv, ops.pack_conv_weight(wt), raw, k, s, ops.SY_CONV_RAW, partials=partials, split_n=split, bn=segs,
               momentum=0.03, eps=1e-3, scale_shift=ss, sync=sync, debug_f32=acc)
    ops.bn_act_apply(raw, ss[0].data_ptr(), ss[1].data_ptr(), split, 1, res, y)
    torch.cuda.synchronize()
    assert sync.tolist() == [0, 0]
    ref = F.conv2d(xb.permute(0, 3, 1, 2).float(), wt, None, s, (k - 1) // 2)            # fp32, TF32 off (conftest)
    # (1) the accumulators: north_star's 1e-3 relative, literally (per element against |ref| + the tensor's rms)
    accn = acc.view(n, ho, wo, co).permute(0, 3, 1, 2)
    rms = float(ref.pow(2).mean().sqrt())
    err = (accn - ref).abs()
    assert torch.isfinite(accn).all()
    assert bool((err <= 1e-3 * ref.abs() + 1e-4 * rms).all()), f"fp32 accumulators: max err {float(err.max()):.3e}, rms {rms:.3e}"
    assert float((accn - ref).norm() / ref.norm()) < 2e-5
    # (2) the stored bf16 result = the rounded accumulator, bit for bit
    rawf = raw.nchw_float()
    assert torch.equal(rawf, accn.to(torch.bfloat16).float())
    # (3) BatchNorm finalize from the stored values: scale / shift per group, running statistics, counters
    for gi, (a, b) in enumerate(((0, split), (split, n))):
        part = rawf[a:b].double()
        mean, var = part.mean((0, 2, 3)), part.var((0, 2, 3), unbiased=False)
        sc = gamma.double() / torch.sqrt(var + 1e-3)
        assert torch.allclose(ss[0, gi].double(), sc, rtol=1e-4, atol=1e-6), f"scale group {gi}"
        assert torch.allclose(ss[1, gi].double(), beta.double() - mean * sc, rtol=1e-4, atol=1e-5 + 1e-4 * float((mean * sc).abs().max())), f"shift group {gi}"
    assert int(nbt[0]) == 2 and (not pair or int(nbt[1]) == 2)
    # (4) the normalise pass on the stored values
    want = torch.cat([F.silu(rawf[a:b] * ss[0, gi][None, :, None, None] + ss[1, gi][None, :, None, None])
                      for gi, (a, b) in enumerate(((0, split), (split, n)))], 0)
    if res is not None:
        want = want + res.nchw_float()
    check_close(y.nchw_float(), want, f"normalise {case}")


# ------------------------------------------------------------------------------------------------ SimOTA at full size
HW = [(75, 120), (38, 60), (19, 30)]
STRIDES = (8, 16, 32)
A_TOTAL = sum(h * w for h, w in HW)


def _synthetic_head_outputs(b, labels_fut, seed, dup_pred=False):
    """Plausible decoded head outputs [b, 11850, 13] (fp32): boxes near their anchors, a few anchors per ground truth
    predicting that box well, low obj / cls logits elsewhere."""
    g = torch.Generator().manual_seed(seed)
    outs, origin = [], []
    for (h, w), s in zip(HW, STRIDES):
        yv, xv = torch.meshgrid(torch.arange(h), torch.arange(w), indexing="ij")
        raw = torch.randn((b, h * w, 4), generator=g) * 0.4
        xy = (raw[..., :2] + torch.stack([xv, yv], -1).reshape(1, -1, 2)) * s
        wh = torch.exp(raw[..., 2:4] + 1.2) * s
        outs.append(torch.cat([xy, wh, torch.randn((b, h * w, 9), generator=g) * 1.5 - 3.0], -1))
        origin.append(raw)
    out, org = torch.cat(outs, 1), torch.cat(origin, 1)
    for bi in range(b):                       # good predictions near every ground truth
        for gt in labels_fut[bi]:
            if gt[3] <= 0:
                continue
            d = (out[bi, :, 0] - gt[1]).abs() + (out[bi, :, 1] - gt[2]).abs()
            idx = torch.topk(d, 12, largest=False).indices
            out[bi, idx, 0:4] = gt[1:5] * (1 + 0.05 * torch.randn((12, 4), generator=g))
            out[bi, idx, 4] = 1.0
            out[bi, idx, 5 + int(gt[0])] = 1.5
            if dup_pred:                      # exact duplicates: equal IoU and equal cost at several anchors
                out[bi, idx[1]] = out[bi, idx[0]]
                out[bi, idx[3]] = out[bi, idx[2]]
    return out.contiguous(), org.contiguous()


def _labels(b, n_gt, seed, dup_gt=False):
    fut, cur = synth.synth_labels(b, 600, 960, n_obj=max(n_gt, 2), seed=seed)
    if n_gt < 2:
        fut[:, n_gt:] = 0
        cur[:, n_gt:] = 0
    if dup_gt and n_gt >= 4:                  # two ground truths with identical class and box: equal cost columns
        fut[:, 3] = fut[:, 2]
        cur[:, 3] = cur[:, 2]
    return fut, cur


@pytest.mark.parametrize("n_gt,ties", [(0, False), (1, False), (12, False), (12, True), (120, False), (120, True)])
def test_simota_bit_exact_full_anchor_count(n_gt, ties):
    b = 3
    fut, cur = _labels(b, n_gt, 7 + n_gt, dup_gt=ties)
    if n_gt >= 12:
        fut[1] = 0                                            # one image without labels (tal_head.py:309-315)
        cur[1] = 0
    outputs, origin = _synthetic_head_outputs(b, fut, 11 + n_gt, dup_pred=ties)
    o = StreamYoloOracle(OracleCfg(gamma=1.0, ignore_thr=0.5, ignore_value=1.6), {})
    grid = tuple(t.float() for t in o.grids(HW, STRIDES))
    ref = o.losses(outputs, origin, grid, (fut, cur), return_aux=True)
    ws = torch.empty(ops.tal_loss_workspace_bytes(b, A_TOTAL, 120, 8), dtype=torch.uint8, device=DEV)
    loss = torch.empty(6, device=DEV)
    fg = torch.empty((b, A_TOTAL), dtype=torch.int32, device=DEV)
    mt = torch.empty((b, A_TOTAL), dtype=torch.int32, device=DEV)
    pi = torch.empty((b, A_TOTAL), device=DEV)
    ops.tal_loss(outputs.to(DEV), origin.to(DEV), fut.to(DEV), cur.to(DEV), HW, STRIDES, 1.0, 0.5, 1.6, True, ws, loss, fg, mt, pi)
    torch.cuda.synchronize()
    aux = ref["aux"]
    nfg = int(aux["fg"].sum())
    assert (n_gt == 0) == (nfg == 0)
    assert torch.equal(fg.cpu().bool(), aux["fg"]), f"foreground set differs ({int((fg.cpu().bool() != aux['fg']).sum())} of {nfg})"
    assert torch.equal(mt.cpu().long(), aux["matched"]), "matched GT ids differ"
    assert torch.allclose(pi.cpu(), aux["pred_iou"], rtol=1e-5, atol=1e-6)
    got = loss.cpu().numpy()
    want = np.array([float(ref[k]) for k in ORDER])[[0, 1, 3, 4, 2, 5]]
    np.testing.assert_allclose(got, want, rtol=2e-4, atol=1e-5)


# ------------------------------------------------------------------------------------------------ the benchmarked models
@pytest.mark.parametrize("tag,depth,width,tal", [("l", 1.0, 1.0, (1.0, 0.5, 1.6)), ("m", 0.67, 0.75, (1.0, 0.4, 1.7))])
def test_benchmarked_model_train_forward_vs_oracle(tag, depth, width, tal):
    """StreamYOLO-l / -m, 600x960, B = 2, train mode: fused FPN features against the bf16-storage oracle with the
    rounding-noise-floor criterion (the same oracle code on inputs nudged by 1e-6), the six losses (within 5 % + twice the
    larger of the oracle's and the product's own deviation under that nudge), the running statistics
    of the first and the deepest BatchNorm."""
    B, H, W = 2, 600, 960
    x = synth.synth_frames(B, H, W)
    tg = synth.synth_labels(B, H, W)
    m = build_product(depth, width, *tal).train()
    with torch.no_grad():
        feats = m.backbone(x.cuda())
        torch.cuda.synchronize()
    o = build_oracle(depth, width, *tal)
    ofeats = o.backbone_off(x)
    pfeats = build_oracle(depth, width, *tal).backbone_off(x * (1 + 1e-6))
    for name, a, b, p in zip(("jian2", "jian1", "jian0"), feats, ofeats, pfeats):
        r, floor = rel(a, b), rel(p, b)
        assert r <= 1.5 * floor + 1e-2, f"{tag} fused {name}: rel l2 {r:.4f} vs rounding-noise floor {floor:.4f}"
    sd = m.state_dict()
    for k in ("backbone.backbone.stem.conv.bn.running_mean", "backbone.backbone.stem.conv.bn.running_var"):
        assert torch.allclose(sd[k].cpu(), o.P[k], rtol=2e-3, atol=2e-4), k
    assert int(sd["backbone.C3_n4.conv3.bn.num_batches_tracked"]) == 2
    m2 = build_product(depth, width, *tal).train()
    with torch.no_grad():
        loss = m2(x.cuda(), (tg[0].cuda(), tg[1].cuda()))
        torch.cuda.synchronize()
    ref = build_oracle(depth, width, *tal).forward(x, tg)
    pert = build_oracle(depth, width, *tal).forward(x * (1 + 1e-6), tg)      # the oracle's own rounding-noise floor on the losses
    # ... and the product's own: it stores the frames in bf16, so the nudge is one bf16 ulp (a smaller one would vanish)
    m3 = build_product(depth, width, *tal).train()
    with torch.no_grad():
        loss_p = m3((x * (1 + 2.0 ** -8)).cuda(), (tg[0].cuda(), tg[1].cuda()))
        torch.cuda.synchronize()
    got = np.array([float(loss[k]) for k in ORDER])
    want = np.array([float(ref[k]) for k in ORDER])
    # A rounding-sized nudge of the input flips SimOTA assignments in either implementation (random-init train-mode BatchNorm nets are
    # chaotic under bf16 storage); the discrepancy between the two must not exceed what each shows against itself.
    floor = np.maximum(np.abs(np.array([float(pert[k]) for k in ORDER]) - want),
                       np.abs(np.array([float(loss_p[k]) for k in ORDER]) - got))
    tol = 2.0 * floor + 5e-2 * np.abs(want) + 5e-3
    assert (np.abs(got - want)[:5] <= tol[:5]).all(), f"{tag} losses {got} vs oracle {want} (noise floor {floor})"
    assert abs(got[5] - want[5]) <= 0.15 + 2.0 * floor[5]
    assert m2.head.hw == [(75, 120), (38, 60), (19, 30)]
