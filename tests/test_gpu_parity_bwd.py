"""GPU parity of the training step's BACKWARD kernels at the benchmarked shapes, against float64 PyTorch on the very
operands the kernels read (the backward counterpart of tests/test_gpu_parity_l.py):

  * the reverse walk checked launch by launch (backward.DEBUG_HOOK) during one forward_backward of StreamYOLO-l at 4 pairs,
    -m and -s at 8 pairs, 600x960, built like bench.py builds them: BatchNorm+SiLU backward, dgamma / dbeta, dW (accumulated
    where a module runs twice), the data gradient accumulated in place -- every conv launch, counted per model;
  * sy_conv2d_wgrad_tc on shapes that reach every split-group count of the reduction (SG = 1, 2, 4, 8) and every tile
    width (BN = 64, 128, 256), accumulating onto a non-zero start;
  * the data gradient as the walk runs it: FUSED, scale 1 / shift 0, accumulated in place through the residual input,
    pair-packed filters, stride 2 through dilate2, under every tiling the planner can be forced to;
  * sy_bn_act_backward at the network's widths (C = 48 ... 1024), the 296-row cap, one and two statistics groups;
  * sy_head_pred_backward at every level of the l / m / s heads and for 1, 3, 8, 20, 27 classes (every compiled
    instantiation and the generic kernel), and the 27-class limit;
  * sy_tal_loss_backward at the full anchor count (A = 11 850) for 0 ... 120 ground truths, gamma 1 and 1.5, loss scales,
    empty images and box edges equal to their ground truth's (the 0.5 tie split of torch.maximum / minimum);
  * the glue backward ops (upsample, SPP max pools, add) at production widths.

Tolerances follow the error model of each result:
  * bf16-stored results (draw, dx, feature gradients): one bf16 rounding plus accumulation noise (check_close);
  * fp32 reductions of K terms t_k (dW, dgamma / dbeta, head dW / db): |err| <= KAPPA * 2^-24 * K * rms(t) + 2^-24 * |ref|.
    K * rms(t) = sqrt(K * sum t^2) bounds sum |t|, and u * K * rms is the typical rounding error of one fp32 running sum of
    K terms of that size; the sum of squares comes from a second float64 reference on the squared operands.  KAPPA = 64
    covers the tail over millions of outputs and the drift of running sums whose terms share a local mean: in the head
    towers of the walk the objectness gradient has one sign over the whole background, and the weight gradient's
    tensor-core K loop (up to ~4 500 pixels per split) then reaches err / (u K rms) ~ 32.  The bar does not grow with the
    largest output.
Every reduction case also recomputes its reference with one unit of the kernel's work left out (one 64-pixel K block,
one partial row, one 256-pixel head row, one 64-channel block at one tap) and asserts that the bar rejects it.
"""
import math

import ctypes as C
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

from oracle.streamyolo_oracle import OracleCfg, StreamYoloOracle  # noqa: E402
from streamyolo_b200 import ops, synth  # noqa: E402
from streamyolo_b200.model import backward, engine  # noqa: E402
from streamyolo_b200.ops import View  # noqa: E402
from test_gpu_model import build_product  # noqa: E402
from test_gpu_ops import check_close  # noqa: E402
from test_gpu_parity_l import A_TOTAL, HW, STRIDES, _labels, _synthetic_head_outputs  # noqa: E402

DEV = "cuda"
F64 = torch.float64
U32 = 2.0 ** -24          # fp32 unit roundoff
KAPPA = 64.0
SY_EINVAL = 1             # include/streamyolo_sm100.h

# (depth, width), (gamma, ignore_thr, ignore_value) of the benchmarked models (bench.py MODELS / TAL, from cfgs/*.py)
MODELS = {"s": ((0.33, 0.50), (1.0, 0.5, 1.5)), "m": ((0.67, 0.75), (1.0, 0.4, 1.7)), "l": ((1.0, 1.0), (1.0, 0.5, 1.6))}


def _gen(seed):
    return torch.Generator(device=DEV).manual_seed(seed)


def nchw64(v: View):
    return v.torch().permute(0, 3, 1, 2).double()


def post_silu(n, h, w, c, seed):
    """NHWC bf16 activations like a BaseConv output: SiLU of a unit normal with a per-channel offset (non-negative mean)"""
    g = _gen(seed)
    mu = torch.rand(c, generator=g, device=DEV) * 2.0 - 1.0
    return View(F.silu(torch.randn((n, h, w, c), generator=g, device=DEV) + mu).to(torch.bfloat16))


def small_grad(n, h, w, c, seed, scale=1e-2):
    g = _gen(seed)
    return View((torch.randn((n, h, w, c), generator=g, device=DEV) * scale).to(torch.bfloat16))


# ------------------------------------------------------------------------------------------------ tolerances
def sum_tol(ref, s2, k, kappa=KAPPA):
    """bar of an fp32 reduction of k terms whose squares sum to s2 (float64), ending at ref"""
    return kappa * U32 * torch.sqrt(k * s2) + U32 * ref.abs()


def sum_ok(got, ref, s2, k):
    err = (got.double() - ref).abs()
    tol = sum_tol(ref, s2, k)
    return bool((err <= tol).all()), float((err / tol.clamp(min=1e-300)).max())


def check_sum(got, ref, s2, k, what):
    assert bool(torch.isfinite(got).all()), f"{what}: non-finite"
    ok, worst = sum_ok(got, ref, s2, k)
    assert ok, f"{what}: outside the fp32 reduction bar, worst err / tol {worst:.3g} (K = {k})"
    return worst


def assert_rejects_sum(got, ref_omit, s2, k, what):
    ok, worst = sum_ok(got, ref_omit, s2, k)
    assert not ok, f"{what}: the bar accepts a reference with one unit of work left out (worst err / tol {worst:.3g})"


def outside_bf16(got, ref, ulp=2.0 ** -7):
    """number of elements outside check_close's bar"""
    got, ref = got.float(), ref.float()
    rms = ref.pow(2).mean().sqrt().item() + 1e-12
    return int(((got - ref).abs() > ulp * ref.abs() + ulp * rms).sum())


# ------------------------------------------------------------------------------------------------ shared references
def bn_act_backward_ref(raw, gy, ss, mi, groups, act):
    """float64 BatchNorm(train) + SiLU backward from the saved statistics.  raw, gy: NCHW float64; ss = [scale | shift][group][C],
    mi = [mean | invstd][group][C]; groups: (first image, end image, group).  Returns draw, dgamma, dbeta, the sums of the
    squared dgamma / dbeta terms and the per-pixel terms dz * xhat, dz."""
    c = raw.shape[1]
    draw, dz_all, t_all = torch.empty_like(raw), torch.empty_like(raw), torch.empty_like(raw)
    dg, db, s2g, s2b = (torch.zeros(c, dtype=F64, device=raw.device) for _ in range(4))
    for a, b, g in groups:
        sc, sh, mu, iv = (t.double()[None, :, None, None] for t in (ss[0, g], ss[1, g], mi[0, g], mi[1, g]))
        z = raw[a:b] * sc + sh
        if act:
            sg = torch.sigmoid(z)
            dz = gy[a:b] * (sg * (1 + z * (1 - sg)))
        else:
            dz = gy[a:b]
        xh = (raw[a:b] - mu) * iv
        t = dz * xh
        draw[a:b] = sc * (dz - dz.mean((0, 2, 3), keepdim=True) - xh * t.mean((0, 2, 3), keepdim=True))
        dg += t.sum((0, 2, 3))
        db += dz.sum((0, 2, 3))
        s2g += t.pow(2).sum((0, 2, 3))
        s2b += dz.pow(2).sum((0, 2, 3))
        dz_all[a:b], t_all[a:b] = dz, t
    return draw, dg, db, s2g, s2b, t_all, dz_all


def conv_backward_checker(ulp=2.0 ** -6):
    """backward.DEBUG_HOOK that checks every recorded conv launch of the walk in float64 on the very tensors the kernels read
    (the gradient buffer as it stood, the saved raw output / statistics, the bf16 weights).  Identical inputs per launch: no
    chaos amplification, so bf16-ulp and fp32-reduction bars hold.  Returns (hook, names of the checked launches)."""
    snap, seen = {}, []

    def hook(stage, r, **kw):
        if stage == "pre":
            snap["gy"] = nchw64(kw["gy"])
            snap["dg"] = kw["dgamma"].double() if kw["acc_bn"] else None
            snap["db"] = kw["dbeta"].double() if kw["acc_bn"] else None
            return
        if stage == "pre_w":
            snap["dw"] = kw["dw"].double() if kw["acc_w"] else None
            # gx is None when this launch is the first contribution to its input's gradient (written, not accumulated)
            snap["gx"] = nchw64(kw["gx"]) if kw["gx"] is not None else 0.0
            return
        mods, raw, xin = r["mods"], nchw64(r["raw"]), nchw64(r["x"])
        name = getattr(mods[0], "_sy_name", "?")
        kh, kw_ = r["k"]
        s, act = r["s"], r["act"]
        n = raw.shape[0]
        sp = r["split"] if 0 < r["split"] < n else n
        groups = [(0, sp, 0), (sp, n, 1)] if sp < n else [(0, n, 0)]
        draw_ref, dg, db, s2g, s2b, _, _ = bn_act_backward_ref(raw, snap["gy"], r["ss"], r["mi"], groups, act)
        del snap["gy"]
        if snap["dg"] is not None:
            dg, db = dg + snap["dg"], db + snap["db"]
        npix = raw.shape[0] * raw.shape[2] * raw.shape[3]
        draw = nchw64(kw["draw"])
        check_close(draw, draw_ref, f"{name}: d raw", ulp=ulp)
        del draw_ref
        check_sum(kw["dgamma"], dg, s2g, npix, f"{name}: dgamma")
        check_sum(kw["dbeta"], db, s2b, npix, f"{name}: dbeta")
        pad = ((kh - 1) // 2, (kw_ - 1) // 2)
        dw_ref = torch.nn.grad.conv2d_weight(xin, kw["dw"].shape, draw, stride=s, padding=pad)
        s2w = torch.nn.grad.conv2d_weight(xin.square(), kw["dw"].shape, draw.square(), stride=s, padding=pad)
        if snap["dw"] is not None:
            dw_ref = dw_ref + snap["dw"]
        check_sum(kw["dw"], dw_ref, s2w, npix, f"{name}: dw")
        del dw_ref, s2w
        wq = torch.cat([mm.conv.weight.detach() for mm in mods], 0).to(torch.bfloat16).double()
        dx_ref = torch.nn.grad.conv2d_input(xin.shape, wq, draw, stride=s, padding=pad) + snap["gx"]
        check_close(nchw64(kw["gx"]), dx_ref, f"{name}: dx (accumulated)", ulp=ulp)
        snap.clear()
        seen.append(name)

    return hook, seen


def run_walk_checked(m, x, tg):
    """one forward_backward of model ``m`` with every conv launch checked in situ; returns the names of the checked launches"""
    hook, seen = conv_backward_checker()
    engine.name_modules(m)
    backward.DEBUG_HOOK = hook
    backward.POISON = True        # the gradient arena starts as NaN: a region read before it was written would show up
    try:
        backward.forward_backward(m, x, tg)
        torch.cuda.synchronize()
    finally:
        backward.DEBUG_HOOK = None
        backward.POISON = False
    for n_, p_ in m.named_parameters():
        assert p_.grad is not None and bool(torch.isfinite(p_.grad).all()), n_
    return seen


# ------------------------------------------------------------------------------------------------ 1. the walk in situ
# checked launches = BaseConv modules - 8 CSP conv2 (ride with their conv1) - 3 head reg towers (ride with their cls twin)
# + 3 (the DFP jian convs run twice) - 1 (the stem has no data gradient): l 125, m 101, s 77 BaseConvs
@pytest.mark.parametrize("tag,pairs,launches", [("l", 4, 116), ("m", 8, 92), ("s", 8, 68)], ids=["l_b4", "m_b8", "s_b8"])
def test_walk_in_situ_benchmarked(tag, pairs, launches):
    (depth, width), (gamma, thr, val) = MODELS[tag]
    m = build_product(depth, width, gamma, thr, val).train()
    x = synth.synth_frames(pairs, 600, 960, seed=4321).cuda()
    tg = tuple(t.cuda() for t in synth.synth_labels(pairs, 600, 960, seed=11))
    seen = run_walk_checked(m, x, tg)
    assert len(seen) == launches, len(seen)


# ------------------------------------------------------------------------------------------------ 2a. weight gradient
def wgrad_variant(ci, co, k, ws_bytes, sms):
    """(BN, ksplit, SG) of sy_conv2d_wgrad_tc from its workspace size (items * 128 * BN * 4 bytes) and the split-group rule
    of conv_wgrad.cu: groups double while SG < 8, Cout * Cin * taps * SG < SMs * 2048 and ksplit >= 16 * SG"""
    bn = 64 if ci <= 64 else (128 if ci <= 128 else 256)
    base = -(-co // 128) * -(-ci // bn) * k * k
    items = ws_bytes // (128 * bn * 4)
    assert items * 128 * bn * 4 == ws_bytes and items % base == 0
    ksplit = items // base
    total, sg = co * ci * k * k, 1
    while sg < 8 and total * sg < sms * 2048 and ksplit >= 16 * sg:
        sg *= 2
    return bn, ksplit, sg


# n, cin, cout, h, w, k, s -- and the (BN, SG) the planner picks on a 132-SM H100
WGRAD_CASES = [
    ((16, 64, 64, 150, 240, 1, 1), (64, 8)),         # L_SHAPES: 1x1 with few channels on the 150 x 240 map, ~258 splits
    ((16, 128, 128, 150, 240, 1, 1), (128, 8)),      # L_SHAPES (conv1 | conv2 pair)
    ((16, 64, 128, 300, 480, 3, 2), (64, 2)),        # L_SHAPES: the largest K (576 000 pixels)
    ((16, 128, 128, 75, 120, 3, 1), (128, 2)),
    ((16, 512, 256, 75, 120, 1, 1), (256, 4)),
    ((16, 512, 512, 38, 60, 1, 1), (256, 2)),
    ((16, 2048, 1024, 19, 30, 1, 1), (256, 1)),      # L_SHAPES: SPP conv2, the most outputs
    ((16, 256, 512, 75, 120, 3, 2), (256, 1)),       # stride 2, odd output height (38)
    ((16, 48, 96, 300, 480, 3, 2), (64, 2)),         # StreamYOLO-m widths (not multiples of 64)
    ((16, 192, 192, 75, 120, 3, 1), (256, 1)),
]


def _wgrad_ws_bytes(n, ci, co, h, w, k, s):
    x = torch.empty((n, h, w, ci), dtype=torch.bfloat16, device=DEV)
    ho, wo = ops.conv_out_hw(h, w, k, s)
    dy = torch.empty((n, ho, wo, co), dtype=torch.bfloat16, device=DEV)
    d = ops.SyConvWgradDesc()
    d.x, d.dy = View(x).st(), View(dy).st()
    d.kh, d.kw, d.stride = k, k, s
    return ops.lib().sy_conv2d_wgrad_workspace_bytes(C.byref(d))


def test_wgrad_cases_cover_every_reduce_variant():
    """The weight-gradient cases below reach every split-group instantiation of wgrad_reduce_kernel and every tile width."""
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    got = [wgrad_variant(c[1], c[2], c[5], _wgrad_ws_bytes(*c), sms) for c, _ in WGRAD_CASES]
    assert {v[2] for v in got} == {1, 2, 4, 8}, got
    assert {v[0] for v in got} == {64, 128, 256}, got


@pytest.mark.parametrize("case,variant", WGRAD_CASES, ids=lambda c: "x".join(map(str, c)))
def test_wgrad_production(case, variant):
    n, ci, co, h, w, k, s = case
    ho, wo = ops.conv_out_hw(h, w, k, s)
    xv, dyv = post_silu(n, h, w, ci, 1), small_grad(n, ho, wo, co, 2)
    start = torch.randn((co, ci, k, k), generator=_gen(3), device=DEV) * 0.1
    dw = start.clone()
    ws = ops.conv2d_wgrad(xv, dyv, k, s, dw, accumulate=True)
    torch.cuda.synchronize()
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    bn, ksplit, sg = wgrad_variant(ci, co, k, ws.numel(), sms)
    if sms == 132:
        assert (bn, sg) == variant, (bn, ksplit, sg)
    x64, dy64 = nchw64(xv), nchw64(dyv)
    pad = (k - 1) // 2
    grad = torch.nn.grad.conv2d_weight(x64, dw.shape, dy64, stride=s, padding=pad)
    s2 = torch.nn.grad.conv2d_weight(x64.square(), dw.shape, dy64.square(), stride=s, padding=pad)
    ref = start.double() + grad
    K = n * ho * wo
    check_sum(dw, ref, s2, K, f"wgrad{case} BN={bn} SG={sg}")
    # one 64-pixel K block left out: the block in the middle of the pixel range (flattened n, oh, ow order)
    p0 = (K // 64 // 2) * 64
    i0, i1 = p0 // (ho * wo), (p0 + 63) // (ho * wo)
    flat_src = dy64[i0:i1 + 1].permute(0, 2, 3, 1).reshape(-1, co)
    flat_dst = torch.zeros_like(flat_src)
    q0 = p0 - i0 * ho * wo
    flat_dst[q0:q0 + 64] = flat_src[q0:q0 + 64]
    blk = flat_dst.reshape(i1 + 1 - i0, ho, wo, co).permute(0, 3, 1, 2)
    part = torch.nn.grad.conv2d_weight(x64[i0:i1 + 1], dw.shape, blk, stride=s, padding=pad)
    assert float(part.abs().max()) > 0
    assert_rejects_sum(dw, ref - part, s2, K, f"wgrad{case}: K block at pixel {p0} left out")


# ------------------------------------------------------------------------------------------------ 2b. data gradient
# forward conv shapes (n, cin, cout, h, w, k, s, conv1 | conv2 pair); the data gradient maps cout -> cin channels
DGRAD_CASES = [
    (16, 64, 128, 300, 480, 3, 2, False),    # the largest: dx is 16 x 300 x 480 x 64
    (16, 128, 128, 150, 240, 1, 1, True),
    (16, 64, 64, 150, 240, 3, 1, False),
    (16, 256, 512, 75, 120, 3, 2, False),    # odd output height
    (16, 512, 512, 19, 30, 3, 1, False),
    (16, 1024, 1024, 19, 30, 1, 1, True),
    (16, 2048, 1024, 19, 30, 1, 1, False),
    (16, 48, 96, 300, 480, 3, 2, False),     # StreamYOLO-m widths
    (16, 192, 192, 75, 120, 1, 1, True),
]
DGRAD_TILINGS = {"planner": {}, "linear": dict(tile_mode=1), "halo": dict(tile_mode=2), "bn64": dict(tile_mode=1, tile_bn=64)}


@pytest.mark.parametrize("case", DGRAD_CASES, ids=lambda c: "x".join(map(str, c)))
def test_dgrad_fused_in_place(case):
    """gx += conv(dilate2(draw) or draw, flipped / transposed filter): FUSED with scale 1, shift 0, no activation, the
    residual input being the output view itself (the walk's in-place accumulation), under every forced tiling."""
    n, ci, co, h, w, k, s, pair = case
    ho, wo = ops.conv_out_hw(h, w, k, s)
    g = _gen(5)
    ws = [(torch.randn((co // 2 if pair else co, ci, k, k), generator=g, device=DEV) / math.sqrt(ci * k * k))
          for _ in range(2 if pair else 1)]
    wpk = ops.pack_conv_weight_dgrad(*ws)
    dyv = small_grad(n, ho, wo, co, 6)
    gx0 = (torch.randn((n, h, w, ci), generator=g, device=DEV) * 1e-2 * math.sqrt(co / ci)).to(torch.bfloat16)
    src = dyv
    if s == 2:
        src = View.empty(n, h, w, co, DEV)
        ops.dilate2(dyv, src)
    one, zero = torch.ones(ci, device=DEV), torch.zeros(ci, device=DEV)
    w64 = torch.cat(ws, 0).to(torch.bfloat16).double()
    dy64, pad = nchw64(dyv), (k - 1) // 2
    ref = nchw64(View(gx0)) + torch.nn.grad.conv2d_input((n, ci, h, w), w64, dy64, stride=s, padding=pad)
    # one 64-channel block of the reduction (cout 0..63) at the centre tap left out
    wb = torch.zeros_like(w64[:64])
    wb[:, :, k // 2, k // 2] = w64[:64, :, k // 2, k // 2]
    ref_omit = ref - torch.nn.grad.conv2d_input((n, ci, h, w), wb, dy64[:, :64], stride=s, padding=pad)
    for name, tiling in DGRAD_TILINGS.items():
        gx = View(gx0.clone())
        ops.conv2d(src, wpk, gx, (k, k), 1, ops.SY_CONV_FUSED, scale=one, shift=zero, act=0, res=gx, **tiling)
        torch.cuda.synchronize()
        got = nchw64(gx)
        check_close(got, ref, f"dgrad{case} {name}")
        assert outside_bf16(got, ref_omit) > 0, f"dgrad{case} {name}: the bar accepts a 64-channel block left out"


# ------------------------------------------------------------------------------------------------ 2c. BatchNorm + SiLU backward
def bn_bwd_rows(npix_group, c):
    """partial rows per statistics group of sy_bn_act_backward (bn_bwd.cu bwd_rows_for)"""
    lanes = min(c // 8, 256)
    per_row = (256 // lanes) * 4 * 2
    return min(296, -(-npix_group // per_row)) if npix_group > 0 else 0


# n, C, h, w, split (0: one statistics group), act, accumulate
BN_CASES = [
    (16, 48, 150, 240, 8, 1, False),     # 42 pixel lanes of 6 chunks (4 idle threads); 296 rows of 973 pixels
    (16, 64, 150, 240, 8, 1, True),
    (16, 96, 75, 120, 8, 0, False),      # 21 x 12 lanes
    (16, 192, 38, 60, 8, 1, True),       # 10 x 24 lanes, 228 rows (below the cap)
    (16, 512, 38, 60, 8, 1, False),      # lanes = 64, PL = 4
    (16, 1024, 19, 30, 8, 0, True),      # lanes = 128, PL = 2
    (8, 1024, 19, 30, 0, 1, False),      # one statistics group
]


def test_bn_cases_reach_the_row_cap():
    assert any(bn_bwd_rows((c[4] or c[0]) * c[2] * c[3], c[1]) == 296 for c in BN_CASES)
    assert any(bn_bwd_rows((c[4] or c[0]) * c[2] * c[3], c[1]) < 296 for c in BN_CASES)


@pytest.mark.parametrize("case", BN_CASES, ids=lambda c: "x".join(map(str, c)))
def test_bn_act_backward_production(case):
    n, c, h, w, split, act, acc = case
    eps = 1e-3
    g = _gen(7)
    mu = torch.rand(c, generator=g, device=DEV) * 4.0 - 2.0                # raw conv outputs: non-zero per-channel means
    sd = torch.rand(c, generator=g, device=DEV) + 0.5
    rawv = View((torch.randn((n, h, w, c), generator=g, device=DEV) * sd + mu).to(torch.bfloat16))
    dyv = small_grad(n, h, w, c, 8)
    raw64, dy64 = nchw64(rawv), nchw64(dyv)
    gamma, beta = torch.rand(c, generator=g, device=DEV) + 0.5, torch.rand(c, generator=g, device=DEV) - 0.5
    groups = [(0, split, 0), (split, n, 1)] if split else [(0, n, 0)]
    mean, invstd = torch.zeros((2, c), device=DEV), torch.ones((2, c), device=DEV)
    for a, b, gi in groups:                  # the statistics the forward saved (fp32)
        mean[gi] = raw64[a:b].mean((0, 2, 3)).float()
        invstd[gi] = (raw64[a:b].var((0, 2, 3), unbiased=False) + eps).rsqrt().float()
    scale = gamma[None] * invstd
    shift = beta[None] - mean * scale
    d0 = torch.randn((2, c), generator=g, device=DEV) if acc else torch.full((2, c), float("nan"), device=DEV)
    dgamma, dbeta = d0[0].clone(), d0[1].clone()
    draw = View.empty(n, h, w, c, DEV)
    ops.bn_act_backward(rawv, dyv, draw, scale, shift, mean, invstd, split, act, dgamma, dbeta, accumulate=acc)
    torch.cuda.synchronize()
    ss, mi = torch.stack([scale, shift]), torch.stack([mean, invstd])
    draw_ref, dg, db, s2g, s2b, t, dz = bn_act_backward_ref(raw64, dy64, ss, mi, groups, act)
    if acc:
        dg, db = dg + d0[0].double(), db + d0[1].double()
    check_close(nchw64(draw), draw_ref, f"bn backward{case}: d raw")
    K = n * h * w
    check_sum(dgamma, dg, s2g, K, f"bn backward{case}: dgamma")
    check_sum(dbeta, db, s2b, K, f"bn backward{case}: dbeta")
    # the reference formula is autograd of F.batch_norm + F.silu (float64, the group's own statistics)
    a, b, _ = groups[0]
    xr = raw64[a:b].clone().requires_grad_(True)
    gr, br = gamma.double().requires_grad_(True), beta.double().requires_grad_(True)
    z = F.batch_norm(xr, None, None, gr, br, True, 0.0, eps)
    (F.silu(z) if act else z).backward(dy64[a:b])
    m64, v64 = raw64[a:b].mean((0, 2, 3)), raw64[a:b].var((0, 2, 3), unbiased=False)
    iv64 = (v64 + eps).rsqrt()
    ss64 = torch.stack([gamma.double() * iv64, beta.double() - m64 * gamma.double() * iv64])[:, None]
    mi64 = torch.stack([m64, iv64])[:, None]
    d_ex, dg_ex, db_ex, _, _, _, _ = bn_act_backward_ref(raw64[a:b], dy64[a:b], ss64, mi64, [(0, b - a, 0)], act)
    assert torch.allclose(d_ex, xr.grad, rtol=1e-9, atol=1e-12 * float(xr.grad.abs().max()))
    assert torch.allclose(dg_ex, gr.grad, rtol=1e-9, atol=1e-9 * float(gr.grad.abs().max()))
    assert torch.allclose(db_ex, br.grad, rtol=1e-9, atol=1e-9 * float(br.grad.abs().max()))
    # one partial row's pixel share of group 0 left out
    rows0 = bn_bwd_rows((b - a) * h * w, c)
    share = -(-((b - a) * h * w) // rows0)
    r = rows0 // 2
    p0, p1 = r * share, min((b - a) * h * w, (r + 1) * share)
    tf, dzf = t.permute(0, 2, 3, 1).reshape(-1, c), dz.permute(0, 2, 3, 1).reshape(-1, c)
    assert_rejects_sum(dgamma, dg - tf[p0:p1].sum(0), s2g, K, f"bn backward{case}: dgamma, row {r} left out")
    assert_rejects_sum(dbeta, db - dzf[p0:p1].sum(0), s2b, K, f"bn backward{case}: dbeta, row {r} left out")


# ------------------------------------------------------------------------------------------------ 2d. head prediction convs
HEAD_LEVELS = [(75, 120, 0), (38, 60, 9000), (19, 30, 11280)]          # anchor offsets in a_total = 11 850
HEAD_CASES = ([(4, 256, h, w, off, 8) for h, w, off in HEAD_LEVELS]     # l_b4
              + [(8, 192, h, w, off, 8) for h, w, off in HEAD_LEVELS]   # m_b8
              + [(8, 128, h, w, off, 8) for h, w, off in HEAD_LEVELS]   # s_b8
              + [(4, 256, 75, 120, 0, nc) for nc in (1, 20, 3, 27)])    # NO = 6, 25 and the generic kernel (8 / 30 / 32 outputs)


def _head_ref(gl, fr, fc, w_reg, w_obj, w_cls):
    """float64 data and weight gradients of the three 1x1 prediction convs; gl [P, NO], fr / fc [P, C]"""
    d_rf = gl[:, :4] @ w_reg + gl[:, 4:5] @ w_obj
    d_cf = gl[:, 5:] @ w_cls
    dw = torch.cat([gl[:, :5].T @ fr, gl[:, 5:].T @ fc], 0)              # [NO, C]
    return d_rf, d_cf, dw


@pytest.mark.parametrize("case", HEAD_CASES, ids=lambda c: "x".join(map(str, c)))
def test_head_pred_backward_production(case):
    b, c, h, w, off, nc = case
    no = 5 + nc
    g = _gen(9)
    cfv, rfv = post_silu(b, h, w, c, 10), post_silu(b, h, w, c, 11)
    w_reg, w_obj, w_cls = [torch.randn((o, c), generator=g, device=DEV) * 0.05 for o in (4, 1, nc)]
    grad_raw = torch.randn((b, A_TOTAL, no), generator=g, device=DEV) * 1e-3     # every anchor set: only the level's are read
    dcf, drf = View.empty(b, h, w, c, DEV), View.empty(b, h, w, c, DEV)
    dws = [torch.full((o, c), float("nan"), device=DEV) for o in (4, 1, nc)]
    dbs = [torch.full((o,), float("nan"), device=DEV) for o in (4, 1, nc)]
    ops.head_pred_backward(grad_raw, cfv, rfv, dcf, drf, w_reg, w_obj, w_cls, A_TOTAL, off, *dws, *dbs)
    torch.cuda.synchronize()
    P = b * h * w
    gl = grad_raw[:, off:off + h * w].double().reshape(P, no)
    fr, fc = rfv.torch().double().reshape(P, c), cfv.torch().double().reshape(P, c)
    w64 = [t.double() for t in (w_reg, w_obj, w_cls)]
    d_rf, d_cf, dw_ref = _head_ref(gl, fr, fc, *w64)
    check_close(drf.torch().double().reshape(P, c), d_rf, f"head{case}: d reg_feat")
    check_close(dcf.torch().double().reshape(P, c), d_cf, f"head{case}: d cls_feat")
    _, _, s2w = _head_ref(gl.square(), fr.square(), fc.square(), *w64)
    dw = torch.cat(dws, 0)
    check_sum(dw, dw_ref, s2w, P, f"head{case}: dW")
    db, db_ref, s2b = torch.cat(dbs), gl.sum(0), gl.square().sum(0)
    check_sum(db, db_ref, s2b, P, f"head{case}: db")
    # one 256-pixel partial row left out
    rows = -(-P // 256)
    r = rows // 2
    q0, q1 = 256 * r, min(P, 256 * r + 256)
    _, _, part = _head_ref(gl[q0:q1], fr[q0:q1], fc[q0:q1], *w64)
    assert_rejects_sum(dw, dw_ref - part, s2w, P, f"head{case}: dW, row {r} left out")
    assert_rejects_sum(db, db_ref - gl[q0:q1].sum(0), s2b, P, f"head{case}: db, row {r} left out")


def test_head_pred_backward_rejects_28_classes():
    b, c, h, w = 1, 64, 8, 10
    cfv, rfv = post_silu(b, h, w, c, 12), post_silu(b, h, w, c, 13)
    w_reg, w_obj, w_cls = [torch.zeros((o, c), device=DEV) for o in (4, 1, 28)]
    grad_raw = torch.zeros((b, h * w, 33), device=DEV)
    dws = [torch.zeros((o, c), device=DEV) for o in (4, 1, 28)]
    dbs = [torch.zeros((o,), device=DEV) for o in (4, 1, 28)]
    with pytest.raises(RuntimeError, match=f"libstreamyolo_sm100 error {SY_EINVAL}:"):
        ops.head_pred_backward(grad_raw, cfv, rfv, View.empty(b, h, w, c, DEV), View.empty(b, h, w, c, DEV), w_reg, w_obj,
                               w_cls, h * w, 0, *dws, *dbs)


# ------------------------------------------------------------------------------------------------ 2e. loss backward
def _edge_ties(outputs, fut):
    """Predictions whose box equals their ground truth's, and predictions sharing its x edges (same cx and w): the 0.5 tie
    split of the IoU gradient.  Modifies ``outputs`` in place."""
    for bi in range(outputs.shape[0]):
        for gt in fut[bi][:6]:
            if gt[3] <= 0:
                continue
            d = (outputs[bi, :, 0:4] - gt[1:5]).abs().sum(1)
            idx = torch.topk(d, 2, largest=False).indices
            outputs[bi, idx[0], 0:4] = gt[1:5]
            outputs[bi, idx[1], 0] = gt[1]
            outputs[bi, idx[1], 2] = gt[3]


# b, ground truths per image, gamma, loss scale
LOSS_CASES = [(4, 0, 1.0, 1.0), (4, 1, 1.5, 1.0), (4, 12, 1.0, 64.0), (8, 12, 1.5, 1.0), (4, 120, 1.5, 0.25),
              (8, 120, 1.0, 1.0)]


@pytest.mark.parametrize("b,n_gt,gamma,gscale", LOSS_CASES)
def test_tal_loss_backward_full_anchor_count(b, n_gt, gamma, gscale):
    """grad_outputs, grad_origin and grad_raw of sy_tal_loss_backward against float64 autograd through the oracle's loss on
    the same fp32 head outputs, after checking that the kernel's assignment equals the oracle's bit for bit.  Bar: the
    kernel evaluates each gradient in a chain of ~2^4 fp32 operations; box edges (and the TAL IoU behind the weights) are
    differences of coordinates up to ~2^10 px for boxes down to ~2^3 px, which costs up to 2^7 of the relative precision:
    |err| <= 2^-24 * 2^4 * 2^7 * 2 = 2^-12 of (|ref| + the rms of the column's non-zero entries); the rms term covers the
    box-size gradients, which are differences of two edge terms and may cancel."""
    fut, cur = _labels(b, n_gt, 17 + n_gt)
    if n_gt >= 12:
        fut[1] = 0                                            # an empty image
        cur[1] = 0
        cur[2] = 0                                            # future labels without current ones: TAL weight 1
    outputs, origin = _synthetic_head_outputs(b, fut, 19 + n_gt, dup_pred=n_gt >= 12)
    _edge_ties(outputs, fut)
    ig_thr, ig_val = 0.5, 1.6
    o = StreamYoloOracle(OracleCfg(gamma=gamma, ignore_thr=ig_thr, ignore_value=ig_val), {})
    grid64 = tuple(t.double() for t in o.grids(HW, STRIDES))
    out64, org64 = outputs.double().requires_grad_(True), origin.double().requires_grad_(True)
    ref = o.losses(out64, org64, grid64, (fut, cur), return_aux=True, dtype=F64)
    (ref["total_loss"] * gscale).backward()
    gout_ref = out64.grad
    gorg_ref = org64.grad if org64.grad is not None else torch.zeros_like(org64)
    ws = torch.empty(ops.tal_loss_workspace_bytes(b, A_TOTAL, 120, 8), dtype=torch.uint8, device=DEV)
    loss = torch.empty(6, device=DEV)
    fg = torch.empty((b, A_TOTAL), dtype=torch.int32, device=DEV)
    mt = torch.empty((b, A_TOTAL), dtype=torch.int32, device=DEV)
    pi = torch.empty((b, A_TOTAL), device=DEV)
    od, ogd, fd, cd = outputs.to(DEV), origin.to(DEV), fut.to(DEV), cur.to(DEV)
    ops.tal_loss(od, ogd, fd, cd, HW, STRIDES, gamma, ig_thr, ig_val, True, ws, loss, fg, mt, pi)
    g_out = torch.full((b, A_TOTAL, 13), float("nan"), device=DEV)
    g_org = torch.full((b, A_TOTAL, 4), float("nan"), device=DEV)
    g_raw = torch.full((b, A_TOTAL, 13), float("nan"), device=DEV)
    ops.tal_loss_backward(od, ogd, fd, HW, STRIDES, gamma, True, ws, gscale, grad_outputs=g_out, grad_origin=g_org,
                          grad_raw=g_raw)
    torch.cuda.synchronize()
    aux = ref["aux"]
    assert torch.equal(fg.cpu().bool(), aux["fg"]), "foreground set differs from the oracle's"
    assert torch.equal(mt.cpu().long(), aux["matched"]), "matched GT ids differ from the oracle's"
    nfg = int(aux["fg"].sum())
    assert (n_gt == 0) == (nfg == 0)
    if n_gt:                                                  # the tie branches are reached
        bi, ai = aux["fg"].nonzero(as_tuple=True)
        t = fut[bi, aux["matched"][bi, ai], 1:5]
        assert int(((outputs[bi, ai, 0] == t[:, 0]) & (outputs[bi, ai, 2] == t[:, 2])).sum()) > 0
    _, _, gs = grid64
    graw_ref = gout_ref.clone()
    graw_ref[..., 0:2] = gout_ref[..., 0:2] * gs[None, :, None] + gorg_ref[..., 0:2]
    graw_ref[..., 2:4] = gout_ref[..., 2:4] * out64.detach()[..., 2:4] + gorg_ref[..., 2:4]
    for got, want, what in ((g_out, gout_ref, "grad_outputs"), (g_org, gorg_ref, "grad_origin"), (g_raw, graw_ref, "grad_raw")):
        got = got.cpu().double()
        assert bool(torch.isfinite(got).all()), what
        nz = (want != 0).sum((0, 1)).clamp(min=1)
        rms = (want.square().sum((0, 1)) / nz).sqrt()                            # per column, over its non-zero entries
        err, tol = (got - want).abs(), 2.0 ** -12 * (want.abs() + rms)
        ratio = err / tol.clamp(min=1e-300)
        worst = int(ratio.argmax())
        assert bool((err <= tol).all()), \
            f"{what}: worst err / tol {float(ratio.max()):.3g} at column {worst % want.shape[2]}: " \
            f"got {float(got.flatten()[worst]):.6g}, want {float(want.flatten()[worst]):.6g}"


# ------------------------------------------------------------------------------------------------ 2f. glue backward
@pytest.mark.parametrize("n,c,hi,wi,ho,wo", [(8, 512, 19, 30, 38, 60), (8, 256, 38, 60, 75, 120)])
def test_upsample_nearest_backward_pan(n, c, hi, wi, ho, wo):
    """the l PAN's two upsamples; the gradient is read from a channel slice of the concat buffer, like in the walk"""
    cat = small_grad(n, ho, wo, 2 * c, 14, scale=1.0)
    dy = cat.ch(c, c)
    x = torch.zeros((n, c, hi, wi), dtype=F64, device=DEV, requires_grad=True)
    F.interpolate(x, size=(ho, wo), mode="nearest").backward(nchw64(dy))
    dx = View.empty(n, hi, wi, c, DEV)
    ops.upsample_nearest_backward(dy, dx)
    torch.cuda.synchronize()
    check_close(nchw64(dx), x.grad, "upsample backward", ulp=2.0 ** -8)        # one rounding of an exact fp32 sum


def test_spp_maxpool_backward_production():
    n, c, h, w = 16, 512, 19, 30
    g = _gen(15)
    xq = (torch.randint(-6, 7, (n, h, w, c), generator=g, device=DEV).float() * 0.25).to(torch.bfloat16)   # ties common
    xv = View(xq)
    dys = [small_grad(n, h, w, c, 16 + i, scale=1.0) for i in range(3)]
    x64 = nchw64(xv).requires_grad_(True)
    for k, d in zip((5, 9, 13), dys):
        F.max_pool2d(x64, k, 1, k // 2).backward(nchw64(d))
    dx = View.empty(n, h, w, c, DEV)
    ops.spp_maxpool_backward(xv, *dys, dx)
    torch.cuda.synchronize()
    check_close(nchw64(dx), x64.grad, "spp backward", ulp=2.0 ** -8)


def test_add_production_slices():
    """y += x into a channel slice of a wider buffer (the walk's accumulation into concat buffers): fp32 add, one rounding"""
    n, c, h, w = 8, 256, 75, 120
    xv = small_grad(n, h, w, c, 19, scale=1.0)
    big = small_grad(n, h, w, 2 * c, 20, scale=1.0)
    before = big.torch().clone()
    y = big.ch(c, c)
    want = (xv.torch().float() + y.torch().float()).to(torch.bfloat16)
    ops.add_(xv, y)
    torch.cuda.synchronize()
    assert torch.equal(y.torch(), want)
    assert torch.equal(big.ch(0, c).torch(), before[..., :c]), "neighbouring slice was overwritten"
