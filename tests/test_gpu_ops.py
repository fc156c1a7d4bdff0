"""GPU: every kernel of libstreamyolo_sm100 (through the C ABI) against a plain PyTorch fp32
reference of the same op evaluated on the SAME bf16-rounded operands.

Tolerances (written here once):
  * conv outputs are stored as bf16: |err| <= 2^-8 * |ref| + 2^-8 * rms(ref)   (one bf16 ulp + accumulation noise)
  * statistic partial sums (fp32): relative 2e-3 of sqrt(count)*rms
  * integer / index / max-pool / copy results: bit exact
"""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

from streamyolo_b200 import ops  # noqa: E402
from streamyolo_b200.ops import View  # noqa: E402

DEV = "cuda"


def bf(t):
    return t.to(torch.bfloat16).float()


def rand_act(n, c, h, w, seed, scale=1.0):
    g = torch.Generator().manual_seed(seed)
    return bf(torch.randn(n, c, h, w, generator=g) * scale).to(DEV)


def rand_w(co, ci, k, seed):
    g = torch.Generator().manual_seed(seed)
    return bf(torch.randn(co, ci, k, k, generator=g) / (ci * k * k) ** 0.5).to(DEV)


def check_close(got, ref, what, ulp=2.0 ** -7):
    got, ref = got.float(), ref.float()
    rms = ref.pow(2).mean().sqrt().item() + 1e-12
    err = (got - ref).abs()
    tol = ulp * ref.abs() + ulp * rms
    bad = (err > tol)
    frac = bad.float().mean().item()
    rel = ((got - ref).norm() / (ref.norm() + 1e-12)).item()
    assert frac == 0.0 and np.isfinite(rel), f"{what}: {bad.sum().item()} / {bad.numel()} outside tolerance, " \
        f"max err {err.max().item():.4g}, rms {rms:.4g}, rel l2 {rel:.3g}"
    return rel


TC_IMPLS = ["tc", "tc_bn64", "tc_halo"]


def tc_impl(impl):
    """ops.conv2d's ``impl`` and tiling keywords of a variant under test.  'tc' = linear M tiles (im2col-mode TMA, the
    default), 'tc_bn64' = linear tiles with the tile width forced to 64 (the BN = 64 kernel on layers the planner gives
    BN = 128, i.e. several N tiles and the M-band walk), 'tc_halo' = one halo load per tile and channel block for the 3x3
    stride-1 convs (linear tiles elsewhere); all are product paths."""
    return {"tc": ("tc", dict(tile_mode=1)), "tc_bn64": ("tc", dict(tile_mode=1, tile_bn=64)),
            "tc_halo": ("tc", dict(tile_mode=2))}.get(impl, (impl, {}))


CONV_CASES = [
    # n, cin, cout, h, w, k, s
    (2, 64, 64, 8, 16, 1, 1),
    (1, 128, 128, 75, 120, 3, 1),
    (2, 64, 128, 150, 240, 3, 2),
    (2, 128, 256, 75, 120, 3, 2),      # odd height -> 38
    (2, 256, 512, 38, 60, 3, 2),
    (2, 512, 1024, 19, 30, 1, 1),
    (3, 8, 16, 15, 20, 3, 1),          # tiny test-model widths
    (2, 16, 32, 15, 20, 3, 2),
    (2, 48, 96, 38, 60, 1, 1),         # StreamYOLO-m widths (not multiples of 64)
    (2, 96, 96, 19, 30, 3, 1),
    (1, 1024, 512, 19, 30, 1, 1),
    (2, 256, 256, 75, 120, 3, 1),      # head tower conv (largest single conv of l)
    (3, 64, 64, 13, 17, 3, 1),         # 221 pixels per image: every linear tile straddles an image boundary
    (5, 32, 64, 9, 7, 3, 2),           # stride 2 on odd sizes, images much smaller than a tile
]


@pytest.mark.parametrize("impl", ["simt"] + TC_IMPLS)
@pytest.mark.parametrize("case", CONV_CASES, ids=lambda c: "x".join(map(str, c)))
def test_conv_raw(case, impl):
    n, ci, co, h, w, k, s = case
    impl, tiling = tc_impl(impl)
    if impl == "simt" and ci * co * h * w * k * k * n > 3e10:
        pytest.skip("too slow on the CUDA-core cross-check kernel")
    x = rand_act(n, ci, h, w, 1)
    wt = rand_w(co, ci, k, 2)
    ref = F.conv2d(x, wt, None, s, (k - 1) // 2)
    xv = ops.from_nchw(x)
    ho, wo = ops.conv_out_hw(h, w, k, s)
    y = View.empty(n, ho, wo, co, DEV)
    y.buf.fill_(float("nan"))
    rows = ops.conv_stat_rows()
    partials = torch.full((rows, 4 * co), float("nan"), device=DEV) if impl == "tc" else None
    split = 1 if n > 1 else 0
    ops.conv2d(xv, ops.pack_conv_weight(wt), y, k, s, ops.SY_CONV_RAW, impl=impl, partials=partials, split_n=split,
               **tiling)
    torch.cuda.synchronize()
    got = y.nchw_float()
    check_close(got, ref, f"conv_{impl}{case}")
    if impl == "tc":
        # per-CTA partial rows [cta][c][group][sum|sumsq]; rows of CTAs that did not run stay NaN
        pr = torch.nan_to_num(partials.view(rows, co, 2, 2)).sum(0).permute(1, 2, 0)
        st = got    # statistics are defined on the stored (rounded) values
        groups = [(0, split), (split, n)] if split else [(0, n)]
        for g, (a0, a1) in enumerate(groups):
            part = st[a0:a1]
            cnt = (a1 - a0) * ho * wo
            rms = part.pow(2).mean().sqrt().item()
            assert torch.allclose(pr[g, 0], part.sum((0, 2, 3)), rtol=0, atol=2e-3 * rms * cnt ** 0.5 + 1e-3), "sum"
            assert torch.allclose(pr[g, 1], part.pow(2).sum((0, 2, 3)), rtol=2e-3, atol=1e-3), "sumsq"


@pytest.mark.parametrize("tiles", TC_IMPLS)
def test_conv_tc_bn_finalize_then_separate_apply(tiles):
    _bn_finalize_then_apply(**tc_impl(tiles)[1])


def _bn_finalize_then_apply(**tiling):
    """RAW conv that also finalizes BatchNorm in its tail (grid barrier + parallel reduce; two groups, two
    parameter segments, running statistics), then the normalise pass with SiLU + residual; against
    F.batch_norm on the stored conv output.  Three launches in a row: the sync counters must come back to zero after each
    (graph replay safe) and num_batches_tracked must count two statistics groups per launch."""
    n, ci, co, h, w = 4, 64, 128, 19, 30
    x, wt = rand_act(n, ci, h, w, 61), rand_w(co, ci, 1, 62)
    g = torch.Generator().manual_seed(63)
    gamma, beta = (torch.rand(co, generator=g) + 0.5).to(DEV), (torch.rand(co, generator=g) - 0.5).to(DEV)
    rm, rv = (torch.rand(co, generator=g) * 0.2).to(DEV), (torch.rand(co, generator=g) + 0.5).to(DEV)
    rm_ref, rv_ref = rm.clone(), rv.clone()
    half = co // 2
    nbt = [torch.zeros((), dtype=torch.long, device=DEV) for _ in range(2)]
    segs = [(gamma[:half].contiguous(), beta[:half].contiguous(), rm[:half], rv[:half], nbt[0], 0),
            (gamma[half:].contiguous(), beta[half:].contiguous(), rm[half:], rv[half:], nbt[1], half)]
    raw = View.empty(n, h, w, co, DEV)
    y = View.empty(n, h, w, co, DEV)
    resid = rand_act(n, co, h, w, 64)
    partials = torch.empty((ops.conv_stat_rows(), 4 * co), device=DEV)
    ss = torch.empty((2, 2, co), device=DEV)
    sync = torch.zeros(2, dtype=torch.int32, device=DEV)
    resid_v, x_v = ops.from_nchw(resid), ops.from_nchw(x)
    for rep in range(3):
        y.buf.fill_(float("nan"))
        rows = ops.conv2d(x_v, ops.pack_conv_weight(wt), raw, 1, 1, ops.SY_CONV_RAW, partials=partials,
                          split_n=2, bn=segs, momentum=0.03, eps=1e-3, scale_shift=ss, sync=sync, act=1, **tiling)
        assert 1 <= rows <= ops.conv_stat_rows()
        ops.bn_act_apply(raw, ss[0].data_ptr(), ss[1].data_ptr(), 2, 1, resid_v, y)
        torch.cuda.synchronize()
        assert sync.tolist() == [0, 0]
        rawf = raw.nchw_float()
        refs = []
        for gi in range(2):
            refs.append(F.batch_norm(rawf[gi * 2:(gi + 1) * 2], rm_ref, rv_ref, gamma, beta, True, 0.03, 1e-3))
        ref = F.silu(torch.cat(refs, 0)) + resid
        check_close(y.nchw_float(), ref, "bn_train_apply")
        assert torch.allclose(rm, rm_ref, rtol=1e-4, atol=1e-5) and torch.allclose(rv, rv_ref, rtol=1e-4, atol=1e-5)
        assert int(nbt[0]) == 2 * (rep + 1) and int(nbt[1]) == 2 * (rep + 1)


@pytest.mark.parametrize("impl", ["simt"] + TC_IMPLS)
def test_conv_fused_residual_slices(impl):
    """FUSED epilogue (scale, shift, SiLU, residual) reading and writing channel slices, in place."""
    impl, tiling = tc_impl(impl)
    n, ci, co, h, w = 2, 64, 64, 19, 30
    x = rand_act(n, ci, h, w, 3)
    wt = rand_w(co, ci, 3, 4)
    g = torch.Generator().manual_seed(5)
    scale = (torch.rand(co, generator=g) + 0.5).to(DEV)
    shift = (torch.rand(co, generator=g) - 0.5).to(DEV)
    resid = rand_act(n, co, h, w, 6)
    ref = F.silu(F.conv2d(x, wt, None, 1, 1) * scale[None, :, None, None] + shift[None, :, None, None]) + resid
    big_in = View.empty(n, h, w, 3 * ci, DEV)
    big_in.buf.fill_(7.0)
    xin = big_in.ch(ci, ci)
    xin.torch().copy_(x.permute(0, 2, 3, 1))
    big_out = View.empty(n, h, w, 2 * co, DEV)
    big_out.buf.fill_(-3.0)
    yv = big_out.ch(co, co)
    yv.torch().copy_(resid.permute(0, 2, 3, 1))      # residual lives where the output goes (in place)
    ops.conv2d(xin, ops.pack_conv_weight(wt), yv, 3, 1, ops.SY_CONV_FUSED, impl=impl, scale=scale, shift=shift,
               act=1, res=yv, **tiling)
    torch.cuda.synchronize()
    check_close(yv.nchw_float(), ref, f"conv_fused_{impl}")
    assert (big_out.ch(0, co).torch() == -3.0).all(), "neighbouring slice was overwritten"


def test_conv_tc_matches_simt_bitwise_mostly():
    """Same operands, two kernels: differences only from fp32 summation order (<= 1 bf16 ulp)."""
    n, ci, co, h, w, k, s = 2, 128, 128, 38, 60, 3, 1
    x, wt = rand_act(n, ci, h, w, 11), rand_w(co, ci, k, 12)
    xv, wp = ops.from_nchw(x), ops.pack_conv_weight(wt)
    a, b = View.empty(n, h, w, co, DEV), View.empty(n, h, w, co, DEV)
    ops.conv2d(xv, wp, a, k, s, ops.SY_CONV_RAW, impl="tc")
    ops.conv2d(xv, wp, b, k, s, ops.SY_CONV_RAW, impl="simt")
    torch.cuda.synchronize()
    diff = (a.torch().float() - b.torch().float()).abs()
    assert (diff > 0).float().mean().item() < 0.05
    check_close(a.torch().float(), b.torch().float(), "tc vs simt")


@pytest.mark.parametrize("impl", ["simt"] + TC_IMPLS)
def test_stem_focus(impl):
    impl, tiling = tc_impl(impl)
    b, h, w, co = 2, 120, 160, 16
    g = torch.Generator().manual_seed(0)
    x = (torch.rand(b, 6, h, w, generator=g) * 255).to(DEV)
    wt = rand_w(co, 12, 3, 7)
    xin = View.empty(2 * b, h // 2, w // 2, 64, DEV)
    ops.focus_pack(x, 2, xin)
    y = View.empty(2 * b, h // 2, w // 2, co, DEV)
    ops.conv2d(xin, ops.pack_stem_weight(wt), y, ops.STEM_K, 1, ops.SY_CONV_RAW, impl=impl, **tiling)
    torch.cuda.synchronize()
    xs = bf(torch.cat([x[:, 0:3], x[:, 3:6]], 0))
    foc = torch.cat([xs[..., ::2, ::2], xs[..., 1::2, ::2], xs[..., ::2, 1::2], xs[..., 1::2, 1::2]], 1)
    packed = xin.nchw_float()
    assert torch.equal(packed[:, 16:28], foc) and (packed[:, 28:32] == 0).all()            # centre tap: exact
    assert (packed[:, 44:64] == 0).all()                                                    # tap padding + row padding
    assert torch.equal(packed[:, 0:12, :, 1:], foc[..., :-1]) and (packed[:, 0:12, :, 0] == 0).all()
    assert torch.equal(packed[:, 32:44, :, :-1], foc[..., 1:]) and (packed[:, 32:44, :, -1] == 0).all()
    ref = F.conv2d(foc, wt, None, 1, 1)
    check_close(y.nchw_float(), ref, "stem")


@pytest.mark.parametrize("groups", [1, 2])
def test_bn_stats_finalize_apply(groups):
    n, c, h, w = 4, 64, 19, 30
    x = rand_act(n, c, h, w, 21, scale=2.0) + 0.7
    x = bf(x)
    xv = ops.from_nchw(x)
    P = ops.stats_num_partials(n, h * w)
    partials = torch.empty((P, 2, c), device=DEV)
    ops.channel_stats(xv, partials)
    g = torch.Generator().manual_seed(22)
    gamma, beta = (torch.rand(c, generator=g) + 0.5).to(DEV), (torch.rand(c, generator=g) - 0.5).to(DEV)
    rm, rv = torch.zeros(c, device=DEV) + 0.1, torch.ones(c, device=DEV) * 0.9
    nbt = torch.zeros((), dtype=torch.long, device=DEV)
    sc = torch.empty((2, 2, c), device=DEV)
    split = n // 2 if groups == 2 else n
    ops.bn_finalize(partials, (P // n) * split if groups == 2 else 0, groups, split * h * w, gamma, beta, rm, rv, nbt,
                    0.03, 1e-3, sc[0], sc[1])
    resid = rand_act(n, c, h, w, 23)
    y = View.empty(n, h, w, c, DEV)
    ops.bn_act_apply(xv, sc[0].data_ptr(), sc[1].data_ptr(), split, 1, ops.from_nchw(resid), y)
    torch.cuda.synchronize()
    rm_ref, rv_ref = torch.zeros(c, device=DEV) + 0.1, torch.ones(c, device=DEV) * 0.9
    refs = []
    for gi in range(groups):
        xs = x[gi * split:(gi + 1) * split]
        refs.append(F.batch_norm(xs, rm_ref, rv_ref, gamma, beta, True, 0.03, 1e-3))
    ref = F.silu(torch.cat(refs, 0)) + resid
    check_close(y.nchw_float(), ref, "bn_apply")
    assert torch.allclose(rm, rm_ref, rtol=1e-4, atol=1e-5) and torch.allclose(rv, rv_ref, rtol=1e-4, atol=1e-5)
    assert int(nbt) == groups


def test_upsample_nearest_index_exact():
    for (hi, wi, ho, wo) in [(19, 30, 38, 60), (38, 60, 75, 120), (8, 10, 15, 20), (4, 5, 8, 10)]:
        x = rand_act(2, 16, hi, wi, 31)
        y = View.empty(2, ho, wo, 32, DEV)
        ops.upsample_nearest(ops.from_nchw(x), y.ch(16, 16))
        torch.cuda.synchronize()
        ref = F.interpolate(x, size=(ho, wo), mode="nearest")
        assert torch.equal(y.ch(16, 16).nchw_float(), ref), (hi, wi, ho, wo)


def test_spp_and_copy_exact():
    x = rand_act(2, 32, 19, 30, 41)
    s = View.empty(2, 19, 30, 128, DEV)
    ops.copy(ops.from_nchw(x), s.ch(0, 32))
    ops.spp_maxpool(s.ch(0, 32), s.ch(32, 32), s.ch(64, 32), s.ch(96, 32))
    torch.cuda.synchronize()
    ref = torch.cat([x] + [F.max_pool2d(x, k, 1, k // 2) for k in (5, 9, 13)], 1)
    assert torch.equal(s.nchw_float(), ref)


@pytest.mark.parametrize("shape", [(2, 64, 15, 20, 8), (2, 64, 15, 20, 3), (1, 32, 9, 11, 80), (8, 256, 75, 120, 8),
                                   (2, 64, 15, 20, 1), (2, 64, 15, 20, 20)],
                         ids=["nc8", "nc3-generic", "nc80-generic", "level0-l", "nc1", "nc20"])
def test_head_pred_decode(shape):
    """Prediction convs + decode against F.conv2d.  Class counts without a compiled instantiation take the generic kernel
    (the reference head accepts any num_classes, tal_head.py:27); the benchmark's level-0 shape (72 000 pixels) takes the
    two-pixels-per-thread variant, whose output must be bit-identical to the one-pixel variant that one image of it
    (9 000 pixels) takes (same per-pixel arithmetic)."""
    b, c, h, w, nc = shape
    cf, rf = rand_act(b, c, h, w, 51), rand_act(b, c, h, w, 52)
    g = torch.Generator().manual_seed(53)
    wr, br = (torch.randn(4, c, generator=g) * 0.05).to(DEV), (torch.randn(4, generator=g) * 0.1).to(DEV)
    wo_, bo = (torch.randn(1, c, generator=g) * 0.05).to(DEV), (torch.randn(1, generator=g) * 0.1).to(DEV)
    wc, bc = (torch.randn(nc, c, generator=g) * 0.05).to(DEV), (torch.randn(nc, generator=g) * 0.1).to(DEV)
    a_total, off, stride = h * w + 37, 37, 16
    for train in (True, False):
        out = torch.zeros((b, a_total, 5 + nc), device=DEV)
        origin = torch.zeros((b, a_total, 4), device=DEV) if train else None
        ops.head_pred_decode(ops.from_nchw(cf), ops.from_nchw(rf), wr, br, wo_, bo, wc, bc, stride, off, a_total, out,
                             origin, sigmoid=not train, decode=True)
        torch.cuda.synchronize()
        reg = F.conv2d(rf, wr[:, :, None, None], br)
        obj = F.conv2d(rf, wo_[:, :, None, None], bo)
        cls = F.conv2d(cf, wc[:, :, None, None], bc)
        raw = torch.cat([reg, obj, cls], 1).flatten(2).permute(0, 2, 1)
        yv, xv = torch.meshgrid(torch.arange(h, device=DEV), torch.arange(w, device=DEV), indexing="ij")
        ref = raw.clone()
        ref[..., 0] = (raw[..., 0] + xv.reshape(-1)) * stride
        ref[..., 1] = (raw[..., 1] + yv.reshape(-1)) * stride
        ref[..., 2:4] = torch.exp(raw[..., 2:4]) * stride
        if not train:
            ref[..., 4:] = raw[..., 4:].sigmoid()
        assert torch.allclose(out[:, off:], ref, rtol=1e-4, atol=1e-4)
        if train:
            assert torch.allclose(origin[:, off:], raw[..., :4], rtol=1e-4, atol=1e-5)
        assert (out[:, :off] == 0).all()
        if nc == 8:
            o1 = torch.zeros((b, a_total, 5 + nc), device=DEV)
            for i in range(b):                         # one image at a time: the one-pixel-per-thread variant
                ops.head_pred_decode(ops.from_nchw(cf[i:i + 1]), ops.from_nchw(rf[i:i + 1]), wr, br, wo_, bo, wc, bc, stride,
                                     off, a_total, o1[i:i + 1], None, sigmoid=not train, decode=True)
            torch.cuda.synchronize()
            assert torch.equal(o1, out)


# ---------------------------------------------------------------------------------------------- backward bricks (SURVEY 8 row a19)
WGRAD_CASES = [
    # n, cin, cout, h, w, k, s
    (2, 64, 64, 19, 30, 1, 1),
    (2, 128, 128, 38, 60, 3, 1),
    (2, 64, 128, 40, 60, 3, 2),        # stride 2
    (2, 128, 256, 75, 120, 3, 2),      # stride 2, odd height -> 38
    (1, 256, 512, 19, 30, 3, 1),       # several M tiles, BN = 256
    (3, 8, 16, 15, 20, 3, 1),          # tiny widths: channel boxes mostly out of bounds
    (2, 96, 96, 19, 30, 3, 1),         # StreamYOLO-m width
    (2, 512, 1024, 19, 30, 1, 1),
    (5, 32, 64, 9, 7, 3, 2),           # fewer pixels than one K block per image
]


@pytest.mark.parametrize("case", WGRAD_CASES, ids=lambda c: "x".join(map(str, c)))
def test_conv_wgrad(case):
    """Tensor-core weight gradient (split-K over pixels + fixed-order reduction) against autograd of F.conv2d on the same
    bf16-rounded operands in fp32.  Tolerance: 2e-4 of the largest gradient entry (fp32 accumulation, other order)."""
    n, ci, co, h, w, k, s = case
    x = rand_act(n, ci, h, w, 21)
    ho, wo = ops.conv_out_hw(h, w, k, s)
    dy = rand_act(n, co, ho, wo, 22)
    wt = torch.zeros(co, ci, k, k, device=DEV, requires_grad=True)
    F.conv2d(x, wt, None, s, (k - 1) // 2).backward(dy)
    ref = wt.grad
    dw = torch.full((co, ci, k, k), float("nan"), device=DEV)
    ops.conv2d_wgrad(ops.from_nchw(x), ops.from_nchw(dy), k, s, dw)
    torch.cuda.synchronize()
    scale = ref.abs().max().item()
    err = (dw - ref).abs().max().item()
    assert torch.isfinite(dw).all() and err <= 2e-4 * scale, f"wgrad{case}: max err {err:.4g} vs max |ref| {scale:.4g}"
    # accumulate mode adds to what is there
    ops.conv2d_wgrad(ops.from_nchw(x), ops.from_nchw(dy), k, s, dw, accumulate=True)
    torch.cuda.synchronize()
    assert (dw - 2 * ref).abs().max().item() <= 4e-4 * scale


@pytest.mark.parametrize("case", [(2, 64, 128, 19, 30, 3), (2, 128, 64, 38, 60, 1), (1, 256, 256, 38, 60, 3)],
                         ids=lambda c: "x".join(map(str, c)))
def test_conv_dgrad_stride1(case):
    """Data gradient of a stride-1 conv = the forward tensor-core kernel on the flipped, channel-transposed filter."""
    n, ci, co, h, w, k = case
    x = rand_act(n, ci, h, w, 31).requires_grad_(True)
    wt = rand_w(co, ci, k, 32)
    dy = rand_act(n, co, h, w, 33)
    F.conv2d(x, wt, None, 1, (k - 1) // 2).backward(dy)
    dx = View.empty(n, h, w, ci, DEV)
    ops.conv2d(ops.from_nchw(dy), ops.pack_conv_weight_dgrad(wt), dx, k, 1, ops.SY_CONV_RAW)
    torch.cuda.synchronize()
    check_close(dx.nchw_float(), x.grad, f"dgrad{case}")


@pytest.mark.parametrize("case", [(4, 64, 128, 19, 30, 3, 2), (2, 128, 64, 38, 60, 1, 0), (4, 32, 32, 16, 20, 3, 2)],
                         ids=lambda c: "x".join(map(str, c)))
def test_baseconv_backward_chain(case):
    """Backward of one whole BaseConv (conv -> train-mode BatchNorm with two statistics groups -> SiLU) through the
    product's kernels: sy_bn_act_backward -> draw (bf16), then the data gradient (forward tensor-core kernel on the
    flipped filter) and the tensor-core weight gradient; against torch autograd in fp32 on the same bf16-rounded operands
    (the conv output is rounded to bf16 with a straight-through estimator, as the product stores it).
    Tolerances: rel l2 1e-2 for dx / dW (draw is stored in bf16), 5e-3 for dgamma / dbeta."""
    n, ci, co, h, w, k, split = case
    eps = 1e-3
    x = rand_act(n, ci, h, w, 41)
    wt = rand_w(co, ci, k, 42)
    g = torch.Generator().manual_seed(43)
    gamma, beta = (torch.rand(co, generator=g) + 0.5).to(DEV), (torch.rand(co, generator=g) - 0.5).to(DEV)
    dy = rand_act(n, co, h, w, 44, scale=0.1)
    # ---- reference
    xr, wr = x.clone().requires_grad_(True), wt.clone().requires_grad_(True)
    gr, br = gamma.clone().requires_grad_(True), beta.clone().requires_grad_(True)
    raw_ref = F.conv2d(xr, wr, None, 1, (k - 1) // 2)
    raw_q = raw_ref + (bf(raw_ref) - raw_ref).detach()
    groups = [(0, split), (split, n)] if split else [(0, n)]
    z = torch.cat([F.batch_norm(raw_q[a:b], None, None, gr, br, True, 0.0, eps) for a, b in groups], 0)
    F.silu(z).backward(dy)
    # ---- product: forward statistics from the stored raw values, like the conv kernel's tail
    xv = ops.from_nchw(x)
    raw = View.empty(n, h, w, co, DEV)
    ops.conv2d(xv, ops.pack_conv_weight(wt), raw, k, 1, ops.SY_CONV_RAW)
    rawf = raw.nchw_float()
    mean = torch.stack([rawf[a:b].mean((0, 2, 3)) for a, b in groups] + ([] if split else [torch.zeros(co, device=DEV)]))
    var = torch.stack([rawf[a:b].var((0, 2, 3), unbiased=False) for a, b in groups] + ([] if split else [torch.ones(co, device=DEV)]))
    invstd = (var + eps).rsqrt()
    scale = (gamma[None] * invstd).contiguous()
    shift = (beta[None] - mean * scale).contiguous()
    # the forward kernel's own statistics (BatchNorm finalize in the conv tail, saved for the backward pass)
    ss, mi = torch.empty((2, 2, co), device=DEV), torch.full((2, 2, co), float("nan"), device=DEV)
    rm, rv, nbt = torch.zeros(co, device=DEV), torch.ones(co, device=DEV), torch.zeros((), dtype=torch.long, device=DEV)
    raw2 = View.empty(n, h, w, co, DEV)
    ops.conv2d(xv, ops.pack_conv_weight(wt), raw2, k, 1, ops.SY_CONV_RAW, split_n=split,
               partials=torch.empty((ops.conv_stat_rows(), 4 * co), device=DEV), bn=[(gamma, beta, rm, rv, nbt, 0)],
               momentum=0.03, eps=eps, scale_shift=ss, sync=torch.zeros(2, dtype=torch.int32, device=DEV), mean_invstd=mi)
    torch.cuda.synchronize()
    ng = len(groups)
    assert torch.equal(raw2.torch(), raw.torch())
    assert torch.allclose(mi[0, :ng], mean[:ng], rtol=1e-4, atol=1e-5) and torch.allclose(mi[1, :ng], invstd[:ng], rtol=1e-4)
    assert torch.allclose(ss[0, :ng], scale[:ng], rtol=1e-4) and torch.allclose(ss[1, :ng], shift[:ng], rtol=1e-4, atol=1e-5)
    draw = View.empty(n, h, w, co, DEV)
    dgamma, dbeta = torch.full((co,), float("nan"), device=DEV), torch.full((co,), float("nan"), device=DEV)
    ops.bn_act_backward(raw, ops.from_nchw(dy), draw, ss[0], ss[1], mi[0], mi[1], split, 1, dgamma, dbeta)
    dx = View.empty(n, h, w, ci, DEV)
    ops.conv2d(draw, ops.pack_conv_weight_dgrad(wt), dx, k, 1, ops.SY_CONV_RAW)
    dw = torch.empty((co, ci, k, k), device=DEV)
    ops.conv2d_wgrad(xv, draw, k, 1, dw)
    torch.cuda.synchronize()

    def rel(a, b):
        return ((a.float() - b.float()).norm() / (b.float().norm() + 1e-12)).item()

    assert rel(dgamma, gr.grad) < 5e-3 and rel(dbeta, br.grad) < 5e-3, (rel(dgamma, gr.grad), rel(dbeta, br.grad))
    assert rel(dx.nchw_float(), xr.grad) < 1e-2, rel(dx.nchw_float(), xr.grad)
    assert rel(dw, wr.grad) < 1e-2, rel(dw, wr.grad)


@pytest.mark.parametrize("case", [(2, 64, 128, 40, 60), (2, 128, 256, 75, 120), (3, 16, 32, 15, 21)],
                         ids=lambda c: "x".join(map(str, c)))
def test_conv_dgrad_stride2(case):
    """Data gradient of a stride-2 3x3 conv: zero insertion + the stride-1 forward kernel on the flipped filter."""
    n, ci, co, h, w = case
    x = rand_act(n, ci, h, w, 51).requires_grad_(True)
    wt = rand_w(co, ci, 3, 52)
    ho, wo = ops.conv_out_hw(h, w, 3, 2)
    dy = rand_act(n, co, ho, wo, 53)
    F.conv2d(x, wt, None, 2, 1).backward(dy)
    dx = View.empty(n, h, w, ci, DEV)
    ops.conv2d_dgrad_stride2(ops.from_nchw(dy), wt, dx)
    torch.cuda.synchronize()
    check_close(dx.nchw_float(), x.grad, f"dgrad_s2{case}")


@pytest.mark.parametrize("hi,wi,ho,wo", [(19, 30, 38, 60), (38, 60, 75, 120), (4, 5, 8, 10), (8, 10, 15, 20)])
def test_upsample_nearest_backward(hi, wi, ho, wo):
    n, c = 2, 64
    x = rand_act(n, c, hi, wi, 61).requires_grad_(True)
    dy = rand_act(n, c, ho, wo, 62)
    F.interpolate(x, size=(ho, wo), mode="nearest").backward(dy)
    dx = View.empty(n, hi, wi, c, DEV)
    ops.upsample_nearest_backward(ops.from_nchw(dy), dx)
    torch.cuda.synchronize()
    check_close(dx.nchw_float(), x.grad, "upsample backward", ulp=2.0 ** -8)


def test_head_pred_backward():
    b, c, h, w, nc = 2, 64, 19, 30, 8
    a_total, off = h * w + 100, 60
    cls_feat, reg_feat = rand_act(b, c, h, w, 71), rand_act(b, c, h, w, 72)
    g = torch.Generator().manual_seed(73)
    w_reg, w_obj, w_cls = [(torch.randn(o, c, generator=g) * 0.1).to(DEV).requires_grad_(True) for o in (4, 1, nc)]
    b_reg, b_obj, b_cls = [torch.zeros(o, device=DEV, requires_grad=True) for o in (4, 1, nc)]
    grad_raw = torch.zeros(b, a_total, 5 + nc, device=DEV)
    gsub = (torch.randn(b, h * w, 5 + nc, generator=g) * 0.05).to(DEV)
    grad_raw[:, off:off + h * w] = gsub
    cf, rf = cls_feat.clone().requires_grad_(True), reg_feat.clone().requires_grad_(True)
    out = torch.cat([F.conv2d(rf, w_reg[:, :, None, None], b_reg), F.conv2d(rf, w_obj[:, :, None, None], b_obj),
                     F.conv2d(cf, w_cls[:, :, None, None], b_cls)], 1)
    out.flatten(2).permute(0, 2, 1).backward(gsub)
    dcf, drf = View.empty(b, h, w, c, DEV), View.empty(b, h, w, c, DEV)
    dws = [torch.full_like(t, float("nan")).detach() for t in (w_reg, w_obj, w_cls)]
    dbs = [torch.full_like(t, float("nan")).detach() for t in (b_reg, b_obj, b_cls)]
    ops.head_pred_backward(grad_raw, ops.from_nchw(cls_feat), ops.from_nchw(reg_feat), dcf, drf, w_reg.detach(),
                           w_obj.detach(), w_cls.detach(), a_total, off, dws[0], dws[1], dws[2], dbs[0], dbs[1], dbs[2])
    torch.cuda.synchronize()
    check_close(dcf.nchw_float(), cf.grad, "d cls_feat")
    check_close(drf.nchw_float(), rf.grad, "d reg_feat")
    for got, ref, name in zip(dws + dbs, [w_reg.grad, w_obj.grad, w_cls.grad, b_reg.grad, b_obj.grad, b_cls.grad],
                              ["dw_reg", "dw_obj", "dw_cls", "db_reg", "db_obj", "db_cls"]):
        assert (got - ref).abs().max().item() <= 2e-4 * ref.abs().max().item() + 1e-7, name


def test_add_and_spp_backward():
    n, c, h, w = 2, 64, 19, 30
    a, b_ = rand_act(n, c, h, w, 81), rand_act(n, c, h, w, 82)
    av, bv = ops.from_nchw(a), ops.from_nchw(b_)
    ops.add_(av, bv)
    torch.cuda.synchronize()
    assert torch.equal(bv.nchw_float(), bf(a + b_))
    # SPP pools: quantised input so that ties are common (first maximum in row-major order must win, like PyTorch)
    g = torch.Generator().manual_seed(83)
    x = (torch.randint(-6, 7, (n, c, h, w), generator=g).float() * 0.25).to(DEV).requires_grad_(True)
    dys = [rand_act(n, c, h, w, 84 + i) for i in range(3)]
    for k, d in zip((5, 9, 13), dys):
        F.max_pool2d(x, k, 1, k // 2).backward(d)
    dx = View.empty(n, h, w, c, DEV)
    ops.spp_maxpool_backward(ops.from_nchw(x.detach()), *[ops.from_nchw(d) for d in dys], dx)
    torch.cuda.synchronize()
    check_close(dx.nchw_float(), x.grad, "spp backward", ulp=2.0 ** -8)
