"""The CPU emulation of the kernels (tests/emul_ops.py, tests/emul_act.py) against the library it stands in for.

Most of the suite's host-side checks -- which buffer feeds which launch, concat slices, group offsets, the backward walk's
gradient routing, the trainer, the streaming tick -- run with every ``ops`` entry point replaced by its emulation.  Those
checks are only as good as the emulation's contract, so here the library and the emulation run on identical inputs (the
emulation on CPU copies) and must agree on:

  * values: bit for bit where the kernel is exact (weight packs, data movement, max pools, Focus, the optimiser step);
    elsewhere within the error model of the kernel's own parity tests (check_close for 16-bit stored results, sum_tol
    for fp32 reductions, the running-statistics bar of test_gpu_ops, loss_bars / grad_bar for the loss);
  * footprint: every output buffer starts as a NaN sentinel, and both sides write exactly the same elements of it
    (channel and image slices, group offsets, anchor-row offsets, origin, the wider buffers around them);
  * semantics: accumulate onto a non-zero start, split_n in {0, 1, n - 1, n, n + 1}, stat_updates = 2, running statistics
    and num_batches_tracked, one and two BatchNorm groups with an uneven p_split, activation codes 0-3, bf16 and fp16;
  * refusals: an argument set the library refuses before launching, the emulation refuses too.

Partial-sum buffers are private to each side and are compared only through what consumes them.

CPU: every name in emul_ops.NAMES and every entry point emul_act wraps has a case in CASES, and every ``ops`` function a
CPU test replaces by name is in NAMES.  The ablations perturb one emulation each (an exact one, a bar-based one and a
footprint-only one) and assert that the case rejects it."""
import ast
import glob
import os
import sys

import numpy as np
import pytest
import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import emul_act  # noqa: E402
import emul_ops  # noqa: E402
from streamyolo_b200 import ops  # noqa: E402
from streamyolo_b200.ops import View  # noqa: E402

DEV = "cuda"
HERE = os.path.dirname(os.path.abspath(__file__))
BF16, F16 = torch.bfloat16, torch.float16
ACT_WRAPPED = ("conv2d", "bn_act_apply", "bn_act_backward")          # what emul_act.wrap replaces
LIB = {n: getattr(ops, n) for n in emul_ops.NAMES}                   # the library's entry points, before any install
SENT = {BF16: 0x7FC1, F16: 0x7E01, torch.float32: 0x7FC00001}       # NaN bit patterns no kernel writes
INT_OF = {BF16: torch.int16, F16: torch.int16, torch.float32: torch.int32}


# ------------------------------------------------------------------------------------------------ helpers
def _g(seed):
    return torch.Generator().manual_seed(seed)


def randn(*shape, seed, scale=1.0, dtype=torch.float32):
    return (torch.randn(shape, generator=_g(seed)) * scale).to(dtype)


def sentinel(shape, dtype=torch.float32):
    return torch.full(shape, SENT[dtype], dtype=INT_OF[dtype]).view(dtype)


def both(t):
    """(device copy, CPU copy) of a CPU tensor"""
    return t.to(DEV), t.clone()


def views(buf, **kw):
    d, c = both(buf)
    return View(d, **kw), View(c, **kw)


def bits(t):
    t = t.detach().cpu().contiguous()
    return t.view(INT_OF[t.dtype]) if t.dtype in INT_OF else t


def written(t):
    return bits(t) != SENT[t.dtype] if t.dtype in SENT else torch.ones_like(t, dtype=torch.bool)


def same_footprint(lib, emu, what):
    wl, we = written(lib), written(emu)
    assert torch.equal(wl, we), f"{what}: the library writes {int(wl.sum())} elements, the emulation {int(we.sum())}, " \
        f"{int((wl != we).sum())} differ"
    return wl


def same_bits(lib, emu, what):
    same_footprint(lib, emu, what)
    assert torch.equal(bits(lib), bits(emu)), f"{what}: {int((bits(lib) != bits(emu)).sum())} elements differ"


def close16(lib, emu, what, ulp=2.0 ** -7):
    """16-bit stored results: the same footprint, then check_close (one rounding plus accumulation noise) on it"""
    from test_gpu_ops import check_close
    m = same_footprint(lib, emu, what)
    check_close(lib.cpu().float()[m], emu.float()[m], what, ulp)


def sum_close(lib, emu, ref, s2, k, what):
    """fp32 reductions of k terms: each side within sum_tol of the float64 reference"""
    from test_gpu_parity_bwd import check_sum
    check_sum(lib.cpu(), ref, s2, k, f"{what} (library)")
    check_sum(emu, ref, s2, k, f"{what} (emulation)")


def stats_close(lib, emu, what):
    """running statistics, scale / shift, mean / invstd: the bar of the kernel's own test (test_gpu_ops)"""
    lib = lib.cpu()
    assert torch.equal(written(lib), written(emu)), f"{what}: footprint"
    m = written(lib)
    assert torch.allclose(lib[m], emu[m], rtol=1e-4, atol=1e-5), f"{what}: {(lib[m] - emu[m]).abs().max():.3g}"


def both_refuse(lib_call, emu_call, what):
    with pytest.raises((RuntimeError, ValueError)) as el:
        lib_call()
        torch.cuda.synchronize()
    with pytest.raises(type(el.value)):
        emu_call()
    torch.cuda.synchronize()


@pytest.fixture
def emul(monkeypatch):
    """emul_ops + emul_act installed with bf16 storage (EXACT = False); the library stays in LIB"""
    emul_act.install(monkeypatch, exact=False)
    return emul_ops


def act_buf(n, h, w, c, seed, dtype=BF16, scale=1.0, offset=0.0):
    return (randn(n, h, w, c, seed=seed, scale=scale) + offset).to(dtype)


# ------------------------------------------------------------------------------------------------ conv2d
def _fused(fn, act, dtype, impl, seed):
    n, h, w, ci, co, k = 3, 11, 13, 24, 32, 3
    xin = act_buf(n, h, w, 3 * ci, seed, dtype)
    wt = randn(co, ci, k, k, seed=seed + 1, scale=(ci * k * k) ** -0.5)
    scale, shift = randn(co, seed=seed + 2).abs() + 0.5, randn(co, seed=seed + 3) * 0.5
    res = act_buf(n, h, w, co, seed + 4, dtype)
    yb = sentinel((n, h, w, 3 * co), dtype)
    yb[..., co:2 * co] = res                          # the residual lives where the output goes (in place)
    if impl == "dw":
        wt = randn(co, 1, k, k, seed=seed + 1, scale=1 / 3)
        xin = act_buf(n, h, w, 3 * co, seed, dtype)
        ci = co
    (xl, xe), (yl, ye) = views(xin, c0=ci, c=ci), views(yb, c0=co, c=co)
    pack = LIB["pack_dw_weight"] if impl == "dw" else LIB["pack_conv_weight"]
    epack = emul_ops.pack_dw_weight if impl == "dw" else emul_ops.pack_conv_weight
    kw = dict(impl=impl, act=act)
    LIB["conv2d"](xl, pack(wt.to(DEV), dtype=dtype), yl, k, 1, ops.SY_CONV_FUSED, scale=scale.to(DEV), shift=shift.to(DEV),
                  res=yl, **kw)
    fn(xe, epack(wt, dtype=dtype), ye, k, 1, ops.SY_CONV_FUSED, scale=scale, shift=shift, res=ye, **kw)
    torch.cuda.synchronize()
    close16(yl.buf, ye.buf, f"conv2d FUSED {impl} act {act} {dtype}")


def case_conv2d_fused(emul):
    for a in (0, 1, 2, 3):
        _fused(emul.conv2d, a, BF16, "tc", 10 + a)
        _fused(emul.conv2d, a, F16, "tc", 20 + a)
    _fused(emul.conv2d, 1, BF16, "simt", 30)
    _fused(emul.conv2d, 3, BF16, "dw", 31)
    _fused(emul.conv2d, 1, F16, "dw", 32)


def _raw_bn(emul, n, split_n, stat_updates, seed):
    """RAW tensor-core conv with the BatchNorm tail: two parameter segments, running statistics, mean / invstd"""
    h, w, ci, co = 9, 14, 32, 64
    x = act_buf(n, h, w, ci, seed)
    wt = randn(co, ci, 1, 1, seed=seed + 1, scale=ci ** -0.5)
    gamma, beta = randn(co, seed=seed + 2).abs() + 0.5, randn(co, seed=seed + 3) * 0.5
    rm, rv = randn(co, seed=seed + 4) * 0.1, randn(co, seed=seed + 5).abs() + 0.5
    sides = []
    for dev, lib in ((DEV, True), ("cpu", False)):
        t = lambda v: v.clone().to(dev)                                                   # noqa: E731
        g, b, m, v = t(gamma), t(beta), t(rm), t(rv)
        nbt = [torch.full((), 7, dtype=torch.long, device=dev) for _ in range(2)]
        segs = [(g[:24], b[:24], m[:24], v[:24], nbt[0], 0), (g[24:], b[24:], m[24:], v[24:], nbt[1], 24)]
        y = View(sentinel((n, h, w, co), BF16).to(dev))
        rows_n = (LIB if lib else emul_ops.__dict__)["conv_stat_rows"]()
        partials = sentinel((rows_n, 4 * co)).to(dev)
        ss, mi = sentinel((2, 2, co)).to(dev), sentinel((2, 2, co)).to(dev)
        sync = torch.zeros(2, dtype=torch.int32, device=dev)
        fn = LIB["conv2d"] if lib else emul.conv2d
        pk = LIB["pack_conv_weight"](wt.to(DEV)) if lib else emul.pack_conv_weight(wt)
        rows = fn(View(x.to(dev)), pk, y, 1, 1, ops.SY_CONV_RAW, impl="tc", partials=partials, split_n=split_n,
                  bn=[s for s in segs], momentum=0.03, eps=1e-3, scale_shift=ss, sync=sync, mean_invstd=mi,
                  stat_updates=stat_updates)
        torch.cuda.synchronize()
        # the sense the host and the kernel tests rely on: the launch writes at most the rows it was given
        assert 1 <= rows <= rows_n, (lib, rows, rows_n)
        sides.append(dict(y=y.buf, ss=ss, mi=mi, rm=m, rv=v, nbt=[int(t_) for t_ in nbt],
                          sums=torch.nan_to_num(partials[:rows].view(rows, co, 2, 2).cpu().double(), nan=0.0).sum(0)))
    (L, E), what = sides, f"conv2d RAW+bn n={n} split_n={split_n} stat_updates={stat_updates}"
    close16(L["y"], E["y"], what + ": y")
    groups = 2 if 0 < split_n < n else 1
    for k in ("ss", "mi"):
        stats_close(L[k][:, :groups], E[k][:, :groups], f"{what}: {k}")
    stats_close(L["rm"], E["rm"], what + ": running_mean")
    stats_close(L["rv"], E["rv"], what + ": running_var")
    ups = groups * (2 if stat_updates == 2 else 1)
    assert L["nbt"] == E["nbt"] == [7 + ups] * 2, (what, L["nbt"], E["nbt"])
    # the partial rows compose into the per-group sums of the stored output (sum, sum of squares): fp32 reductions
    if stat_updates == 2:
        return          # the rows of a repeated single group are private to the kernel; its statistics are checked above
    st = E["y"].double().permute(0, 3, 1, 2)
    sp = split_n if 0 < split_n < n else n
    for gi, (a, b) in enumerate([(0, sp), (sp, n)][:groups]):
        k = (b - a) * h * w
        ref1, ref2 = st[a:b].sum((0, 2, 3)), st[a:b].pow(2).sum((0, 2, 3))
        for j, (ref, s2) in enumerate(((ref1, st[a:b].pow(2).sum((0, 2, 3))), (ref2, st[a:b].pow(4).sum((0, 2, 3))))):
            sum_close(L["sums"][:, gi, j], E["sums"][:, gi, j], ref, s2, k, f"{what}: partial sums group {gi}")


def case_conv2d_raw_bn(emul):
    n = 4
    for split_n in (0, 1, n - 1, n, n + 1):
        _raw_bn(emul, n, split_n, 1, 40 + split_n)
    _raw_bn(emul, n, 0, 2, 50)
    _raw_bn(emul, n, n, 2, 51)


def case_conv2d_refusals(emul):
    x = act_buf(2, 8, 8, 32, 60)
    wt = randn(32, 32, 1, 1, seed=61)
    pk, epk = LIB["pack_conv_weight"](wt.to(DEV)), emul.pack_conv_weight(wt)
    (xl, xe), (yl, ye) = views(x), views(torch.zeros(2, 8, 8, 32, dtype=BF16))
    (hl, he) = views(x.to(F16))[0], views(x.to(F16))[1]
    both_refuse(lambda: LIB["conv2d"](hl, pk, yl, 1, 1, ops.SY_CONV_FUSED),
                lambda: ops.conv2d(he, epk, ye, 1, 1, ops.SY_CONV_FUSED), "mixed storage")
    both_refuse(lambda: LIB["conv2d"](xl, pk, yl, 1, 1, ops.SY_CONV_FUSED, act=4),
                lambda: ops.conv2d(xe, epk, ye, 1, 1, ops.SY_CONV_FUSED, act=4), "act 4")
    pl, pe = torch.empty((LIB["conv_stat_rows"]() - 1, 128), device=DEV), torch.empty((emul.conv_stat_rows() - 1, 128))
    both_refuse(lambda: LIB["conv2d"](xl, pk, yl, 1, 1, ops.SY_CONV_RAW, partials=pl),
                lambda: ops.conv2d(xe, epk, ye, 1, 1, ops.SY_CONV_RAW, partials=pe), "one statistic row short")


def case_conv_stat_rows(emul):
    """the host sizes a RAW launch's partials with conv_stat_rows() and only hands them back: each side's launch accepts
    its own count and writes no more rows than that (case_conv2d_raw_bn) and refuses one row fewer (case_conv2d_refusals);
    and a buffer sized by the emulation's count is one the library accepts (rows >= what the library needs)"""
    x = act_buf(2, 8, 8, 32, 65)
    pk = LIB["pack_conv_weight"](randn(64, 32, 1, 1, seed=66).to(DEV))
    y = View.empty(2, 8, 8, 64, DEV)
    partials = torch.empty((emul.conv_stat_rows(), 4 * 64), device=DEV)
    rows = LIB["conv2d"](View(x.to(DEV)), pk, y, 1, 1, ops.SY_CONV_RAW, partials=partials, split_n=1)
    torch.cuda.synchronize()
    assert 1 <= rows <= emul.conv_stat_rows()
    case_conv2d_refusals(emul)


# ------------------------------------------------------------------------------------------------ BatchNorm glue
def _apply(fn, split_n, act, goff, seed):
    n, h, w, c = 4, 5, 7, 32
    x = act_buf(n, h, w, c, seed)
    ss = torch.stack([randn(2, c, seed=seed + 1).abs() + 0.5, randn(2, c, seed=seed + 2)])
    big = sentinel((n, h, w, 3 * c), BF16)
    res = act_buf(n, h, w, 3 * c, seed + 3)
    (xl, xe), (yl, ye), (rl, re) = views(x), views(big, c0=c, c=c), views(res, c0=0, c=c)
    yo, ro = (c, 2 * c) if goff else (0, 0)        # group 1 writes the next channel block, reads the one after
    ssl = ss.to(DEV)
    LIB["bn_act_apply"](xl, ssl[0], ssl[1], split_n, act, rl, yl, yo, ro)
    fn(xe, ss[0], ss[1], split_n, act, re, ye, yo, ro)
    torch.cuda.synchronize()
    close16(yl.buf, ye.buf, f"bn_act_apply split_n={split_n} act={act} goff={goff}")


def case_bn_act_apply(emul):
    for split_n in (0, 1, 3, 4, 5):
        _apply(emul.bn_act_apply, split_n, 1, True, 70 + split_n)
    for a in (0, 1, 2, 3):
        _apply(emul.bn_act_apply, 2, a, False, 80 + a)
    x = act_buf(2, 4, 4, 16, 85)
    (xl, xe), (yl, ye) = views(x), views(x.clone())
    s = torch.ones((2, 16))
    both_refuse(lambda: LIB["bn_act_apply"](xl, s.to(DEV), s.to(DEV), 1, 1, None, yl, 4, 0),
                lambda: emul.bn_act_apply(xe, s, s, 1, 1, None, ye, 4, 0), "group offset not a multiple of 8")
    both_refuse(lambda: LIB["bn_act_apply"](xl, s.to(DEV), s.to(DEV), 1, 7, None, yl),
                lambda: emul.bn_act_apply(xe, s, s, 1, 7, None, ye), "act 7")


def case_stats_num_partials(emul):
    """the host sizes channel_stats' partials with it and splits them image-major at (P // n) * split: P is a multiple
    of n on both sides (compositions in case_bn_finalize)"""
    for n, hw in ((1, 1), (4, 35), (3, 600), (2, 4500)):
        for p in (LIB["stats_num_partials"](n, hw), emul.stats_num_partials(n, hw)):
            assert p >= n and p % n == 0, (n, hw, p)


def _stats_chain(emul, groups, seed):
    """channel_stats -> bn_finalize -> bn_act_apply, each side on its own partials"""
    n, h, w, c = 4, 9, 70, 32                      # 630 pixels per image: more than one library chunk
    x = act_buf(n, h, w, 2 * c, seed, scale=2.0, offset=0.7)
    gamma, beta = randn(c, seed=seed + 1).abs() + 0.5, randn(c, seed=seed + 2)
    sp = n // 2 if groups == 2 else n
    out = []
    for lib in (True, False):
        dev = DEV if lib else "cpu"
        f = (lambda nm: LIB[nm]) if lib else (lambda nm: getattr(ops, nm))
        xv = View(x.to(dev), c0=c, c=c)
        P = f("stats_num_partials")(n, h * w)
        partials = torch.empty((P, 2, c), device=dev)
        f("channel_stats")(xv, partials)
        rm, rv = torch.full((c,), 0.1, device=dev), torch.full((c,), 0.9, device=dev)
        nbt = torch.zeros((), dtype=torch.long, device=dev)
        ss = sentinel((2, 2, c)).to(dev)
        f("bn_finalize")(partials, (P // n) * sp if groups == 2 else 0, groups, sp * h * w, gamma.to(dev), beta.to(dev),
                         rm, rv, nbt, 0.03, 1e-3, ss[0], ss[1])
        y = View(sentinel((n, h, w, c), BF16).to(dev))
        f("bn_act_apply")(xv, ss[0], ss[1], sp, 1, None, y)
        torch.cuda.synchronize()
        out.append((ss, rm, rv, int(nbt), y.buf))
    (L, E), what = out, f"channel_stats -> bn_finalize -> bn_act_apply, {groups} groups"
    stats_close(L[0][:, :groups], E[0][:, :groups], what + ": scale / shift")
    stats_close(L[1], E[1], what + ": running_mean")
    stats_close(L[2], E[2], what + ": running_var")
    assert L[3] == E[3] == groups
    close16(L[4], E[4], what + ": y")


def case_channel_stats(emul):
    _stats_chain(emul, 1, 90)
    _stats_chain(emul, 2, 91)
    x = act_buf(2, 30, 40, 16, 92)
    (xl, xe) = views(x)
    both_refuse(lambda: LIB["channel_stats"](xl, torch.empty((LIB["stats_num_partials"](2, 1200) - 1, 2, 16), device=DEV)),
                lambda: ops.channel_stats(xe, torch.empty((emul.stats_num_partials(2, 1200) - 1, 2, 16))),
                "one partial row short")


def case_bn_finalize(emul):
    """on one partials tensor ([P][2][C] sums, the entry point's public input): one group, two groups with an uneven
    p_split (``count`` is the pixel count of each group), the refusals"""
    _stats_chain(emul, 2, 95)
    P, c, count = 7, 48, 300
    g = _g(96)
    vals = torch.randn((P, count // 3, c), generator=g) * 1.5 + 0.3
    partials = torch.stack([vals.sum(1), vals.pow(2).sum(1)], 1)                            # [P][2][C]
    gamma, beta = randn(c, seed=97).abs() + 0.5, randn(c, seed=98)
    for groups, p_split in ((1, 0), (2, 2), (2, 5)):
        out = []
        for lib in (True, False):
            dev = DEV if lib else "cpu"
            rm, rv = torch.full((c,), 0.1, device=dev), torch.full((c,), 0.9, device=dev)
            nbt = torch.full((), 3, dtype=torch.long, device=dev)
            ss = sentinel((2, 2, c)).to(dev)
            (LIB["bn_finalize"] if lib else ops.bn_finalize)(partials.to(dev), p_split, groups, count, gamma.to(dev),
                                                             beta.to(dev), rm, rv, nbt, 0.03, 1e-3, ss[0], ss[1])
            torch.cuda.synchronize()
            out.append((ss, rm, rv, int(nbt)))
        (L, E), what = out, f"bn_finalize groups={groups} p_split={p_split}"
        stats_close(L[0][:, :groups], E[0][:, :groups], what + ": scale / shift")
        assert torch.equal(written(L[0].cpu()), written(E[0])), what + ": footprint"
        stats_close(L[1], E[1], what + ": running_mean")
        stats_close(L[2], E[2], what + ": running_var")
        assert L[3] == E[3] == 3 + groups
    z = torch.zeros(c)
    for groups, p_split, cnt in ((3, 0, count), (2, 0, count), (2, P, count), (1, 0, 0)):
        both_refuse(lambda: LIB["bn_finalize"](partials.to(DEV), p_split, groups, cnt, z.to(DEV) + 1, z.to(DEV), None, None,
                                               None, 0.03, 1e-3, torch.empty(2, c, device=DEV), torch.empty(2, c, device=DEV)),
                    lambda: ops.bn_finalize(partials, p_split, groups, cnt, z + 1, z, None, None, None, 0.03, 1e-3,
                                            torch.empty(2, c), torch.empty(2, c)), f"groups={groups} p_split={p_split}")


def _bn_bwd(fn, split_n, act, accumulate, seed):
    from test_gpu_parity_bwd import bn_act_backward_ref
    n, h, w, c = 4, 6, 9, 48
    raw = act_buf(n, h, w, c, seed, offset=0.2)
    dy = act_buf(n, h, w, c, seed + 1, scale=1e-2)
    rawf = raw.float().permute(0, 3, 1, 2)
    sp = split_n if 0 < split_n < n else n
    grp = [(0, sp), (sp, n)] if sp < n else [(0, n)]
    mi, ss = torch.zeros(2, 2, c), torch.zeros(2, 2, c)
    gamma, beta = randn(c, seed=seed + 2).abs() + 0.5, randn(c, seed=seed + 3)
    for gi, (a, b) in enumerate(grp):
        mean, var = rawf[a:b].mean((0, 2, 3)), rawf[a:b].var((0, 2, 3), unbiased=False)
        mi[0, gi], mi[1, gi] = mean, (var + 1e-3).rsqrt()
        ss[0, gi] = gamma * mi[1, gi]
        ss[1, gi] = beta - mean * ss[0, gi]
    start = randn(2, c, seed=seed + 4) if accumulate else torch.zeros(2, c)
    draw_b = sentinel((n, h, w, 2 * c), BF16)
    (rl, re), (dl, de), (wl, we) = views(raw), views(dy), views(draw_b, c0=c, c=c)
    dgl, dbl = start[0].clone().to(DEV), start[1].clone().to(DEV)
    dge, dbe = start[0].clone(), start[1].clone()
    sd, md = ss.to(DEV), mi.to(DEV)
    LIB["bn_act_backward"](rl, dl, wl, sd[0], sd[1], md[0], md[1], split_n, act, dgl, dbl, accumulate=accumulate)
    fn(re, de, we, ss[0], ss[1], mi[0], mi[1], split_n, act, dge, dbe, accumulate=accumulate)
    torch.cuda.synchronize()
    what = f"bn_act_backward split_n={split_n} act={act} accumulate={accumulate}"
    close16(wl.buf, we.buf, what + ": draw")
    _, dg, db, s2g, s2b, _, _ = bn_act_backward_ref(rawf.double(), dy.double().permute(0, 3, 1, 2), ss, mi,
                                                    [(a, b, gi) for gi, (a, b) in enumerate(grp)], act) \
        if act in (0, 1) else _bn_bwd_ref_any(rawf.double(), dy.double().permute(0, 3, 1, 2), ss, mi, grp, act)
    k = n * h * w
    sum_close(dgl, dge, dg + start[0].double(), s2g + start[0].double() ** 2, k + 1, what + ": dgamma")
    sum_close(dbl, dbe, db + start[1].double(), s2b + start[1].double() ** 2, k + 1, what + ": dbeta")


def _bn_bwd_ref_any(raw, gy, ss, mi, grp, act):
    """float64 dgamma / dbeta and the sums of their squared terms for any activation code"""
    c = raw.shape[1]
    dg, db, s2g, s2b = (torch.zeros(c, dtype=torch.float64) for _ in range(4))
    for gi, (a, b) in enumerate(grp):
        sc, sh, mu, iv = (t.double()[None, :, None, None] for t in (ss[0, gi], ss[1, gi], mi[0, gi], mi[1, gi]))
        dz = gy[a:b] * emul_ops._dact(raw[a:b] * sc + sh, act)
        t = dz * (raw[a:b] - mu) * iv
        dg += t.sum((0, 2, 3))
        db += dz.sum((0, 2, 3))
        s2g += t.pow(2).sum((0, 2, 3))
        s2b += dz.pow(2).sum((0, 2, 3))
    return None, dg, db, s2g, s2b, None, None


def case_bn_act_backward(emul):
    for split_n in (0, 1, 3, 4, 5):
        _bn_bwd(emul.bn_act_backward, split_n, 1, split_n == 1, 100 + split_n)
    for a in (0, 1, 2, 3):
        _bn_bwd(emul.bn_act_backward, 2, a, True, 110 + a)


# ------------------------------------------------------------------------------------------------ data movement
def case_focus_pack(emul):
    for dtype in (BF16, F16):
        b, h, w = 2, 12, 18
        x = torch.rand((b, 6, h, w), generator=_g(120)) * 255
        yl, ye = views(sentinel((2 * b, h // 2, w // 2, 64), dtype))
        LIB["focus_pack"](x.to(DEV), 2, yl)
        ops.focus_pack(x, 2, ye)
        torch.cuda.synchronize()
        same_bits(yl.buf, ye.buf, f"focus_pack {dtype}")


def case_upsample_nearest(emul):
    for dtype, (hi, wi, ho, wo) in ((BF16, (5, 7, 10, 14)), (F16, (4, 5, 8, 10)), (BF16, (19, 30, 38, 60))):
        x = act_buf(2, hi, wi, 16, 130, dtype)
        (xl, xe), (yl, ye) = views(x), views(sentinel((2, ho, wo, 48), dtype), c0=16, c=16)
        LIB["upsample_nearest"](xl, yl)
        ops.upsample_nearest(xe, ye)
        torch.cuda.synchronize()
        same_bits(yl.buf, ye.buf, f"upsample_nearest {dtype} {hi}x{wi}->{ho}x{wo}")
    (xl, xe), (yl, ye) = views(act_buf(1, 4, 4, 8, 131)), views(torch.zeros(1, 8, 8, 8, dtype=F16))
    both_refuse(lambda: LIB["upsample_nearest"](xl, yl), lambda: ops.upsample_nearest(xe, ye), "mixed dtypes")


def case_spp_maxpool(emul):
    for dtype in (BF16, F16):
        x = act_buf(2, 9, 11, 16, 140, dtype)
        (xl, xe), (bl, be) = views(x), views(sentinel((2, 9, 11, 64), dtype))
        LIB["spp_maxpool"](xl, bl.ch(16, 16), bl.ch(32, 16), bl.ch(48, 16))
        ops.spp_maxpool(xe, be.ch(16, 16), be.ch(32, 16), be.ch(48, 16))
        torch.cuda.synchronize()
        same_bits(bl.buf, be.buf, f"spp_maxpool {dtype}")


def case_copy(emul):
    for dtype in (BF16, F16):
        x = act_buf(5, 6, 7, 40, 150, dtype)
        (xl, xe), (yl, ye) = views(x, c0=8, c=16, n0=1, n=3), views(sentinel((4, 6, 7, 24), dtype), c0=8, c=16, n0=1, n=3)
        LIB["copy"](xl, yl)
        ops.copy(xe, ye)
        torch.cuda.synchronize()
        same_bits(yl.buf, ye.buf, f"copy {dtype}")


def case_add_(emul):
    x, y = act_buf(3, 5, 6, 32, 160), act_buf(3, 5, 6, 48, 161)
    (xl, xe), (yl, ye) = views(x, c0=8, c=16), views(y, c0=16, c=16)
    LIB["add_"](xl, yl)
    ops.add_(xe, ye)
    torch.cuda.synchronize()
    same_bits(yl.buf, ye.buf, "add_")


def case_dilate2(emul):
    for (h, w, H, W) in ((5, 6, 10, 12), (5, 6, 9, 11)):
        g = act_buf(2, h, w, 16, 170)
        (gl, ge), (dl, de) = views(g), views(sentinel((2, H, W, 16), BF16))
        LIB["dilate2"](gl, dl)
        ops.dilate2(ge, de)
        torch.cuda.synchronize()
        same_bits(dl.buf, de.buf, f"dilate2 {h}x{w}->{H}x{W}")
    (gl, ge), (dl, de) = views(act_buf(2, 5, 6, 16, 171)), views(torch.zeros(2, 12, 12, 16, dtype=BF16))
    both_refuse(lambda: LIB["dilate2"](gl, dl), lambda: ops.dilate2(ge, de), "dilate2 size")


def case_upsample_nearest_backward(emul):
    for (hi, wi, ho, wo) in ((5, 7, 10, 14), (19, 30, 38, 60)):
        dy = act_buf(2, ho, wo, 16, 180, scale=1e-2)
        (dl, de), (xl, xe) = views(dy), views(sentinel((2, hi, wi, 32), BF16), c0=16, c=16)
        LIB["upsample_nearest_backward"](dl, xl)
        ops.upsample_nearest_backward(de, xe)
        torch.cuda.synchronize()
        same_bits(xl.buf, xe.buf, f"upsample_nearest_backward {ho}x{wo}->{hi}x{wi}")


def case_spp_maxpool_backward(emul):
    """a window's gradient goes to its first maximum on both sides; the sums of the routed gradients within the kernel's
    own bar (check_close at 2^-8, test_spp_maxpool_backward_production)"""
    x = act_buf(2, 9, 11, 16, 190)
    d = [act_buf(2, 9, 11, 16, 191 + i, scale=1e-2) for i in range(3)]
    (xl, xe) = views(x)
    dv = [views(t) for t in d]
    (ol, oe) = views(sentinel((2, 9, 11, 48), BF16), c0=16, c=16)
    LIB["spp_maxpool_backward"](xl, *[v[0] for v in dv], ol)
    ops.spp_maxpool_backward(xe, *[v[1] for v in dv], oe)
    torch.cuda.synchronize()
    close16(ol.buf, oe.buf, "spp_maxpool_backward", ulp=2.0 ** -8)


# ------------------------------------------------------------------------------------------------ weight gradient
def case_conv2d_wgrad(emul):
    for (n, h, w, ci, co, k, s) in ((2, 10, 12, 32, 64, 3, 1), (2, 10, 12, 16, 32, 3, 2), (3, 7, 9, 64, 32, 1, 1)):
        x = act_buf(n, h, w, ci, 200)
        ho, wo = ops.conv_out_hw(h, w, k, s)
        dy = act_buf(n, ho, wo, co, 201, scale=1e-2)
        start = randn(co, ci, k, k, seed=202)
        dwl, dwe = start.clone().to(DEV), start.clone()
        LIB["conv2d_wgrad"](View(x.to(DEV)), View(dy.to(DEV)), k, s, dwl, accumulate=True)
        ops.conv2d_wgrad(View(x.clone()), View(dy.clone()), k, s, dwe, accumulate=True)
        torch.cuda.synchronize()
        x64, d64 = x.double().permute(0, 3, 1, 2), dy.double().permute(0, 3, 1, 2)
        ref = torch.nn.grad.conv2d_weight(x64, dwe.shape, d64, stride=s, padding=(k - 1) // 2) + start.double()
        s2 = torch.nn.grad.conv2d_weight(x64 ** 2, dwe.shape, d64 ** 2, stride=s, padding=(k - 1) // 2) + start.double() ** 2
        sum_close(dwl, dwe, ref, s2, n * ho * wo + 1, f"conv2d_wgrad {(n, h, w, ci, co, k, s)}")


# ------------------------------------------------------------------------------------------------ head
def _head_weights(c, nc, seed):
    return [randn(*sh, seed=seed + i, scale=c ** -0.5) for i, sh in enumerate(((4, c), (4,), (1, c), (1,), (nc, c), (nc,)))]


def case_head_pred_decode(emul):
    """one level in the middle of the anchor rows: rows of the other levels and their origin stay untouched on both
    sides; sigmoid / decode on and off; bf16 and fp16 features.  Bar of the forward parity test (FwdChecker)"""
    from test_gpu_parity_bwd import U32, sum_tol
    b, h, w, c, nc, off, a_total, stride = 2, 6, 9, 32, 8, 20, 100, 16
    ws = _head_weights(c, nc, 210)
    for dtype, sigmoid, decode in ((BF16, False, False), (BF16, True, True), (F16, True, True)):
        cf, rf = act_buf(b, h, w, c, 211, dtype), act_buf(b, h, w, c, 212, dtype)
        (cl, ce), (rl, re) = views(cf), views(rf)
        (ol, oe), (gl, ge) = both(sentinel((b, a_total, 5 + nc))), both(sentinel((b, a_total, 4)))
        LIB["head_pred_decode"](cl, rl, *[t.to(DEV) for t in ws], stride, off, a_total, ol, gl, sigmoid, decode)
        ops.head_pred_decode(ce, re, *ws, stride, off, a_total, oe, ge, sigmoid, decode)
        torch.cuda.synchronize()
        what = f"head_pred_decode {dtype} sigmoid={sigmoid} decode={decode}"
        m = same_footprint(ol, oe, what + ": out")
        assert bool(m[:, off:off + h * w].all()) and not bool(m[:, :off].any()) and not bool(m[:, off + h * w:].any())
        same_footprint(gl, ge, what + ": origin")
        f64 = lambda t: t.double().reshape(b, h * w, c)                                  # noqa: E731
        lin, s2 = [], []
        for f, wt, bias in ((f64(rf), ws[0], ws[1]), (f64(rf), ws[2], ws[3]), (f64(cf), ws[4], ws[5])):
            lin.append(f @ wt.double().T + bias.double())
            s2.append(f.square() @ wt.double().square().T + bias.double().square())
        lin, s2 = torch.cat(lin, -1), torch.cat(s2, -1)
        tol = sum_tol(lin, s2, c + 1)
        ref, rt = lin.clone(), tol.clone()
        if decode:
            yv, xv = torch.meshgrid(torch.arange(h), torch.arange(w), indexing="ij")
            ref[..., 0] = (lin[..., 0] + xv.reshape(-1)) * stride
            ref[..., 1] = (lin[..., 1] + yv.reshape(-1)) * stride
            rt[..., 0:2] = tol[..., 0:2] * stride
            ref[..., 2:4] = torch.exp(lin[..., 2:4]) * stride
            rt[..., 2:4] = ref[..., 2:4] * tol[..., 2:4]
        if sigmoid:
            sg = torch.sigmoid(lin[..., 4:])
            ref[..., 4:] = sg
            rt[..., 4:] = sg * (1 - sg) * tol[..., 4:]
        bar = rt + 16 * U32 * ref.abs() + 2.0 ** -126
        rows = slice(off, off + h * w)
        for side, o, g in (("library", ol.cpu(), gl.cpu()), ("emulation", oe, ge)):
            assert bool(((o[:, rows].double() - ref).abs() <= bar).all()), f"{what}: {side} outputs"
            assert bool(((g[:, rows].double() - lin[..., :4]).abs() <= tol[..., :4] + 16 * U32 * lin[..., :4].abs()).all()), \
                f"{what}: {side} origin"
    cf = act_buf(b, h, w, c, 213)
    (cl, ce), (rl, re) = views(cf), views(cf.clone())
    ol, oe = both(torch.zeros(b, a_total, 5 + nc))
    both_refuse(lambda: LIB["head_pred_decode"](cl, rl, *[t.to(DEV) for t in ws], stride, a_total - h * w + 1, a_total, ol,
                                                None, 0, 0),
                lambda: ops.head_pred_decode(ce, re, *ws, stride, a_total - h * w + 1, a_total, oe, None, 0, 0),
                "one anchor row past a_total")


def _head_bwd(emul, name, nc, seed):
    from test_gpu_parity_bwd import check_sum
    b, h, w, c, off, a_total = 2, 5, 7, 32, 15, 80
    g = randn(b, a_total, 5 + nc, seed=seed, scale=1e-2)
    cf, rf = act_buf(b, h, w, c, seed + 1), act_buf(b, h, w, c, seed + 2)
    w_reg, w_obj, w_cls = (randn(*sh, seed=seed + 3 + i, scale=c ** -0.5) for i, sh in enumerate(((4, c), (1, c), (nc, c))))
    starts = [randn(*sh, seed=seed + 10 + i) for i, sh in enumerate(((4, c), (1, c), (nc, c), (4,), (1,), (nc,)))]
    (cl, ce), (rl, re) = views(cf), views(rf)
    (dcl, dce), (drl, dre) = (views(sentinel((b, h, w, 2 * c), BF16), c0=c, c=c) for _ in range(2))
    gl = [s.clone().to(DEV) for s in starts]
    ge = [s.clone() for s in starts]
    LIB[name](g.to(DEV), cl, rl, dcl, drl, w_reg.to(DEV), w_obj.to(DEV), w_cls.to(DEV), a_total, off, *gl, accumulate=True)
    getattr(ops, name)(g, ce, re, dce, dre, w_reg, w_obj, w_cls, a_total, off, *ge, accumulate=True)
    torch.cuda.synchronize()
    what = f"{name} {nc} classes"
    close16(dcl.buf, dce.buf, what + ": d_cls_feat")
    close16(drl.buf, dre.buf, what + ": d_reg_feat")
    gg = g[:, off:off + h * w].double()
    f64 = lambda t: t.double().reshape(b, h * w, c)                                      # noqa: E731
    refs = [(gg[..., 0:4], f64(rf)), (gg[..., 4:5], f64(rf)), (gg[..., 5:], f64(cf))]
    k = b * h * w
    for i, (gs, f) in enumerate(refs):
        ref = torch.einsum("bpo,bpc->oc", gs, f) + starts[i].double()
        s2 = torch.einsum("bpo,bpc->oc", gs ** 2, f ** 2) + starts[i].double() ** 2
        check_sum(gl[i].cpu(), ref, s2, k + 1, f"{what}: dW {i} (library)")
        check_sum(ge[i], ref, s2, k + 1, f"{what}: dW {i} (emulation)")
        refb = gs.sum((0, 1)) + starts[3 + i].double()
        s2b = (gs ** 2).sum((0, 1)) + starts[3 + i].double() ** 2
        check_sum(gl[3 + i].cpu(), refb, s2b, k + 1, f"{what}: db {i} (library)")
        check_sum(ge[3 + i], refb, s2b, k + 1, f"{what}: db {i} (emulation)")


def _head_bwd_refusal(emul, name, nc, c=32):
    b, h, w, a_total = 1, 3, 3, 9
    g = torch.zeros(b, a_total, 5 + nc)
    f = act_buf(b, h, w, c, 220)
    (cl, ce) = views(f)
    wr, wo, wc = torch.zeros(4, c), torch.zeros(1, c), torch.zeros(nc, c)
    outs = [torch.zeros(4, c), torch.zeros(1, c), torch.zeros(nc, c), torch.zeros(4), torch.zeros(1), torch.zeros(nc)]
    (dl, de) = views(torch.zeros(b, h, w, c, dtype=BF16))
    both_refuse(lambda: LIB[name](g.to(DEV), cl, cl, dl, dl, wr.to(DEV), wo.to(DEV), wc.to(DEV), a_total, 0,
                                  *[t.to(DEV) for t in outs]),
                lambda: getattr(ops, name)(g, ce, ce, de, de, wr, wo, wc, a_total, 0, *outs), f"{name} {nc} classes")


def case_head_pred_backward(emul):
    _head_bwd(emul, "head_pred_backward", 8, 230)
    _head_bwd(emul, "head_pred_backward", 27, 240)
    _head_bwd_refusal(emul, "head_pred_backward", 28)


def case_head_pred_backward_wide(emul):
    _head_bwd(emul, "head_pred_backward_wide", 80, 250)
    _head_bwd_refusal(emul, "head_pred_backward_wide", 252)


# ------------------------------------------------------------------------------------------------ loss
def _loss_inputs(b, n_gt):
    from test_gpu_parity_l import _labels, _synthetic_head_outputs
    fut, cur = _labels(b, n_gt, 17 + n_gt)
    outputs, origin = _synthetic_head_outputs(b, fut, 19 + n_gt)
    return outputs, origin, fut, cur


def case_tal_loss_workspace_bytes(emul):
    """the host allocates that many bytes and hands the buffer to tal_loss / tal_loss_backward only: each side's
    tal_loss accepts its own size (case_tal_loss) and refuses one byte less"""
    from test_gpu_parity_l import A_TOTAL, HW, STRIDES
    outputs, origin, fut, cur = _loss_inputs(2, 3)
    for lib in (True, False):
        dev = DEV if lib else "cpu"
        nb = (LIB if lib else emul_ops.__dict__)["tal_loss_workspace_bytes"](2, A_TOTAL, fut.shape[1], 8)
        assert nb > 0
        ws = torch.empty(nb - 1, dtype=torch.uint8, device=dev)
        fn = LIB["tal_loss"] if lib else ops.tal_loss
        with pytest.raises(RuntimeError):
            fn(outputs.to(dev), origin.to(dev), fut.to(dev), cur.to(dev), HW, STRIDES, 1.0, 0.5, 1.6, True, ws,
               torch.empty(6, device=dev))
            torch.cuda.synchronize()


def case_tal_loss(emul):
    """the six losses and the three gradients of each side against float64 autograd through the oracle, with the bars
    of test_simota_reference (loss_bars, grad_bar); the refusal of levels that do not tile a_total"""
    from oracle.streamyolo_oracle import OracleCfg, StreamYoloOracle
    from test_gpu_parity_l import A_TOTAL, HW, STRIDES
    from test_simota_reference import LOSSES, grad_bar, loss_bars
    b, gamma, gscale = 2, 1.5, 2.0
    outputs, origin, fut, cur = _loss_inputs(b, 12)
    o = StreamYoloOracle(OracleCfg(gamma=gamma, ignore_thr=0.5, ignore_value=1.6), {})
    grid64 = tuple(t.double() for t in o.grids(HW, STRIDES))
    out64, org64 = outputs.double().requires_grad_(True), origin.double().requires_grad_(True)
    ref = o.losses(out64, org64, grid64, (fut, cur), return_aux=True, dtype=torch.float64)
    (ref["total_loss"] * gscale).backward()
    want = np.array([float(ref[n]) for n in LOSSES])
    gs = grid64[2]
    graw = out64.grad.clone()
    graw[..., 0:2] = out64.grad[..., 0:2] * gs[None, :, None] + org64.grad[..., 0:2]
    graw[..., 2:4] = out64.grad[..., 2:4] * out64.detach()[..., 2:4] + org64.grad[..., 2:4]
    for lib in (True, False):
        dev, side = (DEV, "library") if lib else ("cpu", "emulation")
        f = (lambda nm: LIB[nm]) if lib else (lambda nm: getattr(ops, nm))
        ws = torch.empty(f("tal_loss_workspace_bytes")(b, A_TOTAL, fut.shape[1], 8), dtype=torch.uint8, device=dev)
        loss = torch.empty(6, device=dev)
        od, ogd, fd, cd = outputs.to(dev), origin.to(dev), fut.to(dev), cur.to(dev)
        f("tal_loss")(od, ogd, fd, cd, HW, STRIDES, gamma, 0.5, 1.6, True, ws, loss)
        g = [sentinel(t.shape).to(dev) for t in (outputs, origin, outputs)]
        f("tal_loss_backward")(od, ogd, fd, HW, STRIDES, gamma, True, ws, gscale, grad_outputs=g[0], grad_origin=g[1],
                               grad_raw=g[2])
        torch.cuda.synchronize()
        got = loss.cpu().double().numpy()
        err, bar = np.abs(got - want), loss_bars(want, int(ref["aux"]["num_fg_raw"]))
        assert (err <= bar).all(), f"tal_loss {side}: losses {got.tolist()} vs {want.tolist()}"
        for t, w_, what in zip(g, (out64.grad, org64.grad, graw), ("grad_outputs", "grad_origin", "grad_raw")):
            t = t.cpu().double().reshape(-1, w_.shape[-1])
            w_ = w_.reshape(-1, w_.shape[-1])
            assert bool(((t - w_).abs() <= grad_bar(w_)).all()), f"tal_loss_backward {side}: {what}"
    bad = [(75, 120), (38, 60), (19, 31)]
    ws_l = torch.empty(LIB["tal_loss_workspace_bytes"](b, A_TOTAL, fut.shape[1], 8), dtype=torch.uint8, device=DEV)
    ws_e = torch.empty(emul.tal_loss_workspace_bytes(b, A_TOTAL, fut.shape[1], 8), dtype=torch.uint8)
    both_refuse(lambda: LIB["tal_loss"](outputs.to(DEV), origin.to(DEV), fut.to(DEV), cur.to(DEV), bad, STRIDES, 1.0, 0.5,
                                        1.6, True, ws_l, torch.empty(6, device=DEV)),
                lambda: ops.tal_loss(outputs, origin, fut, cur, bad, STRIDES, 1.0, 0.5, 1.6, True, ws_e, torch.empty(6)),
                "levels that do not tile a_total")


def case_tal_loss_backward(emul):
    case_tal_loss(emul)


# ------------------------------------------------------------------------------------------------ weights and optimiser
def case_pack_conv_weight(emul):
    for dtype in (BF16, F16):
        a, b_ = randn(16, 24, 3, 3, seed=260), randn(8, 24, 3, 3, seed=261)
        same_bits(LIB["pack_conv_weight"](a.to(DEV), b_.to(DEV), dtype=dtype), ops.pack_conv_weight(a, b_, dtype=dtype),
                  f"pack_conv_weight {dtype}")


def case_pack_conv_weight_dgrad(emul):
    a, b_ = randn(16, 24, 3, 3, seed=262), randn(8, 24, 3, 3, seed=263)
    same_bits(LIB["pack_conv_weight_dgrad"](a.to(DEV), b_.to(DEV)), ops.pack_conv_weight_dgrad(a, b_), "pack_conv_weight_dgrad")


def case_pack_stem_weight(emul):
    for dtype in (BF16, F16):
        w = randn(16, 12, 3, 3, seed=264)
        same_bits(LIB["pack_stem_weight"](w.to(DEV), dtype=dtype), ops.pack_stem_weight(w, dtype=dtype), f"pack_stem {dtype}")


def case_pack_dw_weight(emul):
    for dtype in (BF16, F16):
        w = randn(32, 1, 3, 3, seed=265)
        same_bits(LIB["pack_dw_weight"](w.to(DEV), dtype=dtype), ops.pack_dw_weight(w, dtype=dtype), f"pack_dw {dtype}")


def case_PackBatch(emul):
    ws = [randn(16, 24, 3, 3, seed=266), randn(32, 16, 1, 1, seed=267), randn(16, 12, 3, 3, seed=268)]
    outs = []
    for lib in (True, False):
        dev = DEV if lib else "cpu"
        pb = (LIB["PackBatch"] if lib else ops.PackBatch)(dev)
        w = [t.to(dev) for t in ws]
        o = [sentinel((16, 9, 24), BF16).to(dev), sentinel((32, 1, 16), BF16).to(dev), sentinel((16, 3, 64), BF16).to(dev),
             sentinel((24, 9, 48), BF16).to(dev)]
        pb.add(w[0], o[0], 0)
        pb.add(w[1], o[1], 0)
        pb.add(w[2], o[2], 2)
        pb.add(w[0], o[3], 1, out_pitch=48, co_offset=16)
        pb.run()
        torch.cuda.synchronize()
        outs.append(o)
    for i, (a, b_) in enumerate(zip(*outs)):
        same_bits(a, b_, f"PackBatch item {i}")


def case_sgd_nesterov_ema_step(emul):
    n_total, n_param = 1000, 900
    p, g, e = (randn(n_total, seed=270 + i) for i in range(3))
    m = randn(n_param, seed=273)                 # momentum of the n_param trained values
    for kw in (dict(), dict(nesterov=False, inv_scale=0.5), dict(hyper=torch.tensor([0.02, 0.8, 1e-3, 0.25, 0.99, 0.01])),
               dict(found_inf=torch.ones(1)), dict(found_inf=torch.ones(1), found_inf_ema=True),
               dict(found_inf=torch.zeros(1), found_inf_ema=True)):
        out = []
        for lib in (True, False):
            dev = DEV if lib else "cpu"
            t = [x.clone().to(dev) for x in (p, g, m, e)]
            k = {a: (v.to(dev) if torch.is_tensor(v) else v) for a, v in kw.items()}
            (LIB["sgd_nesterov_ema_step"] if lib else ops.sgd_nesterov_ema_step)(t[0], t[1], t[2], t[3], n_param, 300, 0.01,
                                                                                 ema_decay=0.9998, **k)
            torch.cuda.synchronize()
            out.append(t)
        for a, b_, nm in zip(*out, ("param", "grad", "momentum", "ema")):
            assert torch.equal(a.cpu(), b_), f"sgd_nesterov_ema_step {sorted(kw)}: {nm}"


def case_nonfinite_flag(emul):
    for bad in (None, float("inf"), float("nan")):
        x = randn(1024, seed=280)
        if bad is not None:
            x[517] = bad
        out = []
        for lib in (True, False):
            dev = DEV if lib else "cpu"
            f, c = torch.full((1,), 5.0, device=dev), torch.full((1,), 3, dtype=torch.int32, device=dev)
            (LIB["nonfinite_flag"] if lib else ops.nonfinite_flag)(x.to(dev), f, c)
            torch.cuda.synchronize()
            out.append((float(f), int(c)))
        assert out[0] == out[1] == ((1.0, 4) if bad is not None else (0.0, 3)), (bad, out)


def case_resize_bilinear(emul):
    """the bar of the kernel's own test (test_gpu_train): within 1e-5 of F.interpolate"""
    x = torch.rand((2, 3, 37, 53), generator=_g(290)) * 255
    for size in ((48, 80), (20, 30)):
        ol, oe = both(sentinel((2, 3) + size))
        LIB["resize_bilinear"](x.to(DEV), size, out=ol)
        r = ops.resize_bilinear(x, size, out=oe)
        assert r is oe
        assert torch.allclose(ol.cpu(), oe, rtol=1e-5, atol=1e-5), size
        assert torch.allclose(LIB["resize_bilinear"](x.to(DEV), size).cpu(), ops.resize_bilinear(x, size), rtol=1e-5, atol=1e-5)


def case_scale_labels_(emul):
    lab = randn(3, 7, 5, seed=291).abs() * 100
    a, b_ = both(lab)
    LIB["scale_labels_"](a, 0.75, 1.25)
    assert ops.scale_labels_(b_, 0.75, 1.25) is b_
    torch.cuda.synchronize()
    same_bits(a, b_, "scale_labels_")


# ------------------------------------------------------------------------------------------------ streaming tick
def case_letterbox_sized(emul):
    g = _g(300)
    src = torch.randint(0, 256, (2, 60, 80, 3), generator=g, dtype=torch.uint8)
    sizes = torch.tensor([[60, 80, 48, 64], [50, 70, 48, 64]], dtype=torch.int32)
    ol, oe = both(sentinel((2, 3, 48, 64)))
    LIB["letterbox_sized"](src.to(DEV), sizes.to(DEV), ol)
    ops.letterbox_sized(src, sizes, oe)
    torch.cuda.synchronize()
    same_bits(ol, oe, "letterbox_sized")


def case_stream_gate(emul):
    flags = torch.tensor([1, 0, 1, 0], dtype=torch.int32)
    for status in (None, torch.tensor([0, 0, 3, 1], dtype=torch.int32)):
        out = []
        for lib in (True, False):
            dev = DEV if lib else "cpu"
            s, k = torch.full((4,), 9, dtype=torch.int32, device=dev), torch.full((4,), 9, dtype=torch.int32, device=dev)
            (LIB["stream_gate"] if lib else ops.stream_gate)(status.to(dev) if status is not None else None, flags.to(dev), s, k)
            torch.cuda.synchronize()
            out.append((s.cpu(), k.cpu()))
        assert torch.equal(out[0][0], out[1][0]) and torch.equal(out[0][1], out[1][1]), status


def case_stream_rescale(emul):
    det = randn(3, 5, 7, seed=310).abs() * 100
    count = torch.tensor([2, 5, 3], dtype=torch.int32)
    ratio = torch.tensor([0.5, 0.3125, 1.7])
    for status in (None, torch.tensor([0, 2, 0], dtype=torch.int32)):
        (dl, de), (cl, ce) = both(det), both(count)
        LIB["stream_rescale"](dl, cl, status.to(DEV) if status is not None else None, ratio.to(DEV))
        ops.stream_rescale(de, ce, status, ratio)
        torch.cuda.synchronize()
        same_bits(dl, de, "stream_rescale det")
        assert torch.equal(cl.cpu(), ce)


def case_select_images(emul):
    flags = torch.tensor([1, 0, 1], dtype=torch.int32)
    for dtype in (BF16, F16):
        src = [act_buf(3, 4, 5, 16, 320 + i, dtype) for i in range(2)]
        dst = [sentinel((3, 4, 5, 32), dtype) for _ in range(2)]
        sv = [views(s) for s in src]
        dv = [views(d, c0=8, c=16) for d in dst]
        LIB["select_images"]([s[0] for s in sv], [d[0] for d in dv], flags.to(DEV))
        ops.select_images([s[1] for s in sv], [d[1] for d in dv], flags)
        torch.cuda.synchronize()
        for (dl, de) in dv:
            same_bits(dl.buf, de.buf, f"select_images {dtype}")


def case_postprocess_nms(emul):
    """rows below count: the oracle's (pinned to torchvision's batched_nms); rows past it are private to each side"""
    g = _g(330)
    b, a, nc = 2, 200, 4
    xy = torch.rand((b, a, 2), generator=g) * 300
    wh = torch.rand((b, a, 2), generator=g) * 60 + 4
    pred = torch.cat([xy, wh, torch.rand((b, a, 1 + nc), generator=g)], -1)
    dl, cl = LIB["postprocess_nms"](pred.to(DEV), nc, 0.3, 0.65, max_det=50)
    de, ce = ops.postprocess_nms(pred, nc, 0.3, 0.65, max_det=50)
    torch.cuda.synchronize()
    assert torch.equal(cl.cpu(), ce), (cl.tolist(), ce.tolist())
    for i in range(b):
        assert torch.equal(dl[i, :int(ce[i])].cpu(), de[i, :int(ce[i])]), i


# ------------------------------------------------------------------------------------------------ emul_act's wrappers
def case_act_conv2d(emul):
    """emul_act's conv2d for the kinked codes (the FUSED epilogue)"""
    for a in emul_act.KINKS:
        _fused(ops.conv2d, a, BF16, "tc", 340 + a)
        _fused(ops.conv2d, a, BF16, "dw", 345 + a)


def case_act_bn_act_apply(emul):
    for a in emul_act.KINKS:
        for split_n in (0, 2, 4):
            _apply(ops.bn_act_apply, split_n, a, True, 350 + a + split_n)


def case_act_bn_act_backward(emul):
    for a in emul_act.KINKS:
        _bn_bwd(ops.bn_act_backward, 2, a, True, 360 + a)
        _bn_bwd(ops.bn_act_backward, 0, a, False, 370 + a)


def case_conv2d(emul):
    case_conv2d_fused(emul)
    case_conv2d_raw_bn(emul)
    case_conv2d_refusals(emul)


CASES = {n: globals()["case_" + n] for n in emul_ops.NAMES}
CASES.update({"emul_act." + n: globals()["case_act_" + n] for n in ACT_WRAPPED})


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(CASES))
def test_emulation_conforms(name, emul):
    CASES[name](emul)


# ------------------------------------------------------------------------------------------------ ablations
def _perturbed(monkeypatch, name, fn):
    monkeypatch.setattr(emul_ops, name, fn)
    monkeypatch.setattr(ops, name, fn)


@pytest.mark.gpu
def test_rejects_copy_one_element_off(emul, monkeypatch):
    """an exact entry: a copy that rounds one value differently"""
    base = emul_ops.copy

    def copy(x, y):
        base(x, y)
        y.torch()[0, 0, 0, 0] = y.torch()[0, 0, 0, 0] * 1.01 + 0.01
    _perturbed(monkeypatch, "copy", copy)
    with pytest.raises(AssertionError):
        case_copy(emul)


@pytest.mark.gpu
def test_rejects_bn_finalize_group1_count_scaled_by_rows(emul, monkeypatch):
    """a bar-based entry: group 1's count scaled by its share of the partial rows (count * (P - p_split) / p_split, what
    the emulation once did) instead of the same count per group"""
    base = emul_ops.bn_finalize

    def bn_finalize(partials, p_split, groups, count, gamma, beta, rmean, rvar, nbt, momentum, eps, scale, shift):
        base(partials, p_split, groups, count, gamma, beta, rmean, rvar, nbt, momentum, eps, scale, shift)
        if groups == 2:
            r = partials[p_split:]
            cnt = count * (partials.shape[0] - p_split) / p_split
            mean = r[:, 0].sum(0) / cnt
            var = (r[:, 1].sum(0) / cnt - mean * mean).clamp_min(0)
            scale[1] = gamma.float() * (var + eps).rsqrt()
            shift[1] = beta.float() - mean * scale[1]
    _perturbed(monkeypatch, "bn_finalize", bn_finalize)
    with pytest.raises(AssertionError):
        case_bn_finalize(emul)


@pytest.mark.gpu
def test_rejects_head_pred_decode_one_row_past_its_anchors(emul, monkeypatch):
    """a footprint-only difference: one more anchor row written, with the right values everywhere else"""
    base = emul_ops.head_pred_decode

    def head_pred_decode(cls_feat, reg_feat, *a):
        base(cls_feat, reg_feat, *a)
        off, out = a[7], a[9]
        out[:, off + cls_feat.h * cls_feat.w] = 0.0
    _perturbed(monkeypatch, "head_pred_decode", head_pred_decode)
    with pytest.raises(AssertionError):
        case_head_pred_decode(emul)


@pytest.mark.gpu
def test_rejects_conv_stat_rows_below_the_library(emul, monkeypatch):
    """an emulated row count below this GPU's SM count (114, a PCIe card's, on an H100 SXM): CPU tests would size
    partials the kernel here refuses"""
    monkeypatch.setattr(emul_ops, "conv_stat_rows", lambda: LIB["conv_stat_rows"]() - 1)
    monkeypatch.setattr(ops, "conv_stat_rows", emul_ops.conv_stat_rows)
    with pytest.raises((AssertionError, RuntimeError)):
        case_conv_stat_rows(emul)


# ------------------------------------------------------------------------------------------------ CPU: coverage
def _replaced_by_cpu_tests():
    """names of ``ops`` functions the test modules replace with monkeypatch.setattr(ops, "<name>", ...)"""
    names = {}
    for path in glob.glob(os.path.join(HERE, "test_*.py")):
        tree = ast.parse(open(path).read())
        for node in ast.walk(tree):
            if (isinstance(node, ast.Call) and isinstance(node.func, ast.Attribute) and node.func.attr == "setattr"
                    and len(node.args) >= 2 and isinstance(node.args[0], ast.Name) and node.args[0].id == "ops"
                    and isinstance(node.args[1], ast.Constant) and isinstance(node.args[1].value, str)):
                names.setdefault(node.args[1].value, set()).add(os.path.basename(path))
    return names


def test_every_emulated_entry_point_has_a_conformance_case():
    want = set(emul_ops.NAMES) | {"emul_act." + n for n in ACT_WRAPPED}
    assert set(CASES) == want, (sorted(want - set(CASES)), sorted(set(CASES) - want))
    for n in emul_ops.NAMES:
        assert hasattr(ops, n), f"emul_ops.NAMES lists {n}, which ops does not have"


def test_emul_act_wraps_exactly_the_listed_entry_points(monkeypatch):
    """what emul_act.wrap replaces on ops, found by running it"""
    before = {n: getattr(ops, n) for n in dir(ops)}
    emul_act.wrap(monkeypatch)
    changed = {n for n in before if getattr(ops, n) is not before[n]}
    assert changed == set(ACT_WRAPPED), changed


def test_every_entry_point_cpu_tests_replace_is_emulated():
    replaced = _replaced_by_cpu_tests()
    missing = {n: sorted(f) for n, f in replaced.items() if n not in emul_ops.NAMES}
    assert not missing, f"ops functions replaced by tests but not in emul_ops.NAMES: {missing}"


def test_coverage_check_notices_a_missing_case(monkeypatch):
    """the two coverage tests fail on a name added to NAMES without a case, and on a case removed from the table"""
    monkeypatch.setattr(emul_ops, "NAMES", emul_ops.NAMES + ["select_images_twice"])
    with pytest.raises(AssertionError):
        test_every_emulated_entry_point_has_a_conformance_case()
    monkeypatch.undo()
    monkeypatch.delitem(CASES, "dilate2")
    with pytest.raises(AssertionError):
        test_every_emulated_entry_point_has_a_conformance_case()
