"""GPU parity of every FORWARD launch at the benchmarked shapes, in place, against float64 references (the forward
counterpart of tests/test_gpu_parity_bwd.py):

  * ``FwdChecker`` wraps ops.conv2d, ops.bn_act_apply, ops.head_pred_decode and ops.focus_pack for the length of a forward
    and checks every launch as it happens, on the very tensors it reads (snapshotted in float64 before the launch: CSP
    bottlenecks write their output in place over their residual).  Each reference is built from the MODULE, not from what
    the launch was handed: the conv weights are the module's ``conv.weight`` rounded to bf16, the eval scale / shift the
    float64 fold of its BatchNorm.  An output region that does not overlap the launch's inputs is filled with NaN first,
    so that a pixel the launch never writes shows up; a launch must leave the rest of its output buffer bit for bit alone.
  * run on the forwards bench.py times, built as it builds them (600x960, BN eps 1e-3 / momentum 0.03, use_l1): the train
    plain forward of l / m / s at 8 pairs, the recording forward of a training step (l at 4 pairs, and the still model,
    whose single backbone pass updates the running statistics twice), eval off_pipe of l / m at 8 pairs and on_pipe at
    batch 1, each with its launch count derived from the module tree;
  * the FUSED epilogue (folded scale / shift, SiLU, residual in place or from a slice of another buffer, output into a
    channel slice of a wider buffer) at every distinct eval / on_pipe launch shape, under every tiling;
  * CUDA-graph replays (what bench.py times) bit-identical to eager calls.

Bars follow the error model of each result:
  * bf16-stored results: one bf16 rounding plus accumulation noise (check_close), and a relative L2 error of at most
    2^-8 (one rounding alone gives ~2^-9 / sqrt(3) ~ 1.1e-3);
  * BatchNorm statistics: the bars of tests/test_gpu_parity_l.py (scale 1e-4 relative, shift 1e-4 of |mean * scale|),
    i.e. 1e-4 of (|mean| + std) on the mean and 2e-4 relative on the variance, carried through the running-statistics
    updates (momentum times the per-update bar, plus fp32 rounding of the update);
  * head outputs (fp32 1x1 convs): the fp32-reduction bar of sum_tol, propagated through decode (exp) and sigmoid, plus
    16 fp32 ulps of the evaluation (and the smallest normal fp32, for sigmoids that underflow).
Every conv launch also recomputes its reference with one unit of work left out -- input channels 0-63 at the centre tap,
a 1x1 conv -- and asserts that the bar rejects it.
"""
from collections import Counter

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

from streamyolo_b200 import ops, synth  # noqa: E402
from streamyolo_b200.model import backward, engine  # noqa: E402
from streamyolo_b200.model.network_blocks import BaseConv, CSPLayer  # noqa: E402
from streamyolo_b200.ops import View  # noqa: E402
from test_gpu_model import ORDER, build_product  # noqa: E402
from test_gpu_ops import check_close  # noqa: E402
from test_gpu_parity_bwd import DGRAD_TILINGS, MODELS, U32, nchw64, outside_bf16, post_silu, sum_tol  # noqa: E402
from test_gpu_still import build_still, still_batch  # noqa: E402

DEV = "cuda"
F64 = torch.float64
NAN = float("nan")
FLT_MAX = torch.finfo(torch.float32).max
ULP = 2.0 ** -7           # check_close's default bar
REL_L2 = 2.0 ** -8        # relative L2 bar of a bf16-stored result


# ------------------------------------------------------------------------------------------------ helpers
def conv_launches(model, jian_twice):
    """conv launches of one forward, from the module tree: every BaseConv once, except the CSP conv2s (they ride with their
    conv1) and the head's first reg-tower convs (they ride with their cls twin); the three DFP jian convs launch twice
    where the two frames are not batched (eval, on_pipe, the recording forward)"""
    mods = list(model.modules())
    base = sum(isinstance(m, BaseConv) for m in mods)
    csp = sum(isinstance(m, CSPLayer) for m in mods)
    return base - csp - len(model.head.reg_convs) + (3 if jian_twice else 0)


def _region(buf, v, img0, nimg, goff=0):
    """NHWC view, in ``buf`` (v.buf or a copy of it), of images [img0, img0 + nimg) of ``v`` with the base address moved by
    ``goff`` elements: where a launch with group offsets reads or writes (the batched DFP fusion, tests/emul_ops.py)"""
    _, H, W, Ct = buf.shape
    return buf.as_strided((nimg, H, W, v.c), (H * W * Ct, W * Ct, Ct, 1),
                          buf.storage_offset() + (v.n0 + img0) * H * W * Ct + v.c0 + v.off + goff)


def _n64(t):
    return t.permute(0, 3, 1, 2).to(F64)


def _groups(n, split_n):
    sp = split_n if 0 < split_n < n else n
    return [(0, sp), (sp, n)] if sp < n else [(0, n)]


def _same_bits(a, b):
    return torch.equal(a.view(torch.int16), b.view(torch.int16))


def _sync(t):
    if t.is_cuda:
        torch.cuda.synchronize()


def stem_weight_3x1(w):
    """[O, 12, 3, 3] -> [O, 64, 3, 1]: the 3x3 stem as the 3x1 conv over the W-gathered Focus tensor (ops.focus_pack: the
    left / centre / right column taps at channels 0, 16, 32)"""
    w3 = w.new_zeros((w.shape[0], 64, 3, 1))
    for t, c0 in enumerate((0, 16, 32)):
        w3[:, c0:c0 + 12, :, 0] = w[:, :, :, t]
    return w3


def focus_ref(x, frames):
    """float64 NCHW of what ops.focus_pack writes for the float frames ``x`` [B, 3 * frames, H, W]"""
    xs = torch.cat([x[:, 3 * f:3 * f + 3] for f in range(frames)], 0).to(torch.bfloat16).to(F64)
    foc = torch.cat([xs[..., ::2, ::2], xs[..., 1::2, ::2], xs[..., ::2, 1::2], xs[..., 1::2, 1::2]], 1)
    out = foc.new_zeros((foc.shape[0], 64, foc.shape[2], foc.shape[3]))
    out[:, 16:28] = foc
    out[:, 0:12, :, 1:] = foc[..., :-1]
    out[:, 32:44, :, :-1] = foc[..., 1:]
    return out


def conv_refs(x64, w64, s, sc=None, sh=None, act=1, r64=None):
    """float64 conv (FUSED: silu(conv * scale + shift) + res) and the same with input channels 0-63 at the centre tap left
    out (one unit of the kernel's work)"""
    kh, kw = w64.shape[2], w64.shape[3]
    ref = F.conv2d(x64, w64, None, s, ((kh - 1) // 2, (kw - 1) // 2))
    part = F.conv2d(x64[:, :64], w64[:, :64, kh // 2, kw // 2, None, None], None, s)
    omit = ref - part
    if sc is None:
        return ref, omit

    def epi(t):
        z = t * sc + sh
        z = F.silu(z) if act else z
        return z + r64 if r64 is not None else z
    return epi(ref), epi(omit)


def fused_key(x, y, k, s, res, kind):
    """distinct FUSED launch shape: (n, cin, cout, h, w, kh, kw, stride, operand kind, residual kind)"""
    kh, kw = (k, k) if isinstance(k, int) else k
    rk = "none" if res is None else ("in_place" if (res.buf is y.buf and res.c0 == y.c0 and res.n0 == y.n0) else "slice")
    return (x.n, x.c, y.c, x.h, x.w, kh, kw, s, kind, rk)


def bf16_ratio(got, ref):
    """(worst err / tol under check_close's bar, relative L2 error)"""
    got, ref = got.float(), ref.float()
    err = (got - ref).abs()
    rms = ref.pow(2).mean().sqrt().item() + 1e-12
    return float((err / (ULP * ref.abs() + ULP * rms)).max()), float((got - ref).norm() / (ref.norm() + 1e-12))


# ------------------------------------------------------------------------------------------------ the checker
class FwdChecker:
    """Context manager: every ops.conv2d / bn_act_apply / head_pred_decode / focus_pack launch of ``model`` inside it is
    checked in place against float64 references built from the module tree (see the module docstring).  Run one forward
    first: the map from packed operands to modules is read from the ``_pk`` / ``_pk2`` caches it leaves.
    ``nondegenerate``: FUSED outputs must also be finite and mostly away from zero (calibrated eval statistics).
    After the block: ``n`` counts the launches, ``worst`` holds the worst err / tol ratio per result kind (and the worst
    relative L2 error of the bf16 results), ``fused_shapes`` the distinct FUSED launch shapes."""

    WRAPPED = ("conv2d", "bn_act_apply", "head_pred_decode", "focus_pack")

    def __init__(self, model, nondegenerate=False):
        self.model, self.nondegenerate = model, nondegenerate
        self.n, self.worst = Counter(), {}
        self.fused_shapes = set()
        self.ss = {}                  # data_ptr -> [groups][C] scale / shift rows published by the conv launches
        self.last_mods = None
        self.head_next = 0

    def __enter__(self):
        self.table = self._operands()
        self.orig = {n: getattr(ops, n) for n in self.WRAPPED}
        for n in self.WRAPPED:
            setattr(ops, n, getattr(self, "_" + n))
        return self

    def __exit__(self, *exc):
        for n, f in self.orig.items():
            setattr(ops, n, f)
        return False

    def _operands(self):
        m = self.model
        stem = m.backbone.backbone.stem.conv
        table = {}
        for mod in m.modules():
            if isinstance(mod, BaseConv) and hasattr(mod, "_pk"):
                table[mod._pk.data_ptr()] = ("stem" if mod is stem else "conv", (mod,))
        pairs = [(c.conv1, c.conv2) for c in m.modules() if isinstance(c, CSPLayer)]
        pairs += [(c[0], r[0]) for c, r in zip(m.head.cls_convs, m.head.reg_convs)]
        for a, b in pairs:
            if hasattr(a, "_pk2"):
                table[a._pk2.data_ptr()] = ("pair", (a, b))
        assert table, "no packed operands: run one forward before checking"
        return table

    def _note(self, kind, ratio):
        self.worst[kind] = max(self.worst.get(kind, 0.0), ratio)

    def _close(self, got, want, tol, what, kind):
        err = (got.to(F64) - want).abs()
        ratio = float((err / tol).max())
        self._note(kind, ratio)
        assert not bool(torch.isnan(got).any()) and bool((err <= tol).all()), f"{what}: worst err / tol {ratio:.3g}"

    def _bf16(self, got, ref, what):
        rel = check_close(got, ref, what)
        ratio, rel = bf16_ratio(got, ref)
        self._note("bf16", ratio)
        self._note("rel_l2", rel)
        assert rel <= REL_L2, f"{what}: relative L2 error {rel:.3g} above {REL_L2:.3g}"

    @staticmethod
    def _act(mods):
        return 1 if mods[0].act_name == "silu" else 0

    # -------------------------------------------------------------------- conv
    def _conv2d(self, x, wpk, y, k, s, mode, **a):
        assert wpk.data_ptr() in self.table, "conv launch with an operand that is no module's packed weight"
        kind, mods = self.table[wpk.data_ptr()]
        name = getattr(mods[0], "_sy_name", kind)
        fused = mode == ops.SY_CONV_FUSED
        res = a.get("res")
        x64 = nchw64(x)
        r64 = nchw64(res) if res is not None else None
        bn = None if fused else a.get("bn")
        runs = [(rm.clone(), rv.clone(), int(nbt)) for _, _, rm, rv, nbt, _ in bn] if bn else None
        before = y.buf.clone()
        if not (y.buf is x.buf or (res is not None and y.buf is res.buf)):
            y.torch().fill_(NAN)
        rv_ = self.orig["conv2d"](x, wpk, y, k, s, mode, **a)
        _sync(y.buf)
        self.n["conv"] += 1
        self.last_mods = mods
        w64 = torch.cat([m.conv.weight.detach() for m in mods], 0).to(torch.bfloat16).to(F64)
        if kind == "stem":
            w64 = stem_weight_3x1(w64)
        assert tuple(w64.shape[2:]) == ((k, k) if isinstance(k, int) else tuple(k)), f"{name}: kernel size"
        got = nchw64(y)
        if fused:
            self.fused_shapes.add(fused_key(x, y, k, s, res, kind))
            sc, sh = self._fold(mods)
            ref, omit = conv_refs(x64, w64, s, sc, sh, self._act(mods), r64)
            what = f"{name}: FUSED conv"
        else:
            ref, omit = conv_refs(x64, w64, s)
            what = f"{name}: raw conv"
        del x64, r64
        self._bf16(got, ref, what)
        assert outside_bf16(got, omit) > 0, f"{what}: the bar accepts input channels 0-63 at the centre tap left out"
        del ref, omit
        if fused and self.nondegenerate:
            assert float((got.abs() > 1e-2).double().mean()) >= 0.25, f"{what}: degenerate output"
        if bn:
            self._stats(got, mods, a, runs, name)
        sl = (slice(y.n0, y.n0 + y.n), slice(None), slice(None), slice(y.c0, y.c0 + y.c))
        before[sl] = y.buf[sl]
        assert _same_bits(before, y.buf), f"{what}: writes outside its output view"
        return rv_

    @staticmethod
    def _fold(mods):
        sc, sh = [], []
        for m in mods:
            bn = m.bn
            s_ = bn.weight.detach().to(F64) / torch.sqrt(bn.running_var.to(F64) + bn.eps)
            sc.append(s_)
            sh.append(bn.bias.detach().to(F64) - bn.running_mean.to(F64) * s_)
        return torch.cat(sc)[None, :, None, None], torch.cat(sh)[None, :, None, None]

    def _stats(self, raw, mods, a, runs, name):
        """scale / shift (and mean / invstd) per statistics group from the stored raw values, the running statistics, the
        batch counters, the grid-barrier counters"""
        bn = a["bn"]
        assert len(bn) == len(mods), f"{name}: {len(bn)} BatchNorm segments for {len(mods)} modules"
        c0 = 0
        for seg, m in zip(bn, mods):
            b_ = m.bn
            assert (seg[0] is b_.weight and seg[1] is b_.bias and seg[2] is b_.running_mean and seg[3] is b_.running_var
                    and seg[4] is b_.num_batches_tracked and seg[5] == c0), f"{name}: BatchNorm segment of another module"
            c0 += m.conv.out_channels
        bn0 = mods[0].bn
        eps, mom = bn0.eps, bn0.momentum
        upd = a.get("stat_updates", 1)
        gamma = torch.cat([m.bn.weight.detach() for m in mods]).to(F64)
        beta = torch.cat([m.bn.bias.detach() for m in mods]).to(F64)
        ss, mi = a["scale_shift"], a.get("mean_invstd")
        stats = []
        for gi, (p, q) in enumerate(_groups(raw.shape[0], a.get("split_n", 0))):
            part = raw[p:q]
            mean, var = part.mean((0, 2, 3)), part.var((0, 2, 3), unbiased=False)
            cnt = part.numel() // part.shape[1]
            sc = gamma / torch.sqrt(var + eps)
            sh = beta - mean * sc
            self._close(ss[0, gi], sc, 1e-4 * sc.abs() + 1e-6, f"{name}: scale, group {gi}", "stats")
            self._close(ss[1, gi], sh, 1e-4 * sh.abs() + 1e-5 + 1e-4 * float((mean * sc).abs().max()),
                        f"{name}: shift, group {gi}", "stats")
            if mi is not None:
                self.n["mean_invstd"] += gi == 0
                iv = 1.0 / torch.sqrt(var + eps)
                self._close(mi[0, gi], mean, 1e-4 * (mean.abs() + var.sqrt()) + 1e-6, f"{name}: mean, group {gi}", "stats")
                self._close(mi[1, gi], iv, 1e-4 * iv, f"{name}: invstd, group {gi}", "stats")
            stats.append((mean, var, cnt))
        if upd != 1:
            self.n[f"stat_updates_{upd}"] += 1
        # running statistics: the groups in order, each applied stat_updates times, unbiased variance
        c0 = 0
        for (_, _, rm, rv, nbt, _), (rm0, rv0, nbt0), m in zip(bn, runs, mods):
            sl = slice(c0, c0 + m.conv.out_channels)
            c0 = sl.stop
            want_m, want_v = rm0.to(F64), rv0.to(F64)
            tol_m, tol_v = torch.zeros_like(want_m), torch.zeros_like(want_v)
            for mean, var, cnt in stats:
                for _ in range(upd):
                    want_m = (1 - mom) * want_m + mom * mean[sl]
                    want_v = (1 - mom) * want_v + mom * var[sl] * (cnt / (cnt - 1))
                    tol_m = (1 - mom) * tol_m + mom * 1e-4 * (mean[sl].abs() + var[sl].sqrt())
                    tol_v = (1 - mom) * tol_v + mom * 2e-4 * var[sl] * (cnt / (cnt - 1))
            self._close(rm, want_m, tol_m + 8 * U32 * (want_m.abs() + rm0.abs()) + 1e-12, f"{name}: running_mean", "running")
            self._close(rv, want_v, tol_v + 8 * U32 * (want_v.abs() + rv0.abs()) + 1e-12, f"{name}: running_var", "running")
            assert int(nbt) == nbt0 + len(stats) * upd, f"{name}: num_batches_tracked {int(nbt)}, was {nbt0}"
        if a.get("sync") is not None:
            assert a["sync"].tolist() == [0, 0], f"{name}: grid-barrier counters not back at zero"
        for t in (ss[0], ss[1]):
            self.ss[t.data_ptr()] = t

    # -------------------------------------------------------------------- BatchNorm + SiLU (+ residual) of train mode
    def _bn_act_apply(self, x, scale_ptr, shift_ptr, split_n, act, res, y, y_goff1=0, res_goff1=0):
        sc = scale_ptr if torch.is_tensor(scale_ptr) else self.ss.get(scale_ptr)
        sh = shift_ptr if torch.is_tensor(shift_ptr) else self.ss.get(shift_ptr)
        assert sc is not None and sh is not None, "bn_act_apply: scale / shift not published by a preceding conv launch"
        sc, sh = (t if t.dim() == 2 else t[None] for t in (sc, sh))
        mods = self.last_mods
        name = getattr(mods[0], "_sy_name", "?")
        groups = [(p, q, yo, ro) for (p, q), yo, ro in zip(_groups(x.n, split_n), (0, y_goff1), (0, res_goff1))]
        x64 = nchw64(x)
        r64 = [_n64(_region(res.buf, res, p, q - p, ro)) if res is not None else None for p, q, _, ro in groups]
        before = y.buf.clone()
        if not (y.buf is x.buf or (res is not None and y.buf is res.buf)):
            for p, q, yo, _ in groups:
                _region(y.buf, y, p, q - p, yo).fill_(NAN)
        self.orig["bn_act_apply"](x, scale_ptr, shift_ptr, split_n, act, res, y, y_goff1, res_goff1)
        _sync(y.buf)
        self.n["apply"] += 1
        for gi, (p, q, yo, _) in enumerate(groups):
            z = x64[p:q] * sc[gi].to(F64)[None, :, None, None] + sh[gi].to(F64)[None, :, None, None]
            z = F.silu(z) if self._act(mods) else z
            if r64[gi] is not None:
                z = z + r64[gi]
            self._bf16(_n64(_region(y.buf, y, p, q - p, yo)), z, f"{name}: BatchNorm apply, group {gi}")
            _region(before, y, p, q - p, yo).copy_(_region(y.buf, y, p, q - p, yo))
        assert _same_bits(before, y.buf), f"{name}: BatchNorm apply writes outside its destination"

    # -------------------------------------------------------------------- head prediction convs + decode
    def _head_pred_decode(self, cls_feat, reg_feat, w_reg, b_reg, w_obj, b_obj, w_cls, b_cls, stride, anchor_offset,
                          a_total, out, origin, sigmoid, decode):
        head = self.model.head
        k = self.n["head"] % len(head.strides)
        if k == 0:                    # the three levels must tile [0, A): every anchor row starts as NaN
            self.head_next = 0
            out.fill_(NAN)
            if origin is not None:
                origin.fill_(NAN)
        assert (anchor_offset, stride, a_total) == (self.head_next, head.strides[k], out.shape[1]), \
            f"head level {k}: offset {anchor_offset}, stride {stride}, a_total {a_total}"
        b, h, w, c = cls_feat.n, cls_feat.h, cls_feat.w, cls_feat.c
        cf = cls_feat.torch().to(F64).reshape(b, h * w, c)
        rf = reg_feat.torch().to(F64).reshape(b, h * w, c)
        self.orig["head_pred_decode"](cls_feat, reg_feat, w_reg, b_reg, w_obj, b_obj, w_cls, b_cls, stride, anchor_offset,
                                      a_total, out, origin, sigmoid, decode)
        _sync(out)
        self.n["head"] += 1
        lin, s2 = [], []
        for f, p in ((rf, head.reg_preds[k]), (rf, head.obj_preds[k]), (cf, head.cls_preds[k])):
            wt = p.weight.detach().to(F64).reshape(p.weight.shape[0], -1)
            bias = p.bias.detach().to(F64)
            lin.append(f @ wt.T + bias)
            s2.append(f.square() @ wt.square().T + bias.square())
        lin, s2 = torch.cat(lin, -1), torch.cat(s2, -1)
        tol = sum_tol(lin, s2, c + 1)
        rows = slice(anchor_offset, anchor_offset + h * w)
        if origin is not None:
            self._close(origin[:, rows], lin[..., :4], tol[..., :4] + 16 * U32 * lin[..., :4].abs(), f"head level {k}: origin",
                        "head")
        ref, rt = lin.clone(), tol.clone()
        if decode:
            yv, xv = torch.meshgrid(torch.arange(h, device=lin.device), torch.arange(w, device=lin.device), indexing="ij")
            ref[..., 0] = (lin[..., 0] + xv.reshape(-1)) * stride
            ref[..., 1] = (lin[..., 1] + yv.reshape(-1)) * stride
            rt[..., 0:2] = tol[..., 0:2] * stride
            ref[..., 2:4] = torch.exp(lin[..., 2:4]) * stride
            rt[..., 2:4] = ref[..., 2:4] * tol[..., 2:4]
        if sigmoid:
            sg = torch.sigmoid(lin[..., 4:])
            ref[..., 4:] = sg
            rt[..., 4:] = sg * (1 - sg) * tol[..., 4:]
        # + the smallest normal fp32: a sigmoid that underflows may flush to zero; a box size beyond the fp32 range is inf
        got = out[:, rows]
        over = torch.isinf(got) & (ref.abs() * (1 - rt / ref.abs().clamp(min=1e-300)) > FLT_MAX)
        got = torch.where(over, ref, got.to(F64))
        self._close(got, ref, rt + 16 * U32 * ref.abs() + 2.0 ** -126, f"head level {k}: outputs", "head")
        self.head_next = anchor_offset + h * w
        if self.head_next == a_total:
            assert not bool(torch.isnan(out).any()), "head: the levels leave anchor rows unwritten"
            assert origin is None or not bool(torch.isnan(origin).any()), "head: the levels leave origin rows unwritten"

    # -------------------------------------------------------------------- stem input
    def _focus_pack(self, x, frames, y):
        self.orig["focus_pack"](x, frames, y)
        _sync(y.buf)
        self.n["focus"] += 1
        assert torch.equal(nchw64(y), focus_ref(x, frames)), "Focus packing of the bf16 frames"


# ------------------------------------------------------------------------------------------------ the benchmarked forwards
# distinct FUSED launch shapes of the eval forwards (n, cin, cout, h, w, kh, kw, stride, operand, residual)
FUSED_SHAPES = {  # l / m eval at 8 pairs, l on_pipe at batch 1
    "l_eval": [
        (8, 256, 128, 75, 120, 1, 1, 1, 'conv', 'slice'),
        (8, 256, 256, 19, 30, 3, 3, 1, 'conv', 'none'),
        (8, 256, 256, 38, 60, 3, 3, 1, 'conv', 'none'),
        (8, 256, 256, 75, 120, 1, 1, 1, 'conv', 'none'),
        (8, 256, 256, 75, 120, 3, 3, 1, 'conv', 'none'),
        (8, 256, 512, 19, 30, 3, 3, 1, 'pair', 'none'),
        (8, 256, 512, 38, 60, 3, 3, 1, 'pair', 'none'),
        (8, 256, 512, 75, 120, 3, 3, 1, 'pair', 'none'),
        (8, 512, 256, 38, 60, 1, 1, 1, 'conv', 'none'),
        (8, 512, 256, 38, 60, 1, 1, 1, 'conv', 'slice'),
        (8, 1024, 256, 19, 30, 1, 1, 1, 'conv', 'none'),
        (8, 1024, 512, 19, 30, 1, 1, 1, 'conv', 'slice'),
        (16, 64, 64, 150, 240, 1, 1, 1, 'conv', 'none'),
        (16, 64, 64, 150, 240, 3, 3, 1, 'conv', 'in_place'),
        (16, 64, 64, 300, 480, 3, 1, 1, 'stem', 'none'),
        (16, 64, 128, 300, 480, 3, 3, 2, 'conv', 'none'),
        (16, 128, 128, 75, 120, 1, 1, 1, 'conv', 'none'),
        (16, 128, 128, 75, 120, 3, 3, 1, 'conv', 'in_place'),
        (16, 128, 128, 75, 120, 3, 3, 1, 'conv', 'none'),
        (16, 128, 128, 150, 240, 1, 1, 1, 'conv', 'none'),
        (16, 128, 128, 150, 240, 1, 1, 1, 'pair', 'none'),
        (16, 128, 256, 150, 240, 3, 3, 2, 'conv', 'none'),
        (16, 256, 256, 38, 60, 1, 1, 1, 'conv', 'none'),
        (16, 256, 256, 38, 60, 3, 3, 1, 'conv', 'in_place'),
        (16, 256, 256, 38, 60, 3, 3, 1, 'conv', 'none'),
        (16, 256, 256, 75, 120, 1, 1, 1, 'conv', 'none'),
        (16, 256, 256, 75, 120, 1, 1, 1, 'pair', 'none'),
        (16, 256, 256, 75, 120, 3, 3, 2, 'conv', 'none'),
        (16, 256, 512, 75, 120, 3, 3, 2, 'conv', 'none'),
        (16, 512, 256, 38, 60, 1, 1, 1, 'conv', 'none'),
        (16, 512, 256, 75, 120, 1, 1, 1, 'pair', 'none'),
        (16, 512, 512, 19, 30, 1, 1, 1, 'conv', 'none'),
        (16, 512, 512, 19, 30, 3, 3, 1, 'conv', 'none'),
        (16, 512, 512, 38, 60, 1, 1, 1, 'conv', 'none'),
        (16, 512, 512, 38, 60, 1, 1, 1, 'pair', 'none'),
        (16, 512, 512, 38, 60, 3, 3, 2, 'conv', 'none'),
        (16, 512, 1024, 38, 60, 3, 3, 2, 'conv', 'none'),
        (16, 1024, 512, 19, 30, 1, 1, 1, 'conv', 'none'),
        (16, 1024, 512, 38, 60, 1, 1, 1, 'pair', 'none'),
        (16, 1024, 1024, 19, 30, 1, 1, 1, 'conv', 'none'),
        (16, 1024, 1024, 19, 30, 1, 1, 1, 'pair', 'none'),
        (16, 2048, 1024, 19, 30, 1, 1, 1, 'conv', 'none'),
    ],
    "l_on_pipe": [
        (1, 64, 64, 150, 240, 1, 1, 1, 'conv', 'none'),
        (1, 64, 64, 150, 240, 3, 3, 1, 'conv', 'in_place'),
        (1, 64, 64, 300, 480, 3, 1, 1, 'stem', 'none'),
        (1, 64, 128, 300, 480, 3, 3, 2, 'conv', 'none'),
        (1, 128, 128, 75, 120, 1, 1, 1, 'conv', 'none'),
        (1, 128, 128, 75, 120, 3, 3, 1, 'conv', 'in_place'),
        (1, 128, 128, 75, 120, 3, 3, 1, 'conv', 'none'),
        (1, 128, 128, 150, 240, 1, 1, 1, 'conv', 'none'),
        (1, 128, 128, 150, 240, 1, 1, 1, 'pair', 'none'),
        (1, 128, 256, 150, 240, 3, 3, 2, 'conv', 'none'),
        (1, 256, 128, 75, 120, 1, 1, 1, 'conv', 'slice'),
        (1, 256, 256, 19, 30, 3, 3, 1, 'conv', 'none'),
        (1, 256, 256, 38, 60, 1, 1, 1, 'conv', 'none'),
        (1, 256, 256, 38, 60, 3, 3, 1, 'conv', 'in_place'),
        (1, 256, 256, 38, 60, 3, 3, 1, 'conv', 'none'),
        (1, 256, 256, 75, 120, 1, 1, 1, 'conv', 'none'),
        (1, 256, 256, 75, 120, 1, 1, 1, 'pair', 'none'),
        (1, 256, 256, 75, 120, 3, 3, 1, 'conv', 'none'),
        (1, 256, 256, 75, 120, 3, 3, 2, 'conv', 'none'),
        (1, 256, 512, 19, 30, 3, 3, 1, 'pair', 'none'),
        (1, 256, 512, 38, 60, 3, 3, 1, 'pair', 'none'),
        (1, 256, 512, 75, 120, 3, 3, 1, 'pair', 'none'),
        (1, 256, 512, 75, 120, 3, 3, 2, 'conv', 'none'),
        (1, 512, 256, 38, 60, 1, 1, 1, 'conv', 'none'),
        (1, 512, 256, 38, 60, 1, 1, 1, 'conv', 'slice'),
        (1, 512, 256, 75, 120, 1, 1, 1, 'pair', 'none'),
        (1, 512, 512, 19, 30, 1, 1, 1, 'conv', 'none'),
        (1, 512, 512, 19, 30, 3, 3, 1, 'conv', 'none'),
        (1, 512, 512, 38, 60, 1, 1, 1, 'conv', 'none'),
        (1, 512, 512, 38, 60, 1, 1, 1, 'pair', 'none'),
        (1, 512, 512, 38, 60, 3, 3, 2, 'conv', 'none'),
        (1, 512, 1024, 38, 60, 3, 3, 2, 'conv', 'none'),
        (1, 1024, 256, 19, 30, 1, 1, 1, 'conv', 'none'),
        (1, 1024, 512, 19, 30, 1, 1, 1, 'conv', 'none'),
        (1, 1024, 512, 19, 30, 1, 1, 1, 'conv', 'slice'),
        (1, 1024, 512, 38, 60, 1, 1, 1, 'pair', 'none'),
        (1, 1024, 1024, 19, 30, 1, 1, 1, 'conv', 'none'),
        (1, 1024, 1024, 19, 30, 1, 1, 1, 'pair', 'none'),
        (1, 2048, 1024, 19, 30, 1, 1, 1, 'conv', 'none'),
    ],
    "m_eval": [
        (8, 192, 96, 75, 120, 1, 1, 1, 'conv', 'slice'),
        (8, 192, 192, 19, 30, 3, 3, 1, 'conv', 'none'),
        (8, 192, 192, 38, 60, 3, 3, 1, 'conv', 'none'),
        (8, 192, 192, 75, 120, 1, 1, 1, 'conv', 'none'),
        (8, 192, 192, 75, 120, 3, 3, 1, 'conv', 'none'),
        (8, 192, 384, 19, 30, 3, 3, 1, 'pair', 'none'),
        (8, 192, 384, 38, 60, 3, 3, 1, 'pair', 'none'),
        (8, 192, 384, 75, 120, 3, 3, 1, 'pair', 'none'),
        (8, 384, 192, 38, 60, 1, 1, 1, 'conv', 'none'),
        (8, 384, 192, 38, 60, 1, 1, 1, 'conv', 'slice'),
        (8, 768, 192, 19, 30, 1, 1, 1, 'conv', 'none'),
        (8, 768, 384, 19, 30, 1, 1, 1, 'conv', 'slice'),
        (16, 48, 48, 150, 240, 1, 1, 1, 'conv', 'none'),
        (16, 48, 48, 150, 240, 3, 3, 1, 'conv', 'in_place'),
        (16, 48, 96, 300, 480, 3, 3, 2, 'conv', 'none'),
        (16, 64, 48, 300, 480, 3, 1, 1, 'stem', 'none'),
        (16, 96, 96, 75, 120, 1, 1, 1, 'conv', 'none'),
        (16, 96, 96, 75, 120, 3, 3, 1, 'conv', 'in_place'),
        (16, 96, 96, 75, 120, 3, 3, 1, 'conv', 'none'),
        (16, 96, 96, 150, 240, 1, 1, 1, 'conv', 'none'),
        (16, 96, 96, 150, 240, 1, 1, 1, 'pair', 'none'),
        (16, 96, 192, 150, 240, 3, 3, 2, 'conv', 'none'),
        (16, 192, 192, 38, 60, 1, 1, 1, 'conv', 'none'),
        (16, 192, 192, 38, 60, 3, 3, 1, 'conv', 'in_place'),
        (16, 192, 192, 38, 60, 3, 3, 1, 'conv', 'none'),
        (16, 192, 192, 75, 120, 1, 1, 1, 'conv', 'none'),
        (16, 192, 192, 75, 120, 1, 1, 1, 'pair', 'none'),
        (16, 192, 192, 75, 120, 3, 3, 2, 'conv', 'none'),
        (16, 192, 384, 75, 120, 3, 3, 2, 'conv', 'none'),
        (16, 384, 192, 38, 60, 1, 1, 1, 'conv', 'none'),
        (16, 384, 192, 75, 120, 1, 1, 1, 'pair', 'none'),
        (16, 384, 384, 19, 30, 1, 1, 1, 'conv', 'none'),
        (16, 384, 384, 19, 30, 3, 3, 1, 'conv', 'none'),
        (16, 384, 384, 38, 60, 1, 1, 1, 'conv', 'none'),
        (16, 384, 384, 38, 60, 1, 1, 1, 'pair', 'none'),
        (16, 384, 384, 38, 60, 3, 3, 2, 'conv', 'none'),
        (16, 384, 768, 38, 60, 3, 3, 2, 'conv', 'none'),
        (16, 768, 384, 19, 30, 1, 1, 1, 'conv', 'none'),
        (16, 768, 384, 38, 60, 1, 1, 1, 'pair', 'none'),
        (16, 768, 768, 19, 30, 1, 1, 1, 'conv', 'none'),
        (16, 768, 768, 19, 30, 1, 1, 1, 'pair', 'none'),
        (16, 1536, 768, 19, 30, 1, 1, 1, 'conv', 'none'),
    ],
}

PAIRS = 8


def _build(tag, momentum=0.03):
    (depth, width), (gamma, thr, val) = MODELS[tag]
    m = build_product(depth, width, gamma, thr, val, momentum=momentum)
    engine.name_modules(m)
    return m.train()


def _pairs(pairs):
    return (synth.synth_frames(pairs, 600, 960, seed=4321).cuda(),
            tuple(t.cuda() for t in synth.synth_labels(pairs, 600, 960, seed=11)))


def _report(what, ck):
    print(f"\nFWD {what}: launches {dict(ck.n)}; worst " + ", ".join(f"{k} {v:.3g}" for k, v in sorted(ck.worst.items())))


def _calibrated(tag, x):
    """eval model whose running statistics are the batch statistics of ``x`` (one train-mode forward at BN momentum 1):
    random-init running statistics on 0-255 frames would leave the activations un-normalised"""
    m = _build(tag, momentum=1.0)
    fut, cur = synth.synth_labels(x.shape[0], 600, 960, seed=11)
    with torch.no_grad():
        m(x, (fut.cuda(), cur.cuda()))
    return m.eval()


@pytest.mark.parametrize("tag,launches", [("l", 114), ("m", 90), ("s", 66)])
def test_train_forward_every_launch(tag, launches):
    """the headline path: model(x, targets) in train mode, no gradient (the two frames batched with grouped statistics,
    the DFP jian convs batched with group-offset destinations)"""
    m = _build(tag)
    x, tg = _pairs(PAIRS)
    with torch.no_grad():
        m(x, tg)
        with FwdChecker(m) as ck:
            loss = m(x, tg)
    assert conv_launches(m, jian_twice=False) == launches
    assert ck.n == Counter(conv=launches, apply=launches, head=3, focus=1), ck.n
    assert all(bool(torch.isfinite(loss[k])) for k in ORDER)
    _report(f"{tag} train b{PAIRS}", ck)


def test_recording_forward_every_launch_l_b4():
    """the tape-building forward of a training step (l_b4_ddp): jian not batched, mean / invstd written for the backward"""
    m = _build("l")
    x, tg = _pairs(4)
    with torch.no_grad():
        m(x, tg)
    with FwdChecker(m) as ck:
        _, loss = backward._record(m, x, tg)
    launches = conv_launches(m, jian_twice=True)
    assert launches == 117
    assert ck.n == Counter(conv=launches, apply=launches, head=3, focus=1, mean_invstd=launches), ck.n
    assert bool(torch.isfinite(loss).all())
    _report("l recording b4", ck)


def test_recording_forward_every_launch_still_l():
    """the still model (PIPEHead on [B, 3, H, W]): one backbone + PAFPN pass whose running statistics are updated twice"""
    (depth, width), _ = MODELS["l"]
    m = build_still(depth, width)
    engine.name_modules(m)
    x, labels = still_batch(PAIRS, 600, 960)
    with torch.no_grad():
        m(x, labels)
    with FwdChecker(m) as ck:
        _, loss = backward._record(m, x, labels)
    launches = conv_launches(m, jian_twice=True)
    head = 4 * len(m.head.strides)            # stem, cls | reg pair, cls and reg tower convs per level
    assert ck.n == Counter(conv=launches, apply=launches, head=3, focus=1, mean_invstd=launches,
                           stat_updates_2=launches - 6 - head), ck.n
    assert bool(torch.isfinite(loss).all())
    _report(f"l still recording b{PAIRS}", ck)


@pytest.mark.parametrize("tag,launches", [("l", 117), ("m", 93)])
def test_eval_forward_every_launch(tag, launches):
    x = synth.synth_frames(PAIRS, 600, 960, seed=99).cuda()
    m = _calibrated(tag, x)
    with torch.no_grad(), FwdChecker(m, nondegenerate=True) as ck:
        out = m(x)
    assert conv_launches(m, jian_twice=True) == launches
    assert ck.n == Counter(conv=launches, head=3, focus=1), ck.n
    assert tuple(out.shape) == (PAIRS, 11850, 13)
    assert ck.fused_shapes == set(FUSED_SHAPES[f"{tag}_eval"]), sorted(ck.fused_shapes ^ set(FUSED_SHAPES[f"{tag}_eval"]))
    _report(f"{tag} eval b{PAIRS}", ck)


def test_on_pipe_every_launch_l():
    """streaming at batch 1: the star call, a buffered call on the buffer straight from the previous call, and one on a
    cloned buffer (how bench.py carries it)"""
    m = _calibrated("l", synth.synth_frames(PAIRS, 600, 960, seed=99).cuda())
    f = synth.synth_frames(3, 600, 960, seed=98)[:, :3].contiguous().cuda()
    launches = conv_launches(m, jian_twice=True)
    shapes = set()
    with torch.no_grad():
        buf = None
        for i in range(3):
            with FwdChecker(m, nondegenerate=True) as ck:
                if i == 0:
                    _, buf = m(f[0:1], mode="on_pipe")
                else:
                    _, nb = m(f[i:i + 1], buffer=buf if i == 1 else tuple(t.clone() for t in buf), mode="on_pipe")
                    buf = nb
            assert ck.n == Counter(conv=launches, head=3, focus=1), ck.n
            shapes |= ck.fused_shapes
            _report(f"l on_pipe call {i}", ck)
    assert shapes == set(FUSED_SHAPES["l_on_pipe"]), sorted(shapes ^ set(FUSED_SHAPES["l_on_pipe"]))


# ------------------------------------------------------------------------------------------------ FUSED per shape
FUSED_CASES = sorted(set(c for v in FUSED_SHAPES.values() for c in v))


@pytest.mark.parametrize("case", FUSED_CASES, ids=lambda c: "x".join(map(str, c)))
def test_fused_shape_every_tiling(case):
    """the eval epilogue at one launch shape: random folded scale / shift, SiLU, the residual in place (bottleneck 3x3) or
    from a slice of another buffer (jian), the output a channel slice of a wider buffer holding a sentinel"""
    n, ci, co, h, w, kh, kw, s, kind, rk = case
    g = torch.Generator(device=DEV).manual_seed(sum(v for v in case if isinstance(v, int)))
    if kind == "stem":
        frames = torch.rand((n, 3, 2 * h, 2 * w), generator=g, device=DEV) * 255
        xv = View.empty(n, h, w, 64, DEV)
        ops.focus_pack(frames, 1, xv)
        w12 = (torch.randn((co, 12, 3, 3), generator=g, device=DEV) / 108 ** 0.5).to(torch.bfloat16).float()
        wpk, w64 = ops.pack_stem_weight(w12), stem_weight_3x1(w12.to(F64))
    else:
        xv = post_silu(n, h, w, ci, 1)
        ws = [(torch.randn((c_, ci, kh, kw), generator=g, device=DEV) / (ci * kh * kw) ** 0.5).to(torch.bfloat16).float()
              for c_ in ((co // 2, co // 2) if kind == "pair" else (co,))]
        wpk, w64 = ops.pack_conv_weight(*ws), torch.cat(ws, 0).to(F64)
    ho, wo = ops.conv_out_hw(h, w, kh, s) if kh == kw else (h, w)
    sc = torch.rand(co, generator=g, device=DEV) + 0.5
    sh = torch.rand(co, generator=g, device=DEV) - 0.5
    sentinel = torch.full((n, ho, wo, co + 64), -7.0, dtype=torch.bfloat16, device=DEV)
    r0 = post_silu(n, ho, wo, 2 * co, 2)
    x64 = nchw64(xv)
    res64 = nchw64(r0.ch(co, co)) if rk != "none" else None
    ref, omit = conv_refs(x64, w64, s, sc.to(F64)[None, :, None, None], sh.to(F64)[None, :, None, None], 1, res64)
    del x64
    for tname, tiling in DGRAD_TILINGS.items():
        wide = sentinel.clone()
        y = View(wide).ch(32, co)
        res = None
        if rk == "in_place":
            y.torch().copy_(r0.ch(co, co).torch())
            res = y
        elif rk == "slice":
            res = r0.ch(co, co)
        ops.conv2d(xv, wpk, y, (kh, kw), s, ops.SY_CONV_FUSED, scale=sc, shift=sh, act=1, res=res, **tiling)
        torch.cuda.synchronize()
        got = nchw64(y)
        what = f"FUSED {case} {tname}"
        check_close(got, ref, what)
        assert bf16_ratio(got, ref)[1] <= REL_L2, what
        assert outside_bf16(got, omit) > 0, f"{what}: the bar accepts input channels 0-63 at the centre tap left out"
        wide[..., 32:32 + co] = sentinel[..., 32:32 + co]
        assert _same_bits(wide, sentinel), f"{what}: writes outside its output slice"


# ------------------------------------------------------------------------------------------------ CUDA-graph replay
def test_graph_replay_equals_eager_l():
    """bench.py times CUDA-graph replays; the kernels are deterministic, so a replay must reproduce the eager call bit for
    bit: the six losses of the train plain forward, the eval outputs, and an on_pipe sequence carrying its buffer"""
    from bench import capture
    m = _build("l")
    x, tg = _pairs(PAIRS)
    with torch.no_grad():
        eager = m(x, tg)
        want = torch.stack([eager[k] for k in ORDER]).clone()
        g, out = capture(lambda: m(x, tg))
        g.replay()
        torch.cuda.synchronize()
        assert torch.equal(torch.stack([out[k] for k in ORDER]), want), (torch.stack([out[k] for k in ORDER]), want)
        del g, out
        m.eval()
        want = m(x).clone()
        g, out = capture(lambda: m(x))
        g.replay()
        torch.cuda.synchronize()
        assert torch.equal(out, want)
        del g, out
        f = synth.synth_frames(4, 600, 960, seed=98)[:, :3].contiguous().cuda()
        _, buf = m(f[0:1], mode="on_pipe")
        buf0 = tuple(t.clone() for t in buf)
        eager, cur = [], buf0
        for i in range(1, 4):
            o, nb = m(f[i:i + 1], buffer=cur, mode="on_pipe")
            eager.append(o.clone())
            cur = tuple(t.clone() for t in nb)
        f_static, buf_static = f[1:2].clone(), tuple(t.clone() for t in buf0)

        def frame():
            o2, nb2 = m(f_static, buffer=buf_static, mode="on_pipe")
            for d_, s_ in zip(buf_static, nb2):
                d_.copy_(s_)
            return o2
        g, out = capture(frame)
        for d_, s_ in zip(buf_static, buf0):          # the capture's warm-up call advanced the buffer: start over
            d_.copy_(s_)
        for i in range(1, 4):
            f_static.copy_(f[i:i + 1])
            g.replay()
            torch.cuda.synchronize()
            assert torch.equal(out, eager[i - 1]), f"on_pipe frame {i}"
