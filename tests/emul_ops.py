"""CPU emulation of the ``streamyolo_b200.ops`` entry points in plain PyTorch -- TEST INFRASTRUCTURE ONLY.

The product has no CPU path (``ops.lib()`` raises without the CUDA library and an sm_90 device).  The host-side logic above
the C ABI -- which buffers feed which kernel, in-place concat slices, gradient routing of the backward walk -- is plain
Python, though, and can be checked without a GPU if every kernel call is replaced by a few lines of torch with the same
contract (same arguments, same bf16 rounding points).  ``install(monkeypatch)`` swaps the functions of ``ops`` for these;
tests/test_cpu_backward.py then runs the whole recording forward + backward walk on CPU tensors and compares every
parameter gradient with autograd through the oracle.  Each kernel itself is tested on the GPU against autograd /
the oracle in tests/test_gpu_ops.py and tests/test_gpu_model.py."""
import torch
import torch.nn.functional as F

from oracle.streamyolo_oracle import OracleCfg, StreamYoloOracle
from streamyolo_b200 import ops
from streamyolo_b200.ops import View

PTRS = {}        # data_ptr -> tensor, for the entry points that take raw device pointers (bn_act_apply)
LOSS_STATE = {}  # workspace data_ptr -> what tal_loss leaves for tal_loss_backward


EXACT = False    # True: fp32 "storage" everywhere (no bf16 rounding), so that the emulated product equals the fp32 oracle up to
                 # float roundoff -- a random-init train-mode BatchNorm net amplifies bf16 rounding noise to tens of percent
                 # in the gradients, which would hide routing mistakes


def _bf(t):
    return t.float() if EXACT else t.to(torch.bfloat16)


def _nchw(v: View):
    return v.torch().permute(0, 3, 1, 2).float()


def _store(v: View, t_nchw):
    """one rounding to the view's storage (bf16, fp16, or fp32 in EXACT mode)"""
    v.torch().copy_(t_nchw.permute(0, 2, 3, 1))


def _require(cond, msg):
    """the library's argument checks: it refuses before any launch, with ops._check's RuntimeError"""
    if not cond:
        raise RuntimeError("libstreamyolo_sm100 error 1: " + msg)


ACTS = (ops.SY_ACT_NONE, ops.SY_ACT_SILU, ops.SY_ACT_RELU, ops.SY_ACT_LRELU)


def _act(t, code):
    """the SY_ACT_* activation (include/streamyolo_sm100.h)"""
    _require(code in ACTS, f"act={code} is not an SY_ACT_* code")
    if code == ops.SY_ACT_SILU:
        return F.silu(t)
    if code == ops.SY_ACT_RELU:
        return F.relu(t)
    return F.leaky_relu(t, 0.1) if code == ops.SY_ACT_LRELU else t


def _dact(z, code):
    """its derivative, autograd's value at z = 0 (0 for ReLU, 0.1 for LeakyReLU)"""
    if code == ops.SY_ACT_SILU:
        s = torch.sigmoid(z)
        return s * (1 + z * (1 - s))
    if code == ops.SY_ACT_RELU:
        return (z > 0).to(z.dtype)
    if code == ops.SY_ACT_LRELU:
        return torch.where(z > 0, torch.ones_like(z), torch.full_like(z, 0.1))
    return torch.ones_like(z)


def _unpack(wpk, kh, kw):
    """bf16 [O][kh*kw][I] -> float OIHW"""
    o, taps, i = wpk.shape
    return wpk.float().reshape(o, kh, kw, i).permute(0, 3, 1, 2).contiguous()


def conv_stat_rows():
    """the library's is the SM count (132 on an H100 SXM, 114 on a PCIe card); the host only sizes the partials of a RAW
    launch with it and hands them back, so any count the conv below accepts serves"""
    return 132


def conv2d(x, wpk, y, k, s, mode, impl="tc", scale=None, shift=None, act=1, res=None, partials=None, split_n=0,
           timeline=None, debug_flags=0, bn=None, momentum=0.03, eps=1e-3, scale_shift=None, sync=None, mean_invstd=None,
           debug_f32=None, tile_mode=0, tile_bn=0, stat_updates=1):
    """Returns the number of partial rows written: one row per launch with ``partials`` (the sums of the whole batch,
    [Cout][2 groups][2 (sum, sumsq)] as the library lays out each of its per-CTA rows), 0 without."""
    kh, kw = (k, k) if isinstance(k, int) else k
    dtypes = {x.dtype, y.dtype, wpk.dtype} | ({res.dtype} if res is not None else set())
    if len(dtypes) != 1:
        raise ValueError(f"conv2d: x, y, res and the packed weights must share one storage dtype, got {sorted(map(str, dtypes))}")
    _require(act in ACTS, f"conv2d: act={act} is not an SY_ACT_* code")
    _require(x.dtype != torch.float16 or (mode == ops.SY_CONV_FUSED and not bn and partials is None and impl != "simt"),
             "conv2d: fp16 storage is FUSED mode only, without statistics")
    one_group = not 0 < split_n < x.n
    _require(stat_updates in (0, 1, 2) and (stat_updates != 2 or (bn and one_group)),
             f"conv2d: stat_updates={stat_updates} with split_n={split_n} of {x.n}")
    _require(partials is None or partials.shape[0] >= conv_stat_rows(), "conv2d: too few statistic rows")
    if impl == "dw":                                # depthwise: wpk [kh*kw][C]
        c = wpk.shape[1]
        out = F.conv2d(_nchw(x), wpk.float().t().reshape(c, 1, kh, kw), None, s, ((kh - 1) // 2, (kw - 1) // 2), groups=c)
    else:
        out = F.conv2d(_nchw(x), _unpack(wpk, kh, kw), None, s, ((kh - 1) // 2, (kw - 1) // 2))
    if mode == ops.SY_CONV_FUSED:
        if scale is not None:
            out = out * scale.float()[None, :, None, None] + shift.float()[None, :, None, None]
        out = _act(out, act)
        if res is not None:
            out = out + _nchw(res)
        _store(y, out)
        return 0
    _store(y, out)
    stored = _nchw(y)
    n = stored.shape[0]
    sp = split_n if 0 < split_n < n else n
    groups = [(0, sp), (sp, n)] if sp < n else [(0, n)]
    if partials is not None:
        row = partials[0].view(stored.shape[1], 2, 2)
        for gi, (a, b) in enumerate(groups):
            row[:, gi, 0] = stored[a:b].sum((0, 2, 3))
            row[:, gi, 1] = stored[a:b].pow(2).sum((0, 2, 3))
    if bn:
        c0s = [seg[5] for seg in bn] + [stored.shape[1]]
        for gi, (a, b) in enumerate(groups):
            part = stored[a:b]
            mean = part.mean((0, 2, 3))
            var = part.var((0, 2, 3), unbiased=False)
            cnt = part.numel() / part.shape[1]
            invstd = (var + eps).rsqrt()
            for si, (gamma, beta, rm, rv, nbt, c0) in enumerate(bn):
                sl = slice(c0, c0s[si + 1])
                sc = gamma.detach().float() * invstd[sl]
                scale_shift[0, gi, sl] = sc
                scale_shift[1, gi, sl] = beta.detach().float() - mean[sl] * sc
                if mean_invstd is not None:
                    mean_invstd[0, gi, sl] = mean[sl]
                    mean_invstd[1, gi, sl] = invstd[sl]
                for _ in range(max(stat_updates, 1)):
                    if rm is not None:
                        rm.mul_(1 - momentum).add_(momentum * mean[sl])
                        rv.mul_(1 - momentum).add_(momentum * var[sl] * (cnt / max(cnt - 1, 1)))
                    if nbt is not None:
                        nbt.add_(1)
        PTRS[scale_shift[0].data_ptr()] = scale_shift[0]
        PTRS[scale_shift[1].data_ptr()] = scale_shift[1]
    return 1 if partials is not None else 0


def _strided(v: View, img0, nimg, goff):
    """NHWC torch view of images [img0, img0 + nimg) of ``v`` with the base address moved by ``goff`` elements (the
    group-offset destinations of the batched DFP fusion address image n - B, channels [half, 2 half) that way)."""
    b = v.buf
    H, W, Ct = b.shape[1], b.shape[2], b.shape[3]
    return torch.as_strided(b.view(-1), (nimg, H, W, v.c), (H * W * Ct, W * Ct, Ct, 1),
                            (v.n0 + img0) * H * W * Ct + v.c0 + v.off + goff)


def bn_act_apply(x, scale_ptr, shift_ptr, split_n, act, res, y, y_goff1=0, res_goff1=0):
    """group 1 = the images >= split_n (split_n <= 0: every image, split_n >= n: none); a scale / shift of one row serves a
    launch whose images are all in group 0"""
    scale, shift = (scale_ptr, shift_ptr) if torch.is_tensor(scale_ptr) else (PTRS[scale_ptr], PTRS[shift_ptr])   # [2 groups][C]
    _require((x.n, x.h, x.w, x.c) == (y.n, y.h, y.w, y.c), "bn_act_apply: x/y shape mismatch")
    _require(res is None or (res.n, res.h, res.w, res.c) == (x.n, x.h, x.w, x.c), "bn_act_apply: residual mismatch")
    _require(y_goff1 % 8 == 0 and res_goff1 % 8 == 0, "bn_act_apply: group offsets must be multiples of 8")
    _require(act in ACTS, f"bn_act_apply: act={act} is not an SY_ACT_* code")
    scale, shift = scale.reshape(-1, x.c), shift.reshape(-1, x.c)
    t = _nchw(x)
    n = t.shape[0]
    sp = min(max(split_n, 0), n)
    outs = []
    for gi, (a, b, yo, ro) in enumerate([(0, sp, 0, 0), (sp, n, y_goff1, res_goff1)]):
        if a >= b:
            continue
        out = _act(t[a:b] * scale[gi][None, :, None, None] + shift[gi][None, :, None, None], act)
        if res is not None:
            out = out + _strided(res, a, b - a, ro).permute(0, 3, 1, 2).float()
        outs.append((a, b, yo, out))
    for a, b, yo, out in outs:           # every residual is read before any output is written (in-place residuals)
        _strided(y, a, b - a, yo).copy_(out.permute(0, 2, 3, 1))


def focus_pack(x, frames, y):
    b = x.shape[0]
    xs = torch.cat([x[:, 3 * f:3 * f + 3] for f in range(frames)], 0)
    xs = xs.float() if EXACT else xs.to(y.dtype).float()
    foc = torch.cat([xs[..., ::2, ::2], xs[..., 1::2, ::2], xs[..., ::2, 1::2], xs[..., 1::2, 1::2]], 1)   # [n,12,h,w]
    n, _, h, w = foc.shape
    out = torch.zeros(n, 64, h, w)
    out[:, 16:28] = foc
    out[:, 0:12, :, 1:] = foc[..., :-1]
    out[:, 32:44, :, :-1] = foc[..., 1:]
    _store(y, out)
    assert n == frames * b


def _same_dtype(what, *views):
    if len({v.dtype for v in views}) != 1:
        raise ValueError(f"{what}: the views must share one storage dtype")


def upsample_nearest(x, y):
    _same_dtype("upsample_nearest", x, y)
    _store(y, F.interpolate(_nchw(x), size=(y.h, y.w), mode="nearest"))


def spp_maxpool(x, y5, y9, y13):
    _same_dtype("spp_maxpool", x, y5, y9, y13)
    t = _nchw(x)
    for k, v in ((5, y5), (9, y9), (13, y13)):
        _store(v, F.max_pool2d(t, k, 1, k // 2))


def copy(x, y):
    _same_dtype("copy", x, y)
    _require((x.n, x.h, x.w, x.c) == (y.n, y.h, y.w, y.c), "copy: view mismatch")
    y.torch().copy_(x.torch())


def head_pred_decode(cls_feat, reg_feat, w_reg, b_reg, w_obj, b_obj, w_cls, b_cls, stride, anchor_offset, a_total, out,
                     origin, sigmoid, decode):
    if cls_feat.dtype != reg_feat.dtype:
        raise ValueError("head_pred_decode: the views must share one storage dtype")
    _require(0 <= anchor_offset and anchor_offset + cls_feat.h * cls_feat.w <= a_total, "head_pred: anchor range")
    cf, rf = _nchw(cls_feat), _nchw(reg_feat)
    o = torch.cat([F.conv2d(rf, w_reg[:, :, None, None], b_reg), F.conv2d(rf, w_obj[:, :, None, None], b_obj),
                   F.conv2d(cf, w_cls[:, :, None, None], b_cls)], 1)
    b, no, h, w = o.shape
    flat = o.flatten(2).permute(0, 2, 1).clone()
    sl = slice(anchor_offset, anchor_offset + h * w)
    if origin is not None:
        origin[:, sl] = flat[..., :4]
    if decode:
        yv, xv = torch.meshgrid(torch.arange(h), torch.arange(w), indexing="ij")
        flat[..., 0] = (flat[..., 0] + xv.reshape(-1)) * stride
        flat[..., 1] = (flat[..., 1] + yv.reshape(-1)) * stride
        flat[..., 2:4] = torch.exp(flat[..., 2:4]) * stride
    if sigmoid:
        flat[..., 4:] = torch.sigmoid(flat[..., 4:])
    out[:, sl] = flat


def tal_loss_workspace_bytes(b, a_total, max_labels, num_classes):
    """the host allocates this many bytes and hands the buffer to tal_loss / tal_loss_backward: here it only keys
    LOSS_STATE"""
    return 256


def _loss_oracle(hw, strides, gamma, thr, val, nc):
    o = StreamYoloOracle(OracleCfg(gamma=gamma, ignore_thr=thr, ignore_value=val, num_classes=nc, strides=tuple(strides)), {})
    grid = o.grids(list(hw), o.cfg.strides)
    return o, tuple(g.float() for g in grid)


def tal_loss(outputs, origin, labels_fut, labels_cur, hw, strides, gamma, ignore_thr, ignore_value, use_l1, workspace,
             loss_out, fg_out=None, matched_out=None, pred_iou_out=None):
    _require(sum(h * w for h, w in hw) == outputs.shape[1], "tal_loss: levels give the wrong anchor count")
    _require(workspace.numel() * workspace.element_size() >= tal_loss_workspace_bytes(
        outputs.shape[0], outputs.shape[1], labels_fut.shape[1], outputs.shape[2] - 5), "tal_loss: workspace too small")
    _require(not use_l1 or origin is not None, "tal_loss: use_l1 needs origin preds")
    o, grid = _loss_oracle(hw, strides, gamma, ignore_thr, ignore_value, outputs.shape[2] - 5)
    with torch.enable_grad():
        out_l, org_l = outputs.clone().requires_grad_(True), origin.clone().requires_grad_(True)
        r = o.losses(out_l, org_l, grid, (labels_fut, labels_cur))
        r["total_loss"].backward()
    LOSS_STATE[workspace.data_ptr()] = (out_l.grad, org_l.grad, grid)
    vals = [r["total_loss"], r["iou_loss"], r["conf_loss"], r["cls_loss"], r["l1_loss"], r["num_fg"]]
    loss_out.copy_(torch.tensor([float(v) for v in vals]))


def tal_loss_backward(outputs, origin, labels_fut, hw, strides, gamma, use_l1, workspace, grad_scale=1.0, grad_outputs=None,
                      grad_origin=None, grad_raw=None):
    g_out, g_org, grid = LOSS_STATE[workspace.data_ptr()]
    gs = grid[2]
    if grad_outputs is not None:
        grad_outputs.copy_(g_out * grad_scale)
    if grad_origin is not None:
        grad_origin.copy_(g_org * grad_scale)
    if grad_raw is not None:
        raw = g_out.clone()
        raw[..., 0:2] = g_out[..., 0:2] * gs[None, :, None] + g_org[..., 0:2]
        raw[..., 2:4] = g_out[..., 2:4] * outputs[..., 2:4] + g_org[..., 2:4]
        grad_raw.copy_(raw * grad_scale)


def head_pred_backward(grad_raw, cls_feat, reg_feat, d_cls_feat, d_reg_feat, w_reg, w_obj, w_cls, a_total, anchor_offset,
                       dw_reg, dw_obj, dw_cls, db_reg, db_obj, db_cls, accumulate=False):
    """1 <= classes <= 27, as sy_head_pred_backward"""
    _require(1 <= w_cls.shape[0] <= 27, "head_pred_backward: num_classes out of range")
    _head_pred_bwd(grad_raw, cls_feat, reg_feat, d_cls_feat, d_reg_feat, w_reg, w_obj, w_cls, a_total, anchor_offset, dw_reg,
                   dw_obj, dw_cls, db_reg, db_obj, db_cls, accumulate)


def head_pred_backward_wide(grad_raw, cls_feat, reg_feat, d_cls_feat, d_reg_feat, w_reg, w_obj, w_cls, a_total,
                            anchor_offset, dw_reg, dw_obj, dw_cls, db_reg, db_obj, db_cls, accumulate=False):
    """1 <= classes <= 251 with (5 + classes) x channels x 4 bytes <= 200 KiB, as sy_head_pred_backward_wide"""
    nc = w_cls.shape[0]
    _require(1 <= nc <= 251 and cls_feat.c % 8 == 0 and 4 * (5 + nc) * cls_feat.c <= 200 * 1024,
             "head_pred_backward_wide: num_classes out of range")
    _head_pred_bwd(grad_raw, cls_feat, reg_feat, d_cls_feat, d_reg_feat, w_reg, w_obj, w_cls, a_total, anchor_offset, dw_reg,
                   dw_obj, dw_cls, db_reg, db_obj, db_cls, accumulate)


def _head_pred_bwd(grad_raw, cls_feat, reg_feat, d_cls_feat, d_reg_feat, w_reg, w_obj, w_cls, a_total, anchor_offset,
                   dw_reg, dw_obj, dw_cls, db_reg, db_obj, db_cls, accumulate):
    h, w = cls_feat.h, cls_feat.w
    _require(0 <= anchor_offset and anchor_offset + h * w <= a_total, "head_pred_backward: anchor range")
    g = grad_raw[:, anchor_offset:anchor_offset + h * w]                    # [b, hw, no]
    cf, rf = cls_feat.torch().float().flatten(1, 2), reg_feat.torch().float().flatten(1, 2)   # [b, hw, c]
    d_rf = g[..., 0:4] @ w_reg + g[..., 4:5] @ w_obj
    d_cf = g[..., 5:] @ w_cls
    d_reg_feat.torch().copy_(d_rf.reshape(d_reg_feat.torch().shape))
    d_cls_feat.torch().copy_(d_cf.reshape(d_cls_feat.torch().shape))
    res = [torch.einsum("bpo,bpc->oc", g[..., 0:4], rf), torch.einsum("bpo,bpc->oc", g[..., 4:5], rf),
           torch.einsum("bpo,bpc->oc", g[..., 5:], cf), g[..., 0:4].sum((0, 1)), g[..., 4:5].sum((0, 1)), g[..., 5:].sum((0, 1))]
    for dst, val in zip((dw_reg, dw_obj, dw_cls, db_reg, db_obj, db_cls), res):
        dst.copy_(dst + val.reshape(dst.shape) if accumulate else val.reshape(dst.shape))


def bn_act_backward(raw, dy, draw, scale, shift, mean, invstd, split_n, act, dgamma, dbeta, accumulate=False):
    _require(act in ACTS, f"bn_act_backward: act={act} is not an SY_ACT_* code")
    r, d = _nchw(raw), _nchw(dy)
    n = r.shape[0]
    sp = split_n if 0 < split_n < n else n
    out = torch.empty_like(r)
    dg, db = torch.zeros_like(dgamma), torch.zeros_like(dbeta)
    for gi, (a, b) in enumerate([(0, sp), (sp, n)] if sp < n else [(0, n)]):
        sc, sh, mu, iv = (t[gi][None, :, None, None] for t in (scale, shift, mean, invstd))
        dz = d[a:b] * _dact(r[a:b] * sc + sh, act)
        xh = (r[a:b] - mu) * iv
        m1, m2 = dz.mean((0, 2, 3), keepdim=True), (dz * xh).mean((0, 2, 3), keepdim=True)
        out[a:b] = sc * (dz - m1 - xh * m2)
        db += dz.sum((0, 2, 3))
        dg += (dz * xh).sum((0, 2, 3))
    _store(draw, out)
    dgamma.copy_(dgamma + dg if accumulate else dg)
    dbeta.copy_(dbeta + db if accumulate else db)


def conv2d_wgrad(x, dy, k, s, dw, accumulate=False, workspace=None):
    kh, kw = (k, k) if isinstance(k, int) else k
    g = torch.nn.grad.conv2d_weight(_nchw(x), dw.shape, _nchw(dy), stride=s, padding=((kh - 1) // 2, (kw - 1) // 2))
    dw.copy_(dw + g if accumulate else g)
    return workspace


def dilate2(g, D):
    _require(g.n == D.n and g.c == D.c and D.h in (2 * g.h - 1, 2 * g.h) and D.w in (2 * g.w - 1, 2 * g.w), "dilate2: bad views")
    D.torch().zero_()
    D.torch()[:, ::2, ::2, :][:, :g.h, :g.w] = g.torch()


def upsample_nearest_backward(dy, dx):
    with torch.enable_grad():
        x = torch.zeros(dx.n, dx.c, dx.h, dx.w, requires_grad=True)
        F.interpolate(x, size=(dy.h, dy.w), mode="nearest").backward(_nchw(dy))
    _store(dx, x.grad)


def spp_maxpool_backward(x, d5, d9, d13, dx):
    with torch.enable_grad():
        t = _nchw(x).requires_grad_(True)
        for k, d in ((5, d5), (9, d9), (13, d13)):
            F.max_pool2d(t, k, 1, k // 2).backward(_nchw(d))
    _store(dx, t.grad)


def add_(x, y):
    _require((x.n, x.h, x.w, x.c) == (y.n, y.h, y.w, y.c), "add: view mismatch")
    _store(y, _nchw(x) + _nchw(y))


def sgd_nesterov_ema_step(param, grad, momentum_buf, ema, n_param, decay_begin, lr, momentum=0.9, weight_decay=5e-4,
                          inv_scale=1.0, nesterov=True, ema_decay=0.0, found_inf=None, hyper=None, found_inf_ema=False):
    """what sy_sgd_nesterov_ema_step does, in torch (same order of operations as torch.optim.SGD / yolox ModelEMA); a
    flagged step with ``found_inf_ema`` still moves the EMA towards the unchanged parameters (ModelEMA.update)"""
    one_minus = 1.0 - ema_decay
    if hyper is not None:             # 1 - ema_decay is hyper[5] as the host wrote it, not recomputed from hyper[4]
        lr, momentum, weight_decay, inv_scale, ema_decay, one_minus = (float(v) for v in hyper[:6])
    if found_inf is not None and float(found_inf) != 0.0:
        if found_inf_ema and ema is not None:
            ema.mul_(ema_decay).add_(one_minus * param)
        return
    p = param[:n_param]
    g = grad[:n_param] * inv_scale if inv_scale != 1.0 else grad[:n_param].clone()
    g[decay_begin:] = g[decay_begin:].add(p[decay_begin:], alpha=weight_decay)
    momentum_buf.mul_(momentum).add_(g)
    g = g.add(momentum_buf, alpha=momentum) if nesterov else momentum_buf
    p.add_(g, alpha=-lr)
    if ema is not None:
        ema.mul_(ema_decay).add_(one_minus * param)


def nonfinite_flag(x, flag, count):
    flag.fill_(float(not bool(torch.isfinite(x).all())))
    count.add_(flag.to(torch.int32))


def resize_bilinear(x, size, out=None):
    y = F.interpolate(x, size=size, mode="bilinear", align_corners=False)
    if out is None:
        return y
    _require(tuple(out.shape) == tuple(y.shape) and out.dtype == torch.float32 and out.is_contiguous(),
             "resize_bilinear: bad out")
    return out.copy_(y)


def scale_labels_(labels, sx, sy):
    labels[..., 1::2] = labels[..., 1::2] * sx
    labels[..., 2::2] = labels[..., 2::2] * sy
    return labels


class PackBatch:
    """what ops.PackBatch does, with the torch pack emulations (destinations are filled in place)"""

    def __init__(self, device):
        self.items = []

    def add(self, w, out, mode, out_pitch=0, co_offset=0):
        self.items.append((w, out, mode, out_pitch, co_offset))

    def run(self):
        for w, out, mode, pitch, co in self.items:
            if mode == 2:
                out.copy_(pack_stem_weight(w))
            elif mode == 0:
                out.copy_(pack_conv_weight(w))
            else:
                out[:, :, co:co + w.shape[0]].copy_(pack_conv_weight_dgrad(w))


def letterbox_sized(src, sizes, out):
    """the streaming driver's preproc of each frame.  Deliberately narrower than the library: only rows whose
    destination fills ``out`` (the library puts a smaller one top-left on a canvas of 114)"""
    from oracle import input_oracle
    for i, (h, w, dh, dw) in enumerate(sizes.tolist()):
        assert (dh, dw) == tuple(out.shape[2:]), "emulated for destinations that fill out only"
        out[i] = torch.from_numpy(input_oracle.stream_frame(src[i, :h, :w].numpy(), (dh, dw))[0])


def stream_gate(status, flags, start, keep):
    ok = torch.ones_like(flags) if status is None else (status == 0).to(torch.int32)
    start.copy_(ok * (flags != 0).to(torch.int32))
    keep.copy_(ok)


def stream_rescale(det, count, status, ratio):
    for i in range(det.shape[0]):
        if status is not None and int(status[i]) != 0:
            count[i] = 0
        else:
            det[i, :int(count[i]), :4] /= ratio[i]


def select_images(srcs, dsts, flags):
    _require(1 <= len(srcs) == len(dsts) <= 3, "select_images: 1 to 3 (src, dst) view pairs")
    for s, d in zip(srcs, dsts):
        for i in range(s.n):
            if int(flags[i]):
                d.torch()[i].copy_(s.torch()[i])


def postprocess_nms(pred, num_classes, conf_thre, nms_thre, class_agnostic=False, max_det=None):
    """what sy_postprocess_nms writes, from the NMS oracle; rows past count[i] are zero here and unspecified there"""
    from oracle.postprocess_oracle import postprocess_oracle
    b, a, _ = pred.shape
    max_det = a if max_det is None else max_det
    det = torch.zeros((b, max_det, 7))
    count = torch.zeros((b,), dtype=torch.int32)
    for i, d in enumerate(postprocess_oracle(pred, num_classes, conf_thre, nms_thre, class_agnostic)):
        if d is not None:
            d = d[:max_det]
            det[i, :len(d)] = d
            count[i] = len(d)
    return det, count


NAMES = ["conv_stat_rows", "conv2d", "bn_act_apply", "focus_pack", "upsample_nearest", "spp_maxpool", "copy",
         "head_pred_decode", "tal_loss_workspace_bytes", "tal_loss", "tal_loss_backward", "head_pred_backward",
         "head_pred_backward_wide", "bn_act_backward", "conv2d_wgrad", "dilate2", "upsample_nearest_backward",
         "spp_maxpool_backward", "add_", "pack_conv_weight", "pack_conv_weight_dgrad", "pack_stem_weight",
         "sgd_nesterov_ema_step", "nonfinite_flag", "resize_bilinear", "scale_labels_", "pack_dw_weight",
         "stats_num_partials", "channel_stats", "bn_finalize", "PackBatch", "letterbox_sized", "stream_gate",
         "stream_rescale", "select_images", "postprocess_nms"]


def _view_init(self, buf, c0=0, c=None, n0=0, n=None):
    assert buf.dim() == 4 and buf.is_contiguous()
    self.buf, self.c0, self.n0, self.off = buf, c0, n0, 0
    self.c = buf.shape[3] - c0 if c is None else c
    self.n = buf.shape[0] - n0 if n is None else n


def _pk(t, dtype):
    return _bf(t) if dtype == torch.bfloat16 or EXACT else t.to(dtype)


def pack_conv_weight(*ws, dtype=torch.bfloat16):
    """what sy_pack_conv_weight (mode 0) writes: [sum O][kh*kw][I] in the emulated storage type"""
    return torch.cat([_pk(w.detach().permute(0, 2, 3, 1).reshape(w.shape[0], w.shape[2] * w.shape[3], w.shape[1]), dtype)
                      for w in ws], 0).contiguous()


def pack_conv_weight_dgrad(*ws):
    """mode 1: the forward layout of the flipped, channel-transposed filter, pairs concatenated along co"""
    w = torch.cat([x.detach() for x in ws], 0)
    return pack_conv_weight(w.flip(2, 3).transpose(0, 1).contiguous())


def pack_dw_weight(w, dtype=torch.bfloat16):
    c, _, kh, kw = w.shape
    return _pk(w.detach().reshape(c, kh * kw).t(), dtype).contiguous()


def stats_num_partials(n, hw):
    return n


def channel_stats(x, partials):
    """one partial row per image (stats_num_partials: image-major rows, the same number per image, as the library)"""
    _require(partials.shape[0] >= stats_num_partials(x.n, x.h * x.w), "channel_stats: too few partial rows")
    t = _nchw(x)
    partials[:x.n, 0] = t.sum((2, 3))
    partials[:x.n, 1] = t.pow(2).sum((2, 3))


def bn_finalize(partials, p_split, groups, count, gamma, beta, rmean, rvar, nbt, momentum, eps, scale, shift):
    """group 0 = partial rows [0, p_split), group 1 = the rest; ``count`` is the pixel count of EACH group"""
    _require(groups in (1, 2), f"bn_finalize: groups={groups}")
    _require(partials.shape[0] > 0 and count > 0 and gamma.numel() > 0, "bn_finalize: empty input")
    _require(groups == 1 or 0 < p_split < partials.shape[0], f"bn_finalize: p_split={p_split} of {partials.shape[0]}")
    for gi in range(groups):
        rows = partials[:p_split] if (gi == 0 and groups == 2) else (partials[p_split:] if groups == 2 else partials)
        s1, s2 = rows[:, 0].sum(0), rows[:, 1].sum(0)
        cnt = count
        mean = s1 / cnt
        var = (s2 / cnt - mean * mean).clamp_min(0)
        sc = gamma.detach().float() * (var + eps).rsqrt()
        scale[gi] = sc
        shift[gi] = beta.detach().float() - mean * sc
        if rmean is not None:
            rmean.mul_(1 - momentum).add_(momentum * mean)
            rvar.mul_(1 - momentum).add_(momentum * var * (cnt / max(cnt - 1, 1)))
        if nbt is not None:
            nbt.add_(1)
    PTRS[scale.data_ptr()] = scale
    PTRS[shift.data_ptr()] = shift


def pack_stem_weight(w, dtype=torch.bfloat16):
    """mode 2"""
    o = w.shape[0]
    p = torch.zeros((o, 3, 4, 16), dtype=torch.float32)
    p[:, :, :3, :12] = w.detach().permute(0, 2, 3, 1).float()
    return _pk(p.reshape(o, 3, 64), dtype).contiguous()


def install(monkeypatch, exact=False):
    g = globals()
    for n in NAMES:
        monkeypatch.setattr(ops, n, g[n])
    monkeypatch.setitem(g, "EXACT", exact)
    if exact:
        monkeypatch.setattr(View, "__init__", _view_init)
        monkeypatch.setattr(View, "empty", staticmethod(lambda n, h, w, c, device: View(torch.empty((n, h, w, c), dtype=torch.float32,
                                                                                               device=device))))
        from streamyolo_b200.model import engine

        def as_view_f32(t):
            if isinstance(t, View):
                return t
            p = t.permute(0, 2, 3, 1)
            return View(p if p.is_contiguous() else p.contiguous())

        monkeypatch.setattr(engine, "as_view", as_view_f32)
    PTRS.clear()
    LOSS_STATE.clear()
