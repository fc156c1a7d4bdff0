"""CPU emulation of the ReLU / LeakyReLU activation codes (SY_ACT_RELU, SY_ACT_LRELU) -- TEST INFRASTRUCTURE ONLY.

``install(monkeypatch, exact)`` installs tests/emul_ops.py and then wraps, with the same contract, the three entry points
that take an activation code: ``conv2d`` (FUSED epilogue), ``bn_act_apply`` and ``bn_act_backward``.  Codes 0 / 1 pass
straight through to what was installed before (tests/emul_ops.py, or a wrapper a test put on top of it); codes 2 / 3 run
the same arithmetic here with the activation and its derivative (autograd's convention at z = 0: 0 for ReLU, 0.1 for
LeakyReLU)."""
import torch
import torch.nn.functional as F

import emul_ops
from streamyolo_b200 import ops

KINKS = (ops.SY_ACT_RELU, ops.SY_ACT_LRELU)


def act_fn(t, code):
    return F.relu(t) if code == ops.SY_ACT_RELU else F.leaky_relu(t, 0.1)


def dact(z, code):
    if code == ops.SY_ACT_RELU:
        return (z > 0).to(z.dtype)
    return torch.where(z > 0, torch.ones_like(z), torch.full_like(z, 0.1))


def install(monkeypatch, exact=True):
    emul_ops.install(monkeypatch, exact=exact)
    wrap(monkeypatch)


def wrap(monkeypatch):
    """wrap whatever ops.conv2d / bn_act_apply / bn_act_backward are installed now"""
    base_conv, base_apply, base_bwd = ops.conv2d, ops.bn_act_apply, ops.bn_act_backward

    def conv2d(x, wpk, y, k, s, mode, impl="tc", scale=None, shift=None, act=1, res=None, **kw):
        if mode != ops.SY_CONV_FUSED or act not in KINKS:
            return base_conv(x, wpk, y, k, s, mode, impl=impl, scale=scale, shift=shift, act=act, res=res, **kw)
        kh, kw_ = (k, k) if isinstance(k, int) else k
        pad = ((kh - 1) // 2, (kw_ - 1) // 2)
        if impl == "dw":
            c = wpk.shape[1]
            out = F.conv2d(emul_ops._nchw(x), wpk.float().t().reshape(c, 1, kh, kw_), None, s, pad, groups=c)
        else:
            out = F.conv2d(emul_ops._nchw(x), emul_ops._unpack(wpk, kh, kw_), None, s, pad)
        if scale is not None:
            out = out * scale.float()[None, :, None, None] + shift.float()[None, :, None, None]
        out = act_fn(out, act)
        if res is not None:
            out = out + emul_ops._nchw(res)
        emul_ops._store(y, out)
        return 0

    def bn_act_apply(x, scale_ptr, shift_ptr, split_n, act, res, y, y_goff1=0, res_goff1=0):
        if act not in KINKS:
            return base_apply(x, scale_ptr, shift_ptr, split_n, act, res, y, y_goff1, res_goff1)
        scale, shift = ((scale_ptr, shift_ptr) if torch.is_tensor(scale_ptr)
                        else (emul_ops.PTRS[scale_ptr], emul_ops.PTRS[shift_ptr]))
        scale, shift = scale.reshape(-1, x.c), shift.reshape(-1, x.c)
        t = emul_ops._nchw(x)
        n = t.shape[0]
        sp = min(max(split_n, 0), n)          # group 1 = the images >= split_n, as sy_bn_act_apply
        outs = []
        for gi, (a, b, yo, ro) in enumerate([(0, sp, 0, 0), (sp, n, y_goff1, res_goff1)]):
            if a >= b:
                continue
            out = act_fn(t[a:b] * scale[gi][None, :, None, None] + shift[gi][None, :, None, None], act)
            if res is not None:
                out = out + emul_ops._strided(res, a, b - a, ro).permute(0, 3, 1, 2).float()
            outs.append((a, b, yo, out))
        for a, b, yo, out in outs:           # every residual is read before any output is written (in-place residuals)
            emul_ops._strided(y, a, b - a, yo).copy_(out.permute(0, 2, 3, 1))

    def bn_act_backward(raw, dy, draw, scale, shift, mean, invstd, split_n, act, dgamma, dbeta, accumulate=False):
        if act not in KINKS:
            return base_bwd(raw, dy, draw, scale, shift, mean, invstd, split_n, act, dgamma, dbeta, accumulate=accumulate)
        r, d = emul_ops._nchw(raw), emul_ops._nchw(dy)
        n = r.shape[0]
        sp = split_n if 0 < split_n < n else n
        out = torch.empty_like(r)
        dg, db = torch.zeros_like(dgamma), torch.zeros_like(dbeta)
        for gi, (a, b) in enumerate([(0, sp), (sp, n)] if sp < n else [(0, n)]):
            sc, sh, mu, iv = (t[gi][None, :, None, None] for t in (scale, shift, mean, invstd))
            z = r[a:b] * sc + sh
            dz = d[a:b] * dact(z, act)
            xh = (r[a:b] - mu) * iv
            m1, m2 = dz.mean((0, 2, 3), keepdim=True), (dz * xh).mean((0, 2, 3), keepdim=True)
            out[a:b] = sc * (dz - m1 - xh * m2)
            db += dz.sum((0, 2, 3))
            dg += (dz * xh).sum((0, 2, 3))
        emul_ops._store(draw, out)
        dgamma.copy_(dgamma + dg if accumulate else dg)
        dbeta.copy_(dbeta + db if accumulate else db)

    monkeypatch.setattr(ops, "conv2d", conv2d)
    monkeypatch.setattr(ops, "bn_act_apply", bn_act_apply)
    monkeypatch.setattr(ops, "bn_act_backward", bn_act_backward)
