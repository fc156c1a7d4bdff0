"""CPU ORACLE -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.

Only ``tests/``, ``__graft_entry__.smoke()`` and the ``cpu_baseline`` / ``--impl
reference`` legs of ``bench.py`` may import this module; the product path
(``streamyolo_b200``) never does and fails loudly when its CUDA library is missing.

What it is: a functional (state_dict in, tensors out) fp32 PyTorch restatement of
the StreamYOLO hot path -- CSPDarknet + PAFPN on both frames, DFP fusion,
decoupled head, SimOTA assignment and the Trend-Aware loss -- following

    /root/reference/exps/model/yolox.py      (YOLOX.forward            :28-55)
    /root/reference/exps/model/darknet.py    (CSPDarknet               :97-179)
    /root/reference/exps/model/dfp_pafpn.py  (off_forward / online     :109-228)
    /root/reference/exps/model/tal_head.py   (TALHead                  :152-712)

and the nine yolox==0.3.0 symbols those files import (third-party, pinned at
/root/reference/README.md:67, NOT vendored: SURVEY.md section 8c.1).

Parity pinning: the reference ships no tests or golden vectors ("parity unpinned by
the reference").  This restatement is pinned instead against OUTPUTS OF THE REFERENCE
ITSELF: ``oracle/make_golden.py`` imports the unmodified reference model files (on top
of the yolox shim in ``oracle/ref_shim``) in the build container and writes
``tests/golden/*.npz``; ``tests/test_oracle_golden.py`` checks this file against them.
The shim's nine symbols are restated from the published yolox 0.3.0 sources by memory;
that residual is stated in DESIGN.md.

Storage-precision hook: ``q`` (default identity) is applied exactly where the CUDA
product rounds a tensor to its HBM storage type (bf16): input pixels, conv weights, the
raw conv output in train mode, and every activation after BN+SiLU(+residual).  With
``q=identity`` this is the fp32 reference semantics; with ``q=bf16 round-trip`` it is
the same arithmetic "executed at the product's activation precision" (SURVEY.md 7-H).
"""
import math
from dataclasses import dataclass, field

import torch
import torch.nn.functional as F


@dataclass
class OracleCfg:
    depth: float = 0.33
    width: float = 0.50
    num_classes: int = 8
    gamma: float = 1.0          # cfgs/s_s50_onex_dfp_tal_flip.py:49-50
    ignore_thr: float = 0.5
    ignore_value: float = 1.5
    bn_eps: float = 1e-3        # cfgs/*.py:40-44 (init_yolo)
    bn_momentum: float = 0.03
    strides: tuple = (8, 16, 32)
    in_channels: tuple = (256, 512, 1024)


def bf16_round(t: torch.Tensor) -> torch.Tensor:
    return t.to(torch.bfloat16).to(torch.float32)


def _identity(t):
    return t


class StreamYoloOracle:
    """Functional model: ``state`` is a dict with the reference's state_dict keys."""

    def __init__(self, cfg: OracleCfg, state: dict, q=None):
        self.cfg = cfg
        self.P = {k: v.clone() for k, v in state.items()}
        self.q = q or _identity
        self.training = True
        self.use_l1 = True          # double_trainer.py:209-216 (always on in the shipped schedule)
        self.decode_in_inference = True
        self.bd = max(round(cfg.depth * 3), 1)       # darknet.py:112
        self.fd = round(3 * cfg.depth)               # dfp_pafpn.py:39
        self.hw = None
        self.trace = None           # optional dict name -> tensor (block-boundary dumps)

    # ------------------------------------------------------------------ blocks
    def _note(self, name, t):
        if self.trace is not None:
            self.trace[name] = t.detach().clone()

    def base_conv(self, pfx, x, k, stride, res=None, round_out=True):
        """yolox BaseConv = SiLU(BN(Conv2d(bias=False, pad=(k-1)//2))) [+ residual]."""
        P, q, c = self.P, self.q, self.cfg
        self._note(pfx + ".in", x)
        if res is not None:
            self._note(pfx + ".res", res)
        y = F.conv2d(x, q(P[pfx + ".conv.weight"]), None, stride, (k - 1) // 2)
        g, b = P[pfx + ".bn.weight"], P[pfx + ".bn.bias"]
        if self.training:
            y = q(y)
            n = y.numel() // y.shape[1]
            mean = y.mean((0, 2, 3))
            var = y.var((0, 2, 3), unbiased=False)
            m = c.bn_momentum
            P[pfx + ".bn.running_mean"].mul_(1 - m).add_(m * mean)
            P[pfx + ".bn.running_var"].mul_(1 - m).add_(m * var * (n / max(n - 1, 1)))
            P[pfx + ".bn.num_batches_tracked"] += 1
        else:
            mean, var = P[pfx + ".bn.running_mean"], P[pfx + ".bn.running_var"]
        scale = g * torch.rsqrt(var + c.bn_eps)
        shift = b - mean * scale
        y = F.silu(y * scale[None, :, None, None] + shift[None, :, None, None])
        self._note(pfx, y)                    # what a forward hook on the BaseConv sees
        if res is not None:
            y = y + res
        if round_out:
            y = q(y)
        self._note(pfx + ".out", y)           # the tensor the product stores
        return y

    def csp(self, pfx, x, n, shortcut):
        """yolox CSPLayer: conv3(cat(m(conv1 x), conv2 x)); Bottleneck expansion 1.0."""
        a = self.base_conv(pfx + ".conv1", x, 1, 1)
        b = self.base_conv(pfx + ".conv2", x, 1, 1)
        for i in range(n):
            h = self.base_conv(f"{pfx}.m.{i}.conv1", a, 1, 1)
            a = self.base_conv(f"{pfx}.m.{i}.conv2", h, 3, 1, res=a if shortcut else None)
        return self.base_conv(pfx + ".conv3", torch.cat([a, b], 1), 1, 1)

    def focus(self, pfx, x):
        """yolox Focus: slices in TL, BL, TR, BR order, then BaseConv 3x3."""
        p = torch.cat([x[..., ::2, ::2], x[..., 1::2, ::2], x[..., ::2, 1::2], x[..., 1::2, 1::2]], 1)
        return self.base_conv(pfx + ".conv", p, 3, 1)

    def spp(self, pfx, x):
        x = self.base_conv(pfx + ".conv1", x, 1, 1)
        pools = [F.max_pool2d(x, k, 1, k // 2) for k in (5, 9, 13)]
        return self.base_conv(pfx + ".conv2", torch.cat([x] + pools, 1), 1, 1)

    # ---------------------------------------------------------------- backbone
    def cspdarknet(self, x):
        """darknet.py:167-179 -> (dark3, dark4, dark5)."""
        bb, bd = "backbone.backbone.", self.bd
        x = self.focus(bb + "stem", x)
        x = self.base_conv(bb + "dark2.0", x, 3, 2)
        x = self.csp(bb + "dark2.1", x, bd, True)
        x = self.base_conv(bb + "dark3.0", x, 3, 2)
        d3 = self.csp(bb + "dark3.1", x, bd * 3, True)
        x = self.base_conv(bb + "dark4.0", d3, 3, 2)
        d4 = self.csp(bb + "dark4.1", x, bd * 3, True)
        x = self.base_conv(bb + "dark5.0", d4, 3, 2)
        x = self.spp(bb + "dark5.1", x)
        d5 = self.csp(bb + "dark5.2", x, bd, False)
        return d3, d4, d5

    def pafpn(self, x3):
        """One frame through backbone + PAFPN (dfp_pafpn.py:120-140), un-fused outputs."""
        fd, b = self.fd, "backbone."
        x2, x1, x0 = self.cspdarknet(x3)
        fpn0 = self.base_conv(b + "lateral_conv0", x0, 1, 1)
        f0 = torch.cat([F.interpolate(fpn0, size=x1.shape[2:4], mode="nearest"), x1], 1)
        f0 = self.csp(b + "C3_p4", f0, fd, False)
        fpn1 = self.base_conv(b + "reduce_conv1", f0, 1, 1)
        f1 = torch.cat([F.interpolate(fpn1, size=x2.shape[2:4], mode="nearest"), x2], 1)
        pan2 = self.csp(b + "C3_p3", f1, fd, False)
        p1 = torch.cat([self.base_conv(b + "bu_conv2", pan2, 3, 2), fpn1], 1)
        pan1 = self.csp(b + "C3_n3", p1, fd, False)
        p0 = torch.cat([self.base_conv(b + "bu_conv1", pan1, 3, 2), fpn0], 1)
        pan0 = self.csp(b + "C3_n4", p0, fd, False)
        return pan2, pan1, pan0

    def backbone_off(self, x6):
        """dfp_pafpn.py:109-175 (3-channel input is duplicated, :236-238)."""
        x6 = self.q(x6)
        if x6.shape[1] == 3:
            x6 = torch.cat([x6, x6], 1)
        cur = self.pafpn(x6[:, 0:3])
        sup = self.pafpn(x6[:, 3:6])
        return self._fuse(cur, sup)

    def backbone_on(self, x3, buffer=None):
        """dfp_pafpn.py:177-228: one pass, fuse with the buffered previous frame."""
        cur = self.pafpn(self.q(x3))
        sup = cur if buffer is None else buffer
        return self._fuse(cur, sup), cur

    def _fuse(self, cur, sup):
        outs = []
        for name, c, s in zip(("jian2", "jian1", "jian0"), cur, sup):
            pfx = "backbone." + name
            jc = self._jian(pfx, c)
            js = self._jian(pfx, s)
            y = self.q(torch.cat([jc, js], 1) + c)
            self._note(pfx + ".fused", y)
            outs.append(y)
        return tuple(outs)

    def _jian(self, pfx, x):
        """jianN BaseConv 1x1 (dfp_pafpn.py:83-105); its activated output is not rounded on
        its own: the product adds the residual in fp32 and rounds the sum once."""
        return self.base_conv(pfx, x, 1, 1, round_out=False)

    # -------------------------------------------------------------------- head
    def head_levels(self, feats):
        """tal_head.py:159-171: per level raw [B, 13, H, W] in (reg4, obj1, cls8) order."""
        outs = []
        P = self.P
        for k, x in enumerate(feats):
            x = self.base_conv(f"head.stems.{k}", x, 1, 1)
            cf = self.base_conv(f"head.cls_convs.{k}.0", x, 3, 1)
            cf = self.base_conv(f"head.cls_convs.{k}.1", cf, 3, 1)
            rf = self.base_conv(f"head.reg_convs.{k}.0", x, 3, 1)
            rf = self.base_conv(f"head.reg_convs.{k}.1", rf, 3, 1)
            cls = F.conv2d(cf, P[f"head.cls_preds.{k}.weight"], P[f"head.cls_preds.{k}.bias"])
            reg = F.conv2d(rf, P[f"head.reg_preds.{k}.weight"], P[f"head.reg_preds.{k}.bias"])
            obj = F.conv2d(rf, P[f"head.obj_preds.{k}.weight"], P[f"head.obj_preds.{k}.bias"])
            outs.append(torch.cat([reg, obj, cls], 1))
        return outs

    @staticmethod
    def grids(hw_list, strides):
        """Integer anchor grid (tal_head.py:232-233,248-253): x then y, level-major."""
        xs, ys, ss = [], [], []
        for (h, w), s in zip(hw_list, strides):
            yv, xv = torch.meshgrid(torch.arange(h), torch.arange(w), indexing="ij")
            xs.append(xv.reshape(-1))
            ys.append(yv.reshape(-1))
            ss.append(torch.full((h * w,), s))
        return torch.cat(xs), torch.cat(ys), torch.cat(ss)

    def flatten_decode(self, levels, sigmoid):
        """-> outputs [B, A, 13] decoded, origin_preds [B, A, 4] raw reg (tal_head.py:225-260)."""
        B = levels[0].shape[0]
        self.hw = [tuple(l.shape[-2:]) for l in levels]
        flat = torch.cat([l.flatten(2) for l in levels], 2).permute(0, 2, 1).contiguous()
        gx, gy, gs = self.grids(self.hw, self.cfg.strides)
        gx, gy, gs = gx.float(), gy.float(), gs.float()
        origin = flat[..., :4].clone()
        out = flat.clone()
        if sigmoid:
            out[..., 4:] = out[..., 4:].sigmoid()
        out[..., 0] = (flat[..., 0] + gx) * gs
        out[..., 1] = (flat[..., 1] + gy) * gs
        out[..., 2] = torch.exp(flat[..., 2]) * gs
        out[..., 3] = torch.exp(flat[..., 3]) * gs
        return out, origin, (gx, gy, gs)

    # --------------------------------------------------------------- top level
    def forward(self, x, targets=None, buffer=None, mode="off_pipe"):
        """Mirror of YOLOX.forward (yolox.py:28-55)."""
        assert mode in ("off_pipe", "on_pipe")
        if mode == "off_pipe":
            feats = self.backbone_off(x)
            levels = self.head_levels(feats)
            if self.training:
                assert targets is not None
                outputs, origin, grid = self.flatten_decode(levels, sigmoid=False)
                return self.losses(outputs, origin, grid, targets)
            return self._eval_out(levels)
        feats, buf = self.backbone_on(x, buffer)
        return self._eval_out(self.head_levels(feats)), buf

    def _eval_out(self, levels):
        if self.decode_in_inference:
            return self.flatten_decode(levels, sigmoid=True)[0]
        self.hw = [tuple(l.shape[-2:]) for l in levels]
        flat = torch.cat([l.flatten(2) for l in levels], 2).permute(0, 2, 1).contiguous()
        flat[..., 4:] = flat[..., 4:].sigmoid()
        return flat

    # ---------------------------------------------------------- SimOTA + loss
    @staticmethod
    def pairwise_iou_cxcywh(a, b):
        """yolox bboxes_iou(xyxy=False): no epsilon in the union."""
        tl = torch.max(a[:, None, :2] - a[:, None, 2:] / 2, b[None, :, :2] - b[None, :, 2:] / 2)
        br = torch.min(a[:, None, :2] + a[:, None, 2:] / 2, b[None, :, :2] + b[None, :, 2:] / 2)
        en = (tl < br).all(2).float()
        inter = (br - tl).prod(2) * en
        return inter / (a[:, 2:].prod(1)[:, None] + b[:, 2:].prod(1)[None, :] - inter)

    @staticmethod
    def candidates(gt, gx, gy, gs):
        """get_in_boxes_info (tal_head.py:594-677) on ALL anchors:
        returns in_box[G,A], in_ctr[G,A] (strict > 0 tests, radius 2.5 strides)."""
        xc = (gx * gs + 0.5 * gs)[None, :]
        yc = (gy * gs + 0.5 * gs)[None, :]
        l = (gt[:, 0] - 0.5 * gt[:, 2])[:, None]
        r = (gt[:, 0] + 0.5 * gt[:, 2])[:, None]
        t = (gt[:, 1] - 0.5 * gt[:, 3])[:, None]
        b = (gt[:, 1] + 0.5 * gt[:, 3])[:, None]
        in_box = torch.stack([xc - l, yc - t, r - xc, b - yc], 2).min(2).values > 0.0
        rad = 2.5 * gs[None, :]
        cl, cr = gt[:, 0:1] - rad, gt[:, 0:1] + rad
        ct, cb = gt[:, 1:2] - rad, gt[:, 1:2] + rad
        in_ctr = torch.stack([xc - cl, yc - ct, cr - xc, cb - yc], 2).min(2).values > 0.0
        return in_box, in_ctr

    def assign(self, gt, gt_cls, boxes, obj_logit, cls_logit, grid):
        """SimOTA for one image (tal_head.py:479-592, 679-712), expressed on the FULL anchor
        axis with non-candidates masked out (equivalent to the reference's compaction).
        Returns fg[A] bool, matched_gt[A] int64 (-1 where not fg), pred_iou[A] float."""
        gx, gy, gs = grid
        A, G = boxes.shape[0], gt.shape[0]
        in_box, in_ctr = self.candidates(gt, gx, gy, gs)
        cand = in_box.any(0) | in_ctr.any(0)
        both = in_box & in_ctr
        iou = self.pairwise_iou_cxcywh(gt, boxes)                       # [G, A]
        iou_cost = -torch.log(iou + 1e-8)
        p = (cls_logit.float().sigmoid() * obj_logit.float().sigmoid()[:, None]).sqrt()   # [A, C]
        onehot = F.one_hot(gt_cls.to(torch.int64), self.cfg.num_classes).float()          # [G, C]
        cls_cost = F.binary_cross_entropy(p[None].expand(G, A, -1), onehot[:, None].expand(-1, A, -1),
                                          reduction="none").sum(-1)
        cost = cls_cost + 3.0 * iou_cost + 100000.0 * (~both).float()
        inf = torch.tensor(float("inf"))
        cost_m = torch.where(cand[None], cost, inf)
        iou_m = torch.where(cand[None], iou, -inf)
        n_cand = int(cand.sum())
        kk = min(10, n_cand)
        topv = torch.topk(iou_m, kk, dim=1).values
        dyn_k = torch.clamp(topv.sum(1).int(), min=1)                   # [G]
        order = torch.argsort(cost_m, dim=1, stable=True)               # lowest cost first, low index on ties
        rank = torch.empty_like(order)
        rank.scatter_(1, order, torch.arange(A)[None].expand(G, -1))
        match = (rank < dyn_k[:, None]) & cand[None]                    # [G, A]
        multi = match.sum(0) > 1
        if multi.any():
            best = torch.argmin(torch.where(multi[None], cost, inf), dim=0)   # first minimum
            fix = F.one_hot(best, G).T.bool()
            match = torch.where(multi[None], fix, match)
        fg = match.any(0)
        matched = torch.where(fg, match.float().argmax(0), torch.full((A,), -1))
        pred_iou = (match.float() * iou).sum(0) * fg
        return fg, matched, pred_iou

    def tal_gt_iou(self, gt, sup_gt):
        """Per future-GT trend IoU (tal_head.py:394-403)."""
        if sup_gt.shape[0] == 0:
            return torch.ones(gt.shape[0])
        v = self.pairwise_iou_cxcywh(gt, sup_gt).max(1).values
        return torch.where(v < self.cfg.ignore_thr, torch.full_like(v, self.cfg.ignore_value), v)

    def losses(self, outputs, origin, grid, targets, return_aux=False, dtype=torch.float32):
        """get_losses (tal_head.py:262-470).  targets = (future[B,120,5], current[B,120,5]).  ``dtype``: precision of the
        labels, the TAL weights and the loss terms (outputs, origin and grid are expected in it).  The SimOTA assignment is
        a no-grad constant and always runs in fp32, so a float64 evaluation differentiates the fp32 assignment."""
        c = self.cfg
        fut, cur = targets[0][..., :5].to(dtype), targets[1][..., :5].to(dtype)
        B, A, _ = outputs.shape
        gx, gy, gs = grid
        grid32 = tuple(t.float() for t in grid)
        nl = (fut.sum(2) > 0).sum(1)
        sl = (cur.sum(2) > 0).sum(1)
        fg_all = torch.zeros(B, A, dtype=torch.bool)
        match_all = torch.full((B, A), -1, dtype=torch.int64)
        piou_all = torch.zeros(B, A)
        tiou_all = torch.zeros(B, A, dtype=dtype)
        num_gts = 0
        for b in range(B):
            G, Gs = int(nl[b]), int(sl[b])
            num_gts += G
            if G == 0:
                continue
            gt, gcls = fut[b, :G, 1:5], fut[b, :G, 0]
            with torch.no_grad():
                fg, m, pi = self.assign(gt.float(), gcls.float(), outputs[b, :, :4].detach().float(),
                                        outputs[b, :, 4].detach().float(), outputs[b, :, 5:].detach().float(), grid32)
            fg_all[b], match_all[b], piou_all[b] = fg, m, pi
            tio = self.tal_gt_iou(gt, cur[b, :Gs, 1:5])
            tiou_all[b] = torch.where(fg, tio[m.clamp(min=0)], torch.zeros(A, dtype=dtype))
        n_fg_raw = int(fg_all.sum())
        num_fg = max(n_fg_raw, 1)
        # gather foreground rows in (image, anchor) order like the reference's torch.cat
        bi, ai = fg_all.nonzero(as_tuple=True)
        gtm = match_all[bi, ai]
        reg_t = fut[bi, gtm, 1:5]
        cls_t = F.one_hot(fut[bi, gtm, 0].to(torch.int64), c.num_classes).to(dtype) * piou_all[bi, ai][:, None].to(dtype)
        s, xs, ys = gs[ai], gx[ai], gy[ai]
        l1_t = torch.stack([reg_t[:, 0] / s - xs, reg_t[:, 1] / s - ys,
                            torch.log(reg_t[:, 2] / s + 1e-8), torch.log(reg_t[:, 3] / s + 1e-8)], 1)
        w = 1.0 / (tiou_all[bi, ai] ** c.gamma + 1e-8)
        pb = outputs[bi, ai, :4]
        iou_l = self.iou_loss(pb, reg_t)
        iou_w = ((w * iou_l.sum()) / (w * iou_l).sum()).detach()
        l1_l = (origin[bi, ai] - l1_t).abs()
        w4 = w[:, None].expand(-1, 4)
        l1_w = ((w4 * l1_l.sum()) / (w4 * l1_l).sum()).detach()
        loss_iou = (iou_w * iou_l).sum() / num_fg
        loss_obj = F.binary_cross_entropy_with_logits(outputs[..., 4], fg_all.to(dtype), reduction="sum") / num_fg
        loss_cls = F.binary_cross_entropy_with_logits(outputs[bi, ai, 5:], cls_t, reduction="sum") / num_fg
        loss_l1 = (l1_w * l1_l).sum() / num_fg if self.use_l1 else torch.zeros((), dtype=dtype)
        total = 5.0 * loss_iou + loss_obj + loss_cls + loss_l1
        res = {"total_loss": total, "iou_loss": 5.0 * loss_iou, "l1_loss": loss_l1,
               "conf_loss": loss_obj, "cls_loss": loss_cls, "num_fg": num_fg / max(num_gts, 1)}
        if return_aux:
            res["aux"] = {"fg": fg_all, "matched": match_all, "pred_iou": piou_all, "tal_iou": tiou_all,
                          "iou_w": iou_w, "l1_w": l1_w, "num_fg_raw": n_fg_raw, "num_gts": num_gts}
        return res

    @staticmethod
    def iou_loss(pred, tgt):
        """yolox IOUloss(loss_type='iou'): 1 - IoU^2 with +1e-16 in the union."""
        tl = torch.max(pred[:, :2] - pred[:, 2:] / 2, tgt[:, :2] - tgt[:, 2:] / 2)
        br = torch.min(pred[:, :2] + pred[:, 2:] / 2, tgt[:, :2] + tgt[:, 2:] / 2)
        en = (tl < br).all(1).float()
        inter = (br - tl).prod(1) * en
        union = pred[:, 2:].prod(1) + tgt[:, 2:].prod(1) - inter
        iou = inter / (union + 1e-16)
        return 1 - iou ** 2


# ----------------------------------------------------------------- utilities
def model_shapes(depth: float, width: float, num_classes: int = 8) -> dict:
    """state_dict key -> shape for a StreamYOLO of the given scale, derived analytically
    from the constructors (darknet.py:98-165, dfp_pafpn.py:18-105, tal_head.py:55-131).
    Verified against the reference's real state_dict by tests/test_oracle_golden.py."""
    shapes = {}

    def bc(pfx, cin, cout, k):
        shapes[pfx + ".conv.weight"] = (cout, cin, k, k)
        for n in ("weight", "bias", "running_mean", "running_var"):
            shapes[f"{pfx}.bn.{n}"] = (cout,)
        shapes[pfx + ".bn.num_batches_tracked"] = ()

    def csp(pfx, cin, cout, n):
        mid = int(cout * 0.5)
        bc(pfx + ".conv1", cin, mid, 1)
        bc(pfx + ".conv2", cin, mid, 1)
        bc(pfx + ".conv3", 2 * mid, cout, 1)
        for i in range(n):
            bc(f"{pfx}.m.{i}.conv1", mid, mid, 1)
            bc(f"{pfx}.m.{i}.conv2", mid, mid, 3)

    base = int(width * 64)
    bd = max(round(depth * 3), 1)
    fd = round(3 * depth)
    bb = "backbone.backbone."
    bc(bb + "stem.conv", 12, base, 3)
    bc(bb + "dark2.0", base, base * 2, 3)
    csp(bb + "dark2.1", base * 2, base * 2, bd)
    bc(bb + "dark3.0", base * 2, base * 4, 3)
    csp(bb + "dark3.1", base * 4, base * 4, bd * 3)
    bc(bb + "dark4.0", base * 4, base * 8, 3)
    csp(bb + "dark4.1", base * 8, base * 8, bd * 3)
    bc(bb + "dark5.0", base * 8, base * 16, 3)
    bc(bb + "dark5.1.conv1", base * 16, base * 8, 1)
    bc(bb + "dark5.1.conv2", base * 32, base * 16, 1)
    csp(bb + "dark5.2", base * 16, base * 16, bd)
    c3, c4, c5 = int(256 * width), int(512 * width), int(1024 * width)
    b = "backbone."
    bc(b + "lateral_conv0", c5, c4, 1)
    csp(b + "C3_p4", 2 * c4, c4, fd)
    bc(b + "reduce_conv1", c4, c3, 1)
    csp(b + "C3_p3", 2 * c3, c3, fd)
    bc(b + "bu_conv2", c3, c3, 3)
    csp(b + "C3_n3", 2 * c3, c4, fd)
    bc(b + "bu_conv1", c4, c4, 3)
    csp(b + "C3_n4", 2 * c4, c5, fd)
    bc(b + "jian2", c3, c3 // 2, 1)
    bc(b + "jian1", c4, c4 // 2, 1)
    bc(b + "jian0", c5, c5 // 2, 1)
    hw = int(256 * width)
    for k, cin in enumerate((c3, c4, c5)):
        bc(f"head.stems.{k}", cin, hw, 1)
        for j in range(2):
            bc(f"head.cls_convs.{k}.{j}", hw, hw, 3)
            bc(f"head.reg_convs.{k}.{j}", hw, hw, 3)
        for name, n in (("cls_preds", num_classes), ("reg_preds", 4), ("obj_preds", 1)):
            shapes[f"head.{name}.{k}.weight"] = (n, hw, 1, 1)
            shapes[f"head.{name}.{k}.bias"] = (n,)
    return shapes


def conv_gflop_per_pair(depth, width, height=600, width_px=960, num_classes=8, on_pipe=False):
    """Algorithmic conv FLOPs (2*MAC) of one frame pair, no recompute (SURVEY.md section 8d)."""
    shapes = model_shapes(depth, width, num_classes)
    # spatial size of each conv's OUTPUT
    def hw_of(key):
        s2 = lambda v: (v - 1) // 2 + 1
        h2, w2 = height // 2, width_px // 2
        h4, w4 = s2(h2), s2(w2)
        h8, w8 = s2(h4), s2(w4)
        h16, w16 = s2(h8), s2(w8)
        h32, w32 = s2(h16), s2(w16)
        t = {"stem": (h2, w2), "dark2": (h4, w4), "dark3": (h8, w8), "dark4": (h16, w16), "dark5": (h32, w32),
             "lateral_conv0": (h32, w32), "C3_p4": (h16, w16), "reduce_conv1": (h16, w16), "C3_p3": (h8, w8),
             "bu_conv2": (h16, w16), "C3_n3": (h16, w16), "bu_conv1": (h32, w32), "C3_n4": (h32, w32),
             "jian2": (h8, w8), "jian1": (h16, w16), "jian0": (h32, w32)}
        parts = key.split(".")
        if parts[0] == "head":
            return [(h8, w8), (h16, w16), (h32, w32)][int(parts[2])]
        name = parts[2] if parts[1] == "backbone" else parts[1]
        return t[name]
    total = 0.0
    for k, s in shapes.items():
        if not k.endswith("weight") or ".bn." in k:
            continue
        h, w = hw_of(k)
        fl = 2.0 * s[0] * s[1] * s[2] * s[3] * h * w
        mult = 1 if k.startswith("head.") else (1 if on_pipe else 2)
        total += fl * mult
    return total / 1e9
