"""TALHead: decoupled YOLOX head + SimOTA + Trend-Aware Loss (mirror of
/root/reference/exps/model/tal_head.py).  Towers run on the wgmma conv kernel, the three
prediction convs + box decode are one kernel per level writing [B, A, 5+ncls] directly, and the
whole of get_losses/get_assignments/dynamic_k_matching is ``sy_tal_loss`` (no host sync)."""
import math

import torch
from torch import nn

from . import engine
from .. import ops
from .network_blocks import BaseConv, DWConv


MAX_NUM_CLASSES = 251     # sy_head_pred_decode: compiled instantiations for 8 / 1 / 20 classes, a generic kernel for any other count
                          # (the reference head takes num_classes freely, tal_head.py:27); the training backward takes the same
                          # counts: sy_head_pred_backward up to 27 classes, sy_head_pred_backward_wide above (model/backward.py)


class TALHead(nn.Module):
    def __init__(self, num_classes, width=1.0, strides=[8, 16, 32], in_channels=[256, 512, 1024], act="silu",
                 depthwise=False, gamma=1.5, ignore_thr=0.2, ignore_value=0.2):
        super().__init__()
        if not 1 <= num_classes <= MAX_NUM_CLASSES:
            raise NotImplementedError(f"num_classes={num_classes}: the head kernels take 1..{MAX_NUM_CLASSES} classes")
        self.gamma, self.ignore_thr, self.ignore_value = gamma, ignore_thr, ignore_value
        self.n_anchors = 1
        self.num_classes = num_classes
        self.decode_in_inference = True
        self.cls_convs, self.reg_convs = nn.ModuleList(), nn.ModuleList()
        self.cls_preds, self.reg_preds, self.obj_preds = nn.ModuleList(), nn.ModuleList(), nn.ModuleList()
        self.stems = nn.ModuleList()
        hw = int(256 * width)
        Conv = DWConv if depthwise else BaseConv            # tal_head.py:53
        for cin in in_channels:
            self.stems.append(BaseConv(int(cin * width), hw, 1, 1, act=act))
            self.cls_convs.append(nn.Sequential(Conv(hw, hw, 3, 1, act=act), Conv(hw, hw, 3, 1, act=act)))
            self.reg_convs.append(nn.Sequential(Conv(hw, hw, 3, 1, act=act), Conv(hw, hw, 3, 1, act=act)))
            self.cls_preds.append(nn.Conv2d(hw, self.n_anchors * num_classes, 1, 1, 0))
            self.reg_preds.append(nn.Conv2d(hw, 4, 1, 1, 0))
            self.obj_preds.append(nn.Conv2d(hw, self.n_anchors * 1, 1, 1, 0))
        self.use_l1 = False
        self.strides = strides
        self.hw = None
        self.last_assignment = None     # optional debug dumps (set ``keep_assignment = True``)
        self.keep_assignment = False
        self.activation_dtype = torch.bfloat16      # storage of the tower activations: bf16, or fp16 in eval mode (engine.Ctx)

    def initialize_biases(self, prior_prob):
        v = -math.log((1 - prior_prob) / prior_prob)
        for conv in list(self.cls_preds) + list(self.obj_preds):
            b = conv.bias.view(self.n_anchors, -1)
            b.data.fill_(v)
            conv.bias = torch.nn.Parameter(b.view(-1), requires_grad=True)

    # ------------------------------------------------------------------
    def forward(self, xin, labels=None, imgs=None):
        dt = engine.check_activation_dtype(self.activation_dtype)
        if dt != torch.bfloat16 and self.training:
            raise NotImplementedError("fp16 activation storage runs the eval / streaming forwards only (training stores bf16)")
        views = [engine.as_view(x, dt) if dt != torch.bfloat16 else engine.as_view(x) for x in xin]
        dev = views[0].buf.device
        b = views[0].n
        ctx = engine.Ctx(self.training, b, b, dev, dtype=dt)
        with torch.no_grad(), engine.forward_scope(dev):
            r = self.run(ctx, views, labels)
        return tuple(r) if self.training else r

    def run(self, ctx, views, labels=None):
        """The head on the per-level views: eval -> the [B, A, 5+ncls] outputs; train -> the loss vector [total, iou, conf,
        cls, l1, num_fg].  With a tape (the recording forward) the prediction / decode / loss launches are recorded as
        one ``head`` op."""
        dev = ctx.device
        b = views[0].n
        train = ctx.train
        self.hw = [(v.h, v.w) for v in views]
        a_total = sum(h * w for h, w in self.hw)
        no = 5 + self.num_classes
        out = torch.empty((b, a_total, no), dtype=torch.float32, device=dev)
        origin = torch.empty((b, a_total, 4), dtype=torch.float32, device=dev) if (train and self.use_l1) else None
        off = 0
        levels = []
        for k, v in enumerate(views):
            x = engine.base_conv(ctx, self.stems[k], v)
            # cls_convs[k][0] and reg_convs[k][0] read the same stem output (tal_head.py:159-171): ONE conv launch with
            # 2 x hw output channels and two BatchNorm segments, like the conv1 | conv2 pair of a CSPLayer
            u = engine.conv_pair(ctx, self.cls_convs[k][0], self.reg_convs[k][0], x)
            hw_c = u.c // 2
            cf = engine.base_conv(ctx, self.cls_convs[k][1], u.ch(0, hw_c))
            rf = engine.base_conv(ctx, self.reg_convs[k][1], u.ch(hw_c, hw_c))
            ops.head_pred_decode(cf, rf, _f32(self.reg_preds[k].weight), _f32(self.reg_preds[k].bias),
                                 _f32(self.obj_preds[k].weight), _f32(self.obj_preds[k].bias),
                                 _f32(self.cls_preds[k].weight), _f32(self.cls_preds[k].bias),
                                 self.strides[k], off, a_total, out, origin,
                                 sigmoid=not train, decode=train or self.decode_in_inference)
            levels.append((k, cf, rf, off))
            off += v.h * v.w
        if not train:
            return out
        loss, fut, ws = self._loss(out, origin, labels)
        ctx.rec(t="head", levels=levels, out=out, origin=origin, fut=fut, ws=ws, hw=self.hw, a_total=a_total)
        return loss

    def decode_outputs(self, outputs, dtype=None):
        """Decode raw [B, A, 5+ncls] outputs (tools/eval.py:188 path when decode_in_inference is False)."""
        gx, gy, gs = [], [], []
        for (h, w), s in zip(self.hw, self.strides):
            yv, xv = torch.meshgrid(torch.arange(h), torch.arange(w), indexing="ij")
            gx.append(xv.reshape(-1)), gy.append(yv.reshape(-1)), gs.append(torch.full((h * w,), s))
        gx, gy, gs = (torch.cat(t).to(outputs.device, outputs.dtype) for t in (gx, gy, gs))
        outputs[..., 0] = (outputs[..., 0] + gx) * gs
        outputs[..., 1] = (outputs[..., 1] + gy) * gs
        outputs[..., 2:4] = torch.exp(outputs[..., 2:4]) * gs[:, None]
        return outputs

    def _loss(self, outputs, origin, labels):
        """-> (loss vector, future labels, workspace): the last two are what the loss backward reads"""
        if not self.use_l1:
            # the reference dereferences origin_preds unconditionally (tal_head.py:435) and raises; every
            # shipped schedule sets use_l1 = True (double_trainer.py:209-216)
            raise AttributeError("TALHead.use_l1 must be True in training (reference tal_head.py:435)")
        dev = outputs.device
        fut = labels[0][..., :5].to(dev, torch.float32).contiguous()
        cur = labels[1][..., :5].to(dev, torch.float32).contiguous()
        b, a, no = outputs.shape
        wsb = ops.tal_loss_workspace_bytes(b, a, fut.shape[1], self.num_classes)
        ws = torch.empty((wsb + 255) // 256 * 256, dtype=torch.uint8, device=dev)
        loss = torch.empty(6, dtype=torch.float32, device=dev)
        dumps = {}
        if self.keep_assignment:
            dumps = dict(fg_out=torch.empty((b, a), dtype=torch.int32, device=dev),
                         matched_out=torch.empty((b, a), dtype=torch.int32, device=dev),
                         pred_iou_out=torch.empty((b, a), dtype=torch.float32, device=dev))
        ops.tal_loss(outputs, origin, fut, cur, self.hw, self.strides, float(self.gamma), float(self.ignore_thr),
                     float(self.ignore_value), self.use_l1, ws, loss, **dumps)
        if self.keep_assignment:
            self.last_assignment = dict(dumps, outputs=outputs, origin=origin)
        return loss, fut, ws


def _f32(p):
    """fp32 operand of a prediction conv: weight [O][C], bias [O]"""
    return p.detach().float().contiguous().view(p.shape[0], -1) if p.dim() > 1 else p.detach().float().contiguous()
