"""YOLOX wrapper (mirror of /root/reference/exps/model/yolox.py:11-55)."""
import torch
import torch.nn as nn

from .dfp_pafpn import DFPPAFPN
from .tal_head import TALHead


class YOLOX(nn.Module):
    def __init__(self, backbone=None, head=None):
        super().__init__()
        self.backbone = DFPPAFPN() if backbone is None else backbone
        self.head = TALHead(20) if head is None else head
        # training forward with gradients enabled returns a loss that carries a grad_fn (model/backward.py), so the reference
        # trainer's scaler.scale(loss).backward() works unchanged; False = always the plain (no-gradient) forward
        self.train_with_autograd = True

    @property
    def activation_dtype(self):
        """Storage of every activation and conv operand: torch.bfloat16 (default), or torch.float16 for the eval and
        on_pipe forwards (11 significant bits instead of 8, like the reference's half-precision inference; head outputs stay
        fp32, the on_pipe buffers are fp16).  Setting it sets the backbone's and the head's.  Training runs bf16 only:
        a train-mode forward with fp16 raises NotImplementedError.  ``model.half()`` does not change it."""
        return getattr(self.backbone, "activation_dtype", torch.bfloat16)

    @activation_dtype.setter
    def activation_dtype(self, dtype):
        from . import engine
        engine.check_activation_dtype(dtype)
        self.backbone.activation_dtype = dtype
        self.head.activation_dtype = dtype

    def forward(self, x, targets=None, buffer=None, mode="off_pipe"):
        from . import engine
        with engine.forward_scope(x.device):       # one grid-barrier counter pool rewind for backbone + head
            return self._forward(x, targets, buffer, mode)

    def _forward(self, x, targets=None, buffer=None, mode="off_pipe"):
        assert mode in ["off_pipe", "on_pipe"]
        if self.training and self.activation_dtype != torch.bfloat16:
            raise NotImplementedError("fp16 activation storage runs the eval / streaming forwards only (training stores bf16)")
        if mode == "off_pipe":
            if self.training and self.train_with_autograd and torch.is_grad_enabled():
                # /root/reference/exps/train_utils/double_trainer.py:108-116: outputs = model(inps, targets); loss.backward()
                from . import backward
                assert targets is not None
                return backward.loss_with_autograd(self, x, targets)
            fpn_outs = self.backbone(x, buffer=buffer, mode="off_pipe")
            if self.training:
                assert targets is not None
                loss, iou_loss, conf_loss, cls_loss, l1_loss, num_fg = self.head(fpn_outs, targets, x)
                return {"total_loss": loss, "iou_loss": iou_loss, "l1_loss": l1_loss, "conf_loss": conf_loss,
                        "cls_loss": cls_loss, "num_fg": num_fg}
            return self.head(fpn_outs)
        fpn_outs, buffer_ = self.backbone(x, buffer=buffer, mode="on_pipe")
        return self.head(fpn_outs), buffer_
