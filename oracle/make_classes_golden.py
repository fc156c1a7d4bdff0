"""Generate tests/golden/tiny_c80_120x160.npz and grad_tiny_c80_120x160.npz FROM THE UNMODIFIED REFERENCE (test
infrastructure).  Runs only where /root/reference is mounted:

    python oracle/make_classes_golden.py

The recipe of ``oracle/make_golden.py`` (``run_case``: losses, SimOTA assignment, BN statistics, per-BaseConv output
statistics, eval and on_pipe outputs; ``run_grad_case``: parameter gradient statistics and the prediction-conv gradients)
at the tiny configuration with the reference's ``TALHead(80, ...)`` -- COCO's class count -- and labels drawn from all
80 classes.  Both files also get ``still_*`` entries: the still-image baseline, the reference's
``YOLOX(DFPPAFPN, PIPEHead(80, ...))`` trained on single frames (``model(frames [B, 3, H, W], labels)``, which the
reference's DFPPAFPN duplicates into pairs, dfp_pafpn.py:236-238): losses, assignment, gradient statistics and the
prediction-conv gradients.
"""
import functools
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))

from oracle import make_golden  # noqa: E402  (also puts ref_shim and the reference on sys.path)
from streamyolo_b200 import synth  # noqa: E402

NUM_CLASSES = 80
NAME = "tiny_c80_120x160"
CASE = dict(make_golden.CASES["tiny_120x160"], num_classes=NUM_CLASSES)
GOLD = os.path.join(os.path.dirname(HERE), "tests", "golden")


def build_reference(head_cls):
    """make_golden.build_reference with ``head_cls(NUM_CLASSES, ...)`` as the head"""
    def build(depth, width, gamma, thr, val, momentum=0.03):
        from exps.model.dfp_pafpn import DFPPAFPN
        from exps.model.yolox import YOLOX
        ch = [256, 512, 1024]
        kw = dict(gamma=gamma, ignore_thr=thr, ignore_value=val) if head_cls.__name__ == "TALHead" else {}
        model = YOLOX(DFPPAFPN(depth, width, in_channels=ch), head_cls(NUM_CLASSES, width, in_channels=ch, **kw))
        for m in model.modules():
            if isinstance(m, torch.nn.BatchNorm2d):
                m.eps, m.momentum = 1e-3, momentum
        model.head.initialize_biases(1e-2)
        shapes = {k: tuple(v.shape) for k, v in model.state_dict().items()}
        model.load_state_dict(synth.synth_state_dict(shapes), strict=True)
        model.head.use_l1 = True
        return model, shapes
    return build


def still_case(c):
    """-> (forward entries, gradient entries) of the still model on the first frame of each synthetic pair"""
    from exps.model.pipe_head import PIPEHead
    torch.manual_seed(0)
    model, _ = build_reference(PIPEHead)(c["depth"], c["width"], c["gamma"], c["thr"], c["val"])
    x = synth.synth_frames(c["B"], c["H"], c["W"])[:, :3].contiguous()
    labels, _ = synth.synth_labels(c["B"], c["H"], c["W"], empty_image=c["empty"])
    rec = make_golden.capture_assignment(model)
    model.train()
    loss = model(x, labels)
    loss["total_loss"].backward()
    order = ["total_loss", "iou_loss", "l1_loss", "conf_loss", "cls_loss", "num_fg"]
    fwd = {"still_train_loss": np.array([float(loss[k]) for k in order], np.float64),
           "still_fg_image": np.concatenate([np.full(len(r[1]), r[0], np.int32) for r in rec]),
           "still_fg_anchor": np.concatenate([r[1] for r in rec]),
           "still_fg_gt": np.concatenate([r[2] for r in rec]),
           "still_fg_iou": np.concatenate([r[3] for r in rec])}
    grads = {k: p.grad for k, p in model.named_parameters() if p.grad is not None}
    grd = {"still_total_loss": np.array(float(loss["total_loss"]), np.float64),
           "still_grad_keys": np.array(list(grads)),
           "still_grad_stats": np.stack([make_golden.stat3(g) for g in grads.values()]),
           "still_grad_l2": np.array([float(g.norm()) for g in grads.values()], np.float64)}
    for k, g in grads.items():
        if k.startswith(("head.cls_preds", "head.reg_preds", "head.obj_preds")):
            grd["still_g:" + k] = g.numpy().astype(np.float32)
    return fwd, grd


def add_entries(path, extra):
    with np.load(path) as f:
        d = {k: f[k] for k in f.files}
    d.update(extra)
    np.savez_compressed(path, **d)
    print(path, os.path.getsize(path) // 1024, "KiB")


if __name__ == "__main__":
    torch.set_num_threads(os.cpu_count())
    from exps.model.tal_head import TALHead
    # labels over all 80 classes: make_golden's recipes draw them through synth.synth_labels
    synth.synth_labels = functools.partial(synth.synth_labels, num_classes=NUM_CLASSES)
    make_golden.build_reference = build_reference(TALHead)
    make_golden.run_case(NAME, CASE)
    make_golden.run_grad_case(NAME, CASE)
    fwd, grd = still_case(CASE)
    add_entries(os.path.join(GOLD, NAME + ".npz"), fwd)
    add_entries(os.path.join(GOLD, "grad_" + NAME + ".npz"), grd)
