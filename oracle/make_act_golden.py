"""Generate tests/golden/tiny_{relu,lrelu}_120x160.npz and grad_tiny_{relu,lrelu}_120x160.npz FROM THE UNMODIFIED REFERENCE
(test infrastructure).  Runs only where /root/reference is mounted:

    python oracle/make_act_golden.py

The recipe of ``oracle/make_golden.py`` (``run_case``: losses, SimOTA assignment, BN statistics, per-BaseConv output
statistics, eval and on_pipe outputs; ``run_grad_case``: parameter gradient statistics and the prediction-conv gradients)
at the tiny configuration, with the reference model built with ``act="relu"`` / ``"lrelu"`` in its ``DFPPAFPN`` and
``TALHead`` constructors (every BaseConv's activation, [yolox] ``get_activation``).
"""
import os
import sys

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))

from oracle import make_golden  # noqa: E402  (also puts ref_shim and the reference on sys.path)
from streamyolo_b200 import synth  # noqa: E402

ACT_CASES = {"tiny_" + a + "_120x160": dict(make_golden.CASES["tiny_120x160"], act=a) for a in ("relu", "lrelu")}


def build_reference(act):
    """make_golden.build_reference with ``act`` passed to the reference's DFPPAFPN and TALHead"""
    def build(depth, width, gamma, thr, val, momentum=0.03):
        from exps.model.dfp_pafpn import DFPPAFPN
        from exps.model.tal_head import TALHead
        from exps.model.yolox import YOLOX
        ch = [256, 512, 1024]
        model = YOLOX(DFPPAFPN(depth, width, in_channels=ch, act=act),
                      TALHead(8, width, in_channels=ch, act=act, gamma=gamma, ignore_thr=thr, ignore_value=val))
        for m in model.modules():
            if isinstance(m, torch.nn.BatchNorm2d):
                m.eps, m.momentum = 1e-3, momentum
        model.head.initialize_biases(1e-2)
        shapes = {k: tuple(v.shape) for k, v in model.state_dict().items()}
        model.load_state_dict(synth.synth_state_dict(shapes), strict=True)
        model.head.use_l1 = True
        return model, shapes
    return build


if __name__ == "__main__":
    torch.set_num_threads(os.cpu_count())
    for name, c in ACT_CASES.items():
        make_golden.build_reference = build_reference(c["act"])
        make_golden.run_case(name, c)
        make_golden.run_grad_case(name, c)
