"""CPU: the forward checker of tests/test_gpu_parity_fwd.py (FwdChecker) on the emulated kernels (tests/emul_ops.py, bf16
storage), on the tiny model: it accepts the four forwards bench.py times (train plain, the recording forward of a training
step -- pairs and still frames --, eval off_pipe, on_pipe) with the launch counts of the module tree, and it rejects each of
a set of mutants, emulated kernels made wrong in one way.  This shows that the checker can fail before any GPU time is
spent on it."""
import os
import sys
from collections import Counter

import pytest
import torch

from oracle.make_golden import CASES
from streamyolo_b200 import ops, synth
from streamyolo_b200.model import DFPPAFPN, PIPEHead, YOLOX, backward, engine

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import emul_ops  # noqa: E402
from test_cpu_backward import build_product  # noqa: E402
from test_gpu_parity_fwd import FwdChecker, conv_launches  # noqa: E402

C = CASES["tiny_120x160"]


def _model(momentum=0.03, still=False):
    if still:
        ch = [256, 512, 1024]
        m = YOLOX(DFPPAFPN(C["depth"], C["width"], in_channels=ch), PIPEHead(8, C["width"], in_channels=ch))
        m.load_state_dict(synth.synth_state_dict({k: tuple(v.shape) for k, v in m.state_dict().items()}), strict=True)
        m.head.use_l1 = True
        m.train()
    else:
        m = build_product(C)
    for mod in m.modules():
        if isinstance(mod, torch.nn.BatchNorm2d):
            mod.eps, mod.momentum = 1e-3, momentum
    engine.name_modules(m)
    return m


def _data():
    return synth.synth_frames(C["B"], C["H"], C["W"]), synth.synth_labels(C["B"], C["H"], C["W"])


# each forward: set up (build, warm up / calibrate) and return the checked forward, so that a mutant can be installed for
# the checked forward alone
def run_train():
    m = _model()
    x, tg = _data()
    with torch.no_grad():
        m(x, tg)

    def go():
        with torch.no_grad(), FwdChecker(m) as ck:
            m(x, tg)
        n = conv_launches(m, jian_twice=False)
        assert ck.n == Counter(conv=n, apply=n, head=3, focus=1), ck.n
        return ck
    return go


def run_recording(still=False):
    m = _model(still=still)
    x, tg = _data()
    if still:
        x, tg = x[:, :3].contiguous(), tg[0]
    with torch.no_grad():
        m(x, tg)

    def go():
        with FwdChecker(m) as ck:
            backward._record(m, x, tg)
        n = conv_launches(m, jian_twice=True)
        want = Counter(conv=n, apply=n, head=3, focus=1, mean_invstd=n)
        if still:
            want["stat_updates_2"] = n - 6 - 4 * len(m.head.strides)
        assert ck.n == want, ck.n
        return ck
    return go


def _calibrated():
    m = _model(momentum=1.0)
    x, tg = _data()
    with torch.no_grad():
        m(x, tg)
    return m.eval(), x


def run_eval():
    m, x = _calibrated()

    def go():
        with torch.no_grad(), FwdChecker(m, nondegenerate=True) as ck:
            m(x)
        assert ck.n == Counter(conv=conv_launches(m, jian_twice=True), head=3, focus=1), ck.n
        return ck
    return go


def run_on_pipe():
    m, x = _calibrated()
    n = conv_launches(m, jian_twice=True)

    def go():
        buf = None
        with torch.no_grad():
            for i in range(3):        # star call, buffer straight from the previous call, cloned buffer
                f = x[i % x.shape[0]:i % x.shape[0] + 1, 0:3]
                with FwdChecker(m, nondegenerate=True) as ck:
                    if i == 0:
                        _, buf = m(f, mode="on_pipe")
                    else:
                        _, buf = m(f, buffer=buf if i == 1 else tuple(t.clone() for t in buf), mode="on_pipe")
                assert ck.n == Counter(conv=n, head=3, focus=1), ck.n
        return ck
    return go


FORWARDS = {"train": run_train, "recording": run_recording, "recording_still": lambda: run_recording(still=True),
            "eval": run_eval, "on_pipe": run_on_pipe}


def test_launch_counts_of_the_tiny_tree():
    m = _model()
    assert (conv_launches(m, False), conv_launches(m, True)) == (66, 69)        # 77 BaseConvs, as StreamYOLO-s


@pytest.mark.parametrize("name", list(FORWARDS))
def test_checker_accepts_the_emulated_forward(name, monkeypatch):
    emul_ops.install(monkeypatch)
    ck = FORWARDS[name]()()
    assert ck.worst["bf16"] <= 1.0 and ck.worst["head"] <= 1.0


# ------------------------------------------------------------------------------------------------ mutants
def fused_drops_residual(orig):
    def conv2d(x, wpk, y, k, s, mode, **a):
        if mode == ops.SY_CONV_FUSED:
            a["res"] = None
        return orig(x, wpk, y, k, s, mode, **a)
    return conv2d


def apply_group0_stats_for_group1(orig):
    def bn_act_apply(x, scale_ptr, shift_ptr, split_n, act, res, y, y_goff1=0, res_goff1=0):
        sc, sh = emul_ops.PTRS[scale_ptr].clone(), emul_ops.PTRS[shift_ptr].clone()
        sc[1], sh[1] = sc[0], sh[0]
        return orig(x, sc, sh, split_n, act, res, y, y_goff1, res_goff1)
    return bn_act_apply


def apply_ignores_y_goff1(orig):
    """group 1 written without the channel part of its destination offset: onto group 0's channels (dropping y_goff1
    altogether would address images past the end of the buffer, which the emulation refuses)"""
    def bn_act_apply(x, scale_ptr, shift_ptr, split_n, act, res, y, y_goff1=0, res_goff1=0):
        return orig(x, scale_ptr, shift_ptr, split_n, act, res, y, y_goff1 - y.c if y_goff1 else 0, res_goff1)
    return bn_act_apply


def running_var_biased(orig):
    def conv2d(x, wpk, y, k, s, mode, **a):
        bn = a.get("bn")
        rv0 = [seg[3].clone() for seg in bn] if bn else []
        r = orig(x, wpk, y, k, s, mode, **a)
        if bn:
            raw = y.torch().permute(0, 3, 1, 2).float()
            n = raw.shape[0]
            split = a.get("split_n", 0)
            sp = split if 0 < split < n else n
            c0s = [seg[5] for seg in bn] + [raw.shape[1]]
            for si, seg in enumerate(bn):
                seg[3].copy_(rv0[si])
                for p, q in ([(0, sp), (sp, n)] if sp < n else [(0, n)]):
                    var = raw[p:q, c0s[si]:c0s[si + 1]].var((0, 2, 3), unbiased=False)
                    for _ in range(a.get("stat_updates", 1)):
                        seg[3].mul_(1 - a["momentum"]).add_(a["momentum"] * var)
        return r
    return conv2d


def head_level_one_row_late(orig):
    def head_pred_decode(*args, **kw):
        args = list(args)
        if args[9] == 0:                         # anchor_offset of the first level
            args[9] = args[0].w
        return orig(*args, **kw)
    return head_pred_decode


def conv_skips_one_pixel(orig):
    def conv2d(x, wpk, y, k, s, mode, **a):
        keep = y.torch()[-1, -1, -1].clone()
        r = orig(x, wpk, y, k, s, mode, **a)
        y.torch()[-1, -1, -1] = keep
        return r
    return conv2d


MUTANTS = [("conv2d", fused_drops_residual, "eval"), ("bn_act_apply", apply_group0_stats_for_group1, "train"),
           ("bn_act_apply", apply_ignores_y_goff1, "train"), ("conv2d", running_var_biased, "train"),
           ("conv2d", running_var_biased, "recording_still"), ("head_pred_decode", head_level_one_row_late, "eval"),
           ("head_pred_decode", head_level_one_row_late, "train"), ("conv2d", conv_skips_one_pixel, "train"),
           ("conv2d", conv_skips_one_pixel, "on_pipe")]


@pytest.mark.parametrize("op,mutant,forward", MUTANTS, ids=[f"{m.__name__}-{f}" for _, m, f in MUTANTS])
def test_checker_rejects_mutant(op, mutant, forward, monkeypatch):
    emul_ops.install(monkeypatch)
    go = FORWARDS[forward]()
    monkeypatch.setattr(ops, op, mutant(getattr(ops, op)))
    with pytest.raises(AssertionError):
        go()
