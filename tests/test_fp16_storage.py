"""fp16 activation storage of the eval and on_pipe forwards (``model.activation_dtype = torch.float16``).

CPU (no GPU needed):
  * routing under emulation: the tiny model's eval off_pipe and on_pipe forwards on the torch emulation of the kernels
    (tests/emul_ops.py) with fp16 rounding at every storage point: every buffer created and every packed conv operand is
    fp16, and the outputs lie within twice the rounding-noise floor (+ 1e-3) of the oracle run with fp16 storage rounding;
  * training, the loss.backward() path, the Trainer and the CUDA-core cross-check conv refuse fp16 before any launch;
  * the four conv_tc_f16_kernel instantiations compile without spills or ptxas warnings.

GPU (H100):
  * every launch of the eval forwards of l / m at 8 pairs and of l's on_pipe calls at batch 1, checked in place against
    float64 references on the same fp16 operands (the forward checker of tests/test_gpu_parity_fwd.py with fp16 bars:
    element 2^-10 relative + 2^-10 of the rms, relative L2 2^-11), every distinct FUSED shape under every tiling;
  * the glue kernels and operand packs bit-exact, the depthwise conv and the head prediction against float64;
  * tiny and s end to end against the oracle with fp16 storage rounding, and s's box error against the fp32 oracle;
  * CUDA-graph replays equal eager calls; switching a model to fp16 and back leaves its bf16 outputs bit for bit alone.
"""
import os
import re
import subprocess
import sys
from collections import Counter

import pytest
import torch
import torch.nn.functional as F

from oracle.make_golden import CASES
from oracle.streamyolo_oracle import OracleCfg, StreamYoloOracle, model_shapes
from streamyolo_b200 import ops, synth
from streamyolo_b200.model import DFPPAFPN, TALHead, YOLOX, engine
from streamyolo_b200.ops import View

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import emul_ops  # noqa: E402

F16 = torch.float16
F64 = torch.float64
F16_ULP = 2.0 ** -10          # element bar of an fp16-stored result: one rounding (2^-11) plus accumulation noise
F16_REL_L2 = 2.0 ** -11       # relative L2 bar of an fp16-stored result


def fp16_round(t: torch.Tensor) -> torch.Tensor:
    """the oracle's storage rounding for fp16 activations (bf16_round's counterpart)"""
    return t.to(torch.float16).to(torch.float32)


def rel(a, b):
    a, b = a.float().cpu(), b.float().cpu()
    return ((a - b).norm() / (b.norm() + 1e-12)).item()


def oracle(c, q, momentum=0.03):
    cfg = OracleCfg(depth=c["depth"], width=c["width"], gamma=c.get("gamma", 1.0), ignore_thr=c.get("thr", 0.5),
                    ignore_value=c.get("val", 1.5), bn_momentum=momentum)
    return StreamYoloOracle(cfg, synth.synth_state_dict(model_shapes(c["depth"], c["width"])), q=q)


def duplicated(x):
    """pairs whose support frame is the current frame (as in tests/test_gpu_model.py::test_eval_and_on_pipe_vs_oracle: the
    synthetic weights calibrated on pairs of different frames send some eval boxes to inf, in the oracle as well)"""
    return torch.cat([x[:, 0:3], x[:, 0:3]], 1)


def calibrated_oracle(c, x, tg, q):
    """eval oracle whose running statistics are the batch statistics of one train pass over duplicated(x) (BatchNorm
    momentum 1)"""
    o = oracle(c, q, momentum=1.0)
    o.forward(duplicated(x), tg)
    o.training = False
    return o


def product_from(o, c):
    ch = [256, 512, 1024]
    m = YOLOX(DFPPAFPN(c["depth"], c["width"], in_channels=ch), TALHead(8, c["width"], in_channels=ch))
    for mod in m.modules():
        if isinstance(mod, torch.nn.BatchNorm2d):
            mod.eps = 1e-3
    m.load_state_dict({k: v.clone() for k, v in o.P.items()}, strict=True)
    return m.eval()


def compare_to_oracle(m, o, x, dev, nudge=1e-6):
    """eval off_pipe (on duplicated(x)) and on_pipe (star call on frame 0, buffered call on frame 1) of the product ``m``
    against the oracle ``o``, each judged against the oracle's own rounding-noise floor (the same oracle on inputs nudged by
    ``nudge``, relative): within twice the floor + 1e-3.  Returns the product's eval outputs and the oracle's."""
    xc = duplicated(x)
    with torch.no_grad():
        got = m(xc.to(dev)).float().cpu()
        ref, pert = o.forward(xc), o.forward(xc * (1 + nudge))
        assert bool(torch.isfinite(ref).all()) and bool(torch.isfinite(got).all())
        assert got.shape == ref.shape
        floor = rel(pert[..., :4], ref[..., :4])
        r = rel(got[..., :4], ref[..., :4])
        assert r <= 2 * floor + 1e-3, f"eval boxes: rel l2 {r:.3g}, noise floor {floor:.3g}"
        e, fe = float((got[..., 4:] - ref[..., 4:]).abs().max()), float((pert[..., 4:] - ref[..., 4:]).abs().max())
        assert e <= 2 * fe + 1e-3, f"eval scores: max err {e:.3g}, noise floor {fe:.3g}"
        f0, f1 = x[:1, 0:3], x[1:2, 0:3]
        o1, buf = m(f0.to(dev), mode="on_pipe")
        o2, _ = m(f1.to(dev), buffer=buf, mode="on_pipe")
        assert all(t.dtype == m.activation_dtype for t in buf)
        r1, rbuf = o.forward(f0, mode="on_pipe")
        r2, _ = o.forward(f1, buffer=rbuf, mode="on_pipe")
        p1, pbuf = o.forward(f0 * (1 + nudge), mode="on_pipe")
        p2, _ = o.forward(f1 * (1 + nudge), buffer=pbuf, mode="on_pipe")
        for what, a, b, p in (("on_pipe star", o1, r1, p1), ("on_pipe buffered", o2, r2, p2)):
            fl = rel(p[..., :4], b[..., :4])
            r = rel(a[..., :4], b[..., :4])
            assert r <= 2 * fl + 1e-3, f"{what} boxes: rel l2 {r:.3g}, noise floor {fl:.3g}"
            e, fe = float((a[..., 4:].float().cpu() - b[..., 4:]).abs().max()), float((p[..., 4:] - b[..., 4:]).abs().max())
            assert e <= 2 * fe + 1e-3, f"{what} scores: max err {e:.3g}, noise floor {fe:.3g}"
        for k, (a, b, p) in enumerate(zip(buf, rbuf, pbuf)):
            fl = rel(p, b)
            r = rel(a, b)
            assert r <= 2 * fl + 1e-3, f"on_pipe buffer {k}: rel l2 {r:.3g}, noise floor {fl:.3g}"
    return got, ref


# ================================================================================================ CPU
TINY = CASES["tiny_120x160"]


def _focus_pack_f16(x, frames, y):
    """what sy_focus_pack_f16 writes (emul_ops.focus_pack with fp16 input rounding)"""
    xs = torch.cat([x[:, 3 * f:3 * f + 3] for f in range(frames)], 0).to(F16).float()
    foc = torch.cat([xs[..., ::2, ::2], xs[..., 1::2, ::2], xs[..., ::2, 1::2], xs[..., 1::2, 1::2]], 1)
    n, _, h, w = foc.shape
    out = torch.zeros(n, 64, h, w)
    out[:, 16:28] = foc
    out[:, 0:12, :, 1:] = foc[..., :-1]
    out[:, 32:44, :, :-1] = foc[..., 1:]
    y.torch().copy_(out.permute(0, 2, 3, 1).to(y.dtype))


def _install_f16_emulation(monkeypatch):
    """emul_ops with fp16 rounding at every storage point, plus a log of the dtypes every launch / buffer / operand has"""
    emul_ops.install(monkeypatch, exact=False)
    monkeypatch.setattr(emul_ops, "_bf", lambda t: t.to(F16))
    log = Counter()
    orig_empty = View.empty

    def empty(n, h, w, c, device, dtype=torch.bfloat16):
        log[("view", dtype)] += 1
        return orig_empty(n, h, w, c, device, dtype)
    monkeypatch.setattr(View, "empty", staticmethod(empty))

    def packer(fn, name):
        def pack(*ws, dtype=torch.bfloat16):
            out = fn(*ws)                             # rounded by the patched _bf: fp16
            log[(name, dtype, out.dtype)] += 1
            return out
        return pack
    for name in ("pack_conv_weight", "pack_stem_weight", "pack_dw_weight"):
        monkeypatch.setattr(ops, name, packer(getattr(emul_ops, name), name))
    conv = emul_ops.conv2d

    def conv2d(x, wpk, y, k, s, mode, **a):
        res = a.get("res")
        log[("conv", x.dtype, y.dtype, wpk.dtype, res.dtype if res is not None else None, mode)] += 1
        return conv(x, wpk, y, k, s, mode, **a)
    monkeypatch.setattr(ops, "conv2d", conv2d)

    def focus_pack(x, frames, y):
        log[("focus", y.dtype)] += 1
        _focus_pack_f16(x, frames, y)
    monkeypatch.setattr(ops, "focus_pack", focus_pack)
    return log


def test_fp16_routing_under_emulation(monkeypatch):
    """tiny model, eval off_pipe (frame pairs) and on_pipe (star + buffered): fp16 everywhere, oracle-close"""
    log = _install_f16_emulation(monkeypatch)
    x = synth.synth_frames(TINY["B"], TINY["H"], TINY["W"])
    tg = synth.synth_labels(TINY["B"], TINY["H"], TINY["W"])
    o = calibrated_oracle(TINY, x, tg, fp16_round)
    m = product_from(o, TINY)
    m.activation_dtype = F16
    assert (m.backbone.activation_dtype, m.head.activation_dtype) == (F16, F16)
    compare_to_oracle(m, o, x, "cpu")
    assert log, "no launch was emulated"
    for key, n in log.items():
        assert all(d in (F16, None, ops.SY_CONV_FUSED) for d in key[1:]), (key, n)
    assert sum(n for k, n in log.items() if k[0] == "conv") > 0 and sum(n for k, n in log.items() if k[0] == "view") > 0
    # the operands sit in their own cache slots: the bf16 slots were never filled
    assert not any(hasattr(mod, "_pk") or hasattr(mod, "_pk2") for mod in m.modules())
    assert any(hasattr(mod, "_pkh") for mod in m.modules()) and any(hasattr(mod, "_pk2h") for mod in m.modules())


def _tiny_model():
    ch = [256, 512, 1024]
    m = YOLOX(DFPPAFPN(TINY["depth"], TINY["width"], in_channels=ch), TALHead(8, TINY["width"], in_channels=ch))
    m.head.use_l1 = True
    return m


def test_fp16_refused_outside_eval(monkeypatch):
    """train forward, the loss.backward() path, the Trainer, a stand-alone train-mode backbone / head, and eval on the
    CUDA-core cross-check conv: NotImplementedError before any launch (a launch would fail differently on a CPU host)"""
    from streamyolo_b200.train import Trainer
    x = synth.synth_frames(1, 64, 96)
    tg = synth.synth_labels(1, 64, 96)
    m = _tiny_model().train()
    m.activation_dtype = F16
    with torch.no_grad(), pytest.raises(NotImplementedError):
        m(x, tg)
    with torch.enable_grad(), pytest.raises(NotImplementedError):
        m(x, tg)["total_loss"].backward()
    with pytest.raises(NotImplementedError):
        Trainer(m)
    with pytest.raises(NotImplementedError):
        m.backbone(x)
    with pytest.raises(NotImplementedError):
        m.head([torch.zeros(1, 32, 8, 12), torch.zeros(1, 64, 4, 6), torch.zeros(1, 128, 2, 3)], tg)
    m.eval()
    monkeypatch.setattr(engine, "CONV_IMPL", "simt")
    with torch.no_grad(), pytest.raises(NotImplementedError):
        m(x)
    with pytest.raises(ValueError):
        m.activation_dtype = torch.float32
    assert m.activation_dtype == F16
    m.activation_dtype = torch.bfloat16
    assert (m.backbone.activation_dtype, m.head.activation_dtype) == (torch.bfloat16, torch.bfloat16)


def test_f16_conv_kernels_compile_without_spills(tmp_path):
    """conv_tc_f16_kernel (BN = 64 / 128 x linear / halo) fits its register budget: 0 spill bytes, no ptxas warning"""
    import shutil
    from streamyolo_b200 import build
    if not os.path.exists(build.NVCC) and shutil.which("nvcc") is None:
        pytest.skip("no nvcc")
    nvcc = build.NVCC if os.path.exists(build.NVCC) else shutil.which("nvcc")
    r = subprocess.run([nvcc] + build.COMMON + ["-c", os.path.join(build.CSRC, "conv_tc.cu"), "-o", str(tmp_path / "c.o")],
                       stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=900)
    assert r.returncode == 0, r.stdout
    assert not [ln for ln in r.stdout.splitlines() if ln.startswith("ptxas") and "warning" in ln.lower()], r.stdout
    found = re.findall(r"Compiling entry function '(\w+)'[^\n]*\n[^\n]*\n\s*\d+ bytes stack frame, "
                       r"(\d+) bytes spill stores, (\d+) bytes spill loads", r.stdout)
    f16 = [(n, int(s), int(ld)) for n, s, ld in found if "conv_tc_f16_kernel" in n]
    assert len(f16) == 4, f16
    assert all(s == 0 and ld == 0 for _, s, ld in f16), f16
    assert sum(bool(re.search(r"conv_tc_kernelILi\d+ELb0E", n)) for n, _, _ in found) == 4


# ================================================================================================ GPU
DEV = "cuda"
NAN = float("nan")


def _gpu_helpers():
    from test_gpu_parity_bwd import MODELS, nchw64, outside_bf16
    from test_gpu_parity_fwd import (FUSED_SHAPES, FwdChecker, _same_bits, _sync, conv_launches, conv_refs, fused_key,
                                     stem_weight_3x1)
    from test_gpu_ops import check_close
    return dict(MODELS=MODELS, nchw64=nchw64, outside=outside_bf16, FUSED_SHAPES=FUSED_SHAPES, FwdChecker=FwdChecker,
                same_bits=_same_bits, sync=_sync, conv_launches=conv_launches, conv_refs=conv_refs, fused_key=fused_key,
                stem_weight_3x1=stem_weight_3x1, check_close=check_close)


def f16_close(got, ref, what):
    """one fp16 rounding plus accumulation noise, element-wise and in relative L2"""
    H = _gpu_helpers()
    H["check_close"](got, ref, what, ulp=F16_ULP)
    r = float((got.to(F64) - ref).norm() / (ref.norm() + 1e-300))
    assert r <= F16_REL_L2, f"{what}: relative L2 error {r:.3g} above {F16_REL_L2:.3g}"
    return r


def make_f16_checker(model, nondegenerate=True):
    """tests/test_gpu_parity_fwd.py's FwdChecker for the fp16 eval forwards: operands from the "_pkh" / "_pk2h" slots, conv
    references from the module's weights rounded to fp16, the fp16 bars; the head / NaN-fill / untouched-bytes logic is
    the parent's"""
    H = _gpu_helpers()
    nchw64 = H["nchw64"]

    class F16Checker(H["FwdChecker"]):
        def _operands(self):
            from streamyolo_b200.model.network_blocks import BaseConv, CSPLayer
            m = self.model
            stem = m.backbone.backbone.stem.conv
            table = {}
            for mod in m.modules():
                if isinstance(mod, BaseConv) and hasattr(mod, "_pkh"):
                    table[mod._pkh.data_ptr()] = ("stem" if mod is stem else "conv", (mod,))
            pairs = [(c.conv1, c.conv2) for c in m.modules() if isinstance(c, CSPLayer)]
            pairs += [(c[0], r[0]) for c, r in zip(m.head.cls_convs, m.head.reg_convs)]
            for a, b in pairs:
                if hasattr(a, "_pk2h"):
                    table[a._pk2h.data_ptr()] = ("pair", (a, b))
            assert table, "no fp16 operands: run one fp16 forward before checking"
            return table

        def _conv2d(self, x, wpk, y, k, s, mode, **a):
            res = a.get("res")
            assert mode == ops.SY_CONV_FUSED and x.dtype == y.dtype == wpk.dtype == F16, "fp16 eval launch"
            assert res is None or res.dtype == F16
            assert wpk.data_ptr() in self.table, "conv launch with an operand that is no module's fp16 packed weight"
            kind, mods = self.table[wpk.data_ptr()]
            name = getattr(mods[0], "_sy_name", kind)
            x64 = nchw64(x)
            r64 = nchw64(res) if res is not None else None
            before = y.buf.clone()
            if not (y.buf is x.buf or (res is not None and y.buf is res.buf)):
                y.torch().fill_(NAN)
            rv_ = self.orig["conv2d"](x, wpk, y, k, s, mode, **a)
            H["sync"](y.buf)
            self.n["conv"] += 1
            w64 = torch.cat([m.conv.weight.detach() for m in mods], 0).to(F16).to(F64)
            if kind == "stem":
                w64 = H["stem_weight_3x1"](w64)
            got = nchw64(y)
            self.fused_shapes.add(H["fused_key"](x, y, k, s, res, kind))
            sc, sh = self._fold(mods)
            ref, omit = H["conv_refs"](x64, w64, s, sc, sh, self._act(mods), r64)
            what = f"{name}: fp16 FUSED conv"
            del x64, r64
            r = f16_close(got, ref, what)
            self._note("f16_rel_l2", r)
            assert H["outside"](got, omit, ulp=F16_ULP) > 0, f"{what}: the bar accepts input channels 0-63 at the centre tap left out"
            del ref, omit
            if self.nondegenerate:
                assert float((got.abs() > 1e-2).double().mean()) >= 0.25, f"{what}: degenerate output"
            sl = (slice(y.n0, y.n0 + y.n), slice(None), slice(None), slice(y.c0, y.c0 + y.c))
            before[sl] = y.buf[sl]
            assert H["same_bits"](before, y.buf), f"{what}: writes outside its output view"
            return rv_

        def _focus_pack(self, x, frames, y):
            self.orig["focus_pack"](x, frames, y)
            H["sync"](y.buf)
            self.n["focus"] += 1
            xs = torch.cat([x[:, 3 * f:3 * f + 3] for f in range(frames)], 0).to(F16).to(F64)
            foc = torch.cat([xs[..., ::2, ::2], xs[..., 1::2, ::2], xs[..., ::2, 1::2], xs[..., 1::2, 1::2]], 1)
            out = foc.new_zeros((foc.shape[0], 64, foc.shape[2], foc.shape[3]))
            out[:, 16:28] = foc
            out[:, 0:12, :, 1:] = foc[..., :-1]
            out[:, 32:44, :, :-1] = foc[..., 1:]
            assert y.dtype == F16 and torch.equal(nchw64(y), out), "Focus packing of the fp16 frames"

    return F16Checker(model, nondegenerate=nondegenerate)


def _calibrated_f16(tag):
    from test_gpu_parity_fwd import _calibrated
    x = synth.synth_frames(8, 600, 960, seed=99).cuda()
    m = _calibrated(tag, x)
    m.activation_dtype = F16
    with torch.no_grad():
        m(x)                                          # fills the fp16 operand slots
    return m, x


@pytest.mark.gpu
@pytest.mark.parametrize("tag,launches", [("l", 117), ("m", 93)])
def test_f16_eval_forward_every_launch(tag, launches):
    H = _gpu_helpers()
    m, x = _calibrated_f16(tag)
    with torch.no_grad(), make_f16_checker(m) as ck:
        out = m(x)
    assert ck.n == Counter(conv=launches, head=3, focus=1), ck.n
    assert out.dtype == torch.float32 and tuple(out.shape) == (8, 11850, 13)
    assert ck.fused_shapes == set(H["FUSED_SHAPES"][f"{tag}_eval"]), sorted(ck.fused_shapes ^ set(H["FUSED_SHAPES"][f"{tag}_eval"]))
    print(f"\nFP16 {tag} eval b8: launches {dict(ck.n)}; worst " + ", ".join(f"{k} {v:.3g}" for k, v in sorted(ck.worst.items())))


@pytest.mark.gpu
def test_f16_on_pipe_every_launch_l():
    H = _gpu_helpers()
    m, _ = _calibrated_f16("l")
    f = synth.synth_frames(3, 600, 960, seed=98)[:, :3].contiguous().cuda()
    launches = H["conv_launches"](m, jian_twice=True)
    shapes = set()
    with torch.no_grad():
        buf = None
        for i in range(3):
            with make_f16_checker(m) as ck:
                if i == 0:
                    _, buf = m(f[0:1], mode="on_pipe")
                else:
                    _, buf = m(f[i:i + 1], buffer=buf if i == 1 else tuple(t.clone() for t in buf), mode="on_pipe")
            assert all(t.dtype == F16 for t in buf)
            assert ck.n == Counter(conv=launches, head=3, focus=1), ck.n
            shapes |= ck.fused_shapes
    assert shapes == set(H["FUSED_SHAPES"]["l_on_pipe"]), sorted(shapes ^ set(H["FUSED_SHAPES"]["l_on_pipe"]))


def _f16_cases():
    from test_gpu_parity_fwd import FUSED_SHAPES
    return sorted(set(c for v in FUSED_SHAPES.values() for c in v))


def _post_silu16(n, h, w, c, seed):
    g = torch.Generator(device=DEV).manual_seed(seed)
    mu = torch.rand(c, generator=g, device=DEV) * 2.0 - 1.0
    return View(F.silu(torch.randn((n, h, w, c), generator=g, device=DEV) + mu).to(F16))


@pytest.mark.gpu
@pytest.mark.parametrize("case", _f16_cases(), ids=lambda c: "x".join(map(str, c)))
def test_f16_fused_shape_every_tiling(case):
    """fp16 FUSED epilogue at one eval launch shape under every tiling: folded scale / shift, SiLU, the residual in place or
    from a slice, output into a channel slice of a wider buffer holding a sentinel"""
    from test_gpu_parity_bwd import DGRAD_TILINGS
    H = _gpu_helpers()
    nchw64 = H["nchw64"]
    n, ci, co, h, w, kh, kw, s, kind, rk = case
    g = torch.Generator(device=DEV).manual_seed(sum(v for v in case if isinstance(v, int)))
    if kind == "stem":
        frames = torch.rand((n, 3, 2 * h, 2 * w), generator=g, device=DEV) * 255
        xv = View.empty(n, h, w, 64, DEV, F16)
        ops.focus_pack(frames, 1, xv)
        w12 = (torch.randn((co, 12, 3, 3), generator=g, device=DEV) / 108 ** 0.5).to(F16).float()
        wpk, w64 = ops.pack_stem_weight(w12, dtype=F16), H["stem_weight_3x1"](w12.to(F64))
    else:
        xv = _post_silu16(n, h, w, ci, 1)
        ws = [(torch.randn((c_, ci, kh, kw), generator=g, device=DEV) / (ci * kh * kw) ** 0.5).to(F16).float()
              for c_ in ((co // 2, co // 2) if kind == "pair" else (co,))]
        wpk, w64 = ops.pack_conv_weight(*ws, dtype=F16), torch.cat(ws, 0).to(F64)
    assert wpk.dtype == F16
    ho, wo = ops.conv_out_hw(h, w, kh, s) if kh == kw else (h, w)
    sc = torch.rand(co, generator=g, device=DEV) + 0.5
    sh = torch.rand(co, generator=g, device=DEV) - 0.5
    sentinel = torch.full((n, ho, wo, co + 64), -7.0, dtype=F16, device=DEV)
    r0 = _post_silu16(n, ho, wo, 2 * co, 2)
    res64 = nchw64(r0.ch(co, co)) if rk != "none" else None
    ref, omit = H["conv_refs"](nchw64(xv), w64, s, sc.to(F64)[None, :, None, None], sh.to(F64)[None, :, None, None], 1, res64)
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
        what = f"fp16 FUSED {case} {tname}"
        f16_close(got, ref, what)
        assert H["outside"](got, omit, ulp=F16_ULP) > 0, f"{what}: the bar accepts input channels 0-63 at the centre tap left out"
        wide[..., 32:32 + co] = sentinel[..., 32:32 + co]
        assert H["same_bits"](wide, sentinel), f"{what}: writes outside its output slice"


@pytest.mark.gpu
def test_f16_conv_refusals_and_debug_f32():
    """fp16 runs FUSED only: RAW mode and statistics are refused; the fp32 accumulators of debug_f32 still come out; mixed
    storage dtypes are refused on the host"""
    xv = _post_silu16(2, 19, 30, 64, 3)
    w = torch.randn((64, 64, 3, 3), device=DEV) / 24
    wpk = ops.pack_conv_weight(w, dtype=F16)
    y = View.empty(2, 19, 30, 64, DEV, F16)
    with pytest.raises(RuntimeError, match="FUSED"):
        ops.conv2d(xv, wpk, y, 3, 1, ops.SY_CONV_RAW)
    with pytest.raises(RuntimeError, match="FUSED"):
        ops.conv2d(xv, wpk, y, 3, 1, ops.SY_CONV_FUSED, partials=torch.zeros((ops.conv_stat_rows(), 256), device=DEV))
    with pytest.raises(RuntimeError):
        ops.conv2d(xv, wpk, y, 3, 1, ops.SY_CONV_FUSED, impl="simt")
    with pytest.raises(ValueError):
        ops.conv2d(xv, ops.pack_conv_weight(w), y, 3, 1, ops.SY_CONV_FUSED)
    with pytest.raises(ValueError):
        ops.conv2d(xv, wpk, View.empty(2, 19, 30, 64, DEV), 3, 1, ops.SY_CONV_FUSED)
    dbg = torch.full((2 * 19 * 30, 64), NAN, device=DEV)
    ops.conv2d(xv, wpk, y, 3, 1, ops.SY_CONV_FUSED, debug_f32=dbg)
    torch.cuda.synchronize()
    ref = F.conv2d(xv.torch().permute(0, 3, 1, 2).to(F64), w.to(F16).to(F64), None, 1, 1).permute(0, 2, 3, 1).reshape(-1, 64)
    err = (dbg.to(F64) - ref).abs()
    assert bool((err <= 1e-5 * ref.abs() + 1e-5 * ref.pow(2).mean().sqrt()).all()), float(err.max())
    f16_close(y.torch().permute(0, 3, 1, 2).to(F64), F.silu(ref.reshape(2, 19, 30, 64).permute(0, 3, 1, 2)), "fp16 FUSED")


@pytest.mark.gpu
def test_f16_glue_bit_exact():
    """focus_pack, spp_maxpool, upsample, copy and the fp16 operand packs against torch, bit for bit"""
    g = torch.Generator(device=DEV).manual_seed(7)
    x = torch.rand((2, 6, 64, 96), generator=g, device=DEV) * 255
    y = View.empty(4, 32, 48, 64, DEV, F16)
    ops.focus_pack(x, 2, y)
    xs = torch.cat([x[:, 0:3], x[:, 3:6]], 0).to(F16)
    foc = torch.cat([xs[..., ::2, ::2], xs[..., 1::2, ::2], xs[..., ::2, 1::2], xs[..., 1::2, 1::2]], 1)
    want = torch.zeros((4, 64, 32, 48), dtype=F16, device=DEV)
    want[:, 16:28] = foc
    want[:, 0:12, :, 1:] = foc[..., :-1]
    want[:, 32:44, :, :-1] = foc[..., 1:]
    assert torch.equal(y.torch(), want.permute(0, 2, 3, 1))
    for (h, w) in ((19, 30), (40, 40)):                     # the shared-memory cascade and the direct kernel
        t = (torch.randn((2, h, w, 96), generator=g, device=DEV) * 3).to(F16)
        s = View.empty(2, h, w, 4 * 64, DEV, F16)
        s.ch(0, 64).torch().copy_(t[..., :64])
        ops.spp_maxpool(s.ch(0, 64), s.ch(64, 64), s.ch(128, 64), s.ch(192, 64))
        tn = t[..., :64].permute(0, 3, 1, 2).float()
        for i, k in enumerate((5, 9, 13)):
            ref = F.max_pool2d(tn, k, 1, k // 2).to(F16).permute(0, 2, 3, 1)
            assert torch.equal(s.ch(64 * (i + 1), 64).torch(), ref), (h, w, k)
    t = View((torch.randn((2, 19, 30, 64), generator=g, device=DEV)).to(F16))
    u = View.empty(2, 38, 60, 128, DEV, F16)
    ops.upsample_nearest(t, u.ch(64, 64))
    assert torch.equal(u.ch(64, 64).torch(), F.interpolate(t.torch().permute(0, 3, 1, 2).float(), size=(38, 60)).to(F16).permute(0, 2, 3, 1))
    c = View.empty(2, 19, 30, 64, DEV, F16)
    ops.copy(t, c)
    assert torch.equal(c.torch(), t.torch())
    w = torch.randn((96, 80, 3, 3), generator=g, device=DEV)
    w2 = torch.randn((32, 80, 3, 3), generator=g, device=DEV)
    got = ops.pack_conv_weight(w, w2, dtype=F16)
    assert got.dtype == F16 and torch.equal(got, torch.cat([w, w2]).permute(0, 2, 3, 1).reshape(128, 9, 80).to(F16))
    ws = torch.randn((48, 12, 3, 3), generator=g, device=DEV)
    st = ops.pack_stem_weight(ws, dtype=F16)
    ref = torch.zeros((48, 3, 4, 16), device=DEV)
    ref[:, :, :3, :12] = ws.permute(0, 2, 3, 1)
    assert st.dtype == F16 and torch.equal(st, ref.reshape(48, 3, 64).to(F16))
    wd = torch.randn((64, 1, 5, 5), generator=g, device=DEV)
    dw = ops.pack_dw_weight(wd, dtype=F16)
    assert dw.dtype == F16 and torch.equal(dw, wd.reshape(64, 25).t().to(F16))


@pytest.mark.gpu
@pytest.mark.parametrize("case", [(2, 64, 75, 120, 3, 1), (2, 128, 38, 60, 3, 2), (3, 24, 19, 31, 5, 1), (2, 16, 15, 20, 1, 1),
                                  (1, 256, 150, 240, 3, 2), (2, 48, 37, 59, 5, 2)], ids=lambda c: "x".join(map(str, c)))
def test_f16_dwconv_vs_float64(case):
    n, c, h, w, k, s = case
    g = torch.Generator().manual_seed(1)
    x = torch.randn((n, c, h, w), generator=g).to(F16).cuda()
    wt = (torch.randn((c, 1, k, k), generator=g) / k).cuda()
    wpk = ops.pack_dw_weight(wt, dtype=F16)
    ref = F.conv2d(x.to(F64), wt.to(F16).to(F64), None, s, (k - 1) // 2, groups=c)
    ho, wo = ref.shape[2], ref.shape[3]
    scale = (torch.rand(c, generator=g) + 0.5).cuda()
    shift = (torch.rand(c, generator=g) - 0.5).cuda()
    res = torch.randn((n, c, ho, wo), generator=g).to(F16).cuda()
    y = View.empty(n, ho, wo, c, DEV, F16)
    y.buf.fill_(NAN)
    ops.conv2d(View(x.permute(0, 2, 3, 1).contiguous()), wpk, y, k, s, ops.SY_CONV_FUSED, impl="dw", scale=scale, shift=shift,
               act=1, res=View(res.permute(0, 2, 3, 1).contiguous()))
    torch.cuda.synchronize()
    want = F.silu(ref * scale.to(F64)[None, :, None, None] + shift.to(F64)[None, :, None, None]) + res.to(F64)
    f16_close(y.torch().permute(0, 3, 1, 2).to(F64), want, f"fp16 dwconv fused {case}")
    with pytest.raises(RuntimeError, match="FUSED"):
        ops.conv2d(View(x.permute(0, 2, 3, 1).contiguous()), wpk, y, k, s, ops.SY_CONV_RAW, impl="dw")


@pytest.mark.gpu
@pytest.mark.parametrize("nc", [8, 20, 3])
def test_f16_head_pred_decode_vs_float64(nc):
    """prediction convs (fp32) on fp16 tower features: raw outputs within the fp32-reduction bar of float64, decoded ones
    and sigmoids through the same expressions"""
    from test_gpu_parity_bwd import U32, sum_tol
    g = torch.Generator(device=DEV).manual_seed(nc)
    b, h, w, c = 2, 38, 60, 256
    cf = View((torch.randn((b, h, w, c), generator=g, device=DEV)).to(F16))
    rf = View((torch.randn((b, h, w, c), generator=g, device=DEV)).to(F16))
    wr, wo, wc = (torch.randn((o, c), generator=g, device=DEV) / 16 for o in (4, 1, nc))
    br, bo, bc = (torch.randn((o,), generator=g, device=DEV) for o in (4, 1, nc))
    a = h * w + 100
    out = torch.full((b, a, 5 + nc), NAN, device=DEV)
    ops.head_pred_decode(cf, rf, wr, br, wo, bo, wc, bc, 16, 100, a, out, None, sigmoid=False, decode=False)
    torch.cuda.synchronize()
    f_r, f_c = rf.torch().to(F64).reshape(b, h * w, c), cf.torch().to(F64).reshape(b, h * w, c)
    lin = torch.cat([f_r @ wr.to(F64).T + br.to(F64), f_r @ wo.to(F64).T + bo.to(F64), f_c @ wc.to(F64).T + bc.to(F64)], -1)
    s2 = torch.cat([f_r.square() @ wr.to(F64).square().T, f_r.square() @ wo.to(F64).square().T,
                    f_c.square() @ wc.to(F64).square().T], -1)
    tol = sum_tol(lin, s2, c + 1) + 16 * U32 * lin.abs()
    got = out[:, 100:].to(F64)
    assert bool(((got - lin).abs() <= tol).all()), float(((got - lin).abs() / tol).max())
    assert bool(torch.isnan(out[:, :100]).all()), "head_pred writes outside its anchor rows"
    ops.head_pred_decode(cf, rf, wr, br, wo, bo, wc, bc, 16, 100, a, out, None, sigmoid=True, decode=True)
    torch.cuda.synchronize()
    yv, xv = torch.meshgrid(torch.arange(h, device=DEV), torch.arange(w, device=DEV), indexing="ij")
    raw = got.clone()
    dec = torch.cat([((raw[..., 0] + xv.reshape(-1)) * 16)[..., None], ((raw[..., 1] + yv.reshape(-1)) * 16)[..., None],
                     torch.exp(raw[..., 2:4]) * 16, torch.sigmoid(raw[..., 4:])], -1)
    assert torch.allclose(out[:, 100:].to(F64), dec, rtol=1e-5, atol=1e-6)
    with pytest.raises(ValueError):
        ops.head_pred_decode(cf, View(rf.buf.to(torch.bfloat16)), wr, br, wo, bo, wc, bc, 16, 100, a, out, None, True, True)


@pytest.mark.gpu
@pytest.mark.parametrize("case", ["tiny_120x160", "s_600x960"])
def test_f16_model_vs_oracle(case):
    """eval off_pipe and on_pipe against the oracle with fp16 storage rounding (twice its rounding-noise floor + 1e-3); on
    s at 600x960 the fp16 product's box error against the fp32 oracle is at most a third of the bf16 product's.

    The floor of s nudges the inputs by 1e-4, not 1e-6: the frames are 0-255, where fp16 values are 0.125 apart, so a 1e-6
    nudge moves almost no fp16-rounded input pixel, while the product's fp32 accumulation order differs from the oracle's in
    every layer and the random-init network amplifies that.  Measured on an H100 (2 pairs): the product's deviation from the
    oracle grows smoothly from 1.6e-5 at the stem to 2.6e-2 at the last head convs, about 5x below the bf16 product's at
    every layer; eval boxes 3.2e-2 against a 1e-6-nudge floor of 7.3e-3.  Every launch of the product is checked against
    float64 on its own operands by the tests above; a 1e-4 nudge moves about one input pixel in six across an fp16
    rounding boundary."""
    c = dict(CASES[case])
    b = 2 if case.startswith("tiny") else 1
    x = synth.synth_frames(max(b, 2), c["H"], c["W"])
    tg = synth.synth_labels(max(b, 2), c["H"], c["W"])
    o16 = calibrated_oracle(c, x, tg, fp16_round)
    m = product_from(o16, c).cuda()
    m.activation_dtype = F16
    got16, _ = compare_to_oracle(m, o16, x, DEV, nudge=1e-6 if case.startswith("tiny") else 1e-4)
    if case.startswith("s"):
        o32 = calibrated_oracle(c, x, tg, None)
        xc = duplicated(x)
        ref32 = o32.forward(xc)
        m32 = product_from(o32, c).cuda()
        with torch.no_grad():
            m32.activation_dtype = F16
            e16 = rel(m32(xc.cuda())[..., :4], ref32[..., :4])
            m32.activation_dtype = torch.bfloat16
            e_bf = rel(m32(xc.cuda())[..., :4], ref32[..., :4])
        print(f"\ns 600x960 eval boxes vs fp32 oracle: fp16 storage rel l2 {e16:.3g}, bf16 storage {e_bf:.3g} ({e_bf / e16:.2f}x)")
        assert e16 <= e_bf / 3, (e16, e_bf)


@pytest.mark.gpu
def test_f16_graph_replay_equals_eager_and_switch_back():
    """CUDA-graph replays of fp16 eval (8 pairs) and of an on_pipe sequence equal the eager calls bit for bit; a model
    switched to fp16 and back gives bf16 outputs bit-identical to a model that never was switched"""
    from bench import capture
    from test_gpu_parity_fwd import _calibrated
    x = synth.synth_frames(8, 600, 960, seed=99).cuda()
    m = _calibrated("l", x)
    with torch.no_grad():
        ref_bf16 = m(x).clone()
        m.activation_dtype = F16
        want = m(x).clone()
        assert not torch.equal(want, ref_bf16)
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
        for d_, s_ in zip(buf_static, buf0):
            d_.copy_(s_)
        for i in range(1, 4):
            f_static.copy_(f[i:i + 1])
            g.replay()
            torch.cuda.synchronize()
            assert torch.equal(out, eager[i - 1]), f"fp16 on_pipe frame {i}"
        del g, out
        m.activation_dtype = torch.bfloat16
        assert torch.equal(m(x), ref_bf16), "bf16 eval after an fp16 excursion"
    fresh = _calibrated("l", x)
    with torch.no_grad():
        assert torch.equal(fresh(x), ref_bf16), "bf16 eval of a model never switched"
