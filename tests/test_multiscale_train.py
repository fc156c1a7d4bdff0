"""Multi-scale training (Exp.random_resize every 10 iterations, cfgs/*.py:138-171) with the graphed Trainer: the size set,
the device prologue (pair / frame transform at input_size, then Exp.preprocess into each size's static input), one captured
step per size in one memory pool (train.Trainer.capture_sizes / replay_size), and the kernels at the multi-scale shapes.

CPU (kernels emulated, tests/emul_ops.py): the size formula, eager steps at two sizes whose stride-16 map is odd against
the fp32 oracle, the prologue's preprocess semantics.  GPU: graph replays == eager steps with the sizes interleaved (pair
and still models), no side effects of the capture, every conv launch at the extreme sizes against float64, and the
memory of 22 captured sizes."""
import gc
import os
import random
import sys
from collections import Counter

import pytest
import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import emul_ops  # noqa: E402
import test_cpu_backward as T  # noqa: E402
from oracle.make_golden import CASES  # noqa: E402
from oracle.streamyolo_oracle import OracleCfg, StreamYoloOracle  # noqa: E402
from streamyolo_b200 import data, ops, synth, train  # noqa: E402

MAX_LABELS = 50


# ------------------------------------------------------------------------------------------------ CPU
def test_multiscale_sizes_follow_random_resize():
    """Exp.random_resize: size = randint(50, 70), (16 * int(size * 600 / 960), 16 * size); input_size in the last epoch"""
    want = {(16 * int(s * (600 * 1.0 / 960)), int(16 * s)) for s in range(50, 71)}
    got = train.multiscale_sizes()
    assert len(got) == len(set(got)) == 22
    assert set(got) == want | {(600, 960)}
    assert all(h % 16 == 0 and w % 16 == 0 for h, w in want)
    assert min(want) == (496, 800) and max(want) == (688, 1120)
    rng = random.Random(3)                                   # every draw of the reference's formula is in the set
    for _ in range(200):
        s = rng.randint(50, 70)
        assert (16 * int(s * 600 * 1.0 / 960), int(16 * s)) in got
    assert train.multiscale_sizes((120, 192), (10, 14)) == [(96, 160), (96, 176), (112, 192), (128, 208), (128, 224),
                                                            (120, 192)]


def test_eager_steps_at_two_sizes_match_fp32_oracle(monkeypatch):
    """Trainer.step alternating between 112x176 and 144x224 (stride-16 maps 7x11 and 9x14: odd, so the nearest upsample
    of the 4x6 / 5x7 stride-32 maps runs at a non-2x ratio) on the tiny model: every step's losses equal the fp32 oracle's
    on the parameters the step starts from (the bar of tests/test_cpu_backward.py)."""
    emul_ops.install(monkeypatch, exact=True)
    c = CASES["tiny_120x160"]
    model = T.build_product(c)
    tr = train.Trainer(model, lr=2e-4)
    cfg = OracleCfg(depth=c["depth"], width=c["width"], gamma=c["gamma"], ignore_thr=c["thr"], ignore_value=c["val"])
    for i, (h, w) in enumerate([(112, 176), (144, 224), (112, 176)]):
        x = synth.synth_frames(c["B"], h, w, seed=10 + i)
        tg = synth.synth_labels(c["B"], h, w, seed=20 + i)
        o = StreamYoloOracle(cfg, {k: v.detach().clone() for k, v in model.state_dict().items()})
        with torch.no_grad():
            ref = o.forward(x, tg)
        got = tr.step(x, tg)
        for k in ("total_loss", "iou_loss", "l1_loss", "conf_loss", "cls_loss"):
            assert abs(float(got[k]) - float(ref[k])) <= 2e-5 * abs(float(ref[k])) + 1e-6, (i, (h, w), k)
        assert float(got["num_fg"]) == float(ref["num_fg"])
    assert tr.updates == 3


@pytest.mark.parametrize("still", [False, True], ids=["pair", "still"])
def test_preprocess_is_the_cfg_preprocess(still, monkeypatch):
    """data.preprocess (resize into the static input, labels copied then rescaled) == the cfgs' Exp.preprocess
    (F.interpolate + in-place label scaling of targets[0] and targets[1]); at input_size nothing runs"""
    emul_ops.install(monkeypatch, exact=True)
    b, inp = 3, (120, 192)
    x = synth.synth_frames(b, *inp)[:, :3 if still else 6].contiguous()
    fut, cur = synth.synth_labels(b, *inp)
    labels = fut.clone() if still else (fut.clone(), cur.clone())
    orig = fut.clone() if still else (fut.clone(), cur.clone())

    def reference(x, targets, tsize):          # cfgs/s_s50_onex_dfp_tal_flip.py:160-171
        scale_y, scale_x = tsize[0] / inp[0], tsize[1] / inp[1]
        if scale_x != 1 or scale_y != 1:
            x = F.interpolate(x, size=tsize, mode="bilinear", align_corners=False)
            targets[0][..., 1::2] = targets[0][..., 1::2] * scale_x
            targets[0][..., 2::2] = targets[0][..., 2::2] * scale_y
            targets[1][..., 1::2] = targets[1][..., 1::2] * scale_x
            targets[1][..., 2::2] = targets[1][..., 2::2] * scale_y
        return x, targets

    for size in ((96, 160), (128, 224)):
        want_x, want_l = reference(x.clone(), orig.clone() if still else tuple(t.clone() for t in orig), size)
        out = (torch.full((b, x.shape[1]) + size, float("nan")),
               torch.full_like(fut, float("nan")) if still else tuple(torch.full_like(fut, float("nan")) for _ in range(2)))
        got_x, got_l = data.preprocess(x, labels, size, inp, out=out)
        assert got_x is out[0] and got_l is out[1]
        assert torch.allclose(got_x, want_x, rtol=1e-5, atol=1e-5)
        for g, w_ in zip([got_l] if still else got_l, [want_l] if still else want_l):
            assert torch.allclose(g, w_, rtol=1e-5, atol=1e-5)
        if still:                                   # the cfg rescales images 0 and 1 of a single label tensor only
            assert torch.equal(got_l[2], orig[2]) and not torch.equal(got_l[0], orig[0])
        for g, o in zip([labels] if still else labels, [orig] if still else orig):
            assert torch.equal(g, o)                # the source labels are left as they were
        # without out: the labels are scaled in place, as the cfg does
        src = orig.clone() if still else tuple(t.clone() for t in orig)
        got_x2, got_l2 = data.preprocess(x, src, size, inp)
        assert got_l2 is src and torch.allclose(got_x2, want_x, rtol=1e-5, atol=1e-5)
    same_x, same_l = data.preprocess(x, labels, inp, inp, out=out)
    assert same_x is x and same_l is labels


# ------------------------------------------------------------------------------------------------ GPU
def _bn_buffers(model):
    return {k: v.clone() for k, v in model.state_dict().items() if "running_" in k or "num_batches_tracked" in k}


def _snapshot(tr):
    return (tr.fs.state.clone(), tr.fs.mom.clone(), tr.fs.ema.clone(), _bn_buffers(tr.model), tr.updates)


def _assert_same(a, b, what):
    assert torch.equal(a[0], b[0]), f"{what}: fs.state"
    assert torch.equal(a[1], b[1]), f"{what}: fs.mom"
    assert torch.equal(a[2], b[2]), f"{what}: fs.ema"
    assert a[3].keys() == b[3].keys()
    for k in a[3]:
        assert torch.equal(a[3][k], b[3][k]), f"{what}: {k}"
    assert a[4] == b[4], f"{what}: updates"


class _Inputs:
    """the static uint8 batch of a graphed loop and the per-size prologue: pair_transform / frame_transform into a staging
    buffer at input_size, then Exp.preprocess into the size's static input (at input_size the staging buffer is it).  The
    resized inputs of all other sizes are views of ONE buffer of the largest size: only one size graph runs at a time, and
    each writes its input before it reads it."""

    def __init__(self, b, input_size, still, dev, sizes, seed=1):
        self.b, self.input_size, self.still, self.dev = b, tuple(input_size), still, dev
        self.static = [t.to(dev) for t in synth.synth_uint8_pairs(b, *input_size, seed=seed)]
        if still:
            self.static = self._still(self.static)
        self.c = 3 if still else 6
        self.stage = self._buffers(self.input_size)
        self.shared = torch.empty(b * self.c * max(h * w for h, w in sizes), dtype=torch.float32, device=dev)

    @staticmethod
    def _still(batch):
        frames, ann, counts, mirror = batch
        return [frames[:, 0].contiguous(), ann[:, 0].contiguous(), counts[:, 0].contiguous(), mirror]

    def _buffers(self, size, x=None):
        if x is None:
            x = torch.empty((self.b, self.c) + tuple(size), dtype=torch.float32, device=self.dev)
        if self.still:
            return x, torch.empty((self.b, MAX_LABELS, 5), dtype=torch.float32, device=self.dev)
        return x, tuple(torch.empty((self.b, MAX_LABELS, 5), dtype=torch.float32, device=self.dev) for _ in range(2))

    def load(self, seed):
        """copy a new uint8 batch into the static inputs (what a loop does before every replay)"""
        new = [t.to(self.dev) for t in synth.synth_uint8_pairs(self.b, *self.input_size, seed=seed)]
        for dst, src in zip(self.static, self._still(new) if self.still else new):
            dst.copy_(src)

    def make_inputs(self, size):
        if tuple(size) == self.input_size:
            return self.stage
        return self._buffers(size, self.shared[:self.b * self.c * size[0] * size[1]].view((self.b, self.c) + tuple(size)))

    def prologue(self, size, x, targets):
        frames, ann, counts, mirror = self.static
        fn = data.frame_transform if self.still else data.pair_transform
        fn(frames, ann, counts, mirror, self.input_size, max_labels=MAX_LABELS, out=self.stage)
        data.preprocess(self.stage[0], self.stage[1], size, self.input_size, out=(x, targets))

    def eager(self, size):
        """the same inputs built eagerly into fresh tensors"""
        frames, ann, counts, mirror = self.static
        fn = data.frame_transform if self.still else data.pair_transform
        x, labels = fn(frames, ann, counts, mirror, self.input_size, max_labels=MAX_LABELS)
        return data.preprocess(x, labels, size, self.input_size)


def _graph_equals_eager(build, sizes, input_size, b, still, steps=12, seed=7):
    dev = torch.device("cuda")
    rng = random.Random(seed)
    seq = [sizes[0], sizes[-1]] + [rng.choice(sizes) for _ in range(steps - 2)]       # revisits sizes, random order
    assert len(set(seq)) >= min(3, len(sizes))
    lrs = [1e-4 * (1 + 0.1 * i) for i in range(steps)]
    inp = _Inputs(b, input_size, still, dev, sizes)
    a = build()
    ta = train.Trainer(a, lr=1e-4)
    want = []
    for i, (s, lr) in enumerate(zip(seq, lrs)):
        inp.load(100 + i)
        x, tg = inp.eager(s)
        want.append(float(ta.step(x, tg, lr=lr)["total_loss"]))
    torch.cuda.synchronize()
    del inp
    inp = _Inputs(b, input_size, still, dev, sizes)
    m = build()
    tb = train.Trainer(m, lr=1e-4)
    before = _snapshot(tb)
    tb.capture_sizes(sizes, inp.make_inputs, inp.prologue)
    torch.cuda.synchronize()
    _assert_same(_snapshot(tb), before, "after capture_sizes")
    got = []
    for i, (s, lr) in enumerate(zip(seq, lrs)):
        inp.load(100 + i)
        got.append(float(tb.replay_size(s, lr=lr)["total_loss"]))
    torch.cuda.synchronize()
    assert got == want, (seq, got, want)
    _assert_same(_snapshot(tb), _snapshot(ta), "after the steps")
    return seq


TINY_SIZES = train.multiscale_sizes((120, 192), (10, 14))        # 96x160 .. 128x224 and 120x192; 112x192: 7x12 at stride 16


@pytest.mark.gpu
def test_graph_equals_eager_sizes_interleaved_tiny():
    from test_gpu_model import build_product
    c = CASES["tiny_120x160"]
    seq = _graph_equals_eager(lambda: build_product(c["depth"], c["width"]).train(), TINY_SIZES, (120, 192), 2, False)
    assert (120, 192) in seq


@pytest.mark.gpu
def test_graph_equals_eager_sizes_interleaved_s():
    """StreamYOLO-s at the extreme sizes and input_size, 2 pairs"""
    from test_gpu_parity_fwd import _build
    _graph_equals_eager(lambda: _build("s"), [(496, 800), (688, 1120), (600, 960)], (600, 960), 2, False)


@pytest.mark.gpu
def test_graph_equals_eager_sizes_interleaved_still():
    """the still model (PIPEHead, [B, 3, H, W], one label tensor, stat_updates = 2) through frame_transform"""
    from test_gpu_still import build_still
    c = CASES["tiny_120x160"]
    _graph_equals_eager(lambda: build_still(c["depth"], c["width"]), TINY_SIZES, (120, 192), 3, True)


@pytest.mark.gpu
def test_capture_sizes_has_no_side_effects_after_training():
    """capture in the middle of training (momentum, EMA and updates no longer at their initial values), all 22 sizes of
    the tiny model's scaled set twice over: the state is bit-identical before and after, and a second capture_sizes
    replaces the first"""
    from test_gpu_model import build_product
    c = CASES["tiny_120x160"]
    dev = torch.device("cuda")
    m = build_product(c["depth"], c["width"]).train()
    tr = train.Trainer(m, lr=1e-4)
    x = synth.synth_frames(2, 120, 192).cuda()
    tg = tuple(t.cuda() for t in synth.synth_labels(2, 120, 192))
    for _ in range(3):
        tr.step(x, tg)
    sizes = train.multiscale_sizes((120, 192), (10, 30))
    assert len(sizes) == 22
    inp = _Inputs(2, (120, 192), False, dev, sizes)
    before = _snapshot(tr)
    assert before[4] == 3 and bool(before[1].abs().sum() > 0)
    segments = tr.capture_sizes(sizes, inp.make_inputs, inp.prologue)
    torch.cuda.synchronize()
    assert set(segments) == set(sizes) and set(segments.values()) == {1}
    _assert_same(_snapshot(tr), before, "after capture_sizes")
    tr.capture_sizes(sizes[:3], inp.make_inputs, inp.prologue)
    torch.cuda.synchronize()
    _assert_same(_snapshot(tr), before, "after a second capture_sizes")
    with pytest.raises(KeyError, match="no graph captured"):
        tr.replay_size(sizes[5])


@pytest.mark.gpu
@pytest.mark.parametrize("size", [(496, 800), (688, 1120)], ids=["496x800", "688x1120"])
def test_every_launch_at_the_extreme_sizes_l(size):
    """StreamYOLO-l, 2 pairs, at the smallest and largest multi-scale size: every conv launch of the recording forward
    (FwdChecker) and every recorded conv's backward in situ (run_walk_checked) against float64, with the bars used at
    600x960"""
    from test_gpu_parity_bwd import run_walk_checked
    from test_gpu_parity_fwd import FwdChecker, _build, conv_launches
    from streamyolo_b200.model import backward
    h, w = size
    m = _build("l")
    x = synth.synth_frames(2, h, w, seed=4321).cuda()
    tg = tuple(t.cuda() for t in synth.synth_labels(2, h, w, seed=11))
    with torch.no_grad():
        m(x, tg)
    with FwdChecker(m) as ck:
        _, loss = backward._record(m, x, tg)
    launches = conv_launches(m, jian_twice=True)
    assert launches == 117
    assert ck.n == Counter(conv=launches, apply=launches, head=3, focus=1, mean_invstd=launches), ck.n
    assert bool(torch.isfinite(loss).all())
    print(f"\nFWD l recording b2 {h}x{w}: worst " + ", ".join(f"{k} {v:.3g}" for k, v in sorted(ck.worst.items())))
    seen = run_walk_checked(_build("l"), x, tg)
    assert len(seen) == 116, len(seen)


# Measured on an H100 80GB HBM3 at 700 W (tools/bench_multiscale.py, profiles/h100_multiscale.txt; this test: 1.002):
# max_memory_reserved after capturing all 22 sizes of StreamYOLO-s at 8 pairs is MEASURED_RATIO x that of capturing the
# largest size alone.  One pool per size would hold the intermediates of every size at once.
MEASURED_RATIO = 1.0017
BOUND = 1.1


@pytest.mark.gpu
def test_memory_of_all_sizes_s():
    from test_gpu_parity_fwd import _build
    dev = torch.device("cuda")
    sizes = train.multiscale_sizes()
    largest = max(sizes, key=lambda s: s[0] * s[1])
    peaks = []
    for subset in ([largest], sizes):
        gc.collect()
        torch.cuda.synchronize()
        torch.cuda.empty_cache()
        torch.cuda.reset_peak_memory_stats()
        inp = _Inputs(8, (600, 960), False, dev, subset)
        tr = train.Trainer(_build("s"), lr=1e-4)
        tr.capture_sizes(subset, inp.make_inputs, inp.prologue)
        loss = tr.replay_size(sizes[0] if subset is sizes else largest)["total_loss"]
        torch.cuda.synchronize()
        assert bool(torch.isfinite(loss))
        peaks.append(torch.cuda.max_memory_reserved())
        del tr, inp
    ratio = peaks[1] / peaks[0]
    print(f"\nmax_memory_reserved: largest only {peaks[0] / 2 ** 30:.3f} GiB, all 22 sizes {peaks[1] / 2 ** 30:.3f} GiB, "
          f"ratio {ratio:.3f}")
    assert ratio <= BOUND, (ratio, MEASURED_RATIO)
