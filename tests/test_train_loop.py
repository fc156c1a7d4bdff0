"""The reference trainer's loop on the device (streamyolo_b200/train_loop.py, dropin.install(trainer=True)) and the
non-finite gradient skip (sy_nonfinite_flag, the step's skip-with-EMA mode, train.Trainer(skip_nonfinite=True)).

yolox is not installable here, so the module below stands in for what the reference trainer's module imports from it
(logger, save_checkpoint, load_ckpt, ...), for yolox's InfiniteSampler / YoloBatchSampler / MeterBuffer / yoloxwarmcos
scheduler, and for an Exp and its dataset table; its ``Trainer`` has the attributes the reference ``Trainer.__init__``
sets.

CPU: the orchestration with a stand-in device step (batches, files, labels, mirror bits, lrs, random_resize, log lines,
checkpoints, the evaluated model, the refusals, install), and the skip-with-EMA arithmetic with the kernel emulated.
GPU: the kernel on planted values inside a graph, the skip in a captured step, and the whole loop bit-identical to the
hand-wired capture_sizes loop of INTEGRATION.md for the onex, twox and still layouts, resume and a damaged file.
Two ranks cannot run on one GPU; the per-rank batches are checked on the CPU only."""
import contextlib
import itertools
import math
import os
import sys
import types
from collections import defaultdict, deque

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import emul_ops  # noqa: E402
from oracle.make_golden import CASES  # noqa: E402
from streamyolo_b200 import data, dropin, ops, train, train_loop  # noqa: E402
from streamyolo_b200 import synth  # noqa: E402

TINY = CASES["tiny_120x160"]


# ------------------------------------------------------------------------------------------------ yolox stand-ins
class InfiniteSampler:
    """[yolox 0.3.0] yolox/data/samplers.py InfiniteSampler"""

    def __init__(self, size, shuffle=True, seed=0, rank=0, world_size=1):
        self._size, self._shuffle, self._seed = size, shuffle, int(seed)
        self._rank, self._world_size = rank, world_size

    def __iter__(self):
        yield from itertools.islice(self._infinite_indices(), self._rank, None, self._world_size)

    def _infinite_indices(self):
        g = torch.Generator()
        g.manual_seed(self._seed)
        while True:
            if self._shuffle:
                yield from torch.randperm(self._size, generator=g)
            else:
                yield from torch.arange(self._size)

    def __len__(self):
        return self._size // self._world_size


class YoloBatchSampler(torch.utils.data.sampler.BatchSampler):
    """[yolox 0.3.0] YoloBatchSampler: (mosaic, index) pairs"""

    def __init__(self, *args, mosaic=True, **kwargs):
        super().__init__(*args, **kwargs)
        self.mosaic = mosaic

    def __iter__(self):
        for batch in super().__iter__():
            yield [(self.mosaic, idx) for idx in batch]


class AverageMeter:
    def __init__(self, window_size=50):
        self._deque = deque(maxlen=window_size)
        self._total, self._count = 0.0, 0

    def update(self, value):
        self._deque.append(value)
        self._count += 1
        self._total += value

    @property
    def avg(self):
        return np.mean(np.array(list(self._deque)))

    @property
    def global_avg(self):
        return self._total / max(self._count, 1e-5)

    @property
    def latest(self):
        return self._deque[-1] if len(self._deque) > 0 else None

    def clear(self):
        self._deque.clear()


class MeterBuffer(defaultdict):
    def __init__(self, window_size=20):
        factory = lambda: AverageMeter(window_size=window_size)  # noqa: E731
        super().__init__(factory)

    def get_filtered_meter(self, filter_key="time"):
        return {k: v for k, v in self.items() if filter_key in k}

    def update(self, values=None, **kwargs):
        values = dict(values or {}, **kwargs)
        for k, v in values.items():
            if isinstance(v, torch.Tensor):
                v = v.detach()
            self[k].update(v)

    def clear_meters(self):
        for v in self.values():
            v.clear()


def yolox_warm_cos_lr(lr, min_lr_ratio, total_iters, warmup_total_iters, warmup_lr_start, no_aug_iter, iters):
    min_lr = lr * min_lr_ratio
    if iters <= warmup_total_iters:
        lr = (lr - warmup_lr_start) * pow(iters / float(warmup_total_iters), 2) + warmup_lr_start
    elif iters >= total_iters - no_aug_iter:
        lr = min_lr
    else:
        lr = min_lr + 0.5 * (lr - min_lr) * (1.0 + math.cos(math.pi * (iters - warmup_total_iters)
                                                          / (total_iters - warmup_total_iters - no_aug_iter)))
    return lr


class LRScheduler:
    """[yolox 0.3.0] LRScheduler("yoloxwarmcos", ...)"""

    def __init__(self, lr, iters_per_epoch, total_epochs, warmup_epochs, warmup_lr_start, no_aug_epochs, min_lr_ratio):
        self.args = (lr, min_lr_ratio, iters_per_epoch * total_epochs, iters_per_epoch * warmup_epochs, warmup_lr_start,
                     iters_per_epoch * no_aug_epochs)

    def update_lr(self, iters):
        return yolox_warm_cos_lr(*self.args, iters)


class Log:
    def __init__(self):
        self.lines = []

    def info(self, msg):
        self.lines.append(str(msg))


def save_checkpoint(state, is_best, save_dir, model_name=""):
    os.makedirs(save_dir, exist_ok=True)
    torch.save(state, os.path.join(save_dir, model_name + "_ckpt.pth"))
    if is_best:
        torch.save(state, os.path.join(save_dir, "best_ckpt.pth"))


@contextlib.contextmanager
def adjust_status(module, training=False):
    status = {}
    for m in module.modules():
        status[m] = m.training
        m.training = training
    yield module
    for m in module.modules():
        m.training = status[m]


class SummaryWriter:
    def __init__(self, log_dir):
        self.scalars = []

    def add_scalar(self, tag, value, step):
        self.scalars.append((tag, value, step))


def helpers_module(monkeypatch, name="fake_double_trainer"):
    """the reference trainer's module namespace, registered in sys.modules for the test"""
    mod = types.ModuleType(name)
    mod.logger, mod.save_checkpoint, mod.adjust_status = Log(), save_checkpoint, adjust_status
    mod.load_ckpt = lambda model, ckpt: (model.load_state_dict(ckpt, strict=False), model)[1]
    mod.gpu_mem_usage = lambda: 1234.0
    mod.synchronize = lambda: None
    mod.occupy_mem = lambda rank: None
    mod.SummaryWriter = SummaryWriter
    monkeypatch.setitem(sys.modules, name, mod)

    class Trainer:                          # double_trainer.py:37-72 (the logger setup and GradScaler left out)
        def __init__(self, exp, args):
            self.exp, self.args = exp, args
            self.max_epoch = exp.max_epoch
            self.amp_training = args.fp16
            self.is_distributed = exp.world > 1
            self.rank, self.local_rank = exp.rank, 0
            self.device = exp.device
            self.use_model_ema = exp.ema
            self.save_history_ckpt = exp.save_history_ckpt
            self.data_type = torch.float16 if args.fp16 else torch.float32
            self.input_size = exp.input_size
            self.best_ap = 0
            self.meter = MeterBuffer(window_size=exp.print_interval)
            self.file_name = os.path.join(exp.output_dir, args.experiment_name)
            if self.rank == 0:
                os.makedirs(self.file_name, exist_ok=True)

        def before_iter(self):
            pass

        def after_train(self):
            mod.logger.info("Training of experiment is done and the best AP is {:.2f}".format(self.best_ap * 100))

    Trainer.__module__ = name
    mod.Trainer = Trainer
    return mod


# ------------------------------------------------------------------------------------------------ dataset and Exp
class DoubleTrainTransform:
    def __init__(self, max_labels=50, hsv=True, flip=True):
        self.max_labels = max_labels
        self.trasform1 = types.SimpleNamespace(max_labels=max_labels, hsv=hsv, flip=flip)
        self.trasform2 = types.SimpleNamespace(max_labels=max_labels, hsv=hsv, flip=flip)


class TrainTransform:
    def __init__(self, max_labels=50, hsv=True, flip=True):
        self.max_labels, self.hsv, self.flip = max_labels, hsv, flip


def make_table(root, n, layout, hw=(120, 192), seed=0, jpeg=False, max_rows=7, input_size=(120, 192)):
    """n annotation entries in the reference's layout, the labels scaled into ``input_size`` as ``load_anno_from_ids``
    does; the files are random bytes, or with ``jpeg`` cv2-encoded h x w frames"""
    rng = np.random.default_rng(seed)
    os.makedirs(root, exist_ok=True)
    frames = 1 if layout == "still" else 2
    h, w = hw
    r = min(input_size[0] / h, input_size[1] / w)
    out = []
    for i in range(n):
        paths, labels = [], []
        for f in range(frames):
            p = os.path.join(root, f"{i:04d}_{f}.jpg")
            if jpeg:
                import cv2
                img = (rng.integers(0, 256, (h // 8, w // 8, 3), dtype=np.uint8).repeat(8, 0).repeat(8, 1))
                ok, buf = cv2.imencode(".jpg", img, [cv2.IMWRITE_JPEG_QUALITY, 90])
                assert ok
                buf.tofile(p)
            else:
                rng.integers(0, 256, int(rng.integers(100, 9000)), dtype=np.uint8).tofile(p)
            paths.append(p)
            k = int(rng.integers(0, max_rows + 1))
            x1 = rng.uniform(0, w * 0.6, k)
            y1 = rng.uniform(0, h * 0.6, k)
            res = np.stack([x1, y1, x1 + rng.uniform(6, w * 0.4, k), y1 + rng.uniform(6, h * 0.4, k),
                            rng.integers(0, 8, k).astype(np.float64)], 1) if k else np.zeros((0, 5))
            res[:, :4] *= r
            labels.append(res)
        if frames == 2:
            out.append((labels[0], labels[1], (h, w), (int(h * r), int(w * r)), paths[0], paths[1]))
        else:
            out.append((labels[0], (h, w), (int(h * r), int(w * r)), paths[0]))
    return out


class Loader:
    """what the loop reads of yolox's DataLoader: dataset (the MosaicDetection wrapper), batch_sampler, len, close_mosaic"""

    def __init__(self, dataset, batch_sampler):
        self.dataset, self.batch_sampler = dataset, batch_sampler
        self.closed = 0

    def __len__(self):
        return len(self.batch_sampler)

    def __iter__(self):
        raise AssertionError("the device loop must not iterate the DataLoader")

    def close_mosaic(self):
        self.batch_sampler.mosaic = False
        self.closed += 1


class Evaluator:
    def __init__(self):
        self.calls = []

    def evaluate(self, model, distributed=False, half=False):
        self.calls.append({"model": model, "training": model.training,
                           "state": {k: v.detach().clone() for k, v in model.state_dict().items()}})
        ap = [0.3, 0.2, 0.4, 0.1][len(self.calls) - 1]
        return ap, ap + 0.1, f"summary {len(self.calls)}"


class Exp:
    """the yolox Exp attributes and methods the loop calls, with the shipped cfgs' values where they matter"""

    def __init__(self, table, layout, out, batch=2, max_epoch=2, world=1, rank=0, device="cpu", build=None,
                 input_size=(120, 192), random_size=(10, 14), print_interval=3, ema=True, hsv=False, seed=None):
        self.table, self.layout, self.output_dir = table, layout, out
        self.batch, self.world, self.rank, self.device = batch, world, rank, device
        self.max_epoch, self.no_aug_epochs, self.warmup_epochs = max_epoch, max_epoch, 1
        self.eval_interval, self.print_interval = 10, print_interval
        self.input_size, self.test_size, self.random_size = input_size, input_size, random_size
        self.basic_lr_per_img, self.warmup_lr, self.min_lr_ratio = 0.001 / 64.0, 0, 0.05
        self.momentum, self.weight_decay, self.ema, self.save_history_ckpt = 0.9, 5e-4, ema, True
        self.hsv, self.seed, self.exp_name = hsv, seed, "tiny"
        self.build, self.model = build, None
        self.resizes, self.evaluator = [], Evaluator()
        self.draw = np.random.default_rng(5)

    def get_model(self):
        if self.model is None:
            self.model = self.build()
        return self.model

    def get_optimizer(self, batch_size):            # [yolox] Exp.get_optimizer: the first lr is warmup_lr
        lr = self.warmup_lr if self.warmup_epochs > 0 else self.basic_lr_per_img * batch_size
        return train.build_optimizer(self.model, lr, self.momentum, self.weight_decay)

    def get_data_loader(self, batch_size, is_distributed, no_aug=False, local_rank=0, cache_img=False):
        pre = (TrainTransform if self.layout == "still" else DoubleTrainTransform)(max_labels=5, hsv=self.hsv, flip=True)
        inner = types.SimpleNamespace(annotations=self.table)
        dataset = types.SimpleNamespace(_dataset=inner, preproc=pre)
        if is_distributed:
            batch_size = batch_size // self.world
        sampler = InfiniteSampler(len(self.table), seed=self.seed if self.seed else 0, rank=self.rank,
                                  world_size=self.world)
        self.loader = Loader(dataset, YoloBatchSampler(sampler=sampler, batch_size=batch_size, drop_last=False,
                                                       mosaic=not no_aug))
        return self.loader

    def get_lr_scheduler(self, lr, iters_per_epoch):
        return LRScheduler(lr, iters_per_epoch, self.max_epoch, self.warmup_epochs, self.warmup_lr, self.no_aug_epochs,
                           self.min_lr_ratio)

    def get_evaluator(self, batch_size, is_distributed, testdev=False):
        return self.evaluator

    def eval(self, model, evaluator, is_distributed, half=False):
        return evaluator.evaluate(model, is_distributed, half)

    def random_resize(self, data_loader, epoch, rank, is_distributed):
        if epoch >= self.max_epoch - 1:
            size = self.input_size
        else:
            f = self.input_size[0] * 1.0 / self.input_size[1]
            s = int(self.draw.integers(self.random_size[0], self.random_size[1] + 1))
            size = (16 * int(s * f), int(16 * s))
        self.resizes.append((epoch, size))
        return size


def args_for(**kw):
    a = dict(batch_size=4, fp16=False, cache=False, occupy=False, logger="tensorboard", opts=[], resume=False, ckpt=None,
             start_epoch=None, experiment_name="run")
    a.update(kw)
    return types.SimpleNamespace(**a)


class FakeStep:
    """stand-in for train_loop.DeviceStep: host slots as plain arrays, every replay recorded"""
    log = None

    def __init__(self, tr, table, batch, input_size, sizes, max_bytes, device):
        self.tr, self.fpi, self.sizes = tr, table.frames, sizes
        n, R = batch * self.fpi, table.max_rows
        lab = (batch, self.fpi, R, 5) if self.fpi == 2 else (batch, R, 5)
        cnt = (batch, self.fpi) if self.fpi == 2 else (batch,)
        self.host = [{"bytes": np.zeros((n, max_bytes), np.uint8), "lengths": np.zeros(n, np.int32),
                      "ann": np.zeros(lab), "counts": np.zeros(cnt, np.int32), "mirror": np.zeros(batch, np.int32)}
                     for _ in range(2)]
        self.dev = [None, None]
        self.replays, self.losses, self.status = [], None, []
        self.bad = {}                                   # replay number -> status row
        FakeStep.log = self

    def slot_free(self, s):
        pass

    def h2d(self, s):
        self.dev[s] = {k: v.copy() for k, v in self.host[s].items()}

    def capture(self, s):
        self.captured = (list(self.sizes), {k: v.copy() for k, v in self.dev[s].items()})

    def replay(self, s, size, lr):
        self.replays.append({"slot": self.dev[s], "size": tuple(size), "lr": lr})
        self.tr.updates += 1
        self.tr.fs.ema.mul_(0.5)                        # the EMA copy now differs from the live weights
        k = len(self.replays)
        self.losses = {"total_loss": torch.tensor(10.0 + k), "iou_loss": torch.tensor(2.0), "l1_loss": torch.tensor(1.0),
                       "conf_loss": torch.tensor(3.0 + k), "cls_loss": torch.tensor(4.0), "num_fg": torch.tensor(5.0)}
        self.status.append(self.bad.get(k - 1, np.zeros(len(self.dev[s]["lengths"]), np.int32)))
        return self.losses

    def sync(self, pending):
        return self.status[-pending:]

    def close(self):
        pass


def tiny_build():
    from test_cpu_backward import build_product
    return build_product(TINY)


def run_loop(tmp_path, monkeypatch, layout="onex", n=13, world=1, rank=0, max_epoch=2, args=None, exp_kw=None,
             step=FakeStep, table=None, max_bytes=None):
    emul_ops.install(monkeypatch, exact=True)
    mod = helpers_module(monkeypatch)
    cls = train_loop.device_trainer(mod.Trainer)
    cls.step_class, cls.max_bytes = step, max_bytes
    table = make_table(str(tmp_path / "data"), n, layout) if table is None else table
    exp = Exp(table, layout, str(tmp_path / "out"), world=world, rank=rank, max_epoch=max_epoch, build=tiny_build,
              **(exp_kw or {}))
    t = cls(exp, args or args_for(batch_size=2 * world))
    t.train()
    return t, exp, mod, FakeStep.log


# ------------------------------------------------------------------------------------------------ CPU
@pytest.mark.parametrize("world", [1, 2])
def test_batches_follow_the_batch_sampler_across_epochs(tmp_path, monkeypatch, world):
    """the indices of every replay are what one iterator over the loader's own batch_sampler yields, across the epoch
    boundary, per rank; the loader itself is never iterated"""
    for rank in range(world):
        t, exp, _, log = run_loop(tmp_path / f"r{rank}", monkeypatch, world=world, rank=rank)
        assert t.max_iter == len(exp.loader) == (13 // world + 1) // 2
        assert len(log.replays) == 2 * t.max_iter
        fresh = iter(YoloBatchSampler(sampler=InfiniteSampler(13, rank=rank, world_size=world), batch_size=2,
                                      drop_last=False, mosaic=False))
        want = [[int(i) for _, i in next(fresh)] for _ in range(2 * t.max_iter)]
        assert [_indices_of(r["slot"], exp.table, 2) for r in log.replays] == want
        assert exp.loader.closed == 2                           # before_epoch's close_mosaic, once per epoch


def _indices_of(slot, table, fpi):
    """dataset indices of a slot, found from the bytes of its first frame"""
    out = []
    for b in range(slot["mirror"].shape[0]):
        n = int(slot["lengths"][b * fpi])
        row = slot["bytes"][b * fpi, :n]
        hit = [i for i, a in enumerate(table) if np.array_equal(np.fromfile(a[4] if fpi == 2 else a[3], np.uint8), row)]
        assert len(hit) == 1
        out.append(hit[0])
    return out


@pytest.mark.parametrize("layout", ["onex", "still"])
def test_slots_hold_the_annotation_entries(tmp_path, monkeypatch, layout):
    """bytes and lengths are the files, the labels are the annotation rows zero-padded, counts their lengths; mirror bits
    are 0 / 1 for pairs (both values drawn) and 0 for still"""
    t, exp, _, log = run_loop(tmp_path, monkeypatch, layout=layout, n=9, max_epoch=3)
    fpi = 1 if layout == "still" else 2
    mirrors = []
    for r in log.replays:
        s = r["slot"]
        for b, i in enumerate(_indices_of(s, exp.table, fpi)):
            a = exp.table[i]
            files = (a[4], a[5]) if fpi == 2 else (a[3],)
            labels = (a[0], a[1]) if fpi == 2 else (a[0],)
            for f in range(fpi):
                want = np.fromfile(files[f], np.uint8)
                assert s["lengths"][b * fpi + f] == want.size
                assert np.array_equal(s["bytes"][b * fpi + f, :want.size], want)
                ann = s["ann"][b, f] if fpi == 2 else s["ann"][b]
                cnt = s["counts"][b, f] if fpi == 2 else s["counts"][b]
                assert cnt == len(labels[f])
                assert np.array_equal(ann[:cnt], labels[f])
                assert not ann[cnt:].any()
        mirrors += s["mirror"].tolist()
    assert set(mirrors) == ({0} if layout == "still" else {0, 1})


def _reference_lrs(exp, max_iter, start_epoch, first):
    """the lr the reference's optimizer holds at every iteration: ``first`` at the first, then update_lr(progress + 1)"""
    sched = exp.get_lr_scheduler(exp.basic_lr_per_img * 2, max_iter)
    out, lr = [], first
    for p in range(start_epoch * max_iter, exp.max_epoch * max_iter):
        out.append(lr)
        lr = sched.update_lr(p + 1)
    return out


def test_lrs_sizes_and_random_resize(tmp_path, monkeypatch):
    """every replay's lr is the reference loop's (warmup_lr = 0 first); random_resize every 10 progress iterations, and
    each replay runs at the size in force"""
    t, exp, _, log = run_loop(tmp_path, monkeypatch, n=24, max_epoch=2)
    assert t.max_iter == 12
    assert [r["lr"] for r in log.replays] == _reference_lrs(exp, 12, 0, 0)
    assert [e for e, _ in exp.resizes] == [0, 1]                # progress 9 (epoch 0) and 19 (epoch 1)
    sizes = [r["size"] for r in log.replays]
    assert sizes[:10] == [(120, 192)] * 10
    assert sizes[10:20] == [exp.resizes[0][1]] * 10 and sizes[20:] == [exp.resizes[1][1]] * 4
    assert log.captured[0] == train.multiscale_sizes((120, 192), (10, 14))


def test_log_lines_have_the_reference_format(tmp_path, monkeypatch):
    t, exp, mod, log = run_loop(tmp_path, monkeypatch, n=12, max_epoch=1)
    lines = [ln for ln in mod.logger.lines if ln.startswith("epoch: ")]
    assert len(lines) == 2                                      # iterations 3 and 6 of 6
    import re
    pat = (r"epoch: 1/1, iter: (\d+)/6, mem: 1234Mb, iter_time: \d+\.\d{3}s, data_time: \d+\.\d{3}s, "
           r"total_loss: (\d+\.\d), iou_loss: 2\.0, l1_loss: 1\.0, conf_loss: (\d+\.\d), cls_loss: 4\.0, "
           r"lr: \d\.\d{3}e[-+]\d\d, size: 120, ETA: \d+:\d\d:\d\d$")
    for ln, it in zip(lines, (3, 6)):
        m = re.match(pat, ln)
        assert m, ln
        assert int(m.group(1)) == it and float(m.group(2)) == 10.0 + it and float(m.group(3)) == 3.0 + it
    lr3 = _reference_lrs(exp, 6, 0, 0)[3]
    assert "lr: {:.3e}".format(lr3) in lines[0]


def test_checkpoints_and_the_evaluated_model(tmp_path, monkeypatch):
    """latest / last_epoch / epoch_N every epoch, best when the AP improves, all with the reference's keys and the EMA
    weights; the evaluator gets an eval-mode copy holding the EMA weights, never the training model"""
    t, exp, mod, log = run_loop(tmp_path, monkeypatch, n=8, max_epoch=3)
    d = t.file_name
    assert sorted(os.listdir(d)) == ["best_ckpt.pth", "epoch_1_ckpt.pth", "epoch_2_ckpt.pth", "epoch_3_ckpt.pth",
                                     "last_epoch_ckpt.pth", "latest_ckpt.pth"]
    last = torch.load(os.path.join(d, "last_epoch_ckpt.pth"))
    assert set(last) == {"start_epoch", "model", "optimizer", "best_ap"}
    assert last["start_epoch"] == 3 and last["best_ap"] == pytest.approx(0.4)
    best = torch.load(os.path.join(d, "best_ckpt.pth"))
    assert best["start_epoch"] == 3                             # APs 0.3, 0.2, 0.4: epochs 1 and 3 improved
    ema = t.tr.ema_state_dict()
    for k, v in last["model"].items():
        assert torch.equal(v, ema[k]), k
    assert len(exp.evaluator.calls) == 3
    live = t.model.state_dict()
    for c in exp.evaluator.calls:
        assert c["model"] is t.eval_model and c["model"] is not t.model and not c["training"]
    assert t.eval_model.training                                # adjust_status restored it
    for k, v in exp.evaluator.calls[-1]["state"].items():
        assert torch.equal(v, ema[k]), k
    assert any(not torch.equal(live[k], ema[k]) for k in ema if ema[k].dtype.is_floating_point)
    assert t.tr.updates == 3 * t.max_iter


def test_resume_sets_updates_lr_and_epoch(tmp_path, monkeypatch):
    """--resume: load_reference_checkpoint with max_iter * start_epoch, the checkpoint's lr first, best_ap; -e wins"""
    t, exp, _, _ = run_loop(tmp_path, monkeypatch, n=8, max_epoch=3)
    ckpt = os.path.join(t.file_name, "epoch_1_ckpt.pth")
    want_lr = torch.load(ckpt)["optimizer"]["param_groups"][0]["lr"]
    t2, exp2, _, log = run_loop(tmp_path / "b", monkeypatch, n=8, max_epoch=3, table=exp.table,
                                args=args_for(batch_size=2, resume=True, ckpt=ckpt))
    assert t2.start_epoch == 1 and len(log.replays) == 2 * t2.max_iter
    assert [r["lr"] for r in log.replays] == _reference_lrs(exp2, 4, 1, want_lr)
    assert t2.tr.updates == 3 * 4
    assert t2.best_ap == pytest.approx(0.3)                     # restored: the APs 0.3, 0.2 of this run improve nothing
    assert "best_ckpt.pth" not in os.listdir(t2.file_name)
    t3, _, _, log3 = run_loop(tmp_path / "c", monkeypatch, n=8, max_epoch=3, table=exp.table,
                              args=args_for(batch_size=2, resume=True, ckpt=ckpt, start_epoch=3))
    assert t3.start_epoch == 2 and len(log3.replays) == 4


def test_refusals(tmp_path, monkeypatch):
    with pytest.raises(NotImplementedError, match="no_aug_epochs"):
        _mosaic(tmp_path / "a", monkeypatch)
    with pytest.raises(NotImplementedError, match="hsv"):
        run_loop(tmp_path / "b", monkeypatch, n=6, exp_kw={"hsv": True})
    table = make_table(str(tmp_path / "c"), 4, "onex")
    table[2] = table[2][:2] + ((100, 160),) + table[2][3:]
    with pytest.raises(ValueError, match="one frame size"):
        run_loop(tmp_path / "c", monkeypatch, table=table)


def test_max_bytes_out_of_range_is_refused_before_the_step(tmp_path, monkeypatch):
    """a DeviceTrainer.max_bytes outside [4, 2^28] is refused when the feed starts, before a step is built or a file read"""
    FakeStep.log = None
    with pytest.raises(ValueError, match=r"DeviceTrainer: max_bytes must be an integer in \[4, 2\^28\], not 3"):
        run_loop(tmp_path, monkeypatch, n=6, max_bytes=3)
    assert FakeStep.log is None


def _mosaic(tmp_path, monkeypatch):
    emul_ops.install(monkeypatch, exact=True)
    mod = helpers_module(monkeypatch)
    cls = train_loop.device_trainer(mod.Trainer)
    cls.step_class = FakeStep
    exp = Exp(make_table(str(tmp_path), 6, "onex"), "onex", str(tmp_path / "out"), build=tiny_build)
    exp.no_aug_epochs = 1
    cls(exp, args_for(batch_size=2)).train()


def test_undecoded_frame_raises_at_the_next_sync_point(tmp_path, monkeypatch):
    class Bad(FakeStep):
        def __init__(self, *a):
            super().__init__(*a)
            self.bad = {4: np.array([0, 0, 0, 5], np.int32)}     # replay 5, frame 3: pair 1's support frame

    with pytest.raises(RuntimeError, match=r"dataset index (\d+) \(file .*_1\.jpg\) did not decode: corrupt"):
        run_loop(tmp_path, monkeypatch, n=30, max_epoch=1, step=Bad)
    assert len(FakeStep.log.replays) == 6                       # the print iteration 6 read the ring


def test_install_trainer(monkeypatch):
    mod = helpers_module(monkeypatch, "exps.train_utils.double_trainer")
    base = mod.Trainer
    monkeypatch.setitem(sys.modules, "yolox", types.ModuleType("yolox"))
    dropin.install()
    assert mod.Trainer is base                                  # the default install leaves the trainer alone
    dropin.install(trainer=True)
    first = mod.Trainer
    assert issubclass(first, train_loop.DeviceTrainer) and issubclass(first, base) and first.__name__ == "Trainer"
    dropin.install(trainer=True)
    dropin.install_trainer()
    assert mod.Trainer is first
    monkeypatch.setitem(sys.modules, "yolox", None)             # yolox not importable: nothing happens
    mod.Trainer = base
    dropin.install(trainer=True)
    assert mod.Trainer is base


def test_install_trainer_finds_an_exps_package_on_disk(tmp_path):
    """tools/train.py run from the reference checkout: ``exps`` is an importable package nobody has imported yet when
    install() runs.  It is imported and kept, so exps.train_utils.double_trainer is found and its Trainer replaced, and
    exps.model.* still resolve to this package."""
    import subprocess
    for d in ("exps", "exps/train_utils", "yolox"):
        os.makedirs(tmp_path / d, exist_ok=True)
        (tmp_path / d / "__init__.py").write_text("")
    (tmp_path / "exps" / "train_utils" / "double_trainer.py").write_text("class Trainer:\n    pass\n")
    code = ("import sys; assert 'exps' not in sys.modules; import streamyolo_b200.dropin as d; d.install(trainer=True);"
            "from exps.train_utils.double_trainer import Trainer; from streamyolo_b200.train_loop import DeviceTrainer;"
            "assert issubclass(Trainer, DeviceTrainer), Trainer; import exps; assert exps.__file__.startswith(sys.argv[1]);"
            "from exps.model.yolox import YOLOX; import streamyolo_b200.model as m; assert YOLOX is m.YOLOX; print('ok')")
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    env = dict(os.environ, PYTHONPATH=os.pathsep.join([str(tmp_path), root]))
    r = subprocess.run([sys.executable, "-c", code, str(tmp_path)], cwd=str(tmp_path), env=env, capture_output=True,
                       text=True)
    assert r.returncode == 0 and "ok" in r.stdout, r.stderr


def test_skip_with_ema_is_sgd_skipped_plus_model_ema_update(monkeypatch):
    """a flagged step: parameters and momentum as torch SGD leaves them when GradScaler skips it, the EMA as
    ModelEMA.update; a finite step with the guard as without it"""
    emul_ops.install(monkeypatch, exact=True)        # with sy_nonfinite_flag and the step's skip-with-EMA (found_inf_ema)
    from test_cpu_backward import build_product
    ref = build_product(TINY)
    opt = train.build_optimizer(ref, 0.01)
    ema = train.ModelEMA(ref)
    tr = train.Trainer(build_product(TINY), lr=0.01, skip_nonfinite=True)
    g = torch.randn(tr.fs.n_param, generator=torch.Generator().manual_seed(1)) * 1e-2
    for step, bad in enumerate([False, True, False, True]):
        grad = g * (step + 1)
        if bad:
            grad[len(grad) // 3] = float("nan") if step == 1 else float("-inf")
        for p, q in zip(ref.parameters(), tr.model.parameters()):
            o, n = tr.fs.offset[id(q)]
            p.grad = grad[o:o + n].view(p.shape).clone()
        if not bad:
            opt.step()
        ema.update(ref)
        tr.fs.grad.copy_(grad)
        tr.optimizer_step()
        for k, v in ref.state_dict().items():
            if v.dtype.is_floating_point:
                assert torch.equal(tr.model.state_dict()[k], v), (step, k)
        for k, v in ema.ema.state_dict().items():
            if v.dtype.is_floating_point:
                assert torch.equal(tr.ema_state_dict()[k], v), (step, k)
        for p, q in zip(ref.parameters(), tr.model.parameters()):
            o, n = tr.fs.offset[id(q)]
            assert torch.equal(tr.fs.mom[o:o + n].view(p.shape), opt.state[p]["momentum_buffer"]), step
    assert tr.updates == 4 and int(tr._skipped) == 2
    with pytest.raises(ValueError, match="found_inf"):         # the guard computes its own flag: no second one
        tr.optimizer_step(found_inf=torch.zeros(1))


# ------------------------------------------------------------------------------------------------ GPU
@pytest.mark.gpu
def test_nonfinite_flag_kernel_in_a_graph():
    """NaN, +inf and -inf at the first element, the last and mid-vector, n not a multiple of 4; FLT_MAX, -FLT_MAX and
    subnormals are finite; bad values in every block's range count once per launch.  Captured once, replayed twice per
    case: the flag is reset inside the graph, the counter counts flagged replays only."""
    dev = torch.device("cuda")
    n = 4 * 4000 + 3                                            # 16 blocks of 256 threads
    x = torch.randn(n, device=dev)
    flag = torch.full((1,), 7.0, device=dev)
    count = torch.zeros(1, dtype=torch.int32, device=dev)
    ops.nonfinite_flag(x, flag, count)                          # warm-up outside the graph
    torch.cuda.synchronize()
    assert float(flag) == 0.0 and int(count) == 0
    g = torch.cuda.CUDAGraph()
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        with torch.cuda.graph(g, stream=s):
            ops.nonfinite_flag(x, flag, count)
    base = x.clone()
    tiny = torch.tensor([1e-45, -1e-40, 1.1754942e-38], device=dev)
    finite = [(0, 3.4028234663852886e38), (n - 1, -3.4028234663852886e38), (n // 2, float(tiny[0])),
              (n - 2, float(tiny[1])), (1, float(tiny[2]))]
    want = 0
    for pos in (0, n - 1, n // 2, n - 3, 4 * 4000):
        for v in (float("nan"), float("inf"), float("-inf")):
            x.copy_(base)
            x[pos] = v
            for _ in range(2):
                flag.fill_(0.0)
                g.replay()
                want += 1
            torch.cuda.synchronize()
            assert float(flag) == 1.0 and int(count) == want, (pos, v)
    for v in (float("nan"), float("inf")):                      # every block sees one: the launch still counts once
        x.copy_(base)
        x[::256] = v
        for _ in range(2):
            flag.fill_(0.0)
            g.replay()
            want += 1
        torch.cuda.synchronize()
        assert float(flag) == 1.0 and int(count) == want, v
    x.copy_(base)
    for pos, v in finite:
        x[pos] = v
    assert bool((x[n // 2] != 0) & (x[n // 2].abs() < 1.2e-38))
    for _ in range(2):
        flag.fill_(1.0)                                         # reset by the graph itself
        g.replay()
    torch.cuda.synchronize()
    assert float(flag) == 0.0 and int(count) == want


def _state(tr):
    return tr.fs.state.clone(), tr.fs.mom.clone(), tr.fs.ema.clone(), tr.updates


@pytest.mark.gpu
def test_skip_nonfinite_in_a_captured_step():
    """loss_scale = inf makes every gradient inf / NaN: the guarded captured step leaves parameters and momentum bitwise
    as they were (the forward still updates the BatchNorm statistics, as the reference's forward does on a skipped
    step), moves the EMA as ModelEMA.update does (d from the step's updates) and counts 1.  Finite steps with and without
    the guard are bit-identical."""
    from test_gpu_model import build_product
    dev = torch.device("cuda")
    x = synth.synth_frames(2, 120, 192, seed=3).to(dev)
    tg = tuple(t.to(dev) for t in synth.synth_labels(2, 120, 192, seed=4))
    a = train.Trainer(build_product(TINY["depth"], TINY["width"]).train(), lr=1e-3, skip_nonfinite=True)
    b = train.Trainer(build_product(TINY["depth"], TINY["width"]).train(), lr=1e-3)
    for tr in (a, b):
        for i in range(3):
            tr.step(x, tg, lr=1e-3 * (i + 1))
    torch.cuda.synchronize()
    for u, v in zip(_state(a), _state(b)):
        assert (u == v) if isinstance(u, int) else torch.equal(u, v)
    assert a.skipped_steps() == 0 and b.skipped_steps() == 0
    xs, ts = x.clone(), tuple(t.clone() for t in tg)
    a.capture(xs, ts, loss_scale=float("inf"))                  # its eager warm-up is a skipped step too
    torch.cuda.synchronize()
    assert a.skipped_steps() == 1
    before = _state(a)
    ema_model = train.ModelEMA(a.model)                         # ModelEMA.update on the unchanged weights
    ema_model.ema.load_state_dict(a.ema_state_dict())
    ema_model.updates = a.updates
    a.replay(lr=1e-3)
    ema_model.update(a.model)
    torch.cuda.synchronize()
    after = _state(a)
    n = a.fs.n_param                                # the BatchNorm statistics after it move: the forward ran
    assert torch.equal(after[0][:n], before[0][:n]) and torch.equal(after[1], before[1])
    assert not torch.equal(after[0][n:], before[0][n:])
    assert after[3] == before[3] + 1 and a.skipped_steps() == 2
    got = a.ema_state_dict()
    for k, v in ema_model.ema.state_dict().items():
        if v.dtype.is_floating_point:
            assert torch.equal(got[k], v), k
    assert not torch.equal(after[2], before[2])


@pytest.mark.gpu
def test_capture_sizes_keeps_its_inputs_and_restores_the_skip_counter():
    """The static inputs make_inputs returns are written by every replay (the prologue) and read by it: the Trainer keeps
    them alive as long as the graphs, so no tensor allocated after the capture can be placed in their memory and
    overwritten by a replay.  The capture's eager warm-up (here at loss_scale = inf, a skipped step) leaves the skip
    counter as it found it; the replays count."""
    import gc
    import weakref
    from test_gpu_model import build_product
    dev = torch.device("cuda")
    tr = train.Trainer(build_product(TINY["depth"], TINY["width"]).train(), lr=1e-3, skip_nonfinite=True)
    x0 = synth.synth_frames(2, 120, 192, seed=3).to(dev)
    fut, cur = (t.to(dev) for t in synth.synth_labels(2, 120, 192, seed=4))
    sizes = [(96, 160), (120, 192)]
    refs = []

    def make_inputs(size):                      # fresh tensors, referenced by nobody but the Trainer afterwards
        out = (torch.empty((2, 6) + size, device=dev), (torch.empty_like(fut), torch.empty_like(cur)))
        refs.extend(weakref.ref(t) for t in (out[0], out[1][0], out[1][1]))
        return out

    def prologue(size, x, targets):
        if size == (120, 192):
            x.copy_(x0)
            targets[0].copy_(fut)
            targets[1].copy_(cur)
        else:
            data.preprocess(x0, (fut, cur), size, (120, 192), out=(x, targets))

    state = tr.fs.state[:tr.fs.n_param].clone()
    tr.capture_sizes(sizes, make_inputs, prologue, loss_scale=float("inf"))
    gc.collect()
    torch.cuda.synchronize()
    assert all(r() is not None for r in refs)
    assert tr.skipped_steps() == 0 and torch.equal(tr.fs.state[:tr.fs.n_param], state)
    probes = [torch.full((2, 50, 5), -7.0, device=dev) for _ in range(64)] + [torch.full((), -7.0, device=dev)
                                                                           for _ in range(256)]
    for s in sizes + sizes:
        tr.replay_size(s, 1e-3)
    torch.cuda.synchronize()
    assert all(bool((p == -7.0).all()) for p in probes)
    assert tr.skipped_steps() == 4 and torch.equal(tr.fs.state[:tr.fs.n_param], state)


def _gpu_build(layout):
    if layout == "still":
        from test_gpu_still import build_still
        return lambda: build_still(TINY["depth"], TINY["width"]).train()
    from test_gpu_model import build_product
    return lambda: build_product(TINY["depth"], TINY["width"]).train()


class RecordingStep(train_loop.DeviceStep):
    """the device step, recording what each replay was fed (host slot contents, size, lr) and its losses (device clones)"""
    record = []

    def replay(self, s, size, lr):
        h = {k: v.copy() for k, v in self.host[s].items()}
        out = super().replay(s, size, lr)
        RecordingStep.record.append((h, tuple(size), lr, {k: v.clone() for k, v in out.items()}))
        return out


def _gpu_loop(tmp_path, monkeypatch, layout, table, max_epoch, args=None, run=True):
    mod = helpers_module(monkeypatch)
    cls = train_loop.device_trainer(mod.Trainer)
    cls.step_class = RecordingStep
    RecordingStep.record = []
    exp = Exp(table, layout, str(tmp_path / "out"), max_epoch=max_epoch, device="cuda:0", build=_gpu_build(layout),
              print_interval=4)
    t = cls(exp, args or args_for(batch_size=2))
    if run:
        t.train()
    return t, exp, mod


def _hand_wired(layout, record, table, lr0, input_size=(120, 192), hw=(240, 384), random_size=(10, 14)):
    """INTEGRATION.md's graphed multi-scale loop with device JPEG decode, fed what the drop-in was fed"""
    dev = torch.device("cuda")
    model = _gpu_build(layout)()
    model.head.use_l1 = True
    model.to(dev)
    tr = train.Trainer(model, lr=lr0, momentum=0.9, weight_decay=5e-4, use_ema=True)
    h0 = record[0][0]
    fpi, B, M = (1 if layout == "still" else 2), h0["mirror"].shape[0], 5
    st = {k: torch.from_numpy(v).to(dev) for k, v in h0.items()}
    frames = torch.zeros((B * fpi,) + hw + (3,), dtype=torch.uint8, device=dev)
    status = torch.zeros(B * fpi, dtype=torch.int32, device=dev)
    ws = torch.empty(ops.jpeg_decode_workspace_bytes(B * fpi, st["bytes"].shape[1], *hw), dtype=torch.uint8, device=dev)
    sizes = train.multiscale_sizes(input_size, random_size)
    c = 3 * fpi

    def labels():
        if fpi == 1:
            return torch.empty((B, M, 5), device=dev)
        return tuple(torch.empty((B, M, 5), device=dev) for _ in range(2))

    stage = (torch.empty((B, c) + input_size, device=dev), labels())
    shared = torch.empty(B * c * max(h * w for h, w in sizes), device=dev)

    def make_inputs(size):
        if size == input_size:
            return stage
        return shared[:B * c * size[0] * size[1]].view((B, c) + size), labels()

    def prologue(size, x, targets):
        data.decode_jpeg(st["bytes"], st["lengths"], hw, out=frames, status=status, workspace=ws)
        if fpi == 2:
            data.pair_transform(frames.view(B, 2, hw[0], hw[1], 3), st["ann"], st["counts"], st["mirror"], input_size,
                                max_labels=M, raw=True, out=stage)
        else:
            data.frame_transform(frames, st["ann"], st["counts"], st["mirror"], input_size, max_labels=M, raw=True,
                                 out=stage)
        data.preprocess(stage[0], stage[1], size, input_size, out=(x, targets))

    tr.capture_sizes(sizes, make_inputs, prologue)
    losses = []
    for h, size, lr, _ in record:
        for k, v in h.items():
            st[k].copy_(torch.from_numpy(v))
        out = tr.replay_size(size, lr)
        losses.append({k: v.clone() for k, v in out.items()})
    torch.cuda.synchronize()
    return tr, losses


@pytest.mark.gpu
@pytest.mark.parametrize("layout", ["onex", "twox", "still"])
def test_loop_is_the_hand_wired_graphed_loop(tmp_path, monkeypatch, layout):
    """two epochs of the drop-in (22 iterations of 2 samples, a random_resize size in between) == the hand-wired
    capture_sizes loop fed the same files, labels, mirror bits, sizes and lrs: parameters, BatchNorm buffers, momentum,
    EMA, updates and every iteration's losses bit for bit, and the logged losses are the hand-wired loop's"""
    table = make_table(str(tmp_path / "data"), 22, layout, hw=(240, 384), seed={"onex": 1, "twox": 2, "still": 3}[layout],
                       jpeg=True, max_rows=6)
    t, exp, mod = _gpu_loop(tmp_path, monkeypatch, layout, table, max_epoch=2)
    rec = list(RecordingStep.record)
    assert len(rec) == 22 and len({s for _, s, _, _ in rec}) == 2
    assert rec[0][2] == 0 and t.tr.updates == 22
    tr, losses = _hand_wired(layout, rec, table, lr0=0)
    assert torch.equal(t.tr.fs.state, tr.fs.state)
    assert torch.equal(t.tr.fs.mom, tr.fs.mom)
    assert torch.equal(t.tr.fs.ema, tr.fs.ema)
    assert t.tr.updates == tr.updates
    a, b = t.model.state_dict(), tr.model.state_dict()
    for k in a:
        assert torch.equal(a[k], b[k]), k
    for i, ((_, _, _, got), want) in enumerate(zip(rec, losses)):
        for k in want:
            assert torch.equal(got[k], want[k]), (i, k)
    lines = [ln for ln in mod.logger.lines if ln.startswith("epoch: ")]
    assert len(lines) == 4                                      # iterations 4 and 8 of 11, twice
    for ln, i in zip(lines, (3, 7, 14, 18)):
        for k in ("total_loss", "iou_loss", "l1_loss", "conf_loss", "cls_loss"):
            assert "{}: {:.1f}".format(k, float(losses[i][k])) in ln, (i, k, ln)


@pytest.mark.gpu
def test_resume_from_latest_after_epoch_1(tmp_path, monkeypatch):
    """latest_ckpt.pth after epoch 1 has the reference's keys; --resume gives the state load_reference_checkpoint
    defines, updates = max_iter, and the checkpoint's lr first"""
    table = make_table(str(tmp_path / "data"), 8, "onex", hw=(240, 384), jpeg=True)
    t, exp, _ = _gpu_loop(tmp_path, monkeypatch, "onex", table, max_epoch=1)
    path = os.path.join(t.file_name, "latest_ckpt.pth")
    ckpt = torch.load(path, map_location="cuda")
    assert set(ckpt) == {"start_epoch", "model", "optimizer", "best_ap"} and ckpt["start_epoch"] == 1
    t2, _, _ = _gpu_loop(tmp_path, monkeypatch, "onex", table, max_epoch=2,
                         args=args_for(batch_size=2, resume=True, ckpt=path), run=False)
    t2.before_train()
    try:
        torch.cuda.synchronize()
        m = _gpu_build("onex")().cuda()
        m.head.use_l1 = True
        ref = train.Trainer(m, lr=0.5)
        ref.load_reference_checkpoint(ckpt, t2.max_iter)
        assert t2.tr.updates == t2.max_iter == 4 and t2.start_epoch == 1
        assert torch.equal(t2.tr.fs.state, ref.fs.state) and torch.equal(t2.tr.fs.mom, ref.fs.mom)
        assert torch.equal(t2.tr.fs.ema, ref.fs.ema)
        assert t2._lr == ckpt["optimizer"]["param_groups"][0]["lr"]
    finally:
        t2.after_train()


@pytest.mark.gpu
def test_damaged_file_raises_with_its_index(tmp_path, monkeypatch):
    table = make_table(str(tmp_path / "data"), 8, "onex", hw=(240, 384), jpeg=True)
    k = 5
    path = table[k][5]
    raw = np.fromfile(path, np.uint8)
    raw[len(raw) // 2:len(raw) // 2 + 64] = 0xFF                # markers in the entropy-coded data
    raw[:len(raw) - 200].tofile(path)
    with pytest.raises(RuntimeError, match=rf"dataset index {k} \(file {path}\) did not decode: "):
        _gpu_loop(tmp_path, monkeypatch, "onex", table, max_epoch=1)
