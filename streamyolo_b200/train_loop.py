"""The reference trainer's loop on the device: JPEG files in, one CUDA graph replay per iteration.

The reference's ``tools/train.py`` runs ``exps/train_utils/double_trainer.py: Trainer``: DataLoader workers decode and
resize every frame with cv2, the prefetcher copies the fp32 batch, and each iteration runs the autograd step, torch SGD,
yolox ``ModelEMA`` and DDP's reducer.  ``device_trainer(Trainer)`` is a subclass of that class whose loop replays one
captured step per iteration instead:

    decode_jpeg (sy_jpeg_decode) -> pair_transform / frame_transform (raw=True: load_resized_img's resize +
    DoubleTrainTransform / TrainTransform) -> data.preprocess (Exp.preprocess at the multi-scale size) -> forward +
    backward + bucketed all-reduce + fused SGD-nesterov / EMA step (train.Trainer.capture_sizes / replay_size)

and the host only reads files.  ``dropin.install(trainer=True)`` puts it in place of the reference class, so
``exp.get_trainer(args)`` returns it for every shipped cfg.  ``__init__`` and everything not listed here stay the
reference's; the methods it replaces keep the reference's names (``train``, ``before_train``, ``train_in_epoch``,
``train_in_iter``, ``train_one_iter``, ``before_epoch``, ``after_epoch``, ``after_iter``, ``resume_train``,
``evaluate_and_save_model``, ``save_ckpt``).  The yolox helpers they call (``logger``, ``save_checkpoint``, ``load_ckpt``,
``gpu_mem_usage``, ``synchronize``, ``adjust_status``, ``occupy_mem``, ``SummaryWriter``, ``WandbLogger``) are the ones
the reference class's own module imported.

Batches.  ``exp.get_data_loader`` builds the loader as in the reference, but it is never iterated: no worker starts and
nothing is decoded on the host.  The batches are what one iterator over ``loader.batch_sampler`` yields (yolox's
``YoloBatchSampler``: ``(mosaic, index)`` pairs; one iterator for the whole run, as the prefetcher's ``iter(loader)``),
the files and labels come from the wrapped dataset's ``annotations`` and ``max_labels`` / ``flip`` from the wrapper's
``preproc``.  A pair's mirror bit is one draw with p = 1/2 (``DoubleTrainTransform``'s ``random.randrange(2)``) from a
generator seeded by ``exp.seed`` and the rank; a still frame's is 0 (``TrainTransform``'s default ``mirror=False``).

Feeding.  A host thread reads the files of iteration i + 2 into a pinned slot while the copy of iteration i + 1 (copy
stream, ordered by events) and the replay of iteration i run (feed.DoubleBuffer).  The host synchronises only where
the reference does: at the print iteration (the losses), at ``exp.random_resize`` every 10 iterations (its ``.item()``)
and at the end of an epoch.  Each iteration's JPEG status goes into a device ring that is read at those points; a frame
that did not decode then raises ``RuntimeError`` with its dataset index, file and ``data.JPEG_STATUS`` reason, so up to
9 further steps may have run by then (the reference's ``load_image`` asserts at once, in the worker).

Refused before anything is captured: epochs with mosaic left (``start_epoch < max_epoch - no_aug_epochs``; no shipped
cfg has any) and ``hsv=True`` raise ``NotImplementedError``, frames of more than one size ``ValueError``.

Arguments that change nothing here: ``--cache`` (files are read, not cached images); ``-o/--occupy`` is the reference's
``occupy_mem``; ``--fp16`` does not change the storage (training stores bf16; fp16 activation storage raises as it does
for ``train.Trainer``) and applies no loss scale (bf16 has fp32's exponent range, so a power-of-two scale is exact and
changes nothing), and the input batch and labels stay fp32 where the reference rounds them to fp16 before its
multi-scale resize (double_trainer.py:99-105).  What ``GradScaler`` does that matters is kept: with ``--fp16`` a step
whose gradients are not finite is skipped on the device (``train.Trainer(skip_nonfinite=True)``).

The still cfg (``l_s50_still_dfp_flip.py``) trains on its one ``[B, M, 5]`` label tensor, which is what ``Trainer``
takes.  The reference's prefetcher indexes the collated label tensor as a pair (double_data_prefetcher.py:33, 36-49),
handing ``PIPEHead`` its images 0 and 1 as a tuple, and ``PIPEHead.get_losses`` then fails at ``labels.shape``
(pipe_head.py:271) on the first iteration; the drop-in does not reproduce that.
"""
import copy
import datetime
import os
import sys
import time
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import torch

from . import data, feed, train

RING = 10                     # iterations between two synchronisations at most: random_resize syncs every 10


def _transform_flags(preproc):
    """(max_labels, flip, hsv) of the wrapper's DoubleTrainTransform (flags on its two TrainTransforms) / TrainTransform"""
    inner = getattr(preproc, "trasform1", preproc)
    return int(preproc.max_labels), bool(getattr(inner, "flip", True)), bool(getattr(inner, "hsv", False))


def _index(item):
    """a YoloBatchSampler item (mosaic, index), or a plain index"""
    return int(item[1]) if isinstance(item, (tuple, list)) else int(item)


class BatchTable:
    """What the loop needs of the training dataset (``loader.dataset``, yolox's MosaicDetection wrapper, around
    ``_dataset``): its ``annotations`` (feed.sample: the files, labels and frame size of a dataset index), the frames per
    sample, the one frame size, the most label rows of a frame and the transform's ``max_labels`` and ``flip``."""

    def __init__(self, loader):
        wrapper = loader.dataset
        inner = getattr(wrapper, "_dataset", wrapper)
        self.annotations = inner.annotations
        self.max_labels, self.flip, hsv = _transform_flags(wrapper.preproc)
        if hsv:
            raise NotImplementedError("DeviceTrainer: the cfg's preproc sets hsv=True; HSV augmentation has no device "
                                      "implementation")
        self.frames = 2 if len(self.annotations[0]) == 6 else 1
        self.frame_hw = feed.frame_size(self.annotations, self.frames, "DeviceTrainer")
        self.max_rows = max(1, max(len(lab) for a in self.annotations for lab in feed.sample(a, self.frames)[1]))


class DeviceStep:
    """The device half of the loop: the static inputs and their decode + transform, one captured step per multi-scale
    size (``Trainer.capture_sizes`` in one memory pool), the double buffer and the status ring.  ``DeviceTrainer`` drives
    it through ``host``, ``slot_free``, ``h2d``, ``replay`` and ``sync``; tests put a stand-in with the same methods in its
    place."""

    def __init__(self, tr, table, batch, input_size, sizes, max_bytes, device):
        self.tr, self.batch, self.fpi = tr, batch, table.frames
        self.input_size, self.max_labels = tuple(input_size), table.max_labels
        n, R, dev = batch * self.fpi, table.max_rows, device
        lab = (batch, self.fpi, R, 5) if self.fpi == 2 else (batch, R, 5)
        cnt = (batch, self.fpi) if self.fpi == 2 else (batch,)
        spec = dict(feed.jpeg_spec(batch, self.fpi, max_bytes), ann=(lab, torch.float64), counts=(cnt, torch.int32),
                    mirror=((batch,), torch.int32))
        self.buffer = feed.DoubleBuffer(spec, batch, dev)
        self.host = self.buffer.host
        self.jpeg = feed.JpegBatch(spec, self.fpi, table.frame_hw, self.input_size, dev, table.max_labels, table.flip)
        self.ring = torch.zeros((RING, n), dtype=torch.int32, device=dev)
        c = 3 * self.fpi
        self.stage = self._buffers(self.input_size, dev)
        self.shared = torch.empty(batch * c * max(h * w for h, w in sizes), dtype=torch.float32, device=dev)
        self.sizes, self.dev, self.n_ring, self.losses = sizes, dev, 0, None

    def _buffers(self, size, dev, x=None):
        b, c = self.batch, 3 * self.fpi
        if x is None:
            x = torch.empty((b, c) + tuple(size), dtype=torch.float32, device=dev)
        if self.fpi == 1:
            return x, torch.empty((b, self.max_labels, 5), dtype=torch.float32, device=dev)
        return x, tuple(torch.empty((b, self.max_labels, 5), dtype=torch.float32, device=dev) for _ in range(2))

    def _make_inputs(self, size):
        if tuple(size) == self.input_size:
            return self.stage
        b, c = self.batch, 3 * self.fpi
        return self._buffers(size, self.dev, self.shared[:b * c * size[0] * size[1]].view((b, c) + tuple(size)))

    def _prologue(self, size, x, targets):
        self.jpeg.run(self.stage)
        data.preprocess(self.stage[0], self.stage[1], size, self.input_size, out=(x, targets))

    def capture(self, s):
        """capture every size on the batch in slot s (the capture trains nothing: Trainer.capture_sizes restores the state)"""
        self.buffer.take(s, self.jpeg.inputs, self.batch)
        self.tr.capture_sizes(self.sizes, self._make_inputs, self._prologue)

    def slot_free(self, s):
        """(reader thread) block until the last copy out of host slot s has run"""
        self.buffer.slot_free(s)

    def h2d(self, s):
        self.buffer.h2d(s, self.batch)

    def replay(self, s, size, lr):
        """one step on the batch in slot s at ``size`` with learning rate ``lr``; its status goes into the ring.  Returns
        the graph's loss dict: device tensors that the next replay overwrites."""
        self.buffer.take(s, self.jpeg.inputs, self.batch)
        self.losses = self.tr.replay_size(size, lr)
        self.ring[self.n_ring % RING].copy_(self.jpeg.status)
        self.n_ring += 1
        return self.losses

    def sync(self, pending):
        """synchronise; -> the status rows (numpy) of the last ``pending`` replays, oldest first"""
        assert pending <= RING, (pending, RING)
        rows = self.ring.cpu().numpy()
        return [rows[(self.n_ring - pending + j) % RING] for j in range(pending)]

    def close(self):
        self.buffer.close()


class DeviceTrainer:
    """The loop of the reference trainer (module docstring); combined with the reference class by ``device_trainer``."""

    step_class = DeviceStep   # the device half (a stand-in in the CPU tests)
    virtual_ranks = 1         # ranks run one after another in this process (dropin.install(trainer=True, virtual_ranks=K))
    max_bytes = None          # the longest JPEG file a batch takes; default: the longest training file, rounded up to 4 KiB
    _helpers = None           # the module whose yolox helpers the loop calls (the reference class's)

    def _h(self, name):
        return getattr(sys.modules[self._helpers], name)

    def make_trainer(self, model, **kw):
        return train.Trainer(model, **kw)

    # ---- double_trainer.py:74-93
    def train(self):
        self.before_train()
        try:
            self.train_in_epoch()
        finally:
            self.after_train()

    def train_in_epoch(self):
        for self.epoch in range(self.start_epoch, self.max_epoch):
            self.before_epoch()
            self.train_in_iter()
            self.after_epoch()

    def train_in_iter(self):
        for self.iter in range(self.max_iter):
            self.before_iter()
            self.train_one_iter()
            self.after_iter()

    @property
    def progress_in_iter(self):
        return self.epoch * self.max_iter + self.iter

    # ---- double_trainer.py:133-196
    def before_train(self):
        logger, args, exp = self._h("logger"), self.args, self.exp
        logger.info("args: {}".format(args))
        logger.info("exp value:\n{}".format(exp))
        if str(self.device).startswith("cuda"):
            torch.cuda.set_device(self.local_rank)
        model = exp.get_model()
        model.to(self.device)
        lr0 = exp.get_optimizer(args.batch_size).param_groups[0]["lr"]       # the reference optimiser's first lr
        self._resume = None
        model = self.resume_train(model)
        self.no_aug = self.start_epoch >= self.max_epoch - exp.no_aug_epochs
        if not self.no_aug:
            raise NotImplementedError(f"DeviceTrainer: epochs {self.start_epoch + 1}..{self.max_epoch - exp.no_aug_epochs} "
                                      f"train with mosaic (no_aug_epochs = {exp.no_aug_epochs} of max_epoch = "
                                      f"{self.max_epoch}); mosaic and mixup have no device implementation")
        self.train_loader = exp.get_data_loader(batch_size=args.batch_size, is_distributed=self.is_distributed,
                                                no_aug=self.no_aug, cache_img=args.cache)
        self.table = BatchTable(self.train_loader)
        self._virtual = self._virtual_samplers()
        self.max_iter = len(self.train_loader) if self._virtual is None else len(self._virtual[0])
        self.lr_scheduler = exp.get_lr_scheduler(exp.basic_lr_per_img * args.batch_size, self.max_iter)
        if args.occupy:
            self._h("occupy_mem")(self.local_rank)
        model.head.use_l1 = True                        # before_epoch's switch (no mosaic epoch is left), :209-217
        exp.eval_interval = 1
        self.eval_model = copy.deepcopy(model)          # before the Trainer turns the parameters into views
        vr = {} if self._virtual is None else {"virtual_ranks": self.virtual_ranks}
        self.tr = self.make_trainer(model, lr=lr0, momentum=exp.momentum, weight_decay=exp.weight_decay,
                                    use_ema=exp.ema, skip_nonfinite=bool(args.fp16), **vr)
        if self._resume is not None:
            self.tr.load_reference_checkpoint(self._resume, self.max_iter * self.start_epoch)
            self._resume = None
        self._lr = self.tr.lr                           # what the reference's optimizer holds at the next iteration
        self.model = model
        self._start_feed()
        self.evaluator = exp.get_evaluator(batch_size=args.batch_size, is_distributed=self.is_distributed)
        if self._virtual is not None and not hasattr(self.evaluator, "evaluate_virtual_ranks"):
            raise ValueError(f"DeviceTrainer: virtual ranks evaluate one shard per rank through the device evaluator "
                             f"(dropin.install(evaluators=True)); the cfg's evaluator is a {type(self.evaluator).__name__}")
        if self.rank == 0:
            if args.logger == "tensorboard":
                self.tblogger = self._h("SummaryWriter")(os.path.join(self.file_name, "tensorboard"))
            elif args.logger == "wandb":
                wandb_params = {}
                for k, v in zip(args.opts[0::2], args.opts[1::2]):
                    if k.startswith("wandb-"):
                        wandb_params.update({k.lstrip("wandb-"): v})
                self.wandb_logger = self._h("WandbLogger")(config=vars(exp), **wandb_params)
            else:
                raise ValueError("logger must be either 'tensorboard' or 'wandb'")
        logger.info("Training start...")
        logger.info("\n{}".format(model))

    def _virtual_samplers(self):
        """Virtual ranks (K > 1): the batch sampler of every virtual rank g = rank * K + k of a W x K-rank run, what
        ``get_data_loader`` builds for rank g of W x K (a batch of ``args.batch_size // (W x K)``), rebuilt from the
        loader's own yolox InfiniteSampler (its size, shuffle and seed) and YoloBatchSampler (drop_last, mosaic).  None
        for K = 1: the loader's own batch sampler is iterated."""
        K = self.virtual_ranks
        if K == 1:
            return None
        bs = self.train_loader.batch_sampler
        sampler = getattr(bs, "sampler", None)
        if type(sampler).__name__ != "InfiniteSampler" or type(bs).__name__ != "YoloBatchSampler":
            raise ValueError(f"DeviceTrainer: virtual ranks rebuild yolox's InfiniteSampler inside a YoloBatchSampler; the "
                             f"loader has a {type(sampler).__name__} inside a {type(bs).__name__}")
        G = sampler._world_size * K
        B = self.args.batch_size // G
        if B == 0:
            raise ValueError(f"DeviceTrainer: a batch of {self.args.batch_size} leaves no sample for each of {G} ranks "
                             f"({sampler._world_size} processes x {K} virtual ranks)")
        out = []
        for k in range(K):
            s = type(sampler)(sampler._size, shuffle=sampler._shuffle, seed=sampler._seed)
            s._rank, s._world_size = self.rank * K + k, G      # it takes them from torch.distributed when initialised
            out.append(type(bs)(sampler=s, batch_size=B, drop_last=bs.drop_last, mosaic=bs.mosaic))
        return out

    def resume_train(self, model):
        """double_trainer.py:285-318.  ``--resume``: the checkpoint is read here and loaded into the native Trainer once
        it exists (``load_reference_checkpoint(ckpt, max_iter * start_epoch)``, with ``-e`` and ``best_ap``); ``-c``
        alone: yolox's shape-tolerant ``load_ckpt`` on the model."""
        logger, args = self._h("logger"), self.args
        if args.resume:
            logger.info("resume training")
            ckpt_file = os.path.join(self.file_name, "latest" + "_ckpt.pth") if args.ckpt is None else args.ckpt
            ckpt = torch.load(ckpt_file, map_location=self.device)
            self.best_ap = ckpt.pop("best_ap", 0)
            self.start_epoch = args.start_epoch - 1 if args.start_epoch is not None else ckpt["start_epoch"]
            self._resume = ckpt
            logger.info("loaded checkpoint '{}' (epoch {})".format(args.resume, self.start_epoch))
        else:
            if args.ckpt is not None:
                logger.info("loading checkpoint for fine tuning")
                ckpt = torch.load(args.ckpt, map_location=self.device)["model"]
                model = self._h("load_ckpt")(model, ckpt)
            self.start_epoch = 0
        return model

    # ---- feeding
    def _start_feed(self):
        """the batch iterator, the reader thread, the device step (its graphs captured on the first batch), and the
        reads of the first two iterations"""
        t = self.table
        if self.max_bytes is None:
            max_bytes = feed.default_max_bytes(p for a in t.annotations for p in feed.sample(a, t.frames)[0])
        else:
            max_bytes = feed.check_max_bytes(self.max_bytes, "DeviceTrainer: max_bytes")
        K = self.virtual_ranks
        if self._virtual is None:
            self._batches = iter(self.train_loader.batch_sampler)
            batch = self.train_loader.batch_sampler.batch_size
        else:                                           # the virtual ranks' batches side by side, in rank order
            self._batches = ([i for part in parts for i in part] for parts in zip(*self._virtual))
            batch = K * self._virtual[0].batch_size
        self._rngs = [np.random.default_rng([int(self.exp.seed or 0), int(self.rank) * K + k]) for k in range(K)]
        self._reader = ThreadPoolExecutor(max_workers=1)
        self._left = (self.max_epoch - self.start_epoch) * self.max_iter       # iterations still to be read
        sizes = train.multiscale_sizes(self.exp.input_size, self.exp.random_size)
        self.step = self.step_class(self.tr, t, batch, self.exp.input_size, sizes, max_bytes, self.device)
        self._reads, self._k, self._pending = [], 0, []
        self._submit()
        self._submit()
        self._wait_read()
        self.step.h2d(0)
        self.step.capture(0)
        self._sync_time, self._meter_rows = time.time(), []

    def _submit(self):
        if self._left == 0:
            return
        self._left -= 1
        s = (self._k + len(self._reads)) % 2
        idx = [_index(i) for i in next(self._batches)]
        if self.table.frames == 2:                      # each (virtual) rank draws its own samples' bits
            mirror = np.concatenate([r.integers(0, 2, len(idx) // len(self._rngs)) for r in self._rngs])
        else:
            mirror = np.zeros(len(idx), np.int64)
        self._reads.append((idx, self._reader.submit(self._read, s, idx, mirror)))

    def _read(self, s, idx, mirror):
        """(reader thread) files, labels and mirror bits of one batch -> host slot s"""
        fpi = self.table.frames
        self.step.slot_free(s)
        h = self.step.host[s]
        if len(idx) != h["mirror"].shape[0]:
            raise ValueError(f"DeviceTrainer: the batch sampler yielded {len(idx)} indices, the step takes "
                             f"{h['mirror'].shape[0]} (drop_last=False with an uneven last batch is not supported)")
        ann, counts = h["ann"].reshape(len(idx), fpi, -1, 5), h["counts"].reshape(len(idx), fpi)     # views
        ann[...] = 0
        counts[...] = 0
        for b, i in enumerate(idx):
            files, labels, _ = feed.sample(self.table.annotations[i], fpi)
            feed.read_sample(h, b, i, files, "DeviceTrainer")
            for f, lab in enumerate(labels):
                ann[b, f, :len(lab)] = lab
                counts[b, f] = len(lab)
            h["mirror"][b] = mirror[b]

    def _wait_read(self):
        """block until the read of the next iteration has finished; -> seconds blocked"""
        t0 = time.time()
        self._reads[0][1].result()
        return time.time() - t0

    def _sync_point(self):
        """one of the reference's synchronisations: check the JPEG status of the iterations since the last one, and give
        the meter their iteration time (the wall time since the last one over their count)"""
        n = len(self._pending)
        if n == 0:
            return
        rows = self.step.sync(n)
        now = time.time()
        for idx, st in zip(self._pending, rows):
            feed.check_decoded(st, idx, self.table.annotations, self.table.frames, "DeviceTrainer")
        it = (now - self._sync_time) / n
        for data_time, lr in self._meter_rows:
            self.meter.update(iter_time=it, data_time=data_time, lr=lr)
        self._pending, self._meter_rows, self._sync_time = [], [], now

    # ---- double_trainer.py:95-131
    def train_one_iter(self):
        """One replay.  ``iter_time`` in the meter is the wall time between two synchronisations over the iterations
        between them, ``data_time`` the time the main thread blocked on the reader."""
        s = self._k % 2
        idx, _ = self._reads.pop(0)
        self.step.replay(s, self.input_size, self._lr)
        self._pending.append(idx)
        self._k += 1
        data_time = 0.0
        if self._reads:
            data_time = self._wait_read()
            self.step.h2d(self._k % 2)
        self._submit()
        self._lr = self.lr_scheduler.update_lr(self.progress_in_iter + 1)
        self._meter_rows.append((data_time, self._lr))

    def before_epoch(self):
        logger = self._h("logger")
        logger.info("---> start train epoch{}".format(self.epoch + 1))
        logger.info("--->No mosaic aug now!")
        if hasattr(self.train_loader, "close_mosaic"):
            self.train_loader.close_mosaic()
        logger.info("--->Add additional L1 loss now!")
        self.model.head.use_l1 = True
        self.exp.eval_interval = 1

    # ---- double_trainer.py:231-279
    def after_iter(self):
        if (self.iter + 1) % self.exp.print_interval == 0:
            losses = {k: float(v) for k, v in self.step.losses.items()}     # the graph's vector: read now, never kept
            self._sync_point()
            self.meter.update(**losses)
            left_iters = self.max_iter * self.max_epoch - (self.progress_in_iter + 1)
            eta_seconds = self.meter["iter_time"].global_avg * left_iters
            eta_str = "ETA: {}".format(datetime.timedelta(seconds=int(eta_seconds)))
            progress_str = "epoch: {}/{}, iter: {}/{}".format(self.epoch + 1, self.max_epoch, self.iter + 1, self.max_iter)
            loss_meter = self.meter.get_filtered_meter("loss")
            loss_str = ", ".join(["{}: {:.1f}".format(k, v.latest) for k, v in loss_meter.items()])
            time_meter = self.meter.get_filtered_meter("time")
            time_str = ", ".join(["{}: {:.3f}s".format(k, v.avg) for k, v in time_meter.items()])
            self._h("logger").info(
                "{}, mem: {:.0f}Mb, {}, {}, lr: {:.3e}".format(progress_str, self._h("gpu_mem_usage")(), time_str,
                                                               loss_str, self.meter["lr"].latest)
                + (", size: {:d}, {}".format(self.input_size[0], eta_str)))
            if self.rank == 0 and self.args.logger == "wandb":
                self.wandb_logger.log_metrics({k: v.latest for k, v in loss_meter.items()})
                self.wandb_logger.log_metrics({"lr": self.meter["lr"].latest})
            self.meter.clear_meters()
        if (self.progress_in_iter + 1) % 10 == 0:
            self.input_size = self.exp.random_resize(self.train_loader, self.epoch, self.rank, self.is_distributed)
            self._sync_point()

    # ---- double_trainer.py:221-226, 320-371
    def after_epoch(self):
        self._sync_point()
        self.save_ckpt(ckpt_name="latest")
        if (self.epoch + 1) % self.exp.eval_interval == 0:
            self.tr.all_reduce_norm()
            self.evaluate_and_save_model()

    def evaluate_and_save_model(self):
        """The evaluator gets ``eval_model``, a copy taken before the Trainer was built, holding the EMA weights
        (``tr.ema_state_dict()``), or the live weights without EMA; never the training model itself.  Virtual ranks:
        ``DeviceEvaluator.evaluate_virtual_ranks`` evaluates rank g's ``DistributedSampler`` shard of a W x K-rank run
        with rank g's weights (its EMA BatchNorm buffers), in batches of ``args.batch_size // (W x K)``, and scores
        the rows of all ranks once, in rank order, as the reference's ranks and its gather do."""
        def load(k):
            sd = self.tr.ema_state_dict(k) if self.use_model_ema else self.tr.model_state_dict(k)
            self.eval_model.load_state_dict(sd)

        with self._h("adjust_status")(self.eval_model, training=False):
            if self._virtual is None:
                load(0)
                ap50_95, ap50, summary = self.exp.eval(self.eval_model, self.evaluator, self.is_distributed)
            else:       # every virtual rank's DistributedSampler shard with its own weights, scored once
                ap50_95, ap50, summary = self.evaluator.evaluate_virtual_ranks(
                    self.eval_model, load, self.virtual_ranks, self._virtual[0].batch_size, self.is_distributed)
        update_best_ckpt = ap50_95 > self.best_ap
        self.best_ap = max(self.best_ap, ap50_95)
        if self.rank == 0:
            if self.args.logger == "tensorboard":
                self.tblogger.add_scalar("val/COCOAP50", ap50, self.epoch + 1)
                self.tblogger.add_scalar("val/COCOAP50_95", ap50_95, self.epoch + 1)
            if self.args.logger == "wandb":
                self.wandb_logger.log_metrics({"val/COCOAP50": ap50, "val/COCOAP50_95": ap50_95, "epoch": self.epoch + 1})
            self._h("logger").info("\n" + summary)
        self._h("synchronize")()
        self.save_ckpt("last_epoch", update_best_ckpt)
        if self.save_history_ckpt:
            self.save_ckpt(f"epoch_{self.epoch + 1}")

    def save_ckpt(self, ckpt_name, update_best_ckpt=False):
        """rank 0: yolox ``save_checkpoint`` of ``tr.reference_checkpoint(epoch + 1, best_ap)``, the reference's keys
        (``start_epoch``, ``model``: the EMA weights with EMA, ``optimizer`` in torch.optim.SGD format, ``best_ap``)"""
        if self.rank == 0:
            self._h("logger").info("Save weights to {}".format(self.file_name))
            self._h("save_checkpoint")(self.tr.reference_checkpoint(self.epoch + 1, self.best_ap), update_best_ckpt,
                                       self.file_name, ckpt_name)
            if self.args.logger == "wandb":
                self.wandb_logger.save_checkpoint(self.file_name, ckpt_name, update_best_ckpt)

    def after_train(self):
        reader = getattr(self, "_reader", None)
        if reader is not None:
            reader.shutdown(wait=True, cancel_futures=True)
            self._reader = None
        step = getattr(self, "step", None)
        if step is not None:
            step.close()
        super().after_train()


def device_trainer(base):
    """A subclass of the reference trainer class ``base`` (exps/train_utils/double_trainer.py: Trainer) whose loop is
    DeviceTrainer's; ``__init__`` and everything else stay ``base``'s, and the yolox helpers come from ``base``'s module."""
    return type(base.__name__, (DeviceTrainer, base), {"__module__": base.__module__, "_helpers": base.__module__,
                                                       "__doc__": f"{base.__name__} with its loop on the device "
                                                                  f"(streamyolo_b200.train_loop.DeviceTrainer)"})
