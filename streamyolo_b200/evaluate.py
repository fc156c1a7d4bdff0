"""The validation evaluators' batch loop on the device: JPEG files in, COCO detection rows out, one CUDA graph replay
per batch.

The reference's loop (exps/evaluators/onex_stream_evaluator.py:83-165, twox_stream_evaluator.py:81-163,
still_stream_evaluator.py:62-135) decodes and resizes every frame in the DataLoader's workers (cv2), runs
``model(imgs)`` and ``postprocess`` on the device, then ``convert_to_coco_format`` moves each image's detections to the
host and builds one dict per detection.  Here one replay per batch runs

    decode_jpeg (sy_jpeg_decode) -> the val transform (pair_transform / frame_transform, raw=True: load_resized_img's
    resize + ValTransform) -> model(x) -> postprocess_nms (room for every anchor) -> coco_rows (sy_coco_rows)

and the host only reads files and, once at the end, turns the rows into the reference's ``data_list``, which goes to the
evaluator's own ``evaluate_prediction`` (COCOeval and the per-class table stay the reference's).

    ev = DeviceEvaluator(val_loader, exp.test_size, exp.test_conf, exp.nmsthre, exp.num_classes, rule="onex")
    ap50_95, ap50, summary = ev.evaluate(model)          # what ONEX_COCOEvaluator.evaluate returns
    rows = ev.detections()                               # the same detections as numpy arrays

``DeviceEvaluator`` brings the batch loop; ``evaluate_prediction`` comes from the reference's evaluator class it is
combined with (``device_evaluator(ONEX_COCOEvaluator, "onex")``; ``dropin.install(evaluators=True)`` does this for the
three reference evaluators).
"""
import time
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import torch

from . import feed, ops
from .model import engine

RULES = {"onex": 2, "twox": 2, "still": 1}            # rule -> frames per sample
DROPPED_IDS = (15060, 15061)                         # the ids the onex / twox evaluators always skip


def image_id_table(images, ids, rule):
    """The frame-id rules of the three evaluators as one table: ``ids`` (the image ids of the dataset indices, ``dataset.ids``)
    -> int32 numpy array of the id their detections are emitted under, -1 where they are dropped.  ``images`` =
    ``dataset.coco.dataset['images']``, indexed by id as the reference indexes it.

      onex  (onex_stream_evaluator.py:188-207): dropped if the id is 15060 / 15061, images[id + 1].fid == 0 or
            images[id].fid == 0 (that branch sets idd but appends nothing); otherwise id + 1
      twox  (twox_stream_evaluator.py:184-216): as onex, and also dropped if images[id + 2].fid == 0 or images[id].fid == 1;
            otherwise id + 2
      still (still_stream_evaluator.py:156-167): every image under its own id

    An id whose rule reads past the end of ``images`` raises ValueError (the reference raises IndexError there as soon as
    that image has a detection)."""
    if rule not in RULES:
        raise ValueError(f"image_id_table: rule must be one of {sorted(RULES)}, not {rule!r}")
    out = np.full(len(ids), -1, np.int32)
    for k, i in enumerate(int(v) for v in ids):
        if rule == "still":
            out[k] = i
            continue
        if i in DROPPED_IDS:
            continue
        ahead = 2 if rule == "twox" else 1
        if not (0 <= i and i + ahead < len(images)):
            raise ValueError(f"image_id_table: image id {i} reads images[{i + ahead}] of {len(images)} ({rule} rule)")
        if images[i + 1]["fid"] == 0 or (rule == "twox" and images[i + 2]["fid"] == 0) or images[i]["fid"] == 0:
            continue
        if rule == "twox" and images[i]["fid"] == 1:
            continue
        out[k] = i + ahead
    return out


def sampler_batches(loader):
    """The dataset indices of every batch ``loader`` yields, from its own batch sampler (so the padding repeats of a
    DistributedSampler are evaluated, as the reference's loop evaluates them)."""
    if getattr(loader, "batch_sampler", None) is None:
        raise ValueError("DeviceEvaluator: the loader must batch its samples (batch_size set)")
    return [[int(i) for i in b] for b in loader.batch_sampler]


def empty_rows():
    return {"bbox": np.zeros((0, 4), np.float32), "score": np.zeros(0, np.float32), "image_id": np.zeros(0, np.int64),
            "category_id": np.zeros(0, np.int64)}


def merge_ranks(parts):
    """Rows of every rank -> one set of rows, rank-major (what ``gather`` + ``itertools.chain`` give the reference)."""
    return {k: np.concatenate([p[k] for p in parts]) for k in empty_rows()}


def coco_dicts(rows):
    """The reference's data_list: one dict per row, with the Python values ``convert_to_coco_format`` stores."""
    return [{"image_id": i, "category_id": c, "bbox": b, "score": s, "segmentation": []}
            for i, c, b, s in zip(rows["image_id"].tolist(), rows["category_id"].tolist(), rows["bbox"].tolist(),
                                  rows["score"].tolist())]


class EvalBatch:
    """The work of one batch on static buffers -- what ``DeviceEvaluator`` captures as a CUDA graph per batch size.
    Inputs (``jpeg.inputs``): ``bytes`` uint8 [F * B, max_bytes] and ``lengths`` int32 [F * B] (the files of the B samples,
    F = 2 frames per sample for pairs, current frame first, 1 for still), ``image_id`` int32 [B] (-1: emit nothing).
    Outputs: ``jpeg.status`` int32 [F * B] (data.JPEG_STATUS) and ``rows`` (ops.coco_rows' five tensors)."""

    def __init__(self, model, batch, frames, frame_hw, input_size, max_bytes, conf_thre, nms_thre, class_ids, ratio, device):
        self.model, self.conf_thre, self.nms_thre = model, float(conf_thre), float(nms_thre)
        self.jpeg = feed.JpegBatch(batch_spec(batch, frames, max_bytes), frames, frame_hw, input_size, device)
        self.x = torch.empty((batch, 3 * frames, input_size[0], input_size[1]), dtype=torch.float32, device=device)
        self.ratio = torch.full((batch,), ratio, dtype=torch.float32, device=device)
        self.class_ids = class_ids
        self.rows = None

    def run(self):
        self.jpeg.run((self.x, None))
        with torch.no_grad():
            raw = self.model(self.x)
        det, count = ops.postprocess_nms(raw, self.model.head.num_classes, self.conf_thre, self.nms_thre,
                                         max_det=raw.shape[1])
        self.rows = ops.coco_rows(det, count, self.ratio, self.jpeg.inputs["image_id"], self.class_ids,
                                  status=self.jpeg.status, out=self.rows)


def _sample(dataset, index, frames):
    """(file paths, (h, w)) of a dataset index (the layout of feed.sample)"""
    files, _, hw = feed.sample(dataset.annotations[index], frames)
    return files, hw


def batch_spec(batch, frames, max_bytes):
    """the fields of an evaluated batch (feed.jpeg_spec and the output ids)"""
    return dict(feed.jpeg_spec(batch, frames, max_bytes), image_id=((batch,), torch.int32))


class DeviceEvaluator:
    """The reference evaluators' ``evaluate`` with the batch loop on the device (module docstring).  The constructor takes
    the reference evaluator's arguments, plus

      rule       "onex", "twox" or "still": which evaluator's frame-id rules and dataset layout (a class attribute in the
                 classes ``device_evaluator`` builds)
      max_bytes  the longest JPEG file a batch takes; default: the longest file evaluated, rounded up to 4 KiB

    Every evaluated frame must have one size (Argoverse-HD: 1200 x 1920): the sizes of the dataset's ``img_info`` are
    checked here, and a file of another size makes ``evaluate`` raise."""

    rule = None

    def __init__(self, dataloader, img_size, confthre, nmsthre, num_classes, testdev=False, per_class_mAP=True, rule=None,
                 max_bytes=None):
        self.dataloader, self.img_size, self.confthre, self.nmsthre = dataloader, img_size, confthre, nmsthre
        self.num_classes, self.testdev, self.per_class_mAP = num_classes, testdev, per_class_mAP
        nxt = type(self).__mro__[type(self).__mro__.index(DeviceEvaluator) + 1]
        if nxt is not object:                         # the reference evaluator's own constructor
            super().__init__(dataloader, img_size, confthre, nmsthre, num_classes, testdev, per_class_mAP)
        self.rule = rule if rule is not None else self.rule
        if self.rule not in RULES:
            raise ValueError(f"DeviceEvaluator: rule must be one of {sorted(RULES)}, not {self.rule!r}")
        self.max_bytes = None if max_bytes is None else feed.check_max_bytes(max_bytes, "DeviceEvaluator: max_bytes")
        ds = dataloader.dataset
        if len(ds.class_ids) != num_classes:
            raise ValueError(f"DeviceEvaluator: the dataset's class table has {len(ds.class_ids)} entries for "
                             f"{num_classes} classes")
        if not all(-2 ** 31 <= int(c) < 2 ** 31 for c in ds.class_ids):
            raise ValueError("DeviceEvaluator: class ids must fit in int32")
        self.frames_per_image = RULES[self.rule]
        self._use_batches(sampler_batches(dataloader))
        self._rows = None
        self.capture_seconds = None

    def _use_batches(self, batches):
        """the batches (dataset indices) the next evaluation runs, their one frame size and image-id table"""
        ds = self.dataloader.dataset
        self.batches = batches
        used = sorted({i for b in self.batches for i in b})
        self.frame_hw = feed.frame_size([ds.annotations[i] for i in used], self.frames_per_image, "DeviceEvaluator")
        self.ratio = min(self.img_size[0] / float(self.frame_hw[0]), self.img_size[1] / float(self.frame_hw[1]))
        images = None if self.rule == "still" else ds.coco.dataset["images"]
        self.table = dict(zip(used, image_id_table(images, [ds.ids[i] for i in used], self.rule).tolist()))

    def detections(self):
        """The rows of the last ``evaluate`` (after the gather, on rank 0 with several ranks) as numpy arrays: ``bbox`` fp32
        [N, 4] xywh in frame pixels, ``score`` fp32 [N], ``image_id`` int64 [N], ``category_id`` int64 [N]; None before."""
        return None if self._rows is None else {k: v.copy() for k, v in self._rows.items()}

    def _capture(self, model, sizes, max_bytes, device):
        """one EvalBatch and its graph per batch size, the graphs in one memory pool (they replay one at a time)"""
        class_ids = torch.tensor([int(c) for c in self.dataloader.dataset.class_ids], dtype=torch.int32, device=device)
        pool, out = torch.cuda.graph_pool_handle(), {}
        for b in sorted(sizes, reverse=True):
            t = EvalBatch(model, b, self.frames_per_image, self.frame_hw, self.img_size, max_bytes, self.confthre,
                          self.nmsthre, class_ids, self.ratio, device)
            out[b] = (t, engine.capture_graph(t.run, device, pool))
        return out

    def evaluate(self, model, distributed=False, half=False, trt_file=None, decoder=None, test_size=None):
        """The reference's ``evaluate``: -> ``evaluate_prediction(data_list, statistics)`` (ap50_95, ap50, summary on the
        main process).  ``half=True`` calls ``model.half()`` as the reference does; the activation storage is
        ``model.activation_dtype``.  ``trt_file`` and ``decoder`` are not supported (NotImplementedError).

        The graphs are captured at the start of every call, because the weights change between epochs: one eager warm-up
        batch and one capture per batch size (the full one and a partial last one), each a few forwards' time.

        Timing statistics: under graphs the reference's per-stage split does not exist.  "forward" is the device time of
        every batch's replay but the last (CUDA events around it) and covers decode, transform, forward, NMS and the
        COCO rows; "NMS" is 0.  The "Average forward / NMS / inference time" line keeps its format."""
        if trt_file is not None or decoder is not None:
            raise NotImplementedError("DeviceEvaluator: trt_file and decoder are not supported")
        rows, infer_ms = self._rows_of(model, half)
        return self._score(rows, infer_ms, len(self.dataloader) - 1, distributed, next(model.parameters()).device)

    def evaluate_virtual_ranks(self, model, load_rank, virtual_ranks, batch_size, distributed=False, half=False):
        """``evaluate`` as a run of W x K ranks does it when this process runs K of them (``virtual_ranks``, W processes
        when ``distributed``): virtual rank g = rank * K + k evaluates the indices ``DistributedSampler(num_replicas=W * K,
        rank=g, shuffle=False)`` gives it, in batches of ``batch_size``, after ``load_rank(k)`` has put its weights into
        ``model``; the rows are concatenated in rank order (gathered over the W processes) and scored once, and the
        statistics are the sums over the W x K ranks.  The loader's own batches are evaluated again by ``evaluate``."""
        import torch.distributed as dist
        world, rank = (dist.get_world_size(), dist.get_rank()) if distributed else (1, 0)
        ds, own = self.dataloader.dataset, self.batches
        parts, infer_ms, n_batches = [], 0.0, 0
        try:
            for k in range(virtual_ranks):
                sampler = torch.utils.data.distributed.DistributedSampler(ds, num_replicas=world * virtual_ranks,
                                                                          rank=rank * virtual_ranks + k, shuffle=False)
                idx = [int(i) for i in sampler]
                self._use_batches([idx[i:i + batch_size] for i in range(0, len(idx), batch_size)])
                load_rank(k)
                rows, ms = self._rows_of(model, half)
                parts.append(rows)
                infer_ms += ms
                n_batches += len(self.batches) - 1
        finally:
            self._use_batches(own)
        return self._score(merge_ranks(parts), infer_ms, n_batches, distributed, next(model.parameters()).device)

    def _rows_of(self, model, half):
        """the rows of ``self.batches`` -> (rows, device ms of every replay but the last)"""
        model = model.eval()
        if half:
            model = model.half()
        device = next(model.parameters()).device
        if model.head.num_classes != self.num_classes:
            raise ValueError(f"DeviceEvaluator: the model has {model.head.num_classes} classes, the evaluator "
                             f"{self.num_classes}")
        ds, fpi = self.dataloader.dataset, self.frames_per_image
        max_bytes = self.max_bytes or feed.default_max_bytes(p for i in self.table for p in _sample(ds, i, fpi)[0])
        ops.lib()
        t0 = time.perf_counter()
        graphs = self._capture(model, {len(b) for b in self.batches}, max_bytes, device)
        torch.cuda.synchronize()
        self.capture_seconds = time.perf_counter() - t0
        rows, infer_ms = self._loop(graphs, max_bytes, device)
        del graphs
        return rows, infer_ms

    def _score(self, rows, infer_ms, n_batches, distributed, device):
        """gather the rows of every process to rank 0 in rank order and score them (evaluate_prediction)"""
        statistics = torch.tensor([infer_ms / 1000.0, 0.0, n_batches], dtype=torch.float32, device=device)
        if distributed:
            import torch.distributed as dist
            parts = [None] * dist.get_world_size() if dist.get_rank() == 0 else None
            dist.gather_object(rows, parts, dst=0)
            rows = merge_ranks(parts) if dist.get_rank() == 0 else empty_rows()
            dist.reduce(statistics, dst=0)
        self._rows = rows
        result = self.evaluate_prediction(coco_dicts(rows), statistics)
        if distributed:
            torch.distributed.barrier()
        return result

    def _loop(self, graphs, max_bytes, device):
        """Replay every batch.  A host thread reads the files of batch i + 2 into a pinned slot while the copy of batch
        i + 1 (copy stream, into a device slot) and the replay of batch i run; the rows of batch i - 1 are read back while
        batch i replays.  -> (rows, device ms of every replay but the last)."""
        n_batches, fpi = len(self.batches), self.frames_per_image
        b_max = max(len(b) for b in self.batches)
        ds, cur = self.dataloader.dataset, torch.cuda.current_stream(device)
        buf = feed.DoubleBuffer(batch_spec(b_max, fpi, max_bytes), b_max, device)
        cap = graphs[b_max][0].rows[0].shape[0]
        h_rows = [(feed.pinned((cap, 4), torch.float32), feed.pinned((cap,), torch.float32), feed.pinned((cap,), torch.int32),
                   feed.pinned((cap,), torch.int32), feed.pinned((1,), torch.int32), feed.pinned((b_max * fpi,), torch.int32))
                  for _ in range(2)]
        out_done = [torch.cuda.Event() for _ in range(2)]
        timing = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(n_batches)]
        parts = []

        def read(i):                                  # host thread: files of batch i -> host slot i % 2
            s, batch = i % 2, self.batches[i]
            buf.slot_free(s)
            for b, k in enumerate(batch):
                feed.read_sample(buf.host[s], b, k, _sample(ds, k, fpi)[0], "DeviceEvaluator")
            buf.host[s]["image_id"][:len(batch)] = [self.table[k] for k in batch]

        def h2d(i, fut):
            fut.result()
            buf.h2d(i % 2, len(self.batches[i]))

        def collect(i):                               # rows of batch i, out of pinned slot i % 2
            s, batch = i % 2, self.batches[i]
            out_done[s].synchronize()
            bbox, score, ids, cat, total, status = h_rows[s]
            feed.check_decoded(status, batch, ds.annotations, fpi, "DeviceEvaluator")
            n = int(total[0])
            parts.append({"bbox": bbox[:n].numpy().copy(), "score": score[:n].numpy().copy(),
                          "image_id": ids[:n].numpy().astype(np.int64), "category_id": cat[:n].numpy().astype(np.int64)})

        with ThreadPoolExecutor(max_workers=1) as reader:
            try:
                reads = {i: reader.submit(read, i) for i in range(min(2, n_batches))}
                h2d(0, reads.pop(0))
                for i, batch in enumerate(self.batches):
                    s, b = i % 2, len(batch)
                    t, g = graphs[b]
                    buf.take(s, t.jpeg.inputs, b)
                    timing[i][0].record(cur)
                    g.replay()
                    timing[i][1].record(cur)
                    rows = t.rows
                    m = rows[0].shape[0]
                    for dst, src in zip(h_rows[s][:4], rows[:4]):
                        dst[:m].copy_(src, non_blocking=True)
                    h_rows[s][4].copy_(rows[4], non_blocking=True)
                    h_rows[s][5][:b * fpi].copy_(t.jpeg.status, non_blocking=True)
                    out_done[s].record(cur)
                    if i + 1 < n_batches:
                        h2d(i + 1, reads.pop(i + 1))
                    if i + 2 < n_batches:
                        reads[i + 2] = reader.submit(read, i + 2)
                    if i >= 1:
                        collect(i - 1)
                collect(n_batches - 1)
            finally:
                buf.close()
        infer_ms = sum(a.elapsed_time(e) for a, e in timing[:-1])
        return (merge_ranks(parts) if parts else empty_rows()), infer_ms


def device_evaluator(base, rule):
    """A subclass of the reference evaluator class ``base`` (ONEX_COCOEvaluator, TWOX_COCOEvaluator or
    STILL_COCOEvaluator) whose ``evaluate`` is DeviceEvaluator's; ``evaluate_prediction`` and everything else stay
    ``base``'s."""
    if rule not in RULES:
        raise ValueError(f"device_evaluator: rule must be one of {sorted(RULES)}, not {rule!r}")
    return type(base.__name__, (DeviceEvaluator, base), {"rule": rule, "__module__": base.__module__,
                                                         "__doc__": f"{base.__name__} with the batch loop on the device "
                                                                    f"(streamyolo_b200.evaluate.DeviceEvaluator)"})
