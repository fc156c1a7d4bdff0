"""The JPEG input path of the device loops (evaluate.DeviceEvaluator, train_loop.DeviceTrainer): the Argoverse sample
layout, the file reader, the pinned double buffer between the reader thread and the replays, and the decode + transform
a captured batch starts with.  A field spec is ``{name: (shape, dtype)}``, every field sample-major (dim 0: the batch's
samples, or their F frames: 2 per sample for pairs, 1 for still)."""
import os

import numpy as np
import torch

from . import data, ops


def sample(a, frames):
    """(files, labels, (h, w)) of annotation entry ``a``: pairs (``frames`` = 2) ``(res, support_res, img_info,
    resized_info, file, support_file)``, frame 0 being ``file`` and label 0 ``res`` (the future boxes); still (1) ``(res,
    img_info, resized_info, file)``.  Labels: float64 [n, 5] rows x1, y1, x2, y2, cls, as ``pull_item`` returns them."""
    if frames == 2:
        return (a[4], a[5]), (a[0], a[1]), tuple(int(v) for v in a[2])
    return (a[3],), (a[0],), tuple(int(v) for v in a[1])


def frame_size(annotations, frames, who):
    """The one (h, w) of the frames of ``annotations``; ValueError if they have several (a graph decodes one size)."""
    sizes = {sample(a, frames)[2] for a in annotations}
    if len(sizes) != 1:
        raise ValueError(f"{who}: one frame size per loop; the samples' img_info hold {sorted(sizes)}")
    return sizes.pop()


def default_max_bytes(files):
    """The row length a batch of ``files`` needs: the longest file, rounded up to 4 KiB, at least 4096."""
    return max(4096, -(-max(os.path.getsize(p) for p in files) // 4096) * 4096)


def check_max_bytes(value, name):
    """``value`` as an int, or ValueError naming ``name`` (e.g. "DeviceEvaluator: max_bytes")."""
    if int(value) != value or not 4 <= value <= 1 << 28:
        raise ValueError(f"{name} must be an integer in [4, 2^28], not {value}")
    return int(value)


def jpeg_spec(batch, frames, max_bytes):
    """the fields every JPEG batch has: its files' bytes and lengths"""
    return {"bytes": ((batch * frames, max_bytes), torch.uint8), "lengths": ((batch * frames,), torch.int32)}


def pinned(shape, dtype):
    """a zeroed page-locked host tensor, which a non-blocking copy can read or write while the host goes on"""
    return torch.zeros(shape, dtype=dtype, pin_memory=True)


def read_sample(host, b, index, files, who):
    """(reader thread) The ``files`` of dataset index ``index``, sample ``b`` of the batch -> its rows of a host slot's
    ``bytes`` and ``lengths`` (numpy); ValueError if a file is longer than the rows."""
    max_bytes = host["bytes"].shape[1]
    for f, path in enumerate(files):
        a = np.fromfile(path, np.uint8)
        if a.size > max_bytes:
            raise ValueError(f"{who}: dataset index {index}: {path} has {a.size} bytes, more than max_bytes = {max_bytes}")
        host["bytes"][b * len(files) + f, :a.size] = a
        host["lengths"][b * len(files) + f] = a.size


def check_decoded(status, indices, annotations, frames, who):
    """RuntimeError naming the first frame of a batch that did not decode: ``status`` the int32 status of its frames
    (``frames`` per sample), ``indices`` its dataset indices."""
    for k, v in enumerate(np.asarray(status)[:len(indices) * frames].tolist()):
        if v != 0:
            i = indices[k // frames]
            raise RuntimeError(f"{who}: dataset index {i} (file {sample(annotations[i], frames)[0][k % frames]}) did not "
                               f"decode: {data.JPEG_STATUS.get(v, f'status {v}')}")


class DoubleBuffer:
    """Two pinned host slots (``host[s]``: numpy views, for the reader thread) and two device slots of the fields ``spec``
    for up to ``batch`` samples, a copy stream and two events per slot, so that the read of batch i + 2, the copy of
    batch i + 1 and the replay of batch i overlap:

      h2d_done[s]  the copy out of host slot s has run: the reader waits on it (``slot_free``) before it writes the slot
      in_used[s]   the replay has taken device slot s in (``take``): the copy stream waits on it before it writes the slot"""

    def __init__(self, spec, batch, device):
        self.device = device
        self.rows = {k: shape[0] // batch for k, (shape, _) in spec.items()}      # rows per sample
        self._host = [{k: pinned(shape, dt) for k, (shape, dt) in spec.items()} for _ in range(2)]
        self.host = [{k: v.numpy() for k, v in h.items()} for h in self._host]
        self.dev = [{k: torch.zeros(shape, dtype=dt, device=device) for k, (shape, dt) in spec.items()} for _ in range(2)]
        self.copy = torch.cuda.Stream(device=device)
        self.h2d_done = [torch.cuda.Event() for _ in range(2)]
        self.in_used = [torch.cuda.Event() for _ in range(2)]

    def slot_free(self, s):
        """(reader thread) block until the last copy out of host slot s has run"""
        self.h2d_done[s].synchronize()

    def h2d(self, s, n):
        """the first ``n`` samples of host slot s -> device slot s, on the copy stream"""
        self.copy.wait_event(self.in_used[s])
        with torch.cuda.stream(self.copy):
            for k, v in self.dev[s].items():
                m = n * self.rows[k]
                v[:m].copy_(self._host[s][k][:m], non_blocking=True)
        self.h2d_done[s].record(self.copy)

    def take(self, s, inputs, n):
        """the first ``n`` samples of device slot s -> ``inputs`` (static tensors of the spec's fields holding n samples),
        on the current stream after their copy"""
        cur = torch.cuda.current_stream(self.device)
        cur.wait_event(self.h2d_done[s])
        for k, v in inputs.items():
            v.copy_(self.dev[s][k][:n * self.rows[k]])
        self.in_used[s].record(cur)

    def close(self):
        torch.cuda.current_stream(self.device).synchronize()
        self.copy.synchronize()


class JpegBatch:
    """The static inputs of a captured batch and the decode + transform its graph starts with, F = ``frames`` per sample:
    ``inputs`` (device tensors of the fields ``spec``), ``frames`` uint8 [F * B, h, w, 3], ``status`` int32 [F * B]
    (data.JPEG_STATUS) and the decode workspace.  With ``ann``, ``counts`` and ``mirror`` fields it is the train
    transform (``max_labels``, ``flip``), without them the validation transform."""

    def __init__(self, spec, frames, hw, input_size, device, max_labels=50, flip=False):
        self.fpi, self.hw, self.input_size = frames, tuple(hw), tuple(input_size)
        self.kw = dict(max_labels=max_labels, flip=flip, raw=True)
        self.inputs = {k: torch.zeros(shape, dtype=dt, device=device) for k, (shape, dt) in spec.items()}
        n, max_bytes = self.inputs["bytes"].shape
        self.frames = torch.zeros((n, self.hw[0], self.hw[1], 3), dtype=torch.uint8, device=device)
        self.status = torch.zeros((n,), dtype=torch.int32, device=device)
        self.workspace = torch.empty(ops.jpeg_decode_workspace_bytes(n, max_bytes, *self.hw), dtype=torch.uint8,
                                     device=device)

    def run(self, out):
        """decode, then pair_transform / frame_transform (``raw=True``) into ``out`` = (x, labels)"""
        i = self.inputs
        data.decode_jpeg(i["bytes"], i["lengths"], self.hw, out=self.frames, status=self.status, workspace=self.workspace)
        labels = (i["ann"], i["counts"], i["mirror"]) if "ann" in i else (None, None, None)
        if self.fpi == 2:
            data.pair_transform(self.frames.view(-1, 2, self.hw[0], self.hw[1], 3), *labels, self.input_size, out=out,
                                **self.kw)
        else:
            data.frame_transform(self.frames, *labels, self.input_size, out=out, **self.kw)
