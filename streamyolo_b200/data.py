"""The data loader's image transforms on the device, from the uint8 BGR frames the dataset holds to the model's input.

``pair_transform`` = DoubleTrainTransform(max_labels, hsv=False, flip) / DoubleValTransform
(/root/reference/exps/data/data_augment_flip.py:141-234) for a batch of frame pairs, ``frame_transform`` =
TrainTransform / ValTransform (:170-263) for a batch of single frames, ``stream_frame`` = the streaming
driver's preproc (sAP/streamyolo/streamyolo_det.py:57-60, 176-181), ``stream_frames_sized`` the same for frames of
different sizes (the evaluation preproc, data_augment_flip.py:151-167, per frame).  They are bit-identical to the cv2 / numpy host code
they replace (sy_pair_labels, sy_frame_labels, sy_letterbox); INTEGRATION.md shows where they plug in.
"""
import operator

import numpy as np
import torch

from . import ops

# per-image status of decode_jpeg (SY_JPEG_* of include/streamyolo_sm100.h)
JPEG_STATUS = {0: "ok", 1: "malformed or truncated header, or invalid tables", 2: "unsupported JPEG variant "
               "(progressive, arithmetic, lossless, 12-bit, not YCbCr 4:2:0 / 4:2:2 / 4:4:4, or several scans)",
               3: "EXIF orientation other than 1", 4: "image size differs from the batch size",
               5: "corrupt or truncated entropy-coded data"}


def _fit(h, w, size):
    """the scale and (int-truncated) size of an h x w image fitted into ``size`` (preproc, load_resized_img)"""
    r = min(size[0] / h, size[1] / w)
    return r, (int(h * r), int(w * r))


def pair_transform(frames, ann, counts, mirror, input_size, max_labels=50, flip=True, raw=False, hsv=False, out=None):
    """Train / validation transform of a batch of frame pairs.

    frames  uint8 CUDA [B, 2, h, w, 3], BGR, current frame first: the two images of ``pull_item`` (``raw=True``: what
            cv2.imread returned, and load_resized_img's resize runs first)
    ann     float64 [B, 2, M, 5] rows x1, y1, x2, y2, cls as ``pull_item`` scales them (frame 0: the future boxes), or None
            for the validation transform (no labels, no mirror)
    counts  int32 [B, 2] valid rows of ``ann``
    mirror  int32 [B] the pair's random mirror bit (``random.randrange(2)`` of DoubleTrainTransform)
    out     ``(x, (labels_fut, labels_cur))`` of an earlier call to write into (static buffers for CUDA-graph capture)

    -> ``(x, (labels_fut, labels_cur))``: x fp32 [B, 6, H, W], labels fp32 [B, max_labels, 5] (cls, cx, cy, w, h), or
    ``(x, None)`` without annotations.  Nothing is read back to the host."""
    if hsv:
        raise NotImplementedError("pair_transform: HSV augmentation has no device implementation (no TAL cfg enables it)")
    ops._require(torch.is_tensor(frames) and frames.dtype == torch.uint8 and frames.dim() == 5 and frames.shape[1] == 2
                 and frames.shape[4] == 3 and frames.is_contiguous(), "pair_transform: frames must be contiguous uint8 [B, 2, h, w, 3]")
    b, _, h, w, _ = frames.shape
    mid = _fit(h, w, input_size)[1] if raw else (h, w)
    r, dst = _fit(mid[0], mid[1], input_size)
    if out is None:
        x = torch.empty((b, 6, input_size[0], input_size[1]), dtype=torch.float32, device=frames.device)
        labels = None
        if ann is not None:
            labels = tuple(torch.empty((b, max_labels, 5), dtype=torch.float32, device=frames.device) for _ in range(2))
    else:
        x, labels = out
    ops._require(tuple(x.shape) == (b, 6, input_size[0], input_size[1]), "pair_transform: out image must be [B, 6, H, W]")
    flags = None
    if ann is not None:
        ops._require(labels is not None and labels[0].shape[1] == max_labels, "pair_transform: out labels must be [B, max_labels, 5]")
        flags = torch.empty((b, 2), dtype=torch.int32, device=frames.device)
        ops.pair_labels(ann, counts, mirror if flip else None, flip, mid[1], r, labels[0], labels[1], flags)
    ops.letterbox(frames.view(2 * b, h, w, 3), mid, dst, x, flags)
    return x, labels


def frame_transform(frames, ann, counts, mirror, input_size, max_labels=50, flip=True, raw=False, out=None):
    """Train / validation transform of a batch of single frames: TrainTransform(max_labels, hsv=False, flip) / ValTransform
    (/root/reference/exps/data/data_augment_flip.py:170-263), the dataset transform of the still-image baseline
    (cfgs/l_s50_still_dfp_flip.py).

    frames  uint8 CUDA [B, h, w, 3], BGR (``raw=True``: what cv2.imread returned, and load_resized_img's resize runs first)
    ann     float64 [B, M, 5] rows x1, y1, x2, y2, cls, or None for the validation transform (no labels, no mirror)
    counts  int32 [B] valid rows of ``ann``
    mirror  int32 [B] each frame's random mirror bit (``random.randrange(2)`` of TrainTransform)
    out     ``(x, labels)`` of an earlier call to write into (static buffers for CUDA-graph capture)

    -> ``(x, labels)``: x fp32 [B, 3, H, W], labels fp32 [B, max_labels, 5] (cls, cx, cy, w, h), or ``(x, None)`` without
    annotations.  Nothing is read back to the host."""
    ops._require(torch.is_tensor(frames) and frames.dtype == torch.uint8 and frames.dim() == 4 and frames.shape[3] == 3
                 and frames.is_contiguous(), "frame_transform: frames must be contiguous uint8 [B, h, w, 3]")
    b, h, w, _ = frames.shape
    mid = _fit(h, w, input_size)[1] if raw else (h, w)
    r, dst = _fit(mid[0], mid[1], input_size)
    if out is None:
        x = torch.empty((b, 3, input_size[0], input_size[1]), dtype=torch.float32, device=frames.device)
        labels = None
        if ann is not None:
            labels = torch.empty((b, max_labels, 5), dtype=torch.float32, device=frames.device)
    else:
        x, labels = out
    ops._require(torch.is_tensor(x) and tuple(x.shape) == (b, 3, input_size[0], input_size[1]),
                 "frame_transform: out image must be [B, 3, H, W]")
    flags = None
    if ann is not None:
        ops._require(torch.is_tensor(labels) and labels.dim() == 3 and labels.shape[1] == max_labels,
                     "frame_transform: out labels must be [B, max_labels, 5]")
        flags = torch.empty((b,), dtype=torch.int32, device=frames.device)
        ops.frame_labels(ann, counts, mirror if flip else None, flip, mid[1], r, labels, flags)
    ops.letterbox(frames, mid, dst, x, flags)
    return x, labels


def preprocess(x, labels, tsize, input_size, out=None):
    """``Exp.preprocess(x, labels, tsize)`` (StreamYOLO's cfgs/s_s50_onex_dfp_tal_flip.py:160-171, the same in every
    cfg) on the device: at a multi-scale size ``tsize`` other than ``input_size`` a bilinear resize (sy_resize_bilinear) and
    ``labels[0][..., 1::2] *= sx``, ``labels[0][..., 2::2] *= sy``, the same for ``labels[1]`` (sy_scale_labels).  As in
    the cfgs, ``labels`` is the (future, current) pair, or for a still model one label tensor whose images 0 and 1 are
    rescaled.  At ``input_size`` nothing runs and ``(x, labels)`` come back as they are.

    out  ``(x, labels)`` static buffers of size ``tsize`` (a CUDA graph's inputs): the resize writes there and the labels are
         copied there before they are scaled, so ``labels`` is left unchanged.  Without it the labels are scaled in place,
         like the cfgs do."""
    scale_y, scale_x = tsize[0] / input_size[0], tsize[1] / input_size[1]
    if scale_x == 1 and scale_y == 1:
        return x, labels
    if out is not None:
        l_out = out[1]
        if torch.is_tensor(labels):
            l_out.copy_(labels)
        else:
            for dst, src in zip(l_out, labels):
                dst.copy_(src)
        labels = l_out
    x = ops.resize_bilinear(x, tuple(tsize), out=None if out is None else out[0])
    for t in (labels[0], labels[1]):
        ops.scale_labels_(t, scale_x, scale_y)
    return x, labels


def stream_frame(frame, size=(600, 960), out=None):
    """streamyolo_det.preproc(frame, size) followed by torch.from_numpy(.).float()[None]: uint8 CUDA [h, w, 3] BGR ->
    fp32 [1, 3, H, W], a plain (possibly non-uniform) cv2-exact resize without pad or mirror."""
    ops._require(torch.is_tensor(frame) and frame.dtype == torch.uint8 and frame.dim() == 3 and frame.shape[2] == 3
                 and frame.is_contiguous(), "stream_frame: frame must be contiguous uint8 [h, w, 3]")
    h, w, _ = frame.shape
    if out is None:
        out = torch.empty((1, 3, size[0], size[1]), dtype=torch.float32, device=frame.device)
    ops._require(tuple(out.shape) == (1, 3, size[0], size[1]), "stream_frame: out must be [1, 3, H, W]")
    ops.letterbox(frame.view(1, h, w, 3), (h, w), size, out)
    return out


def _sizes_list(sizes, who):
    """``sizes`` ([(h, w), ...] or an int [n, 2] array) as a list of int pairs, each at least 1x1"""
    out = [tuple(int(v) for v in s) for s in np.asarray(sizes).reshape(-1, 2).tolist()]
    ops._require(len(out) > 0 and all(h >= 1 and w >= 1 for h, w in out), f"{who}: sizes must be (h, w) pairs of at least 1")
    return out


def sized_table(sizes, input_size, in_scale=None):
    """The per-frame transform of frames of different sizes into one ``input_size`` (H, W) model input.

    A frame whose driver size (int(h * in_scale), int(w * in_scale)) is ``input_size`` gets the streaming driver's plain
    resize to H x W and the ratio ``in_scale`` (streamyolo_det.py:57-60, 176-181, 82); every other frame (all of them without
    ``in_scale``) the evaluation preproc: r = min(H / h, W / w), a resize to (int(h * r), int(w * r)) and the 114 pad, with
    the ratio r its boxes are divided by (data_augment_flip.py:151-167, onex_stream_evaluator.py:182).

    -> (int32 numpy [n, 4] rows h, w, dst_h, dst_w -- sy_letterbox_sized's table -- and the n ratios as Python floats)."""
    rows, ratios = [], []
    for h, w in _sizes_list(sizes, "sized_table"):
        if in_scale is not None and (int(h * in_scale), int(w * in_scale)) == tuple(input_size):
            r, dst = in_scale, tuple(input_size)
        else:
            r, dst = _fit(h, w, input_size)
        ops._require(min(dst) >= 1, f"sized_table: a {h}x{w} frame fitted into {tuple(input_size)} is empty")
        rows.append((h, w, dst[0], dst[1]))
        ratios.append(r)
    return np.array(rows, np.int32), ratios


def stream_frames_sized(frames, sizes, input_size, out=None, in_scale=None):
    """``preproc`` per frame for frames of different sizes (sy_letterbox_sized).

    frames  uint8 CUDA [n, max_h, max_w, 3] slots (decode_jpeg_sized's output): frame i BGR at the top-left of slot i
    sizes   the n frames' (h, w), each within the slot
    in_scale  with it, a frame of driver size ``input_size`` takes the driver's plain resize (see sized_table)

    -> ``(x, ratios)``: x fp32 [n, 3, H, W], what ``preproc(frame_i, input_size)`` gives with the 114 pad, and each frame's
    ratio (the r its boxes are divided by)."""
    sizes = _sizes_list(sizes, "stream_frames_sized")
    ops._require(torch.is_tensor(frames) and frames.dtype == torch.uint8 and frames.dim() == 4 and frames.shape[3] == 3
                 and frames.is_contiguous() and frames.shape[0] == len(sizes),
                 f"stream_frames_sized: frames must be contiguous uint8 [{len(sizes)}, max_h, max_w, 3]")
    n, sh, sw, _ = frames.shape
    for i, (h, w) in enumerate(sizes):
        ops._require(h <= sh and w <= sw, f"stream_frames_sized: frame {i} of {h}x{w} is larger than the {sh}x{sw} slot")
    table, ratios = sized_table(sizes, input_size, in_scale)
    if out is None:
        out = torch.empty((n, 3, input_size[0], input_size[1]), dtype=torch.float32, device=frames.device)
    ops._require(tuple(out.shape) == (n, 3, input_size[0], input_size[1]), "stream_frames_sized: out must be [n, 3, H, W]")
    ops.letterbox_sized(frames, torch.from_numpy(table).to(frames.device), out)
    return out, ratios


def pack_jpeg(files, max_bytes):
    """Host side of device JPEG decoding: the file contents ``files`` (``bytes`` or uint8 numpy arrays, e.g.
    ``np.fromfile(path, np.uint8)``) -> (uint8 [N, max_bytes] zero-padded rows, int32 [N] lengths), both numpy, for the
    dataset's ``pull_item`` / collate.  A file longer than ``max_bytes`` raises ValueError."""
    rows = np.zeros((len(files), max_bytes), np.uint8)
    lengths = np.zeros(len(files), np.int32)
    for i, f in enumerate(files):
        a = np.frombuffer(f, np.uint8) if isinstance(f, (bytes, bytearray, memoryview)) else np.asarray(f, np.uint8).ravel()
        if a.size > max_bytes:
            raise ValueError(f"pack_jpeg: file {i} has {a.size} bytes, more than max_bytes = {max_bytes}")
        rows[i, :a.size] = a
        lengths[i] = a.size
    return rows, lengths


_JPEG_WS = {}


def decode_jpeg(streams, lengths, hw, out=None, status=None, workspace=None):
    """Decode a batch of JPEG files on the device into what cv2.imread returns for them (sy_jpeg_decode).

    streams   uint8 CUDA [N, max_bytes] file bytes (pack_jpeg's rows, copied to the device)
    lengths   int32 CUDA [N]
    hw        (H, W) every frame must have
    out, status, workspace   uint8 [N, H, W, 3], int32 [N] and the uint8 workspace to write into (static buffers for
              CUDA-graph capture); new ones when omitted (the workspace is then cached per device and shape)

    -> ``(frames, status)``: frames uint8 [N, H, W, 3] BGR, the ``raw=True`` input of pair_transform (viewed as
    [N / 2, 2, H, W, 3]) and frame_transform; status int32 [N], 0 where the frame decoded, else a JPEG_STATUS code and
    that frame is left as it was.  Nothing is read back: check_jpeg_status is the synchronising check."""
    ops._require(torch.is_tensor(streams) and streams.dim() == 2 and streams.is_cuda,
                 "decode_jpeg: streams must be a CUDA uint8 [N, max_bytes] tensor")
    n, max_bytes = streams.shape
    h, w = hw
    dev = streams.device
    if out is None:
        out = torch.empty((n, h, w, 3), dtype=torch.uint8, device=dev)
    if status is None:
        status = torch.empty((n,), dtype=torch.int32, device=dev)
    ops._require(tuple(out.shape) == (n, h, w, 3), f"decode_jpeg: out must be [{n}, {h}, {w}, 3]")
    if workspace is None:
        key = (dev, n, max_bytes, h, w)
        if key not in _JPEG_WS:
            _JPEG_WS[key] = torch.empty(ops.jpeg_decode_workspace_bytes(n, max_bytes, h, w), dtype=torch.uint8, device=dev)
        workspace = _JPEG_WS[key]
    ops.jpeg_decode(streams, lengths, out, status, workspace)
    return out, status


def check_jpeg_status(status):
    """Synchronising check of decode_jpeg's status: raises RuntimeError naming the first frame that did not decode and why."""
    st = status.cpu().tolist()
    for i, s in enumerate(st):
        if s != 0:
            raise RuntimeError(f"decode_jpeg: frame {i} did not decode: {JPEG_STATUS.get(s, f'status {s}')}")


def decode_jpeg_sized(streams, lengths, sizes, max_hw, out=None, status=None, workspace=None):
    """Decode a batch of JPEG files of different sizes on the device (sy_jpeg_decode_sized).

    streams, lengths  as decode_jpeg
    sizes     the (h, w) each frame must have: host pairs (checked against ``max_hw`` here) or an int32 CUDA [N, 2] tensor
              (static for CUDA-graph capture; a frame larger than the slot then gets status 4)
    max_hw    (max_h, max_w) of the output slots
    out, status, workspace   uint8 [N, max_h, max_w, 3], int32 [N] and the workspace to write into, as decode_jpeg

    -> ``(frames, status)``: frame i what cv2.imread returns for file i, at the top-left of slot i (the rest of the slot is
    not written); status as decode_jpeg.  Nothing is read back."""
    mh, mw = (int(v) for v in max_hw)
    if not torch.is_tensor(sizes):
        hw = _sizes_list(sizes, "decode_jpeg_sized")
        for i, (h, w) in enumerate(hw):
            ops._require(h <= mh and w <= mw, f"decode_jpeg_sized: frame {i} of {h}x{w} is larger than the {mh}x{mw} slot")
        sizes = torch.tensor(hw, dtype=torch.int32)
    ops._require(sizes.dtype == torch.int32 and tuple(sizes.shape) == (sizes.shape[0], 2),
                 "decode_jpeg_sized: sizes must be int32 [N, 2]")
    ops._require(torch.is_tensor(streams) and streams.dim() == 2 and streams.dtype == torch.uint8 and streams.is_cuda,
                 "decode_jpeg_sized: streams must be a CUDA uint8 [N, max_bytes] tensor")
    n, max_bytes = streams.shape
    ops._require(sizes.shape[0] == n, f"decode_jpeg_sized: {sizes.shape[0]} sizes for {n} files")
    dev = streams.device
    sizes = sizes.to(dev)
    if out is None:
        out = torch.empty((n, mh, mw, 3), dtype=torch.uint8, device=dev)
    if status is None:
        status = torch.empty((n,), dtype=torch.int32, device=dev)
    ops._require(tuple(out.shape) == (n, mh, mw, 3), f"decode_jpeg_sized: out must be [{n}, {mh}, {mw}, 3]")
    if workspace is None:
        key = (dev, n, max_bytes, mh, mw)
        if key not in _JPEG_WS:
            _JPEG_WS[key] = torch.empty(ops.jpeg_decode_sized_workspace_bytes(n, max_bytes, mh, mw), dtype=torch.uint8,
                                        device=dev)
        workspace = _JPEG_WS[key]
    ops.jpeg_decode_sized(streams, lengths, sizes, out, status, workspace)
    return out, status


# per-image status of encode_jpeg (SY_JPEG_ENCODE_* of include/streamyolo_sm100.h)
ENCODE_STATUS = {0: "ok", 1: "the file does not fit in max_bytes", 2: "its size is outside the slot"}
_ENC_WS = {}


def encode_jpeg(frames, quality=95, sizes=None, max_bytes=None, out=None, workspace=None):
    """Encode uint8 BGR frames on the device into the files cv2.imencode(".jpg", frame, [cv2.IMWRITE_JPEG_QUALITY,
    quality]) returns, byte for byte (sy_jpeg_encode: baseline, 4:2:0, standard Huffman tables, JFIF), which
    cv2.imwrite(path, frame, ...) would write.

    frames    uint8 CUDA [n, h, w, 3]; or slots [n, max_h, max_w, 3] (decode_jpeg_sized's or the streaming detector's
              ``frames``) with ``sizes``
    sizes     each frame's (h, w) at the top-left of its slot: host pairs (checked here) or an int32 CUDA [n, 2] tensor
              (read on the device only, static for CUDA-graph capture)
    max_bytes the longest file to make room for (the row length of the output); default ``ops.jpeg_encode_max_bytes``
              of the slot, which no frame of the slot's size exceeds
    out       ``(buf, lengths, status)``: uint8 [n, max_bytes], int64 [n] and int32 [n] device buffers to write into.  The
              call then only enqueues the encode (capturable) and returns ``out``; ``jpeg_files(*out)`` reads them back
    workspace the uint8 workspace (ops.jpeg_encode_workspace_bytes) to use; cached per device and shape when omitted

    -> a list of n ``bytes``, the files (one synchronisation).  A file longer than ``max_bytes`` raises ValueError
    naming the frame."""
    ops._require(torch.is_tensor(frames) and frames.dtype == torch.uint8 and frames.dim() == 4 and frames.shape[3] == 3
                 and frames.is_contiguous() and frames.is_cuda,
                 "encode_jpeg: frames must be a contiguous CUDA uint8 [n, h, w, 3] tensor")
    try:
        quality = operator.index(quality)
    except TypeError:
        raise RuntimeError(f"encode_jpeg: quality must be an integer in 1..100, not {quality!r}") from None
    ops._require(1 <= quality <= 100, f"encode_jpeg: quality must be an integer in 1..100, not {quality}")
    n, mh, mw, _ = frames.shape
    dev = frames.device
    if sizes is None:
        sizes = [(mh, mw)] * n
    if not torch.is_tensor(sizes):
        hw = _sizes_list(sizes, "encode_jpeg")
        ops._require(len(hw) == n, f"encode_jpeg: {len(hw)} sizes for {n} frames")
        for i, (h, w) in enumerate(hw):
            ops._require(h <= mh and w <= mw, f"encode_jpeg: frame {i} of {h}x{w} is larger than the {mh}x{mw} slot")
        sizes = torch.tensor(hw, dtype=torch.int32)
    ops._require(sizes.dtype == torch.int32 and tuple(sizes.shape) == (n, 2), f"encode_jpeg: sizes must be int32 [{n}, 2]")
    sizes = sizes.to(dev).contiguous()
    if out is None:
        if max_bytes is None:
            max_bytes = ops.jpeg_encode_max_bytes(mh, mw)
        buf = torch.empty((n, int(max_bytes)), dtype=torch.uint8, device=dev)
        lengths = torch.empty((n,), dtype=torch.int64, device=dev)
        status = torch.empty((n,), dtype=torch.int32, device=dev)
    else:
        buf, lengths, status = out
        ops._require(torch.is_tensor(buf) and buf.dim() == 2 and (max_bytes is None or buf.shape[1] == max_bytes),
                     "encode_jpeg: out's buffer must be uint8 [n, max_bytes]")
    if workspace is None:
        key = (dev, n, mh, mw, buf.shape[1])
        if key not in _ENC_WS:
            _ENC_WS[key] = torch.empty(ops.jpeg_encode_workspace_bytes(n, mh, mw, buf.shape[1]), dtype=torch.uint8,
                                       device=dev)
        workspace = _ENC_WS[key]
    ops.jpeg_encode(frames, sizes, quality, buf, lengths, status, workspace)
    if out is not None:
        return out
    return jpeg_files(buf, lengths, status)


def jpeg_files(buf, lengths, status, present=None, stage=None):
    """encode_jpeg's output -> a list of ``bytes``: exactly each file's length is copied back, with one synchronisation.
    ``lengths`` / ``status`` may already be on the host; ``present``: which rows to read (None for the others, whose status
    is not checked); ``stage``: a page-locked uint8 host tensor of at least the files' total length to copy through (a new
    one otherwise).  A file that did not fit raises ValueError naming its frame."""
    n = buf.shape[0]
    present = [True] * n if present is None else [bool(p) for p in present]
    st, ln = status.cpu().tolist(), lengths.cpu().tolist()
    for i in range(n):
        if present[i] and st[i] != 0:
            raise ValueError(f"encode_jpeg: frame {i} was not encoded: {ENCODE_STATUS.get(st[i], f'status {st[i]}')}"
                             + (f" (max_bytes = {buf.shape[1]})" if st[i] == 1 else ""))
    total = sum(l for l, p in zip(ln, present) if p)
    if stage is None or stage.numel() < total:
        stage = torch.empty((max(total, 1),), dtype=torch.uint8, pin_memory=True)
    spans, at = [], 0
    for i in range(n):
        if not present[i]:
            spans.append(None)
            continue
        stage[at:at + ln[i]].copy_(buf[i, :ln[i]], non_blocking=True)
        spans.append((at, at + ln[i]))
        at += ln[i]
    torch.cuda.current_stream(buf.device).synchronize()
    host = stage.numpy()
    return [None if sp is None else host[sp[0]:sp[1]].tobytes() for sp in spans]


def _device_int32(v, dev, what):
    """``v`` (numpy, a list or a tensor) as a contiguous int32 tensor on ``dev``"""
    t = v if torch.is_tensor(v) else torch.from_numpy(np.ascontiguousarray(np.asarray(v)))
    ops._require(not t.is_floating_point() and not t.is_complex(), f"draw_boxes: {what} must be integers, not {t.dtype}")
    return t.to(device=dev, dtype=torch.int32).contiguous()


def draw_boxes(frames, boxes, labels, counts, palette, sizes=None, out=None):
    """Draw detections as the sAP toolkit's visualisation does (vis_obj_fancy of sAP/vis/vis_det_th.py with
    show_label=False, show_score=False; sy_draw_boxes): each box filled at 0.8 / 0.2 over the frame, then outlined two
    pixels wide, in its label's palette colour, later boxes over earlier ones.

    frames    uint8 CUDA [n, h, w, 3]; or slots [n, max_h, max_w, 3] with ``sizes`` (decode_jpeg_sized's output)
    boxes     int32 [n, K, 4] x1, y1, x2, y2, already rounded (vis_obj_fancy's ``bboxes.round().astype(np.int32)``); or a
              list of n [k_i, 4] arrays, which sets ``counts``
    labels    int32 [n, K] (or a list of n [k_i] arrays), each in [0, P)
    counts    int32 [n]: the first counts[i] boxes of row i are drawn (None with lists)
    palette   uint8 [P, 3] in the frames' channel order: (B, G, R) for BGR frames
    sizes     each frame's (h, w) at the top-left of its slot: host pairs or an int32 CUDA [n, 2] tensor
    out       None: draw in place on ``frames`` and return them.  A uint8 tensor of ``frames``' shape: draw ``frames``
              into it, leaving ``frames`` alone; only the pixels a box touches are written, so ``out`` should hold a copy
              of the frames.  With ``out`` every other argument must already be a CUDA tensor, and the call only enqueues
              the kernel (capturable in a CUDA graph, which then follows the boxes and counts written before each replay)

    Host arguments are copied to the device (no synchronisation); nothing is read back."""
    ops._require(torch.is_tensor(frames) and frames.dtype == torch.uint8 and frames.dim() == 4 and frames.shape[3] == 3
                 and frames.is_contiguous() and frames.is_cuda,
                 "draw_boxes: frames must be a contiguous CUDA uint8 [n, h, w, 3] tensor")
    n, mh, mw, _ = frames.shape
    dev = frames.device
    if out is not None:
        args = {"boxes": boxes, "labels": labels, "counts": counts, "palette": palette}
        if sizes is not None:
            args["sizes"] = sizes
        for k, v in args.items():
            ops._require(torch.is_tensor(v) and v.is_cuda, f"draw_boxes: with out=, {k} must be a CUDA tensor")
    if isinstance(boxes, (list, tuple)):
        ops._require(counts is None and isinstance(labels, (list, tuple)) and len(boxes) == n and len(labels) == n,
                     f"draw_boxes: give {n} box arrays and {n} label arrays, and no counts")
        bl = [np.asarray(b, np.int64).reshape(-1, 4) for b in boxes]
        ll = [np.asarray(l, np.int64).reshape(-1) for l in labels]
        ops._require(all(len(b) == len(l) for b, l in zip(bl, ll)), "draw_boxes: each frame needs one label per box")
        k = max([1] + [len(b) for b in bl])
        bx, lb = np.zeros((n, k, 4), np.int64), np.zeros((n, k), np.int64)
        for i, (b, l) in enumerate(zip(bl, ll)):
            bx[i, :len(b)], lb[i, :len(l)] = b, l
        boxes, labels, counts = bx, lb, [len(b) for b in bl]
    for name, v in (("boxes", boxes), ("labels", labels), ("counts", counts)):
        if not torch.is_tensor(v):
            a = np.asarray(v)
            ops._require(a.dtype.kind in "iub" and (a.size == 0 or (a.min() >= -2 ** 31 and a.max() < 2 ** 31)),
                         f"draw_boxes: {name} must be int32 values")
    boxes, labels, counts = (_device_int32(v, dev, k) for v, k in ((boxes, "boxes"), (labels, "labels"),
                                                                    (counts, "counts")))
    pal = palette if torch.is_tensor(palette) else torch.from_numpy(np.ascontiguousarray(np.asarray(palette, np.uint8)))
    pal = pal.to(dev).contiguous()
    if sizes is None:
        sizes = [(mh, mw)] * n
    if not torch.is_tensor(sizes):
        hw = _sizes_list(sizes, "draw_boxes")
        ops._require(len(hw) == n, f"draw_boxes: {len(hw)} sizes for {n} frames")
        for i, (h, w) in enumerate(hw):
            ops._require(h <= mh and w <= mw, f"draw_boxes: frame {i} of {h}x{w} is larger than the {mh}x{mw} slot")
        sizes = torch.tensor(hw, dtype=torch.int32)
    ops._require(sizes.dtype == torch.int32 and tuple(sizes.shape) == (n, 2), f"draw_boxes: sizes must be int32 [{n}, 2]")
    sizes = sizes.to(dev).contiguous()
    if boxes.dim() == 3 and boxes.data_ptr() % 16:
        boxes = boxes.clone()
    return ops.draw_boxes(frames, sizes, boxes, labels, counts, pal, frames if out is None else out)


def imrescale_size(h, w, scale):
    """The (h, w) mmcv.imrescale(img, scale) gives an h x w image (mmcv.image.rescale_size with a number:
    ``int(w * scale + 0.5), int(h * scale + 0.5)``); ValueError for a scale <= 0, as mmcv raises, and for an empty result,
    which cv2.resize refuses."""
    if not scale > 0:
        raise ValueError(f"Invalid scale {scale}, must be positive.")
    out = int(h * float(scale) + 0.5), int(w * float(scale) + 0.5)
    if min(out) < 1:
        raise ValueError(f"imrescale: a {h}x{w} image at scale {scale} is empty ({out[0]}x{out[1]})")
    return out


def resize_sized(frames, sizes, dst_sizes, out_hw=None, out=None):
    """Resize frames of different sizes as cv2.resize(img, (dst_w, dst_h), interpolation=INTER_LINEAR) does, bit for bit
    (sy_resize_sized; mmcv.imrescale's bilinear resize with ``dst_sizes`` from imrescale_size).

    frames    uint8 CUDA [n, slot_h, slot_w, 3] slots (decode_jpeg_sized's output), channel order kept
    sizes     each frame's (h, w) at the top-left of its slot; dst_sizes: each frame's (dst_h, dst_w)
    out_hw    the output slots' (h, w): the largest dst size by default
    out       uint8 [n, out_h, out_w, 3] to write into; with it and an int32 CUDA [n, 4] ``sizes`` table (h, w, dst_h,
              dst_w; ``dst_sizes`` None) the call only enqueues (capturable)

    -> ``out``: frame i at the top-left of slot i; the rest of each slot is not written."""
    ops._require(torch.is_tensor(frames) and frames.dtype == torch.uint8 and frames.dim() == 4 and frames.shape[3] == 3
                 and frames.is_contiguous() and frames.is_cuda,
                 "resize_sized: frames must be a contiguous CUDA uint8 [n, slot_h, slot_w, 3] tensor")
    n, sh, sw, _ = frames.shape
    dev = frames.device
    if torch.is_tensor(sizes):
        ops._require(dst_sizes is None, "resize_sized: with a sizes table, give no dst_sizes")
        table = sizes
    else:
        src, dst = _sizes_list(sizes, "resize_sized"), _sizes_list(dst_sizes, "resize_sized")
        ops._require(len(src) == n and len(dst) == n, f"resize_sized: give {n} sizes and {n} dst sizes")
        for i, (h, w) in enumerate(src):
            ops._require(h <= sh and w <= sw, f"resize_sized: frame {i} of {h}x{w} is larger than the {sh}x{sw} slot")
        table = torch.tensor([s + d for s, d in zip(src, dst)], dtype=torch.int32)
        if out_hw is None and out is None:
            out_hw = (max(h for h, _ in dst), max(w for _, w in dst))
        if out is not None:
            out_hw = tuple(out.shape[1:3])
        for i, (h, w) in enumerate(dst):
            ops._require(h <= out_hw[0] and w <= out_hw[1], f"resize_sized: frame {i} resized to {h}x{w} is larger "
                         f"than the {out_hw[0]}x{out_hw[1]} output slot")
    if out is None:
        ops._require(out_hw is not None, "resize_sized: give out_hw or out")
        out = torch.empty((n, int(out_hw[0]), int(out_hw[1]), 3), dtype=torch.uint8, device=dev)
    return ops.resize_sized(frames, table.to(dev).contiguous(), out)


# vis_det's box and text colour (0, 255, 0): the same in RGB and BGR order
VIS_DET_GREEN = (0, 255, 0)


def draw_outlines(frames, boxes, points, sizes=None, counts=None, n_points=None, color=VIS_DET_GREEN):
    """Draw detections as the sAP toolkit's vis_det does (sAP/det/__init__.py:152-174; sy_draw_outlines), in place:
    each box as cv2.rectangle(img, (x1, y1), (x2, y2), color, thickness=1) draws it, and the listed pixels (the label
    text the host rasterised with cv2.putText) in the same colour.

    frames    uint8 CUDA [n, h, w, 3]; or slots [n, max_h, max_w, 3] with ``sizes``
    boxes     int32 [n, K, 4] x1, y1, x2, y2, already rounded (vis_det's ``bboxes.round().astype(np.int32)``), with
              ``counts``; or a list of n [k_i, 4] arrays
    points    int32 [n, M] pixel indices y * w + x within each frame, with ``n_points``; or a list of n index arrays
    sizes     each frame's (h, w) at the top-left of its slot: host pairs or an int32 CUDA [n, 2] tensor
    color     3 values in the frames' channel order

    With every argument a CUDA tensor the call only enqueues the kernel (capturable in a CUDA graph, which then follows
    what is written to the tensors before each replay); host arguments are copied to the device (no synchronisation).
    Only the pixels a box or a listed index touches are written.  -> ``frames``."""
    ops._require(torch.is_tensor(frames) and frames.dtype == torch.uint8 and frames.dim() == 4 and frames.shape[3] == 3
                 and frames.is_contiguous() and frames.is_cuda,
                 "draw_outlines: frames must be a contiguous CUDA uint8 [n, h, w, 3] tensor")
    n, mh, mw, _ = frames.shape
    dev = frames.device

    def rows(v, c, width, what):
        if torch.is_tensor(v):
            ops._require(torch.is_tensor(c), f"draw_outlines: give {what} counts with a {what} tensor")
            return v, c
        ops._require(c is None and len(v) == n, f"draw_outlines: give {n} {what} arrays and no counts")
        arrs = [np.asarray(a, np.int64).reshape((-1, 4) if width == 4 else (-1,)) for a in v]
        ops._require(all(a.size == 0 or (a.min() >= -2 ** 31 and a.max() < 2 ** 31) for a in arrs),
                     f"draw_outlines: {what} must be int32 values")
        k = max([1] + [len(a) for a in arrs])
        packed = np.zeros((n, k, 4) if width == 4 else (n, k), np.int32)
        for i, a in enumerate(arrs):
            packed[i, :len(a)] = a
        return torch.from_numpy(packed), torch.tensor([len(a) for a in arrs], dtype=torch.int32)

    boxes, counts = rows(boxes, counts, 4, "box")
    points, n_points = rows(points, n_points, 1, "point")
    if sizes is None:
        sizes = [(mh, mw)] * n
    if not torch.is_tensor(sizes):
        hw = _sizes_list(sizes, "draw_outlines")
        ops._require(len(hw) == n, f"draw_outlines: {len(hw)} sizes for {n} frames")
        for i, (h, w) in enumerate(hw):
            ops._require(h <= mh and w <= mw, f"draw_outlines: frame {i} of {h}x{w} is larger than the {mh}x{mw} slot")
        sizes = torch.tensor(hw, dtype=torch.int32)
    boxes, counts, points, n_points, sizes = (t.to(dev).contiguous() for t in (boxes, counts, points, n_points, sizes))
    if boxes.data_ptr() % 16:
        boxes = boxes.clone()
    return ops.draw_outlines(frames, sizes, boxes, counts, points, n_points, color)


# the band colour of the sAP toolkit's vis_contrast.py (RGB [241, 159, 93], :106) in BGR order
CONTRAST_BAND_BGR = (93, 159, 241)


def splice_frames(a, b, splits, sizes=None, horizontal=False, color=CONTRAST_BAND_BGR):
    """Compose split-screen frames as the sAP toolkit's vis_contrast.py does (:148-165; sy_splice_frames): frame B from
    the split line on, frame A before it, and a band of ``color`` over both, written into ``a`` in place.

    a, b      uint8 CUDA [n, h, w, 3], or slots [n, max_h, max_w, 3] with ``sizes`` (decode_jpeg_sized's output); two
              different tensors of one shape
    splits    per frame (split, band_start, band_end): columns, or rows with ``horizontal``, at or past ``split`` take B's
              pixels, and [band_start, band_end) takes the band colour.  Host triples or an int32 CUDA [n, 3] tensor
    sizes     each pair's (h, w) at the top-left of its slots: host pairs (checked here) or an int32 CUDA [n, 2] tensor
    color     the band colour in the frames' channel order: the script's, for BGR frames, by default

    Host arguments are copied to the device (no synchronisation); with every argument a CUDA tensor the call only
    enqueues the kernel, so it can be captured in a CUDA graph, which then follows the splits and sizes written before
    each replay.  Pixels outside each frame, and A's pixels before the split outside the band, are not written."""
    ops._require(torch.is_tensor(a) and a.dtype == torch.uint8 and a.dim() == 4 and a.shape[3] == 3
                 and a.is_contiguous() and a.is_cuda, "splice_frames: a must be a contiguous CUDA uint8 [n, h, w, 3] tensor")
    n, mh, mw, _ = a.shape
    dev = a.device
    if not torch.is_tensor(splits):
        sp = np.asarray(splits, np.int64).reshape(-1, 3) if len(splits) else np.zeros((0, 3), np.int64)
        ops._require(len(sp) == n, f"splice_frames: {len(sp)} splits for {n} frames")
        ops._require(sp.size == 0 or (sp.min() >= -2 ** 31 and sp.max() < 2 ** 31), "splice_frames: splits must be "
                     "int32 values")
        splits = torch.from_numpy(sp.astype(np.int32))
    ops._require(splits.dtype == torch.int32 and tuple(splits.shape) == (n, 3), f"splice_frames: splits must be int32 "
                 f"[{n}, 3]")
    if sizes is None:
        sizes = [(mh, mw)] * n
    if not torch.is_tensor(sizes):
        hw = _sizes_list(sizes, "splice_frames")
        ops._require(len(hw) == n, f"splice_frames: {len(hw)} sizes for {n} frames")
        for i, (h, w) in enumerate(hw):
            ops._require(h <= mh and w <= mw, f"splice_frames: frame {i} of {h}x{w} is larger than the {mh}x{mw} slot")
        sizes = torch.tensor(hw, dtype=torch.int32)
    ops._require(sizes.dtype == torch.int32 and tuple(sizes.shape) == (n, 2), f"splice_frames: sizes must be int32 [{n}, 2]")
    return ops.splice_frames(a, b, sizes.to(dev).contiguous(), splits.to(dev).contiguous(), horizontal, color)
