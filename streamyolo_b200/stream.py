"""The streaming detector: the sAP driver's per-frame loop (sAP/streamyolo/streamyolo_det.py:150-195) as ONE CUDA graph
replay per frame, for one camera stream or several batched together, each stream with a frame size of its own.

    det = StreamDetector(model, frame_hw=(1200, 1920), in_scale=0.5, streams=1)   # model in eval(), weights loaded
    det.reset()                                   # every stream starts a sequence (det.reset(i): stream i only)
    bboxes, scores, labels = det.step(frame)[0]   # what the driver's inference() returns for that frame

One tick runs, for the S streams at once: the resize of each stream's uint8 frame with its own transform (data.sized_table:
the driver's plain resize, ``data.stream_frame``, for a frame whose driver size is the input size, the evaluation
letterbox otherwise; sy_letterbox_sized), the backbone + PAFPN on the current frames, the per-stream choice of the support features
(the current ones for a stream that starts a sequence -- the star node of dfp_pafpn.py:177-228 -- the carried buffer
otherwise), the DFP fusion, the buffer update, the head, the NMS (``sy_postprocess_nms`` with room for every anchor) and
the division of each stream's boxes by its own ratio (``in_scale`` for the driver's resize; sy_stream_rescale).  Around
the replay ``step`` copies the frames in and the detections out through pinned host memory and synchronises once.

Streams of different sizes, fed JPEG bytes (a camera rig):

    det = StreamDetector(model, frame_sizes=[(1200, 1920), (2048, 1550), (1550, 2048)], input_size=(600, 960),
                         in_scale=0.5, jpeg_max_bytes=1 << 20)
    for (bboxes, scores, labels) in det.step_jpeg([jpeg0, jpeg1, None]):   # None: no frame from that camera this tick
        ...
    det.last_status()                             # per stream: 0 decoded, a data.JPEG_STATUS code, or NO_FRAME

Then the tick starts with the decode of the S files (sy_jpeg_decode_sized) into slots of the largest size.  A stream whose
frame did not decode, or that got none, keeps its carried features, starts no sequence and returns no detections
(sy_stream_gate, sy_stream_rescale): all decided on the device, still one replay and one synchronisation per tick.

Raw camera frames (YUV, as ISPs, hardware codecs, V4L2 and GMSL deliver them):

    det = StreamDetector(model, frame_sizes=[(1200, 1920), (1080, 1920)], input_size=(600, 960), frame_format="nv12")
    det.step([nv12_0, nv12_1])                    # uint8 [h * 3 // 2, w] each, what cv2.cvtColor(COLOR_YUV2BGR_NV12) takes

Then the tick starts with the conversion of the S frames to BGR (sy_yuv_to_bgr_sized, cv2.cvtColor bit for bit) into the
slots; only each frame's own bytes cross to the device.  Raw sensor frames (8-bit Bayer mosaics, before any ISP) likewise:

    det = StreamDetector(model, frame_sizes=[(1200, 1920)] * 8, input_size=(600, 960), frame_format="bayer_rggb",
                         demosaic="ea")
    det.step(raws)                                # uint8 [h, w] each, what cv2.cvtColor(COLOR_BayerRGGB2BGR_EA) takes

and the tick starts with their demosaicing (sy_bayer_to_bgr_sized, cv2.cvtColor bit for bit).

The graph reads the weights and the folded BatchNorm as they were at capture: after ``load_state_dict`` (or any other
change of the weights or running statistics) call ``capture()`` again.  Nothing checks this per frame.
"""
import time

import numpy as np
import torch

from . import data, feed, ops
from .model import engine


class StreamTick:
    """The work of one tick on static buffers -- what ``StreamDetector`` captures as a CUDA graph.  ``frames`` (uint8
    [S, max_h, max_w, 3] slots, stream i's frame at the top-left of slot i) and ``flags`` (int32 [S], set = the stream
    starts a sequence) are the inputs; ``table`` holds the static int32 [S, 4] rows of data.sized_table and ``ratio`` (fp32
    [S]) each stream's box ratio.  With ``jpeg_max_bytes`` the inputs are ``bytes`` (uint8 [S, jpeg_max_bytes]) and
    ``lengths`` (int32 [S], 0 = no frame) instead of ``frames``, decoded inside the tick into ``frames`` with a per-stream
    ``status``.  ``raw`` ([S, A, 5 + nc] head outputs), ``det`` ([S, A, 7] rows x1, y1, x2, y2 -- divided by the stream's
    ratio --, obj, class_conf, class_pred) and ``count`` ([S] rows of ``det``) are the outputs; ``buffer`` holds each
    stream's features carried to the next tick.  With a YUV ``frame_format`` (an ops.YUV_FORMATS key) the input is ``yuv``
    (uint8 [S, max_bytes], stream i's frame in cv2's layout in the first bytes of row i), converted inside the tick into
    ``frames``; with a Bayer one (BAYER_FORMATS) it is ``bayer`` (uint8 [S, max_bytes], stream i's [h, w] mosaic in the
    first h * w bytes of row i), demosaiced inside the tick into ``frames`` with ``demosaic`` (an ops.DEMOSAIC key).
    With ``record_quality`` the tick ends with the JPEG encode of the frames in ``frames`` (``rec_out``, ``rec_len``,
    ``rec_status``).  With ``record_boxes`` = (fp32 score threshold, uint8 [P, 3] BGR palette on the device)
    the encode reads ``rec_frames`` instead: a copy of ``frames`` with the tick's detections drawn (sy_vis_det_boxes,
    sy_draw_boxes), so ``frames``, which a later tick may read again, is never drawn on."""

    def __init__(self, model, table, ratios, size, streams, conf_thre, nms_thre, device, jpeg_max_bytes=None,
                 forecast=None, clear_on_empty=False, queries=0, frame_format="bgr", record_quality=None,
                 record_boxes=None, demosaic="bilinear"):
        self.model, self.size = model, tuple(size)
        self.conf_thre, self.nms_thre = float(conf_thre), float(nms_thre)
        table = np.asarray(table, np.int32)
        slot = (int(table[:, 0].max()), int(table[:, 1].max()))
        self.frames = torch.zeros((streams, slot[0], slot[1], 3), dtype=torch.uint8, device=device)
        self.flags = torch.ones((streams,), dtype=torch.int32, device=device)
        self.table = torch.from_numpy(table).to(device)
        self.ratio = torch.tensor(ratios, dtype=torch.float32, device=device)
        self.start = torch.zeros((streams,), dtype=torch.int32, device=device)
        self.keep = torch.ones((streams,), dtype=torch.int32, device=device)
        self.x = torch.empty((streams, 3, size[0], size[1]), dtype=torch.float32, device=device)
        self.ctx = engine.Ctx(False, streams, streams, torch.device(device), dtype=model.activation_dtype)
        self.buffer = None
        self.raw = self.det = self.count = None
        self.status = None
        self.yuv = self.bayer = None
        if frame_format in BAYER_FORMATS:
            self.bayer_pattern, self.demosaic = frame_format[len("bayer_"):], demosaic
            self.bayer = torch.zeros((streams, int((table[:, 0] * table[:, 1]).max())), dtype=torch.uint8, device=device)
            self.bayer_sizes = self.table[:, :2].contiguous()
        elif frame_format != "bgr":
            self.yuv_format = frame_format
            self.yuv = torch.zeros((streams, max(int(np.prod(frame_shape(frame_format, h, w))) for h, w in table[:, :2])),
                                   dtype=torch.uint8, device=device)
            self.yuv_sizes = self.table[:, :2].contiguous()
        # forecast = (match_iou_th, max_tracks): the tick ends with the tracks' update from its detections, each stream
        # gated by start / keep; fc_dt (int32 [S], set by the host) is the frames since the stream's previous update
        self.fc = self.fc_dt = None
        if forecast is not None:
            self.fc_th = float(forecast[0])
            self.fc = ops.ForecastState(streams, forecast[1], device)
            self.fc_dt = torch.zeros((streams,), dtype=torch.int32, device=device)
        self.fc_clear = bool(clear_on_empty)
        # queries = Q > 0: the tick then extrapolates the updated tracks to up to Q queries per stream (sy_forecast_
        # extrap_queries): fc_qdt (fp32 [S, Q]) and fc_nq (int32 [S]) are inputs set by the host, fc_qout the outputs
        self.fc_q = int(queries)
        if self.fc_q:
            self.fc_qdt = torch.zeros((streams, self.fc_q), dtype=torch.float32, device=device)
            self.fc_nq = torch.zeros((streams,), dtype=torch.int32, device=device)
            self.fc_wh = torch.from_numpy(np.ascontiguousarray(table[:, [1, 0]])).to(device)   # (W, H)
            self.fc_qout = None
        if jpeg_max_bytes is not None:
            self.bytes = torch.zeros((streams, jpeg_max_bytes), dtype=torch.uint8, device=device)
            self.lengths = torch.zeros((streams,), dtype=torch.int32, device=device)
            self.status = torch.zeros((streams,), dtype=torch.int32, device=device)
            self.sizes = self.table[:, :2].contiguous()
            self.workspace = torch.empty(ops.jpeg_decode_sized_workspace_bytes(streams, jpeg_max_bytes, *slot),
                                         dtype=torch.uint8, device=device)
        # record_quality: the tick ends with the JPEG encode of every slot's frame (sy_jpeg_encode) into rec_out, file i
        # in the first rec_len[i] bytes of row i, rec_status[i] its SY_JPEG_ENCODE_* status
        self.rec_q = record_quality
        if record_quality is not None:
            rec_bytes = ops.jpeg_encode_max_bytes(*slot)
            self.rec_sizes = self.table[:, :2].contiguous()
            self.rec_out = torch.zeros((streams, rec_bytes), dtype=torch.uint8, device=device)
            self.rec_len = torch.zeros((streams,), dtype=torch.int64, device=device)
            self.rec_status = torch.zeros((streams,), dtype=torch.int32, device=device)
            self.rec_ws = torch.empty(ops.jpeg_encode_workspace_bytes(streams, *slot, rec_bytes), dtype=torch.uint8,
                                      device=device)
        # record_boxes: the frames are copied to rec_frames and the detections drawn there before the encode; vb holds
        # sy_vis_det_boxes's (boxes, labels, counts), allocated by the first (warm-up) run
        self.rec_boxes = record_boxes
        if record_boxes is not None:
            self.vb_th, self.vb_palette = record_boxes
            self.rec_frames = torch.zeros_like(self.frames)
            self.vb = None

    def run(self):
        ctx, net, head = self.ctx, self.model.backbone, self.model.head
        if self.status is not None:
            ops.jpeg_decode_sized(self.bytes, self.lengths, self.sizes, self.frames, self.status, self.workspace)
        if self.yuv is not None:
            ops.yuv_to_bgr_sized(self.yuv, self.yuv_sizes, self.yuv_format, self.frames)
        if self.bayer is not None:
            ops.bayer_to_bgr_sized(self.bayer, self.bayer_sizes, self.bayer_pattern, self.demosaic, self.frames)
        ops.stream_gate(self.status, self.flags, self.start, self.keep)
        ops.letterbox_sized(self.frames, self.table, self.x)
        with torch.no_grad(), engine.forward_scope(ctx.device):
            cur = engine.pafpn_frames(ctx, net, self.x, 1)
            if self.buffer is None:
                self.buffer = tuple(ctx.empty(v.n, v.h, v.w, v.c) for v in cur)
            ops.select_images(cur, self.buffer, self.start)
            fused = engine.dfp_fuse(ctx, net, cur, self.buffer)
            ops.select_images(cur, self.buffer, self.keep)
            self.raw = head.run(ctx, fused)
            self.det, self.count = ops.postprocess_nms(self.raw, head.num_classes, self.conf_thre, self.nms_thre,
                                                       max_det=self.raw.shape[1])
            ops.stream_rescale(self.det, self.count, self.status, self.ratio)
            if self.fc is not None:
                ops.forecast_update(self.fc, self.det, self.count, self.fc_dt, self.start, self.keep, self.fc_th,
                                    clear_on_empty=self.fc_clear)
            if self.fc_q:
                self.fc_qout = ops.forecast_extrap_queries(self.fc, self.fc_qdt, self.fc_nq, self.fc_wh, self.fc_qout)
        if self.rec_q is not None:
            rec = self.frames
            if self.rec_boxes is not None:
                self.vb = ops.vis_det_boxes(self.det, self.count, self.vb_th, *(self.vb or ()))
                self.rec_frames.copy_(self.frames)
                ops.draw_boxes(self.rec_frames, self.rec_sizes, *self.vb, self.vb_palette, self.rec_frames)
                rec = self.rec_frames
            ops.jpeg_encode(rec, self.rec_sizes, self.rec_q, self.rec_out, self.rec_len, self.rec_status, self.rec_ws)


NO_FRAME = -1     # last_status() of a stream that was given no frame


def input_size_for(frame_sizes, in_scale, input_size=None):
    """The model input size of a rig: ``input_size`` when given, else the driver's (int(h * in_scale), int(w * in_scale))
    of the largest frame (by area; the first of equal ones)."""
    if input_size is not None:
        return tuple(int(v) for v in input_size)
    h, w = max(frame_sizes, key=lambda s: s[0] * s[1])
    return int(h * in_scale), int(w * in_scale)


def jpeg_files(files, streams, max_bytes):
    """step_jpeg's inputs as S uint8 numpy arrays (``None``: no frame this tick, an empty array), or an error: a list of S
    entries, each ``bytes`` / ``bytearray`` / ``memoryview``, a uint8 numpy array or CPU tensor, or None, and at most
    ``max_bytes`` long."""
    if not isinstance(files, (list, tuple)) or len(files) != streams:
        raise ValueError(f"StreamDetector.step_jpeg: give a list of {streams} files (None for no frame)")
    out = []
    for i, f in enumerate(files):
        if f is None:
            a = np.zeros(0, np.uint8)
        elif isinstance(f, (bytes, bytearray, memoryview)):
            a = np.frombuffer(f, np.uint8)
        else:
            a = f.numpy() if torch.is_tensor(f) and not f.is_cuda else f
            if not isinstance(a, np.ndarray) or a.dtype != np.uint8:
                raise TypeError(f"StreamDetector.step_jpeg: file {i} must be bytes or a uint8 array, not "
                                f"{getattr(a, 'dtype', type(a).__name__)}")
            a = np.ascontiguousarray(a).reshape(-1)
        if a.size > max_bytes:
            raise ValueError(f"StreamDetector.step_jpeg: file {i} has {a.size} bytes, more than jpeg_max_bytes = {max_bytes}")
        out.append(a)
    return out


def route_status(status, present, flags):
    """The host's bookkeeping after a JPEG tick: -> (the per-stream status last_status() reports -- NO_FRAME for a stream
    given no frame --, the start flags of the next tick).  A stream whose frame decoded has started (or continued) its
    sequence, so its flag clears; one that was gated keeps its flag, so that a sequence starts at its next decoded frame."""
    st = np.where(np.asarray(present, bool), np.asarray(status, np.int32), NO_FRAME).astype(np.int32)
    return st, np.where(st == 0, 0, np.asarray(flags, np.int32)).astype(np.int32)


def sized_output(det):
    """one stream's NMS rows (numpy fp32 [n, 7]) whose boxes the device already divided by the stream's ratio -> the
    driver's (bboxes, scores, labels)"""
    return det[:, :4].copy(), det[:, 4] * det[:, 5], det[:, 6].astype(np.int32)


FRAME_FORMATS = ("bgr",) + tuple(ops.YUV_FORMATS)
# raw 8-bit Bayer mosaics, named by the colour order of their top-left 2x2 (ops.BAYER_PATTERNS)
BAYER_FORMATS = tuple("bayer_" + p for p in ops.BAYER_PATTERNS)
# the smallest Bayer frame: one whole 2x2 colour cell.  cv2 is reproducible at every size on a contiguous frame; below
# 3 rows or columns it is black (and so is the device's)
BAYER_MIN_HW = (2, 2)


def record_boxes_args(record_boxes, record_quality, num_classes):
    """``StreamDetector(record_boxes=(score_th, palette))`` -> (the fp32 threshold sy_vis_det_boxes takes, the uint8
    [P, 3] palette in BGR order), or ValueError"""
    if record_quality is None:
        raise ValueError("StreamDetector: record_boxes draws on the recorded frames: it takes record_quality")
    if not isinstance(record_boxes, (tuple, list)) or len(record_boxes) != 2:
        raise ValueError(f"StreamDetector: record_boxes must be None or (score_th, palette), not {record_boxes!r}")
    th, palette = record_boxes
    if isinstance(th, bool) or not isinstance(th, (int, float, np.integer, np.floating)) or not np.isfinite(th):
        raise ValueError(f"StreamDetector: record_boxes's score_th must be a finite number, not {th!r}")
    try:
        pal = np.asarray(palette)
    except Exception:
        pal = None
    if pal is None or pal.dtype.kind not in "iu" or pal.ndim != 2 or pal.shape[1] != 3 or pal.size == 0 \
            or pal.min() < 0 or pal.max() > 255:
        raise ValueError("StreamDetector: record_boxes's palette must be a list of (R, G, B) integer triples in 0..255")
    if len(pal) < num_classes:
        raise ValueError(f"StreamDetector: record_boxes's palette has {len(pal)} colours for {num_classes} classes")
    # vis_obj_fancy filters only when score_th > 0 (vis_det_th.py:81), then compares fp32 scores with it in fp32
    return (float(np.float32(th)) if th > 0 else -np.inf), np.ascontiguousarray(pal[:, ::-1].astype(np.uint8))


def frame_shape(fmt, h, w):
    """the uint8 array ``step`` takes for one h x w frame of ``fmt`` (a FRAME_FORMATS or BAYER_FORMATS entry), in cv2's
    layout"""
    if fmt == "bgr":
        return h, w, 3
    if fmt in BAYER_FORMATS:
        return h, w
    return (h * 3 // 2, w) if fmt in ("nv12", "nv21", "i420", "yv12") else (h, w, 2)


def step_frames(frames, streams, frame_hw, fmt="bgr"):
    """``frames`` (numpy, CPU or CUDA tensor) as a uint8 [S, *frame_shape] tensor, or RuntimeError; [*frame_shape] for
    one stream."""
    s, shape = streams, frame_shape(fmt, *frame_hw)
    src = frames if torch.is_tensor(frames) else torch.from_numpy(np.ascontiguousarray(frames))
    one = ", ".join(str(v) for v in shape)
    ops._require(src.dtype == torch.uint8 and (tuple(src.shape) == (s, *shape) or (s == 1 and tuple(src.shape) == shape)),
                 f"StreamDetector.step: frames must be uint8 [{s}, {one}]" + (f" or [{one}]" if s == 1 else "")
                 + f", not {src.dtype} {list(src.shape)}")
    return src.reshape(s, *shape)


class StreamDetector:
    """``model`` (YOLOX with a DFPPAFPN backbone, in eval mode, weights loaded) on ``streams`` camera streams of
    ``frame_hw`` uint8 BGR frames, at the driver's input size ``(int(h * in_scale), int(w * in_scale))``.  The activation
    storage is ``model.activation_dtype`` (``torch.float16`` for the driver's ``model.half()``).  The constructor captures
    the tick (after one warm-up run); every stream starts a sequence at the first ``step``.

    Streams of their own sizes and JPEG input:
      frame_sizes     [(h, w), ...], one per stream (default: ``frame_hw`` for every stream); with the default
                      ``streams=1`` it also sets the number of streams
      input_size      the model's (H, W); default: the driver's size of the largest frame (input_size_for).  Only with
                      ``frame_sizes`` or ``jpeg_max_bytes``: without them the input size is the driver's, as above
      jpeg_max_bytes  the longest JPEG file ``step_jpeg`` takes.  The replay then starts with the decode of the streams'
                      files, so such a detector takes files only (``step_jpeg``); without it, it takes decoded frames only
                      (``step``)
    Forecast (the sAP toolkit's pps_forecast_kf.py online):
      forecast        True: the tick ends with each stream's track update from its detections (sy_forecast_update:
                      Kalman predict, greedy IoU association, Kalman update), gated as the feature buffer is: a stream
                      that starts a sequence clears its tracks, one without a decoded frame keeps them.  ``step`` and
                      ``step_jpeg`` then take ``fidx``, each stream's frame index, and ``forecast(fidx)`` extrapolates
                      the tracks to a query frame.  The detections ``step`` returns do not change.
      match_iou_th    the association's IoU threshold (inclusive)
      max_tracks      the most detections one stream's update takes; a tick with more raises RuntimeError naming the
                      stream, whose tracks are then left as they were
    Raw camera frames:
      frame_format    "bgr" (the default): ``step`` and ``submit`` take uint8 BGR [h, w, 3] frames.  "nv12", "nv21",
                      "i420", "yv12" (4:2:0: uint8 [h * 3 // 2, w], even h and w) or "yuyv", "uyvy" (4:2:2: uint8
                      [h, w, 2], even w): they take the camera's frames in cv2's layout, and the replay starts with their
                      conversion to BGR (sy_yuv_to_bgr_sized, cv2.cvtColor(COLOR_YUV2BGR_NV12, _NV21, _I420, _YV12,
                      _YUY2, _UYVY) bit for bit).  "bayer_rggb", "bayer_bggr", "bayer_gbrg", "bayer_grbg" (BAYER_FORMATS:
                      8-bit sensor mosaics, uint8 [h, w], named by the colour order of the top-left 2x2; h and w at least
                      2): the replay starts with their demosaicing (sy_bayer_to_bgr_sized, cv2.cvtColor(COLOR_BayerRGGB2BGR,
                      _BGGR2BGR, _GBRG2BGR, _GRBG2BGR, with the _EA codes for ``demosaic="ea"``) bit for bit).  Not with
                      ``jpeg_max_bytes``
      demosaic        with a Bayer frame_format: "bilinear" (the default, cv2's COLOR_Bayer*2BGR) or "ea" (edge-aware,
                      COLOR_Bayer*2BGR_EA)
    The sAP toolkit's streamer (sAP/forecast/streamer.py, see streamyolo_b200.streamer), with ``forecast=True``:
      clear_on_empty  True: an empty detection leaves the stream without tracks, as the streamer's association does
                      (the default keeps the predicted tracks, as pps_forecast_kf.py does)
      queries         Q > 0: the tick ends with the extrapolation of each stream's updated tracks to up to Q queries
                      (sy_forecast_extrap_queries), given to ``step`` / ``step_jpeg`` as ``query_dt`` and read back
                      with the detections, one synchronisation per tick (``last_queries``)
      ``submit`` / ``poll`` / ``receive`` run a tick without waiting for it, and ``publish`` / ``query`` extrapolate the
      tracks of the last received tick while the next one is in flight (the wall-clock streamer)
    Recording what the cameras saw:
      record_quality  None (the default) or a JPEG quality 1..100: the tick ends with the encode of every stream's BGR
                      frame -- the decoded, converted or given frame the resize reads -- into the file cv2.imencode(".jpg",
                      frame, [cv2.IMWRITE_JPEG_QUALITY, record_quality]) makes (sy_jpeg_encode), and ``last_jpeg``
                      reads the files back.  The detections do not change
      record_boxes    None (the default) or ``(score_th, palette)``, with ``record_quality``: each recorded frame has the
                      tick's own detections drawn on it first, as the sAP toolkit's vis_det_th.py draws a result file
                      (vis_obj_fancy without text: boxes filled at 0.8 / 0.2 and outlined two pixels wide in their class
                      colour), the rows with score >= score_th (``score_th`` <= 0: every row).  ``palette``: a list of
                      (R, G, B) per class, in the order of the toolkit's ``color_palette``, at least ``num_classes`` long.
                      Drawn on a copy: the detections, forecasts and every other output do not change
    Each stream's frame is transformed as data.sized_table says and its boxes divided by its own ratio (``ratios``): a frame
    of driver size ``input_size`` gets the driver's plain resize and ``in_scale``.  ``frame_hw`` is the slot the frames are
    stored in: the largest height and width (the frame size when every stream has one size)."""

    def __init__(self, model, frame_hw=(1200, 1920), in_scale=0.5, streams=1, conf_thre=0.01, nms_thre=0.65,
                 frame_sizes=None, input_size=None, jpeg_max_bytes=None, forecast=False, match_iou_th=0.3,
                 max_tracks=1024, clear_on_empty=False, queries=0, frame_format="bgr", record_quality=None,
                 record_boxes=None, demosaic="bilinear"):
        if model.training:
            raise ValueError("StreamDetector: the model must be in eval mode (model.eval())")
        if int(streams) != streams or streams < 1:
            raise ValueError(f"StreamDetector: streams must be a positive integer, not {streams}")
        if input_size is not None and frame_sizes is None and jpeg_max_bytes is None:
            raise ValueError("StreamDetector: input_size takes frame_sizes or jpeg_max_bytes; without them the input size "
                             "is the driver's (int(h * in_scale), int(w * in_scale))")
        streams = int(streams)
        sizes = [tuple(int(v) for v in s) for s in ([frame_hw] * streams if frame_sizes is None else frame_sizes)]
        if len(sizes) != streams and frame_sizes is not None and streams == 1:
            streams = len(sizes)                      # streams defaults to one: frame_sizes then sets the count
        if len(sizes) != streams or any(len(s) != 2 for s in sizes):
            raise ValueError(f"StreamDetector: frame_sizes must hold {streams} (h, w) pairs, not {frame_sizes}")
        size = input_size_for(sizes, in_scale, input_size)
        if min(size) < 1 or min(min(s) for s in sizes) < 1:
            raise ValueError(f"StreamDetector: frames {sizes} at in_scale {in_scale} give input size {size}")
        if jpeg_max_bytes is not None:
            jpeg_max_bytes = feed.check_max_bytes(jpeg_max_bytes, "StreamDetector: jpeg_max_bytes")
        if frame_format not in FRAME_FORMATS + BAYER_FORMATS:
            raise ValueError(f"StreamDetector: unknown frame_format {frame_format!r} (one of "
                             f"{', '.join(FRAME_FORMATS + BAYER_FORMATS)})")
        if demosaic not in ops.DEMOSAIC:
            raise ValueError(f"StreamDetector: unknown demosaic {demosaic!r} (one of {', '.join(ops.DEMOSAIC)})")
        if demosaic != "bilinear" and frame_format not in BAYER_FORMATS:
            raise ValueError(f"StreamDetector: demosaic={demosaic!r} takes a Bayer frame_format "
                             f"({', '.join(BAYER_FORMATS)}), not {frame_format!r}")
        if frame_format != "bgr" and jpeg_max_bytes is not None:
            raise ValueError(f"StreamDetector: frame_format {frame_format!r} takes raw frames, jpeg_max_bytes JPEG "
                             "files: give one or the other")
        if frame_format in BAYER_FORMATS:
            small = [s for s in sizes if s[0] < BAYER_MIN_HW[0] or s[1] < BAYER_MIN_HW[1]]
            if small:
                raise ValueError(f"StreamDetector: {frame_format} frames need at least {BAYER_MIN_HW[0]} rows and "
                                 f"{BAYER_MIN_HW[1]} columns (one whole colour cell); not {small[0]}")
        elif frame_format != "bgr":
            sub420 = len(frame_shape(frame_format, 2, 2)) == 2
            odd = [s for s in sizes if s[1] % 2 or (sub420 and s[0] % 2)]
            if odd:
                raise ValueError(f"StreamDetector: {frame_format} frames need an even width"
                                 + (" and height" if sub420 else "") + f", as cv2 requires; not {odd[0]}")
        if forecast and (int(max_tracks) != max_tracks or not 1 <= max_tracks <= 1 << 20):
            raise ValueError(f"StreamDetector: max_tracks must be an integer in [1, 2^20], not {max_tracks}")
        if int(queries) != queries or not 0 <= queries <= 65535:
            raise ValueError(f"StreamDetector: queries must be an integer in [0, 65535], not {queries}")
        if (clear_on_empty or queries) and not forecast:
            raise ValueError("StreamDetector: clear_on_empty and queries take forecast=True")
        if record_quality is not None and (isinstance(record_quality, bool) or not isinstance(record_quality, (int, np.integer))
                                           or not 1 <= record_quality <= 100):
            raise ValueError(f"StreamDetector: record_quality must be None or an integer in 1..100, not {record_quality!r}")
        if record_boxes is not None:
            record_boxes = record_boxes_args(record_boxes, record_quality, model.head.num_classes)
        try:
            table, ratios = data.sized_table(sizes, size, in_scale)
        except RuntimeError as e:
            raise ValueError(f"StreamDetector: {e}") from None
        dev = next(model.parameters()).device
        ops.lib()
        self.model, self.streams, self.in_scale, self.size = model, streams, in_scale, size
        self.frame_sizes, self.ratios = sizes, ratios
        self.jpeg_max_bytes = jpeg_max_bytes
        self.frame_format, self.demosaic = frame_format, demosaic
        self.forecasting = bool(forecast)
        self.queries = int(queries)
        self._tick = StreamTick(model, table, ratios, size, streams, conf_thre, nms_thre, dev, self.jpeg_max_bytes,
                                (match_iou_th, int(max_tracks)) if forecast else None, clear_on_empty, self.queries,
                                frame_format, None if record_quality is None else int(record_quality),
                                None if record_boxes is None else (record_boxes[0],
                                                                   torch.from_numpy(record_boxes[1]).to(dev)),
                                demosaic)
        self.record_quality = None if record_quality is None else int(record_quality)
        if self.record_quality is not None:
            self._rec_len = feed.pinned((streams,), torch.int64)
            self._rec_status = feed.pinned((streams,), torch.int32)
            self._rec_rows = None                 # the streams the last tick has a file for
            self._rec_stage = None
        if self.forecasting:
            self._fc_dt = feed.pinned((streams,), torch.int32)
            self._fc_meta = feed.pinned((streams, 4), torch.int32)
            self._fc_wh = torch.tensor([(w, h) for h, w in sizes], dtype=torch.int32, device=dev)
            self._fc_out = None
        if self.queries:
            self._q_dt = feed.pinned((streams, self.queries), torch.float32)
            self._q_n = feed.pinned((streams,), torch.int32)
            self._q_out = None
            self._queries = None
        self._pub = None                          # publish / query: the published tracks, their stream and events
        self._inflight = None
        self.frame_hw = tuple(self._tick.frames.shape[1:3])          # the slot: the largest height and width
        if self.jpeg_max_bytes is None:
            self._inputs()
        else:
            self._jstage = feed.pinned((streams, self.jpeg_max_bytes), torch.uint8)
            self._jlen = feed.pinned((streams,), torch.int32)
            self._status = feed.pinned((streams,), torch.int32)
        self._last_status = None
        self._flags = feed.pinned((streams,), torch.int32)
        self._graph = None
        self.capture()

    def capture(self):
        """(Re-)capture the tick: reads the model's current weights and folded BatchNorm.  Call it after
        ``load_state_dict``.  Every stream starts a sequence at the next ``step``."""
        self._graph = None
        t = self._tick
        self._graph = engine.capture_graph(t.run, t.frames.device)
        self._det = feed.pinned((self.streams, t.raw.shape[1], 7), torch.float32)
        self._count = feed.pinned((self.streams,), torch.int32)
        if self.queries:
            self._q_out = tuple(feed.pinned(tuple(o.shape), o.dtype) for o in t.fc_qout)
        self._inflight = None
        if self.forecasting:                      # the warm-up run went through the update: no stream has tracks yet
            t.fc.meta.zero_()
            self._fc_last = [None] * self.streams         # each stream's frame index at its last update
        self.reset()

    def reset(self, stream=None):
        """Start a new sequence at the next ``step``: on every stream, or on stream ``stream`` only."""
        if stream is None:
            self._flags.fill_(1)
        else:
            if not 0 <= stream < self.streams:
                raise ValueError(f"StreamDetector.reset: stream {stream} not in [0, {self.streams})")
            self._flags[stream] = 1

    def step(self, frames, fidx=None, query_dt=None):
        """One frame per stream -> a list of S ``(bboxes, scores, labels)`` numpy tuples, what the driver's inference()
        returns (boxes in frame pixels, float32 [n, 4]; scores float32 [n]; labels int32 [n]).  ``frames``: a list of S
        frames, frame i uint8 BGR [h_i, w_i, 3] of stream i's size; or, when every stream has the same size, uint8
        [S, h, w, 3] ([h, w, 3] for one stream).  Each a numpy array, a CPU tensor or a CUDA tensor.  A detector built with
        ``jpeg_max_bytes`` takes files only: ``step`` raises RuntimeError there, use ``step_jpeg``.  With ``forecast=True``,
        ``fidx`` gives each stream's frame index (a list of S ints; an int for one stream), and the tick updates the
        stream's tracks with its detections (see ``forecast``).  With ``queries``, ``query_dt`` gives each stream's query
        offsets (a list of S sequences of at most Q frame counts, floats; None: none) that the tick extrapolates the
        updated tracks to (see ``last_queries``)."""
        fidx = self._fidx(fidx, "step")
        self._stage_frames(frames, "step")
        self._queries_in(query_dt, "step")
        return self._run(None, fidx)

    def _inputs(self):
        """the tick's buffer ``step`` copies the frames to (``frames``, ``yuv`` for a YUV frame_format or ``bayer`` for a
        Bayer one), each stream's frame shape in it and the pinned stage (stream i's frame staged at the start of row i)"""
        t = self._tick
        self._in = t.yuv if t.yuv is not None else t.bayer if t.bayer is not None else t.frames
        self._shapes = [frame_shape(self.frame_format, h, w) for h, w in self.frame_sizes]
        self._stage = feed.pinned(tuple(self._in.shape), torch.uint8)

    def _stage_frames(self, frames, what):
        """``frames`` of ``step`` copied (asynchronously) into the tick's input buffer"""
        t = self._tick
        if self.jpeg_max_bytes is not None:
            raise RuntimeError(f"StreamDetector.{what}: this detector was built with jpeg_max_bytes, and its replay decodes "
                               "the streams' files: feed it with step_jpeg (build one with frame_sizes alone for decoded "
                               "frames)")
        if isinstance(frames, (list, tuple)):
            ops._require(len(frames) == self.streams, f"StreamDetector.step: give a list of {self.streams} frames, one per stream")
            for i, (f, shape, (h, w)) in enumerate(zip(frames, self._shapes, self.frame_sizes)):
                ops._require(f is not None, f"StreamDetector.step: frame {i} is None: every stream takes a frame per tick")
                src = f if torch.is_tensor(f) else torch.from_numpy(np.ascontiguousarray(f))
                ops._require(src.dtype == torch.uint8 and tuple(src.shape) == shape, f"StreamDetector.step: frame {i} must "
                             f"be uint8 {list(shape)}, not {src.dtype} {list(src.shape)}")
                n = src.numel()
                dst = t.frames[i, :h, :w] if self._in is t.frames else self._in[i, :n].view(shape)
                if src.is_cuda:
                    dst.copy_(src)
                else:                                 # only the frame's own bytes cross, not the whole slot
                    stage = self._stage[i].view(-1)[:n].view(shape)
                    stage.copy_(src)
                    dst.copy_(stage, non_blocking=True)
        else:
            ops._require(all(s == self.frame_hw for s in self.frame_sizes),
                         f"StreamDetector.step: give a list of {self.streams} frames, one per stream")
            src = step_frames(frames, self.streams, self.frame_hw, self.frame_format)
            dst = self._in.view(src.shape)            # one size: each slot holds exactly one frame
            if src.is_cuda:
                dst.copy_(src)
            else:
                stage = self._stage.view(src.shape)
                stage.copy_(src)
                dst.copy_(stage, non_blocking=True)

    def last_raw(self):
        """A device copy of the last tick's head outputs [S, A, 5 + nc] (what the driver keeps as ``results_raw``)."""
        return self._tick.raw.clone()

    def step_jpeg(self, files, fidx=None, query_dt=None):
        """One JPEG file per stream -> a list of S ``(bboxes, scores, labels)`` tuples as ``step`` returns them, with one
        host synchronisation.  ``files``: a list of S entries, each the file's bytes (``bytes``, or a uint8 numpy array or
        CPU tensor) of at most ``jpeg_max_bytes``, or None when the stream has no frame this tick.  A stream whose file
        did not decode (see ``last_status``) or that got None returns empty arrays, keeps its carried features and, if it
        was to start a sequence, starts it at its next decoded frame.  ``fidx``: as for ``step``; such a stream's tracks
        are left as they were."""
        if self.jpeg_max_bytes is None:
            raise RuntimeError("StreamDetector.step_jpeg: construct the detector with jpeg_max_bytes")
        t = self._tick
        files = jpeg_files(files, self.streams, self.jpeg_max_bytes)
        fidx = self._fidx(fidx, "step_jpeg")
        stage = self._jstage.numpy()
        for i, a in enumerate(files):
            stage[i, :a.size] = a
            self._jlen[i] = a.size
            if a.size:
                t.bytes[i, :a.size].copy_(self._jstage[i, :a.size], non_blocking=True)
        t.lengths.copy_(self._jlen, non_blocking=True)
        self._queries_in(query_dt, "step_jpeg")
        return self._run([a.size > 0 for a in files], fidx)

    def _queries_in(self, query_dt, what):
        """``query_dt`` of step / step_jpeg into the pinned query inputs, copied to the tick's"""
        if not self.queries:
            if query_dt is not None:
                raise ValueError(f"StreamDetector.{what}: query_dt takes a detector built with queries > 0")
            return
        query_dt = [None] * self.streams if query_dt is None else query_dt
        if not isinstance(query_dt, (list, tuple)) or len(query_dt) != self.streams \
                or any(q is not None and len(q) > self.queries for q in query_dt):
            raise ValueError(f"StreamDetector.{what}: query_dt must hold {self.streams} sequences of at most "
                             f"{self.queries} frame counts (None for none)")
        self._q_dt.zero_()
        for i, q in enumerate(query_dt):
            n = 0 if q is None else len(q)
            self._q_n[i] = n
            if n:
                self._q_dt[i, :n] = torch.from_numpy(np.asarray(q, np.float32))
        t = self._tick
        t.fc_qdt.copy_(self._q_dt, non_blocking=True)
        t.fc_nq.copy_(self._q_n, non_blocking=True)

    def _fidx(self, fidx, what):
        """``fidx`` of step / step_jpeg as a list of S ints (None without forecast)"""
        if not self.forecasting:
            if fidx is not None:
                raise ValueError(f"StreamDetector.{what}: fidx takes a detector built with forecast=True")
            return None
        if isinstance(fidx, (int, np.integer)) and self.streams == 1:
            fidx = [fidx]
        if not isinstance(fidx, (list, tuple, np.ndarray)) or len(fidx) != self.streams \
                or any(int(v) != v for v in fidx):
            raise ValueError(f"StreamDetector.{what}: with forecast=True give fidx, {self.streams} frame indices "
                             "(an int for one stream)")
        return [int(v) for v in fidx]

    def _dt(self, fidx):
        """frames from each stream's last update to ``fidx`` (0 for a stream without one), into the pinned dt"""
        for i, (f, last) in enumerate(zip(fidx, self._fc_last)):
            d = 0 if last is None else f - last
            if not -2 ** 31 <= d < 2 ** 31:
                raise ValueError(f"StreamDetector: stream {i}: frame index {f} is {d} frames from its last update")
            self._fc_dt[i] = d

    def _run(self, present, fidx=None):
        """Replay the tick on the staged inputs and return the detections; ``present`` (JPEG ticks only): which streams
        were given a file; ``fidx``: the streams' frame indices (forecast only)."""
        self._launch(present, fidx)
        torch.cuda.current_stream().synchronize()
        return self._finish(present, fidx)

    def _launch(self, present, fidx):
        """the replay and the copies out of ``_run``, queued on the current stream"""
        if self._inflight is not None:
            raise RuntimeError("StreamDetector: a submitted tick is still in flight: receive() it first")
        t = self._tick
        t.flags.copy_(self._flags, non_blocking=True)
        if fidx is not None:
            self._dt(fidx)
            t.fc_dt.copy_(self._fc_dt, non_blocking=True)
        if self._pub is not None:                 # the tick rewrites the tracks a pending publish copies
            torch.cuda.current_stream().wait_event(self._pub["copied"])
        self._graph.replay()
        self._det.copy_(t.det, non_blocking=True)
        self._count.copy_(t.count, non_blocking=True)
        if present is not None:
            self._status.copy_(t.status, non_blocking=True)
        if fidx is not None:
            self._fc_meta.copy_(t.fc.meta, non_blocking=True)
        if self.queries:
            for h, d in zip(self._q_out, t.fc_qout):
                h.copy_(d, non_blocking=True)
        if self.record_quality is not None:
            self._rec_len.copy_(t.rec_len, non_blocking=True)
            self._rec_status.copy_(t.rec_status, non_blocking=True)

    def _finish(self, present, fidx):
        """the host's side of ``_run`` once the tick and its copies are done -> the detections"""
        t = self._tick
        if present is None:
            updated = [True] * self.streams
            self._flags.zero_()
        else:
            self._last_status, nxt = route_status(self._status.numpy(), present, self._flags.numpy())
            updated = (self._last_status == 0).tolist()
            self._flags.copy_(torch.from_numpy(nxt))
        if self.record_quality is not None:
            self._rec_rows = list(updated)
        if fidx is not None:
            over = [i for i in range(self.streams) if self._fc_meta[i, 3] != 0]
            if over:
                raise RuntimeError(f"StreamDetector: stream {over[0]}'s detection has more rows than max_tracks = "
                                   f"{t.fc.max_tracks}; its tracks were left as they were (build the detector with a "
                                   "larger max_tracks)")
            for i, u in enumerate(updated):
                if u:
                    self._fc_last[i] = fidx[i]
        if self.queries:
            box, score, label, track, count = (h.numpy() for h in self._q_out)
            n_q, meta = self._q_n.tolist(), self._fc_meta.numpy()
            self._queries = [[None if meta[i, 0] == 0 else
                              (box[i, k, :n].copy(), score[i, k, :n].copy(), label[i, k, :n].copy(), track[i, k, :n].copy())
                              for k, n in enumerate(count[i, :n_q[i]].tolist())] for i in range(self.streams)]
        det = self._det.numpy()
        return [sized_output(det[i, :n]) for i, n in enumerate(self._count.tolist())]

    def last_jpeg(self):
        """The last tick's frames as JPEG files (a detector built with ``record_quality``): per stream the ``bytes``
        cv2.imencode(".jpg", frame, [cv2.IMWRITE_JPEG_QUALITY, record_quality]) returns for the BGR frame the tick
        detected on, or None for a stream without a frame that tick (no file, or one that did not decode).  Copies exactly
        each file's length back, with one synchronisation; None before the first tick."""
        if self.record_quality is None:
            raise RuntimeError("StreamDetector.last_jpeg: build the detector with record_quality")
        if self._rec_rows is None:
            return None
        t = self._tick
        total = sum(int(l) for l, r in zip(self._rec_len.tolist(), self._rec_rows) if r)
        if self._rec_stage is None or self._rec_stage.numel() < total:
            self._rec_stage = feed.pinned((max(2 * total, 1),), torch.uint8)
        return data.jpeg_files(t.rec_out, self._rec_len, self._rec_status, self._rec_rows, self._rec_stage)

    def last_queries(self):
        """The extrapolations of the last ``step`` / ``step_jpeg`` (a detector built with ``queries``): per stream, one
        entry per ``query_dt`` offset, ``(ltwh, scores, labels, tracks)`` as ``forecast`` returns them, or None where the
        stream has no track after its update (the streamer then emits empty arrays of its own dtypes)"""
        if not self.queries:
            raise RuntimeError("StreamDetector.last_queries: build the detector with queries > 0")
        return self._queries

    def submit(self, frames, fidx=None):
        """``step`` without the wait: stage ``frames`` and queue the replay and its copies, then return.  ``poll`` tells
        when it is done and ``receive`` then returns what ``step`` returns.  One tick at a time."""
        fidx = self._fidx(fidx, "submit")
        if self._inflight is not None:
            raise RuntimeError("StreamDetector.submit: a submitted tick is still in flight: receive() it first")
        if self.queries:
            raise RuntimeError("StreamDetector.submit: a detector built with queries runs its ticks with step / step_jpeg")
        self._stage_frames(frames, "submit")
        self._launch(None, fidx)
        done = torch.cuda.Event()
        done.record()
        self._inflight = (done, fidx)

    def poll(self, timeout):
        """True once the submitted tick is done, waiting at most ``timeout`` seconds for it (the toolkit's
        ``Pipe.poll(timeout)``); False when it is still running then"""
        if self._inflight is None:
            raise RuntimeError("StreamDetector.poll: no tick was submitted")
        done = self._inflight[0]
        end = time.perf_counter() + max(float(timeout), 0.0)
        while not done.query():
            if time.perf_counter() >= end:
                return False
        return True

    def receive(self):
        """The submitted tick's detections, as ``step`` returns them; waits for it when ``poll`` has not seen it done"""
        if self._inflight is None:
            raise RuntimeError("StreamDetector.receive: no tick was submitted")
        done, fidx = self._inflight
        done.synchronize()
        self._inflight = None
        return self._finish(None, fidx)

    def publish(self):
        """Copy the tracks of the last received tick to the buffers ``query`` reads, on a stream of their own: a tick
        submitted after this waits for the copy, and no tick in flight writes what a query reads"""
        if not self.forecasting:
            raise RuntimeError("StreamDetector.publish: build the detector with forecast=True")
        if self._inflight is not None:
            raise RuntimeError("StreamDetector.publish: receive() the submitted tick first")
        t = self._tick
        if self._pub is None:
            self._pub = {"state": ops.ForecastState(self.streams, t.fc.max_tracks, t.fc.x.device),
                         "stream": torch.cuda.Stream(t.fc.x.device), "copied": torch.cuda.Event(), "out": None,
                         "host": None, "dt": feed.pinned((self.streams, 1), torch.float32),
                         "n": torch.ones((self.streams,), dtype=torch.int32, device=t.fc.x.device),
                         "meta": feed.pinned((self.streams, 4), torch.int32)}
        p = self._pub
        p["stream"].wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(p["stream"]):
            for name in ("x", "P", "label", "score", "track", "meta"):
                getattr(p["state"], name).copy_(getattr(t.fc, name))
            p["copied"].record()
        p["meta"].copy_(self._fc_meta)

    def query(self, dt):
        """The published tracks extrapolated ``dt`` frames ahead (a list of S numbers, fp32 frame counts; a number for
        one stream) -> per stream ``(ltwh, scores, labels, tracks)`` as ``forecast`` returns them, or None where the
        stream had no track.  One launch (sy_forecast_extrap_queries) and one synchronisation of the publish stream: it
        does not wait for a tick in flight."""
        if self._pub is None:
            raise RuntimeError("StreamDetector.query: publish() the tracks first")
        p = self._pub
        dt = [dt] if np.ndim(dt) == 0 else list(dt)
        if len(dt) != self.streams:
            raise ValueError(f"StreamDetector.query: give {self.streams} offsets")
        p["dt"][:, 0] = torch.from_numpy(np.asarray(dt, np.float32))
        with torch.cuda.stream(p["stream"]):
            d = p["dt"].to(p["state"].x.device, non_blocking=True)
            p["out"] = ops.forecast_extrap_queries(p["state"], d, p["n"], self._fc_wh, p["out"])
            if p["host"] is None:
                p["host"] = tuple(feed.pinned(tuple(o.shape), o.dtype) for o in p["out"])
            for h, o in zip(p["host"], p["out"]):
                h.copy_(o, non_blocking=True)
        p["stream"].synchronize()
        box, score, label, track, count = (h.numpy() for h in p["host"])
        return [None if p["meta"][i, 0] == 0 else
                (box[i, 0, :n].copy(), score[i, 0, :n].copy(), label[i, 0, :n].copy(), track[i, 0, :n].copy())
                for i, n in enumerate(count[:, 0].tolist())]

    def forecast(self, fidx):
        """Each stream's tracks extrapolated to its frame index ``fidx`` (a list of S ints; an int for one stream) ->
        a list of S ``(ltwh, scores, labels, tracks)`` numpy tuples: float32 [n, 4] boxes in frame pixels, float32 [n],
        int32 [n], int32 [n].  The sAP toolkit's forecast (sAP/forecast/pps_forecast_kf.py:258-273): the tracks matched
        at the last update move by their Kalman velocity times the frames since that update, the others stay; boxes are
        clipped to the stream's frame and dropped below 75 pixels (extrap_clean_up).  One launch, one synchronisation."""
        if not self.forecasting:
            raise RuntimeError("StreamDetector.forecast: build the detector with forecast=True")
        fidx = self._fidx(fidx, "forecast")
        t = self._tick
        self._dt(fidx)
        dt = self._fc_dt.to(t.fc.x.device, non_blocking=True)
        out = ops.forecast_extrap(t.fc, dt, self._fc_wh)
        if self._fc_out is None:
            self._fc_out = tuple(feed.pinned(tuple(o.shape), o.dtype) for o in out)
        for h, d in zip(self._fc_out, out):
            h.copy_(d, non_blocking=True)
        torch.cuda.current_stream().synchronize()
        box, score, label, track, count = (h.numpy() for h in self._fc_out)
        return [(box[i, :n].copy(), score[i, :n].copy(), label[i, :n].copy(), track[i, :n].copy())
                for i, n in enumerate(count.tolist())]

    def last_status(self):
        """Per-stream int32 status of the last ``step_jpeg``: 0 where the frame decoded, a data.JPEG_STATUS code where it
        did not, NO_FRAME (-1) where the stream got no file; None before the first ``step_jpeg``."""
        return None if self._last_status is None else self._last_status.copy()
