"""The streaming detector: the sAP driver's per-frame loop (sAP/streamyolo/streamyolo_det.py:150-195) as ONE CUDA graph
replay per frame, for one camera stream or several batched together.

    det = StreamDetector(model, frame_hw=(1200, 1920), in_scale=0.5, streams=1)   # model in eval(), weights loaded
    det.reset()                                   # every stream starts a sequence (det.reset(i): stream i only)
    bboxes, scores, labels = det.step(frame)[0]   # what the driver's inference() returns for that frame

One tick runs, for the S streams at once: the driver's resize of the S uint8 frames (``data.stream_frame`` at batch S), the
backbone + PAFPN on the current frames, the per-stream choice of the support features (the current ones for a stream
that starts a sequence -- the star node of dfp_pafpn.py:177-228 -- the carried buffer otherwise), the DFP fusion, the
buffer update, the head and the NMS (``sy_postprocess_nms`` with room for every anchor).  Around the replay ``step``
copies the frames in and the detections out through pinned host memory and synchronises once.

The graph reads the weights and the folded BatchNorm as they were at capture: after ``load_state_dict`` (or any other
change of the weights or running statistics) call ``capture()`` again.  Nothing checks this per frame.
"""
import numpy as np
import torch

from . import ops
from .model import engine


class StreamTick:
    """The work of one tick on static buffers -- what ``StreamDetector`` captures as a CUDA graph.  ``frames`` (uint8
    [S, h, w, 3]) and ``flags`` (int32 [S], set = the stream starts a sequence) are the inputs; ``raw`` ([S, A, 5 + nc] head
    outputs), ``det`` ([S, A, 7] rows x1, y1, x2, y2, obj, class_conf, class_pred) and ``count`` ([S] rows of ``det``) are
    the outputs; ``buffer`` holds each stream's features carried to the next tick."""

    def __init__(self, model, frame_hw, size, streams, conf_thre, nms_thre, device):
        self.model, self.size = model, tuple(size)
        self.conf_thre, self.nms_thre = float(conf_thre), float(nms_thre)
        h, w = frame_hw
        self.frames = torch.zeros((streams, h, w, 3), dtype=torch.uint8, device=device)
        self.flags = torch.ones((streams,), dtype=torch.int32, device=device)
        self.x = torch.empty((streams, 3, size[0], size[1]), dtype=torch.float32, device=device)
        self.ctx = engine.Ctx(False, streams, streams, torch.device(device), dtype=model.activation_dtype)
        self.buffer = None
        self.raw = self.det = self.count = None

    def run(self):
        ctx, net, head = self.ctx, self.model.backbone, self.model.head
        s, h, w, _ = self.frames.shape
        ops.letterbox(self.frames, (h, w), self.size, self.x)
        with torch.no_grad(), engine.forward_scope(ctx.device):
            cur = engine.pafpn_frames(ctx, net, self.x, 1)
            if self.buffer is None:
                self.buffer = tuple(ctx.empty(v.n, v.h, v.w, v.c) for v in cur)
            ops.select_images(cur, self.buffer, self.flags)
            fused = engine.dfp_fuse(ctx, net, cur, self.buffer)
            for c, b in zip(cur, self.buffer):
                ops.copy(c, b)
            self.raw = head.run(ctx, fused)
            self.det, self.count = ops.postprocess_nms(self.raw, head.num_classes, self.conf_thre, self.nms_thre,
                                                       max_det=self.raw.shape[1])


def step_frames(frames, streams, frame_hw):
    """``frames`` (numpy, CPU or CUDA tensor) as a uint8 [S, h, w, 3] tensor, or RuntimeError; [h, w, 3] for one stream."""
    s, (h, w) = streams, frame_hw
    src = frames if torch.is_tensor(frames) else torch.from_numpy(np.ascontiguousarray(frames))
    ops._require(src.dtype == torch.uint8 and (tuple(src.shape) == (s, h, w, 3) or (s == 1 and tuple(src.shape) == (h, w, 3))),
                 f"StreamDetector.step: frames must be uint8 [{s}, {h}, {w}, 3]" + (f" or [{h}, {w}, 3]" if s == 1 else "")
                 + f", not {src.dtype} {list(src.shape)}")
    return src.reshape(s, h, w, 3)


def driver_output(det, in_scale):
    """The driver's inference() conversion of one frame's NMS rows (numpy fp32 [n, 7]): boxes / in_scale,
    obj * class_conf, the class as int32."""
    return det[:, :4] / in_scale, det[:, 4] * det[:, 5], det[:, 6].astype(np.int32)


class StreamDetector:
    """``model`` (YOLOX with a DFPPAFPN backbone, in eval mode, weights loaded) on ``streams`` camera streams of
    ``frame_hw`` uint8 BGR frames, at the driver's input size ``(int(h * in_scale), int(w * in_scale))``.  The activation
    storage is ``model.activation_dtype`` (``torch.float16`` for the driver's ``model.half()``).  The constructor captures
    the tick (after one warm-up run); every stream starts a sequence at the first ``step``."""

    def __init__(self, model, frame_hw=(1200, 1920), in_scale=0.5, streams=1, conf_thre=0.01, nms_thre=0.65):
        if model.training:
            raise ValueError("StreamDetector: the model must be in eval mode (model.eval())")
        if int(streams) != streams or streams < 1:
            raise ValueError(f"StreamDetector: streams must be a positive integer, not {streams}")
        h, w = (int(v) for v in frame_hw)
        size = (int(h * in_scale), int(w * in_scale))
        if min(h, w, *size) < 1:
            raise ValueError(f"StreamDetector: frame {frame_hw} at in_scale {in_scale} gives input size {size}")
        dev = next(model.parameters()).device
        ops.lib()
        self.model, self.streams, self.frame_hw, self.in_scale, self.size = model, int(streams), (h, w), in_scale, size
        self._tick = StreamTick(model, (h, w), size, self.streams, conf_thre, nms_thre, dev)
        self._stage = torch.empty((self.streams, h, w, 3), dtype=torch.uint8).pin_memory()
        self._flags = torch.ones((self.streams,), dtype=torch.int32).pin_memory()
        self._graph = None
        self.capture()

    def capture(self):
        """(Re-)capture the tick: reads the model's current weights and folded BatchNorm.  Call it after
        ``load_state_dict``.  Every stream starts a sequence at the next ``step``."""
        self._graph = None
        t = self._tick
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            t.run()                                   # packs the conv operands and folds BatchNorm outside the graph
        torch.cuda.current_stream().wait_stream(side)
        torch.cuda.synchronize()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=engine.graph_capture_stream(t.frames.device)):
            t.run()
        self._graph = g
        a = t.raw.shape[1]
        self._det = torch.empty((self.streams, a, 7), dtype=torch.float32).pin_memory()
        self._count = torch.empty((self.streams,), dtype=torch.int32).pin_memory()
        self.reset()

    def reset(self, stream=None):
        """Start a new sequence at the next ``step``: on every stream, or on stream ``stream`` only."""
        if stream is None:
            self._flags.fill_(1)
        else:
            if not 0 <= stream < self.streams:
                raise ValueError(f"StreamDetector.reset: stream {stream} not in [0, {self.streams})")
            self._flags[stream] = 1

    def step(self, frames):
        """One frame per stream -> a list of S ``(bboxes, scores, labels)`` numpy tuples, what the driver's inference()
        returns (boxes in frame pixels, float32 [n, 4]; scores float32 [n]; labels int32 [n]).  ``frames``: uint8 BGR
        [S, h, w, 3] ([h, w, 3] for one stream), a numpy array, a CPU tensor or a CUDA tensor."""
        t = self._tick
        src = step_frames(frames, self.streams, self.frame_hw)
        if src.is_cuda:
            t.frames.copy_(src)
        else:
            self._stage.copy_(src)
            t.frames.copy_(self._stage, non_blocking=True)
        t.flags.copy_(self._flags, non_blocking=True)
        self._graph.replay()
        self._det.copy_(t.det, non_blocking=True)
        self._count.copy_(t.count, non_blocking=True)
        torch.cuda.current_stream().synchronize()
        self._flags.zero_()
        det = self._det.numpy()
        return [driver_output(det[i, :n], self.in_scale) for i, n in enumerate(self._count.tolist())]

    def last_raw(self):
        """A device copy of the last tick's head outputs [S, A, 5 + nc] (what the driver keeps as ``results_raw``)."""
        return self._tick.raw.clone()
