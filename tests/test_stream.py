"""The streaming detector (streamyolo_b200.stream): the sAP driver's per-frame loop as one CUDA graph per tick.

CPU (no GPU needed):
  * the tick the graph captures, run under the torch emulation of the kernels (tests/emul_ops.py, fp32 storage) with the
    per-stream resize, the start / keep gate, the per-image select, the NMS and the box division emulated too, reproduces
    the fp32 oracle's on_pipe forward per stream -- the star call for a stream that starts a sequence, the buffered call
    otherwise -- over a sequence with mixed resets;
  * the host's output conversion and the argument checks;
  * select_images_kernel compiles without spills.

GPU (H100):
  * sy_select_images against torch, bit for bit, on odd shapes, channel slices, bf16 and fp16, flags clear / set / mixed,
    and inside a CUDA graph whose flags change between replays;
  * StreamYOLO-s at 1200x1920 -> 600x960, one stream, bf16 and fp16 storage: every frame's raw outputs and detections are
    bit-identical to the driver's eager loop; three streams with mixed resets bit-identical to eager calls at batch 3;
    after load_state_dict + capture() the detector follows the new weights.
"""
import os
import sys

import numpy as np
import pytest
import torch

from oracle import input_oracle
from oracle.make_golden import CASES
from oracle.postprocess_oracle import postprocess_oracle
from streamyolo_b200 import data, ops, stream, synth
from streamyolo_b200.ops import View

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import emul_ops  # noqa: E402

CONF, NMS = 0.01, 0.65        # the driver's inference() defaults


def uint8_frames(n, h, w, seed):
    """seeded BGR camera-like frames: the synthetic float frames, rounded to uint8 HWC"""
    return synth.synth_frames(n, h, w, seed=seed)[:, :3].permute(0, 2, 3, 1).round().clamp(0, 255).to(torch.uint8).contiguous()


def driver_inference(result0, nc, in_scale):
    """the driver's inference() on one frame's head outputs, with the NMS oracle (pinned to torchvision.ops.batched_nms)"""
    d = postprocess_oracle(result0[None], nc, CONF, NMS)[0]
    d = np.zeros((0, 7), np.float32) if d is None else d.numpy()
    return d[:, :4] / in_scale, d[:, 4] * d[:, 5], d[:, 6].astype(np.int32)


def same_dets(a, b):
    return all(x.dtype == y.dtype and x.shape == y.shape and np.array_equal(x, y) for x, y in zip(a, b))


# ================================================================================================ CPU
TINY = CASES["tiny_120x160"]


def test_tick_follows_oracle_on_pipe_per_stream_and_divides_boxes(monkeypatch):
    """three streams over four ticks (tick 0: every stream starts; tick 2: stream 1 restarts; tick 3: streams 0 and 2): each
    stream's head outputs equal the fp32 oracle's on_pipe call on that stream alone -- star after a reset, buffered on the
    stream's previous frame otherwise -- to float roundoff, and the buffered streams really differ from a star call"""
    from test_fp16_storage import calibrated_oracle, product_from
    emul_ops.install(monkeypatch, exact=True)
    x = synth.synth_frames(TINY["B"], TINY["H"], TINY["W"])
    o = calibrated_oracle(TINY, x, synth.synth_labels(TINY["B"], TINY["H"], TINY["W"]), None)
    m = product_from(o, TINY)
    # undecoded boxes: the random-init tiny net sends some exp(w), exp(h) to 1e30 and beyond, where a relative error says
    # nothing about the routing
    o.decode_in_inference = m.head.decode_in_inference = False
    S, size, fhw = 3, (TINY["H"], TINY["W"]), (2 * TINY["H"], 2 * TINY["W"])
    table, ratios = data.sized_table([fhw] * S, size, 0.5)          # every frame of driver size: the plain resize
    assert table.tolist() == [[fhw[0], fhw[1], size[0], size[1]]] * S and ratios == [0.5] * S
    tick = stream.StreamTick(m, table, ratios, size, S, CONF, NMS, "cpu")
    resets = [(0, 1, 2), (), (1,), (0, 2)]
    bufs = [None] * S
    for t, rs in enumerate(resets):
        frames = uint8_frames(S, fhw[0], fhw[1], seed=100 + t)
        tick.frames.copy_(frames)
        tick.flags.copy_(torch.tensor([int(i in rs) for i in range(S)], dtype=torch.int32))
        tick.run()
        assert tuple(tick.raw.shape) == (S, sum(h * w for h, w in m.head.hw), 13)
        for i in range(S):
            xi = torch.from_numpy(input_oracle.stream_frame(frames[i].numpy(), size))
            with torch.no_grad():
                star, cur = o.forward(xi, mode="on_pipe")
                want, bufs[i] = (star, cur) if i in rs else o.forward(xi, buffer=bufs[i], mode="on_pipe")
            got = tick.raw[i:i + 1]
            err = float((got - want).norm() / want.norm())
            assert err < 1e-4, f"tick {t} stream {i}: rel l2 {err:.3g}"
            if i not in rs:
                assert float((star - want).norm() / want.norm()) > 100 * err, f"tick {t} stream {i}: buffer had no effect"
            d = postprocess_oracle(got, 8, CONF, NMS)[0]
            n = 0 if d is None else len(d)
            if n:
                d[:, :4] /= 0.5                                       # the boxes divided by the stream's ratio
            assert int(tick.count[i]) == n and (n == 0 or torch.equal(tick.det[i, :n], d))


def test_sized_output_conversion():
    """the boxes as the device left them (divided by the stream's ratio, see test_stream_rescale_is_numpys_division),
    obj * class_conf, the class as int32: the driver's inference() on its numpy rows, in arrays of their own (the rows
    are the pinned buffer the next tick overwrites)"""
    rows = np.array([[10.5, 20.25, 110.0, 220.75, 0.9, 0.5, 3.0], [0.0, 1.0, 2.0, 3.0, 0.25, 0.75, 7.0]], np.float32)
    b, s, lab = stream.sized_output(rows)
    assert b.dtype == np.float32 and np.array_equal(b, rows[:, :4]) and not np.shares_memory(b, rows)
    assert s.dtype == np.float32 and np.array_equal(s, np.array([0.9 * 0.5, 0.25 * 0.75], np.float32))
    assert lab.dtype == np.int32 and lab.tolist() == [3, 7]
    b, s, lab = stream.sized_output(np.zeros((0, 7), np.float32))
    assert b.shape == (0, 4) and s.shape == (0,) and lab.shape == (0,)


def test_argument_checks():
    """a train-mode model, streams < 1 and an empty input size are refused before any launch; frames of the wrong shape or
    dtype are refused by step()"""
    from test_fp16_storage import _tiny_model
    m = _tiny_model()
    with pytest.raises(ValueError, match="eval"):
        stream.StreamDetector(m.train())
    m.eval()
    for bad in (0, -1, 1.5):
        with pytest.raises(ValueError, match="streams"):
            stream.StreamDetector(m, streams=bad)
    with pytest.raises(ValueError, match="input size"):
        stream.StreamDetector(m, frame_hw=(1, 1920), in_scale=0.5)
    ok = np.zeros((12, 16, 3), np.uint8)
    assert tuple(stream.step_frames(ok, 1, (12, 16)).shape) == (1, 12, 16, 3)
    assert tuple(stream.step_frames(torch.zeros((2, 12, 16, 3), dtype=torch.uint8), 2, (12, 16)).shape) == (2, 12, 16, 3)
    for bad, s in ((ok, 2), (ok.astype(np.float32), 1), (np.zeros((12, 16, 4), np.uint8), 1), (np.zeros((16, 12, 3), np.uint8), 1),
                   (np.zeros((3, 12, 16, 3), np.uint8), 2)):
        with pytest.raises(RuntimeError, match="frames must be uint8"):
            stream.step_frames(bad, s, (12, 16))


def test_select_kernel_compiles_without_spills(tmp_path):
    """select_images_kernel: 0 spill bytes, no stack frame, no ptxas warning"""
    import re
    import shutil
    import subprocess
    from streamyolo_b200 import build
    if not os.path.exists(build.NVCC) and shutil.which("nvcc") is None:
        pytest.skip("no nvcc")
    nvcc = build.NVCC if os.path.exists(build.NVCC) else shutil.which("nvcc")
    r = subprocess.run([nvcc] + build.COMMON + build.SOURCES["bn_glue.cu"] + ["-c", os.path.join(build.CSRC, "bn_glue.cu"),
                       "-o", str(tmp_path / "g.o")], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=600)
    assert r.returncode == 0, r.stdout
    assert not [ln for ln in r.stdout.splitlines() if ln.startswith("ptxas") and "warning" in ln.lower()], r.stdout
    found = re.findall(r"Compiling entry function '(\w*select_images_kernel\w*)'[^\n]*\n[^\n]*\n\s*(\d+) bytes stack frame, "
                       r"(\d+) bytes spill stores, (\d+) bytes spill loads", r.stdout)
    assert len(found) == 1 and found[0][1:] == ("0", "0", "0"), found


# ================================================================================================ GPU
DEV = "cuda"


def _bits(t):
    return t.view(torch.int16)


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16], ids=["bf16", "fp16"])
def test_select_images_vs_torch(dtype):
    """odd shapes, channel slices of wider buffers (pitch > c), one, two and three pairs, > 2048 channels, flags clear /
    set / mixed: flagged images are copied, every other byte of the destinations keeps its poisoned bits"""
    g = torch.Generator(device=DEV).manual_seed(5)
    n = 5
    levels = [(7, 9, 24, 40, 8), (4, 5, 40, 56, 16), (2, 3, 64, 64, 0)]    # h, w, c, pitch, channel offset
    srcs, dsts = [], []
    for h, w, c, pitch, c0 in levels:
        srcs.append(View(torch.randint(-32768, 32767, (n, h, w, pitch + 8), generator=g, device=DEV, dtype=torch.int16)
                         .view(dtype)).ch(c0 + 8 if c0 else 0, c))
        dsts.append(View(torch.randint(-32768, 32767, (n, h, w, pitch), generator=g, device=DEV, dtype=torch.int16)
                         .view(dtype)).ch(c0, c))
    for flags in ([0] * n, [1] * n, [1, 0, 0, 1, 1], [0, 1, 0, 0, 0]):
        for k in (1, 2, 3):
            before = [d.buf.clone() for d in dsts]
            fl = torch.tensor(flags, dtype=torch.int32, device=DEV)
            ops.select_images(srcs[:k], dsts[:k], fl)
            torch.cuda.synchronize()
            for j, (s, d, b) in enumerate(zip(srcs, dsts, before)):
                want = b.clone()
                if j < k:
                    for i in range(n):
                        if flags[i]:
                            want[i, :, :, d.c0:d.c0 + d.c] = s.torch()[i]
                assert torch.equal(_bits(d.buf), _bits(want)), (flags, k, j)
                d.buf.copy_(b)
    big_s = View(torch.randn((2, 2, 3, 2056), generator=g, device=DEV).to(dtype))
    big_d = View(torch.randn((2, 2, 3, 2056), generator=g, device=DEV).to(dtype))
    keep = big_d.buf.clone()
    ops.select_images([big_s], [big_d], torch.tensor([0, 1], dtype=torch.int32, device=DEV))
    torch.cuda.synchronize()
    assert torch.equal(_bits(big_d.buf[0]), _bits(keep[0])) and torch.equal(_bits(big_d.buf[1]), _bits(big_s.buf[1]))
    with pytest.raises(RuntimeError):
        ops.select_images(srcs[:1], dsts[1:2], torch.ones(n, dtype=torch.int32, device=DEV))     # shape mismatch
    with pytest.raises(RuntimeError):
        ops.select_images(srcs + srcs[:1], dsts + dsts[:1], torch.ones(n, dtype=torch.int32, device=DEV))
    with pytest.raises(RuntimeError):
        ops.select_images(srcs, dsts, torch.ones(n, dtype=torch.int64, device=DEV))


@pytest.mark.gpu
def test_select_images_in_a_graph_follows_the_flags():
    """one captured launch, flags rewritten before each replay"""
    g = torch.Generator(device=DEV).manual_seed(6)
    src = View(torch.randn((4, 6, 10, 32), generator=g, device=DEV).to(torch.bfloat16))
    dst = View(torch.randn((4, 6, 10, 32), generator=g, device=DEV).to(torch.bfloat16))
    flags = torch.zeros(4, dtype=torch.int32, device=DEV)
    graph = torch.cuda.CUDAGraph()
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.graph(graph, stream=side):
        ops.select_images([src], [dst], flags)
    torch.cuda.synchronize()
    for fl in ([0, 0, 1, 0], [1, 0, 0, 1]):
        keep = dst.buf.clone()
        flags.copy_(torch.tensor(fl, dtype=torch.int32))
        graph.replay()
        torch.cuda.synchronize()
        for i in range(4):
            assert torch.equal(dst.buf[i], src.buf[i] if fl[i] else keep[i]), (fl, i)


def _model_s(dtype, seed=99):
    from test_gpu_parity_fwd import _calibrated
    m = _calibrated("s", synth.synth_frames(8, 600, 960, seed=seed).cuda())
    m.activation_dtype = dtype
    return m


FRAME_HW, IN_SCALE, SIZE = (1200, 1920), 0.5, (600, 960)


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16], ids=["bf16", "fp16"])
def test_one_stream_bit_identical_to_driver_loop(dtype):
    """8 frames, a new sequence at frames 0 and 5; numpy frames for even frames, CUDA frames for odd ones"""
    m = _model_s(dtype)
    nc = m.head.num_classes
    det = stream.StreamDetector(m, frame_hw=FRAME_HW, in_scale=IN_SCALE, streams=1, conf_thre=CONF, nms_thre=NMS)
    assert det.size == SIZE
    frames = uint8_frames(8, *FRAME_HW, seed=31)
    buffer = None
    n_dets = []
    for i in range(8):
        if i in (0, 5):
            det.reset()
            buffer = None
        with torch.no_grad():
            x = data.stream_frame(frames[i].cuda(), SIZE)
            result, buffer = m(x, buffer=buffer, mode="on_pipe")
            want = driver_inference(result[0].cpu(), nc, IN_SCALE)
        got = det.step(frames[i].numpy() if i % 2 == 0 else frames[i].cuda())
        assert len(got) == 1
        raw = det.last_raw()
        assert raw.shape == result.shape and torch.equal(raw, result), f"frame {i}: raw head outputs"
        assert same_dets(got[0], want), f"frame {i}: detections"
        n_dets.append(len(want[2]))
    assert all(n > 0 for n in n_dets), n_dets
    print(f"\n{dtype} detections per frame: {n_dets}")


@pytest.mark.gpu
def test_three_streams_mixed_resets_bit_identical_to_batch3():
    """S = 3 over four ticks (every stream starts; none; stream 1 restarts; streams 0 and 2 restart) against two eager
    calls at batch 3: model(frames, mode='on_pipe') for the current features, then model(frames, buffer=mix) with mix[i]
    the current features of a restarting stream and the previous ones otherwise"""
    m = _model_s(torch.float16)
    nc = m.head.num_classes
    S = 3
    det = stream.StreamDetector(m, frame_hw=FRAME_HW, in_scale=IN_SCALE, streams=S)
    prev = None
    for t, rs in enumerate([(0, 1, 2), (), (1,), (0, 2)]):
        for i in rs:
            det.reset(i)
        frames = uint8_frames(S, *FRAME_HW, seed=200 + t)
        with torch.no_grad():
            x = torch.cat([data.stream_frame(frames[i].cuda(), SIZE) for i in range(S)])
            _, cur = m(x, mode="on_pipe")
            cur = tuple(c.clone() for c in cur)
            mix = tuple(torch.stack([c[i] if (i in rs or prev is None) else p[i] for i in range(S)]).contiguous(
                memory_format=torch.channels_last) for c, p in zip(cur, prev or cur))
            result, _ = m(x, buffer=mix, mode="on_pipe")
        got = det.step(frames)
        raw = det.last_raw()
        assert torch.equal(raw, result), f"tick {t}: raw head outputs"
        for i in range(S):
            assert same_dets(got[i], driver_inference(result[i].cpu(), nc, IN_SCALE)), f"tick {t} stream {i}"
        prev = cur


@pytest.mark.gpu
def test_capture_after_load_state_dict_follows_new_weights():
    m = _model_s(torch.bfloat16)
    nc = m.head.num_classes
    det = stream.StreamDetector(m, frame_hw=FRAME_HW, in_scale=IN_SCALE)
    frame = uint8_frames(1, *FRAME_HW, seed=41)[0]
    old = det.step(frame.numpy())
    other = _model_s(torch.bfloat16, seed=7).state_dict()
    other = {k: (v * 0.9 if k.endswith("conv.weight") else v) for k, v in other.items()}
    m.load_state_dict(other)
    det.capture()
    got = det.step(frame.numpy())
    with torch.no_grad():
        result, _ = m(data.stream_frame(frame.cuda(), SIZE), mode="on_pipe")
    assert torch.equal(det.last_raw(), result)
    assert same_dets(got[0], driver_inference(result[0].cpu(), nc, IN_SCALE))
    assert not same_dets(got[0], old[0])
    with pytest.raises(ValueError):
        det.reset(1)
    with pytest.raises(RuntimeError, match="frames must be uint8"):
        det.step(np.zeros((600, 960, 3), np.uint8))
